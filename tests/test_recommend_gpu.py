"""Batched offline recommendation (gorse_b200_recommend) against the composed path: the library's single-stage entries
(query_excluding, item_to_item, user_to_user, fm_rank) called one after another, with the exclude sets grown, the candidates
merged, filtered and replaced and the decay applied in Python (recommend_model.chain).  Items identical, every score
identical bit for bit, for several stage orders, without a ranker, with an FM ranker and replacement, and with an embedding
slot whose softmax chunks couple the final candidates.  Also: calls of more than one chunk against smaller calls,
repeatability, argument errors, a per-user restatement over the oracle's brute force and fm_oracle that uses no
library entry, the exact-scan switch, and one test per chaining rule on the device."""
import types

import numpy as np
import pytest

import fm_oracle
import recommend_model as rm

pytestmark = pytest.mark.gpu

N_ITEMS, N_USERS, DIM = 400, 70, 16


@pytest.fixture(scope="module")
def ctx(gb):
    c = gb.Context(0)
    yield c
    c.close()


def mapped_collection(gb, ctx, rng, dim, distance, items, sparse=False):
    """a collection holding `items` in shuffled slots -> (collection, slot_of_item, item_of_slot)"""
    perm = rng.permutation(np.asarray(items))
    coll = gb.VectorCollection(ctx, 0 if sparse else dim, distance)
    if sparse:
        vecs = []
        for _ in perm:
            ind = np.sort(rng.choice(40, size=int(rng.integers(1, 6)), replace=False)).astype(np.uint32)
            vecs.append((ind, rng.random(ind.size).astype(np.float32) + 0.1))
        coll.add(sparse=vecs)
    else:
        coll.X = rng.standard_normal((perm.size, dim)).astype(np.float32) * 0.5   # slot order, for the oracle
        coll.add(values=coll.X)
    soi = np.full(N_ITEMS, -1, np.int64)
    soi[perm] = np.arange(perm.size)
    return coll, soi, perm.astype(np.int32)


@pytest.fixture(scope="module")
def world(gb, ctx):
    rng = np.random.default_rng(5)
    w = types.SimpleNamespace()
    w.live = (rng.random(N_ITEMS) > 0.12).astype(np.uint8)
    w.E0 = []
    w.ctx_items = []
    for u in range(N_USERS):
        fb = rng.choice(N_ITEMS, size=int(rng.integers(0, 14)), replace=False).tolist()
        w.ctx_items.append(fb[: max(1, len(fb) // 2)] + ([-1] if u % 4 == 0 else []) if fb else [])
        w.E0.append(fb + [-1] * int(u % 3 == 0))
    w.cf, w.cf_soi, w.cf_ios = mapped_collection(gb, ctx, rng, DIM, gb.DISTANCE_DOT, [i for i in range(N_ITEMS) if i % 5])
    w.user_vecs = rng.standard_normal((N_USERS, DIM)).astype(np.float32)
    w.i2i = {}
    w.i2i["euc"] = mapped_collection(gb, ctx, rng, DIM, gb.DISTANCE_EUCLIDEAN, [i for i in range(N_ITEMS) if i % 3])
    w.i2i["dot"] = mapped_collection(gb, ctx, rng, DIM, gb.DISTANCE_DOT, [i for i in range(N_ITEMS) if i % 7])
    w.i2i["sparse"] = mapped_collection(gb, ctx, rng, DIM, gb.DISTANCE_DOT, list(range(N_ITEMS)), sparse=True)
    w.u2u = {}
    for name, sparse in (("dense", False), ("sparse", True)):
        coll = gb.VectorCollection(ctx, 0 if sparse else DIM, gb.DISTANCE_DOT if sparse else gb.DISTANCE_EUCLIDEAN)
        if sparse:
            vecs = []
            for _ in range(N_USERS + 10):
                ind = np.sort(rng.choice(30, size=int(rng.integers(1, 5)), replace=False)).astype(np.uint32)
                vecs.append((ind, np.ones(ind.size, np.float32)))
            coll.add(sparse=vecs)
        else:
            coll.X = rng.standard_normal((N_USERS + 10, DIM)).astype(np.float32) * 0.5
            coll.add(values=coll.X)
        fb = [rng.choice(N_ITEMS, size=int(rng.integers(0, 25)), replace=True).tolist() for _ in range(N_USERS + 10)]
        slots = np.arange(N_USERS, dtype=np.int64)
        slots[::9] = -1
        w.u2u[name] = (coll, slots, fb, (rng.random(N_ITEMS) > 0.2).astype(np.uint8))
    w.pop = (rng.choice(N_ITEMS, 30, replace=False).astype(np.int32), rng.standard_normal(30))
    w.latest = (rng.choice(N_ITEMS, 20, replace=False).astype(np.int32), np.arange(20, 0, -1).astype(np.float64) * 1e9)
    w.ext = []
    for u in range(N_USERS):
        it = rng.choice(N_ITEMS, size=int(rng.integers(0, 12)), replace=True).astype(np.int32)   # duplicates survive one stage
        w.ext.append((it, np.zeros(it.size)))
    w.repl = []
    for u in range(N_USERS):
        ids = [i for i in w.E0[u] if i >= 0][:6] + rng.choice(N_ITEMS, 2, replace=False).tolist()
        ids = list(dict.fromkeys(ids))
        w.repl.append([(i, (u + i) % 2) for i in ids])
    yield w
    for c in [w.cf] + [v[0] for v in w.i2i.values()] + [v[0] for v in w.u2u.values()]:
        c.close()


N = {"i2i_euc": 12, "i2i_dot": 9, "i2i_sparse": 7, "u2u_dense": 10, "u2u_sparse": 8, "cf": 15}


def lib_stages(gb, w, names):
    out = []
    for nm in names:
        if nm == "pop":
            out.append(gb.ListStage(*w.pop))
        elif nm == "latest":
            out.append(gb.ListStage(*w.latest))
        elif nm == "ext":
            out.append(gb.ListStage(per_user=w.ext))
        elif nm == "cf":
            out.append(gb.CollaborativeStage())
        elif nm.startswith("i2i"):
            coll, soi, ios = w.i2i[nm[4:]]
            out.append(gb.ItemToItemStage(coll, N[nm], w.ctx_items, soi, ios, score_scale=0.5 if nm == "i2i_sparse" else 1.0))
        else:
            coll, slots, fb, ok = w.u2u[nm[4:]]
            out.append(gb.UserToUserStage(coll, N[nm], slots, fb, ok))
    return out


def composed_stages(w, names, users):
    """the same stages through the single-stage entries, for the users `users`"""
    out = []
    E0 = [w.E0[u] for u in users]
    for nm in names:
        if nm == "pop":
            out.append(rm.list_stage(*w.pop))
        elif nm == "latest":
            out.append(rm.list_stage(*w.latest))
        elif nm == "ext":
            out.append(rm.external_stage([w.ext[u] for u in users]))
        elif nm == "cf":
            ex = [[int(w.cf_soi[i]) if i >= 0 else -1 for i in e] for e in E0]
            rows, _ = w.cf.query_excluding(w.user_vecs[users], ex, N["cf"])
            cf_rows = [(w.cf_ios[s], sc.astype(np.float64)) for s, sc in rows]
            out.append(rm.collaborative_stage(cf_rows, w.live, N["cf"]))
        elif nm.startswith("i2i"):
            coll, soi, ios = w.i2i[nm[4:]]
            n, scale = N[nm], 0.5 if nm == "i2i_sparse" else 1.0
            ctxs = [[int(soi[i]) if i >= 0 else -1 for i in w.ctx_items[u]] for u in users]

            def run(E, coll=coll, soi=soi, ios=ios, n=n, scale=scale, ctxs=ctxs):
                rows, _ = coll.item_to_item(ctxs, [[int(soi[i]) for i in sorted(e) if soi[i] >= 0] for e in E], n, score_scale=scale)
                return [[(int(ios[s]), float(v)) for s, v in zip(*r)] for r in rows]
            out.append(run)
        else:
            coll, slots, fb, ok = w.u2u[nm[4:]]

            def run(E, coll=coll, slots=slots, fb=fb, ok=ok, n=N[nm]):
                rows, _ = coll.user_to_user(slots[users], fb, [sorted(e) for e in E], n, N_ITEMS, ok)
                return [[(int(i), float(v)) for i, v in zip(*r)] for r in rows]
            out.append(run)
    return out


def fm_model(gb, ctx, dims, bs, seed=3):
    rng = np.random.default_rng(seed)
    nf, k = 500, 8
    params = fm_oracle.random_params(rng, nf, k, dims)
    inp = fm_oracle.random_input(rng, nf, [0] * N_USERS, N_ITEMS, dims)
    fm = gb.FMRanker(ctx, nf, k, 6, bs, dims, params)
    fm.oracle = fm_oracle.Model(nf, k, 6, bs, dims, params)
    return fm, inp


def sub_input(inp, users):
    """the FM rows of `users` (the item table stays the dictionary's)"""
    s = types.SimpleNamespace(**vars(inp))
    s.n_users = len(users)
    s.user_feat = np.ascontiguousarray(inp.user_feat[users])
    rows = [(inp.user_lab_off[u], inp.user_lab_off[u + 1]) for u in users]
    s.user_lab_off = np.zeros(len(users) + 1, np.int64)
    np.cumsum([b - a for a, b in rows], out=s.user_lab_off[1:])
    s.user_lab_idx = np.ascontiguousarray(np.concatenate([inp.user_lab_idx[a:b] for a, b in rows] + [np.zeros(1, np.int32)]), np.int32)
    s.user_lab_val = np.ascontiguousarray(np.concatenate([inp.user_lab_val[a:b] for a, b in rows] + [np.zeros(1, np.float32)]), np.float32)
    return s


def fm_rank_fn(fm, inp, oracle=False):
    def rank(cands):
        s = types.SimpleNamespace(**vars(inp))
        s.cand_off = np.zeros(len(cands) + 1, np.int64)
        np.cumsum([len(c) for c in cands], out=s.cand_off[1:])
        s.cand_items = np.ascontiguousarray(np.concatenate([np.asarray(c, np.int32) for c in cands] + [np.zeros(1, np.int32)]), np.int32)
        sc = fm.oracle.rank(s)[0] if oracle else fm.rank(s)[0]
        return [sc[a:b] for a, b in zip(s.cand_off[:-1], s.cand_off[1:])]
    return rank


def check_same(got, want):
    assert len(got) == len(want)
    for u, ((gi, gs), wrow) in enumerate(zip(got, want)):
        wi = np.array([i for i, _ in wrow], np.int32)
        ws = np.array([s for _, s in wrow], np.float64)
        assert gi.tolist() == wi.tolist(), f"user {u}: items differ"
        assert gs.tobytes() == ws.tobytes(), f"user {u}: scores differ"


ORDERS = [("pop", "cf", "i2i_euc", "u2u_dense", "latest"),
          ("ext", "i2i_dot", "u2u_sparse", "cf", "pop"),
          ("i2i_sparse", "cf", "ext", "i2i_euc", "u2u_dense"),
          ("latest", "pop")]


@pytest.mark.parametrize("order", ORDERS, ids=lambda o: "-".join(o))
@pytest.mark.parametrize("ranker", ["none", "fm", "fm_slot"])
def test_equals_composed_path(gb, ctx, world, order, ranker):
    w = world
    users = list(range(N_USERS))
    cf = (w.cf, w.user_vecs, w.cf_soi, w.cf_ios, N["cf"])
    fm = inp = None
    if ranker != "none":
        fm, inp = fm_model(gb, ctx, (32,) if ranker == "fm_slot" else (), 7 if ranker == "fm_slot" else 1024)
    try:
        kw = dict(ranker=(fm, inp), replacement=w.repl, positive_decay=0.5, read_decay=0.75) if fm else {}
        got, stats = gb.recommend(ctx, w.E0, N_ITEMS, w.live, lib_stages(gb, w, order), cf=cf, **kw)
        want = rm.chain(w.E0, w.live, composed_stages(w, order, users), rank=fm_rank_fn(fm, inp) if fm else None,
                        replacement=w.repl if fm else None, positive_decay=0.5, read_decay=0.75)
        check_same(got, want)
        assert stats["candidates"] == sum(len(r) for r in want)
        assert sum(len(r) for r in want) > 0
        again, _ = gb.recommend(ctx, w.E0, N_ITEMS, w.live, lib_stages(gb, w, order), cf=cf, **kw)
        for (a, b), (c, d) in zip(got, again):
            assert a.tobytes() == c.tobytes() and b.tobytes() == d.tobytes()
    finally:
        if fm:
            fm.close()


def test_slot_chunks_follow_final_candidates(gb, ctx, world):
    """with batch_size 7 the softmax couples the rows of each chunk of the final list: ranking every candidate alone gives
    other scores, so agreeing with the composed path pins the chunking"""
    w = world
    order = ("pop", "i2i_euc")
    fm, inp = fm_model(gb, ctx, (32,), 7)
    with fm:
        got, _ = gb.recommend(ctx, w.E0, N_ITEMS, w.live, lib_stages(gb, w, order), ranker=(fm, inp))
        rank = fm_rank_fn(fm, inp)

        def rank_alone(cands):   # every candidate in a call of its own: no coupling
            return [np.array([rank([[i] if v == u else [] for v in range(N_USERS)])[u][0] for i in c], np.float32) for u, c in enumerate(cands)]
        alone = rm.chain(w.E0, w.live, composed_stages(w, order, list(range(N_USERS))), rank=rank_alone)
    assert any(g[1].tobytes() != np.array([s for _, s in a], np.float64).tobytes() for g, a in zip(got, alone) if len(a) > 1)


def test_many_chunks_match_small_calls(gb, ctx):
    """more users than one chunk (sm_count * 1024) answer as the same users sent in smaller calls"""
    rng = np.random.default_rng(11)
    nu, ni = 140000, 3000
    live = (rng.random(ni) > 0.1).astype(np.uint8)
    E0 = [rng.choice(ni, size=int(rng.integers(0, 6)), replace=False).tolist() for _ in range(nu)]
    coll = gb.VectorCollection(ctx, DIM, gb.DISTANCE_DOT)
    coll.add(values=rng.standard_normal((2000, DIM)).astype(np.float32))
    fb = [rng.choice(ni, size=4).tolist() for _ in range(2000)]
    slots = rng.integers(-1, 2000, nu)
    pop = (rng.choice(ni, 40, replace=False).astype(np.int32), rng.standard_normal(40))
    stages = [gb.ListStage(*pop), gb.UserToUserStage(coll, 10, slots, fb)]
    try:
        big, stats = gb.recommend(ctx, E0, ni, live, stages)
        assert stats["chunks"] >= 2
        cut = 70001
        small = []
        for a, b in ((0, cut), (cut, nu)):
            st = [gb.ListStage(*pop), gb.UserToUserStage(coll, 10, slots[a:b], fb)]
            small += gb.recommend(ctx, E0[a:b], ni, live, st)[0]
        for (a, b), (c, d) in zip(big, small):
            assert a.tobytes() == c.tobytes() and b.tobytes() == d.tobytes()
    finally:
        coll.close()


def test_argument_errors(gb, ctx, world):
    w = world
    st = lib_stages(gb, w, ("pop", "i2i_euc"))

    def err(**kw):
        args = dict(exclude_lists=w.E0, n_items=N_ITEMS, item_live=w.live, stages=st)
        args.update(kw)
        with pytest.raises(gb.GorseB200Error) as e:
            gb.recommend(ctx, **args)
        assert e.value.status == -1, e.value.message

    err(exclude_lists=[[N_ITEMS]] + w.E0[1:])
    err(exclude_lists=[[3, 3]] + w.E0[1:])
    err(stages=[gb.ListStage(np.array([N_ITEMS], np.int32), np.zeros(1))])
    err(stages=[gb.ListStage(np.array([1], np.int32), np.array([np.nan]))])
    err(stages=[gb.CollaborativeStage()])   # no CF inputs
    coll, soi, ios = w.i2i["euc"]
    bad = ios.copy()
    bad[0] = -1   # a live slot without an item
    err(stages=[gb.ItemToItemStage(coll, 5, w.ctx_items, soi, bad)])
    bad = soi.copy()
    bad[int(ios[0])] = int(ios.size)   # a slot past the collection
    err(stages=[gb.ItemToItemStage(coll, 5, w.ctx_items, bad, ios)])
    err(stages=[gb.ItemToItemStage(coll, 5, [[N_ITEMS]] + w.ctx_items[1:], soi, ios)])
    bad = soi.copy()
    bad[int(np.nonzero(soi < 0)[0][0])] = soi[int(ios[0])]   # two items naming one slot
    err(stages=[gb.ItemToItemStage(coll, 5, w.ctx_items, bad, ios)])
    c2, slots, fb, ok = w.u2u["dense"]
    err(stages=[gb.UserToUserStage(c2, 5, np.full(N_USERS, 10 ** 6), fb, ok)])
    fm, inp = fm_model(gb, ctx, (), 1024)
    with fm:
        err(ranker=(fm, inp), replacement=w.repl, positive_decay=float("nan"))
        err(ranker=(fm, inp), replacement=[[(N_ITEMS, 1)]] + w.repl[1:])
        bad_inp = types.SimpleNamespace(**vars(inp))
        bad_inp.item_feat = np.full(N_ITEMS, 10 ** 6, np.int32)
        err(ranker=(fm, bad_inp))


# ---- a per-user restatement of Pipeline.Recommend over the oracle's brute force and fm_oracle: no library entry involved --
def oracle_stages(orc, w, names):
    """the dense stages restated per user: QueryVectors / QueryItemToItem / QueryUserToUser on the oracle's brute force,
    the reference's float64 map sums and TopKFilter, the user-to-user item filter after the cut"""
    out = []
    for nm in names:
        if nm in ("pop", "latest"):
            out.append(rm.list_stage(*getattr(w, nm)))
        elif nm == "ext":
            out.append(rm.external_stage(w.ext))
        elif nm == "cf":
            rows = []
            for u in range(N_USERS):
                k = N["cf"] + len(w.E0[u])
                oi, od = orc.bruteforce_search(w.cf.X, w.user_vecs[u], k, metric=orc.METRIC_NEG_DOT)
                ex = {int(w.cf_soi[i]) for i in w.E0[u] if i >= 0 and w.cf_soi[i] >= 0}
                keep = [(int(w.cf_ios[s]), float(np.float32(-d))) for s, d in zip(oi, od) if int(s) not in ex]
                rows.append(([i for i, _ in keep], [s for _, s in keep]))
            out.append(rm.collaborative_stage(rows, w.live, N["cf"]))
        elif nm == "i2i_euc":
            coll, soi, ios = w.i2i["euc"]

            def run(E, coll=coll, soi=soi, ios=ios, n=N[nm]):
                res = []
                for u, e in enumerate(E):
                    acc = {}
                    for it in w.ctx_items[u]:
                        if it < 0 or soi[it] < 0:
                            continue
                        c = int(soi[it])
                        oi, od = orc.bruteforce_search(coll.X, coll.X[c], n + 1, metric=orc.METRIC_EUCLIDEAN)
                        ids, sc = orc.similar_scores(True, 1.0, c, n, oi.astype(np.int32), -od)
                        for s, v in zip(ids, sc):
                            if int(ios[s]) not in e:
                                acc[int(s)] = acc.get(int(s), 0.0) + float(v)
                    best = sorted(acc.items(), key=lambda t: (-t[1], t[0]))[:n]
                    res.append([(int(ios[s]), v) for s, v in best])
                return res
            out.append(run)
        elif nm == "u2u_dense":
            coll, slots, fb, ok = w.u2u["dense"]

            def run(E, coll=coll, slots=slots, fb=fb, ok=ok, n=N[nm]):
                res = []
                for u, e in enumerate(E):
                    c = int(slots[u])
                    if c < 0:
                        res.append([])
                        continue
                    oi, od = orc.bruteforce_search(coll.X, coll.X[c], n + 1, metric=orc.METRIC_EUCLIDEAN)
                    ids, sc = orc.similar_scores(True, 1.0, c, n, oi.astype(np.int32), -od)
                    acc = {}
                    for v, s in zip(ids, sc):
                        for it in fb[int(v)]:
                            if int(it) not in e:
                                acc[int(it)] = acc.get(int(it), 0.0) + float(s)
                    best = sorted(acc.items(), key=lambda t: (-t[1], t[0]))[:n]
                    res.append([(i, v) for i, v in best if ok[i]])
                return res
            out.append(run)
        else:
            raise ValueError(nm)
    return out


@pytest.mark.parametrize("ranker", ["none", "fm", "fm_slot"])
def test_equals_oracle_restatement(gb, ctx, orc, world, ranker):
    w = world
    order = ("pop", "cf", "i2i_euc", "ext", "u2u_dense", "latest")
    fm = inp = None
    if ranker != "none":
        fm, inp = fm_model(gb, ctx, (32,) if ranker == "fm_slot" else (), 7 if ranker == "fm_slot" else 1024)
    try:
        kw = dict(ranker=(fm, inp), replacement=w.repl, positive_decay=0.5, read_decay=0.75) if fm else {}
        got, _ = gb.recommend(ctx, w.E0, N_ITEMS, w.live, lib_stages(gb, w, order), cf=(w.cf, w.user_vecs, w.cf_soi, w.cf_ios, N["cf"]), **kw)
        want = rm.chain(w.E0, w.live, oracle_stages(orc, w, order), rank=fm_rank_fn(fm, inp, oracle=True) if fm else None,
                        replacement=w.repl if fm else None, positive_decay=0.5, read_decay=0.75)
        check_same(got, want)
    finally:
        if fm:
            fm.close()


def test_exact_scan_gives_the_same_answer(gb, ctx, monkeypatch):
    """collections large enough for the tensor-core sweep, answered again with GORSE_B200_TOPK_EXACT=1"""
    rng = np.random.default_rng(21)
    ni, nu, d = 40000, 300, 32
    E0 = [rng.choice(ni, size=int(rng.integers(0, 8)), replace=False).tolist() for _ in range(nu)]
    live = (rng.random(ni) > 0.05).astype(np.uint8)
    ident = np.arange(ni, dtype=np.int64)
    cf = gb.VectorCollection(ctx, d, gb.DISTANCE_DOT)
    cf.add(values=rng.standard_normal((ni, d)).astype(np.float32))
    i2 = gb.VectorCollection(ctx, d, gb.DISTANCE_EUCLIDEAN)
    i2.add(values=rng.standard_normal((ni, d)).astype(np.float32))
    vecs = rng.standard_normal((nu, d)).astype(np.float32)
    try:
        def run():
            st = [gb.CollaborativeStage(), gb.ItemToItemStage(i2, 50, [e[::-1] for e in E0], ident, ident.astype(np.int32))]
            return gb.recommend(ctx, E0, ni, live, st, cf=(cf, vecs, ident, ident.astype(np.int32), 50))
        fast, _ = run()
        monkeypatch.setenv("GORSE_B200_TOPK_EXACT", "1")
        exact, _ = run()
        assert sum(len(a) for a, _ in fast) > 0
        for (a, b), (c, e) in zip(fast, exact):
            assert a.tobytes() == c.tobytes() and b.tobytes() == e.tobytes()
    finally:
        cf.close()
        i2.close()


# ---- one device test per chaining rule, each showing on its data that the rule changes the answer ------------------------
def items_of(rows):
    return [r[0].tolist() for r in rows]


def test_rule_duplicate_in_a_stage_is_ranked_twice(gb, ctx):
    live = np.ones(20, np.uint8)
    ext = gb.ListStage(per_user=[(np.array([5, 5, 6], np.int32), np.zeros(3))])
    later = gb.ListStage(np.array([5, 7], np.int32), np.array([1.0, 2.0]))
    got, _ = gb.recommend(ctx, [[]], 20, live, [ext, later])
    assert items_of(got) == [[5, 5, 6, 7]]   # the duplicate survives its stage; the later list no longer returns 5


def test_rule_earlier_stage_moves_the_later_cut(gb, ctx, world):
    w = world
    i2i = lib_stages(gb, w, ("i2i_euc",))[0]
    alone, _ = gb.recommend(ctx, w.E0, N_ITEMS, np.ones(N_ITEMS, np.uint8), [i2i])
    u = max(range(N_USERS), key=lambda u: len(alone[u][0]))
    assert len(alone[u][0]) == N["i2i_euc"]
    top = alone[u][0][:1].astype(np.int32)
    after, _ = gb.recommend(ctx, w.E0, N_ITEMS, np.ones(N_ITEMS, np.uint8), [gb.ListStage(top, np.zeros(1)), i2i])
    row = after[u][0][1:].tolist()
    assert len(row) == N["i2i_euc"] and row[:-1] == alone[u][0][1:].tolist()
    assert row[-1] not in alone[u][0].tolist()   # the row took another n-th entry


def test_rule_cf_row_is_cut_before_the_filter(gb, ctx, world):
    w = world
    cf = (w.cf, w.user_vecs, w.cf_soi, w.cf_ios, N["cf"])
    live = np.ones(N_ITEMS, np.uint8)
    alone, _ = gb.recommend(ctx, w.E0, N_ITEMS, live, [gb.CollaborativeStage()], cf=cf)
    assert all(len(r[0]) == N["cf"] for r in alone)
    top = np.array([alone[0][0][0]], np.int32)
    after, _ = gb.recommend(ctx, w.E0, N_ITEMS, live, [gb.ListStage(top, np.zeros(1)), gb.CollaborativeStage()], cf=cf)
    assert after[0][0].tolist() == alone[0][0].tolist()   # the list's item, then n - 1 from the CF stage: fewer than n


def test_rule_non_live_item_is_dropped_but_excludes(gb, ctx, world):
    w = world
    i2i = lib_stages(gb, w, ("i2i_euc",))[0]
    live = np.ones(N_ITEMS, np.uint8)
    alone, _ = gb.recommend(ctx, w.E0, N_ITEMS, live, [i2i])
    u = max(range(N_USERS), key=lambda u: len(alone[u][0]))
    x = int(alone[u][0][0])
    live[x] = 0
    plain, _ = gb.recommend(ctx, w.E0, N_ITEMS, live, [i2i])
    first, _ = gb.recommend(ctx, w.E0, N_ITEMS, live, [gb.ListStage(np.array([x], np.int32), np.zeros(1)), i2i])
    assert x not in plain[u][0].tolist() and x not in first[u][0].tolist()
    assert len(plain[u][0]) == N["i2i_euc"] - 1   # dropped after the merge
    assert len(first[u][0]) == N["i2i_euc"]       # excluded by the list, so the row took another entry


def test_rule_replacement_only_when_live_and_new(gb, ctx):
    fm, inp = fm_model(gb, ctx, (), 1024)
    live = np.ones(N_ITEMS, np.uint8)
    live[4] = 0
    E0 = [[1, 2, 4]] + [[]] * (N_USERS - 1)
    stages = [gb.ListStage(np.array([3, 9], np.int32), np.zeros(2))]
    repl = [[(3, 1), (4, 1), (2, 0)]] + [[]] * (N_USERS - 1)
    with fm:
        got, _ = gb.recommend(ctx, E0, N_ITEMS, live, stages, ranker=(fm, inp), replacement=repl)
    assert sorted(got[0][0].tolist()) == [2, 3, 9]   # 3 is a candidate already, 4 is not live, 2 is appended


def test_rule_decay_after_ranking_then_resort(gb, ctx):
    fm, inp = fm_model(gb, ctx, (), 1024)
    live = np.ones(N_ITEMS, np.uint8)
    stages = [gb.ListStage(np.arange(10, 30, dtype=np.int32), np.zeros(20))]
    E0 = [[]] * N_USERS
    with fm:
        plain, _ = gb.recommend(ctx, E0, N_ITEMS, live, stages, ranker=(fm, inp))
        top = int(plain[0][0][0])
        decay = -4.0 if plain[0][1][0] > 0 else 4.0   # sends the top item to the bottom
        repl = [[(top, 1)]] + [[]] * (N_USERS - 1)
        dec, _ = gb.recommend(ctx, E0, N_ITEMS, live, stages, ranker=(fm, inp), replacement=repl, positive_decay=decay)
    s_plain = dict(zip(plain[0][0].tolist(), plain[0][1].tolist()))
    assert dict(zip(dec[0][0].tolist(), dec[0][1].tolist()))[top] == s_plain[top] * decay
    assert dec[0][0][-1] == top
    assert dec[0][0].tolist() != plain[0][0].tolist() and dec[0][0][0] != top
    assert np.all(np.diff(dec[0][1]) <= 0)   # re-sorted after the decay


def test_rule_no_ranker_merged_order_no_replacement(gb, ctx):
    live = np.ones(20, np.uint8)
    stages = [gb.ListStage(np.array([3, 1], np.int32), np.array([0.1, 0.9])), gb.ListStage(np.array([2], np.int32), np.array([5.0]))]
    got, _ = gb.recommend(ctx, [[]], 20, live, stages, replacement=[[(7, 1)]])
    assert items_of(got) == [[3, 1, 2]] and got[0][1].tolist() == [0.1, 0.9, 5.0]
