"""Batched item-to-item recommendation (gorse_b200_vecdb_item_to_item): for many users at once, what
Recommender.recommendItemToItem does per user (logics/recommend.go:244-283) -- QueryItemToItem for every context item in
order, float64 sums per neighbour without the exclude set, the best n.  Checked against the reference's known answers, a
Python restatement of the recommender over the oracle's brute force, the per-item vecdb_query path, itself with the
tensor-core sweep turned off, and an oracle that sums in the wrong order."""
import ctypes as C

import numpy as np
import pytest

gpu = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx(gb):
    c = gb.Context(0)
    yield c
    c.close()


# ---- the oracle: recommendItemToItem + QueryItemToItem restated over the oracle's searches -----------------------------
class Dense:
    def __init__(self, X, euclid):
        self.X, self.euclid = X, euclid

    def neighbours(self, orc, c, allow, n, scale):
        """QueryItemToItem(c): top n + 1 of the allowed rows, drop c, drop Dot scores <= 0, stop at n"""
        ids = np.nonzero(allow)[0]
        oi, od = orc.bruteforce_search(np.ascontiguousarray(self.X[ids]), self.X[c], n + 1,
                                       metric=orc.METRIC_EUCLIDEAN if self.euclid else orc.METRIC_NEG_DOT)
        return orc.similar_scores(self.euclid, scale, c, n, ids[oi].astype(np.int32), -od)


class Sparse:
    def __init__(self, vecs):
        self.vecs = vecs   # list of (indices, values)

    def neighbours(self, orc, c, allow, n, scale):
        rows = sorted(set(np.nonzero(allow)[0].tolist()) | {c})
        off = np.concatenate([[0], np.cumsum([len(self.vecs[r][0]) for r in rows])]).astype(np.int64)
        ind = np.concatenate([np.asarray(self.vecs[r][0], np.uint32) for r in rows] + [np.zeros(0, np.uint32)])
        val = np.concatenate([np.asarray(self.vecs[r][1], np.float32) for r in rows] + [np.zeros(0, np.float32)])
        oi, od = orc.sparse_bruteforce_search(off, ind, val, rows.index(c), n)
        return orc.similar_scores(False, scale, -1, n, np.asarray(rows, np.int32)[oi], od)


def expected(orc, store, allow, dead, contexts, excludes, n, scale, reverse=False):
    cache, out = {}, []
    for ctx_u, ex_u in zip(contexts, excludes):
        acc, drop = {}, set(int(s) for s in ex_u)
        order = list(ctx_u)[::-1] if reverse else list(ctx_u)
        for c in order:
            c = int(c)
            if c < 0 or dead[c]:
                continue   # GetVectors finds nothing
            if c not in cache:
                cache[c] = store.neighbours(orc, c, allow, n, scale)
            for j, s in zip(*cache[c]):
                if int(j) not in drop:
                    acc[int(j)] = acc.get(int(j), 0.0) + float(s)
        best = sorted(acc.items(), key=lambda t: (-t[1], t[0]))[:n]
        out.append((np.array([b[0] for b in best], np.int64), np.array([b[1] for b in best], np.float64)))
    return out


def assert_rows_equal(got, want):
    """scores bit-identical (float64 bytes); slots identical except for the order of exact ties (and which tied slots the
    cut keeps)"""
    assert len(got) == len(want)
    for r, ((gs, gv), (ws, wv)) in enumerate(zip(got, want)):
        assert gv.tobytes() == wv.tobytes(), f"row {r}: scores differ"
        if gs.tolist() != ws.tolist():
            for v in np.unique(wv)[1:]:
                assert set(gs[gv == v].tolist()) == set(ws[wv == v].tolist()), f"row {r}"


# ---- random collections and users ---------------------------------------------------------------------------------------
def categories_of(rng, N):
    return [[int(rng.integers(0, 3))] + ([5] if i % 97 == 0 else []) for i in range(N)]


def dense_collection(gb, ctx, rng, N, d, distance):
    X = (rng.standard_normal((N, d)) * 0.5).astype(np.float32)
    X[: N // 10] *= 3
    hidden = (rng.random(N) < 0.08).astype(np.uint8)
    cats = categories_of(rng, N)
    col = gb.VectorCollection(ctx, d, distance)
    col.add(X, hidden=hidden, timestamps=rng.integers(0, 1000, N), categories=cats)
    dead = np.zeros(N, bool)
    dead[col.delete_before(30)] = True
    return col, Dense(X, distance == gb.DISTANCE_EUCLIDEAN), hidden, dead, cats


def sparse_collection(gb, ctx, rng, N):
    vecs = []
    for i in range(N):
        f = np.sort(rng.choice(300, size=int(rng.integers(1, 12)), replace=False)).astype(np.uint32)
        v = (rng.random(f.size) + 0.1).astype(np.float32)
        if i % 7 == 0:
            v[0] = -v[0]   # some dots <= 0, which QueryItemToItem drops
        vecs.append((f, v))
    hidden = (rng.random(N) < 0.08).astype(np.uint8)
    cats = categories_of(rng, N)
    col = gb.VectorCollection(ctx, 0, gb.DISTANCE_DOT)
    col.add(sparse=vecs, hidden=hidden, timestamps=rng.integers(0, 1000, N), categories=cats)
    dead = np.zeros(N, bool)
    dead[col.delete_before(30)] = True
    return col, Sparse(vecs), hidden, dead, cats


def make_users(rng, N, hidden, dead, n_users, max_ctx=12, heavy=()):
    """contexts with -1, deleted and hidden slots and repeats; exclusions with -1; some empty users; `heavy` = long contexts"""
    hid, ded = np.nonzero(hidden)[0], np.nonzero(dead)[0]
    contexts, excludes = [], []
    for u in range(n_users):
        m = int(heavy[u % len(heavy)]) if heavy and u % 3 == 0 else int(rng.integers(0, max_ctx + 1))
        c = rng.integers(0, N, m).astype(np.int64)
        if u % 8 == 0:
            c = c[:0]
        if m >= 4 and u % 4 == 1:
            c[0], c[1] = -1, int(ded[u % len(ded)])
            c[2] = int(hid[u % len(hid)])
            c[3] = c[min(5, m - 1)] if m > 5 else c[2]   # a repeated item
        contexts.append(c)
        e = rng.choice(N, size=int(rng.integers(0, 30)), replace=False).astype(np.int64)
        if u % 5 == 2 and c.size:
            e = np.unique(np.concatenate([e, c[c >= 0][:3]]))   # the user's own items, as the feedback exclude set
        if u % 3 == 0 and e.size >= 2:
            e[:2] = -1
        excludes.append(rng.permutation(e))
    return contexts, excludes


def allow_mask(hidden, dead, cats, want=()):
    a = (hidden == 0) & ~dead
    for w in want:
        a &= np.array([w in c for c in cats])
    return a


# ---- tests --------------------------------------------------------------------------------------------------------------
@gpu
def test_reference_known_answers(gb, ctx):
    # logics/recommend_test.go:72-136.  Embedding: source (0,0) without category, near (0.1,0), far (10,0), hidden (0.05,0)
    # hidden; category "movie" (id 7), CacheSize 2.
    with gb.VectorCollection(ctx, 2, gb.DISTANCE_EUCLIDEAN) as col:
        X = np.array([[0, 0], [0.1, 0], [10, 0], [0.05, 0]], np.float32)
        col.add(X, hidden=[0, 0, 0, 1], categories=[[], [7], [7], [7]])
        rows, _ = col.item_to_item([[0]], [[0]], 2, categories=[7])
        d = [np.float32(np.sqrt(np.float32(0.1) ** 2)), np.float32(10)]
        assert rows[0][0].tolist() == [1, 2]
        assert rows[0][1].tolist() == [1 / (1 - (-float(d[0]))), 1 / (1 - (-float(d[1])))]
    # tags: source {0: 1}, near {0: 2}, unrelated {1: 1}
    with gb.VectorCollection(ctx, 0, gb.DISTANCE_DOT) as col:
        col.add(sparse=[([0], [1.0]), ([0], [2.0]), ([1], [1.0])])
        rows, _ = col.item_to_item([[0]], [[0]], 2)
        assert rows[0][0].tolist() == [1] and rows[0][1].tolist() == [2.0]


@gpu
@pytest.mark.parametrize("kind,scale", [("euclid", 1.0), ("dot", 1.0), ("sparse", 1.0), ("sparse", 0.5)])
def test_matches_the_oracle(gb, orc, ctx, kind, scale):
    rng = np.random.default_rng(11 if kind == "euclid" else 12 if kind == "dot" else 13)
    N, n = 3000, 20
    if kind == "sparse":
        col, store, hidden, dead, cats = sparse_collection(gb, ctx, rng, N)
    else:
        col, store, hidden, dead, cats = dense_collection(gb, ctx, rng, N, 32, gb.DISTANCE_EUCLIDEAN if kind == "euclid" else gb.DISTANCE_DOT)
    with col:
        contexts, excludes = make_users(rng, N, hidden, dead, 96)
        rows, st = col.item_to_item(contexts, excludes, n, score_scale=scale)
        want = expected(orc, store, allow_mask(hidden, dead, cats), dead, contexts, excludes, n, scale)
        assert_rows_equal(rows, want)
        assert all(len(r[0]) <= n for r in rows) and any(len(r[0]) == n for r in rows)
        assert [len(r[0]) for r in rows][0] == 0   # empty context
        if kind == "euclid":
            # the order of the sums is observable: summed backwards, at least one score differs in its last bits.  (Dot
            # scores are fp32 values, and a few of them add up exactly in float64 in any order; 1 / (1 + dist) does not.)
            rev = expected(orc, store, allow_mask(hidden, dead, cats), dead, contexts, excludes, n, scale, reverse=True)
            assert any(g[1].tobytes() != r[1].tobytes() for g, r in zip(rows, rev))
        # a category filter, and one (category 5) that leaves fewer candidates than n
        for want_c in ([1], [5]):
            rows, _ = col.item_to_item(contexts[:48], excludes[:48], n, categories=want_c, score_scale=scale)
            assert_rows_equal(rows, expected(orc, store, allow_mask(hidden, dead, cats, want_c), dead, contexts[:48], excludes[:48], n, scale))


@gpu
@pytest.mark.parametrize("kind", ["dot", "sparse"])
def test_both_accumulators(gb, orc, ctx, kind):
    rng = np.random.default_rng(21)
    N, n = 2500, 50
    if kind == "sparse":
        col, store, hidden, dead, cats = sparse_collection(gb, ctx, rng, N)
    else:
        col, store, hidden, dead, cats = dense_collection(gb, ctx, rng, N, 16, gb.DISTANCE_DOT)
    with col:
        # |C_u| * n above the shared-memory table for every third user
        contexts, excludes = make_users(rng, N, hidden, dead, 30, heavy=(150, 300))
        rows, st = col.item_to_item(contexts, excludes, n)
        assert st["shared_users"] > 0 and st["global_users"] > 0, st
        assert st["shared_users"] + st["global_users"] == 30
        assert_rows_equal(rows, expected(orc, store, allow_mask(hidden, dead, cats), dead, contexts, excludes, n, 1.0))


@gpu
def test_sweep_and_exact_neighbour_paths(gb, orc, ctx):
    rng = np.random.default_rng(31)
    n = 30
    # >= 32768 vectors: the tensor-core sweep answers most neighbour rows
    col, store, hidden, dead, cats = dense_collection(gb, ctx, rng, 40000, 64, gb.DISTANCE_DOT)
    with col:
        contexts, excludes = make_users(rng, 40000, hidden, dead, 64, max_ctx=8)
        rows, st = col.item_to_item(contexts, excludes, n)
        assert st["context_items"] >= 64 and st["exact_rows"] < st["context_items"] // 2, st
        assert_rows_equal(rows, expected(orc, store, allow_mask(hidden, dead, cats), dead, contexts, excludes, n, 1.0))
    # a small collection: the exact kernel answers all of them
    col, store, hidden, dead, cats = dense_collection(gb, ctx, rng, 1500, 24, gb.DISTANCE_EUCLIDEAN)
    with col:
        contexts, excludes = make_users(rng, 1500, hidden, dead, 40)
        rows, st = col.item_to_item(contexts, excludes, n)
        assert st["exact_rows"] == st["context_items"] > 0, st
        assert_rows_equal(rows, expected(orc, store, allow_mask(hidden, dead, cats), dead, contexts, excludes, n, 1.0))


@gpu
@pytest.mark.parametrize("kind", ["euclid", "sparse"])
def test_repeatable_and_path_independent(gb, ctx, monkeypatch, kind):
    rng = np.random.default_rng(41)
    N, n = 40000 if kind == "euclid" else 4000, 40
    if kind == "sparse":
        col, _, hidden, dead, _ = sparse_collection(gb, ctx, rng, N)
    else:
        col, _, hidden, dead, _ = dense_collection(gb, ctx, rng, N, 32, gb.DISTANCE_EUCLIDEAN)
    with col:
        contexts, excludes = make_users(rng, N, hidden, dead, 200, heavy=(200,))
        a, sa = col.item_to_item(contexts, excludes, n)
        b, _ = col.item_to_item(contexts, excludes, n)
        monkeypatch.setenv("GORSE_B200_TOPK_EXACT", "1")
        c, sc = col.item_to_item(contexts, excludes, n)
        if kind == "euclid":
            assert sa["exact_rows"] < sa["context_items"] and sc["exact_rows"] == sc["context_items"]
        for (ga, va), (gb_, vb), (gc, vc) in zip(a, b, c):
            assert ga.tolist() == gb_.tolist() == gc.tolist()
            assert va.tobytes() == vb.tobytes() == vc.tobytes()


@gpu
@pytest.mark.parametrize("kind,scale", [("euclid", 1.0), ("sparse", 0.5)])
def test_matches_the_per_item_path(gb, orc, ctx, kind, scale):
    """vecdb_query(c, topK = n + 1) per context item + similar_scores + a host sum: what the library served before.  Dense
    vecdb_query runs the same top-k pipeline as item_to_item, so the oracle's restatement is checked too."""
    rng = np.random.default_rng(51)
    N, n = 3000, 25
    if kind == "sparse":
        col, store, hidden, dead, cats = sparse_collection(gb, ctx, rng, N)
    else:
        col, store, hidden, dead, cats = dense_collection(gb, ctx, rng, N, 32, gb.DISTANCE_EUCLIDEAN)
    metric = gb.METRIC_NEG_DOT if kind == "sparse" else gb.METRIC_EUCLIDEAN
    with col:
        contexts, excludes = make_users(rng, N, hidden, dead, 12)
        rows, _ = col.item_to_item(contexts, excludes, n, categories=[2], score_scale=scale)
        assert_rows_equal(rows, expected(orc, store, allow_mask(hidden, dead, cats, [2]), dead, contexts, excludes, n, scale))
        _, _, _, live = col.get(np.arange(N))
        for (gs, gv), ctx_u, ex_u in zip(rows, contexts, excludes):
            acc, drop = {}, set(ex_u.tolist())
            for c in ctx_u.tolist():
                if c < 0 or not live[c]:
                    continue
                q = [col.get_sparse(c)] if kind == "sparse" else col.get([c])[0]
                s, v, cnt = col.query(q, [2], n + 1)
                ids, sc = gb.similar_scores(metric, scale, c, n, s[0, :cnt[0]].astype(np.int32), -v[0, :cnt[0]])
                for j, x in zip(ids.tolist(), sc.tolist()):
                    if j not in drop:
                        acc[j] = acc.get(j, 0.0) + x
            best = sorted(acc.items(), key=lambda t: (-t[1], t[0]))[:n]
            assert_rows_equal([(gs, gv)], [(np.array([b[0] for b in best], np.int64), np.array([b[1] for b in best], np.float64))])


def raw_call(gb, h, ctx_lists, ex_lists, n=10, scale=1.0):
    from gorse_b200 import _lib

    nu = len(ctx_lists)
    co = np.concatenate([[0], np.cumsum([len(x) for x in ctx_lists])]).astype(np.int64)
    cs = np.asarray([x for l in ctx_lists for x in l], np.int64)
    eo = np.concatenate([[0], np.cumsum([len(x) for x in ex_lists])]).astype(np.int64)
    es = np.asarray([x for l in ex_lists for x in l], np.int64)
    m = max(n, 1)
    slots, scores, cnt = np.zeros(nu * m + 1, np.int64), np.zeros(nu * m + 1, np.float64), np.zeros(nu + 1, np.int32)
    return _lib.lib.gorse_b200_vecdb_item_to_item(h, nu, gb.ptr(co), gb.ptr(cs) if cs.size else None, gb.ptr(eo), gb.ptr(es) if es.size else None,
                                                  None, 0, n, scale, gb.ptr(slots), gb.ptr(scores), gb.ptr(cnt), None)


@gpu
def test_errors(gb, ctx):
    from gorse_b200 import _lib

    d = 8
    X = np.random.default_rng(0).standard_normal((100, d)).astype(np.float32)
    with gb.VectorCollection(ctx, d, gb.DISTANCE_COSINE) as col:
        col.add(X)
        assert raw_call(gb, col.h, [[1]], [[]]) == _lib.ERR_UNSUPPORTED
    with gb.VectorCollection(ctx, 0, gb.DISTANCE_DOT) as col:
        col.add(sparse=[([1, 2], [1.0, 2.0]), ([2], [1.0])])
        assert raw_call(gb, col.h, [[0]], [[]], n=129) == _lib.ERR_UNSUPPORTED
        assert raw_call(gb, col.h, [[0]], [[]], n=128) == _lib.OK
    with gb.VectorCollection(ctx, d, gb.DISTANCE_EUCLIDEAN) as col:
        col.add(X)
        assert raw_call(gb, col.h, [[1]], [[]], n=1025) == _lib.ERR_UNSUPPORTED
        assert raw_call(gb, col.h, [[1]], [[]], n=1024) == _lib.OK
        assert raw_call(gb, col.h, [[1], [2]], [[5, 5], []]) == _lib.ERR_ARG             # a slot excluded twice
        assert b"twice" in _lib.lib.gorse_b200_last_error()
        assert raw_call(gb, col.h, [[1], [2]], [[5, -1, -1], []]) == _lib.OK             # -1 may repeat
        assert raw_call(gb, col.h, [[1, 100]], [[]]) == _lib.ERR_ARG                     # not a slot
        assert raw_call(gb, col.h, [[1, -2]], [[]]) == _lib.ERR_ARG
        assert raw_call(gb, col.h, [[1]], [[]], scale=float("nan")) == _lib.ERR_ARG
        rows, _ = col.item_to_item([[1, 2], []], [[], []], 0)                             # n <= 0: nothing
        assert [len(r[0]) for r in rows] == [0, 0]
        Xn = X[:2].copy()
        Xn[1, 3] = np.nan
        col.add(Xn)
        with pytest.raises(gb.GorseB200Error) as ei:                                     # a NaN score, as in vecdb_query
            col.item_to_item([[100]], [[]], 10)
        assert ei.value.status == _lib.ERR_ARG


def test_null_collection_fails_without_a_device(gb):
    from gorse_b200 import _lib

    assert raw_call(gb, None, [[0]], [[]]) == _lib.ERR_ARG
    assert b"NULL" in _lib.lib.gorse_b200_last_error()
