"""Batched user-to-user recommendation (gorse_b200_vecdb_user_to_user): for many users at once, what
Recommender.recommendUserToUser does per user (logics/recommend.go:285-348) -- QueryUserToUser, every similar user's positive
feedback items summed in float64 without the exclude set, the best n, then the item filter.  Checked against the reference's
known answer, a Python restatement of the recommender over the oracle's brute force, the per-user vecdb_query path, itself
with the tensor-core sweep turned off, and an oracle that sums the neighbours in the wrong order."""
import numpy as np
import pytest

gpu = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx(gb):
    c = gb.Context(0)
    yield c
    c.close()


# ---- the oracle: recommendUserToUser + QueryUserToUser restated over the oracle's searches -----------------------------
class Dense:
    def __init__(self, X, euclid):
        self.X, self.euclid = X, euclid

    def neighbours(self, orc, c, allow, n, scale):
        """QueryUserToUser(c): top n + 1 of the allowed rows, drop c, drop Dot scores <= 0, stop at n"""
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


def aggregate(nbrs, feedback, ex_u, n, item_ok, reverse=False):
    """recommendUserToUser's loop over the similar users, TopKFilter(n), then the item filter"""
    acc, drop = {}, set(int(x) for x in ex_u)
    pairs = list(zip(*nbrs))
    for v, s in pairs[::-1] if reverse else pairs:
        if int(v) < len(feedback):
            for it in feedback[int(v)]:
                if int(it) not in drop:
                    acc[int(it)] = acc.get(int(it), 0.0) + float(s)
    best = sorted(acc.items(), key=lambda t: (-t[1], t[0]))[:n]
    best = [b for b in best if item_ok is None or item_ok[b[0]]]
    return np.array([b[0] for b in best], np.int64), np.array([b[1] for b in best], np.float64)


def expected(orc, store, allow, dead, user_slots, feedback, excludes, n, scale, item_ok=None, reverse=False):
    cache, out = {}, []
    for c, ex_u in zip(user_slots, excludes):
        c = int(c)
        if c < 0 or dead[c]:
            out.append((np.zeros(0, np.int64), np.zeros(0, np.float64)))   # GetVectors finds nothing
            continue
        if c not in cache:
            cache[c] = store.neighbours(orc, c, allow, n, scale)
        out.append(aggregate(cache[c], feedback, ex_u, n, item_ok, reverse))
    return out


def assert_rows_equal(got, want):
    """scores bit-identical (float64 bytes); items identical except for the order of exact ties (and which tied items the
    cut keeps)"""
    assert len(got) == len(want)
    for r, ((gs, gv), (ws, wv)) in enumerate(zip(got, want)):
        assert gv.tobytes() == wv.tobytes(), f"row {r}: scores differ"
        if gs.tolist() != ws.tolist():
            for v in np.unique(wv)[1:]:
                assert set(gs[gv == v].tolist()) == set(ws[wv == v].tolist()), f"row {r}"


# ---- random collections, feedback and users -----------------------------------------------------------------------------
def dense_collection(gb, ctx, rng, N, d, distance):
    X = (rng.standard_normal((N, d)) * 0.5).astype(np.float32)
    X[: N // 10] *= 3
    hidden = (rng.random(N) < 0.08).astype(np.uint8)
    col = gb.VectorCollection(ctx, d, distance)
    col.add(X, hidden=hidden, timestamps=rng.integers(0, 1000, N))
    dead = np.zeros(N, bool)
    dead[col.delete_before(30)] = True
    return col, Dense(X, distance == gb.DISTANCE_EUCLIDEAN), hidden, dead


def sparse_collection(gb, ctx, rng, N):
    vecs = []
    for i in range(N):
        f = np.sort(rng.choice(300, size=int(rng.integers(1, 12)), replace=False)).astype(np.uint32)
        v = (rng.random(f.size) + 0.1).astype(np.float32)
        if i % 7 == 0:
            v[0] = -v[0]   # some dots <= 0, which QueryUserToUser drops
        vecs.append((f, v))
    hidden = (rng.random(N) < 0.08).astype(np.uint8)
    col = gb.VectorCollection(ctx, 0, gb.DISTANCE_DOT)
    col.add(sparse=vecs, hidden=hidden, timestamps=rng.integers(0, 1000, N))
    dead = np.zeros(N, bool)
    dead[col.delete_before(30)] = True
    return col, Sparse(vecs), hidden, dead


def make_feedback(rng, rows, n_items, max_len=12, heavy_share=0.0, heavy_len=0):
    """item rows per slot: some empty, some repeating an item (two positive feedback types), a few popular items"""
    fb = []
    for v in range(rows):
        m = heavy_len if rng.random() < heavy_share else int(rng.integers(0, max_len + 1))
        r = np.where(rng.random(m) < 0.3, rng.integers(0, 8, m), rng.integers(0, n_items, m)).astype(np.int32)
        if v % 9 == 0:
            r = r[:0]
        if v % 5 == 1 and r.size >= 3:
            r[2] = r[0]
        fb.append(r)
    return fb


def make_users(rng, N, hidden, dead, n_users, n_items):
    """query slots with -1, deleted, hidden and repeated users; exclusions with -1; some users with no exclusions"""
    hid, ded = np.nonzero(hidden)[0], np.nonzero(dead)[0]
    slots = rng.integers(0, N, n_users).astype(np.int64)
    for u in range(n_users):
        if u % 11 == 3:
            slots[u] = -1
        elif u % 11 == 5:
            slots[u] = int(ded[u % len(ded)])
        elif u % 11 == 7:
            slots[u] = int(hid[u % len(hid)])
        elif u % 11 == 9:
            slots[u] = slots[u - 1]
    excludes = []
    for u in range(n_users):
        e = rng.choice(n_items, size=int(rng.integers(0, 25)), replace=False).astype(np.int64)
        if u % 3 == 0 and e.size >= 2:
            e[:2] = -1
        excludes.append(rng.permutation(e))
    return slots, excludes


def allow_mask(hidden, dead):
    return (hidden == 0) & ~dead


# ---- tests --------------------------------------------------------------------------------------------------------------
@gpu
def test_reference_known_answer(gb, ctx):
    # logics/recommend_test.go:346-395.  user_1 at (0,0), user_2 at (1,0); user_2 clicked item_20 .. item_23 (indices 0 .. 3),
    # item_22 is hidden and item_23 older than the TTL; CacheSize 10.
    with gb.VectorCollection(ctx, 2, gb.DISTANCE_EUCLIDEAN) as col:
        col.add(np.array([[0, 0], [1, 0]], np.float32))
        rows, st = col.user_to_user([0], [[], [0, 1, 2, 3]], [[]], 10, 4, item_ok=[1, 1, 0, 0])
        assert rows[0][0].tolist() == [0, 1] and rows[0][1].tolist() == [0.5, 0.5]
        assert st["query_users"] == 1


@gpu
@pytest.mark.parametrize("kind,scale", [("euclid", 1.0), ("euclid", 0.5), ("dot", 1.0), ("dot", 0.5), ("sparse", 1.0), ("sparse", 0.5)])
def test_matches_the_oracle(gb, orc, ctx, kind, scale):
    rng = np.random.default_rng({"euclid": 11, "dot": 12, "sparse": 13}[kind])
    N, n, n_items = 3000, 20, 400
    if kind == "sparse":
        col, store, hidden, dead = sparse_collection(gb, ctx, rng, N)
    else:
        col, store, hidden, dead = dense_collection(gb, ctx, rng, N, 32, gb.DISTANCE_EUCLIDEAN if kind == "euclid" else gb.DISTANCE_DOT)
    with col:
        fb = make_feedback(rng, N - 37, n_items)   # the last slots have no feedback row
        slots, excludes = make_users(rng, N, hidden, dead, 96, n_items)
        ok = (rng.random(n_items) > 0.1).astype(np.uint8)
        allow = allow_mask(hidden, dead)
        rows, st = col.user_to_user(slots, fb, excludes, n, n_items, item_ok=ok, score_scale=scale)
        assert_rows_equal(rows, expected(orc, store, allow, dead, slots, fb, excludes, n, scale, ok))
        assert all(len(r[0]) <= n for r in rows) and any(len(r[0]) == n for r in rows)
        assert any(len(r[0]) == n - 1 for r in rows)   # a filtered item inside the cut
        live = [s for s in slots if s >= 0 and not dead[s]]
        assert st["query_users"] == len(set(live)) and len(set(live)) < len(live)
        assert [len(rows[u][0]) for u in range(len(slots)) if slots[u] < 0 or dead[slots[u]]] == [0] * (len(slots) - len(live))
        # no filter
        rows, _ = col.user_to_user(slots, fb, excludes, n, n_items, score_scale=scale)
        assert_rows_equal(rows, expected(orc, store, allow, dead, slots, fb, excludes, n, scale))
        if kind == "euclid":
            # the order of the sums is observable: summed over the neighbours backwards, at least one score differs
            rev = expected(orc, store, allow, dead, slots, fb, excludes, n, scale, reverse=True)
            assert any(g[1].tobytes() != r[1].tobytes() for g, r in zip(rows, rev))


@gpu
def test_cut_before_filter(gb, ctx):
    # user 0 at (0,0); user 1 at (1,0): s = 1/2; user 2 at (2,0): s = 1/3.  Sums: item 0 = 1/2 + 1/3, item 1 = 1/2,
    # items 2 and 3 = 1/3.  The first 3 are items 0, 1, 2; item 1 is filtered, and item 3, below the cut, does not move up.
    with gb.VectorCollection(ctx, 2, gb.DISTANCE_EUCLIDEAN) as col:
        col.add(np.array([[0, 0], [1, 0], [2, 0]], np.float32))
        rows, _ = col.user_to_user([0], [[], [0, 1], [0, 2, 3]], [[]], 3, 4, item_ok=[1, 0, 1, 1])
        assert rows[0][0].tolist() == [0, 2]
        assert rows[0][1].tolist() == [0.5 + 1 / 3, 1 / 3]
        rows, _ = col.user_to_user([0], [[], [0, 1], [0, 2, 3]], [[]], 3, 4)
        assert rows[0][0].tolist() == [0, 1, 2]


@gpu
def test_repeated_items_are_not_lost(gb, ctx):
    # the nearest neighbour's row holds item 5 300 times among other items; the second one's holds item 7 7000 times.
    # n = 1: 300 + 3 adds, the shared-memory table; n = 2: above it, the global row.
    with gb.VectorCollection(ctx, 2, gb.DISTANCE_EUCLIDEAN) as col:
        col.add(np.array([[0, 0], [0.3, 0], [0.7, 0.2]], np.float32))
        fb = [[], [5] * 150 + [1, 2, 3] + [5] * 150, [7] * 7000 + [5]]
        _, s1, _ = col.query(np.array([[0, 0]], np.float32), topk=3)
        s = [1 / (1 - float(x)) for x in s1[0, 1:]]   # the two neighbours' scores
        for n, path in ((1, "shared_users"), (2, "global_users")):
            rows, st = col.user_to_user([0], fb, [[2]], n, 10)
            assert st[path] == 1, st
            acc = {}
            for v in range(1, n + 1):
                for it in fb[v]:
                    if it != 2:
                        acc[it] = acc.get(it, 0.0) + s[v - 1]
            best = sorted(acc.items(), key=lambda t: (-t[1], t[0]))[:n]
            assert rows[0][0].tolist() == [b[0] for b in best]
            assert rows[0][1].tobytes() == np.array([b[1] for b in best], np.float64).tobytes()


@gpu
@pytest.mark.parametrize("kind", ["dot", "sparse"])
def test_both_accumulators(gb, orc, ctx, kind):
    rng = np.random.default_rng(21)
    N, n, n_items = 2500, 40, 3000
    if kind == "sparse":
        col, store, hidden, dead = sparse_collection(gb, ctx, rng, N)
    else:
        col, store, hidden, dead = dense_collection(gb, ctx, rng, N, 16, gb.DISTANCE_DOT)
    with col:
        # about a third of the rows are long: a user whose neighbours hold more than 6144 entries takes a global row
        fb = make_feedback(rng, N, n_items, heavy_share=0.3, heavy_len=500)
        slots, excludes = make_users(rng, N, hidden, dead, 60, n_items)
        ok = (rng.random(n_items) > 0.1).astype(np.uint8)
        rows, st = col.user_to_user(slots, fb, excludes, n, n_items, item_ok=ok)
        assert st["shared_users"] > 0 and st["global_users"] > 0, st
        assert_rows_equal(rows, expected(orc, store, allow_mask(hidden, dead), dead, slots, fb, excludes, n, 1.0, ok))


@gpu
def test_sweep_and_exact_neighbour_paths(gb, orc, ctx):
    rng = np.random.default_rng(31)
    n, n_items = 30, 1000
    # >= 32768 vectors and >= 64 query rows: the tensor-core sweep answers most neighbour rows
    col, store, hidden, dead = dense_collection(gb, ctx, rng, 40000, 64, gb.DISTANCE_DOT)
    with col:
        fb = make_feedback(rng, 40000, n_items)
        slots, excludes = make_users(rng, 40000, hidden, dead, 120, n_items)
        rows, st = col.user_to_user(slots, fb, excludes, n, n_items)
        assert st["query_users"] >= 64 and st["exact_rows"] < st["query_users"] // 2, st
        assert_rows_equal(rows, expected(orc, store, allow_mask(hidden, dead), dead, slots, fb, excludes, n, 1.0))
    # a small collection: the exact kernel answers all of them
    col, store, hidden, dead = dense_collection(gb, ctx, rng, 1500, 24, gb.DISTANCE_EUCLIDEAN)
    with col:
        fb = make_feedback(rng, 1500, n_items)
        slots, excludes = make_users(rng, 1500, hidden, dead, 40, n_items)
        rows, st = col.user_to_user(slots, fb, excludes, n, n_items)
        assert st["exact_rows"] == st["query_users"] > 0, st
        assert_rows_equal(rows, expected(orc, store, allow_mask(hidden, dead), dead, slots, fb, excludes, n, 1.0))


@gpu
@pytest.mark.parametrize("kind", ["euclid", "sparse"])
def test_repeatable_and_path_independent(gb, ctx, monkeypatch, kind):
    rng = np.random.default_rng(41)
    N, n, n_items = 40000 if kind == "euclid" else 4000, 40, 2000
    if kind == "sparse":
        col, _, hidden, dead = sparse_collection(gb, ctx, rng, N)
    else:
        col, _, hidden, dead = dense_collection(gb, ctx, rng, N, 32, gb.DISTANCE_EUCLIDEAN)
    with col:
        fb = make_feedback(rng, N, n_items, heavy_share=0.3, heavy_len=500)
        slots, excludes = make_users(rng, N, hidden, dead, 200, n_items)
        ok = (rng.random(n_items) > 0.1).astype(np.uint8)
        a, sa = col.user_to_user(slots, fb, excludes, n, n_items, item_ok=ok)
        b, _ = col.user_to_user(slots, fb, excludes, n, n_items, item_ok=ok)
        monkeypatch.setenv("GORSE_B200_TOPK_EXACT", "1")
        c, sc = col.user_to_user(slots, fb, excludes, n, n_items, item_ok=ok)
        assert sa["shared_users"] > 0 and sa["global_users"] > 0, sa
        if kind == "euclid":
            assert sa["exact_rows"] < sa["query_users"] and sc["exact_rows"] == sc["query_users"]
        for (ga, va), (gb_, vb), (gc, vc) in zip(a, b, c):
            assert ga.tolist() == gb_.tolist() == gc.tolist()
            assert va.tobytes() == vb.tobytes() == vc.tobytes()


@gpu
@pytest.mark.parametrize("kind,scale", [("euclid", 1.0), ("sparse", 0.5)])
def test_matches_the_per_user_path(gb, orc, ctx, kind, scale):
    """vecdb_query(u, topK = n + 1) per user + similar_scores + a host aggregation: what the library served before.  Dense
    vecdb_query runs the same top-k pipeline as user_to_user, so the oracle's restatement is checked too."""
    rng = np.random.default_rng(51)
    N, n, n_items = 3000, 25, 300
    if kind == "sparse":
        col, store, hidden, dead = sparse_collection(gb, ctx, rng, N)
    else:
        col, store, hidden, dead = dense_collection(gb, ctx, rng, N, 32, gb.DISTANCE_EUCLIDEAN)
    metric = gb.METRIC_NEG_DOT if kind == "sparse" else gb.METRIC_EUCLIDEAN
    with col:
        fb = make_feedback(rng, N - 5, n_items)
        slots, excludes = make_users(rng, N, hidden, dead, 24, n_items)
        ok = (rng.random(n_items) > 0.1).astype(np.uint8)
        rows, _ = col.user_to_user(slots, fb, excludes, n, n_items, item_ok=ok, score_scale=scale)
        assert_rows_equal(rows, expected(orc, store, allow_mask(hidden, dead), dead, slots, fb, excludes, n, scale, ok))
        _, _, _, live = col.get(np.arange(N))
        for (gs, gv), c, ex_u in zip(rows, slots.tolist(), excludes):
            if c < 0 or not live[c]:
                assert gs.size == 0
                continue
            q = [col.get_sparse(c)] if kind == "sparse" else col.get([c])[0]
            s, v, cnt = col.query(q, (), n + 1)
            nbrs = gb.similar_scores(metric, scale, c, n, s[0, :cnt[0]].astype(np.int32), -v[0, :cnt[0]])
            assert_rows_equal([(gs, gv)], [aggregate(nbrs, fb, ex_u, n, ok)])


def raw_call(gb, h, slots, fb_lists, ex_lists, n=10, n_items=50, scale=1.0, fb_off=None):
    from gorse_b200 import _lib

    nu = len(slots)
    sl = np.asarray(slots, np.int64)
    fo = np.concatenate([[0], np.cumsum([len(x) for x in fb_lists])]).astype(np.int64) if fb_off is None else np.asarray(fb_off, np.int64)
    fi = np.asarray([x for l in fb_lists for x in l], np.int32)
    eo = np.concatenate([[0], np.cumsum([len(x) for x in ex_lists])]).astype(np.int64)
    es = np.asarray([x for l in ex_lists for x in l], np.int64)
    m = max(n, 1)
    items, scores, cnt = np.zeros(nu * m + 1, np.int64), np.zeros(nu * m + 1, np.float64), np.zeros(nu + 1, np.int32)
    return _lib.lib.gorse_b200_vecdb_user_to_user(h, nu, gb.ptr(sl), len(fo) - 1, gb.ptr(fo), gb.ptr(fi) if fi.size else None, n_items, None,
                                                  gb.ptr(eo), gb.ptr(es) if es.size else None, n, scale, gb.ptr(items), gb.ptr(scores),
                                                  gb.ptr(cnt), None)


@gpu
def test_errors(gb, ctx):
    from gorse_b200 import _lib

    d = 8
    X = np.random.default_rng(0).standard_normal((100, d)).astype(np.float32)
    fb = [[1, 2], [3]]
    with gb.VectorCollection(ctx, d, gb.DISTANCE_COSINE) as col:
        col.add(X)
        assert raw_call(gb, col.h, [1], fb, [[]]) == _lib.ERR_UNSUPPORTED
    with gb.VectorCollection(ctx, 0, gb.DISTANCE_DOT) as col:
        col.add(sparse=[([1, 2], [1.0, 2.0]), ([2], [1.0])])
        assert raw_call(gb, col.h, [0], fb, [[]], n=129) == _lib.ERR_UNSUPPORTED
        assert raw_call(gb, col.h, [0], fb, [[]], n=128) == _lib.OK
    with gb.VectorCollection(ctx, d, gb.DISTANCE_EUCLIDEAN) as col:
        col.add(X)
        assert raw_call(gb, col.h, [1], fb, [[]], n=1025) == _lib.ERR_UNSUPPORTED
        assert raw_call(gb, col.h, [1], fb, [[]], n=1024) == _lib.OK
        assert raw_call(gb, col.h, [1, 2], fb, [[5, 5], []]) == _lib.ERR_ARG           # an item excluded twice
        assert b"twice" in _lib.lib.gorse_b200_last_error()
        assert raw_call(gb, col.h, [1, 2], fb, [[5, -1, -1], []]) == _lib.OK           # -1 may repeat
        assert raw_call(gb, col.h, [1], fb, [[50]]) == _lib.ERR_ARG                    # not an item
        assert raw_call(gb, col.h, [1], fb, [[-2]]) == _lib.ERR_ARG
        assert raw_call(gb, col.h, [100], fb, [[]]) == _lib.ERR_ARG                    # not a slot
        assert raw_call(gb, col.h, [-2], fb, [[]]) == _lib.ERR_ARG
        assert raw_call(gb, col.h, [1], [[1, 50]], [[]]) == _lib.ERR_ARG               # a feedback entry outside the items
        assert raw_call(gb, col.h, [1], [[1, -1]], [[]]) == _lib.ERR_ARG
        assert raw_call(gb, col.h, [1], [[1, 2]], [[]], fb_off=[0, 2, 1]) == _lib.ERR_ARG   # decreasing offsets
        assert raw_call(gb, col.h, [1], fb, [[]], scale=float("nan")) == _lib.ERR_ARG
        assert raw_call(gb, col.h, [1], [], [[]]) == _lib.OK                           # no feedback rows at all
        rows, _ = col.user_to_user([1, 2], fb, [[], []], 0, 50)                         # n <= 0: nothing
        assert [len(r[0]) for r in rows] == [0, 0]
        Xn = X[:2].copy()
        Xn[1, 3] = np.nan
        col.add(Xn)
        with pytest.raises(gb.GorseB200Error) as ei:                                   # a NaN score, as in vecdb_query
            col.user_to_user([100], fb, [[]], 10, 50)
        assert ei.value.status == _lib.ERR_ARG


def test_null_collection_fails_without_a_device(gb):
    from gorse_b200 import _lib

    assert raw_call(gb, None, [0], [[1]], [[]]) == _lib.ERR_ARG
    assert b"NULL" in _lib.lib.gorse_b200_last_error()
