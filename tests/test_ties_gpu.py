"""Every search under exact ties: each entry's answer equals the strict spec -- the first k allowed candidates by (score
descending, slot ascending), the entry's exclusions dropped as it documents them -- ids, score bits, counts and -1 padding,
with no tie waiver.  The data makes ties common and the scores exact by construction: dense entries are odd multiples of 1/4
in [-7/4, 7/4] (exact in bf16 and fp32, never 0, so no product is -0), so every dot and squared distance at these d is an
exact fp32 value in any summation order and float64 numpy gives the kernels' bits; sparse values are 1 or a few dyadic idf
weights, so sparse dots are exact too.  Rows are planted in several copies so that tie groups straddle the cuts, including
the exact kernel's round boundary at rank 2048.  The CPU tests check those premises: the float64 scores equal the oracle's,
the data sets have ties at the cut, and the reversed rule (slot descending) gives other answers on them."""
import functools

import numpy as np
import pytest

import session_model as sm
import test_item_to_item_gpu as i2i
import test_recall_gpu as recall
import test_user_to_user_gpu as u2u

gpu = pytest.mark.gpu

GRID = np.array([-7, -5, -3, -1, 1, 3, 5, 7], np.float32) / 4
INDEX_K = (1, 100, 128, 129, 256, 257, 512, 513)   # across the sweep's class limits 128 / 256 / 512
BIG_K = (2048, 2049, 4100)                          # across the exact kernel's rounds of 2048
NQ = 64                                             # query rows: >= 64 for the sweep


@pytest.fixture(scope="module")
def ctx(gb):
    c = gb.Context(0)
    yield c
    c.close()


# ---- the spec -------------------------------------------------------------------------------------------------------------
def first_k(scores, slots, allowed, excluded, self_slot, k, reverse=False):
    """the first k allowed candidates but self_slot by (score desc, slot asc), then without the excluded slots.
    -0.0 and +0.0 are one score (numpy compares them equal).  reverse: ties by slot descending instead."""
    keep = allowed & (slots != self_slot)
    s, v = slots[keep], scores[keep]
    order = np.lexsort((-s if reverse else s, -v))[:max(k, 0)]
    s, v = s[order], v[order]
    drop = np.isin(s, np.asarray(excluded, np.int64))
    return s[~drop], v[~drop]


def tied_at(v, k):
    """the candidate at rank k (1-based) scores like the one after it: a tie group straddles the cut at k"""
    return 0 < k < len(v) and v[k - 1] == v[k]


# ---- tie-heavy data with exact scores ---------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def dense_data(seed, n_base, copies, d, nq):
    """n_base grid rows, each stored copies / 2 .. 3 copies / 2 times at scattered slots (uneven, so that the tie groups do not
    line up with the cuts); nq grid queries, every fourth a stored row"""
    rng = np.random.default_rng(seed)
    base = GRID[rng.integers(0, GRID.size, (n_base, d))]
    times = rng.integers(max(copies // 2, 1), copies * 3 // 2 + 1, n_base)
    X = np.ascontiguousarray(base[rng.permutation(np.repeat(np.arange(n_base), times))])
    Q = GRID[rng.integers(0, GRID.size, (nq, d))]
    Q[::4] = X[rng.choice(len(X), len(Q[::4]), replace=False)]
    return X, np.ascontiguousarray(Q)


def dense_scores(Q, X, euclid):
    """"higher is closer" fp32 scores: the dot, or minus float32(sqrt(float64 squared distance)).  Every partial sum is an
    exact float64 value, so any summation order gives these bits; sqrt rounded to float64 then to fp32 is the correctly
    rounded fp32 sqrt."""
    q, x = Q.astype(np.float64), X.astype(np.float64)
    dot = q @ x.T
    if not euclid:
        return dot.astype(np.float32)
    sq = (q * q).sum(1)[:, None] + (x * x).sum(1)[None, :] - 2 * dot
    return -np.sqrt(sq).astype(np.float32)


@functools.lru_cache(maxsize=None)
def sparse_data(seed, n, n_features, idf):
    """n sparse vectors of 2..8 features from a small vocabulary, value 1 (dots count shared features) or the feature's
    weight from `idf`; every fifth vector repeats an earlier one"""
    rng = np.random.default_rng(seed)
    w = np.asarray(idf, np.float32)[rng.integers(0, len(idf), n_features)] if idf else np.ones(n_features, np.float32)
    vecs = []
    for i in range(n):
        if i % 5 == 4:
            vecs.append(vecs[int(rng.integers(0, i))])
            continue
        f = np.sort(rng.choice(n_features, int(rng.integers(2, 9)), replace=False)).astype(np.uint32)
        vecs.append((f, w[f]))
    A = np.zeros((n, n_features), np.float64)
    for i, (f, v) in enumerate(vecs):
        A[i, f] = v
    return vecs, A


def sparse_scores(Aq, A):
    return (Aq @ A.T).astype(np.float32)


SWEEP = dict(seed=1, n_base=10000, copies=4, d=64, nq=NQ)      # N ~ 40 000: the tensor-core sweep
SMALL = dict(seed=2, n_base=800, copies=8, d=16, nq=16)        # N ~ 6 400: the exact kernel, k up to 4100
AGG = dict(seed=4, n_base=1250, copies=2, d=16, nq=0)          # N ~ 2 500: the aggregators' dense Dot collection
COS = dict(seed=6, n_base=1000, copies=3, d=32, nq=32)         # N ~ 3 000: Cosine
SPARSE = dict(ones=(3, 3000, 40, ()), idf=(5, 3000, 40, (1.0, 1.5, 0.75)))


def stored_queries(X, nq):
    return np.random.default_rng(8).choice(len(X), nq, replace=False).astype(np.int64)


def index_specs(X, Q, euclid, kmax, reverse=False):
    """the spec lists (slots, scores) of the index's three searches -- stored rows [0, nq), stored rows stored_queries(X, nq),
    the vectors Q -- cut at kmax"""
    slots, allow, nq = np.arange(len(X)), np.ones(len(X), bool), len(Q)
    qs = stored_queries(X, nq)
    out = {}
    for name, Qm, selfs in (("range", X[:nq], np.arange(nq)), ("indices", X[qs], qs), ("vectors", Q, [-1] * nq)):
        S = dense_scores(Qm, X, euclid)
        out[name] = [first_k(S[r], slots, allow, (), int(selfs[r]), kmax, reverse) for r in range(nq)]
    return out


# ---- premises (CPU) ------------------------------------------------------------------------------------------------------------
def test_float64_scores_are_the_oracles(orc):
    rng = np.random.default_rng(0)
    for p in (SWEEP, SMALL, COS):
        X, Q = dense_data(**p)
        rows = rng.choice(len(X), 200)
        for euclid in (False, True):
            S = dense_scores(Q[:4], X[rows], euclid)
            for i in range(4):
                for j, r in enumerate(rows):
                    want = -orc.euclidean(Q[i], X[r]) if euclid else orc.dot(Q[i], X[r])
                    assert S[i, j].tobytes() == np.float32(want).tobytes()
    for seed, n, nf, idf in SPARSE.values():
        vecs, A = sparse_data(seed, n, nf, idf)
        S = sparse_scores(A[:20], A)
        for i in range(20):
            for j in rng.choice(n, 100):
                want = orc.sparse_dot(vecs[i][0], vecs[i][1], vecs[j][0], vecs[j][1])
                assert S[i, j].tobytes() == np.float32(want).tobytes()


@pytest.mark.parametrize("euclid", [False, True])
@pytest.mark.parametrize("data,ks,share", [("sweep", INDEX_K, 0.75), ("small", BIG_K, 0.9)])
def test_dense_data_ties_at_every_cut(euclid, data, ks, share):
    """in at least `share` of the rows of every search a tie group straddles each cut k (for the small set: rank 2048, the
    exact kernel's first round), and there the reversed rule keeps other slots"""
    X, Q = dense_data(**(SWEEP if data == "sweep" else SMALL))
    kmax = max(ks) + 1
    specs, rev = index_specs(X, Q, euclid, kmax), index_specs(X, Q, euclid, kmax, reverse=True)
    for name in specs:
        for k in ks:
            tied = [r for r, (_, v) in enumerate(specs[name]) if tied_at(v, k)]
            assert len(tied) >= share * len(specs[name]), (name, k, len(tied))
            for r in tied:
                assert rev[name][r][0][:k].tolist() != specs[name][r][0][:k].tolist()


@pytest.mark.parametrize("kind", list(SPARSE))
def test_sparse_data_ties_at_the_cut(kind):
    vecs, A = sparse_data(*SPARSE[kind])
    S = sparse_scores(A[:200], A)
    slots = np.arange(len(vecs))
    for k in (1, 10, 100, 128):
        tied = 0
        for r in range(200):
            s, v = first_k(S[r], slots, S[r] > 0, (), r, k + 1)
            rs, _ = first_k(S[r], slots, S[r] > 0, (), r, k, True)
            if tied_at(v, k):
                tied += 1
                assert rs.tolist() != s[:k].tolist()
        assert tied >= 140, (k, tied)


# ---- the brute-force index -----------------------------------------------------------------------------------------------------
def check_index(got, specs, k, prune0):
    idx, dist, cnt = got
    assert len(specs) == len(cnt)
    for r, (s, v) in enumerate(specs):
        s, dd = s[:k], (-v[:k]).astype(np.float32)   # the index returns distances: -dot, or the Euclidean distance
        if prune0:
            s, dd = s[dd > 0], dd[dd > 0]
        c = len(s)
        assert cnt[r] == c, (r, k)
        assert idx[r, :c].tolist() == s.tolist(), (r, k)
        assert dist[r, :c].tobytes() == dd.tobytes(), (r, k)
        assert (idx[r, c:] == -1).all() and (dist[r, c:] == 0).all()


@pytest.fixture(scope="module", params=["negdot", "euclid"])
def sweep_index(request, gb, ctx):
    euclid = request.param == "euclid"
    X, Q = dense_data(**SWEEP)
    ix = gb.BruteforceIndex(ctx, X.shape[1], gb.METRIC_EUCLIDEAN if euclid else gb.METRIC_NEG_DOT)
    ix.add(X)
    yield ix, Q, stored_queries(X, NQ), index_specs(X, Q, euclid, max(INDEX_K))
    ix.close()


@gpu
@pytest.mark.parametrize("prune0", [False, True])
@pytest.mark.parametrize("path", ["sweep", "exact"])
def test_index(gb, sweep_index, monkeypatch, path, prune0):
    ix, Q, qs, specs = sweep_index
    if path == "exact":
        monkeypatch.setenv("GORSE_B200_TOPK_EXACT", "1")
    ix.stage1_stats()
    for k in INDEX_K:
        for name, search in (("range", lambda: ix.search_range(0, NQ, k, prune0)), ("indices", lambda: ix.search_indices(qs, k, prune0)),
                             ("vectors", lambda: ix.search_vectors(Q, k, prune0))):
            got = search()
            ms, flop, fallback = ix.stage1_stats()
            if path == "sweep" and k <= 512:
                assert ms > 0 and fallback <= NQ // 4, (name, k, fallback)   # the sweep answered most rows
            else:
                assert ms == 0
            check_index(got, specs[name], k, prune0)


@gpu
@pytest.mark.parametrize("metric", ["negdot", "euclid"])
def test_index_exact_kernel_rounds(gb, ctx, metric):
    euclid = metric == "euclid"
    X, Q = dense_data(**SMALL)
    qs, specs = stored_queries(X, len(Q)), index_specs(X, Q, euclid, max(BIG_K))
    with gb.BruteforceIndex(ctx, X.shape[1], gb.METRIC_EUCLIDEAN if euclid else gb.METRIC_NEG_DOT) as ix:
        ix.add(X)
        for k in INDEX_K + BIG_K:
            for prune0 in (False, True):
                check_index(ix.search_range(0, len(Q), k, prune0), specs["range"], k, prune0)
                check_index(ix.search_indices(qs, k, prune0), specs["indices"], k, prune0)
                check_index(ix.search_vectors(Q, k, prune0), specs["vectors"], k, prune0)


# ---- vector collections --------------------------------------------------------------------------------------------------------
def collection_meta(rng, N):
    hidden = (rng.random(N) < 0.08).astype(np.uint8)
    cats = [[int(rng.integers(0, 3))] for _ in range(N)]
    return hidden, rng.integers(0, 1000, N), cats


def allowed(hidden, dead, cats, want=()):
    a = (hidden == 0) & ~dead
    for w in want:
        a &= np.array([w in c for c in cats])
    return a


def tie_exclusions(rng, S, allow, n, N, hidden, dead):
    """per row: the two lowest slots of the tie group at rank n (the ones the cut would keep), random slots, a hidden and a
    deleted slot, and -1 entries"""
    slots, out = np.arange(N), []
    for r in range(S.shape[0]):
        s, v = first_k(S[r], slots, allow, (), -1, n)
        group = np.sort(s[v == v[-1]])[:2]
        e = np.unique(np.concatenate([group, rng.choice(N, 4), rng.choice(np.flatnonzero(hidden), 1), rng.choice(np.flatnonzero(dead), 1)]))
        out.append(rng.permutation(np.concatenate([e, [-1] * int(r % 3)]).astype(np.int64)))
    return out


def assert_same(got_rows, want_rows):
    assert len(got_rows) == len(want_rows)
    for r, ((gs, gv), (ws, wv)) in enumerate(zip(got_rows, want_rows)):
        assert np.asarray(gs).tolist() == np.asarray(ws).tolist(), f"row {r}"
        assert np.asarray(gv).tobytes() == np.asarray(wv).tobytes(), f"row {r}: scores differ"


def query_rows(slots, scores, cnt):
    k = slots.shape[1]
    for q, c in enumerate(cnt):
        assert (slots[q, c:] == -1).all() and (scores[q, c:] == 0).all()
    assert (cnt <= k).all()
    return [(slots[q, :c], scores[q, :c]) for q, c in enumerate(cnt)]


@pytest.fixture(scope="module", params=["dot", "euclid"])
def dense_collection(request, gb, ctx):
    euclid = request.param == "euclid"
    X, Q = dense_data(**SWEEP)
    rng = np.random.default_rng(9)
    hidden, ts, cats = collection_meta(rng, len(X))
    Qc = np.concatenate([Q, X[rng.choice(len(X), 32)]])   # 96 rows
    col = gb.VectorCollection(ctx, X.shape[1], gb.DISTANCE_EUCLIDEAN if euclid else gb.DISTANCE_DOT)
    col.add(X, hidden=hidden, timestamps=ts, categories=cats)
    dead = np.zeros(len(X), bool)
    dead[col.delete_before(30)] = True
    yield col, X, Qc, hidden, dead, cats, dense_scores(Qc, X, euclid)
    col.close()


@gpu
@pytest.mark.parametrize("path", ["sweep", "exact"])
def test_collection_query(dense_collection, monkeypatch, path):
    col, X, Q, hidden, dead, cats, S = dense_collection
    if path == "exact":
        monkeypatch.setenv("GORSE_B200_TOPK_EXACT", "1")
    slots = np.arange(len(X))
    for want_c in ((), (1,)):
        allow = allowed(hidden, dead, cats, want_c)
        for topk in (1, 100, 129, 300):
            got = query_rows(*col.query(Q, want_c, topk))
            assert_same(got, [first_k(S[r], slots, allow, (), -1, topk) for r in range(len(Q))])
            if topk == 100:
                assert sum(tied_at(first_k(S[r], slots, allow, (), -1, 101)[1], 100) for r in range(len(Q))) >= len(Q) // 2


@gpu
@pytest.mark.parametrize("path", ["sweep", "exact"])
def test_collection_query_excluding(dense_collection, monkeypatch, path):
    col, X, Q, hidden, dead, cats, S = dense_collection
    if path == "exact":
        monkeypatch.setenv("GORSE_B200_TOPK_EXACT", "1")
    rng = np.random.default_rng(10)
    slots, n = np.arange(len(X)), 100
    for want_c in ((), (2,)):
        allow = allowed(hidden, dead, cats, want_c)
        excl = tie_exclusions(rng, S, allow, n, len(X), hidden, dead)
        rows, exact = col.query_excluding(Q, excl, n, categories=want_c)
        assert_same(rows, [first_k(S[r], slots, allow, excl[r], -1, n + len(excl[r])) for r in range(len(Q))])
        assert exact < len(Q) // 4 if path == "sweep" else exact == len(Q)


@gpu
def test_cosine_collection_query(gb, orc, ctx):
    X, Q = dense_data(**COS)
    rng = np.random.default_rng(11)
    hidden, ts, cats = collection_meta(rng, len(X))
    with gb.VectorCollection(ctx, X.shape[1], gb.DISTANCE_COSINE) as col:
        col.add(X, hidden=hidden, timestamps=ts, categories=cats)
        dead = np.zeros(len(X), bool)
        dead[col.delete_before(30)] = True
        for want_c in ((), (0,)):
            allow = allowed(hidden, dead, cats, want_c)
            for topk in (1, 50, 300):
                got = query_rows(*col.query(Q, want_c, topk))
                want = recall.cosine_expected(orc, X, allow, Q, [()] * len(Q), topk)
                assert_same(got, want)
                if topk == 50:   # the copies tie at the cut
                    assert sum(len(w[1]) > 0 and (w[1] == w[1][-1]).sum() > 1 for w in want) >= len(Q) // 4


# ---- sparse ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("kind", list(SPARSE))
def test_sparse_index(gb, ctx, kind):
    vecs, A = sparse_data(*SPARSE[kind])
    N = len(vecs)
    S, slots = sparse_scores(A, A), np.arange(N)
    off = np.concatenate([[0], np.cumsum([len(f) for f, _ in vecs])]).astype(np.int64)
    with gb.SparseIndex(ctx) as ix:
        ix.add(off, np.concatenate([f for f, _ in vecs]), np.concatenate([v for _, v in vecs]))
        for k in (1, 10, 100, 128):
            idx, dot, cnt = ix.search_range(0, N, k)
            for r in range(N):
                s, v = first_k(S[r], slots, S[r] > 0, (), r, k)   # positive dots only
                c = len(s)
                assert cnt[r] == c and idx[r, :c].tolist() == s.tolist() and dot[r, :c].tobytes() == v.tobytes(), (r, k)
                assert (idx[r, c:] == -1).all()


@gpu
@pytest.mark.parametrize("kind", list(SPARSE))
def test_sparse_collection_query(gb, ctx, kind):
    vecs, A = sparse_data(*SPARSE[kind])
    N = len(vecs)
    rng = np.random.default_rng(12)
    hidden, ts, cats = collection_meta(rng, N)
    qrows = rng.choice(N, 200, replace=False)
    S, slots = sparse_scores(A[qrows], A), np.arange(N)
    with gb.VectorCollection(ctx, 0, gb.DISTANCE_DOT) as col:
        col.add(sparse=vecs, hidden=hidden, timestamps=ts, categories=cats)
        dead = np.zeros(N, bool)
        dead[col.delete_before(30)] = True
        for want_c in ((), (1,)):
            allow = allowed(hidden, dead, cats, want_c)
            for topk in (1, 20, 128):
                got = query_rows(*col.query([vecs[r] for r in qrows], want_c, topk))
                assert_same(got, [first_k(S[r], slots, allow & (S[r] > 0), (), -1, topk) for r in range(len(qrows))])


# ---- aggregators ------------------------------------------------------------------------------------------------------------------
class Spec:
    """QueryItemToItem / QueryUserToUser over the strict spec: the first n allowed neighbours but c, Dot scores > 0 only"""

    def __init__(self, S):
        self.S = S   # [N, N] fp32 scores

    def neighbours(self, orc, c, allow, n, scale):
        s, v = first_k(self.S[c], np.arange(self.S.shape[0]), allow, (), c, n)
        return s[v > 0].astype(np.int32), v[v > 0].astype(np.float64) * scale


def ranked(acc, n):
    """the first n sums by (sum desc, id asc), and whether more sums equal the n-th than n admits"""
    best = sorted(acc.items(), key=lambda t: (-t[1], t[0]))
    over = 0 < n < len(best) and best[n - 1][1] == best[n][1]
    best = best[:n]
    return (np.array([b[0] for b in best], np.int64), np.array([b[1] for b in best], np.float64)), over


def item_to_item_spec(store, allow, dead, contexts, excludes, n):
    out, over = [], 0
    for ctx_u, ex_u in zip(contexts, excludes):
        acc, drop = {}, set(int(x) for x in ex_u)
        for c in ctx_u.tolist():
            if c < 0 or dead[c]:
                continue
            for j, s in zip(*store.neighbours(None, c, allow, n, 1.0)):
                if int(j) not in drop:
                    acc[int(j)] = acc.get(int(j), 0.0) + float(s)
        row, o = ranked(acc, n)
        out.append(row)
        over += o
    return out, over


def user_to_user_spec(store, allow, dead, user_slots, feedback, excludes, n, item_ok):
    out, over = [], 0
    for c, ex_u in zip(user_slots.tolist(), excludes):
        acc, drop = {}, set(int(x) for x in ex_u)
        if c >= 0 and not dead[c]:
            for v, s in zip(*store.neighbours(None, c, allow, n, 1.0)):
                for it in feedback[int(v)].tolist():
                    if it not in drop:
                        acc[it] = acc.get(it, 0.0) + float(s)
        (ids, sc), o = ranked(acc, n)
        keep = np.array([item_ok is None or bool(item_ok[i]) for i in ids], bool)
        out.append((ids[keep] if ids.size else ids, sc[keep] if ids.size else sc))
        over += o
    return out, over


def agg_collection(gb, ctx, kind):
    """(collection, spec store, hidden, dead, cats): the dense Dot collection AGG or the sparse one"""
    rng = np.random.default_rng(13)
    if kind == "dense":
        X, _ = dense_data(**AGG)
        N, S = len(X), dense_scores(X, X, False)
    else:
        vecs, A = sparse_data(*SPARSE["idf"])
        N, S = len(vecs), sparse_scores(A, A)
    hidden, ts, cats = collection_meta(rng, N)
    if kind == "dense":
        col = gb.VectorCollection(ctx, X.shape[1], gb.DISTANCE_DOT)
        col.add(X, hidden=hidden, timestamps=ts, categories=cats)
    else:
        col = gb.VectorCollection(ctx, 0, gb.DISTANCE_DOT)
        col.add(sparse=vecs, hidden=hidden, timestamps=ts, categories=cats)
    dead = np.zeros(N, bool)
    dead[col.delete_before(30)] = True
    return col, Spec(S), hidden, dead, cats


@gpu
@pytest.mark.parametrize("kind", ["dense", "sparse"])
def test_item_to_item(gb, ctx, kind):
    col, store, hidden, dead, cats = agg_collection(gb, ctx, kind)
    N, n = len(hidden), 50
    rng = np.random.default_rng(14)
    with col:
        # every third user's |C_u| * n is above the shared-memory table: both accumulators run
        contexts, excludes = i2i.make_users(rng, N, hidden, dead, 60, heavy=(150, 300))
        rows, st = col.item_to_item(contexts, excludes, n)
        assert st["shared_users"] > 0 and st["global_users"] > 0, st
        want, over = item_to_item_spec(store, allowed(hidden, dead, cats), dead, contexts, excludes, n)
        assert over >= 5, over   # rows whose n-th sum ties beyond the cut: select_first_n's second select
        assert_same(rows, want)
        rows, _ = col.item_to_item(contexts, excludes, n, categories=[1])
        assert_same(rows, item_to_item_spec(store, allowed(hidden, dead, cats, (1,)), dead, contexts, excludes, n)[0])


@gpu
@pytest.mark.parametrize("kind", ["dense", "sparse"])
def test_user_to_user(gb, ctx, kind):
    col, store, hidden, dead, _ = agg_collection(gb, ctx, kind)
    N, n, n_items = len(hidden), 20, 400
    rng = np.random.default_rng(15)
    with col:
        # a third of the feedback rows are long: a user with 8 or more of them among its 20 neighbours holds more adds than
        # the shared-memory table and takes a global row
        fb = u2u.make_feedback(rng, N, n_items, heavy_share=0.3, heavy_len=800)
        slots, excludes = u2u.make_users(rng, N, hidden, dead, 90, n_items)
        allow = allowed(hidden, dead, [()] * N)
        for ok in (None, (rng.random(n_items) > 0.1).astype(np.uint8)):
            rows, st = col.user_to_user(slots, fb, excludes, n, n_items, item_ok=ok)
            assert st["shared_users"] > 0 and st["global_users"] > 0, st
            want, over = user_to_user_spec(store, allow, dead, slots, fb, excludes, n, ok)
            assert over >= 5, over
            assert_same(rows, want)


@gpu
@pytest.mark.parametrize("kind", ["dense", "sparse"])
def test_session_recommend(gb, ctx, kind):
    col, store, hidden, dead, _ = agg_collection(gb, ctx, kind)
    N, n = len(hidden), 50
    rng = np.random.default_rng(16)
    with col:
        contexts, excludes = i2i.make_users(rng, N, hidden, dead, 60, heavy=(150, 300))
        nb = sm.oracle_neighbours(None, store, hidden, dead, n, 1.0)
        ok = (rng.random(N) >= 0.08).astype(np.uint8)
        for context_size, top in ((3, 20), (400, n)):
            rows, st = col.session_recommend(contexts, excludes, n, context_size, top, item_ok=ok)
            if context_size == 400:
                assert st["shared_sessions"] > 0 and st["global_sessions"] > 0, st
            assert_same(rows, sm.session_rows(nb, contexts, excludes, context_size, top, ok))


# ---- compaction -----------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("kind", ["dense", "sparse"])
def test_compaction_keeps_tied_answers(gb, ctx, kind):
    """DESIGN §8.12: compaction renames slots in order, so every tie keeps its order and every cut keeps the same members"""
    rng = np.random.default_rng(17)
    if kind == "dense":
        X, Q = dense_data(seed=7, n_base=9000, copies=4, d=32, nq=80)   # ~36 000 slots, > 32 768 live after the deletes
        N, Sq = len(X), dense_scores(Q, X, False)
    else:
        vecs, A = sparse_data(*SPARSE["ones"])
        N = len(vecs)
        qrows = rng.choice(N, 80, replace=False)
        Q, Sq = [vecs[r] for r in qrows], sparse_scores(A[qrows], A)
    hidden, ts, cats = collection_meta(rng, N)
    ts[rng.random(N) < 0.02] = 10   # about 5 % of the slots are deleted
    with gb.VectorCollection(ctx, X.shape[1] if kind == "dense" else 0, gb.DISTANCE_DOT) as col:
        if kind == "dense":
            col.add(X, hidden=hidden, timestamps=ts, categories=cats)
        else:
            col.add(sparse=vecs, hidden=hidden, timestamps=ts, categories=cats)
        dead = np.zeros(N, bool)
        dead[col.delete_before(30)] = True
        allow, slots = allowed(hidden, dead, cats), np.arange(N)
        excl = tie_exclusions(rng, Sq, allow, 50, N, hidden, dead) if kind == "dense" else None
        contexts, ex_items = i2i.make_users(rng, N, hidden, dead, 40)

        def answers(rename):
            """query, query_excluding and item_to_item, with every slot-valued input renamed through `rename` (None: as is)"""
            def ren(a):
                a = np.asarray(a, np.int64)
                return a if rename is None else np.where(a >= 0, rename[np.maximum(a, 0)], -1)
            out = [query_rows(*col.query(Q, (), 100))]
            if kind == "dense":
                out.append(col.query_excluding(Q, [ren(e) for e in excl], 50)[0])
            out.append(col.item_to_item([ren(c) for c in contexts], [ren(e) for e in ex_items], 20)[0])
            return out

        before = answers(None)
        want = [first_k(Sq[r], slots, allow & (Sq[r] > 0 if kind == "sparse" else True), (), -1, 100) for r in range(80)]
        assert_same(before[0], want)
        if kind == "dense":
            assert_same(before[1], [first_k(Sq[r], slots, allow, excl[r], -1, 50 + len(excl[r])) for r in range(80)])
        new_slot, _, _ = col.compact()
        assert col.count()[0] == int((~dead).sum()) and (new_slot[dead] == -1).all()
        after = answers(new_slot)
        for b, a in zip(before, after):
            assert_same([(new_slot[np.asarray(s, np.int64)], v) for s, v in b], a)
