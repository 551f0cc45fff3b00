"""Batched entries past one chunk: every entry that splits a call into chunks on the host is called with enough rows for at
least three full chunks and a partial last one, and its answers are compared with the strict spec of tests/test_ties_gpu.py
-- the first k allowed candidates by (score descending, slot ascending), exclusions dropped as the entry documents them --
on every row within 64 of a chunk boundary, on the first and last row and on a seeded sample of 1,000 more: ids, score bits,
counts and padding.  Each call is also compared, whole, with the same rows sent in calls smaller than one chunk.  The data is
tie-heavy with exact scores (grid-valued dense vectors, count-valued sparse ones), so the tie order and the cut are pinned in
the later chunks too.  The chunk sizes are restated from the code and every test asserts that its call made the chunks it
is meant to make, so the coverage cannot quietly shrink to one chunk."""
import functools

import numpy as np
import pytest

import recommend_model as rm
import session_model as sm
from test_ties_gpu import GRID, check_index, dense_scores, first_k, item_to_item_spec, sparse_data, tied_at, user_to_user_spec

gpu = pytest.mark.gpu

H100_SMS = 132   # the CPU tests size their data as the GPU tests do on an H100 SXM


# ---- the chunk sizes, restated from the code ---------------------------------------------------------------------------------
def dense_chunk(sm_count):
    """query rows of one chunk of recall::recall_rows (topk.cu: cq = sm_count * mma::GROUP_ROWS * 8, GROUP_ROWS = 128)"""
    return sm_count * 128 * 8


def user_chunk(sm_count):
    """users of one stage-B chunk: item-to-item, session and user-to-user (neighbour_call in item_to_item.cu:
    cu = sm_count * 1024) and gorse_b200_recommend (plan in recommend.cu: at most sm_count * 1024 users)"""
    return sm_count * 1024


def sparse_chunk(ntiles, k):
    """queries of one chunk of the sparse tiled search's list path, k <= 128 (sparse.cu tiled_search: TILE_LIST_BYTES /
    (ntiles * (8 k + 4)), TILE_LIST_BYTES = 512 MB, at least one query)"""
    return max(1, (512 << 20) // (ntiles * (8 * k + 4)))


SPARSE_TILE = 8192   # stored rows per tile (sparse.cu TILE)


def past_three(chunk):
    """a row count of three full chunks and a partial fourth"""
    return 3 * chunk + chunk // 3 + 7


def assert_chunks(n, chunk, at_least=3):
    assert n > at_least * chunk and n % chunk != 0, (n, chunk)


def check_rows(n, chunk, seed, extra=()):
    """the rows within 64 of every chunk boundary, the first and the last row, 1,000 seeded random rows and `extra`"""
    rows = {0, n - 1, *(int(x) for x in extra)}
    for b in range(chunk, n, chunk):
        rows.update(range(max(b - 64, 0), min(b + 64, n)))
    rows.update(np.random.default_rng(seed).choice(n, 1000, replace=False).tolist())
    return np.array(sorted(rows), np.int64)


@pytest.fixture(scope="module")
def ctx(gb):
    c = gb.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def sms():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


# ---- data and the spec ---------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def grid_rows(seed, n, n_base, d):
    """n grid rows (odd multiples of 1/4, exact scores) drawn from n_base distinct rows, so that ties are common"""
    rng = np.random.default_rng(seed)
    base = GRID[rng.integers(0, GRID.size, (n_base, d))]
    return np.ascontiguousarray(base[rng.integers(0, n_base, n)])


def hot_row(d, sign_seed):
    """a row of +-7/4: its own copies are its unique best Dot and Euclidean neighbours"""
    return (np.where(np.random.default_rng(sign_seed).random(d) < 0.5, -7, 7) / 4).astype(np.float32)


def index_data(sms, d=16):
    """the search_range index: past_three(dense_chunk) grid rows; 2,500 copies of one hot row planted in chunk 2 and of
    another in chunk 3, so that the window hands those query rows to the exact kernel after chunk 1"""
    cq = dense_chunk(sms)
    N = past_three(cq)
    X = grid_rows(1, N, N // 4, d).copy()
    rng = np.random.default_rng(2)
    for c, seed in ((1, 3), (2, 4)):
        X[cq * c + rng.choice(cq, 2500, replace=False)] = hot_row(d, seed)
    return X


def top_specs(Qm, X, euclid, ks, selfs=None, allow=None, positive=False, scores=None):
    """first_k of every row of Qm over X, cut at ks[r] (positive: Dot > 0 only).  The k-th largest allowed score of a row is
    found by a partition first and first_k runs on the candidates at or above it: the same answer as first_k over the whole
    row.  scores(a, b) -> the fp32 score block of rows [a, b) (default: dense_scores)."""
    ks = np.broadcast_to(np.asarray(ks, np.int64), (len(Qm) if scores is None else len(ks),))
    nq, N, out = len(ks), X.shape[0], []
    for a in range(0, nq, 64):
        b = min(a + 64, nq)
        S = scores(a, b) if scores is not None else dense_scores(Qm[a:b], X, euclid)
        S2 = S.astype(np.float32).copy()
        if allow is not None:
            S2[:, ~allow] = -np.inf
        if positive:
            S2[~(S > 0)] = -np.inf
        if selfs is not None:
            sl = np.asarray(selfs[a:b], np.int64)
            S2[np.nonzero(sl >= 0)[0], sl[sl >= 0]] = -np.inf
        for r in range(b - a):
            k = int(min(max(ks[a + r], 1), N))
            thr = np.partition(S2[r], N - k)[N - k]
            cand = np.flatnonzero((S2[r] >= thr) & np.isfinite(S2[r]))
            out.append(first_k(S[r][cand], cand, np.ones(cand.size, bool), (), -1, int(ks[a + r])))
    return out


class NeighbourSpec:
    """QueryItemToItem / QueryUserToUser over the strict spec for the slots the checked users need, computed in blocks:
    the first n allowed neighbours but c, Dot scores > 0 only (the interface of test_ties_gpu.Spec)"""

    def __init__(self, scores, N, allow, n, slots):
        slots = np.unique(np.asarray([s for s in slots if s >= 0], np.int64))
        rows = top_specs(None, np.zeros((N, 1)), False, np.full(slots.size, n), selfs=slots, allow=allow, positive=True,
                         scores=lambda a, b: scores(slots[a:b]))
        self.nb = {int(c): (s.astype(np.int32), v.astype(np.float64)) for c, (s, v) in zip(slots, rows)}

    def neighbours(self, orc, c, allow, n, scale):
        s, v = self.nb[int(c)]
        return s, v * scale


def dense_block(X):
    return lambda rows: dense_scores(X[rows], X, False)


def sparse_block(A):
    return lambda rows: (A[rows] @ A.T).astype(np.float32)


def sparse_csr(vecs):
    off = np.concatenate([[0], np.cumsum([len(f) for f, _ in vecs])]).astype(np.int64)
    return off, np.concatenate([f for f, _ in vecs]), np.concatenate([v for _, v in vecs])


def split_rows(flat, off):
    return np.split(flat, off[1:-1])


def same_rows(got, want, what):
    assert len(got) == len(want), what
    for r, ((gs, gv), (ws, wv)) in enumerate(zip(got, want)):
        assert np.asarray(gs).tolist() == np.asarray(ws).tolist(), (what, r)
        assert np.asarray(gv).tobytes() == np.asarray(wv).tobytes(), (what, r, "scores differ")


def in_pieces(n, size):
    return [(a, min(a + size, n)) for a in range(0, n, size)]


# ---- premises (CPU) ------------------------------------------------------------------------------------------------------------
def test_premises(orc):
    """float64 scores of the data equal the oracle's, the boundary rows of the search_range data have tie groups at the cut
    k = 100, the hot rows' copies tie at the top, and top_specs equals first_k over whole rows"""
    X = index_data(H100_SMS)
    cq, N = dense_chunk(H100_SMS), len(X)
    rng = np.random.default_rng(0)
    rows, cols = rng.choice(N, 4), rng.choice(N, 200)
    for euclid in (False, True):
        S = dense_scores(X[rows], X[cols], euclid)
        for i, r in enumerate(rows):
            for j, c in enumerate(cols):
                want = -orc.euclidean(X[r], X[c]) if euclid else orc.dot(X[r], X[c])
                assert S[i, j].tobytes() == np.float32(want).tobytes()
    vecs, A = sparse_data(5, 4000, 40, (1.0, 1.5, 0.75))
    S = (A[:10] @ A.T).astype(np.float32)
    for i in range(10):
        for j in rng.choice(len(vecs), 50):
            assert S[i, j].tobytes() == np.float32(orc.sparse_dot(*vecs[i], *vecs[j])).tobytes()
    bnd = np.array([b + o for b in range(cq, N, cq) for o in range(-64, 64, 8)])
    for euclid in (False, True):
        specs = top_specs(X[bnd], X, euclid, 101, selfs=bnd)
        assert sum(tied_at(v, 100) for _, v in specs) >= 0.9 * len(bnd), euclid
        whole = [first_k(s, np.arange(N), np.ones(N, bool), (), int(q), 101) for q, s in zip(bnd[:8], dense_scores(X[bnd[:8]], X, euclid))]
        same_rows(specs[:8], whole, "top_specs")
        hot = np.flatnonzero((X == hot_row(16, 3)).all(1))
        assert len(hot) == 2500 and (hot >= cq).all() and (hot < 2 * cq).all()
        s, v = top_specs(X[hot[:1]], X, euclid, 600, selfs=hot[:1])[0]
        assert (v == v[0]).all() and s.tolist() == [int(x) for x in hot[1:601]]


# ---- 1. the dense index ----------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module", params=["negdot", "euclid"])
def range_index(request, gb, ctx, sms):
    euclid = request.param == "euclid"
    X = index_data(sms)
    ix = gb.BruteforceIndex(ctx, X.shape[1], gb.METRIC_EUCLIDEAN if euclid else gb.METRIC_NEG_DOT)
    ix.add(X)
    rows = check_rows(len(X), dense_chunk(sms), 20)
    yield ix, X, euclid, rows, top_specs(X[rows], X, euclid, 600, selfs=rows)
    ix.close()


@gpu
@pytest.mark.parametrize("k", [100, 600])
def test_index_search_range(range_index, sms, k):
    ix, X, euclid, rows, specs = range_index
    N, cq = len(X), dense_chunk(sms)
    assert_chunks(N, cq)
    for prune0 in (False, True):
        ix.stage1_stats()
        idx, dist, cnt = ix.search_range(0, N, k, prune0)
        ms, _, fallback = ix.stage1_stats()
        if k == 100:   # the sweep answered the rows, and the window handed the hot copies of chunks 2 and 3 to the exact kernel
            assert ms > 0 and fallback >= 4000, fallback
        check_index((idx[rows], dist[rows], cnt[rows]), specs, k, prune0)
        assert not (idx == np.arange(N)[:, None]).any()   # no row returns its own slot, in any chunk
        if not prune0:
            assert (cnt == k).all()
            whole = idx, dist, cnt
    for a, b in in_pieces(N, cq // 2):   # the same rows in calls of half a chunk
        i2, d2, c2 = ix.search_range(a, b, k)
        assert i2.tobytes() == whole[0][a:b].tobytes() and d2.tobytes() == whole[1][a:b].tobytes() and c2.tobytes() == whole[2][a:b].tobytes()


@gpu
def test_index_query_similar(gb, range_index, sms):
    ix, X, euclid, rows, specs = range_index
    N, n = len(X), 100
    ids, sc, cnt = ix.query_similar(0, N, n)
    for r, (s, v) in zip(rows, specs):
        wi, ws = gb.similar_scores(gb.METRIC_EUCLIDEAN if euclid else gb.METRIC_NEG_DOT, 1.0, -1, n, s[:n], (-v[:n]).astype(np.float32))
        c = len(wi)
        assert cnt[r] == c and ids[r, :c].tolist() == wi.tolist() and sc[r, :c].tobytes() == ws.tobytes(), r
        assert (ids[r, c:] == -1).all() and (sc[r, c:] == 0).all()
    for a, b in ((0, 1000), (dense_chunk(sms) - 500, dense_chunk(sms) + 500), (N - 777, N)):
        i2, s2, c2 = ix.query_similar(a, b, n)
        assert i2.tobytes() == ids[a:b].tobytes() and s2.tobytes() == sc[a:b].tobytes() and c2.tobytes() == cnt[a:b].tobytes()


@pytest.fixture(scope="module", params=["negdot", "euclid"])
def query_index(request, gb, ctx, sms):
    """N = 40,000 grid rows of d = 32; past_three(dense_chunk) query rows: stored slots for search_indices, and for
    search_vectors the same rows with every third one a fresh grid row"""
    euclid = request.param == "euclid"
    X = grid_rows(5, 40000, 12000, 32)
    nq = past_three(dense_chunk(sms))
    rng = np.random.default_rng(6)
    qs = rng.integers(0, len(X), nq).astype(np.int64)
    Q = X[qs].copy()
    Q[::3] = GRID[rng.integers(0, GRID.size, (len(Q[::3]), X.shape[1]))]
    rows = check_rows(nq, dense_chunk(sms), 21)
    specs = {"indices": top_specs(X[qs[rows]], X, euclid, 600, selfs=qs[rows]), "vectors": top_specs(Q[rows], X, euclid, 600)}
    ix = gb.BruteforceIndex(ctx, X.shape[1], gb.METRIC_EUCLIDEAN if euclid else gb.METRIC_NEG_DOT)
    ix.add(X)
    yield ix, qs, Q, rows, specs
    ix.close()


@gpu
@pytest.mark.parametrize("k", [100, 600])
@pytest.mark.parametrize("entry", ["indices", "vectors"])
def test_index_search_queries(query_index, sms, entry, k):
    ix, qs, Q, rows, specs = query_index
    nq, cq = len(qs), dense_chunk(sms)
    assert_chunks(nq, cq)
    search = (lambda a, b, p: ix.search_indices(qs[a:b], k, p)) if entry == "indices" else (lambda a, b, p: ix.search_vectors(Q[a:b], k, p))
    for prune0 in (False, True):
        idx, dist, cnt = search(0, nq, prune0)
        check_index((idx[rows], dist[rows], cnt[rows]), specs[entry], k, prune0)
        if entry == "indices":
            assert not (idx == qs[:, None]).any()   # no row returns its own slot, in any chunk
        if not prune0:
            whole = idx, dist, cnt
    for a, b in in_pieces(nq, cq // 2):
        i2, d2, c2 = search(a, b, False)
        assert i2.tobytes() == whole[0][a:b].tobytes() and d2.tobytes() == whole[1][a:b].tobytes() and c2.tobytes() == whole[2][a:b].tobytes()


# ---- 2. the collection's query_excluding ---------------------------------------------------------------------------------------------
def exclusion_sizes(nq, cq, n):
    """|E_q| per row so that k_q = n + |E_q| falls in every class -- 128, 256, 512 and the exact kernel -- in every chunk but
    the second, which has no exact-class row; every seventh row has none"""
    r = np.arange(nq)
    size = np.select([r % 7 == 0, r % 4 == 1, r % 4 == 2, r % 4 == 3], [0, 60, 300, 700], 5 + r % 23)
    size[(size == 700) & ((r % 40 != 3) | (r // cq == 1))] = 20   # exact-class rows are one in 40: their lists are long
    return size.astype(np.int64)


@pytest.fixture(scope="module", params=["dot", "euclid"])
def excluding_collection(request, gb, ctx, sms):
    euclid = request.param == "euclid"
    X = grid_rows(7, 40000, 12000, 32)
    N, n, cq = len(X), 100, dense_chunk(sms)
    nq = past_three(cq)
    rng = np.random.default_rng(8)
    hidden = (rng.random(N) < 0.08).astype(np.uint8)
    ts = rng.integers(0, 1000, N)
    Q = X[rng.integers(0, N, nq)].copy()
    Q[::2] = GRID[rng.integers(0, GRID.size, (len(Q[::2]), X.shape[1]))]
    col = gb.VectorCollection(ctx, X.shape[1], gb.DISTANCE_EUCLIDEAN if euclid else gb.DISTANCE_DOT)
    col.add(X, hidden=hidden, timestamps=ts)
    dead = np.zeros(N, bool)
    dead[col.delete_before(30)] = True
    allow = (hidden == 0) & ~dead
    size = exclusion_sizes(nq, cq, n)
    off = np.concatenate([[0], np.cumsum(size)])
    start = rng.integers(0, N, nq)
    flat = (np.repeat(start, size) + (np.arange(off[-1]) - np.repeat(off[:-1], size)) * 7919) % N   # distinct slots per row
    excl = split_rows(flat.astype(np.int64), off)
    rows = check_rows(nq, cq, 22)
    # the checked rows exclude the two lowest slots of the tie group at rank n and one hidden and one deleted slot
    first = top_specs(Q[rows], X, euclid, n, allow=allow)
    for r, (s, v) in zip(rows, first):
        group = np.sort(s[v == v[-1]])[:2]
        extra = np.concatenate([group, rng.choice(np.flatnonzero(hidden), 1), rng.choice(np.flatnonzero(dead), 1)])
        if size[r]:
            excl[r] = np.unique(np.concatenate([excl[r], extra]))
    specs = top_specs(Q[rows], X, euclid, [n + len(excl[r]) for r in rows], allow=allow)
    specs = [(s[~np.isin(s, excl[r])], v[~np.isin(s, excl[r])]) for r, (s, v) in zip(rows, specs)]
    yield col, Q, excl, rows, specs, n
    col.close()


@gpu
def test_collection_query_excluding(excluding_collection, sms):
    col, Q, excl, rows, specs, n = excluding_collection
    nq, cq = len(Q), dense_chunk(sms)
    assert_chunks(nq, cq)
    k = n + np.array([len(e) for e in excl])
    for c in range(-(-nq // cq)):   # every class holds rows in every chunk, but the exact class in chunk 2
        kc = k[c * cq:(c + 1) * cq]
        for lo, hi in ((1, 128), (129, 256), (257, 512), (513, 1 << 30)):
            assert ((kc >= lo) & (kc <= hi)).any() == (c != 1 or hi < 513), (c, lo)
    got, exact = col.query_excluding(Q, excl, n)
    assert exact >= (k > 512).sum()
    same_rows([got[r] for r in rows], specs, "spec")
    pieces = []
    for a, b in in_pieces(nq, cq // 2):
        pieces += col.query_excluding(Q[a:b], excl[a:b], n)[0]
    same_rows(pieces, got, "pieces")


# ---- 3. item-to-item and session ------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def aggregator_data(kind, N):
    """(fp32 score block callable, dense rows or sparse vectors) of an aggregators' Dot collection of N slots"""
    if kind == "dense":
        X = grid_rows(9, N, N // 3, 16)
        return dense_block(X), X
    vecs, A = sparse_data(10, N, 60, (1.0, 1.5, 0.75))
    return sparse_block(A), vecs


def make_collection(gb, ctx, kind, N, seed):
    block, data = aggregator_data(kind, N)
    rng = np.random.default_rng(seed)
    hidden = (rng.random(N) < 0.08).astype(np.uint8)
    ts = rng.integers(0, 1000, N)
    if kind == "dense":
        col = gb.VectorCollection(ctx, data.shape[1], gb.DISTANCE_DOT)
        col.add(data, hidden=hidden, timestamps=ts)
    else:
        col = gb.VectorCollection(ctx, 0, gb.DISTANCE_DOT)
        col.add(sparse=data, hidden=hidden, timestamps=ts)
    dead = np.zeros(N, bool)
    dead[col.delete_before(30)] = True
    return col, block, hidden, dead


def i2i_users(rng, N, nu, cu, heavy_every, hot):
    """context and exclusion lists of nu users: 0 to 6 context slots (some -1), every heavy_every-th user from the second
    chunk on a heavy one with 400 slots of the pool `hot` (live slots, so that 400 n adds exceed the shared table), so the first chunk has no global-row user"""
    m = rng.integers(0, 7, nu)
    u = np.arange(nu)
    heavy = (u >= cu) & (u % heavy_every == 5)
    m[heavy] = 400
    off = np.concatenate([[0], np.cumsum(m)])
    flat = rng.integers(0, N, off[-1]).astype(np.int64)
    flat[rng.random(off[-1]) < 0.03] = -1
    ctxs = split_rows(flat, off)
    for h in np.flatnonzero(heavy):
        ctxs[h] = rng.choice(hot, 400).astype(np.int64)
    ex_m = rng.integers(0, 5, nu)
    eoff = np.concatenate([[0], np.cumsum(ex_m)])
    ex = split_rows(((np.repeat(rng.integers(0, N, nu), ex_m) + (np.arange(eoff[-1]) - np.repeat(eoff[:-1], ex_m)) * 101) % N).astype(np.int64), eoff)
    return ctxs, ex, np.flatnonzero(heavy)


@pytest.fixture(scope="module", params=["dense", "sparse"])
def i2i_world(request, gb, ctx, sms):
    kind = request.param
    cq, cu = dense_chunk(sms), user_chunk(sms)
    N = cq + 30000 if kind == "dense" else 60000   # dense: more distinct context rows than one chunk of the neighbour table
    col, block, hidden, dead = make_collection(gb, ctx, kind, N, 11)
    rng = np.random.default_rng(12)
    nu = past_three(cu)
    hot = rng.choice(np.flatnonzero(~dead), 1000, replace=False)
    ctxs, ex, heavy = i2i_users(rng, N, nu, cu, 997, hot)
    rows = check_rows(nu, cu, 23, extra=heavy[::40])
    allow = (hidden == 0) & ~dead
    need = [c for r in rows for c in ctxs[r].tolist()]
    store = NeighbourSpec(block, N, allow, 20, need)
    yield col, store, hidden, dead, allow, ctxs, ex, rows, heavy
    col.close()


@gpu
def test_item_to_item(i2i_world, sms):
    col, store, hidden, dead, allow, ctxs, ex, rows, heavy = i2i_world
    nu, cu, n = len(ctxs), user_chunk(sms), 20
    assert_chunks(nu, cu)
    assert heavy.min() >= cu and (heavy // cu == 1).any()   # no heavy user in chunk 1, heavy users in the chunks after it
    got, st = col.item_to_item(ctxs, ex, n)
    assert st["shared_users"] + st["global_users"] == nu and st["global_users"] == len(heavy), st
    if col.dim > 0:
        assert st["context_items"] > dense_chunk(sms), st   # stage A's neighbour table takes more than one chunk
    want, _ = item_to_item_spec(store, allow, dead, [ctxs[r] for r in rows], [ex[r] for r in rows], n)
    same_rows([got[r] for r in rows], want, "spec")
    pieces = []
    for a, b in in_pieces(nu, cu // 2):
        pieces += col.item_to_item(ctxs[a:b], ex[a:b], n)[0]
    same_rows(pieces, got, "pieces")


@gpu
def test_session_recommend(i2i_world, sms):
    col, store, hidden, dead, allow, ctxs, ex, rows, heavy = i2i_world
    nu, cu, n = len(ctxs), user_chunk(sms), 20
    assert_chunks(nu, cu)
    N = len(hidden)
    ok = (np.random.default_rng(13).random(N) >= 0.1).astype(np.uint8)
    nb = sm.oracle_neighbours(None, store, hidden, dead, n, 1.0)
    for context_size, top in ((3, 15), (400, n)):
        got, st = col.session_recommend(ctxs, ex, n, context_size, top, item_ok=ok)
        assert st["shared_sessions"] + st["global_sessions"] == nu, st
        same_rows([got[r] for r in rows], sm.session_rows(nb, [ctxs[r] for r in rows], [ex[r] for r in rows], context_size, top, ok), "spec")
    pieces = []
    for a, b in in_pieces(nu, cu // 2):
        pieces += col.session_recommend(ctxs[a:b], ex[a:b], n, 400, n, item_ok=ok)[0]
    same_rows(pieces, got, "pieces")


# ---- 4. user-to-user -----------------------------------------------------------------------------------------------------------------
def u2u_feedback(rng, N, n_items):
    """item rows per slot: every third slot 800 items, so that users with enough such neighbours take a global row"""
    m = np.where(np.arange(N) % 3 == 0, 800, rng.integers(0, 12, N))
    off = np.concatenate([[0], np.cumsum(m)])
    items = np.where(rng.random(off[-1]) < 0.3, rng.integers(0, 8, off[-1]), rng.integers(0, n_items, off[-1])).astype(np.int32)
    return split_rows(items, off)


@pytest.fixture(scope="module", params=["dense", "sparse"])
def u2u_world(request, gb, ctx, sms):
    kind = request.param
    N, n_items, cu = 40000, 5000, user_chunk(sms)
    col, block, hidden, dead = make_collection(gb, ctx, kind, N, 14)
    rng = np.random.default_rng(15)
    fb = u2u_feedback(rng, N, n_items)
    nu = past_three(cu)
    slots = rng.integers(0, N, nu).astype(np.int64)
    slots[np.arange(nu) % 11 == 3] = -1
    m = rng.integers(0, 6, nu)
    off = np.concatenate([[0], np.cumsum(m)])
    ex = split_rows(((np.repeat(rng.integers(0, n_items, nu), m) + (np.arange(off[-1]) - np.repeat(off[:-1], m)) * 13) % n_items).astype(np.int64), off)
    rows = check_rows(nu, cu, 24)
    allow = (hidden == 0) & ~dead
    store = NeighbourSpec(block, N, allow, 20, slots[rows].tolist())
    yield col, store, dead, allow, slots, fb, ex, rows, n_items
    col.close()


@gpu
def test_user_to_user(u2u_world, sms):
    col, store, dead, allow, slots, fb, ex, rows, n_items = u2u_world
    nu, cu, n = len(slots), user_chunk(sms), 20
    assert_chunks(nu, cu)
    # heavy users (more feedback entries than the shared-memory table's 6,144) in every chunk
    lens = np.array([len(f) for f in fb])
    work = np.array([lens[store.nb[int(s)][0]].sum() if s >= 0 and not dead[s] else 0 for s in slots[rows]])
    for c in range(-(-nu // cu)):
        assert (work[rows // cu == c] > 6144).any(), c
    ok = (np.random.default_rng(16).random(n_items) > 0.1).astype(np.uint8)
    for item_ok in (None, ok):
        got, st = col.user_to_user(slots, fb, ex, n, n_items, item_ok=item_ok)
        assert st["global_users"] > 0 and st["shared_users"] > 0 and st["shared_users"] + st["global_users"] <= nu, st
        want, _ = user_to_user_spec(store, allow, dead, slots[rows], fb, [ex[r] for r in rows], n, item_ok)
        same_rows([got[r] for r in rows], want, "spec")
    # the same users in calls of half a chunk: the same rows, and the routing counts of the chunks add up to the whole call's
    pieces, routed = [], np.zeros(2, np.int64)
    for a, b in in_pieces(nu, cu // 2):
        rows_p, st_p = col.user_to_user(slots[a:b], fb, ex[a:b], n, n_items, item_ok=ok)
        pieces += rows_p
        routed += (st_p["shared_users"], st_p["global_users"])
    same_rows(pieces, got, "pieces")
    assert routed.tolist() == [st["shared_users"], st["global_users"]], (routed, st)


# ---- 5. the sparse list path ------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sparse_world(gb, ctx):
    N = 20 * SPARSE_TILE
    vecs, A = sparse_data(17, N, 60, ())
    ix = gb.SparseIndex(ctx)
    ix.add(*sparse_csr(vecs))
    yield ix, vecs, A
    ix.close()


@gpu
@pytest.mark.parametrize("k", [1, 100, 128])
def test_sparse_index_search_range(sparse_world, k):
    ix, vecs, A = sparse_world
    N, ntiles = len(vecs), 20
    chunk = sparse_chunk(ntiles, k)
    chunks = -(-N // chunk)
    if k > 1:   # k = 1 fits 2.2M queries in one chunk
        assert_chunks(N, chunk)
    rows = check_rows(N, chunk, 25)
    ix.stats()
    idx, dot, cnt = ix.search_range(0, N, k)
    assert ix.stats()["tiles"] == ntiles * chunks
    specs = top_specs(None, A, False, np.full(rows.size, k), selfs=rows, positive=True, scores=lambda a, b: (A[rows[a:b]] @ A.T).astype(np.float32))
    for r, (s, v) in zip(rows, specs):
        c = len(s)
        assert cnt[r] == c and idx[r, :c].tolist() == s.tolist() and dot[r, :c].tobytes() == v.tobytes(), (r, k)
        assert (idx[r, c:] == -1).all() and (dot[r, c:] == 0).all()
    assert not (idx == np.arange(N)[:, None]).any()
    for a, b in in_pieces(N, max(chunk // 2, 20000)):
        i2, d2, c2 = ix.search_range(a, b, k)
        assert i2.tobytes() == idx[a:b].tobytes() and d2.tobytes() == dot[a:b].tobytes() and c2.tobytes() == cnt[a:b].tobytes()


@gpu
@pytest.mark.parametrize("k", [100, 128])
def test_sparse_collection_query(gb, ctx, sparse_world, k):
    _, vecs, A = sparse_world
    N, ntiles = len(vecs), 20
    chunk = sparse_chunk(ntiles, k)
    nq = past_three(chunk)
    assert_chunks(nq, chunk)
    rng = np.random.default_rng(26)
    hidden = (rng.random(N) < 0.08).astype(np.uint8)
    cats = [[int(c)] for c in rng.integers(0, 3, N)]
    qrows = rng.integers(0, N, nq)
    Q = [vecs[r] for r in qrows]
    rows = check_rows(nq, chunk, 27)
    with gb.VectorCollection(ctx, 0, gb.DISTANCE_DOT) as col:
        col.add(sparse=vecs, hidden=hidden, timestamps=np.full(N, 100), categories=cats)
        for want_c in ((), (1,)):
            allow = (hidden == 0) & (np.array([c[0] for c in cats]) == 1 if want_c else True)
            slots, scores, cnt = col.query(Q, want_c, k)
            specs = top_specs(None, A, False, np.full(rows.size, k), allow=allow, positive=True,
                              scores=lambda a, b: (A[qrows[rows[a:b]]] @ A.T).astype(np.float32))
            for r, (s, v) in zip(rows, specs):
                c = len(s)
                assert cnt[r] == c and slots[r, :c].tolist() == s.tolist() and scores[r, :c].tobytes() == v.tobytes(), (r, k, want_c)
                assert (slots[r, c:] == -1).all() and (scores[r, c:] == 0).all()
        for a, b in in_pieces(nq, chunk // 2):
            s2, v2, c2 = col.query(Q[a:b], (1,), k)
            assert s2.tobytes() == slots[a:b].tobytes() and v2.tobytes() == scores[a:b].tobytes() and c2.tobytes() == cnt[a:b].tobytes()


# ---- 6. gorse_b200_recommend -------------------------------------------------------------------------------------------------------------
@gpu
def test_recommend_item_to_item_and_user_to_user(gb, ctx, sms, i2i_world, u2u_world):
    """an item-to-item stage on the dense collection of i2i_world (its slots are the items) and a user-to-user stage on
    u2u_world's, over past_three(sm_count * 1024) users, against the per-user chaining of recommend_model"""
    col_i, store_i, hidden_i, dead_i, allow_i, ctxs, ex_i, rows, _ = i2i_world
    col_u, store_u, dead_u, allow_u, slots, fb, _, rows_u, n_items = u2u_world
    if col_i.dim == 0 or col_u.dim == 0:
        pytest.skip("the dense collections carry this test")
    nu, cu = len(ctxs), user_chunk(sms)
    assert len(slots) == nu and rows.tolist() != [] and n_items <= len(hidden_i)
    ni = len(hidden_i)
    E0 = ex_i
    live = np.ones(ni, np.uint8)
    ok = (np.random.default_rng(18).random(ni) > 0.1).astype(np.uint8)
    ident = np.arange(ni)
    fb_i = [f.astype(np.int32) for f in fb]
    stages = [gb.ItemToItemStage(col_i, 20, [c.astype(np.int32) for c in ctxs], ident, ident.astype(np.int32)),
              gb.UserToUserStage(col_u, 20, slots, fb_i, ok)]
    got, st = gb.recommend(ctx, E0, ni, live, stages)
    assert st["chunks"] >= 4, st
    chk = np.intersect1d(rows, rows_u)
    chk_slots = slots[chk]

    def i2i_stage(E):
        want, _ = item_to_item_spec(store_i, allow_i, dead_i, [ctxs[u] for u in chk], [sorted(e) for e in E], 20)
        return [[(int(i), float(v)) for i, v in zip(*w)] for w in want]

    def u2u_stage(E):
        want, _ = user_to_user_spec(store_u, allow_u, dead_u, chk_slots, fb, [sorted(e) for e in E], 20, ok)
        return [[(int(i), float(v)) for i, v in zip(*w)] for w in want]

    want = rm.chain([E0[u] for u in chk], live, [i2i_stage, u2u_stage])
    for u, w in zip(chk, want):
        items, scores = got[u]
        assert items.tolist() == [i for i, _ in w] and scores.tolist() == [s for _, s in w], u
