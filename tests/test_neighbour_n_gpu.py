"""Neighbour recommenders at every n: item-to-item, session, user-to-user, their gorse_b200_recommend stages and the neighbour
cache, from n = 1 to the dense limit 1024 (sparse: to 128), against the strict specs of tests/test_ties_gpu.py and
tests/test_chunks_gpu.py -- the first n allowed neighbours by (score descending, slot ascending), float64 sums in context
order, the first n sums by (sum descending, id ascending).  The n values straddle every limit that code sizes by n: the top-k
sweep's k classes 128 / 256 / 512 and the exact kernel above them, the table kernel's rounds of 128 entries, the stage-B sort
of pow2_at_least(top) entries written in rounds of 256, the user-to-user item filter in rounds of 256, the shared-memory
accumulator's TABLE_KEYS = 6144 adds, the recommend stages' lists of more than 256 items, and the neighbour cache's fill,
save and load chunks.  The data is tie-heavy with exact scores (grid-valued dense vectors, count-valued sparse ones), and a
few Dot rows have fewer positive neighbours than n, so the table kernel drops entries in later rounds.  A random fp32
collection pins the float64 summation order against the oracle's brute force.  The constants are restated from the code
and the CPU tests assert that the data crosses each of them; every GPU case asserts the path it was built for (exact rows,
users per accumulator, cache rows computed, held and left out, load stats), so the coverage cannot quietly shrink to n <= 50."""
import functools
import io
import struct

import numpy as np
import pytest

import recommend_model as rm
import session_model as sm
import test_item_to_item_gpu as i2i
import test_user_to_user_gpu as u2u
from test_chunks_gpu import NeighbourSpec, grid_rows, same_rows, sparse_block, top_specs
from test_ties_gpu import dense_scores, item_to_item_spec, sparse_data, user_to_user_spec

gpu = pytest.mark.gpu

DENSE_N = (1, 2, 100, 127, 128, 129, 255, 256, 257, 511, 512, 513, 1000, 1024)
SPARSE_N = (1, 100, 127, 128)

# ---- the limits, restated from the code ---------------------------------------------------------------------------------------
MAX_N_DENSE, MAX_N_SPARSE = 1024, 128   # stages.cuh
CLASS_K = (128, 256, 512)               # topk.cu: the sweep's k classes; a larger k takes the exact kernel
SWEEP_MIN_VECTORS, SWEEP_MIN_ROWS = 32768, 64   # topk_mma.cu mma_path_eligible (d <= 4096, Dot or Euclidean)
TABLE_ROUND = 128                       # topk.cu table_kernel<128>: a row's entries are compacted in rounds of 128
TABLE_KEYS = 6144                       # aggregate.cuh: a user takes the shared-memory table when its adds are at most this
FILL_CHUNK_BYTES = 64 << 20             # item_to_item.cu: rows of one fill chunk = FILL_CHUNK_BYTES / (16 n + 24)
STAGE_BYTES = 64 << 20                  # snapshot.cu: one staging buffer of the neighbour cache's save and load
NBR_HEADER = 48                         # include/gorse_b200.h: the neighbour cache stream's header; a row is 8 + 8 count bytes


def sweep_class(k):
    """the sweep's class of a row of k neighbours (topk.cu class_of): 0, 1, 2, or 3 = the exact kernel.  The class a row takes
    is not observable from outside the library, so it is restated here; the GPU cases observe the exact kernel's rows."""
    return next((t for t, c in enumerate(CLASS_K) if k <= c), len(CLASS_K))


def fill_chunk(n):
    return max(1, FILL_CHUNK_BYTES // (16 * n + 24))


def load_chunk(n):
    """rows of one load chunk (snapshot.cu ncache_load: R = STAGE_BYTES / (8 n + 4))"""
    return max(1, STAGE_BYTES // (8 * n + 4))


def save_chunks(counts):
    """chunks of a save of rows with these entry counts (snapshot.cu ncache_save: whole rows of 8 + 8 count bytes, at most
    cap = min(STAGE_BYTES, max(64 KB, all rows' bytes)) per chunk)"""
    b = 8 + 8 * np.asarray(counts, np.int64)
    cap = min(STAGE_BYTES, max(64 << 10, int(b.sum())))
    chunks, used = 1, 0
    for x in b.tolist():
        if used + x > cap:
            chunks, used = chunks + 1, 0
        used += x
    return chunks


@pytest.fixture(scope="module")
def ctx(gb):
    c = gb.Context(0)
    yield c
    c.close()


# ---- data -----------------------------------------------------------------------------------------------------------------------
N_BIG, N_ITEMS = 36000, 3000
N_CACHE = 40000


@functools.lru_cache(maxsize=None)
def big_rows():
    """N_BIG grid rows of d = 16 from N_BIG / 4 base rows, every value's sign set by one pattern sigma, except for the rows
    whose first four magnitudes are (7, 7, 7, >= 5) / 4 -- about 1 in 128, picked by value so that copies agree -- which carry
    -sigma: their Dot is positive with one another only, so they have fewer positive neighbours than n for n >= 300.
    -> (X, minority mask)"""
    X = np.abs(grid_rows(31, N_BIG, N_BIG // 4, 16))
    sigma = np.where(np.arange(16) % 3 == 0, -1, 1).astype(np.float32)
    few = (X[:, 0] == 1.75) & (X[:, 1] == 1.75) & (X[:, 2] == 1.75) & (X[:, 3] >= 1.25)
    return np.ascontiguousarray(X * np.where(few[:, None], -sigma, sigma)), few


@functools.lru_cache(maxsize=None)
def big_meta():
    """hidden, timestamps (about 3 % below the deletion cut 30) and one category per slot"""
    rng = np.random.default_rng(32)
    return (rng.random(N_BIG) < 0.08).astype(np.uint8), rng.integers(0, 1000, N_BIG), rng.integers(0, 3, N_BIG)


def planted_contexts(n, pool):
    """two users of floor(6144 / n) distinct live context slots (the shared table, |C_u| n <= TABLE_KEYS) and two of one
    more (a global row)"""
    k = TABLE_KEYS // n
    return [pool[i:i + m].astype(np.int64) for i, m in ((0, k), (7, k), (3, k + 1), (11, k + 1))]


@functools.lru_cache(maxsize=None)
def big_users():
    """96 users of test_item_to_item_gpu.make_users (contexts with -1, hidden, deleted and repeated slots; exclusions with
    -1), the pool the planted users draw from, the user-to-user slots, feedback rows and item filter"""
    hidden, ts, _ = big_meta()
    dead = ts < 30
    rng = np.random.default_rng(33)
    ctxs, excl = i2i.make_users(rng, N_BIG, hidden, dead, 96, max_ctx=8)
    live = np.flatnonzero(~dead)
    pool = rng.choice(live, 80, replace=False)
    slots, uex = u2u.make_users(rng, N_BIG, hidden, dead, 96, N_ITEMS)
    # seven feedback items per slot, 30 % of them one of 16 popular items; a slot's row holds six of them (big_feedback)
    items = np.where(rng.random((N_BIG, 7)) < 0.3, rng.integers(0, 16, (N_BIG, 7)), rng.integers(0, N_ITEMS, (N_BIG, 7))).astype(np.int32)
    ok = (rng.random(N_ITEMS) >= 1 / 3).astype(np.uint8)   # the filter drops a third of the items
    cand = rng.choice(live[~big_rows()[1][live]], 60, replace=False)   # user-to-user users planted by W_u at n = 1024
    return ctxs, excl, pool, slots, uex, items, ok, cand


class Lists:
    """QueryItemToItem / QueryUserToUser lists of the slots the checked users need, built once at the largest n; the list
    at a smaller n is the first n entries of it (the interface of test_ties_gpu.Spec)"""

    def __init__(self, nb):
        self.nb = nb

    def neighbours(self, orc, c, allow, n, scale):
        s, v = self.nb[int(c)]
        return s[:n], v[:n] * scale


def dense_lists(orc, X, euclid, allow, slots, nmax=MAX_N_DENSE):
    """Dot: NeighbourSpec (scores > 0 only); Euclidean: the first nmax of top_specs, scored 1 / (1 + distance) by the
    oracle's QueryItemToItem post-processing"""
    N, block = len(X), (lambda rows: dense_scores(X[rows], X, euclid))
    if not euclid:
        return Lists(NeighbourSpec(block, N, allow, nmax, slots).nb)
    slots = np.unique(np.asarray([s for s in slots if s >= 0], np.int64))
    rows = top_specs(None, X, True, np.full(slots.size, nmax), selfs=slots, allow=allow, scores=lambda a, b: block(slots[a:b]))
    return Lists({int(c): orc.similar_scores(True, 1.0, -1, nmax, s.astype(np.int32), v) for c, (s, v) in zip(slots, rows)})


def sparse_lists(A, allow, slots):
    return Lists(NeighbourSpec(sparse_block(A), A.shape[0], allow, MAX_N_SPARSE, slots).nb)


def big_allow(cat=None):
    hidden, ts, cats = big_meta()
    a = (hidden == 0) & (ts >= 30)
    return a if cat is None else a & (cats == cat)


@functools.lru_cache(maxsize=None)
def big_lists(orc, euclid, cat=None):
    X, _ = big_rows()
    ctxs, _, pool, slots, _, _, _, cand = big_users()
    need = np.concatenate([np.concatenate(ctxs), pool, slots, cand])
    return dense_lists(orc, X, euclid, big_allow(cat), need)


def live_len(ctx_u, dead):
    return sum(1 for c in ctx_u if c >= 0 and not dead[c])


def u2u_work(lists, slots, fb, dead, n):
    """W_u: the feedback entries of user u's n neighbours (0 for a user without a vector)"""
    return np.array([0 if s < 0 or dead[s] else sum(len(fb[v]) for v in lists.nb[int(s)][0][:n]) for s in slots])


@functools.lru_cache(maxsize=None)
def big_feedback(orc, euclid):
    """the feedback rows: six items per slot, seven for the hot slots -- up to 60 slots in the 1024 neighbours of two planted
    candidates and in neither list of two others.  -> (rows, the four planted users): the first two have W_u = 6144 at
    n = 1024 (the shared table), the last two more (a global row)"""
    lists = big_lists(orc, euclid)
    _, _, _, _, _, items, _, cand = big_users()
    full = [int(c) for c in cand if len(lists.nb[int(c)][0]) == MAX_N_DENSE]
    cold = set(lists.nb[full[0]][0].tolist()) | set(lists.nb[full[1]][0].tolist())
    warm = [c for c in full[2:] if set(lists.nb[c][0].tolist()) - cold][:2]
    hot = np.array(sorted((set(lists.nb[warm[0]][0].tolist()) | set(lists.nb[warm[1]][0].tolist())) - cold), np.int64)
    hot = np.random.default_rng(34).permutation(hot)[:60]
    m = np.full(N_BIG, 6)
    m[hot] = 7
    return [items[s, :m[s]] for s in range(N_BIG)], np.array(full[:2] + warm, np.int64)


# ---- premises (CPU) ------------------------------------------------------------------------------------------------------------
def test_premises_limits():
    """the n values cover every sweep class and both sides of each class limit, the dense and sparse maxima, one and more
    table rounds; the planted users straddle TABLE_KEYS; the cache data takes the fill, save and load chunks the cases need"""
    for c in CLASS_K:
        assert c in DENSE_N and c + 1 in DENSE_N
    assert {sweep_class(n) for n in DENSE_N} == {0, 1, 2, 3}
    assert [n for n in DENSE_N if sweep_class(n) == 3][0] == 513
    assert max(DENSE_N) == MAX_N_DENSE and max(SPARSE_N) == MAX_N_SPARSE and min(DENSE_N) == 1
    assert any(-(-n // TABLE_ROUND) > 2 for n in DENSE_N)
    assert any(n > 256 for n in DENSE_N)   # stage-B writes and the user-to-user filter take more than one round of 256
    for n in (100, 1024):
        k = TABLE_KEYS // n
        assert k * n <= TABLE_KEYS < (k + 1) * n
    assert TABLE_KEYS // 1024 == 6 and TABLE_KEYS // 100 == 61
    # the neighbour cache at n = 1024 over N_CACHE full Euclidean lists
    fc, lc = fill_chunk(1024), load_chunk(1024)
    assert (fc, lc) == (4090, 8188)
    assert -(-N_CACHE // fc) >= 9
    small = 2 * fc + fc // 2
    assert small % fc != 0 and small < N_CACHE
    assert save_chunks(np.full(N_CACHE, 1024)) >= 4 and save_chunks(np.full(N_CACHE, 1024)) == -(-N_CACHE // (STAGE_BYTES // (8 + 8 * 1024)))
    assert -(-N_CACHE // lc) >= 4
    assert lc < lc + lc // 2 < 2 * lc   # the smaller pool's cut falls inside the second load chunk
    assert N_CACHE * (8 * 1024 + 4) < 400 << 20


def test_premises_data(orc):
    """the big collection crosses the sweep's limits, its scores are the oracle's, some Dot rows have fewer positive
    neighbours than n at several table rounds, and the user-to-user candidates give users on both sides of TABLE_KEYS"""
    X, few = big_rows()
    hidden, ts, _ = big_meta()
    dead = ts < 30
    assert len(X) >= SWEEP_MIN_VECTORS and 200 < few.sum() < 400
    assert (X.astype(np.float32).view(np.uint32) & 0xFFFF == 0).all()   # bf16-exact
    rng = np.random.default_rng(0)
    for euclid in (False, True):
        cols = rng.choice(N_BIG, 100)
        S = dense_scores(X[:3], X[cols], euclid)
        for i in range(3):
            for j, c in enumerate(cols):
                want = -orc.euclidean(X[i], X[c]) if euclid else orc.dot(X[i], X[c])
                assert S[i, j].tobytes() == np.float32(want).tobytes()
    ctxs, _, pool, slots, _, _, _, _ = big_users()
    distinct = {c for u in ctxs for c in u.tolist() if c >= 0 and not dead[c]}
    assert len(distinct) >= SWEEP_MIN_ROWS
    assert len({s for s in slots.tolist() if s >= 0 and not dead[s]}) >= SWEEP_MIN_ROWS
    dot = big_lists(orc, False)
    short = [len(dot.nb[c][0]) for c in distinct if few[c]]
    assert any(TABLE_ROUND < k < 1000 for k in short), short   # the table kernel drops entries after its first round
    assert any(len(dot.nb[c][0]) == MAX_N_DENSE for c in distinct)
    for euclid in (False, True):
        lists = big_lists(orc, euclid)
        fb, planted = big_feedback(orc, euclid)
        assert len(planted) == 4
        w = u2u_work(lists, planted, fb, dead, MAX_N_DENSE)
        assert w[0] == w[1] == TABLE_KEYS and (w[2:] > TABLE_KEYS).all(), w


# ---- A. item-to-item ------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module", params=["dot", "euclid"])
def big(request, gb, ctx, orc):
    euclid = request.param == "euclid"
    X, _ = big_rows()
    hidden, ts, cats = big_meta()
    col = gb.VectorCollection(ctx, X.shape[1], gb.DISTANCE_EUCLIDEAN if euclid else gb.DISTANCE_DOT)
    col.add(X, hidden=hidden, timestamps=ts, categories=[[int(c)] for c in cats])
    dead = np.zeros(N_BIG, bool)
    dead[col.delete_before(30)] = True
    assert (dead == (ts < 30)).all() and col.storage()[0] == 2
    yield col, euclid, hidden, dead, big_lists(orc, euclid)
    col.close()


def i2i_users(n, dead):
    """the 96 users, and at n = 100 and 1024 the four planted ones"""
    ctxs, excl, pool, _, _, _, _, _ = big_users()
    ctxs, excl = list(ctxs), list(excl)
    if n in (100, 1024):
        extra = planted_contexts(n, pool)
        ctxs += extra
        excl += [np.array([-1, int(pool[40])], np.int64)] * len(extra)
    return ctxs, excl


@gpu
@pytest.mark.parametrize("path", ["sweep", "exact"])
def test_item_to_item(orc, big, monkeypatch, path):
    col, euclid, hidden, dead, lists = big
    if path == "exact":
        monkeypatch.setenv("GORSE_B200_TOPK_EXACT", "1")
    allow = big_allow()
    for n in DENSE_N:
        ctxs, excl = i2i_users(n, dead)
        got, st = col.item_to_item(ctxs, excl, n)
        want, _ = item_to_item_spec(lists, allow, dead, ctxs, excl, n)
        same_rows(got, want, ("i2i", n))
        live = [live_len(c, dead) for c in ctxs]
        heavy = sum(m * n > TABLE_KEYS for m in live)
        assert (st["shared_users"], st["global_users"]) == (len(ctxs) - heavy, heavy), (n, st)
        if n in (100, 1024):
            assert st["shared_users"] >= 2 and st["global_users"] >= 2, (n, st)
        assert st["context_items"] >= SWEEP_MIN_ROWS
        assert (st["exact_rows"] == st["context_items"]) == (path == "exact" or sweep_class(n) == 3), (n, st)
        assert max(len(r[0]) for r in got) == n
    if path == "sweep":   # a category filter at n = 513
        n = 513
        ctxs, excl = i2i_users(n, dead)
        got, _ = col.item_to_item(ctxs, excl, n, categories=[1])
        want, _ = item_to_item_spec(big_lists(orc, euclid, 1), big_allow(1), dead, ctxs, excl, n)
        same_rows(got, want, ("i2i category", n))


@functools.lru_cache(maxsize=None)
def sparse_world():
    vecs, A = sparse_data(5, 4000, 40, (1.0, 1.5, 0.75))
    rng = np.random.default_rng(34)
    N = len(vecs)
    hidden, ts = (rng.random(N) < 0.08).astype(np.uint8), rng.integers(0, 1000, N)
    dead = ts < 30
    ctxs, excl = i2i.make_users(rng, N, hidden, dead, 96, max_ctx=8)
    pool = rng.choice(np.flatnonzero(~dead), 80, replace=False)
    ctxs += planted_contexts(100, pool)
    excl += [np.zeros(0, np.int64)] * 4
    allow = (hidden == 0) & ~dead
    return vecs, A, hidden, ts, ctxs, excl, allow


@gpu
def test_item_to_item_sparse(gb, ctx):
    vecs, A, hidden, ts, ctxs, excl, allow = sparse_world()
    N = len(vecs)
    lists = sparse_lists(A, allow, np.concatenate(ctxs))
    dead = ts < 30
    with gb.VectorCollection(ctx, 0, gb.DISTANCE_DOT) as col:
        col.add(sparse=vecs, hidden=hidden, timestamps=ts)
        col.delete_before(30)
        for n in SPARSE_N:
            got, st = col.item_to_item(ctxs, excl, n)
            same_rows(got, item_to_item_spec(lists, allow, dead, ctxs, excl, n)[0], ("sparse i2i", n))
            heavy = sum(live_len(c, dead) * n > TABLE_KEYS for c in ctxs)
            assert st["global_users"] == heavy and (n != 100 or heavy >= 2), (n, st)


# ---- order-sensitive sums against the oracle -------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("kind", ["euclid", "dot"])
def test_float64_sums_equal_the_oracle(gb, orc, ctx, kind):
    """random fp32 vectors (N = 3,000, the exact scan): item-to-item and user-to-user sums at n = 100, 513 and 1024 equal the
    oracle's brute force summed in context / neighbour order, bit for bit"""
    rng = np.random.default_rng(35 if kind == "euclid" else 36)
    N = 3000
    col, store, hidden, dead, cats = i2i.dense_collection(gb, ctx, rng, N, 32, gb.DISTANCE_EUCLIDEAN if kind == "euclid" else gb.DISTANCE_DOT)
    with col:
        assert col.storage()[0] == 4
        ctxs, excl = i2i.make_users(rng, N, hidden, dead, 32, max_ctx=6)
        fb = u2u.make_feedback(rng, N, 2000)
        slots, uex = u2u.make_users(rng, N, hidden, dead, 32, 2000)
        ok = (rng.random(2000) > 0.3).astype(np.uint8)
        allow = i2i.allow_mask(hidden, dead, cats)
        for n in (100, 513, 1024):
            got, st = col.item_to_item(ctxs, excl, n)
            assert st["exact_rows"] == st["context_items"] > 0
            i2i.assert_rows_equal(got, i2i.expected(orc, store, allow, dead, ctxs, excl, n, 1.0))
            if kind == "euclid" and n == 1024:
                rev = i2i.expected(orc, store, allow, dead, ctxs, excl, n, 1.0, reverse=True)
                assert any(g[1].tobytes() != r[1].tobytes() for g, r in zip(got, rev))
            got, _ = col.user_to_user(slots, fb, uex, n, 2000, item_ok=ok)
            u2u.assert_rows_equal(got, u2u.expected(orc, store, allow, dead, slots, fb, uex, n, 1.0, ok))


# ---- collections smaller than n ----------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("N", [300, 1025])
@pytest.mark.parametrize("kind", ["dot", "euclid"])
def test_small_collections(gb, orc, ctx, N, kind):
    """N = 300 is below most n; at N = 1,025 every Euclidean list holds exactly n = 1024 entries.  Every one-slot context
    answers its whole neighbour list."""
    euclid = kind == "euclid"
    X = grid_rows(37, N, N // 4, 16)
    rng = np.random.default_rng(38)
    ctxs = [rng.integers(0, N, int(rng.integers(1, 5))).astype(np.int64) for _ in range(40)] + [np.array([s], np.int64) for s in range(0, N, 37)]
    excl = [np.zeros(0, np.int64)] * len(ctxs)
    allow, dead = np.ones(N, bool), np.zeros(N, bool)
    lists = dense_lists(orc, X, euclid, allow, np.arange(N))
    fb = [rng.integers(0, 500, 6).astype(np.int32) for _ in range(N)]
    slots = rng.integers(0, N, 40).astype(np.int64)
    uex = [np.zeros(0, np.int64)] * 40
    with gb.VectorCollection(ctx, 16, gb.DISTANCE_EUCLIDEAN if euclid else gb.DISTANCE_DOT) as col:
        col.add(X)
        for n in DENSE_N:
            got, _ = col.item_to_item(ctxs, excl, n)
            same_rows(got, item_to_item_spec(lists, allow, dead, ctxs, excl, n)[0], ("i2i", N, n))
            for (s, _), c in zip(got[40:], ctxs[40:]):
                assert len(s) == len(lists.nb[int(c[0])][0][:n])
                if euclid:
                    assert len(s) == min(n, N - 1)
            got, _ = col.user_to_user(slots, fb, uex, n, 500)
            same_rows(got, user_to_user_spec(lists, allow, dead, slots, fb, uex, n, None)[0], ("u2u", N, n))


# ---- B. session ---------------------------------------------------------------------------------------------------------------------
@gpu
def test_session_recommend(big):
    """top 1, n and 1024 at n = 1, 100 and 1024: the stage-B sort is sized by top, not by n"""
    col, euclid, hidden, dead, lists = big
    ok = (np.random.default_rng(39).random(N_BIG) >= 0.15).astype(np.uint8)
    for n in (1, 100, 1024):
        ctxs, excl = i2i_users(n, dead)
        nb = sm.oracle_neighbours(None, lists, hidden, dead, n, 1.0)
        for top in sorted({1, n, 1024}):
            for context_size, item_ok in ((3, ok), (1000, None)):
                got, st = col.session_recommend(ctxs, excl, n, context_size, top, item_ok=item_ok)
                assert st["shared_sessions"] + st["global_sessions"] == len(ctxs), st
                want = sm.session_rows(nb, ctxs, excl, context_size, top, item_ok)
                same_rows(got, want, ("session", n, top, context_size))
                if top == 1024 and n > 1 and item_ok is None:
                    assert max(len(r[0]) for r in want) > 256   # the answer is written in more than one round
                if top > n == 1:
                    assert max(len(r[0]) for r in want) > 1


# ---- C. user-to-user ---------------------------------------------------------------------------------------------------------------
@gpu
def test_user_to_user(orc, big):
    col, euclid, hidden, dead, lists = big
    _, _, _, slots, uex, _, ok, _ = big_users()
    fb, planted = big_feedback(orc, euclid)
    allow = big_allow()
    over_total = 0
    for n in DENSE_N:
        s, e = slots, list(uex)
        if n == 1024:
            s = np.concatenate([slots, planted])
            e += [np.array([-1], np.int64)] * len(planted)
        for item_ok in (None, ok):
            got, st = col.user_to_user(s, fb, e, n, N_ITEMS, item_ok=item_ok)
            want, over = user_to_user_spec(lists, allow, dead, s, fb, e, n, item_ok)
            same_rows(got, want, ("u2u", n, item_ok is None))
            w = u2u_work(lists, s, fb, dead, n)
            assert (st["shared_users"], st["global_users"]) == (int(((w > 0) & (w <= TABLE_KEYS)).sum()), int((w > TABLE_KEYS).sum())), (n, st)
            if n == 1024:
                assert (w == TABLE_KEYS).sum() >= 2 and (w > TABLE_KEYS).sum() >= 2
            if item_ok is None:
                over_total += over
                if n >= 512:
                    assert max(len(r[0]) for r in want) == n
            elif n >= 512:   # the filter keeps entries that are not a prefix, past the first round of 256
                assert any(len(r[0]) > 256 and len(r[0]) < n for r in want)
    assert over_total >= 5, over_total


@gpu
def test_user_to_user_sparse(gb, ctx):
    vecs, A, hidden, ts, _, _, allow = sparse_world()
    N = len(vecs)
    dead = ts < 30
    rng = np.random.default_rng(40)
    slots, uex = u2u.make_users(rng, N, hidden, dead, 96, N_ITEMS)
    fb = [rng.integers(0, N_ITEMS, 6).astype(np.int32) for _ in range(N)]
    ok = (rng.random(N_ITEMS) >= 1 / 3).astype(np.uint8)
    lists = sparse_lists(A, allow, slots)
    with gb.VectorCollection(ctx, 0, gb.DISTANCE_DOT) as col:
        col.add(sparse=vecs, hidden=hidden, timestamps=ts)
        col.delete_before(30)
        for n in SPARSE_N:
            got, _ = col.user_to_user(slots, fb, uex, n, N_ITEMS, item_ok=ok)
            same_rows(got, user_to_user_spec(lists, allow, dead, slots, fb, uex, n, ok)[0], ("sparse u2u", n))


# ---- D. recommend stages --------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("n", [100, 257, 1024])
def test_recommend_stages(gb, ctx, orc, big, n):
    """a per-user list of 600 entries, each item twice (rec_grow's duplicate branch at p = 1024), then ItemToItemStage and
    UserToUserStage at n on the big collection (its slots are the items): one call equals the composed path of the
    single-stage entries"""
    from test_recommend_gpu import check_same

    col, euclid, hidden, dead, lists = big
    ctxs, _ = i2i_users(n, dead)
    _, _, _, slots, _, _, ok_items, _ = big_users()
    fb = big_feedback(orc, euclid)[0]
    nu = len(slots)
    ok = np.zeros(N_BIG, np.uint8)   # the stage's dictionary is the collection's slots; the feedback names the first N_ITEMS
    ok[:N_ITEMS] = ok_items
    ctxs = ctxs[:nu]
    rng = np.random.default_rng(41 + n)
    E0 = [np.unique(rng.integers(0, N_BIG, int(rng.integers(0, 20)))).tolist() + ([-1] if u % 3 == 0 else []) for u in range(nu)]
    dup = []
    for u in range(nu):
        it = rng.choice(N_BIG, 300, replace=False).astype(np.int32)
        dup.append((rng.permutation(np.concatenate([it, it])), np.zeros(600)))
    live = (rng.random(N_BIG) > 0.05).astype(np.uint8)
    ident = np.arange(N_BIG, dtype=np.int64)
    stages = [gb.ListStage(per_user=dup), gb.ItemToItemStage(col, n, ctxs, ident, ident.astype(np.int32)),
              gb.UserToUserStage(col, n, slots, fb, ok)]
    got, st = gb.recommend(ctx, E0, N_BIG, live, stages)

    def i2i_run(E):
        rows, _ = col.item_to_item(ctxs, [sorted(e) for e in E], n)
        return [[(int(s), float(v)) for s, v in zip(*r)] for r in rows]

    def u2u_run(E):
        rows, _ = col.user_to_user(slots, fb, [sorted(e) for e in E], n, N_BIG, ok)
        return [[(int(i), float(v)) for i, v in zip(*r)] for r in rows]

    want = rm.chain(E0, live, [rm.external_stage(dup), i2i_run, u2u_run])
    check_same(got, want)
    assert st["candidates"] == sum(len(r) for r in want)
    assert max(len(i2i_run([set(e) for e in E0])[u]) for u in range(nu)) == n   # a stage appends n items


# ---- E. the neighbour cache at n = 1024 -----------------------------------------------------------------------------------------------
class Counting(io.BytesIO):
    """a stream that counts the writes it is handed (the save's header, then one per chunk)"""

    def __init__(self):
        super().__init__()
        self.writes = 0

    def write(self, b):
        self.writes += 1
        return super().write(b)


def cache_entries(gb, a, b, rng, N, n=MAX_N_DENSE, users=160):
    """item-to-item, session, user-to-user and both recommend stages on a and b: the same answers, bit for bit"""
    ctxs = [rng.integers(0, N, int(rng.integers(1, 5))).tolist() for _ in range(users)]
    excl = [np.unique(rng.integers(0, N, 3)).tolist() for _ in range(users)]
    same_rows(a.item_to_item(ctxs, excl, n)[0], b.item_to_item(ctxs, excl, n)[0], "i2i")
    ok = (np.arange(N) % 3 != 0).astype(np.uint8)
    same_rows(a.session_recommend(ctxs, excl, n, 2, n, item_ok=ok)[0], b.session_recommend(ctxs, excl, n, 2, n, item_ok=ok)[0], "session")
    fb = [rng.integers(0, 500, 3).tolist() for _ in range(N)]
    slots = rng.integers(-1, N, users).astype(np.int64)
    uex = [[] for _ in slots]
    same_rows(a.user_to_user(slots, fb, uex, n, 500)[0], b.user_to_user(slots, fb, uex, n, 500)[0], "u2u")
    ident = np.arange(N, dtype=np.int64)
    out = [gb.recommend(c.ctx, excl, N, np.ones(N, np.uint8), [gb.ItemToItemStage(c, n, ctxs, ident, ident.astype(np.int32)),
                                                                gb.UserToUserStage(c, n, slots, fb)])[0] for c in (a, b)]
    same_rows(out[0], out[1], "recommend")


def held_rows(s):
    """(row ranks, entry counts) of a stream, parsed by the documented format"""
    rows = struct.unpack_from("<q", s, 40)[0]
    at, ranks, counts = NBR_HEADER, [], []
    for _ in range(rows):
        r, c = struct.unpack_from("<ii", s, at)
        ranks.append(r)
        counts.append(c)
        at += 8 + 8 * c
    assert at == len(s)
    return ranks, np.array(counts, np.int64)


@functools.lru_cache(maxsize=None)
def cache_rows():
    """N_CACHE grid rows as big_rows builds them: the Dot of two rows is positive exactly when both carry the same sign
    pattern, so a minority row's list holds the other minority rows and every other list is full.  The lists' lengths
    differ between the rows of every chunk.  -> (X, entry count of each row's list at n = 1024)"""
    X = np.abs(grid_rows(42, N_CACHE, N_CACHE // 4, 16))
    sigma = np.where(np.arange(16) % 3 == 0, -1, 1).astype(np.float32)
    few = (X[:, 0] == 1.75) & (X[:, 1] == 1.75) & (X[:, 2] == 1.75) & (X[:, 3] >= 1.25)
    X = np.ascontiguousarray(X * np.where(few[:, None], -sigma, sigma))
    return X, np.where(few, min(MAX_N_DENSE, int(few.sum()) - 1), MAX_N_DENSE).astype(np.int64)


def test_premises_cache_rows():
    X, cnt = cache_rows()
    assert 100 < (cnt < MAX_N_DENSE).sum() < 500 and len(X) == N_CACHE
    S = dense_scores(X[:200], X, False)
    assert (cnt[:200] == np.minimum(MAX_N_DENSE, (S > 0).sum(1) - 1)).all()   # positive Dots but the row's own
    lc = load_chunk(MAX_N_DENSE)
    for k in range(-(-N_CACHE // lc)):   # short lists in every load chunk
        assert (cnt[k * lc:(k + 1) * lc] < MAX_N_DENSE).any()
    assert save_chunks(cnt) >= 4


@gpu
def test_neighbour_cache_chunks(gb, ctx):
    n, N = MAX_N_DENSE, N_CACHE
    X, cnt = cache_rows()
    fc, lc = fill_chunk(n), load_chunk(n)
    length = NBR_HEADER + int((8 + 8 * cnt).sum())
    at = lambda rows: NBR_HEADER + int((8 + 8 * cnt[:rows]).sum())   # the stream's offset of row `rows`
    src, off = (gb.VectorCollection(ctx, 16, gb.DISTANCE_DOT) for _ in range(2))
    try:
        for c in (src, off):
            c.add(X)
        # fill: every list, in ceil(N / 4090) >= 9 chunks; then every entry answers from the cache as its uncached twin
        src.neighbour_cache(n, N)
        st = src.neighbour_cache_fill()
        assert (st["computed"], st["rows"], st["left_out"]) == (N, N, 0), st
        cache_entries(gb, src, off, np.random.default_rng(43), N)
        st = src.neighbour_cache_stats()
        assert st["computed"] == N and st["served"] > 0 and st["rows"] == N, st
        # save: the header, then >= 4 chunks of whole rows
        out = Counting()
        assert src.save_neighbour_cache(out) == length
        nbr = out.getvalue()
        assert len(nbr) == length and out.writes == 1 + save_chunks(cnt) >= 5
        ranks, counts = held_rows(nbr)
        assert ranks == list(range(N)) and (counts == cnt).all()
        snap = io.BytesIO()
        assert (src.save(snap) == np.arange(N)).all()
        with gb.Context(0) as ctx2:
            dst = gb.VectorCollection.load(ctx2, io.BytesIO(snap.getvalue()))
            try:
                # load into a full pool: ceil(N / 8188) >= 4 chunks through the two staging buffers, each chunk's rows and
                # counts arriving whole
                dst.neighbour_cache(n, N)
                assert dst.load_neighbour_cache(io.BytesIO(nbr)) == dict(loaded=N, dropped=0, bytes=len(nbr))
                again = Counting()
                dst.save_neighbour_cache(again)
                assert again.getvalue() == nbr
                cache_entries(gb, dst, src, np.random.default_rng(44), N)
                st = dst.neighbour_cache_stats()
                assert st["computed"] == 0 and st["served"] > 0, st
                # load into a pool of 1.5 chunks: the cut falls inside the second chunk
                kept = lc + lc // 2
                dst.neighbour_cache(n, kept)
                assert dst.load_neighbour_cache(io.BytesIO(nbr)) == dict(loaded=kept, dropped=N - kept, bytes=len(nbr))
                again = Counting()
                dst.save_neighbour_cache(again)
                s = again.getvalue()
                assert held_rows(s)[0] == list(range(kept)) and s[NBR_HEADER:] == nbr[NBR_HEADER:at(kept)]
                cache_entries(gb, dst, src, np.random.default_rng(45), N)
                st = dst.neighbour_cache_stats()
                assert st["rows"] == kept and st["computed"] > 0, st   # the rows past the pool are computed, not held
            finally:
                dst.close()
        # fill into a pool that ends inside the third fill chunk
        cap = 2 * fc + fc // 2
        off.neighbour_cache(n, cap)
        st = off.neighbour_cache_fill()
        assert (st["computed"], st["rows"], st["left_out"]) == (cap, cap, N - cap), st
        again = Counting()
        off.save_neighbour_cache(again)
        assert held_rows(again.getvalue())[0] == list(range(cap)) and again.getvalue()[NBR_HEADER:] == nbr[NBR_HEADER:at(cap)]
    finally:
        src.close()
        off.close()
