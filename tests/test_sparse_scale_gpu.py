"""The tiled sparse search (csrc/sparse.cu) at sizes that cross every boundary of its layout: several tiles of 8192 rows plus a
remainder, a head feature held by most rows, queries of 25,000 features next to queries of one, empty rows, allow masks that
hide a tile's best rows, external query vectors and count-valued vectors with exact ties at the k-th place.  Every answer must
equal the oracle's sparse brute force bit for bit -- rows, dot bits and order, the order being (dot desc, row asc) -- through
the index's search_range, the collection's query, and one sparse case each of item-to-item, user-to-user and session
recommendation against their restated recommenders.  The stats hook shows that both accumulation paths ran."""
import numpy as np
import pytest

import session_model as sm
import test_item_to_item_gpu as i2i
import test_user_to_user_gpu as u2u

pytestmark = pytest.mark.gpu

TILE = 8192
N = 3 * TILE + 1234
F = 30000
HEAVY = (5, TILE + 17, 2 * TILE + 4000, 3 * TILE + 600)   # rows with 25,000 features, one in every tile


@pytest.fixture(scope="module")
def ctx(gb):
    c = gb.Context(0)
    yield c
    c.close()


def make_vectors(seed, count_valued):
    """N rows: 0..40 uniform features, feature 0 (the head) in 70 % of them, every 13th row empty, every 29th row a single
    feature, the HEAVY rows 25,000 features; values 1 (dots count shared features) or positive floats with a few negatives"""
    rng = np.random.default_rng(seed)
    vecs = []
    for r in range(N):
        if r in HEAVY:
            f = rng.choice(F, size=25000, replace=False)
        elif r % 13 == 0:
            f = np.zeros(0, np.int64)
        elif r % 29 == 0:
            f = rng.choice(F, size=1)
        else:
            f = rng.choice(np.arange(1, F), size=int(rng.integers(0, 41)), replace=False)
            if rng.random() < 0.7:
                f = np.concatenate([[0], f])
        f = np.sort(f).astype(np.uint32)
        if count_valued:
            v = np.ones(f.size, np.float32)
        else:
            v = (rng.random(f.size) * 2 + 0.05).astype(np.float32)
            v[rng.random(f.size) < 0.05] *= -1
        vecs.append((f, v))
    return vecs


def pack(vecs):
    off = np.concatenate([[0], np.cumsum([len(v[0]) for v in vecs])]).astype(np.int64)
    ind = np.concatenate([v[0] for v in vecs]).astype(np.uint32)
    val = np.concatenate([v[1] for v in vecs]).astype(np.float32)
    return off, ind, val


class Data:
    """the vectors, their CSR and the oracle's dots of every row with a query, memoised per query"""

    def __init__(self, orc, count_valued):
        self.orc, self.count_valued = orc, count_valued
        self.vecs = make_vectors(7 if count_valued else 8, count_valued)
        self.off, self.ind, self.val = pack(self.vecs)
        self.cache = {}

    def dots(self, q, vec=None):
        """the oracle's dot of every row with stored row q (q itself left out), or with the external vector `vec` (q = -1,
        memoised by its bytes): (rows, dots)"""
        key = q if vec is None else (vec[0].tobytes(), vec[1].tobytes())
        if key not in self.cache:
            qi, qv = self.vecs[q] if vec is None else vec
            qi, qv = np.ascontiguousarray(qi, np.uint32), np.ascontiguousarray(qv, np.float32)
            oi, od = np.zeros(N, np.int32), np.zeros(N, np.float32)
            m = self.orc.lib().gbo_sparse_bruteforce_search(self.off, self.ind, self.val, N, qi, qv, len(qi), q, N, oi, od)
            self.cache[key] = (oi[:m].copy(), od[:m].copy())
        return self.cache[key]

    def first_k(self, q, k, allow=None, vec=None):
        """the oracle's positive dots, allowed rows only, in (dot desc, row asc) order, cut at k"""
        oi, od = self.dots(q, vec)
        keep = od > 0
        if allow is not None:
            keep &= allow[oi]
        oi, od = oi[keep], od[keep]
        o = np.lexsort((oi, -od.astype(np.float64)))[:k]
        return oi[o], od[o]


@pytest.fixture(scope="module", params=["idf", "count"])
def data(request, orc):
    return Data(orc, request.param == "count")


def query_rows(data):
    """the heavy rows, the rows around each tile edge, empty and single-feature rows, and a seeded sample"""
    rng = np.random.default_rng(3)
    edges = [e + d for e in range(0, N, TILE) for d in (-1, 0, 1) if 0 <= e + d < N]
    rows = set(HEAVY) | set(edges) | {0, 13, 29, 58, N - 1} | set(rng.integers(0, N, 60).tolist())
    return sorted(rows)


def assert_equal(idx, dot, cnt, want_i, want_d, k, what):
    assert cnt == len(want_i), what
    assert idx[:cnt].tolist() == want_i.tolist(), what
    assert dot[:cnt].tobytes() == want_d.tobytes(), what
    assert (idx[cnt:] == -1).all() and (dot[cnt:] == 0).all(), what


def test_data_crosses_the_boundaries(data):
    lens = np.diff(data.off)
    assert (lens == 0).sum() > 1000 and (lens == 1).sum() > 500 and lens.max() == 25000
    assert (data.ind == 0).sum() > 0.6 * N   # the head feature
    if data.count_valued:                    # count-valued: exact ties at the k-th place for most queries
        ties = 0
        for q in query_rows(data)[:40]:
            _, od = data.first_k(q, N)
            ties += len(od) > 100 and od[99] == od[100]
        assert ties >= 20


@pytest.mark.parametrize("k", [1, 100, 128])
def test_search_range(gb, ctx, data, k):
    with gb.SparseIndex(ctx) as ix:
        ix.add(data.off, data.ind, data.val)
        ix.stats()
        rows = query_rows(data)
        idx, dot, cnt = ix.search_range(0, N, k)
        st = ix.stats()
        for q in rows:
            assert_equal(idx[q], dot[q], cnt[q], *data.first_k(q, k), k, f"row {q}")
        # both accumulation paths ran: the heavy rows' tiles pull, the rest push
        assert st["push"] > 0 and st["pull"] > 0, st
        assert st["tiles"] >= 4 and st["search_ms"] > 0, st
        # a range that starts inside the data, through a heavy row
        q0, q1 = HEAVY[1] - 3, HEAVY[1] + 500
        i2, d2, c2 = ix.search_range(q0, q1, k)
        assert i2.tolist() == idx[q0:q1].tolist() and d2.tobytes() == dot[q0:q1].tobytes() and c2.tolist() == cnt[q0:q1].tolist()


@pytest.fixture(scope="module")
def collection(gb, ctx, data):
    """the data as a sparse collection; hidden: 5 % of the rows plus, for query row HEAVY[0], its best rows in the second tile"""
    rng = np.random.default_rng(11)
    hidden = (rng.random(N) < 0.05).astype(np.uint8)
    oi, od = data.first_k(HEAVY[0], N)
    tile1 = oi[(oi >= TILE) & (oi < 2 * TILE)][:150]
    hidden[tile1] = 1
    col = gb.VectorCollection(ctx, 0, gb.DISTANCE_DOT)
    col.add(sparse=data.vecs, hidden=hidden, timestamps=np.full(N, 1000))
    yield col, hidden == 0, tile1
    col.close()


@pytest.mark.parametrize("k", [1, 100, 128])
def test_collection_query(data, collection, k):
    col, allow, tile1 = collection
    rows = query_rows(data)
    rng = np.random.default_rng(k)
    ext = []
    for j, q in enumerate(rows[:24]):   # stored vectors, and variants of them: a feature past every stored one, values scaled
        f, v = data.vecs[q]
        if j % 3 == 1:
            f, v = np.concatenate([f, [F + 5]]).astype(np.uint32), np.concatenate([v, [2.0]]).astype(np.float32)
        elif j % 3 == 2:
            v = (v * np.float32(rng.random() + 0.5)).astype(np.float32)
        ext.append((f, v))
    ext.append((np.zeros(0, np.uint32), np.zeros(0, np.float32)))                        # an empty query
    ext.append((np.array([0], np.uint32), np.array([1.0], np.float32)))                   # the head feature alone
    ext.append((np.arange(0, F, 2, dtype=np.uint32), np.ones(F // 2, np.float32)))        # 15,000 features
    slots, scores, cnt = col.query(ext, (), k)
    for j, vec in enumerate(ext):
        assert_equal(slots[j], scores[j], cnt[j], *data.first_k(-1, k, allow, vec=vec), k, f"query {j}")
    # the hidden rows were the first query's best in the second tile
    if k >= 100:
        oi, _ = data.first_k(HEAVY[0], k)
        assert np.isin(tile1, oi).any()
        got, _, _ = col.query([data.vecs[HEAVY[0]]], (), k)
        assert not np.isin(tile1, got[0]).any()


# ---- the recommenders whose neighbour stage is the sparse search (float values: no ties inside the neighbour lists) ------
@pytest.fixture(scope="module")
def rec(gb, ctx, orc):
    d = Data(orc, False)
    rng = np.random.default_rng(21)
    hidden = (rng.random(N) < 0.05).astype(np.uint8)
    col = gb.VectorCollection(ctx, 0, gb.DISTANCE_DOT)
    ts = rng.integers(0, 1000, N)
    ts[list(HEAVY)], hidden[list(HEAVY)] = 1000, 0   # the heavy rows stay queryable
    col.add(sparse=d.vecs, hidden=hidden, timestamps=ts)
    dead = np.zeros(N, bool)
    dead[col.delete_before(30)] = True
    yield col, i2i.Sparse(d.vecs), hidden, dead, rng, orc
    col.close()


def contexts_with_heavy(rng, hidden, dead, n_users):
    contexts, excludes = i2i.make_users(rng, N, hidden, dead, n_users, max_ctx=4)
    for u in range(0, n_users, 4):
        contexts[u] = np.concatenate([[HEAVY[(u // 4) % len(HEAVY)]], contexts[u]]).astype(np.int64)
    return contexts, excludes


def test_item_to_item(rec):
    col, store, hidden, dead, rng, orc = rec
    contexts, excludes = contexts_with_heavy(rng, hidden, dead, 16)
    rows, _ = col.item_to_item(contexts, excludes, 30)
    want = i2i.expected(orc, store, i2i.allow_mask(hidden, dead, [()] * N), dead, contexts, excludes, 30, 1.0)
    i2i.assert_rows_equal(rows, want)
    assert any(len(r[0]) == 30 for r in rows)


def test_user_to_user(rec):
    col, store, hidden, dead, rng, orc = rec
    slots = np.array(list(HEAVY) + rng.integers(0, N, 10).tolist(), np.int64)
    fb = u2u.make_feedback(rng, N, 500)
    excludes = [rng.choice(500, size=5, replace=False).astype(np.int64) for _ in slots]
    ok = (rng.random(500) > 0.1).astype(np.uint8)
    rows, _ = col.user_to_user(slots, fb, excludes, 30, 500, item_ok=ok)
    want = u2u.expected(orc, u2u.Sparse(store.vecs), u2u.allow_mask(hidden, dead), dead, slots, fb, excludes, 30, 1.0, ok)
    u2u.assert_rows_equal(rows, want)
    assert any(len(r[0]) > 0 for r in rows)


def test_session_recommend(rec):
    col, store, hidden, dead, rng, orc = rec
    contexts, excludes = contexts_with_heavy(rng, hidden, dead, 16)
    nb = sm.oracle_neighbours(orc, store, hidden, dead, 30, 1.0)
    rows, _ = col.session_recommend(contexts, excludes, 30, 3, 40)
    i2i.assert_rows_equal(rows, sm.session_rows(nb, contexts, excludes, 3, 40))
    assert any(len(r[0]) > 0 for r in rows)

