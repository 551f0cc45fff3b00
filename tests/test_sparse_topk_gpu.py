"""Sparse searches past 128 neighbours: the wide path of the tiled sparse search (csrc/sparse.cu), which writes each query's
score row and emits it in sorted rounds of 2048, behind gorse_b200_sparse_index_search_range and the sparse collection query.
The data crosses every boundary of the layout: several tiles of 8192 rows plus a remainder, a head feature held by most rows
(the push path), rows of 25,000 features (the pull path), empty rows, and count-valued vectors whose dots tie at the cut and at
the round boundary.  Every answer must equal the oracle's sparse brute force bit for bit -- rows, dot bits and order (dot
desc, row asc) -- with the rows past the count padded with -1 / 0; the first 128 entries must equal the k = 128 answer of the
list path."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

TILE = 8192
N = 3 * TILE + 1234
F = 30000
HEAVY = (5, TILE + 17, 2 * TILE + 4000, 3 * TILE + 600)   # rows with 25,000 features, one in every tile
KS = (129, 2048, 2049, 5000, N)


@pytest.fixture(scope="module")
def ctx(gb):
    c = gb.Context(0)
    yield c
    c.close()


def make_vectors(seed, count_valued):
    """N rows: 0..40 uniform features, the head feature 0 in 70 % of them, every 13th row empty, every 29th row a single
    feature, the HEAVY rows 25,000 features; values 1 (dots count shared features) or positive idf-like floats with a few
    negatives"""
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


class Oracle:
    """the oracle's positive dots of every stored vector with a query, memoised per query: a stored row q (left out of its own
    answer) or an external vector (q = -1)"""

    def __init__(self, orc, vecs):
        self.orc, self.vecs = orc, vecs
        self.off, self.ind, self.val = pack(vecs)
        self.cache = {}

    def dots(self, q, vec=None):
        key = q if vec is None else (vec[0].tobytes(), vec[1].tobytes())
        if key not in self.cache:
            qi, qv = self.vecs[q] if vec is None else vec
            qi, qv = np.ascontiguousarray(qi, np.uint32), np.ascontiguousarray(qv, np.float32)
            n = len(self.vecs)
            oi, od = np.zeros(n, np.int32), np.zeros(n, np.float32)
            m = self.orc.lib().gbo_sparse_bruteforce_search(self.off, self.ind, self.val, n, qi, qv, len(qi), q, n, oi, od)
            keep = od[:m] > 0
            self.cache[key] = (oi[:m][keep].copy(), od[:m][keep].copy())
        return self.cache[key]

    def first_k(self, q, k, allow=None, vec=None):
        """the allowed positive dots in (dot desc, row asc) order, cut at k"""
        oi, od = self.dots(q, vec)
        if allow is not None:
            keep = allow[oi]
            oi, od = oi[keep], od[keep]
        o = np.lexsort((oi, -od.astype(np.float64)))[:k]
        return oi[o], od[o]


@pytest.fixture(scope="module", params=["idf", "count"])
def data(request, orc):
    count_valued = request.param == "count"
    o = Oracle(orc, make_vectors(7 if count_valued else 8, count_valued))
    o.count_valued = count_valued
    return o


def div_up(a, b):
    return (a + b - 1) // b


def query_rows():
    """the heavy rows, the rows around each tile edge, empty and single-feature rows, and a seeded sample"""
    rng = np.random.default_rng(3)
    edges = [e + d for e in range(0, N, TILE) for d in (-1, 0, 1) if 0 <= e + d < N]
    return sorted(set(HEAVY) | set(edges) | {0, 13, 29, 58, N - 1} | set(rng.integers(0, N, 40).tolist()))


def assert_equal(idx, dot, cnt, want_i, want_d, what):
    assert cnt == len(want_i), what
    assert idx[:cnt].tolist() == want_i.tolist(), what
    assert dot[:cnt].tobytes() == want_d.tobytes(), what
    assert (idx[cnt:] == -1).all() and (dot[cnt:] == 0).all(), what


@pytest.fixture(scope="module")
def index(gb, ctx, data):
    """the data in a sparse index, with its k = 128 answer over all rows (the list path)"""
    with gb.SparseIndex(ctx) as ix:
        ix.add(data.off, data.ind, data.val)
        yield ix, ix.search_range(0, N, 128)


def test_data_has_ties_at_the_cuts(data):
    """count-valued dots tie at the round boundary (2048 / 2049) and at k = 129 for many query rows"""
    if not data.count_valued:
        pytest.skip("idf values")
    ties = {129: 0, 2048: 0}
    for q in query_rows():
        _, od = data.first_k(q, N)
        for k in ties:
            ties[k] += len(od) > k and od[k - 1] == od[k]
    assert ties[129] >= 10 and ties[2048] >= 10, ties


@pytest.mark.parametrize("k", KS)
def test_search_range(index, data, k):
    ix, (i128, d128, c128) = index
    ix.stats()
    idx, dot, cnt = ix.search_range(0, N, k)
    st = ix.stats()
    assert idx.shape == (N, k)
    for q in query_rows():
        assert_equal(idx[q], dot[q], cnt[q], *data.first_k(q, k), f"row {q}")
    # rows with fewer positive dots than k are padded; the rest are full
    assert (cnt < k).any() and (cnt == 0).any()
    if k <= 2049:
        assert (cnt == k).any()
    # the first 128 entries are the list path's answer
    assert (np.minimum(cnt, 128) == c128).all()
    assert idx[:, :128].tobytes() == i128.tobytes() and dot[:, :128].tobytes() == d128.tobytes()
    # the score rows of all N queries do not fit one chunk: more tiles walked than one pass over the index has
    assert st["tiles"] > div_up(N, TILE) and st["push"] > 0 and st["pull"] > 0, st
    # a range that starts inside the data, through a heavy row
    q0, q1 = HEAVY[1] - 3, HEAVY[1] + 300
    i2, d2, c2 = ix.search_range(q0, q1, k)
    assert i2.tobytes() == idx[q0:q1].tobytes() and d2.tobytes() == dot[q0:q1].tobytes() and c2.tolist() == cnt[q0:q1].tolist()


def test_search_range_past_the_index_size(index, data):
    """k larger than the index: the answers are the k = N ones, the rest of each row padding"""
    ix, _ = index
    rows = np.array(HEAVY + (13, 100, N - 1), np.int64)
    for q in rows:
        idx, dot, cnt = ix.search_range(int(q), int(q) + 1, 3 * N)
        assert_equal(idx[0], dot[0], cnt[0], *data.first_k(int(q), 3 * N), f"row {q}")


# ---- the collection query -------------------------------------------------------------------------------------------------
class Collection:
    """the data as a sparse collection after a master-style cycle: 5 % hidden, categories {r % 3} (+ 3 on even rows), 300
    rows upserted with scaled values (their old slots tombstoned, the new versions appended), and every 17th row written at
    an old timestamp and deleted by delete_before.  `store` is the oracle over the slots; `allow(cats)` the candidates."""

    def __init__(self, gb, ctx, orc, data):
        rng = np.random.default_rng(11)
        self.col = gb.VectorCollection(ctx, 0, gb.DISTANCE_DOT)
        self.hidden = rng.random(N) < 0.05
        ts = np.full(N, 1000)
        ts[::17] = 10
        self.cats = [[r % 3] + ([3] if r % 2 == 0 else []) for r in range(N)]
        self.col.add(sparse=data.vecs, hidden=self.hidden, timestamps=ts, categories=self.cats)
        up = np.sort(np.concatenate([list(HEAVY), rng.choice(N, 296, replace=False)]))
        up = np.unique(up)
        new = [(data.vecs[r][0], (data.vecs[r][1] * np.float32(1.5)).astype(np.float32)) for r in up]
        first = self.col.add(sparse=new, hidden=np.zeros(len(up), np.uint8), timestamps=np.full(len(up), 2000),
                             categories=[self.cats[r] for r in up], replace=up)
        assert first == N
        self.dead = np.zeros(N + len(up), bool)
        self.dead[up] = True
        self.dead[self.col.delete_before(30)] = True
        assert self.dead[N:].sum() == 0 and self.dead[:N:17].all()
        self.hidden = np.concatenate([self.hidden, np.zeros(len(up), bool)])
        self.cats += [self.cats[r] for r in up]
        self.store = Oracle(orc, list(data.vecs) + new)

    def allow(self, cats=()):
        ok = ~self.dead & ~self.hidden
        for c in cats:
            ok &= np.array([c in cs for cs in self.cats])
        return ok


@pytest.fixture(scope="module")
def collection(gb, ctx, orc, data):
    c = Collection(gb, ctx, orc, data)
    yield c
    c.col.close()


def external_queries(data):
    """stored vectors and variants of them (a feature past every stored one, values scaled), an empty query, the head feature
    alone, and 15,000 features"""
    rng = np.random.default_rng(5)
    ext = []
    for j, q in enumerate(query_rows()[:18]):
        f, v = data.vecs[q]
        if j % 3 == 1:
            f, v = np.concatenate([f, [F + 5]]).astype(np.uint32), np.concatenate([v, [2.0]]).astype(np.float32)
        elif j % 3 == 2:
            v = (v * np.float32(rng.random() + 0.5)).astype(np.float32)
        ext.append((f, v))
    ext.append((np.zeros(0, np.uint32), np.zeros(0, np.float32)))
    ext.append((np.array([0], np.uint32), np.array([1.0], np.float32)))
    ext.append((np.arange(0, F, 2, dtype=np.uint32), np.ones(F // 2, np.float32)))
    return ext


@pytest.mark.parametrize("k", KS)
def test_collection_query(data, collection, k):
    c = collection
    ext = external_queries(data)
    for cats in ((), (3,)):
        allow = c.allow(cats)
        slots, scores, cnt = c.col.query(ext, cats, k)
        for j, vec in enumerate(ext):
            assert_equal(slots[j], scores[j], cnt[j], *c.store.first_k(-1, k, allow, vec=vec), f"query {j}, categories {cats}")
        assert cnt[-3] == 0 and cnt[-2] > 128 and (cnt < k).any()
        # the first 128 entries are the list path's answer
        s128, d128, c128 = c.col.query(ext, cats, 128)
        assert (np.minimum(cnt, 128) == c128).all()
        assert slots[:, :128].tobytes() == s128.tobytes() and scores[:, :128].tobytes() == d128.tobytes()


def test_collection_query_past_the_slot_count(data, collection):
    """topK above every slot: the answers are complete and the rest of each row is padding"""
    c = collection
    ext = external_queries(data)[-4:]
    k = 2 * len(c.dead)
    slots, scores, cnt = c.col.query(ext, (), k)
    for j, vec in enumerate(ext):
        assert_equal(slots[j], scores[j], cnt[j], *c.store.first_k(-1, k, c.allow(), vec=vec), f"query {j}")


def test_collection_query_after_compact(gb, ctx, orc, data):
    """compaction renames the slots and changes no answer"""
    c = Collection(gb, ctx, orc, data)
    try:
        ext = external_queries(data)
        before = {k: c.col.query(ext, (3,), k) for k in (129, 2049, N)}
        new_slot, _, _ = c.col.compact()
        assert c.col.count() == (int((~c.dead).sum()), int((~c.dead).sum()))
        for k, (slots, scores, cnt) in before.items():
            s2, d2, c2 = c.col.query(ext, (3,), k)
            assert c2.tolist() == cnt.tolist(), k
            assert d2.tobytes() == scores.tobytes(), k
            renamed = np.where(slots >= 0, new_slot[np.maximum(slots, 0)], -1)
            assert s2.tolist() == renamed.tolist(), k
    finally:
        c.col.close()
