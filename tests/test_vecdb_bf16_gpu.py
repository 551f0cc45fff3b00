"""bf16 storage of dense vector collections (gorse_b200_vecdb_create, gorse_b200_vecdb_storage): a collection whose values are
all bf16-exact keeps its rows at 2 bytes a value and answers every entry exactly as its fp32 twin -- the same slots, tie order
and score bits, the same stored bits and the same snapshot stream.  The twin holds the same vectors in fp32: it is built from
them plus one vector that is not bf16-exact, added last with an older timestamp, then deleted and compacted away.  Also: the
promotion to fp32 by add, add_item_factors and load (in a later staging chunk too), and bit patterns kept exactly."""
import io
import struct
import types

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

DISTANCES = ("DOT", "EUCLIDEAN", "COSINE")
DIMS = (16, 64, 128, 200, 1024, 3072)   # 200: the one-thread (dist_any) scan; 16 .. 128: the quad scan; 1024, 3072: wide rows
N_Q, N_USERS = 48, 64
HEADER = struct.Struct("<8sIiiIqqq")
INEXACT = np.float32(1.0) + np.float32(2.0 ** -20)   # low 16 bits not zero


def exact(x):
    """x truncated to bf16: the low 16 bits cleared"""
    return (np.ascontiguousarray(x, np.float32).view(np.uint32) & np.uint32(0xFFFF0000)).view(np.float32)


def tie_heavy(rng, n, dim):
    """bf16-exact values: small multiples of 1/2 (exact scores, many ties) mixed with truncated normals, and repeated rows"""
    v = (rng.integers(-2, 3, (n, dim)) * 0.5).astype(np.float32)
    wild = rng.random((n, dim)) < 0.25
    v[wild] = exact(rng.standard_normal(int(wild.sum())))[:]
    dup = rng.random(n) < 0.2
    v[dup] = v[rng.integers(0, n, int(dup.sum()))]
    v[np.all(v == 0, axis=1), 0] = 1.0   # no zero rows (Cosine)
    return v


@pytest.fixture(scope="module")
def ctx(gb):
    c = gb.Context(0)
    yield c
    c.close()


def build_pair(gb, ctx, dim, dist, X, rng):
    """the bf16 collection and its fp32 twin, written alike; -> (bf16, twin, meta)"""
    n = len(X)
    meta = dict(hidden=rng.random(n) < 0.05, timestamps=rng.integers(1000, 3000, n),
                categories=[np.flatnonzero(rng.random(3) < 0.5).tolist() for _ in range(n)])
    d = getattr(gb, "DISTANCE_" + dist)
    a, b = gb.VectorCollection(ctx, dim, d), gb.VectorCollection(ctx, dim, d)
    assert a.add(X, **meta) == b.add(X, **meta) == 0
    odd = exact(rng.standard_normal(dim))
    odd[0] = INEXACT
    assert b.add(odd[None], timestamps=[10]) == n
    assert b.storage()[0] == 4
    assert np.array_equal(b.delete_before(11), [n])
    new_slot = b.compact()[0]
    assert np.array_equal(new_slot[:n], np.arange(n)) and new_slot[n] == -1
    return a, b, meta


def workload(rng, X, n_ids):
    n = len(X)
    dim = X.shape[1]

    def pick(k):
        s = rng.integers(0, n, k)
        s[rng.random(k) > 0.93] = -1
        return s

    def ids(k):
        s = rng.integers(0, n_ids, k)
        s[rng.random(k) > 0.9] = -1
        return s

    w = types.SimpleNamespace(n_ids=n_ids)
    w.q = (rng.integers(-2, 3, (N_Q, dim)) * 0.5).astype(np.float32)
    w.q[: N_Q // 4] = X[rng.integers(0, n, N_Q // 4)]   # stored rows as queries: exact ties at the top
    w.excl = [np.unique(pick(int(rng.integers(0, 12)))) for _ in range(N_Q)]
    w.ctx = [pick(int(rng.integers(1, 8))) for _ in range(N_USERS)]
    w.ex = [np.unique(pick(int(rng.integers(0, 10)))) for _ in range(N_USERS)]
    w.user_slots = pick(N_USERS)
    w.fb = [rng.integers(0, n_ids, int(rng.integers(0, 6))) for _ in range(n)]
    w.ex_items = [np.unique(ids(int(rng.integers(0, 8)))) for _ in range(N_USERS)]
    w.item_ok = (rng.random(n_ids) > 0.1).astype(np.uint8)
    w.slot_ok = (rng.random(n) > 0.1).astype(np.uint8)
    w.ctx_items = [ids(int(rng.integers(1, 8))) for _ in range(N_USERS)]
    w.item_live = (rng.random(n_ids) > 0.05).astype(np.uint8)
    w.soi = np.full(n_ids, -1, np.int64)
    w.ios = np.full(n, -1, np.int32)
    for s in range(min(n, n_ids)):
        w.soi[s], w.ios[s] = s, s
    return w


def rows_of(slots, scores, cnt):
    return [(slots[q, :c].copy(), scores[q, :c].copy()) for q, c in enumerate(cnt)]


def answers(gb, ctx, col, w, recommenders=True):
    out = {"query": rows_of(*col.query(w.q, (), 20)), "query_categories": rows_of(*col.query(w.q, (1,), 20)),
           "query_excluding": col.query_excluding(w.q, w.excl, 15, categories=(0,))[0]}
    if col.distance == gb.DISTANCE_COSINE or not recommenders:   # the batched recommenders refuse Cosine
        return out
    out["item_to_item"] = col.item_to_item(w.ctx, w.ex, 10, categories=(0,))[0]
    out["session_recommend"] = col.session_recommend(w.ctx, w.ex, 10, 3, 15, item_ok=w.slot_ok)[0]
    out["user_to_user"] = col.user_to_user(w.user_slots, w.fb, w.ex_items, 10, w.n_ids, w.item_ok)[0]
    stages = [gb.ItemToItemStage(col, 10, w.ctx_items, w.soi, w.ios, score_scale=0.5), gb.UserToUserStage(col, 10, w.user_slots, w.fb, w.item_ok)]
    out["recommend"] = gb.recommend(ctx, w.ex_items, w.n_ids, w.item_live, stages)[0]
    return out


def assert_same(a, b):
    assert a.keys() == b.keys()
    for name in a:
        assert len(a[name]) == len(b[name]), name
        for (s0, v0), (s1, v1) in zip(a[name], b[name]):
            assert np.array_equal(s0, s1), name   # the same slots in the same (tie) order
            assert np.asarray(v0).tobytes() == np.asarray(v1).tobytes(), name   # the same score bits


def ties(rows):
    return sum(int(np.sum(v[1:] == v[:-1])) for _, v in rows)


def stream(col):
    buf = io.BytesIO()
    col.save(buf)
    return buf.getvalue()


def stored(col):
    live, slots = col.count()
    vals, hid, ts, alive = col.get(np.arange(slots + 2, dtype=np.int64) - 1)   # slots -1 and `slots` are not live
    return (live, slots), vals.tobytes(), hid.tobytes(), ts.tobytes(), alive.tobytes()


def check_twins(gb, ctx, a, b, X, w):
    assert a.storage()[0] == 2 and b.storage()[0] == 4
    assert stored(a) == stored(b)
    assert np.array_equal(a.get(np.arange(len(X)))[0].view(np.uint32), X.view(np.uint32))
    assert stream(a) == stream(b)
    ra, rb = answers(gb, ctx, a, w), answers(gb, ctx, b, w)
    assert_same(ra, rb)
    assert ties(ra["query"]) > 0
    return ra


@pytest.mark.parametrize("dist", DISTANCES)
@pytest.mark.parametrize("dim", DIMS)
def test_bf16_collection_answers_as_its_fp32_twin(gb, ctx, dim, dist):
    rng = np.random.default_rng(dim * 7 + len(dist))
    n = 1500 if dim >= 1024 else 3000
    X = tie_heavy(rng, n, dim)
    a, b, meta = build_pair(gb, ctx, dim, dist, X, rng)
    try:
        # rows: exactly half the twin's bytes (capacity = n after one add / a compaction); the bf16 collection also holds its
        # upload staging (at most 64 MB of fp32 rows), which the twin released when it was promoted
        (va, da), (vb, db) = a.storage(), b.storage()
        stage = min(n, (64 << 20) // (4 * dim)) * dim * 4
        assert (va, vb) == (2, 4) and db - da == n * dim * 2 - stage
        w = workload(rng, X, n + 50)
        check_twins(gb, ctx, a, b, X, w)
        # the same deletes and compaction on both: the same tombstones, maps and answers; a stays bf16
        assert np.array_equal(a.delete_before(1500), b.delete_before(1500))
        ma, mb = a.compact(), b.compact()
        # compaction releases the staging: the rest of the two is alike
        assert np.array_equal(ma[0], mb[0]) and mb[2] - ma[2] == (int(ma[0].max()) + 1) * dim * 2
        live = np.flatnonzero(ma[0] >= 0)
        w = workload(rng, X[live], n + 50)
        check_twins(gb, ctx, a, b, X[live], w)
        # a snapshot of the bf16 collection loads as bf16 and answers alike
        c = gb.VectorCollection.load(ctx, io.BytesIO(stream(a)))
        try:
            assert c.storage()[0] == 2
            assert stored(c) == stored(a)
            assert_same(answers(gb, ctx, c, w), answers(gb, ctx, a, w))
        finally:
            c.close()
    finally:
        a.close()
        b.close()


@pytest.mark.parametrize("exact_scan", [False, True])
@pytest.mark.parametrize("dist", ("DOT", "EUCLIDEAN"))
def test_tensor_core_sweep_and_exact_scan(gb, ctx, monkeypatch, dist, exact_scan):
    """d = 128, 32 768+ vectors, 64 query rows: the tensor-core sweep serves the bf16 collection and its twin alike (and the
    exact scan with GORSE_B200_TOPK_EXACT=1)"""
    if exact_scan:
        monkeypatch.setenv("GORSE_B200_TOPK_EXACT", "1")
    rng = np.random.default_rng(128 + exact_scan)
    n = 33000
    X = tie_heavy(rng, n, 128)
    a, b, _ = build_pair(gb, ctx, 128, dist, X, rng)
    try:
        w = workload(rng, X, n)
        w.q, w.excl = np.concatenate([w.q, w.q[:16]]), w.excl + w.excl[:16]   # 64 rows
        assert len(w.q) == 64
        check_twins(gb, ctx, a, b, X, w)
    finally:
        a.close()
        b.close()


def test_empty_and_sparse_storage(gb, ctx):
    with gb.VectorCollection(ctx, 64, gb.DISTANCE_DOT) as d, gb.VectorCollection(ctx, 0, gb.DISTANCE_DOT) as s:
        assert d.storage()[0] == 2 and s.storage()[0] == 0
        s.add(sparse=[(np.array([1, 5], np.uint32), np.array([0.3, 0.7], np.float32))])
        assert s.storage()[0] == 0
        # an empty collection promotes for free
        d.add(np.full((3, 64), INEXACT, np.float32))
        assert d.storage()[0] == 4


def test_promotion_by_add(gb, ctx):
    """40 000 bf16 rows, then one vector that is not bf16-exact: the collection becomes fp32, its earlier answers stay, and it
    answers as a collection that held the same vectors in fp32 from the start"""
    rng = np.random.default_rng(40000)
    n, dim = 40000, 64
    X = tie_heavy(rng, n, dim)
    odd = exact(rng.standard_normal(dim))
    odd[3] = INEXACT
    w = workload(rng, X, n)
    with gb.VectorCollection(ctx, dim, gb.DISTANCE_EUCLIDEAN) as a, gb.VectorCollection(ctx, dim, gb.DISTANCE_EUCLIDEAN) as ref:
        a.add(X, timestamps=np.full(n, 100))
        assert a.storage()[0] == 2
        before = answers(gb, ctx, a, w, recommenders=False)
        a.add(odd[None], timestamps=[50])
        assert a.storage()[0] == 4
        ref.add(np.concatenate([X, odd[None]]), timestamps=np.concatenate([np.full(n, 100), [50]]))
        assert ref.storage()[0] == 4
        assert stored(a) == stored(ref) and stream(a) == stream(ref)
        assert_same(answers(gb, ctx, a, w, recommenders=False), answers(gb, ctx, ref, w, recommenders=False))
        a.delete_before(100)   # the inexact vector goes; the collection stays fp32
        assert a.storage()[0] == 4
        assert_same(answers(gb, ctx, a, w, recommenders=False), before)
        a.compact()
        assert a.storage()[0] == 4
        assert_same(answers(gb, ctx, a, w, recommenders=False), before)


def test_promotion_by_add_item_factors(gb, ctx):
    from gorse_b200 import _lib, synth

    U, I, d = 300, 200, 32
    off, items = synth.make_feedback(U, I, 4000, seed=3)
    with gb.CFModel(ctx, U, I, d, off, items) as m:
        m.init_normal(0.0, 0.1, 3)
        P, Q = m.get_factors()
        slot = np.zeros(I, np.int64)
        with gb.VectorCollection(ctx, d, gb.DISTANCE_DOT) as col:   # ordinary factors: fp32
            gb.check(_lib.lib.gorse_b200_vecdb_add_item_factors(col.h, m.h, None, 0, None, None, gb.ptr(slot)))
            assert col.storage()[0] == 4
            got = col.get(slot[slot >= 0])[0]
            assert np.array_equal(got.view(np.uint32), Q[slot >= 0].view(np.uint32))
        m.set_factors(P, exact(Q))
        with gb.VectorCollection(ctx, d, gb.DISTANCE_DOT) as col, gb.VectorCollection(ctx, d, gb.DISTANCE_DOT) as twin:
            gb.check(_lib.lib.gorse_b200_vecdb_add_item_factors(col.h, m.h, None, 0, None, None, gb.ptr(slot)))
            assert col.storage()[0] == 2   # factors truncated to bf16: stays bf16
            gb.check(_lib.lib.gorse_b200_vecdb_add_item_factors(twin.h, m.h, None, 0, None, None, gb.ptr(slot)))
            present = slot >= 0
            assert np.array_equal(col.get(slot[present])[0].view(np.uint32), exact(Q)[present].view(np.uint32))
            twin.add(np.full((1, d), INEXACT, np.float32), timestamps=[-1])
            twin.delete_before(0)
            twin.compact()
            assert stream(col) == stream(twin)
            q = exact(P[:64])
            excl = [slot[items[off[u]:off[u + 1]]] for u in range(64)]
            assert_same({"r": col.query_excluding(q, excl, 10)[0]}, {"r": twin.query_excluding(q, excl, 10)[0]})


@pytest.fixture(scope="module")
def wide_stream(gb, ctx):
    """a bf16-exact stream of 40 000 x 1024 values: 164 MB, three 64 MB staging chunks on load"""
    rng = np.random.default_rng(1024)
    n, dim = 40000, 1024
    X = exact(rng.standard_normal((n, dim)).astype(np.float32))
    with gb.VectorCollection(ctx, dim, gb.DISTANCE_DOT) as col:
        col.add(X, timestamps=np.arange(n))
        s = stream(col)
    _, _, d, _, _, n_s, _, ncat = HEADER.unpack_from(s)
    assert (d, n_s) == (dim, n) and 4 * n * dim > 2 * (64 << 20)
    return types.SimpleNamespace(X=X, s=s, values=len(s) - 4 * n * dim)


def test_load_exact_stream_is_bf16(gb, ctx, wide_stream):
    with gb.VectorCollection.load(ctx, io.BytesIO(wide_stream.s)) as col:
        assert col.storage()[0] == 2
        assert np.array_equal(col.get(np.arange(len(wide_stream.X)))[0].view(np.uint32), wide_stream.X.view(np.uint32))
        assert stream(col) == wide_stream.s


@pytest.mark.parametrize("row", [0, 17000, 39999])   # the first, second and last (third) staging chunk
def test_load_promotes_at_the_first_inexact_value(gb, ctx, wide_stream, row):
    dim = wide_stream.X.shape[1]
    X = wide_stream.X.copy()
    X[row, 5] = INEXACT
    s = bytearray(wide_stream.s)
    s[wide_stream.values:] = X.tobytes()
    with gb.VectorCollection.load(ctx, io.BytesIO(bytes(s))) as col:
        assert col.storage()[0] == 4
        assert np.array_equal(col.get(np.arange(len(X)))[0].view(np.uint32), X.view(np.uint32))
        assert stream(col) == bytes(s)
        assert col.query(X[row:row + 1], (), 5)[2][0] == 5 and dim == 1024


def test_bit_patterns_survive(gb, ctx):
    bits = np.array([0x00000000, 0x80000000, 0x7F800000, 0xFF800000,    # +-0, +-Inf
                     0x00010000, 0x807F0000, 0x00400000, 0x80010000,    # bf16 subnormals
                     0x7FC10000, 0xFFA50000, 0x7F810000, 0xFFFF0000,    # NaNs with payloads in the high half
                     0x3F800000, 0xC2480000, 0x01000000, 0x7F7F0000], np.uint32)
    X = np.stack([np.roll(bits, k) for k in range(4)]).view(np.float32)
    with gb.VectorCollection(ctx, 16, gb.DISTANCE_DOT) as col:
        col.add(X)
        assert col.storage()[0] == 2
        assert np.array_equal(col.get(np.arange(4))[0].view(np.uint32), X.view(np.uint32))
        s = stream(col)
        assert s[-X.nbytes:] == X.tobytes()
        with gb.VectorCollection.load(ctx, io.BytesIO(s)) as back:
            assert back.storage()[0] == 2
            assert np.array_equal(back.get(np.arange(4))[0].view(np.uint32), X.view(np.uint32))
