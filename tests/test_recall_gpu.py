"""Batched CF recall (gorse_b200_vecdb_query_excluding): for many users at once, QueryVectors(topK = n + |E_u|) followed by
dropping E_u, as the worker does per user (worker/pipeline.go:403-449).  Checked against the reference's known answer, the
oracle's brute force, gorse_b200_vecdb_query, itself with the tensor-core sweep turned off, and a BPR model handed off to a
collection."""
import ctypes as C

import numpy as np
import pytest

gpu = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx(gb):
    c = gb.Context(0)
    yield c
    c.close()


def expected(orc, X, allow, Q, excl, n, metric):
    """the oracle's top n + |E_q| over the allowed rows, mapped back to slots, minus E_q"""
    ids = np.nonzero(allow)[0]
    Xa = np.ascontiguousarray(X[ids])
    out = []
    for q in range(Q.shape[0]):
        oi, od = orc.bruteforce_search(Xa, Q[q], n + len(excl[q]), metric=metric)
        drop = set(int(s) for s in excl[q])
        keep = np.array([int(ids[i]) not in drop for i in oi], bool)
        out.append((ids[oi][keep].astype(np.int64), (-od[keep]).astype(np.float32)))
    return out


def assert_rows_equal(got, want):
    """scores bit-identical; slots identical except for the order of exact fp32 ties (and which tied slots a cut keeps)"""
    assert len(got) == len(want)
    for r, ((gs, gv), (ws, wv)) in enumerate(zip(got, want)):
        assert gv.tobytes() == wv.tobytes(), f"row {r}: scores differ"
        if gs.tolist() != ws.tolist():
            vals = np.unique(wv)
            for v in vals[1:]:   # every tie group but the lowest (the one a cut may split) holds the same slots
                assert set(gs[gv == v].tolist()) == set(ws[wv == v].tolist()), f"row {r}"


@gpu
def test_reference_known_answer(gb, ctx):
    # worker/worker_test.go:166-221: items i = 0..9 at (i, 1), the user at (1, 0), items 4..9 excluded, n = 100
    with gb.VectorCollection(ctx, 2, gb.DISTANCE_DOT) as col:
        col.add(np.array([[i, 1] for i in range(10)], np.float32))
        rows, exact = col.query_excluding(np.array([[1, 0]], np.float32), [list(range(4, 10))], 100)
        assert rows[0][0].tolist() == [3, 2, 1, 0] and rows[0][1].tolist() == [3.0, 2.0, 1.0, 0.0]   # the score-0 item stays
        assert exact == 1


def random_collection(gb, ctx, rng, N, d, distance=None):
    X = (rng.standard_normal((N, d)) * 0.5).astype(np.float32)
    X[: N // 10] *= 3   # a popular head: large norms rank high for many users, like trained item factors
    hidden = (rng.random(N) < 0.08).astype(np.uint8)
    ts = rng.integers(0, 1000, N)
    cats = [[int(rng.integers(0, 3))] + ([5] if i % 997 == 0 else []) for i in range(N)]
    col = gb.VectorCollection(ctx, d, gb.DISTANCE_DOT if distance is None else distance)
    col.add(X, hidden=hidden, timestamps=ts, categories=cats)
    dead = np.zeros(N, bool)
    dead[col.delete_before(30)] = True
    return col, X, hidden, dead, cats


def exclusion_lists(orc, rng, X, allow, Q, N, sizes):
    """one list per row: random slots (some hidden or deleted), -1 entries, and adversarial rows that exclude exactly
    their true top 200"""
    ids = np.nonzero(allow)[0]
    excl = []
    for q, m in enumerate(sizes):
        if m == "top200":
            oi, _ = orc.bruteforce_search(np.ascontiguousarray(X[ids]), Q[q], 200, metric=orc.METRIC_NEG_DOT)
            e = ids[oi].astype(np.int64)
        else:
            e = rng.choice(N, size=m, replace=False).astype(np.int64)
            if m >= 4 and q % 3 == 0:
                e[:2] = -1   # ids the collection does not hold
        excl.append(rng.permutation(e))
    return excl


def row_sizes(rng, nq):
    # |E| for n = 100: mostly k <= 128, then each class, above 512, empty rows and adversarial rows
    sizes = [int(x) for x in rng.integers(0, 28, nq)]
    for i in range(0, nq, 16):
        sizes[i] = 0
    for i in range(3, nq, 13):
        sizes[i] = int(rng.integers(29, 156))
    for i in range(5, nq, 29):
        sizes[i] = int(rng.integers(157, 412))
    for i in range(7, nq, 61):
        sizes[i] = int(rng.integers(413, 900))
    for i in range(9, nq, 37):
        sizes[i] = "top200"
    return sizes


@gpu
@pytest.mark.parametrize("N,nq", [(5000, 96), (40000, 512)])
def test_dot_matches_the_oracle(gb, orc, ctx, N, nq):
    rng = np.random.default_rng(N)
    d, n = 64, 100
    col, X, hidden, dead, cats = random_collection(gb, ctx, rng, N, d)
    with col:
        Q = rng.standard_normal((nq, d)).astype(np.float32)
        allow = (hidden == 0) & ~dead
        excl = exclusion_lists(orc, rng, X, allow, Q, N, row_sizes(rng, nq))
        excl[1] = np.unique(np.concatenate([np.nonzero(hidden)[0][:5], np.nonzero(dead)[0][:5]])).astype(np.int64)   # unreachable slots
        rows, exact = col.query_excluding(Q, excl, n)
        assert_rows_equal(rows, expected(orc, X, allow, Q, excl, n, orc.METRIC_NEG_DOT))
        assert [len(r[0]) for r in rows][0] == n   # |E| = 0
        if N >= 32768:
            assert exact < nq // 2, exact   # the tensor-core sweep answered most rows
        # a category filter, and one (category 5) that leaves fewer items than k_q
        for want in ([1], [5]):
            allow_c = allow & np.array([want[0] in c for c in cats])
            rows, _ = col.query_excluding(Q[:64], excl[:64], n, categories=want)
            assert_rows_equal(rows, expected(orc, X, allow_c, Q[:64], excl[:64], n, orc.METRIC_NEG_DOT))
            if want == [5]:
                assert all(len(r[0]) == int(allow_c.sum()) - len(set(excl[i].tolist()) & set(np.nonzero(allow_c)[0].tolist()))
                           for i, r in enumerate(rows))


def cosine_expected(orc, X, allow, Q, excl, n):
    """the collection's Cosine query restated: 1 - q.x / (|q| |x|) with the reference's fp32 dots, ascending, then slot"""
    ids = np.nonzero(allow)[0]
    nx = np.array([np.sqrt(orc.dot(X[i], X[i])) for i in ids], np.float32)
    out = []
    for q in range(Q.shape[0]):
        nq_ = np.sqrt(orc.dot(Q[q], Q[q]))
        dist = np.array([np.float32(1) - orc.dot(Q[q], X[i]) / (nq_ * nx[j]) for j, i in enumerate(ids)], np.float32)
        order = np.lexsort((ids, dist))[: n + len(excl[q])]
        keep = ~np.isin(ids[order], excl[q])
        out.append((ids[order][keep].astype(np.int64), (-dist[order][keep]).astype(np.float32)))
    return out


@gpu
@pytest.mark.parametrize("dist,d", [("euclid", 40), ("cosine", 32)])
def test_euclidean_and_cosine_match_vecdb_query(gb, orc, ctx, dist, d):
    """vecdb_query and query_excluding run one top-k pipeline; a sample of rows is also checked against the oracle (Euclidean)
    or a restatement of the Cosine query"""
    rng = np.random.default_rng(d)
    N, nq, n = 40000, 128, 50
    gd = gb.DISTANCE_EUCLIDEAN if dist == "euclid" else gb.DISTANCE_COSINE
    col, X, hidden, dead, cats = random_collection(gb, ctx, rng, N, d, gd)
    with col:
        Q = rng.standard_normal((nq, d)).astype(np.float32)
        sizes = [0 if i % 8 == 0 else int(rng.integers(1, 300)) for i in range(nq)]
        excl = [rng.choice(N, size=m, replace=False).astype(np.int64) for m in sizes]
        rows, _ = col.query_excluding(Q, excl, n)
        allow = (hidden == 0) & ~dead
        sample = list(range(0, nq, 16))
        if dist == "euclid":
            want = expected(orc, X, allow, Q[sample], [excl[q] for q in sample], n, orc.METRIC_EUCLIDEAN)
        else:
            want = cosine_expected(orc, X, allow, Q[sample], [excl[q] for q in sample], n)
        assert_rows_equal([rows[q] for q in sample], want)
        kmax = n + max(sizes)
        s, sc, cnt = col.query(Q, [], kmax)   # a prefix of the top kmax is the top k_q (one total order)
        for q in range(nq):
            k = n + sizes[q]
            ws, wv = s[q, :min(k, cnt[q])], sc[q, :min(k, cnt[q])]
            keep = ~np.isin(ws, excl[q])
            assert rows[q][0].tolist() == ws[keep].tolist() and rows[q][1].tobytes() == wv[keep].tobytes(), q


@gpu
def test_path_independence_and_repeatability(gb, orc, ctx, monkeypatch):
    rng = np.random.default_rng(7)
    N, nq, d, n = 40000, 256, 64, 100
    col, X, hidden, dead, cats = random_collection(gb, ctx, rng, N, d)
    with col:
        Q = rng.standard_normal((nq, d)).astype(np.float32)
        excl = exclusion_lists(orc, rng, X, (hidden == 0) & ~dead, Q, N, row_sizes(rng, nq))
        a, ea = col.query_excluding(Q, excl, n)
        b, eb = col.query_excluding(Q, excl, n)
        monkeypatch.setenv("GORSE_B200_TOPK_EXACT", "1")
        c, ec = col.query_excluding(Q, excl, n)
        assert ea < nq and ec == nq
        for (sa, va), (sb, vb), (sc_, vc) in zip(a, b, c):
            assert sa.tolist() == sb.tolist() == sc_.tolist()
            assert va.tobytes() == vb.tobytes() == vc.tobytes()


def raw_call(gb, h, Q, off, ex, n=10):
    from gorse_b200 import _lib

    nq = Q.shape[0]
    total = nq * n + int(off[-1])
    slots, scores, cnt = np.zeros(max(total, 1), np.int64), np.zeros(max(total, 1), np.float32), np.zeros(max(nq, 1), np.int32)
    return _lib.lib.gorse_b200_vecdb_query_excluding(h, nq, gb.ptr(Q), None, 0, n, gb.ptr(off), gb.ptr(ex) if ex.size else None,
                                                     gb.ptr(slots), gb.ptr(scores), gb.ptr(cnt), None)


@gpu
def test_errors(gb, ctx):
    from gorse_b200 import _lib

    d = 16
    with gb.VectorCollection(ctx, d, gb.DISTANCE_DOT) as col:
        col.add(np.random.default_rng(0).standard_normal((100, d)).astype(np.float32))
        Q = np.ones((2, d), np.float32)
        off = np.array([0, 2, 3], np.int64)
        assert raw_call(gb, col.h, Q, off, np.array([5, 5, 1], np.int64)) == _lib.ERR_ARG          # a slot twice in one row
        assert b"twice" in _lib.lib.gorse_b200_last_error()
        assert raw_call(gb, col.h, Q, off, np.array([5, -1, -1], np.int64)) == _lib.OK             # -1 may repeat
        assert raw_call(gb, col.h, Q, off, np.array([5, 100, 1], np.int64)) == _lib.ERR_ARG        # not a slot
        assert raw_call(gb, col.h, Q, off, np.array([5, -2, 1], np.int64)) == _lib.ERR_ARG
        assert raw_call(gb, col.h, Q, np.array([1, 2, 3], np.int64), np.array([5, 6, 1], np.int64)) == _lib.ERR_ARG   # excl_off[0] != 0
        Qn = Q.copy()
        Qn[1, 3] = np.nan
        with pytest.raises(gb.GorseB200Error) as ei:   # a NaN score, as in vecdb_query
            col.query_excluding(Qn, [[], []], 10)
        assert ei.value.status == _lib.ERR_ARG
        rows, _ = col.query_excluding(Q, [[1], []], 0)   # n <= 0: nothing
        assert [len(r[0]) for r in rows] == [0, 0]
    with gb.VectorCollection(ctx, 0, gb.DISTANCE_DOT) as col:
        col.add(sparse=[([1, 2], [1.0, 2.0])])
        assert raw_call(gb, col.h, np.ones((1, 2), np.float32), np.array([0, 0], np.int64), np.zeros(0, np.int64)) == _lib.ERR_UNSUPPORTED


def test_null_collection_fails_without_a_device(gb):
    from gorse_b200 import _lib

    Q = np.ones((1, 4), np.float32)
    assert raw_call(gb, None, Q, np.array([0, 0], np.int64), np.zeros(0, np.int64)) == _lib.ERR_ARG
    assert b"NULL" in _lib.lib.gorse_b200_last_error()


@gpu
def test_bpr_hand_off_round_trip(gb, orc, ctx):
    """train, hand the item factors to a collection (master/tasks.go:925-961), recall for every user excluding the training
    rows: the oracle over the downloaded factors gives the same rows"""
    from gorse_b200 import _lib, synth

    U, I, d, n = 600, 400, 32, 20
    off, items = synth.make_feedback(U, 360, 9000, seed=5)   # items 360.. have no feedback: not in the collection
    with gb.CFModel(ctx, U, I, d, off, items) as m, gb.VectorCollection(ctx, d, gb.DISTANCE_DOT) as col:
        m.init_normal(0.0, 0.1, 3)
        for ep in range(5):
            m.bpr_epoch(0.05, 0.01, int(off[-1]), 11 + ep)
        P, Q = m.get_factors()
        slot = np.zeros(I, np.int64)
        gb.check(_lib.lib.gorse_b200_vecdb_add_item_factors(col.h, m.h, None, 0, None, None, gb.ptr(slot)))
        excl = [slot[items[off[u]:off[u + 1]]] for u in range(U)]
        rows, _ = col.query_excluding(P, excl, n)
        present = slot >= 0
        X = np.zeros((int(present.sum()), d), np.float32)
        X[slot[present]] = Q[present]
        assert_rows_equal(rows, expected(orc, X, np.ones(len(X), bool), P, excl, n, orc.METRIC_NEG_DOT))
