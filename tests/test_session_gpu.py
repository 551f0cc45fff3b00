"""Batched session recommendation (gorse_b200_vecdb_session_recommend): for many sessions at once, what the REST server's
session recommendation does per request (server/rest.go:1069-1173).  Checked against the reference's known answer, the
Python restatement of the handler (session_model.py) over the oracle's neighbour query, gorse_b200_vecdb_item_to_item,
itself with the tensor-core sweep turned off, and its limits."""
import numpy as np
import pytest

import session_model as sm
from test_item_to_item_gpu import assert_rows_equal, dense_collection, make_users, sparse_collection

gpu = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx(gb):
    c = gb.Context(0)
    yield c
    c.close()


def collection(gb, ctx, rng, kind, N, d=32):
    if kind == "sparse":
        return sparse_collection(gb, ctx, rng, N)
    return dense_collection(gb, ctx, rng, N, d, gb.DISTANCE_EUCLIDEAN)


def item_masks(rng, N):
    holes = (rng.random(N) >= 0.08).astype(np.uint8)    # about 8 % of the items fail the filter
    sparse = (rng.random(N) < 0.04).astype(np.uint8)    # most lists are emptied and do not count
    return {"none": None, "ones": np.ones(N, np.uint8), "holes": holes, "sparse": sparse}


@gpu
def test_reference_known_answer(gb, ctx):
    # server/rest_test.go:1803-1886: a tags collection, ContextSize 4, n = 3; "1".."5" exist only as vectors, "100" is
    # hidden; category "*" holds "7" and "9"
    vecs = [([0], [1.0]), ([1], [1.0]), ([2], [1.0]), ([3], [1.0]), ([4], [1.0]), ([3], [1.0]), ([2, 3], [1.0, 1.0]), ([1, 2, 3], [1.0] * 3),
            ([0, 1, 2, 3], [1.0] * 4), ([0], [100.0])]
    with gb.VectorCollection(ctx, 0, gb.DISTANCE_DOT) as col:
        col.add(sparse=vecs, hidden=[0] * 9 + [1])
        ok = np.zeros(10, np.uint8)
        ok[5:9] = 1
        ctx_s, ex_s = [[0, 1, 2, 3, 4]], [[0, 1, 2, 3, 4]]
        rows, st = col.session_recommend(ctx_s, ex_s, 100, 4, 3, item_ok=ok)
        assert rows[0][0].tolist() == [8, 7, 6] and rows[0][1].tolist() == [4.0, 3.0, 2.0]
        rows, _ = col.session_recommend(ctx_s, ex_s, 100, 4, 100 + 3, item_ok=ok)   # offset 100: nothing past it
        assert len(rows[0][0]) == 4
        ok_star = np.zeros(10, np.uint8)
        ok_star[[6, 8]] = 1
        rows, _ = col.session_recommend(ctx_s, ex_s, 100, 4, 3, item_ok=ok_star)
        assert rows[0][0].tolist() == [8, 6] and rows[0][1].tolist() == [4.0, 2.0]


@gpu
@pytest.mark.parametrize("kind,scale", [("euclid", 1.0), ("euclid", 0.5), ("sparse", 1.0), ("sparse", 0.5)])
def test_matches_the_restatement(gb, orc, ctx, kind, scale):
    rng = np.random.default_rng(61 if kind == "euclid" else 62)
    N, n = 3000, 20
    col, store, hidden, dead, _ = collection(gb, ctx, rng, kind, N)
    with col:
        contexts, excludes = make_users(rng, N, hidden, dead, 96)
        nb = sm.oracle_neighbours(orc, store, hidden, dead, n, scale)
        for name, ok in item_masks(rng, N).items():
            for context_size in (1, 3, 100):
                for top in (5, n, 3 * n):
                    rows, _ = col.session_recommend(contexts, excludes, n, context_size, top, item_ok=ok, score_scale=scale)
                    want = sm.session_rows(nb, contexts, excludes, context_size, top, ok)
                    assert_rows_equal(rows, want)
                    assert all(len(r[0]) <= top for r in rows)
            # the cut is observable: a larger context_size changes some rows
            a, _ = col.session_recommend(contexts, excludes, n, 1, n, item_ok=ok, score_scale=scale)
            b, _ = col.session_recommend(contexts, excludes, n, 100, n, item_ok=ok, score_scale=scale)
            assert any(x[0].tolist() != y[0].tolist() for x, y in zip(a, b)), name
        # top above the candidate count: every candidate
        rows, _ = col.session_recommend(contexts, excludes, n, 100, 1024, score_scale=scale)
        assert any(0 < len(r[0]) < 1024 for r in rows) and max(len(r[0]) for r in rows) < 1024


@gpu
@pytest.mark.parametrize("kind", ["euclid", "sparse"])
def test_equals_item_to_item_without_the_filter_and_the_cut(gb, ctx, kind):
    rng = np.random.default_rng(71)
    N, n = 3000, 25
    col, _, hidden, dead, _ = collection(gb, ctx, rng, kind, N)
    with col:
        contexts, excludes = make_users(rng, N, hidden, dead, 80)
        want, _ = col.item_to_item(contexts, excludes, n)
        got, _ = col.session_recommend(contexts, excludes, n, max(len(c) for c in contexts), n)
        for (gs, gv), (ws, wv) in zip(got, want):
            assert gs.tolist() == ws.tolist() and gv.tobytes() == wv.tobytes()


@gpu
@pytest.mark.parametrize("kind", ["euclid", "sparse"])
def test_both_accumulators(gb, orc, ctx, kind):
    rng = np.random.default_rng(81)
    N, n = 2500, 50
    col, store, hidden, dead, _ = collection(gb, ctx, rng, kind, N, d=16)
    with col:
        # |C_s| * n above the shared-memory table for every third session
        contexts, excludes = make_users(rng, N, hidden, dead, 30, heavy=(150, 300))
        nb = sm.oracle_neighbours(orc, store, hidden, dead, n, 1.0)
        ok = item_masks(rng, N)["holes"]
        for context_size in (2, 400):
            rows, st = col.session_recommend(contexts, excludes, n, context_size, n, item_ok=ok)
            assert st["shared_sessions"] > 0 and st["global_sessions"] > 0, st
            assert st["shared_sessions"] + st["global_sessions"] == 30
            assert_rows_equal(rows, sm.session_rows(nb, contexts, excludes, context_size, n, ok))


@gpu
@pytest.mark.parametrize("kind", ["euclid", "sparse"])
def test_repeatable_and_path_independent(gb, ctx, monkeypatch, kind):
    rng = np.random.default_rng(91)
    N, n = 40000 if kind == "euclid" else 4000, 40
    col, _, hidden, dead, _ = collection(gb, ctx, rng, kind, N)
    with col:
        contexts, excludes = make_users(rng, N, hidden, dead, 200, heavy=(200,))
        ok = item_masks(rng, N)["holes"]
        a, sa = col.session_recommend(contexts, excludes, n, 10, 30, item_ok=ok)
        b, _ = col.session_recommend(contexts, excludes, n, 10, 30, item_ok=ok)
        monkeypatch.setenv("GORSE_B200_TOPK_EXACT", "1")
        c, sc = col.session_recommend(contexts, excludes, n, 10, 30, item_ok=ok)
        if kind == "euclid":
            assert sa["exact_rows"] < sa["context_items"] and sc["exact_rows"] == sc["context_items"]
        for (ga, va), (gb_, vb), (gc, vc) in zip(a, b, c):
            assert ga.tolist() == gb_.tolist() == gc.tolist()
            assert va.tobytes() == vb.tobytes() == vc.tobytes()


@gpu
def test_single_session(gb, orc, ctx):
    rng = np.random.default_rng(95)
    N, n = 3000, 20
    col, store, hidden, dead, _ = collection(gb, ctx, rng, "euclid", N)
    with col:
        contexts, excludes = make_users(rng, N, hidden, dead, 8)
        nb = sm.oracle_neighbours(orc, store, hidden, dead, n, 1.0)
        for c, e in zip(contexts, excludes):
            rows, _ = col.session_recommend([c], [e], n, 5, 10)
            assert_rows_equal(rows, sm.session_rows(nb, [c], [e], 5, 10))


def raw_call(gb, h, ctx_lists, ex_lists, n=10, top=10, context_size=100):
    from gorse_b200 import _lib

    ns = len(ctx_lists)
    co = np.concatenate([[0], np.cumsum([len(x) for x in ctx_lists])]).astype(np.int64)
    cs = np.asarray([x for l in ctx_lists for x in l], np.int64)
    eo = np.concatenate([[0], np.cumsum([len(x) for x in ex_lists])]).astype(np.int64)
    es = np.asarray([x for l in ex_lists for x in l], np.int64)
    m = max(top, 1)
    slots, scores, cnt = np.zeros(ns * m + 1, np.int64), np.zeros(ns * m + 1, np.float64), np.zeros(ns + 1, np.int32)
    return _lib.lib.gorse_b200_vecdb_session_recommend(h, ns, gb.ptr(co), gb.ptr(cs) if cs.size else None, gb.ptr(eo), gb.ptr(es) if es.size else None,
                                                       None, n, context_size, top, 1.0, gb.ptr(slots), gb.ptr(scores), gb.ptr(cnt), None)


@gpu
def test_limits(gb, ctx):
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
        assert raw_call(gb, col.h, [[1]], [[]], n=0) == _lib.ERR_UNSUPPORTED
        assert raw_call(gb, col.h, [[1]], [[]], top=1025) == _lib.ERR_UNSUPPORTED
        assert raw_call(gb, col.h, [[1]], [[]], top=1024) == _lib.OK
        assert raw_call(gb, col.h, [[1, 100]], [[]]) == _lib.ERR_ARG                      # not a slot
        assert raw_call(gb, col.h, [[1]], [[100]]) == _lib.ERR_ARG
        rows, _ = col.session_recommend([[1, 2], []], [[], []], 10, 5, 0)                  # top <= 0: nothing
        assert [len(r[0]) for r in rows] == [0, 0]
        with pytest.raises(ValueError):
            col.session_recommend([[1]], [[]], 10, 5, 10, item_ok=np.ones(99, np.uint8))
        Xn = X[:2].copy()
        Xn[1, 3] = np.nan
        col.add(Xn)
        with pytest.raises(gb.GorseB200Error) as ei:                                      # a NaN score, as in vecdb_query
            col.session_recommend([[100]], [[]], 10, 5, 10)
        assert ei.value.status == _lib.ERR_ARG
