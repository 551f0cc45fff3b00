"""The one dense top-k pipeline (tensor-core sweep, window kernel, exact kernel) behind the brute-force index and the vector
collection's query: the index on the sweep for k above 128, the same answers with the sweep turned off, a k the index could
not answer before, and a batched collection query on the sweep, each against the oracle's brute force."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx(gb):
    c = gb.Context(0)
    yield c
    c.close()


def dataset(rng, N, d):
    X = (rng.standard_normal((N, d)) * 0.5).astype(np.float32)
    X[: N // 10] *= 3   # a popular head, as in trained factors
    X[1:4] = X[0]       # duplicates of row 0: Euclidean distance 0, which prune0 drops
    return X


def assert_like_oracle(gi, gd, oi, od):
    """distances bit-identical to the oracle's; ids identical except for the order of exact fp32 ties (ours: ascending id;
    the oracle's comes from Go's heap) and which tied ids the cut at k keeps"""
    assert len(gi) == len(oi) and gd.tobytes() == od.tobytes()
    assert (np.lexsort((gi, gd)) == np.arange(len(gi))).all()
    for v in np.unique(od)[:-1]:
        assert set(gi[gd == v].tolist()) == set(oi[od == v].tolist())


def check_rows(orc, X, qs, k, prune0, om, got):
    idx, dist, cnt = got
    for r, q in enumerate(qs):
        oi, od = orc.bruteforce_search(X, X[q], k, prune0=prune0, metric=om, self_index=int(q))
        c = cnt[r]
        assert_like_oracle(idx[r, :c], dist[r, :c], oi, od)
        assert (idx[r, c:] == -1).all() and int(q) not in idx[r, :c].tolist()


@pytest.mark.parametrize("prune0", [False, True])
@pytest.mark.parametrize("metric", ["euclid", "negdot"])
@pytest.mark.parametrize("k", [129, 300, 512])
def test_index_on_the_sweep_above_k_128(gb, orc, ctx, k, metric, prune0):
    rng = np.random.default_rng(k)
    N, d, nq = 40000, 64, 64
    X = dataset(rng, N, d)
    gm, om = (gb.METRIC_EUCLIDEAN, orc.METRIC_EUCLIDEAN) if metric == "euclid" else (gb.METRIC_NEG_DOT, orc.METRIC_NEG_DOT)
    with gb.BruteforceIndex(ctx, d, gm) as ix:
        ix.add(X)
        ix.stage1_stats()
        got = ix.search_range(0, nq, k, prune0=prune0)
        ms, flop, _ = ix.stage1_stats()
        assert ms > 0 and flop == 2.0 * nq * N * d   # one sweep answered the call
        check_rows(orc, X, range(nq), k, prune0, om, got)
        qs = rng.choice(N, 64, replace=False).astype(np.int64)
        check_rows(orc, X, qs, k, prune0, om, ix.search_indices(qs, k, prune0=prune0))


@pytest.mark.parametrize("metric", ["euclid", "negdot"])
def test_index_answers_do_not_depend_on_the_path(gb, ctx, monkeypatch, metric):
    rng = np.random.default_rng(3)
    N, d, k = 40000, 128, 100
    X = dataset(rng, N, d)
    Q = rng.standard_normal((96, d)).astype(np.float32)
    qs = rng.choice(N, 80, replace=False).astype(np.int64)
    gm = gb.METRIC_EUCLIDEAN if metric == "euclid" else gb.METRIC_NEG_DOT
    with gb.BruteforceIndex(ctx, d, gm) as ix:
        ix.add(X)

        def answers():
            out = []
            for prune0 in (False, True):
                out += [ix.search_vectors(Q, k, prune0), ix.search_indices(qs, k, prune0), ix.search_range(100, 300, k, prune0)]
            return out

        ix.stage1_stats()
        swept = answers()
        assert ix.stage1_stats()[0] > 0
        monkeypatch.setenv("GORSE_B200_TOPK_EXACT", "1")
        exact = answers()
        assert ix.stage1_stats()[0] == 0
    for a, b in zip(swept, exact):
        for x, y in zip(a, b):
            assert x.tobytes() == y.tobytes()


def test_index_answers_a_k_above_the_old_shared_memory_limit(gb, orc, ctx):
    # d = 16, k = 7000: a warp-per-query list of 7000 entries does not fit in shared memory; the exact kernel sorts in rounds
    rng = np.random.default_rng(5)
    N, d, k = 9000, 16, 7000
    X = dataset(rng, N, d)
    with gb.BruteforceIndex(ctx, d, gb.METRIC_EUCLIDEAN) as ix:
        ix.add(X)
        check_rows(orc, X, [0, 17, N - 1], k, False, orc.METRIC_EUCLIDEAN, ix.search_indices(np.array([0, 17, N - 1], np.int64), k))
        Q = rng.standard_normal((2, d)).astype(np.float32)
        idx, dist, cnt = ix.search_vectors(Q, k)
        for q in range(2):
            oi, od = orc.bruteforce_search(X, Q[q], k, metric=orc.METRIC_EUCLIDEAN)
            assert cnt[q] == k
            assert_like_oracle(idx[q], dist[q], oi, od)


@pytest.mark.parametrize("distance", ["dot", "euclid"])
def test_batched_collection_query_on_the_sweep(gb, orc, ctx, distance):
    rng = np.random.default_rng(9)
    N, d, nq, topk = 40000, 64, 96, 100
    X = dataset(rng, N, d)
    hidden = (rng.random(N) < 0.1).astype(np.uint8)
    gd, om = (gb.DISTANCE_DOT, orc.METRIC_NEG_DOT) if distance == "dot" else (gb.DISTANCE_EUCLIDEAN, orc.METRIC_EUCLIDEAN)
    with gb.VectorCollection(ctx, d, gd) as col:
        col.add(X, hidden=hidden)
        Q = rng.standard_normal((nq, d)).astype(np.float32)
        slots, scores, cnt = col.query(Q, [], topk)
        ids = np.nonzero(hidden == 0)[0]
        Xa = np.ascontiguousarray(X[ids])
        for q in range(0, nq, 3):
            oi, od = orc.bruteforce_search(Xa, Q[q], topk, metric=om)
            assert cnt[q] == topk
            assert_like_oracle(slots[q], -scores[q], ids[oi], od)
