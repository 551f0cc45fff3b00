"""The tensor-core stage of the brute-force search (csrc/topk_mma.cu): wgmma GEMM + fused threshold filter, then the
exact re-rank.  Results must equal the oracle's ann.Bruteforce bit for bit (indices AND distances), like the exact
scan; the dense stage-1 scores are checked against a bf16 matmul to validate descriptors / swizzle / accumulator layout."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx(gb):
    c = gb.Context(0)
    yield c
    c.close()


def assert_same_neighbours(idx, dist, oi, od):
    """Distances bit-exact and ascending; ids identical wherever a distance is unique.  Exact fp32 ties (they do occur among
    4*10^4 candidates) may come out in a different order: the reference's tie order is an artefact of Go's heap that no
    reference test pins, ours is (distance, index).  Ids strictly inside the k-th distance must match as sets."""
    assert dist.tobytes() == od.tobytes()
    if idx.tolist() == oi.tolist():
        return
    last = od[-1]
    for v in np.unique(od):
        ours, theirs = set(idx[dist == v].tolist()), set(oi[od == v].tolist())
        if v < last:
            assert ours == theirs, (v, ours, theirs)
        else:
            assert len(ours) == len(theirs)


def bf16_round(x):
    u = x.astype(np.float32).view(np.uint32).astype(np.uint64)
    u = (u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000
    return u.astype(np.uint32).view(np.float32)


@pytest.mark.parametrize("metric,d", [("negdot", 128), ("negdot", 64), ("euclid", 64), ("negdot", 40)])
def test_stage1_scores_match_bf16_matmul(gb, ctx, metric, d):
    N = 33000
    rng = np.random.default_rng(d)
    X = rng.standard_normal((N, d)).astype(np.float32)
    X /= np.linalg.norm(X, axis=1, keepdims=True)
    gm = gb.METRIC_EUCLIDEAN if metric == "euclid" else gb.METRIC_NEG_DOT
    with gb.BruteforceIndex(ctx, d, gm) as ix:
        ix.add(X)
        got = ix.stage1_scores(100, 400)
    Xb = bf16_round(X).astype(np.float64)
    want = Xb[100:400] @ Xb.T
    if metric == "euclid":
        want = want - 0.5 * (X.astype(np.float64) ** 2).sum(1)[None, :]
    acc_err = 0.0
    assert np.abs(got - want).max() < 2e-3 + acc_err, np.abs(got - want).max()
    # and the error bound the filter relies on: |stage-1 score - exact| <= eps = (1.02 * 2^-8 [+ n_mma * 2^-11]) * |q| * max|x|
    exact = X[100:400].astype(np.float64) @ X.astype(np.float64).T
    if metric == "euclid":
        exact = exact - 0.5 * (X.astype(np.float64) ** 2).sum(1)[None, :]
    assert np.abs(got - exact).max() <= 1.02 / 256 + acc_err


@pytest.mark.parametrize("metric,d,k", [("negdot", 128, 100), ("euclid", 64, 100), ("negdot", 64, 10), ("euclid", 128, 37)])
def test_tensor_path_equals_oracle(gb, orc, ctx, metric, d, k):
    N, NQ = 40000, 300
    rng = np.random.default_rng(d + k)
    X = rng.standard_normal((N, d)).astype(np.float32)
    if metric == "negdot":
        X /= np.linalg.norm(X, axis=1, keepdims=True)  # cosine via -dot on unit vectors (BASELINE config 4)
    gm = gb.METRIC_EUCLIDEAN if metric == "euclid" else gb.METRIC_NEG_DOT
    om = orc.METRIC_EUCLIDEAN if metric == "euclid" else orc.METRIC_NEG_DOT
    with gb.BruteforceIndex(ctx, d, gm) as ix:
        ix.add(X)
        idx, dist, cnt = ix.search_range(1000, 1000 + NQ, k)       # all-pairs form (self excluded)
        fb = ix.stage1_stats()[2]
        qv = rng.standard_normal((128, d)).astype(np.float32)
        idx2, dist2, cnt2 = ix.search_vectors(qv, k, prune0=(metric == "euclid"))
    assert fb <= 3, f"{fb} of {NQ} rows needed the exact fallback"
    oi, od, oc, _ = orc.bruteforce_all(X, 1000, 1000 + NQ, k, metric=om, n_threads=8)
    assert cnt.tolist() == oc.tolist()
    n_same = 0
    for r in range(NQ):
        assert_same_neighbours(idx[r, :cnt[r]], dist[r, :cnt[r]], oi[r, :oc[r]], od[r, :oc[r]])
        n_same += idx[r].tolist() == oi[r].tolist()
    assert n_same >= NQ - 10  # ties are rare
    for q in range(0, 128, 9):
        oi, od = orc.bruteforce_search(X, qv[q], k, prune0=(metric == "euclid"), metric=om)
        assert cnt2[q] == len(oi)
        assert_same_neighbours(idx2[q, :cnt2[q]], dist2[q, :cnt2[q]], oi, od)


def test_adversarial_inputs_fall_back_exactly(gb, orc, ctx):
    # many exact duplicates (ties at the k-th place) and wildly varying norms: the filter must stay sound
    N, d, k = 33000, 64, 20
    rng = np.random.default_rng(1)
    X = rng.standard_normal((N, d)).astype(np.float32)
    X[::3] = X[0]                      # 11000 identical vectors
    X[1::3] *= rng.uniform(0.01, 50, size=(len(X[1::3]), 1)).astype(np.float32)
    with gb.BruteforceIndex(ctx, d, gb.METRIC_NEG_DOT) as ix:
        ix.add(X)
        idx, dist, cnt = ix.search_range(0, 96, k)
    for q in range(0, 96, 7):
        oi, od = orc.bruteforce_search(X, X[q], k, metric=orc.METRIC_NEG_DOT, self_index=q)
        assert dist[q].tobytes() == od.tobytes()          # same distance multiset, ascending
        assert sorted(zip(od.tolist(), oi.tolist()))[0][0] == dist[q][0]
        strict = od < od[-1]                               # members strictly inside the k-th distance are pinned
        assert set(oi[strict].tolist()) <= set(idx[q].tolist())
