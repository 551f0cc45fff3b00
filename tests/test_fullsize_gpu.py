"""BASELINE.json's FULL sizes, checked through size-independent properties and spot checks against the oracle
(the oracle cannot run whole configs in seconds, so it is used on samples):
  C2  BPR 1M x 100K x 10M, d=64: sampler validity on 10^6 triples, a sampled triple stream applied in order is bit-exact
      vs the oracle on the full tables, one epoch keeps the factors finite and moves hot and cold rows
  C3  eALS at full size lives in tests/test_xl_als_gpu.py
  C4  top-100 over 1M x 128: every row sorted, self-free, k results; 12 rows bit-exact vs the oracle's Bruteforce
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def test_c2_bpr_full_size(gb, orc):
    from gorse_b200 import synth

    U, I, R, d = 1_000_000, 100_000, 10_000_000, 64
    off, items = synth.make_feedback(U, I, R, seed=1000, zipf_s=1.0, exact=True)
    assert off[-1] == R
    rng = np.random.default_rng(0)
    P = (rng.standard_normal((U, d)) * 0.01).astype(np.float32)
    Q = (rng.standard_normal((I, d)) * 0.01).astype(np.float32)
    with gb.Context(0) as ctx, gb.CFModel(ctx, U, I, d, off, items) as m:
        # integer path at full size: every sampled triple is valid, users are uniform
        t = m.bpr_sample_triples(seed=5, first_step=123456789, n=1_000_000)
        u, i, j = t[:, 0].astype(np.int64), t[:, 1].astype(np.int64), t[:, 2].astype(np.int64)
        key = np.sort(np.repeat(np.arange(U, dtype=np.int64), np.diff(off)) * I + items)  # all (u, item) pairs
        assert np.isin(u * I + i, key, assume_unique=False).all()          # i in R_u
        assert not np.isin(u * I + j, key, assume_unique=False).any()      # j not in R_u
        assert j.min() >= 0 and j.max() < I
        cnt = np.bincount(u, minlength=U)
        assert abs(cnt.mean() - 1.0) < 1e-9 and cnt.max() < 12              # uniform over users (model.go:452-458)
        # the oracle's restatement of the sampler agrees on a prefix
        want = orc.bpr_sample_triples(I, off, items, np.arange(U, dtype=np.int32), 5, 123456789, 20000)
        assert t[:20000].tobytes() == want.tobytes()
        # float path at full table size: in-order application == reference with Jobs = 1, bit for bit
        m.set_factors(P, Q)
        m.bpr_apply_triples(t[:20000], 0.05, 0.01, gb.SCATTER_STORE, gb.ORDER_SEQUENTIAL)
        Pg, Qg = m.get_factors()
        Po, Qo = P.copy(), Q.copy()
        orc.bpr_apply_triples(Po, Qo, t[:20000], 0.05, 0.01)
        assert Pg.tobytes() == Po.tobytes() and Qg.tobytes() == Qo.tobytes()
        # one epoch (rounds of 8192 triples): finite, and both the hottest and a cold item moved
        m.set_factors(P, Q)
        m.bpr_epoch(0.05, 0.01, R, 77)
        P1, Q1 = m.get_factors()
    assert np.isfinite(P1).all() and np.isfinite(Q1).all()
    pop = np.bincount(items, minlength=I)
    hot, cold = int(pop.argmax()), int(np.argsort(pop)[I // 2])
    assert not np.array_equal(Q1[hot], Q[hot]) and not np.array_equal(Q1[cold], Q[cold])
    moved = (np.abs(P1 - P).max(axis=1) > 0).mean()
    assert moved > 0.99  # ~every user is drawn ~10 times per epoch


def test_c4_topk_full_size(gb, orc):
    N, d, k, NQ = 1_000_000, 128, 100, 4096
    rng = np.random.default_rng(0)
    X = rng.standard_normal((N, d), dtype=np.float32)
    X /= np.linalg.norm(X, axis=1, keepdims=True)
    with gb.Context(0) as ctx, gb.BruteforceIndex(ctx, d, gb.METRIC_NEG_DOT) as ix:
        ix.add(X)
        idx, dist, cnt = ix.search_range(500_000, 500_000 + NQ, k)
    assert (cnt == k).all()
    assert (np.diff(dist, axis=1) >= 0).all()                                   # ascending distances
    assert not (idx == np.arange(500_000, 500_000 + NQ)[:, None]).any()         # never the query itself
    assert all(len(set(r.tolist())) == k for r in idx[::97])                    # no duplicates
    for q in range(0, NQ, 350):
        oi, od = orc.bruteforce_search(X, X[500_000 + q], k, metric=orc.METRIC_NEG_DOT, self_index=500_000 + q)
        assert dist[q].tobytes() == od.tobytes()
        if idx[q].tolist() != oi.tolist():  # only exact fp32 ties may differ in order
            for v in np.unique(od[od < od[-1]]):
                assert set(idx[q][dist[q] == v].tolist()) == set(oi[od == v].tolist())
