"""The round semantics of the atomic-scatter BPR epoch against an independent model.

An epoch with atomic scatter runs its step stream in rounds of 8192 triples: every triple of a round reads its rows as
the previous round left them, and the round's updates are then all added.  The model below applies the same triples
round by round in numpy; only the order of float additions into a row may differ from the GPU.  Applying the triples one
after the other (the oracle, the reference with Jobs = 1) must differ by far more than the tolerance, so that a pipelining
bug that reads a row one round stale, or one that reads a row mid-round, cannot pass.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROUND = 8192
LR, REG = 0.05, 0.01
U, I, R = 50_000, 10_000, 500_000


def rounds_model(P, Q, uij, lr, reg):
    P = P.copy()
    Q = Q.copy()
    lr, reg = np.float32(lr), np.float32(reg)
    for r0 in range(0, len(uij), ROUND):
        t = uij[r0:r0 + ROUND]
        t = t[t[:, 2] >= 0]
        u, i, j = t[:, 0], t[:, 1], t[:, 2]
        p, qi, qj = P[u], Q[i], Q[j]
        diff = (p * qi).sum(1, dtype=np.float32) - (p * qj).sum(1, dtype=np.float32)
        with np.errstate(over="ignore"):
            e = np.exp(-diff)
            g = (e / (np.float32(1) + e))[:, None]
        np.add.at(Q, i, lr * (g * p - reg * qi))
        np.add.at(Q, j, lr * (-g * p - reg * qj))
        np.add.at(P, u, lr * (g * (qi - qj) - reg * p))
    return P, Q


@pytest.fixture(scope="module")
def data():
    from gorse_b200 import synth

    off, items = synth.make_feedback(U - 1, I, R - I, seed=21, zipf_s=1.0, exact=True)
    # one user who holds every item: its triples have no valid negative (j = -1) and update nothing
    items = np.concatenate([items, np.arange(I, dtype=np.int32)])
    off = np.concatenate([off, [off[-1] + I]]).astype(np.int64)
    return off, items


@pytest.fixture(scope="module")
def ctx(gb):
    c = gb.Context(0)
    yield c
    c.close()


@pytest.mark.parametrize("d", [16, 32, 64, 128, 3, 8, 10, 48, 80, 256])
def test_round_epoch_matches_round_model(gb, orc, ctx, data, d):
    off, items = data
    n = int(off[-1])
    assert n % ROUND != 0   # the last round is partial
    rng = np.random.default_rng(d)
    P0 = (rng.standard_normal((U, d)) * 0.1).astype(np.float32)
    Q0 = (rng.standard_normal((I, d)) * 0.1).astype(np.float32)
    with gb.CFModel(ctx, U, I, d, off, items) as m:
        uij = m.bpr_sample_triples(seed=77, first_step=0, n=n)
        m.set_factors(P0, Q0)
        m.bpr_epoch(LR, REG, n, 77, gb.SCATTER_ATOMIC)
        Pg, Qg = m.get_factors()
    assert (uij[:, 2] == -1).any()
    Pm, Qm = rounds_model(P0, Q0, uij, LR, REG)
    Ps, Qs = P0.copy(), Q0.copy()
    orc.bpr_apply_triples(Ps, Qs, uij, LR, REG)
    tol = 1e-5 * max(np.abs(Pm).max(), np.abs(Qm).max())
    for got, model in ((Pg, Pm), (Qg, Qm)):
        assert np.isfinite(got).all()
        assert np.abs(got.astype(np.float64) - model).max() <= tol
    # negative control: the sequential order is told apart by a wide margin
    assert max(np.abs(Ps.astype(np.float64) - Pg).max(), np.abs(Qs.astype(np.float64) - Qg).max()) >= 100 * tol
