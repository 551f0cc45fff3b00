"""Round epochs in sequence, and after every other writer of the factor tables.

test_bpr_rounds_gpu.py checks one atomic-scatter epoch from freshly set factors.  Fit runs many epochs back to back,
and other calls write P and Q between them.  Here every epoch is checked against the numpy round model of
test_bpr_rounds_gpu.py, started from get_factors(): two and three epochs in a row at round counts of either parity, and
an epoch after set_factors, init_normal, bpr_apply_triples, a store-scatter epoch and an eALS epoch.  State that one
epoch call left behind and the next one used without refreshing (a stale copy of a table, or a barrier counter that
is not reset) would make the epoch miss the model by far more than the tolerance.
"""
import numpy as np
import pytest

from test_bpr_rounds_gpu import LR, REG, ROUND, rounds_model

pytestmark = pytest.mark.gpu

U, I, R = 20_000, 5_000, 200_000


@pytest.fixture(scope="module")
def data():
    from gorse_b200 import synth

    off, items = synth.make_feedback(U, I, R, seed=5, zipf_s=1.0, exact=True)
    users = np.repeat(np.arange(U, dtype=np.int32), np.diff(off))
    order = np.argsort(items, kind="stable")
    item_off = np.concatenate([[0], np.cumsum(np.bincount(items, minlength=I))]).astype(np.int64)
    return off, items, item_off, users[order]


@pytest.fixture(scope="module")
def ctx(gb):
    c = gb.Context(0)
    yield c
    c.close()


def steps(n_rounds):
    return (n_rounds - 1) * ROUND + 1000   # a partial last round


def check_epoch(gb, m, n, seed, lr=LR):
    P0, Q0 = m.get_factors()
    uij = m.bpr_sample_triples(seed=seed, first_step=0, n=n)
    m.bpr_epoch(lr, REG, n, seed, gb.SCATTER_ATOMIC)
    Pg, Qg = m.get_factors()
    Pm, Qm = rounds_model(P0, Q0, uij, lr, REG)
    tol = 1e-5 * max(np.abs(Pm).max(), np.abs(Qm).max())
    for got, model in ((Pg, Pm), (Qg, Qm)):
        assert np.isfinite(got).all()
        assert np.abs(got.astype(np.float64) - model).max() <= tol


def start(d, seed=0):
    rng = np.random.default_rng(seed)
    return ((rng.standard_normal((U, d)) * 0.1).astype(np.float32),
            (rng.standard_normal((I, d)) * 0.1).astype(np.float32))


@pytest.mark.parametrize("epochs", [2, 3])
@pytest.mark.parametrize("n_rounds", [5, 6])
@pytest.mark.parametrize("d", [16, 64, 128, 8, 48])
def test_back_to_back_epochs(gb, ctx, data, d, n_rounds, epochs):
    off, items, _, _ = data
    with gb.CFModel(ctx, U, I, d, off, items) as m:
        m.set_factors(*start(d))
        for e in range(epochs):
            check_epoch(gb, m, steps(n_rounds), 100 + e)


@pytest.mark.parametrize("writer", ["set_factors", "init_normal", "bpr_apply_triples", "store_epoch", "als_epoch"])
def test_epoch_after_other_writer(gb, ctx, data, writer):
    off, items, item_off, item_users = data
    d, n = 64, steps(5)
    lr = LR
    with gb.CFModel(ctx, U, I, d, off, items, item_off, item_users) as m:
        m.set_factors(*start(d))
        m.bpr_epoch(LR, REG, n, 1, gb.SCATTER_ATOMIC)
        if writer == "set_factors":
            m.set_factors(*start(d, seed=7))
        elif writer == "init_normal":
            m.init_normal(0.0, 0.1, 3)
        elif writer == "bpr_apply_triples":
            m.bpr_apply_triples(m.bpr_sample_triples(seed=9, first_step=0, n=20_000), LR, REG)
        elif writer == "store_epoch":
            m.bpr_epoch(LR, REG, n, 2, gb.SCATTER_STORE)
        else:
            m.als_epoch(0.06, 0.001)
            # eALS leaves factors up to ~5, 50 times the others here; at lr = 0.05 the order of the float additions
            # alone then moves the epoch ~1.4e-5 of the largest factor away from the model
            lr = LR / 10
        check_epoch(gb, m, n, 4, lr)
