"""GPU parity of the eALS ("CCD") epoch against the oracle (model/cf/model.go:641-738) through the C-ABI.
The path is deterministic for any Jobs (each row writes only itself); the GPU sums over a row's feedback
lane-parallel and the Gram matrix block-parallel, so parity is reassociation-limited: tolerance 1e-4 relative
(north_star), measured against the row's largest entry."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx(gb):
    c = gb.Context(0)
    yield c
    c.close()


def rel_err(a, b):
    scale = np.maximum(np.abs(b).max(axis=1, keepdims=True), 1e-12)
    return (np.abs(a - b) / scale).max()


@pytest.mark.parametrize("d,U,I,R", [(16, 400, 150, 6000), (8, 200, 80, 2000), (64, 300, 100, 5000),
                                      (128, 200, 60, 3000), (10, 150, 50, 1500), (160, 60, 40, 900),
                                      (96, 250, 70, 4000), (32, 500, 30, 9000), (128, 2000, 40, 9000)])
def test_one_epoch_matches_oracle(gb, orc, ctx, d, U, I, R):
    from gorse_b200 import synth

    off, items = synth.make_feedback(U, I, R, seed=d)
    # users / items without feedback must still be visited (they get (0-b)/(0+w*S_ff+reg), SURVEY App. A)
    off = np.concatenate([off, [off[-1], off[-1]]]).astype(np.int64)
    U += 2
    ioff, iusers = gb.transpose_csr(off, items, I + 1)
    I += 1
    rng = np.random.default_rng(d)
    P = (rng.standard_normal((U, d)) * 0.1).astype(np.float32)
    Q = (rng.standard_normal((I, d)) * 0.1).astype(np.float32)
    with gb.CFModel(ctx, U, I, d, off, items, ioff, iusers) as m:
        m.set_factors(P, Q)
        m.als_epoch(0.06, 0.001)
        P1, Q1 = m.get_factors()
        m.als_epoch(0.06, 0.001)
        P2, Q2 = m.get_factors()
    Po, Qo = P.copy(), Q.copy()
    orc.als_epoch(Po, Qo, off, items, ioff, iusers, 0.06, 0.001)
    assert rel_err(P1, Po) < 1e-4 and rel_err(Q1, Qo) < 1e-4, (rel_err(P1, Po), rel_err(Q1, Qo))
    orc.als_epoch(Po, Qo, off, items, ioff, iusers, 0.06, 0.001)
    assert rel_err(P2, Po) < 1e-4 and rel_err(Q2, Qo) < 1e-4, (rel_err(P2, Po), rel_err(Q2, Qo))
    assert np.isfinite(P2).all() and not np.array_equal(P1, P)


def check_long_rows(gb, orc, ctx, d):
    # a hot item with thousands of users (no shared-memory staging) next to tiny rows
    from gorse_b200 import synth

    U, I = 3000, 40
    off, items = synth.make_feedback(U, I, 20000, seed=3, zipf_s=1.3)
    ioff, iusers = gb.transpose_csr(off, items, I)
    assert np.diff(ioff).max() > 1500
    rng = np.random.default_rng(0)
    P = (rng.standard_normal((U, d)) * 0.1).astype(np.float32)
    Q = (rng.standard_normal((I, d)) * 0.1).astype(np.float32)
    with gb.CFModel(ctx, U, I, d, off, items, ioff, iusers) as m:
        m.set_factors(P, Q)
        m.als_epoch(0.06, 0.01)
        P1, Q1 = m.get_factors()
    Po, Qo = P.copy(), Q.copy()
    orc.als_epoch(Po, Qo, off, items, ioff, iusers, 0.06, 0.01)
    assert rel_err(P1, Po) < 1e-4 and rel_err(Q1, Qo) < 1e-4, (rel_err(P1, Po), rel_err(Q1, Qo))


def test_long_rows_take_every_row_class(gb, orc, ctx):
    check_long_rows(gb, orc, ctx, 32)


# Below d = 128 the long rows take the Gram form: d = 16 / 10 / 48 check that it updates every coordinate when d is not a
# multiple of 32, d = 10 that the partial stride is padded (10 * 11 floats is not a multiple of 4); d = 160 takes S and the
# long rows above 128.
@pytest.mark.parametrize("d", [16, 10, 48, 160])
def test_long_rows_at_other_d(gb, orc, ctx, d):
    check_long_rows(gb, orc, ctx, d)


def test_deterministic_run_to_run(gb, orc, ctx):
    from gorse_b200 import synth

    off, items = synth.make_feedback(500, 200, 8000, seed=1)
    ioff, iusers = gb.transpose_csr(off, items, 200)
    rng = np.random.default_rng(0)
    P = (rng.standard_normal((500, 16)) * 0.1).astype(np.float32)
    Q = (rng.standard_normal((200, 16)) * 0.1).astype(np.float32)
    outs = []
    for _ in range(2):
        with gb.CFModel(ctx, 500, 200, 16, off, items, ioff, iusers) as m:
            m.set_factors(P, Q)
            m.als_epoch(0.06, 0.001)
            outs.append(m.get_factors())
    assert outs[0][0].tobytes() == outs[1][0].tobytes() and outs[0][1].tobytes() == outs[1][1].tobytes()


def test_full_fit_matches_oracle_ndcg(gb, orc, ctx):
    from gorse_b200 import synth

    U, I, d = 800, 300, 8
    off, items = synth.make_feedback(U, I, 20000, seed=9, n_clusters=6)
    train, test = synth.leave_one_out(off, items, seed=1)
    neg = synth.sample_negatives(I, train, test, 100, seed=2)
    ioff, iusers = gb.transpose_csr(train[0], train[1], I)
    rng = np.random.default_rng(3)
    P0 = (rng.standard_normal((U, d)) * 0.1).astype(np.float32)
    Q0 = (rng.standard_normal((I, d)) * 0.1).astype(np.float32)
    Po, Qo = P0.copy(), Q0.copy()
    for _ in range(10):
        orc.als_epoch(Po, Qo, train[0], train[1], ioff, iusers, 0.015, 0.05)
    want = orc.evaluate(Po, Qo, test[0], test[1], neg[0], neg[1], 10)[0]
    base = orc.evaluate(P0, Q0, test[0], test[1], neg[0], neg[1], 10)[0]
    with gb.CFModel(ctx, U, I, d, train[0], train[1], ioff, iusers) as m:
        m.set_factors(P0, Q0)
        for _ in range(10):
            m.als_epoch(0.015, 0.05)
        got = m.evaluate(test[0], test[1], neg[0], neg[1], 10)[0]
    assert want > base + 0.1 and abs(got - want) < 0.01, (base, want, got)
