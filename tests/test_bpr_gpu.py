"""GPU parity of the BPR path against the oracle (model/cf/model.go:408-540), through the C-ABI.

  level 1  bit-exact: Predict; one conflict-free batch with SCATTER_STORE; arbitrary triple streams with
           ORDER_SEQUENTIAL (= the reference with Jobs=1 on that stream)
  level 1' SCATTER_ATOMIC within 1e-5 relative (north_star tolerance: 1e-4 relative on fp32 factors)
  integer  the on-device sampler == the oracle's restatement of it, bit for bit; validity of every triple
  level 3  a full multi-epoch fit reaches the oracle fit's NDCG@10 within 0.01
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

DIMS = [16, 64, 128, 32, 8, 10, 24, 40, 256]


def make(U=300, I=120, R=3000, d=16, seed=0, std=0.1, clusters=0):
    from gorse_b200 import synth

    off, items = synth.make_feedback(U, I, R, seed=seed, n_clusters=clusters)
    rng = np.random.default_rng(seed + 100)
    P = (rng.standard_normal((U, d)) * std).astype(np.float32)
    Q = (rng.standard_normal((I, d)) * std).astype(np.float32)
    return off, items, P, Q


@pytest.fixture(scope="module")
def ctx(gb):
    c = gb.Context(0)
    yield c
    c.close()


@pytest.mark.parametrize("d", DIMS)
def test_predict_bit_exact(gb, orc, ctx, d):
    off, items, P, Q = make(d=d, std=1.0)
    with gb.CFModel(ctx, 300, 120, d, off, items) as m:
        m.set_factors(P, Q)
        rng = np.random.default_rng(1)
        us = rng.integers(0, 300, 500).astype(np.int32)
        its = rng.integers(0, 120, 500).astype(np.int32)
        got = m.predict(us, its)
        want = np.array([orc.dot(P[u], Q[i]) for u, i in zip(us, its)], np.float32)
        assert got.tobytes() == want.tobytes()
        P2, Q2 = m.get_factors()
        assert P2.tobytes() == P.tobytes() and Q2.tobytes() == Q.tobytes()


@pytest.mark.parametrize("d", DIMS)
def test_conflict_free_batch_store_bit_exact(gb, orc, ctx, d):
    from gorse_b200 import synth

    off, items, P, Q = make(d=d, std=0.5)
    t = synth.conflict_free_triples(off, items, 120, 50, seed=3)
    assert len(t) >= 20
    with gb.CFModel(ctx, 300, 120, d, off, items) as m:
        m.set_factors(P, Q)
        m.bpr_apply_triples(t, 0.05, 0.01, gb.SCATTER_STORE, gb.ORDER_HOGWILD)
        Pg, Qg = m.get_factors()
    Po, Qo = P.copy(), Q.copy()
    orc.bpr_apply_triples(Po, Qo, t, 0.05, 0.01)
    assert Pg.tobytes() == Po.tobytes()
    assert Qg.tobytes() == Qo.tobytes()
    assert not np.array_equal(Po, P)


@pytest.mark.parametrize("d", [16, 64, 10])
def test_conflict_free_batch_atomic_within_tolerance(gb, orc, ctx, d):
    from gorse_b200 import synth

    off, items, P, Q = make(d=d, std=0.5)
    t = synth.conflict_free_triples(off, items, 120, 50, seed=4)
    with gb.CFModel(ctx, 300, 120, d, off, items) as m:
        m.set_factors(P, Q)
        m.bpr_apply_triples(t, 0.05, 0.01, gb.SCATTER_ATOMIC, gb.ORDER_HOGWILD)
        Pg, Qg = m.get_factors()
    Po, Qo = P.copy(), Q.copy()
    orc.bpr_apply_triples(Po, Qo, t, 0.05, 0.01)
    np.testing.assert_allclose(Pg, Po, rtol=1e-5, atol=1e-7)
    np.testing.assert_allclose(Qg, Qo, rtol=1e-5, atol=1e-7)


@pytest.mark.parametrize("d", [16, 64, 128, 8])
def test_sequential_order_equals_reference_jobs1_bit_exact(gb, orc, ctx, d):
    # an arbitrary (conflicting) triple stream applied in order == model.go:448-490 with Jobs = 1
    off, items, P, Q = make(U=60, I=30, R=500, d=d, std=0.3)
    with gb.CFModel(ctx, 60, 30, d, off, items) as m:
        m.set_factors(P, Q)
        t = m.bpr_sample_triples(seed=11, first_step=0, n=2000)
        m.bpr_apply_triples(t, 0.05, 0.01, gb.SCATTER_STORE, gb.ORDER_SEQUENTIAL)
        Pg, Qg = m.get_factors()
    Po, Qo = P.copy(), Q.copy()
    orc.bpr_apply_triples(Po, Qo, t, 0.05, 0.01)
    assert Pg.tobytes() == Po.tobytes() and Qg.tobytes() == Qo.tobytes()


def test_sampler_matches_oracle_and_is_valid(gb, orc, ctx):
    off, items, P, Q = make(U=400, I=150, R=6000, d=16, seed=5)
    # a user with every item (no valid negative) and users without feedback
    full = np.arange(150, dtype=np.int32)
    items = np.concatenate([items, full])
    off = np.concatenate([off, [off[-1] + 150, off[-1] + 150, off[-1] + 150]]).astype(np.int64)
    U = len(off) - 1
    active = np.nonzero(np.diff(off) > 0)[0].astype(np.int32)
    with gb.CFModel(ctx, U, 150, 16, off, items) as m:
        got = m.bpr_sample_triples(seed=1234, first_step=77, n=20000)
    want = orc.bpr_sample_triples(150, off, items, active, 1234, 77, 20000)
    assert got.tobytes() == want.tobytes()
    for u, i, j in got[:3000]:
        row = items[off[u]:off[u + 1]]
        assert len(row) > 0 and i in row
        assert (j == -1 and len(row) == 150) or (j >= 0 and j not in row)
    assert (got[:, 2] == -1).sum() > 0
    # distribution: users uniform over the active ones (model.go:452-458)
    cnt = np.bincount(got[:, 0], minlength=U)[active]
    exp = 20000 / len(active)
    assert abs(cnt.mean() - exp) < 1e-9 and cnt.std() < 3 * np.sqrt(exp)


def test_init_normal_statistics(gb, orc, ctx):
    # the reference's own RNG tests are statistical (common/util/random_test.go:25-62): mean/std within tolerance
    off, items, P, Q = make(U=2000, I=500, R=8000, d=16)
    with gb.CFModel(ctx, 2000, 500, 16, off, items) as m:
        m.init_normal(1.0, 2.0, 42)
        P1, Q1 = m.get_factors()
        m.init_normal(1.0, 2.0, 42)
        P2, Q2 = m.get_factors()
        m.init_normal(1.0, 2.0, 43)
        P3, _ = m.get_factors()
    assert P1.tobytes() == P2.tobytes() and Q1.tobytes() == Q2.tobytes() and P1.tobytes() != P3.tobytes()
    for X in (P1, Q1):
        assert abs(X.mean() - 1.0) < 0.1 and abs(X.std() - 2.0) < 0.1
    assert abs(np.corrcoef(P1[:500].ravel(), Q1.ravel())[0, 1]) < 0.05


def test_argument_errors(gb, orc, ctx):
    off, items, P, Q = make()
    with gb.CFModel(ctx, 300, 120, 16, off, items) as m:
        with pytest.raises(gb.GorseB200Error) as e:
            m.bpr_apply_triples(np.array([[0, 500, 1]], np.int32), 0.05, 0.01)
        assert e.value.status == -1
        with pytest.raises(gb.GorseB200Error):
            m.predict(np.array([300], np.int32), np.array([0], np.int32))
        m.bpr_apply_triples(np.zeros((0, 3), np.int32), 0.05, 0.01)  # empty input is fine
        with pytest.raises(gb.GorseB200Error) as e:
            m.als_epoch(0.06, 0.001)  # no item CSR
        assert e.value.status == -6
    bad_off = off.copy()
    bad_off[5] = bad_off[4] - 1
    with pytest.raises(gb.GorseB200Error):
        gb.CFModel(ctx, 300, 120, 16, bad_off, items)


def ndcg_of(orc, P, Q, test, neg):
    return orc.evaluate(P, Q, test[0], test[1], neg[0], neg[1], 10)[0]


def test_full_fit_matches_oracle_ndcg(gb, orc, ctx):
    # level 3: planted-cluster data; GPU Hogwild epochs (SCATTER_ATOMIC: no update is lost) vs oracle sequential
    # epochs from the same init.  SCATTER_STORE is the parity mode: with ~10^4 triples in flight on a 400-item
    # table its racy read-modify-write loses most updates (measured NDCG 0.07 vs 0.49), exactly as the
    # reference's lock-free goroutines would at that concurrency, so it is not the training default.
    scatter = "atomic"
    from gorse_b200 import synth

    U, I, d = 1500, 400, 16
    off, items = synth.make_feedback(U, I, 30000, seed=9, n_clusters=8)
    train, test = synth.leave_one_out(off, items, seed=1)
    neg = synth.sample_negatives(I, train, test, 100, seed=2)
    rng = np.random.default_rng(3)
    P0 = (rng.standard_normal((U, d)) * 0.001).astype(np.float32)
    Q0 = (rng.standard_normal((I, d)) * 0.001).astype(np.float32)
    n_steps, epochs, lr, reg = int(train[0][-1]), 30, 0.05, 0.01
    active = np.nonzero(np.diff(train[0]) > 0)[0].astype(np.int32)
    Po, Qo = P0.copy(), Q0.copy()
    for ep in range(epochs):
        t = orc.bpr_sample_triples(I, train[0], train[1], active, 1000 + ep, 0, n_steps)
        orc.bpr_apply_triples(Po, Qo, t, lr, reg)
    base = ndcg_of(orc, P0, Q0, test, neg)
    want = ndcg_of(orc, Po, Qo, test, neg)
    assert want > base + 0.1, (base, want)
    with gb.CFModel(ctx, U, I, d, train[0], train[1]) as m:
        m.set_factors(P0, Q0)
        for ep in range(epochs):
            m.bpr_epoch(lr, reg, n_steps, 1000 + ep, gb.SCATTER_ATOMIC if scatter == "atomic" else gb.SCATTER_STORE)
        Pg, Qg = m.get_factors()
        got_dev = m.evaluate(test[0], test[1], neg[0], neg[1], 10)[0]
    got = ndcg_of(orc, Pg, Qg, test, neg)
    assert np.isfinite(Pg).all() and np.isfinite(Qg).all()
    assert abs(got - want) < 0.01, (base, want, got)
    assert got_dev == got  # device Evaluate == oracle Evaluate on the same factors


@pytest.mark.parametrize("d", [64, 128])
def test_atomic_epochs_repeat_up_to_rounding(gb, ctx, d):
    """Epochs with atomic scatter run in rounds whose triples read the rows the previous round left: the same factors and
    seeds give the same factors on every run, except for the order of float additions into a row that several triples of
    one round update.  Zipf(1) data with many rounds per epoch and a heavy popularity head."""
    from gorse_b200 import synth

    U, I, R = 200_000, 20_000, 2_000_000
    off, items = synth.make_feedback(U, I, R, seed=d, zipf_s=1.0, exact=True)
    rng = np.random.default_rng(d)
    P0 = (rng.standard_normal((U, d)) * 0.01).astype(np.float32)
    Q0 = (rng.standard_normal((I, d)) * 0.01).astype(np.float32)
    runs = []
    for _ in range(2):
        with gb.CFModel(ctx, U, I, d, off, items) as m:
            m.set_factors(P0, Q0)
            for ep in range(3):
                m.bpr_epoch(0.05, 0.01, R, 500 + ep, gb.SCATTER_ATOMIC)
            runs.append(m.get_factors())
    (P1, Q1), (P2, Q2) = runs
    assert not np.array_equal(Q1, Q0)
    for a, b in ((P1, P2), (Q1, Q2)):
        assert np.isfinite(a).all()
        assert np.abs(a.astype(np.float64) - b).max() <= 1e-5 * np.abs(a).max()
