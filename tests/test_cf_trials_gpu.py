"""gorse_b200_cf_fit_trials: the trials of a model search fitted in one call, each as its own solo fit.

BPR trials share every epoch's triples and run in bpr_trials_round_kernel; an epoch with atomic scatter is reproducible
only up to the order of float additions into a row, so BPR trials are held to their solo fits within a tolerance and to
the round model (numpy, round by round) after one epoch.  ALS trials run the solo epoch's kernels on their own tables and
equal their solo fits bit for bit.
"""
import numpy as np
import pytest

from test_bpr_rounds_gpu import rounds_model

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx(gb):
    c = gb.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def clusters(gb):
    """test_fit_gpu.py's planted-cluster set"""
    from gorse_b200 import synth

    U, I = 1200, 300
    off, items = synth.make_feedback(U, I, 24000, seed=4, n_clusters=6)
    train, test = synth.leave_one_out(off, items, seed=1)
    neg = synth.sample_negatives(I, train, test, 100, seed=2)
    ioff, iusers = gb.transpose_csr(train[0], train[1], I)
    return U, I, train, test, neg, ioff, iusers


@pytest.fixture(scope="module")
def zipf():
    """test_bpr_rounds_gpu.py's 50K-user Zipf set, with a user who holds every item (triples without a negative)"""
    from gorse_b200 import synth

    U, I, R = 50_000, 10_000, 500_000
    off, items = synth.make_feedback(U - 1, I, R - I, seed=21, zipf_s=1.0, exact=True)
    items = np.concatenate([items, np.arange(I, dtype=np.int32)])
    off = np.concatenate([off, [off[-1] + I]]).astype(np.int64)
    return U, I, off, items


def solo(gb, ctx, data, d, kind, **kw):
    U, I, train, test, neg, ioff, iusers = data
    with gb.CFModel(ctx, U, I, d, train[0], train[1], ioff, iusers) as m:
        res = m.fit(kind, test[0], test[1], neg[0], neg[1], **kw)
        P, Q = m.get_factors()
    return res, P, Q


def batched(gb, ctx, data, d, trials, progress=None, item_csr=True):
    U, I, train, test, neg, ioff, iusers = data
    with gb.CFModel(ctx, U, I, d, train[0], train[1], *((ioff, iusers) if item_csr else ())) as m:
        return m.fit_trials(trials, test[0], test[1], neg[0], neg[1], progress=progress, factors=True)


def maxdiff(a, b):
    return float(np.abs(a.astype(np.float64) - b).max())


def fields(r):
    return (r.ndcg, r.precision, r.recall, r.epochs_run, r.early_stopped, r.best_epoch, r.cancelled)


@pytest.mark.parametrize("d", [16, 32, 64, 128])
def test_one_epoch_matches_round_model(gb, orc, ctx, zipf, d):
    """each model reads its rows one round stale, neither more nor less; at d = 128 the three models take two launches"""
    U, I, off, items = zipf
    n = int(off[-1])
    hp = [(0.05, 0.01), (0.02, 0.05), (0.08, 0.001)]
    none_off = np.zeros(U + 1, np.int64)
    none = np.zeros(0, np.int32)
    with gb.CFModel(ctx, U, I, d, off, items) as m:
        m.init_normal(0.0, 0.1, 9)
        P0, Q0 = m.get_factors()
        uij = m.bpr_sample_triples(seed=10, first_step=0, n=n)   # epoch 1 of a fit at seed 9
        trials = [("bpr", dict(lr=lr, reg=reg, n_epochs=1, init_stddev=0.1, seed=9)) for lr, reg in hp]
        res, out = m.fit_trials(trials, none_off, none, none_off, none, factors=True)
    assert (uij[:, 2] == -1).any()
    for (lr, reg), r, (Pg, Qg) in zip(hp, res, out):
        assert r.epochs_run == 1 and not r.cancelled
        Pm, Qm = rounds_model(P0, Q0, uij, lr, reg)
        tol = 1e-5 * max(np.abs(Pm).max(), np.abs(Qm).max())
        assert np.isfinite(Pg).all() and np.isfinite(Qg).all()
        assert max(maxdiff(Pg, Pm), maxdiff(Qg, Qm)) <= tol
        Ps, Qs = P0.copy(), Q0.copy()
        orc.bpr_apply_triples(Ps, Qs, uij, lr, reg)
        assert max(maxdiff(Ps, Pg), maxdiff(Qs, Qg)) >= 100 * tol


@pytest.mark.parametrize("d", [16, 32, 64, 128])
def test_bpr_trials_match_solo_fits(gb, orc, ctx, clusters, d):
    U, I, train, test, neg, ioff, iusers = clusters
    lrs, regs = [0.05, 0.02, 0.1], [0.01, 0.03, 0.005]
    kws = [dict(lr=lr, reg=reg, n_epochs=12, verbose=5, seed=3) for lr, reg in zip(lrs, regs)]
    rng = np.random.default_rng(d)
    P0 = rng.standard_normal((U, d)).astype(np.float32)
    Q0 = rng.standard_normal((I, d)).astype(np.float32)
    with gb.CFModel(ctx, U, I, d, train[0], train[1], ioff, iusers) as m:
        m.set_factors(P0, Q0)
        res, out = m.fit_trials([("bpr", kw) for kw in kws], test[0], test[1], neg[0], neg[1], factors=True)
        Pc, Qc = m.get_factors()
    assert Pc.tobytes() == P0.tobytes() and Qc.tobytes() == Q0.tobytes()   # the model's own factors are not touched
    solos = [solo(gb, ctx, clusters, d, "bpr", **kw) for kw in kws]
    for k, (r, (P, Q)) in enumerate(zip(res, out)):
        _, Ps, Qs = solos[k]
        tol = 1e-4 * max(np.abs(Ps).max(), np.abs(Qs).max())
        assert max(maxdiff(P, Ps), maxdiff(Q, Qs)) <= tol, k
        # the neighbouring trial's parameters give another model: swapped parameters cannot pass
        _, Pn, Qn = solos[(k + 1) % len(kws)]
        assert max(maxdiff(P, Pn), maxdiff(Q, Qn)) > 10 * tol, k
        want = orc.evaluate(P, Q, test[0], test[1], neg[0], neg[1], 10)
        assert (r.ndcg, r.precision, r.recall) == tuple(want)
        assert r.epochs_run == 12 and not r.early_stopped and not r.cancelled
    assert res[0].ndcg > 0.15


@pytest.mark.parametrize("d", [16, 64])
def test_mixed_batch_and_als_bit_for_bit(gb, ctx, clusters, d):
    """ALS trials equal their solo fits bit for bit in a batch with BPR trials, which match theirs; n_epochs differ"""
    trials = [("bpr", dict(lr=0.05, reg=0.01, n_epochs=7)), ("als", dict(reg=0.015, alpha=0.05, n_epochs=5)),
              ("bpr", dict(lr=0.02, reg=0.02, n_epochs=4)), ("als", dict(reg=0.06, alpha=0.001, n_epochs=7))]
    for _, kw in trials:
        kw.update(verbose=2, seed=5)
    seen = []
    res, out = batched(gb, ctx, clusters, d, trials, progress=lambda ep, states: seen.append((ep, states)) or False)
    assert [ep for ep, _ in seen] == list(range(1, 8))
    for k, (kind, kw) in enumerate(trials):
        r, (P, Q) = res[k], out[k]
        rs, Ps, Qs = solo(gb, ctx, clusters, d, kind, **kw)
        assert r.epochs_run == kw["n_epochs"] == rs.epochs_run
        if kind == "als":
            assert P.tobytes() == Ps.tobytes() and Q.tobytes() == Qs.tobytes(), k
            assert fields(r) == fields(rs), k
        else:
            assert max(maxdiff(P, Ps), maxdiff(Q, Qs)) <= 1e-4 * max(np.abs(Ps).max(), np.abs(Qs).max()), k
        # the callback: each trial's epochs, its evaluations (every 2 epochs and its last) and when it finished
        n_ep = kw["n_epochs"]
        for ep, states in seen:
            run, ndcg, finished = states[k]
            assert run == min(ep, n_ep) and finished == (ep >= n_ep)
            assert (ndcg >= 0) == (ep <= n_ep and (ep % 2 == 0 or ep == n_ep))


def test_batch_larger_than_one_launch(gb, ctx, clusters):
    """17 BPR trials at d = 16 (16 per launch) and 3 at d = 128 (2 per launch)"""
    for d, n in ((16, 17), (128, 3)):
        kws = [dict(lr=0.01 + 0.005 * k, reg=0.01, n_epochs=3, verbose=3, seed=8) for k in range(n)]
        res, out = batched(gb, ctx, clusters, d, [("bpr", kw) for kw in kws])
        for k in (0, n - 2, n - 1):
            _, Ps, Qs = solo(gb, ctx, clusters, d, "bpr", **kws[k])
            P, Q = out[k]
            assert max(maxdiff(P, Ps), maxdiff(Q, Qs)) <= 1e-4 * max(np.abs(Ps).max(), np.abs(Qs).max()), (d, k)
            assert res[k].epochs_run == 3


def test_early_stop_inside_a_batch(gb, ctx, clusters):
    U, I, train, test, neg, ioff, iusers = clusters
    common = dict(n_epochs=20, verbose=2, patience=4, seed=1)
    trials = [("bpr", dict(lr=0.05, reg=0.01, **common)), ("bpr", dict(lr=0.0, reg=0.0, **common)),
              ("bpr", dict(lr=0.03, reg=0.01, **common))]
    res, out = batched(gb, ctx, clusters, 16, trials)
    rs, _, _ = solo(gb, ctx, clusters, 16, "bpr", **trials[1][1])
    # lr = 0: NDCG never improves on epoch 0, so the trial stops where its solo fit stops, on its initial factors
    assert rs.early_stopped and rs.epochs_run == 6
    assert fields(res[1]) == fields(rs)
    with gb.CFModel(ctx, U, I, 16, train[0], train[1]) as m:
        m.init_normal(0.0, 0.001, 1)
        P0, Q0 = m.get_factors()
    assert out[1][0].tobytes() == P0.tobytes() and out[1][1].tobytes() == Q0.tobytes()
    for k in (0, 2):
        r2, Ps, Qs = solo(gb, ctx, clusters, 16, "bpr", **trials[k][1])
        assert res[k].epochs_run == r2.epochs_run
        assert max(maxdiff(out[k][0], Ps), maxdiff(out[k][1], Qs)) <= 1e-4 * max(np.abs(Ps).max(), np.abs(Qs).max()), k


def test_cancel(gb, ctx, clusters):
    trials = [("als", dict(reg=0.015, alpha=0.05, n_epochs=2)), ("bpr", dict(lr=0.05, n_epochs=10)),
              ("als", dict(reg=0.06, n_epochs=10))]
    for _, kw in trials:
        kw.update(verbose=2, seed=2)
    seen = []

    def progress(ep, states):
        seen.append((ep, states))
        return ep >= 3

    res, _ = batched(gb, ctx, clusters, 16, trials, progress=progress)
    assert [ep for ep, _ in seen] == [1, 2, 3]
    assert [[s[1] >= 0 for s in states] for _, states in seen] == [[False] * 3, [True] * 3, [False] * 3]
    # trial 0 finished at epoch 2 and keeps its result
    rs, _, _ = solo(gb, ctx, clusters, 16, "als", **trials[0][1])
    assert fields(res[0]) == fields(rs) and not res[0].cancelled
    for r in res[1:]:
        assert r.cancelled and r.epochs_run == 3 and (r.ndcg, r.precision, r.recall) == (0.0, 0.0, 0.0)


def test_device_side_argument_errors(gb, ctx, clusters):
    U, I, train, test, neg, ioff, iusers = clusters
    with gb.CFModel(ctx, U, I, 48, train[0], train[1], ioff, iusers) as m:
        with pytest.raises(gb.GorseB200Error) as ei:
            m.fit_trials([("als", {}), ("bpr", {})], test[0], test[1], neg[0], neg[1])
        assert ei.value.status == gb._lib.ERR_UNSUPPORTED and "trial 1" in ei.value.message
    with gb.CFModel(ctx, U, I, 16, train[0], train[1]) as m:
        with pytest.raises(gb.GorseB200Error) as ei:
            m.fit_trials([("bpr", {}), ("als", {})], test[0], test[1], neg[0], neg[1])
        assert ei.value.status == gb._lib.ERR_STATE and "item CSR" in ei.value.message
