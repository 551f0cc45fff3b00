"""gorse_b200_fm_fit_trials: every trial of a batched call equals its own solo gorse_b200_fm_fit / _fit_emb call bit for bit --
parameters, both Adam moments, every result field and the sequence of progress states -- for the slot-free model and
models with slots, trials that leave early (n_epochs, patience, divergence), one trial, several groups, cancels, plain
launches, and against the CPU restatement (fm_oracle) for the first steps."""
import numpy as np
import pytest

import fm_oracle

pytestmark = pytest.mark.gpu

RESULT_FIELDS = ("auc", "precision", "recall", "accuracy", "cost", "epochs_run", "best_epoch", "early_stopped", "diverged", "cancelled", "steps")


@pytest.fixture(scope="module")
def ctx(gb):
    with gb.Context(0) as c:
        yield c


def same(a, b):
    """bitwise, every NaN counting as one value (NaN payloads are not pinned)"""
    a, b = np.array(a, np.float32), np.array(b, np.float32)
    a[np.isnan(a)] = np.nan
    b[np.isnan(b)] = np.nan
    return a.tobytes() == b.tobytes()


def solo(gb, ctx, nf, nd, tr, te, p0, emb, kw, cancel_at=None):
    seq = []

    def prog(ep, n, auc):
        seq.append((ep, auc))
        return cancel_at is not None and ep == cancel_at

    t = gb.FMTrainer(ctx, nf, nd, **kw)
    if emb is None:
        out = t.fit(tr, te, p0, progress=prog, moments=True)
    else:
        out = t.fit_emb(tr, te, p0, emb.dims, emb.table, emb.mask, emb.train_rows, emb.test_rows, progress=prog, moments=True)
    return out, seq


def batched(gb, ctx, nf, nd, tr, te, pins, emb, base, trials, cancel_at=None):
    calls = []

    def prog(ep, states):
        calls.append((ep, states))
        return cancel_at is not None and ep == cancel_at

    e = None if emb is None else (emb.dims, emb.table, emb.mask, emb.train_rows, emb.test_rows)
    out = gb.FMTrainer(ctx, nf, nd, **base).fit_trials(trials, tr, te, pins, emb=e, progress=prog, moments=True)
    return out, calls


def trial_seq(calls, i):
    """trial i's (epoch, auc) as the callback saw it while the trial was in the batch"""
    seq = []
    for ep, states in calls:
        run, auc, fin = states[i]
        if (ep == 0 and auc != -1.0) or (ep > 0 and run == ep):
            seq.append((ep, auc))
            if fin:
                break
    return seq


def assert_same(g, o, what):
    (pg, rg, mg), (po, ro, mo) = g, o
    assert same(pg, po), (what, "params", int(np.sum(pg.view(np.uint32) != po.view(np.uint32))))
    assert same(mg, mo), (what, "moments")
    for f in RESULT_FIELDS:
        assert same([rg[f]], [ro[f]]), (what, f, rg[f], ro[f])


def check_all(gb, ctx, nf, nd, tr, te, pins, emb, base, trials, cancel_at=None, solo_cancel=None):
    out, calls = batched(gb, ctx, nf, nd, tr, te, pins, emb, base, trials, cancel_at)
    assert len(out) == len(trials)
    for i, (over, p0) in enumerate(zip(trials, pins)):
        ref, seq = solo(gb, ctx, nf, nd, tr, te, p0, emb, {**base, **over}, solo_cancel(i) if solo_cancel else cancel_at)
        assert_same(out[i], ref, f"trial {i}")
        got = trial_seq(calls, i)
        assert [e for e, _ in got] == [e for e, _ in seq] and same([a for _, a in got], [a for _, a in seq]), (i, got, seq)
    return out, calls


def ctr(seed, nf, n_train, n_test, everywhere=None):
    rng = np.random.default_rng(seed)
    tr = fm_oracle.random_ctr(rng, nf, n_train)
    te = fm_oracle.random_ctr(rng, nf, n_test)
    if everywhere is not None:   # one feature in every training row
        off, idx, val, tgt = tr
        idx = idx.copy()
        idx[off[:-1] + 1] = everywhere
        tr = (off, idx, val, tgt)
    return rng, tr, te


MIXED = [dict(lr=0.01), dict(lr=0.003, reg=0.01), dict(lr=0.05, optimizer=1), dict(lr=0.02, reg=0.001, optimizer=1), dict(lr=0.001, reg=0.0)]


@pytest.mark.parametrize("k", [8, 16, 32])
def test_slot_free_trials_equal_their_solo_fits(gb, ctx, k):
    nf = 203
    rng, tr, te = ctr(k, nf, 2100, 400, everywhere=7)   # batches of 300: a partial last batch
    pins = [fm_oracle.init_params(rng, nf, k, s) for s in (0.1, 0.05, 0.2, 0.1, 0.01)]
    base = dict(n_factors=k, n_epochs=3, batch_size=300, verbose=1, patience=0)
    check_all(gb, ctx, nf, 6, tr, te, pins, None, base, MIXED)


def test_feature_indices_above_2_24(gb, ctx):
    nf, k = (1 << 24) + 64, 8
    rng = np.random.default_rng(6)
    tr, te = fm_oracle.random_ctr(rng, 1 << 20, 500), fm_oracle.random_ctr(rng, 1 << 20, 100)
    for off, idx, _, _ in (tr, te):
        m = rng.random(idx.size) < 0.5
        m[off[:-1]] = False
        idx[m] = rng.integers((1 << 24) - 40, (1 << 24) + 60, int(m.sum()))
    pins = []
    for s in (0.1, 0.05):
        p0 = np.zeros(1 + nf * k + nf, np.float32)
        p0[1:] = (rng.standard_normal(nf * k + nf) * s).astype(np.float32)
        pins.append(p0)
    base = dict(n_factors=k, n_epochs=2, batch_size=128, verbose=1, patience=0, max_steps=5)
    check_all(gb, ctx, nf, 6, tr, te, pins, None, base, [dict(lr=0.01), dict(lr=0.03, optimizer=1)])


@pytest.mark.parametrize("dims,bs", [((24,), 7), ((5, 24, 64), 16)])
def test_slot_trials_equal_their_solo_fits(gb, ctx, dims, bs):
    nf, k = 120, 8
    rng = np.random.default_rng(len(dims))
    tr, te = fm_oracle.random_ctr(rng, nf, 150), fm_oracle.random_ctr(rng, nf, 60)
    emb = fm_oracle.random_embeddings(rng, 40, dims, 150, 60)   # absent embeddings: masked slots and row -1
    assert (emb.train_rows == -1).any() and (emb.mask == 0).any()
    pins = [fm_oracle.init_params(rng, nf, k, s, dims) for s in (0.1, 0.3, 0.05)]
    base = dict(n_factors=k, n_epochs=2, batch_size=bs, verbose=1, patience=0)
    check_all(gb, ctx, nf, 5, tr, te, pins, emb, base, MIXED[:3])


def test_trials_that_leave(gb, ctx):
    nf, k = 120, 8
    rng, tr, te = ctr(8, nf, 1500, 500)
    pins = [fm_oracle.init_params(rng, nf, k, 0.1) for _ in range(5)]
    pins[4][1 + 3] = np.inf          # a non-finite row 0 read by every padded position
    trials = [dict(lr=0.01, n_epochs=2), dict(lr=0.01, n_epochs=5), dict(lr=0.0, n_epochs=6), dict(lr=0.02, n_epochs=6),
              dict(lr=50.0, n_epochs=6)]
    base = dict(n_factors=k, batch_size=100, verbose=1, patience=2)
    out, _ = check_all(gb, ctx, nf, 6, tr, te, pins, None, base, trials)
    assert out[0][1]["epochs_run"] == 2
    assert out[2][1]["early_stopped"] == 1   # lr 0: the AUC never improves
    assert out[4][1]["diverged"] == 1


def test_one_trial_equals_the_solo_entry(gb, ctx):
    nf, k = 150, 16
    rng, tr, te = ctr(9, nf, 900, 200)
    check_all(gb, ctx, nf, 4, tr, te, [fm_oracle.init_params(rng, nf, k, 0.1)], None,
              dict(n_factors=k, n_epochs=3, batch_size=128, verbose=2, patience=0), [dict(lr=0.01)])


def test_several_groups(gb, ctx):
    nf, k = 60, 8
    rng, tr, te = ctr(10, nf, 200, 80)
    n = 17                            # one more than a group holds
    pins = [fm_oracle.init_params(rng, nf, k, 0.05 + 0.01 * i) for i in range(n)]
    trials = [dict(lr=0.002 * (i + 1), optimizer=i % 2, n_epochs=1 + i % 3) for i in range(n)]
    _, calls = check_all(gb, ctx, nf, 5, tr, te, pins, None, dict(n_factors=k, batch_size=64, verbose=1, patience=0), trials)
    assert sum(1 for ep, _ in calls if ep == 0) == 2


@pytest.mark.parametrize("at", [0, 2])
def test_cancel(gb, ctx, at):
    nf, k = 80, 8
    rng, tr, te = ctr(11, nf, 600, 100)
    pins = [fm_oracle.init_params(rng, nf, k, 0.1) for _ in range(3)]
    trials = [dict(lr=0.01, n_epochs=1), dict(lr=0.02, n_epochs=5), dict(lr=0.005, optimizer=1, n_epochs=5)]
    base = dict(n_factors=k, batch_size=64, verbose=2, patience=0)
    out, calls = check_all(gb, ctx, nf, 6, tr, te, pins, None, base, trials, cancel_at=at)
    assert calls[-1][0] == at
    assert [o[1]["cancelled"] for o in out] == ([1, 1, 1] if at == 0 else [0, 1, 1])


def test_plain_launches_equal_the_graph(gb, ctx, monkeypatch):
    nf, k = 120, 8
    rng = np.random.default_rng(12)
    tr, te = fm_oracle.random_ctr(rng, nf, 300), fm_oracle.random_ctr(rng, nf, 80)
    emb = fm_oracle.random_embeddings(rng, 30, (12,), 300, 80)
    pins = [fm_oracle.init_params(rng, nf, k, s, (12,)) for s in (0.1, 0.2, 0.05)]
    base = dict(n_factors=k, n_epochs=2, batch_size=64, verbose=1, patience=0)
    g, _ = batched(gb, ctx, nf, 5, tr, te, pins, emb, base, MIXED[:3])
    monkeypatch.setenv("GORSE_B200_FM_FIT_NO_GRAPH", "1")
    p, _ = batched(gb, ctx, nf, 5, tr, te, pins, emb, base, MIXED[:3])
    for i in range(3):
        assert_same(g[i], p[i], f"trial {i}")


def test_one_trial_of_a_mixed_batch_equals_the_restatement(gb, ctx):
    nf, k = 203, 16
    rng, tr, te = ctr(13, nf, 2100, 300)
    pins = [fm_oracle.init_params(rng, nf, k, s) for s in (0.1, 0.05, 0.2, 0.1, 0.01)]
    base = dict(n_factors=k, n_epochs=2, batch_size=300, verbose=1, patience=0, max_steps=3)
    out, _ = batched(gb, ctx, nf, 6, tr, te, pins, None, base, MIXED)
    for i in (1, 2):   # an Adam and an SGD trial
        ref = fm_oracle.fit(nf, 6, tr, te, pins[i], **{**base, **MIXED[i]})
        assert out[i][1]["steps"] == 3
        assert_same(out[i], ref, f"trial {i} against the restatement")
