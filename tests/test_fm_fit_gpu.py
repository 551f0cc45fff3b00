"""gorse_b200_fm_fit against the CPU restatement of the reference's AFM.Fit (fm_oracle/fm_fit_oracle.c): parameters and both
Adam moments bit-identical after 1, 2 and 7 steps and after whole epochs, the evaluation metrics and the Verbose / Patience /
NaN-break / cancel bookkeeping, a fitted model ranked by gorse_b200_fm_rank, and every argument error."""
import ctypes as C
import os

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
    """bitwise, every NaN counting as one value (the device and the CPU propagate different NaN payloads)"""
    a, b = np.array(a, np.float32), np.array(b, np.float32)
    a[np.isnan(a)] = np.nan
    b[np.isnan(b)] = np.nan
    return a.tobytes() == b.tobytes()


def data(seed, nf, n_train, n_test, everywhere=None, high=None):
    rng = np.random.default_rng(seed)
    low = min(nf, 1 << 20)        # ids and labels below 2^20; `high` adds the large ones
    tr = fm_oracle.random_ctr(rng, low, n_train)
    te = fm_oracle.random_ctr(rng, low, n_test)
    if everywhere is not None:   # one feature in every training row, with a numerical value
        off, idx, val, tgt = tr
        idx, val = idx.copy(), val.copy()
        idx[off[:-1] + 1] = everywhere
        val[off[:-1] + 1] = rng.standard_normal(len(off) - 1).astype(np.float32)
        tr = (off, idx, val, tgt)
    if high is not None:         # replace half the label features by indices above 2^24 (they travel as float32)
        for off, idx, _, _ in (tr, te):
            m = rng.random(idx.size) < 0.5
            m[off[:-1]] = False
            idx[m] = rng.integers(high[0], high[1], int(m.sum()))
    return rng, tr, te


def both(gb, ctx, nf, nd, tr, te, p0, moments=True, **kw):
    t = gb.FMTrainer(ctx, nf, nd, **kw)
    pg, rg, mg = t.fit(tr, te, p0, moments=moments)
    po, ro, mo = fm_oracle.fit(nf, nd, tr, te, p0, **kw)
    return (pg, rg, mg), (po, ro, mo)


def assert_same(g, o, what):
    (pg, rg, mg), (po, ro, mo) = g, o
    assert same(pg, po), (what, "params", int(np.sum(pg.view(np.uint32) != po.view(np.uint32))))
    if mg is not None:
        assert same(mg, mo), (what, "moments")
    for f in RESULT_FIELDS:
        assert same([rg[f]], [ro[f]]), (what, f, rg[f], ro[f])


CASES = [(k, opt, reg, 7) for k in (8, 16, 32) for opt in (0, 1) for reg in (0.0, 0.01)] + \
        [(16, opt, 0.01, bs) for opt in (0, 1) for bs in (1024, 1)]


@pytest.mark.parametrize("k,opt,reg,bs", CASES)
def test_steps_and_epochs_bit_identical(gb, ctx, k, opt, reg, bs):
    nf = 203                      # nf and nf k with 8-lane blocks (203 % 16 = 11): every fusing case of the optimiser
    n_train = 2100 if bs != 1 else 300
    rng, tr, te = data(k * 10 + opt + bs, nf, n_train, 400)
    p0 = fm_oracle.init_params(rng, nf, k, 0.1)
    kw = dict(n_factors=k, lr=0.01 if opt == 0 else 0.05, reg=reg, optimizer=opt, batch_size=bs, verbose=1, patience=0)
    for steps in (1, 2, 7):
        g, o = both(gb, ctx, nf, 6, tr, te, p0, n_epochs=3, max_steps=steps, **kw)
        assert g[1]["steps"] == steps
        assert_same(g, o, f"{steps} steps")
    g, o = both(gb, ctx, nf, 9, tr, te, p0, n_epochs=2, **kw)   # num_dimension 9 > the longest row: extra padding
    assert g[1]["epochs_run"] == 2 and np.any(g[2][0] != 0) == (opt == 0)
    assert_same(g, o, "epochs")


def test_feature_in_every_row_and_mixed_lengths(gb, ctx):
    nf, k = 150, 16
    rng, tr, te = data(5, nf, 3000, 300, everywhere=7)
    p0 = fm_oracle.init_params(rng, nf, k, 0.1)
    g, o = both(gb, ctx, nf, 0, tr, te, p0, n_factors=k, n_epochs=3, lr=0.01, batch_size=1024, verbose=1, patience=0)
    assert_same(g, o, "everywhere")


def test_feature_indices_above_2_24(gb, ctx):
    nf, k = (1 << 24) + 64, 8
    rng, tr, te = data(6, nf, 500, 100, high=((1 << 24) - 40, (1 << 24) + 60))
    p0 = np.zeros(1 + nf * k + nf, np.float32)
    p0[1:] = (rng.standard_normal(nf * k + nf) * 0.1).astype(np.float32)
    g, o = both(gb, ctx, nf, 6, tr, te, p0, n_factors=k, n_epochs=2, lr=0.01, batch_size=128, verbose=1, patience=0, max_steps=5)
    assert_same(g, o, "above 2^24")


@pytest.mark.parametrize("bad", ["inf", "nan"])
def test_non_finite_row_0(gb, ctx, bad):
    nf, k = 80, 8
    rng, tr, te = data(7, nf, 600, 100)
    p0 = fm_oracle.init_params(rng, nf, k, 0.1)
    p0[1 + 3] = np.float32(bad)     # V[0][3]: every padded position reads it
    g, o = both(gb, ctx, nf, 8, tr, te, p0, n_factors=k, n_epochs=2, lr=0.01, batch_size=64, verbose=1, patience=0)
    assert np.isnan(g[0]).any()
    assert_same(g, o, bad)


def test_verbose_patience_nan_break_and_cancel(gb, ctx):
    nf, k = 120, 8
    rng, tr, te = data(8, nf, 1500, 500)
    p0 = fm_oracle.init_params(rng, nf, k, 0.1)
    base = dict(n_factors=k, batch_size=100)
    # Verbose 3 over 7 epochs: evaluations at 0, 3, 6, 7
    g, o = both(gb, ctx, nf, 6, tr, te, p0, n_epochs=7, lr=0.01, verbose=3, patience=0, **base)
    assert_same(g, o, "verbose")
    # a large step makes the AUC fall: Patience stops early
    g, o = both(gb, ctx, nf, 6, tr, te, p0, n_epochs=30, lr=0.5, verbose=1, patience=2, **base)
    assert o[1]["early_stopped"] == 1
    assert_same(g, o, "patience")
    # SGD with a huge step diverges: the NaN break
    g, o = both(gb, ctx, nf, 6, tr, te, p0, n_epochs=30, lr=1e6, optimizer=1, verbose=1, patience=0, **base)
    assert o[1]["diverged"] == 1 and o[1]["epochs_run"] < 30
    assert_same(g, o, "diverged")
    # cancel after the epoch-0 evaluation and after epoch 2
    for at in (0, 2):
        t = gb.FMTrainer(ctx, nf, 6, n_epochs=5, lr=0.01, verbose=1, patience=0, **base)
        seen = []
        pg, rg, _ = t.fit(tr, te, p0, progress=lambda ep, n, auc: seen.append((ep, n)) or ep == at)
        po, ro, _ = fm_oracle.fit(nf, 6, tr, te, p0, n_epochs=5, lr=0.01, verbose=1, patience=0, cancel_epoch=at, **base)
        assert rg["cancelled"] == 1 and seen == [(e, 5) for e in range(at + 1)]
        assert same(pg, po) and all(same([rg[f]], [ro[f]]) for f in RESULT_FIELDS), at


def test_plain_launches_equal_the_graph(gb, ctx):
    nf, k = 100, 16
    rng, tr, te = data(9, nf, 1000, 100)
    p0 = fm_oracle.init_params(rng, nf, k, 0.1)
    kw = dict(n_factors=k, n_epochs=2, lr=0.01, batch_size=64, verbose=1, patience=0)
    a = gb.FMTrainer(ctx, nf, 6, **kw).fit(tr, te, p0, moments=True)
    os.environ["GORSE_B200_FM_FIT_NO_GRAPH"] = "1"
    try:
        b = gb.FMTrainer(ctx, nf, 6, **kw).fit(tr, te, p0, moments=True)
    finally:
        del os.environ["GORSE_B200_FM_FIT_NO_GRAPH"]
    assert a[0].tobytes() == b[0].tobytes() and a[2].tobytes() == b[2].tobytes() and a[1] == b[1]


def test_fitted_model_ranks_like_the_restatement(gb, ctx):
    nf, k = 90, 16
    rng, tr, te = data(10, nf, 800, 100)
    p0 = fm_oracle.init_params(rng, nf, k, 0.1)
    params, _, _ = gb.FMTrainer(ctx, nf, 6, n_factors=k, n_epochs=3, lr=0.01, batch_size=128, verbose=1, patience=0).fit(tr, te, p0)
    inp = fm_oracle.random_input(rng, nf, [0, 5, 300, 40], 60)
    with gb.FMRanker(ctx, nf, k, 6, 1024, (), params) as fm:
        sg, og, _ = fm.rank(inp)
    so, oo = fm_oracle.Model(nf, k, 6, 1024, (), params).rank(inp)
    assert sg.tobytes() == so.tobytes() and og.tolist() == oo.tolist()


def test_unsupported_and_argument_errors(gb, ctx):
    from gorse_b200 import _lib

    nf, k = 30, 8
    rng, tr, te = data(11, nf, 50, 20)
    p0 = fm_oracle.init_params(rng, nf, k, 0.1)

    def call(nf=nf, nd=4, n_emb=0, tr=tr, te=te, pin=p0, **kw):
        t = gb.FMTrainer(ctx, nf, nd, n_emb=n_emb, **{**dict(n_factors=k, n_epochs=1), **kw})
        try:
            t.fit(tr, te, pin)
        except gb.GorseB200Error as e:
            return e.status
        return _lib.OK

    assert call() == _lib.OK
    assert call(n_emb=1) == _lib.ERR_UNSUPPORTED
    assert call(n_factors=33, pin=fm_oracle.init_params(rng, nf, 33)) == _lib.ERR_UNSUPPORTED
    assert call(verbose=0) == _lib.ERR_ARG
    assert call(optimizer=2) == _lib.ERR_ARG
    assert call(batch_size=0) == _lib.ERR_ARG
    assert call(n_epochs=-1) == _lib.ERR_ARG
    assert call(patience=-1) == _lib.ERR_ARG
    assert call(max_steps=-1) == _lib.ERR_ARG
    assert call(nf=0, pin=np.zeros(1, np.float32)) == _lib.ERR_ARG
    assert call(nd=-1) == _lib.ERR_ARG
    off, idx, val, tgt = tr
    assert call(tr=(off + 1, idx, val, tgt)) == _lib.ERR_ARG                       # offsets not from 0
    bad = off.copy()
    bad[3] = bad[5]
    assert call(tr=(bad, idx, val, tgt)) == _lib.ERR_ARG                            # decreasing offsets
    for v in (nf, -1):
        i2 = idx.copy()
        i2[4] = v
        assert call(tr=(off, i2, val, tgt)) == _lib.ERR_ARG                         # feature outside the table
    big = (1 << 24) + 2
    i2 = idx.copy()
    i2[4] = big + 1                                                                 # rounds to 2^24 + 4 >= n_features
    assert call(nf=big + 2, tr=(off, i2, val, tgt), pin=np.zeros(1 + (big + 2) * (k + 1), np.float32)) == _lib.ERR_ARG
    toff, tidx, tval, ttgt = te
    t2 = tidx.copy()
    t2[0] = nf
    assert call(te=(toff, t2, tval, ttgt)) == _lib.ERR_ARG                          # the test rows are checked too
    p = _lib.FMFitParams(k, 1, 0.01, 0.0, 0, 16, 1, 0, 0)
    r = _lib.FMFitResult()
    n, o_, i_, v_, t_ = len(off) - 1, off, idx, val, tgt
    P = _lib.ptr
    out = np.zeros_like(p0)
    assert lib_fit(_lib, ctx, nf, p, n, P(o_), P(i_), P(v_), None, P(p0), P(out), r) == _lib.ERR_ARG              # NULL targets
    assert lib_fit(_lib, ctx, nf, p, n, P(o_), P(i_), P(v_), P(t_), None, P(out), r) == _lib.ERR_ARG               # NULL params_in
    assert lib_fit(_lib, ctx, nf, p, n, P(o_), None, P(v_), P(t_), P(p0), P(out), r) == _lib.ERR_ARG               # NULL indices
    for wrong in (p0.size - 1, p0.size + 1, 1 + nf * (k + 2) + nf):                                               # another model's length
        assert lib_fit(_lib, ctx, nf, p, n, P(o_), P(i_), P(v_), P(t_), P(p0), P(out), r, n_params=wrong) == _lib.ERR_ARG
    with pytest.raises(ValueError):
        gb.FMTrainer(ctx, nf, 4, n_factors=k).fit(tr, te, fm_oracle.init_params(rng, nf, k + 1))
    assert _lib.lib.gorse_b200_fm_fit(ctx.h, nf, 4, 0, None, 0, *([None] * 4), 0, *([None] * 4), P(p0), p0.size, P(out), None, None,
                                      None, C.byref(r)) == _lib.ERR_ARG                                            # NULL params


def lib_fit(_lib, ctx, nf, p, n, off, idx, val, tgt, pin, pout, r, n_params=None):
    n_params = 1 + nf * (p.n_factors + 1) if n_params is None else n_params
    return _lib.lib.gorse_b200_fm_fit(ctx.h, nf, 4, 0, C.byref(p), n, off, idx, val, tgt, 0, None, None, None, None, pin, n_params, pout, None,
                                      None, None, C.byref(r))
