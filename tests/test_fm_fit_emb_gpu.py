"""gorse_b200_fm_fit_emb against the CPU restatement of the reference's AFM.Fit with item-embedding slots
(fm_oracle/fm_fit_oracle.c): every parameter tensor and both Adam moments bit-identical after 1, 2 and 7 steps and after
whole epochs, absent embeddings, the softmax's partner-row rule for batches smaller and larger than the dim, non-finite
parameters, the evaluation in chunks, the loop's bookkeeping, plain launches, the slot-free model, a fitted model in the
ranker, and the entry's limits and argument errors."""
import ctypes as C
import os
import types

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


def problem(seed, nf, k, dims, n_train, n_test, n_rows=50, std=0.1, **kw):
    rng = np.random.default_rng(seed)
    tr, te = fm_oracle.random_ctr(rng, nf, n_train), fm_oracle.random_ctr(rng, nf, n_test)
    emb = fm_oracle.random_embeddings(rng, n_rows, dims, n_train, n_test, **kw)
    return rng, tr, te, emb, fm_oracle.init_params(rng, nf, k, std, dims)


def gpu_fit(gb, ctx, nf, nd, tr, te, emb, p0, progress=None, **kw):
    return gb.FMTrainer(ctx, nf, nd, **kw).fit_emb(tr, te, p0, emb.dims, emb.table, emb.mask, emb.train_rows, emb.test_rows, progress=progress,
                                                   moments=True)


def assert_same(g, o, what, k=None, nf=None, dims=()):
    (pg, rg, mg), (po, ro, mo) = g, o
    if not same(pg, po) and k:
        names, o_ = ["B", "V", "W"], [0, 1, 1 + nf * k, 1 + nf * k + nf]
        for s, d in enumerate(dims):
            for n, ln in zip(("H", "AW", "Ab", "EW", "Eb"), (k * d, d * k, k, d * k, k)):
                names.append(f"{n}{s}")
                o_.append(o_[-1] + ln)
        bad = [n for i, n in enumerate(names) if not same(pg[o_[i]:o_[i + 1]], po[o_[i]:o_[i + 1]])]
        raise AssertionError((what, "params differ in", bad))
    assert same(pg, po), (what, "params")
    assert same(mg, mo), (what, "moments")
    for f in RESULT_FIELDS:
        assert same([rg[f]], [ro[f]]), (what, f, rg[f], ro[f])


def check(gb, ctx, nf, nd, tr, te, emb, p0, what, **kw):
    k = kw.get("n_factors", 16)
    assert_same(gpu_fit(gb, ctx, nf, nd, tr, te, emb, p0, **kw), fm_oracle.fit(nf, nd, tr, te, p0, emb=emb, **kw), what, k, nf, emb.dims.tolist())


CASES = [(k, opt, reg, 7, dims) for k, dims in ((8, (5,)), (16, (24, 5)), (32, (64, 3, 17))) for opt in (0, 1) for reg in (0.0, 0.01)] + \
        [(16, 0, 0.01, 1024, (768,)), (16, 1, 0.01, 1, (24, 40)), (8, 0, 0.0002, 300, (5, 24, 64))]


@pytest.mark.parametrize("k,opt,reg,bs,dims", CASES)
def test_steps_and_epochs_bit_identical(gb, ctx, k, opt, reg, bs, dims):
    nf = 203
    n_train = {7: 150, 1: 40, 300: 700, 1024: 1300}[bs]    # every size leaves a partial last batch
    rng, tr, te, emb, p0 = problem(k + opt + bs, nf, k, dims, n_train, 120)
    kw = dict(n_factors=k, lr=0.01, reg=reg, optimizer=opt, batch_size=bs, verbose=1, patience=0)
    for steps in (1, 2, 7) if bs != 1024 else (1, 2):
        check(gb, ctx, nf, 6, tr, te, emb, p0, f"{steps} steps", n_epochs=50, max_steps=steps, **kw)
    check(gb, ctx, nf, 6, tr, te, emb, p0, "epochs", n_epochs=2, **kw)


@pytest.mark.parametrize("n_emb", [4, 8])
def test_many_slots_add_vx_gradients_in_heap_order(gb, ctx, n_emb):
    dims = tuple(3 + 2 * s for s in range(n_emb))
    rng, tr, te, emb, p0 = problem(n_emb, 60, 8, dims, 40, 30, std=0.5)
    check(gb, ctx, 60, 5, tr, te, emb, p0, "slots", n_factors=8, n_epochs=2, batch_size=16, verbose=1, lr=0.01)


@pytest.mark.parametrize("mode", ["no_item", "masked", "all_absent", "one_row"])
def test_absent_embeddings(gb, ctx, mode):
    kwp = dict(no_item=dict(p_no_item=0.6, p_absent=0.0), masked=dict(p_no_item=0.0, p_absent=0.6), all_absent=dict(p_no_item=1.0),
               one_row=dict())[mode]
    n_train = 1 if mode == "one_row" else 50
    rng, tr, te, emb, p0 = problem(21, 80, 16, (24, 5), n_train, 40, **kwp)
    check(gb, ctx, 80, 5, tr, te, emb, p0, mode, n_factors=16, n_epochs=3, batch_size=16, verbose=1, lr=0.01)
    if mode == "no_item":     # a NULL mask: every embedding present
        emb.mask = None
        check(gb, ctx, 80, 5, tr, te, emb, p0, "NULL mask", n_factors=16, n_epochs=2, batch_size=16, verbose=1, lr=0.01)


@pytest.mark.parametrize("bs,dim", [(7, 24), (40, 24), (24, 24), (9, 6), (33, 5)])
def test_partner_row_rule(gb, ctx, bs, dim):
    rng, tr, te, emb, p0 = problem(bs * dim, 90, 8, (dim,), 3 * bs + 2, 2 * bs + 3, std=0.5)
    check(gb, ctx, 90, 5, tr, te, emb, p0, "partner", n_factors=8, n_epochs=2, batch_size=bs, verbose=1, lr=0.02)


@pytest.mark.parametrize("where", ["H", "AW", "EW", "V0"])
def test_non_finite_parameters(gb, ctx, where):
    nf, k, d = 70, 8, 24
    rng, tr, te, emb, p0 = problem(31, nf, k, (d,), 40, 30)
    base = 1 + nf * k + nf
    at = {"H": base + 5, "AW": base + k * d + 9, "EW": base + 2 * k * d + k + 11, "V0": 1 + 3}[where]
    p0 = p0.copy()
    p0[at] = np.inf if where != "AW" else np.nan
    g = gpu_fit(gb, ctx, nf, 9, tr, te, emb, p0, n_factors=k, n_epochs=1, batch_size=16, verbose=1, max_steps=2)
    o = fm_oracle.fit(nf, 9, tr, te, p0, emb=emb, n_factors=k, n_epochs=1, batch_size=16, verbose=1, max_steps=2)
    assert np.isnan(o[0]).any()
    # parameters and moments only: the evaluations see NaN predictions, whose place in Go's sort (and so the AUC) is unpinned
    assert same(g[0], o[0]) and same(g[2], o[2]) and g[1]["steps"] == o[1]["steps"] == 2, where


def test_loop_bookkeeping_and_chunked_evaluation(gb, ctx):
    nf, k = 120, 16
    rng, tr, te, emb, p0 = problem(41, nf, k, (24,), 200, 700)     # test lists longer than one chunk of 64
    kw = dict(n_factors=k, batch_size=64, lr=0.01)
    check(gb, ctx, nf, 6, tr, te, emb, p0, "verbose 3", n_epochs=7, verbose=3, patience=0, **kw)
    check(gb, ctx, nf, 6, tr, te, emb, p0, "patience", n_epochs=12, verbose=1, patience=2, **kw)
    check(gb, ctx, nf, 6, tr, te, emb, p0, "diverge", n_epochs=6, verbose=1, patience=0, n_factors=k, batch_size=64, lr=1e30, optimizer=1)
    for ce in (0, 2):
        g = gpu_fit(gb, ctx, nf, 6, tr, te, emb, p0, progress=lambda ep, n, auc: ep == ce, n_epochs=5, verbose=1, **kw)
        assert_same(g, fm_oracle.fit(nf, 6, tr, te, p0, emb=emb, cancel_epoch=ce, n_epochs=5, verbose=1, **kw), f"cancel {ce}")
        assert g[1]["cancelled"] == 1


def test_plain_launches_equal_the_graph(gb, ctx):
    rng, tr, te, emb, p0 = problem(51, 100, 16, (24, 5), 150, 60)
    kw = dict(n_factors=16, n_epochs=3, batch_size=32, verbose=1)
    a = gpu_fit(gb, ctx, 100, 6, tr, te, emb, p0, **kw)
    os.environ["GORSE_B200_FM_FIT_NO_GRAPH"] = "1"
    try:
        b = gpu_fit(gb, ctx, 100, 6, tr, te, emb, p0, **kw)
    finally:
        del os.environ["GORSE_B200_FM_FIT_NO_GRAPH"]
    assert_same(a, b, "no graph")


def test_no_slots_equals_fm_fit(gb, ctx):
    rng = np.random.default_rng(61)
    nf, k = 203, 16
    tr, te = fm_oracle.random_ctr(rng, nf, 500), fm_oracle.random_ctr(rng, nf, 100)
    p0 = fm_oracle.init_params(rng, nf, k, 0.1)
    none = fm_oracle.Embeddings((), [], None, np.zeros(500, np.int32), np.zeros(100, np.int32))
    kw = dict(n_factors=k, n_epochs=3, batch_size=64, verbose=1)
    a = gpu_fit(gb, ctx, nf, 6, tr, te, none, p0, **kw)
    b = gb.FMTrainer(ctx, nf, 6, **kw).fit(tr, te, p0, moments=True)
    assert_same(a, b, "n_emb = 0")


def test_fitted_model_ranks_as_the_restatement(gb, ctx):
    nf, k, dims = 150, 16, (24, 5)
    rng, tr, te, emb, p0 = problem(71, nf, k, dims, 200, 50)
    pg, _, _ = gpu_fit(gb, ctx, nf, 6, tr, te, emb, p0, n_factors=k, n_epochs=3, batch_size=32, verbose=1)
    inp = fm_oracle.random_input(rng, nf, [40, 9, 70], 25, dims)
    with gb.FMRanker(ctx, nf, k, 6, 32, dims, pg) as r:
        s, o, _ = r.rank(inp)
    ws, wo = fm_oracle.Model(nf, k, 6, 32, dims, pg).rank(inp)
    assert same(s, ws) and o.tolist() == wo.tolist()


def test_limits_and_argument_errors(gb, ctx):
    from gorse_b200 import _lib

    nf, k = 40, 8
    rng, tr, te, emb, p0 = problem(81, nf, k, (5,), 20, 10, n_rows=6)

    def call(dims=(5,), kk=k, rows=None, params=None, table=True, n_emb=None):
        t = gb.FMTrainer(ctx, nf, 4, n_factors=kk, n_epochs=1)
        d = np.asarray(dims, np.int32)
        tabs = [fm_oracle.to_bf16(np.zeros((6, int(x)), np.float32)) for x in d]
        arr = (C.c_void_p * max(len(tabs), 1))(*[x.ctypes.data for x in tabs])
        want = 1 + nf * kk + nf + sum(kk * (3 * int(x) + 2) for x in d)
        p = np.zeros(want if params is None else params, np.float32)
        out = np.zeros(p.size, np.float32)
        er = emb.train_rows.copy() if rows is None else rows
        res = _lib.FMFitResult()
        P = lambda a: a.ctypes.data_as(C.c_void_p)
        off, idx, val, tgt = (np.ascontiguousarray(a) for a in tr)
        toff, tidx, tval, ttgt = (np.ascontiguousarray(a) for a in te)
        return _lib.lib.gorse_b200_fm_fit_emb(ctx.h, nf, 4, C.byref(t.params), 20, P(off), P(idx), P(val), P(tgt), P(er), 10, P(toff), P(tidx),
                                              P(tval), P(ttgt), P(emb.test_rows), d.size if n_emb is None else n_emb, P(d), 6,
                                              arr if table else None, None, P(p), p.size, P(out), None, None, None, C.byref(res))

    assert call() == _lib.OK
    assert call(kk=33) == _lib.ERR_UNSUPPORTED
    assert call(dims=(1025,)) == _lib.ERR_UNSUPPORTED
    assert call(dims=(2,) * 9) == _lib.ERR_UNSUPPORTED
    bad = emb.train_rows.copy()
    bad[3] = 6
    assert call(rows=bad) == _lib.ERR_ARG and b"table row" in _lib.lib.gorse_b200_last_error()
    bad[3] = -2
    assert call(rows=bad) == _lib.ERR_ARG
    assert call(params=7) == _lib.ERR_ARG
    assert call(table=False) == _lib.ERR_ARG
    with pytest.raises(Exception):   # gorse_b200_fm_fit itself still takes no model with slots
        gb.FMTrainer(ctx, nf, 4, n_factors=k, n_epochs=1, n_emb=1).fit(tr, te, np.zeros(1 + nf * k + nf, np.float32))
