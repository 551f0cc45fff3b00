"""CPU checks of the FM training restatement (fm_oracle/fm_fit_oracle.c): the shared Log and Pow, the replayed backward heap
and that another order of the logit's three gradients is detectable, the optimiser pieces against the reference's own
compiled kernels, the Precision / Recall / Accuracy known answers, the AUC against a brute-force pair count, the Fit
loop's bookkeeping, and that gorse_b200_fm_fit rejects a NULL context without a device."""
import ctypes as C

import numpy as np
import pytest

import fm_oracle


def test_log_agrees_with_numpy_after_rounding():
    """The restated Log against numpy's float64 log rounded to float32.  The loss only takes it on [1, 2]; agreement with
    math32's amd64 assembly is not pinned, so this bounds how far the restated algorithm is from a correctly rounded one."""
    rng = np.random.default_rng(7)
    x = np.concatenate([rng.uniform(1, 2, 20000), rng.uniform(1e-30, 1e30, 2000), [1.0, 2.0, 1.5, np.float32(1 + 2 ** -23)]]).astype(np.float32)
    got = np.array([fm_oracle.logf(v) for v in x], np.float32)
    want = np.log(x.astype(np.float64)).astype(np.float32)
    ulps = np.abs(got.view(np.int32).astype(np.int64) - want.view(np.int32).astype(np.int64))
    assert ulps.max() <= 1 and np.mean(ulps != 0) < 0.1, (ulps.max(), np.mean(ulps != 0))   # float32 arithmetic: within 1 ulp
    assert fm_oracle.logf(1.0) == 0.0
    assert fm_oracle.logf(0.0) == -np.inf and fm_oracle.logf(np.inf) == np.inf
    assert np.isnan(fm_oracle.logf(-1.0)) and np.isnan(fm_oracle.logf(np.nan))
    assert fm_oracle.logf(np.float32(1e-45)) == np.float32(np.log(np.float64(np.float32(1e-45))))   # subnormal


def test_pow_steps():
    for beta in (0.9, 0.999):
        for t in (0, 1, 2, 7, 100, 1000, 123457):
            want = np.float32(np.float64(np.float32(beta)) ** t)
            got = fm_oracle.pow_steps(beta, t)
            assert abs(int(got.view(np.int32)) - int(want.view(np.int32))) <= 1, (beta, t, got, want)


def test_backward_heap_order_of_the_logit_gradients():
    # Tensor.Backward over AFM.Forward + BCEWithLogits pops Mul(p, y) first, then Abs(p), then ReLU(p)
    assert fm_oracle.p_grad_order() == [1, 2, 0]


def _small_problem(seed=3, nf=60, n_train=700, n_test=200):
    rng = np.random.default_rng(seed)
    tr = fm_oracle.random_ctr(rng, nf, n_train)
    te = fm_oracle.random_ctr(rng, nf, n_test)
    return rng, nf, tr, te


def test_another_order_of_the_logit_gradients_is_detectable():
    rng, nf, tr, te = _small_problem()
    p0 = fm_oracle.init_params(rng, nf, 8, 0.3)
    kw = dict(n_factors=8, n_epochs=3, lr=0.05, reg=0.01, batch_size=7, verbose=1, patience=0)
    ref, _, _ = fm_oracle.fit(nf, 6, tr, te, p0, **kw)
    # (a + b) + c: only the term added last matters, the first two commute
    try:
        differ = []
        for order in ([0, 1, 2], [0, 2, 1]):   # Abs last, Mul last
            fm_oracle.set_p_grad_order(order)
            other, _, _ = fm_oracle.fit(nf, 6, tr, te, p0, **kw)
            differ.append(other.tobytes() != ref.tobytes())
        fm_oracle.set_p_grad_order([2, 1, 0])  # ReLU last, as replayed
        same, _, _ = fm_oracle.fit(nf, 6, tr, te, p0, **kw)
    finally:
        fm_oracle.set_p_grad_order(None)
    assert all(differ), differ
    assert same.tobytes() == ref.tobytes()


def test_optimiser_pieces_equal_the_reference_kernels():
    import oracle

    oracle.build()
    if not oracle.ref_available():
        pytest.skip("oracle/_ref/libfloats_ref.so is not built (reference project not found)")
    L = C.CDLL(oracle.REF_SO)
    fp = C.POINTER(C.c_float)
    L._mm512_mul_const_add_to.argtypes = [fp, fp, fp, fp, C.c_int64]
    L._mm512_mul_const_add.argtypes = [fp, fp, fp, C.c_int64]

    def P(a):
        return a.ctypes.data_as(fp)

    # The committed Go assembly keeps the 8-lane block as vmulps + vaddps (floats_avx512.s:160-161); gcc, which built
    # oracle/_ref, contracts it into an FMA (tests/test_oracle_floats.py).  So the 8-lane block is checked against the
    # two-rounding form and every other element against the compiled kernel.
    rng = np.random.default_rng(9)
    for n in (1, 2, 7, 8, 9, 15, 16, 17, 24, 25, 31, 32, 40, 100, 1000, 16 * 200 + 8, 16 * 200 + 13):
        a, b = rng.standard_normal(n).astype(np.float32), rng.standard_normal(n).astype(np.float32)
        body = n // 16 * 16
        blk = np.zeros(n, bool)
        if n - body >= 8:
            blk[body:body + 8] = True
        for c in (np.float32(0.1) - np.float32(0.0), np.float32(1) - np.float32(0.9), np.float32(-3.3e-3), np.float32(2e-4)):
            cc = np.array([c], np.float32)
            two = (a * c + b).astype(np.float32)   # numpy rounds the product, then the sum
            d = np.zeros(n, np.float32)
            L._mm512_mul_const_add_to(P(a), P(cc), P(b), P(d), n)
            got = fm_oracle.mul_const_add_to(a, c, b)
            assert got[~blk].tobytes() == d[~blk].tobytes() and got[blk].tobytes() == two[blk].tobytes(), (n, c)
            d = b.copy()
            L._mm512_mul_const_add(P(a), P(cc), P(d), n)
            got = fm_oracle.mul_const_add(a, c, b)
            assert got[~blk].tobytes() == d[~blk].tobytes() and got[blk].tobytes() == two[blk].tobytes(), (n, c)


def test_precision_recall_accuracy_known_answers():
    # model/ctr/evaluator_test.go:22-46
    assert fm_oracle.metrics([1, 1, 1], [1])[0] == np.float32(0.75)
    assert fm_oracle.metrics([], [])[0] == 0
    assert fm_oracle.metrics([1, -1, -1, -1], [])[1] == np.float32(0.25)
    assert fm_oracle.metrics([], [])[1] == 0
    assert fm_oracle.metrics([1, 1, -1, -1], [1, 1, -1, -1])[2] == np.float32(0.5)
    assert fm_oracle.metrics([], [])[2] == 0


def test_auc_against_a_brute_force_pair_count():
    rng = np.random.default_rng(5)
    for n_pos, n_neg in ((1, 1), (10, 0), (0, 10), (37, 51), (500, 300)):
        pos = np.round(rng.standard_normal(n_pos), 1).astype(np.float32)   # rounding makes ties
        neg = np.round(rng.standard_normal(n_neg), 1).astype(np.float32)
        auc = fm_oracle.metrics(pos, neg)[3]
        if n_pos * n_neg == 0:
            assert auc == 0
            continue
        pairs = int((neg[None, :] < pos[:, None]).sum())   # exact while below 2^24
        assert auc == np.float32(np.float32(pairs) / np.float32(n_pos * n_neg)), (auc, pairs)


def test_fit_bookkeeping():
    rng, nf, tr, te = _small_problem(seed=4)
    p0 = fm_oracle.init_params(rng, nf, 8)
    kw = dict(n_factors=8, lr=0.01, batch_size=64)
    n_batches = (len(tr[0]) - 1 + 63) // 64
    _, r, m = fm_oracle.fit(nf, 6, tr, te, p0, n_epochs=5, verbose=2, patience=0, **kw)
    assert r["epochs_run"] == 5 and r["steps"] == 5 * n_batches and not r["early_stopped"] and not r["cancelled"]
    assert np.any(m != 0)
    # the same epochs stopped by max_steps give the same parameters
    a, _, _ = fm_oracle.fit(nf, 6, tr, te, p0, n_epochs=2, verbose=1, patience=0, **kw)
    b, rb, _ = fm_oracle.fit(nf, 6, tr, te, p0, n_epochs=5, verbose=1, patience=0, max_steps=2 * n_batches + 3, **kw)
    c, _, _ = fm_oracle.fit(nf, 6, tr, te, p0, n_epochs=5, verbose=1, patience=0, max_steps=2 * n_batches, **kw)
    assert rb["steps"] == 2 * n_batches + 3 and a.tobytes() == c.tobytes() and a.tobytes() != b.tobytes()
    # cancelled after epoch 2: the parameters of two epochs, a zero score
    d, rd, _ = fm_oracle.fit(nf, 6, tr, te, p0, n_epochs=5, verbose=1, patience=0, cancel_epoch=2, **kw)
    assert rd["cancelled"] == 1 and rd["auc"] == 0 and rd["precision"] == 0 and d.tobytes() == a.tobytes()
    # patience 1 on a learning rate that makes AUC fall stops early
    _, re_, _ = fm_oracle.fit(nf, 6, tr, te, p0, n_factors=8, lr=5.0, batch_size=64, n_epochs=30, verbose=1, patience=1)
    assert re_["early_stopped"] == 1 or re_["diverged"] == 1


def test_null_context_fails_without_a_device(gb):
    from gorse_b200 import _lib

    p = _lib.FMFitParams()
    assert _lib.lib.gorse_b200_fm_fit_params_default(C.byref(p)) == _lib.OK
    assert (p.n_factors, p.n_epochs, p.batch_size, p.verbose, p.patience, p.optimizer) == (16, 50, 1024, 10, 10, _lib.FM_ADAM)
    r = _lib.FMFitResult()
    assert _lib.lib.gorse_b200_fm_fit(None, 4, 2, 0, C.byref(p), 0, *([None] * 4), 0, *([None] * 4), None, 0, None, None, None,
                                      None, C.byref(r)) == _lib.ERR_ARG
    assert b"NULL" in _lib.lib.gorse_b200_last_error()
