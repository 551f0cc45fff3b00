"""CPU checks of the FM ranker's restatement (fm_oracle): the reference's softmax known answer, its floats pieces against
the reference's own compiled kernels, the property that rows are independent without embeddings, that the chunk coupling of
the softmax is detectable, the shared double exp against numpy, and that the C entry points reject a NULL handle without a
device."""
import ctypes as C

import numpy as np
import pytest

import fm_oracle


def test_softmax_known_answer():
    # common/nn/op_test.go:534-539
    y = fm_oracle.softmax(np.array([[3.0, 1.0, 0.2]], np.float32))
    assert np.allclose(y[0], [0.8360188027814407, 0.11314284146556013, 0.05083835575299916], atol=1e-6, rtol=0)
    assert fm_oracle.softmax(np.array([[3.0, 1.0, 0.2]], np.float32), coupled=False).tobytes() == y.tobytes()


def test_softmax_coupling_uses_row_r_dim_plus_c_mod_b():
    rng = np.random.default_rng(3)
    x = rng.standard_normal((5, 7)).astype(np.float32) * 3
    y = fm_oracle.softmax(x)
    flat = x.reshape(-1)
    mx = x.max(axis=1)
    e = np.array([np.float32(np.exp(np.float64(np.float32(flat[i] - mx[i % 5])))) for i in range(flat.size)], np.float32).reshape(5, 7)
    s = np.zeros(5, np.float32)
    for r in range(5):
        acc = e[r, 0]
        for c in range(1, 7):
            acc = np.float32(acc + e[r, c])
        s[r] = acc
    want = (e.reshape(-1) / s[np.arange(35) % 5]).astype(np.float32).reshape(5, 7)
    assert np.allclose(y, want, rtol=1e-6, atol=0)   # numpy's exp may differ from the restated one in the last bit
    assert not np.allclose(y, fm_oracle.softmax(x, coupled=False), rtol=1e-3)


def test_exp_agrees_with_numpy_after_rounding():
    """The shared double exp against numpy's, both rounded to float32, on the softmax's range.  Agreement with Go's amd64
    assembly is not pinned; this counts how often the restatement differs from another correctly rounded-ish exp."""
    rng = np.random.default_rng(11)
    x = np.concatenate([rng.uniform(-110, 0, 20000), rng.uniform(-1, 1, 5000), rng.uniform(0, 88, 5000),
                        [0.0, -0.0, 1e-9, -1e-9, -np.inf, np.inf, 89.0, -104.0]]).astype(np.float32)
    got = np.array([fm_oracle.exp(v) for v in x], np.float32)
    with np.errstate(over="ignore"):
        want = np.exp(x.astype(np.float64)).astype(np.float32)
    mism = int(np.sum(got.view(np.uint32) != want.view(np.uint32)))
    assert mism <= 3, mism
    assert fm_oracle.exp(np.nan) != fm_oracle.exp(np.nan)


def test_pieces_equal_the_reference_kernels():
    import oracle

    oracle.build()
    if not oracle.ref_available():
        pytest.skip("oracle/_ref/libfloats_ref.so is not built (reference project not found)")
    L = C.CDLL(oracle.REF_SO)
    fp = C.POINTER(C.c_float)
    L._mm512_mm.argtypes = [C.c_bool, C.c_bool, C.c_int64, C.c_int64, C.c_int64, fp, C.c_int64, fp, C.c_int64, fp, C.c_int64]
    L._mm512_mul_to.argtypes = [fp, fp, fp, C.c_int64]
    L._mm512_add_const.argtypes = [fp, fp, C.c_int64]

    def P(a):
        return a.ctypes.data_as(fp)

    rng = np.random.default_rng(5)
    for transA, m, n, k in [(0, 7, 16, 32), (0, 3, 8, 768), (0, 5, 33, 64), (1, 16, 1, 9), (1, 32, 1, 40), (1, 1, 1, 16), (0, 300, 16, 7)]:
        a = rng.standard_normal(m * k).astype(np.float32)
        b = rng.standard_normal(k * n).astype(np.float32)
        lda = m if transA else k
        c1, c2 = np.zeros(m * n, np.float32), np.zeros(m * n, np.float32)
        L._mm512_mm(bool(transA), False, m, n, k, P(a), lda, P(b), n, P(c1), n)
        fm_oracle.mm(transA, 0, m, n, k, a, lda, b, n, c2, n)
        assert c1.tobytes() == c2.tobytes(), (transA, m, n, k)
    for n in (1, 7, 16, 17, 100, 1000):
        a, b = rng.standard_normal(n).astype(np.float32), rng.standard_normal(n).astype(np.float32)
        c = np.zeros(n, np.float32)
        L._mm512_mul_to(P(a), P(b), P(c), n)
        assert c.tobytes() == fm_oracle.mul_to(a, b).tobytes()
        d = a.copy()
        cc = np.array([0.37], np.float32)
        L._mm512_add_const(P(d), P(cc), n)
        assert d.tobytes() == fm_oracle.add_const(a, cc[0]).tobytes()


def test_rows_are_independent_without_embeddings():
    """model_test.go:261-292: one BatchPredict over many rows == one call per row"""
    rng = np.random.default_rng(1)
    nf, k = 40, 8
    m = fm_oracle.Model(nf, k, 4, 1024, (), fm_oracle.random_params(rng, nf, k))
    rows = [(rng.integers(0, nf, L).astype(np.int32), rng.standard_normal(L).astype(np.float32)) for L in (2, 8, 0, 5, 3)]
    batched = m.batch_predict(rows)
    single = np.array([m.batch_predict([r])[0] for r in rows], np.float32)
    assert batched.tobytes() == single.tobytes()


def test_coupling_is_detectable_with_embeddings():
    rng = np.random.default_rng(2)
    nf, k, d = 30, 8, 32
    params = fm_oracle.random_params(rng, nf, k, (d,))
    inp = fm_oracle.random_input(rng, nf, [40, 9], 25, (d,))
    for bs, differ in ((1024, True), (7, True), (1, False)):
        m = fm_oracle.Model(nf, k, 3, bs, (d,), params)
        coupled, _ = m.rank(inp)
        rowwise, _ = m.rank(inp, coupled=False)
        assert (coupled.tobytes() != rowwise.tobytes()) == differ, bs


def test_order_is_score_descending_ties_by_position():
    rng = np.random.default_rng(4)
    nf, k = 20, 8
    m = fm_oracle.Model(nf, k, 3, 1024, (), fm_oracle.random_params(rng, nf, k))
    inp = fm_oracle.random_input(rng, nf, [30], 6)   # 30 candidates from 6 items: ties
    s, o = m.rank(inp)
    want = sorted(range(30), key=lambda t: (-s[t], t))
    assert o.tolist() == want


def test_null_handle_fails_without_a_device(gb):
    from gorse_b200 import _lib

    h = C.c_void_p()
    assert _lib.lib.gorse_b200_fm_rank(None, 1, *([None] * 4), 0, *([None] * 11)) == _lib.ERR_ARG
    assert b"NULL" in _lib.lib.gorse_b200_last_error()
    p = np.zeros(1 + 4 * 9, np.float32)
    assert _lib.lib.gorse_b200_fm_create(None, 4, 8, 2, 1024, 0, None, p.ctypes.data_as(C.c_void_p), p.size, C.byref(h)) == _lib.ERR_ARG
    assert _lib.lib.gorse_b200_fm_destroy(None) == _lib.OK
