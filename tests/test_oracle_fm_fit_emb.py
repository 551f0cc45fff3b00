"""CPU checks of the restatement of AFM.Fit for models with item-embedding slots (fm_oracle/fm_fit_oracle.c), the checker of
gorse_b200_fm_fit_emb: floats.MM's four transpose cases and floats.Dot against the reference's compiled kernels (live when
oracle/_ref is built, and always against their stored outputs), the known answers of common/nn/op_test.go for MatMul, ReLU,
Softmax and the graphs that reuse a tensor, the replayed backward heap on the graph with slots, the gradients against an
independent float64 statement of the same rules (and, where the softmax couples a row only with itself, against the
numerical gradient), and that each pinned rule changes the parameters when it is replaced by its alternative."""
import ctypes as C
import os

import numpy as np
import pytest

import fm_oracle


def _mm(tA, tB, m, n, k, a, b):
    c = np.zeros(m * n, np.float32)
    fm_oracle.mm(tA, tB, m, n, k, a, m if tA else k, b, k if tB else n, c, n)
    return c


MM_SHAPES = [(0, 1, 9, 24, 16), (0, 1, 9, 29, 8), (0, 1, 5, 7, 32), (0, 1, 4, 16, 768), (0, 1, 3, 8, 61), (0, 1, 6, 5, 1),
             (1, 0, 24, 16, 300), (1, 0, 29, 8, 1024), (1, 0, 5, 32, 7), (1, 0, 16, 29, 33), (1, 1, 5, 9, 20), (0, 0, 7, 29, 24)]
DOT_LENGTHS = (1, 5, 8, 15, 16, 24, 31, 32, 61, 768)
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "fm_mm_golden.npz")


def mm_inputs():
    """the seeded operands of every shape, in order"""
    rng = np.random.default_rng(7)
    mms = [(rng.standard_normal(m * k).astype(np.float32), rng.standard_normal(k * n).astype(np.float32)) for _, _, m, n, k in MM_SHAPES]
    dots = [(rng.standard_normal(n).astype(np.float32), rng.standard_normal(n).astype(np.float32)) for n in DOT_LENGTHS]
    return mms, dots


def reference_outputs():
    """_mm512_mm and _mm512_dot of oracle/_ref on mm_inputs(), or None when it is not built"""
    import oracle

    oracle.build()
    if not oracle.ref_available():
        return None
    L = C.CDLL(oracle.REF_SO)
    fp = C.POINTER(C.c_float)
    L._mm512_mm.argtypes = [C.c_bool, C.c_bool, C.c_int64, C.c_int64, C.c_int64, fp, C.c_int64, fp, C.c_int64, fp, C.c_int64]
    L._mm512_dot.restype = C.c_float
    L._mm512_dot.argtypes = [fp, fp, C.c_int64]
    mms, dots = mm_inputs()
    out = {}
    for i, ((tA, tB, m, n, k), (a, b)) in enumerate(zip(MM_SHAPES, mms)):
        c = np.zeros(m * n, np.float32)
        L._mm512_mm(bool(tA), bool(tB), m, n, k, a.ctypes.data_as(fp), m if tA else k, b.ctypes.data_as(fp), k if tB else n, c.ctypes.data_as(fp), n)
        out[f"mm{i}"] = c
    out["dot"] = np.array([L._mm512_dot(a.ctypes.data_as(fp), b.ctypes.data_as(fp), a.size) for a, b in dots], np.float32)
    return out


def check_mm(want):
    mms, dots = mm_inputs()
    for i, ((tA, tB, m, n, k), (a, b)) in enumerate(zip(MM_SHAPES, mms)):
        assert want[f"mm{i}"].tobytes() == _mm(tA, tB, m, n, k, a, b).tobytes(), (tA, tB, m, n, k)
    assert want["dot"].tobytes() == np.array([fm_oracle.dot(a, b) for a, b in dots], np.float32).tobytes()


def test_mm_transpose_cases_equal_the_reference_kernels_stored_outputs():
    """dx0 = dy x1^T is floats.Dot per element (lane accumulators and a tree, not a chain); dx1 = x0^T dy is a chain over the
    batch.  Shapes cover the 16-lane body, the 8-lane block and the scalar tail of both the output and the contraction.
    The stored outputs are the reference's compiled kernels' (tests/golden/make_fm_mm_golden.py), so this holds the
    restatement to them where oracle/_ref cannot be built."""
    check_mm(np.load(GOLDEN))


def test_mm_transpose_cases_equal_the_reference_kernel():
    want = reference_outputs()
    if want is None:
        pytest.skip("oracle/_ref/libfloats_ref.so is not built (reference project not found)")
    check_mm(want)
    stored = np.load(GOLDEN)
    assert all(stored[k].tobytes() == v.tobytes() for k, v in want.items())


def test_dot_is_not_a_chain():
    rng = np.random.default_rng(8)
    differ = 0
    for _ in range(20):
        a, b = rng.standard_normal(768).astype(np.float32), rng.standard_normal(768).astype(np.float32)
        chain = np.zeros(1, np.float32)
        fm_oracle.mm(0, 0, 1, 1, 768, a, 768, b, 1, chain, 1)
        assert abs(fm_oracle.dot(a, b) - chain[0]) < 1e-3
        differ += fm_oracle.dot(a, b) != chain[0]
    assert differ >= 10


def test_matmul_known_answers():
    # common/nn/op_test.go:375-430: all four transpose cases of [[1,2,3],[4,5,6]] x (a 3 x 2 matrix), forward and dy = ones
    x, y = np.arange(1, 7, dtype=np.float32).reshape(1, 2, 3), np.arange(1, 7, dtype=np.float32).reshape(1, 3, 2)
    for t1, t2 in [(0, 0), (1, 0), (0, 1), (1, 1)]:
        xa, ya = (x.transpose(0, 2, 1) if t1 else x), (y.transpose(0, 2, 1) if t2 else y)
        z, gx, gy = fm_oracle.op_bmm(np.ascontiguousarray(xa), np.ascontiguousarray(ya), t1, t2)
        assert z.reshape(2, 2).tolist() == [[22, 28], [49, 64]]
        wx, wy = np.array([[3, 7, 11], [3, 7, 11]], np.float32), np.array([[5, 5], [7, 7], [9, 9]], np.float32)
        assert gx.reshape(xa.shape[1:]).tolist() == (wx.T if t1 else wx).tolist()
        assert gy.reshape(ya.shape[1:]).tolist() == (wy.T if t2 else wy).tolist()


def test_softmax_known_answer_and_gradient():
    # common/nn/op_test.go:534-545: the forward values, and the backward (seeded with ones) against the numerical gradient
    # with op_test.go's step and tolerances (:24-57).  One row couples only with itself, so both index rules agree there.
    x = np.array([[3.0, 1.0, 0.2]], np.float32)
    y, g = fm_oracle.op_softmax(x)
    assert np.allclose(y[0], [0.8360188027814407, 0.11314284146556013, 0.05083835575299916], atol=1e-6, rtol=0)
    eps = 1e-4
    num = np.zeros(3, np.float32)
    for i in range(3):
        lo, hi = x.copy(), x.copy()
        lo[0, i] -= np.float32(eps)
        hi[0, i] += np.float32(eps)
        num[i] = np.sum((fm_oracle.op_softmax(hi)[0].astype(np.float64) - fm_oracle.op_softmax(lo)[0]) / (2 * eps))
    assert np.all(np.abs(g[0] - num) <= 5e-3 + 1e-2 * np.abs(num))
    assert fm_oracle.op_softmax(x, coupled=False)[1].tobytes() == g.tobytes()


def test_softmax_backward_uses_the_sum_of_row_i_mod_b():
    rng = np.random.default_rng(21)
    x, dy = (rng.standard_normal((5, 7)) * 2).astype(np.float32), rng.standard_normal((5, 7)).astype(np.float32)
    y, g = fm_oracle.op_softmax(x, dy)
    gx = (y * dy).astype(np.float32)
    sm = np.zeros(5, np.float32)
    for r in range(5):
        acc = gx[r, 0]
        for c in range(1, 7):
            acc = np.float32(acc + gx[r, c])
        sm[r] = acc
    want = (gx.reshape(-1) - (y.reshape(-1) * sm[np.arange(35) % 5]).astype(np.float32)).astype(np.float32)
    assert g.reshape(-1).tobytes() == want.tobytes()
    assert not np.allclose(g, fm_oracle.op_softmax(x, dy, coupled=False)[1], rtol=1e-3)


def _backward(inputs, kinds, x):
    """gradient of the last op with respect to the leaf x, walking the replayed pop order: kinds are 'add' (two inputs),
    'square' and 'double' (one); -1 names the leaf.  A tensor's gradient is assigned by its first consumer popped and added
    to by the later ones; an op is popped only when its output's gradient is complete."""
    order = fm_oracle.heap_order(inputs)
    assert sorted(order) == list(range(len(inputs)))
    val = {-1: x}
    for o, (kind, inp) in enumerate(zip(kinds, inputs)):
        val[o] = {"add": lambda a: val[a[0]] + val[a[1]], "square": lambda a: val[a[0]] ** 2, "double": lambda a: 2 * val[a[0]]}[kind](inp)
    grad, done = {len(inputs) - 1: np.ones_like(x)}, set()
    for o in order:
        assert all(c in done for c in range(len(inputs)) if o in inputs[c]), "popped before a consumer"
        gs = {"add": [grad[o], grad[o]], "square": [2 * val[inputs[o][0]] * grad[o]], "double": [2 * grad[o]]}[kinds[o]]
        for i, g in zip(inputs[o], gs):
            grad[i] = grad[i] + g if i in grad else g
        done.add(o)
    return val[len(inputs) - 1], grad[-1]


def test_reused_tensors_known_answers():
    # common/nn/op_test.go:583-626 (TestReuseLeaf, TestReuseNode, TestDependency): the values, and gradients 2, 4x and 6x
    x = np.arange(1, 7, dtype=np.float64)
    y, g = _backward([(-1, -1)], ["add"], x)                                         # x + x
    assert y.tolist() == [2, 4, 6, 8, 10, 12] and g.tolist() == [2] * 6
    y, g = _backward([(-1,), (0, 0)], ["square", "add"], x)                          # x^2 + x^2
    assert y.tolist() == [2, 8, 18, 32, 50, 72] and g.tolist() == (4 * x).tolist()
    y, g = _backward([(-1,), (0,), (0, 1)], ["square", "double", "add"], x)          # x^2 + 2 x^2: Mul pops before Pow
    assert y.tolist() == [3, 12, 27, 48, 75, 108] and g.tolist() == (6 * x).tolist()
    assert fm_oracle.heap_order([(-1,), (0,), (0, 1)]) == [2, 1, 0]


def test_relu_known_answer():
    # common/nn/op_test.go:520-532
    y, g = fm_oracle.op_unary("relu", np.array([[1, -2, 3], [-4, 5, -6]], np.float32))
    assert y.tolist() == [[1, 0, 3], [0, 5, 0]] and g.tolist() == [[1, 0, 1], [0, 1, 0]]


def test_backward_heap_on_the_slot_graph():
    """The logit's order does not depend on the slots; vx's does, and is no simple pattern: equal generations leave the
    container/heap as its sift-down leaves them.  These are the orders the kernels use."""
    want = [[0], [1, 0], [2, 1, 0], [1, 3, 2, 0], [3, 4, 2, 1, 0], [4, 5, 1, 2, 3, 0], [3, 6, 4, 2, 5, 1, 0], [7, 4, 2, 5, 3, 1, 6, 0],
            [8, 5, 6, 2, 1, 4, 3, 7, 0]]
    for n in range(9):
        p, vx = fm_oracle.backward_order(n)
        assert p == [1, 2, 0] == fm_oracle.p_grad_order() and vx == want[n], n
    import re, os
    src = open(os.path.join(os.path.dirname(fm_oracle.__file__), "..", "gorse_b200", "csrc", "fm_fit.cu")).read()
    tab = re.search(r"VX_ORDER\[.*?= \{(.*?)\};", src, re.S).group(1)
    assert [[int(v) for v in row.split(",")] for row in re.findall(r"\{([^{}]*)\}", tab)] == want


def _problem(seed, nf=30, k=8, dims=(5,), n_train=13, n_test=9, n_rows=6, **kw):
    rng = np.random.default_rng(seed)
    tr, te = fm_oracle.random_ctr(rng, nf, n_train), fm_oracle.random_ctr(rng, nf, n_test)
    emb = fm_oracle.random_embeddings(rng, n_rows, dims, n_train, n_test, **kw)
    p0 = fm_oracle.random_params(rng, nf, k, dims)
    return nf, k, tr, te, emb, p0


def _f64_step_grads(nf, k, tr, emb, p0, D, rows):
    """The gradients of one batch by the same rules in float64 numpy: -> (loss, grad of the slot tensors, concatenated)"""
    off, idx, val, tgt = tr
    P = p0.astype(np.float64)
    B = len(rows)
    V, W = P[1:1 + nf * k].reshape(nf, k), P[1 + nf * k:1 + nf * k + nf]
    X, I = np.zeros((B, D)), np.zeros((B, D), np.int64)
    for b, r in enumerate(rows):
        n = off[r + 1] - off[r]
        I[b, :n], X[b, :n] = idx[off[r]:off[r + 1]], val[off[r]:off[r + 1]]
    vx = np.einsum("bdk,bd->bk", V[I], X)
    p = (W[I] * X).sum(1) + 0.5 * (vx ** 2 - np.einsum("bdk,bd->bk", V[I] ** 2, X ** 2)).sum(1) + P[0]
    o, cache = 1 + nf * k + nf, []
    for s, d in enumerate(emb.dims):
        H, AW, Ab = P[o:o + k * d].reshape(k, d), P[o + k * d:o + 2 * k * d].reshape(d, k), P[o + 2 * k * d:o + 2 * k * d + k]
        EW, Eb = P[o + 2 * k * d + k:o + 3 * k * d + k].reshape(d, k), P[o + 3 * k * d + k:o + 3 * k * d + 2 * k]
        o += 3 * k * d + 2 * k
        e = np.zeros((B, d))
        for b, r in enumerate(rows):
            t = emb.train_rows[r]
            if t >= 0 and (emb.mask is None or emb.mask[t, s]):
                e[b] = (emb.table[s][t].astype(np.uint32) << 16).view(np.float32)
        h = e @ AW + Ab
        hr = np.maximum(h, 0)
        z = (hr @ H).reshape(-1)
        part = np.arange(B * d) % B
        ex = np.exp(z - z.reshape(B, d).max(1)[part])
        y = ex / ex.reshape(B, d).sum(1)[part]
        att = y.reshape(B, d) * e
        enc = att @ EW + Eb
        p = p + (vx * enc).sum(1)
        cache.append((H, EW, e, h, hr, y, att))
    t = tgt[rows].astype(np.float64)
    loss = np.mean(np.maximum(p, 0) - p * (t + 1) / 2 + np.log1p(np.exp(-np.abs(p))))
    with np.errstate(over="ignore"):
        sig = 1 / (1 + np.exp(-p))
    dp = (sig - (t + 1) / 2) / B
    grads = []
    for (H, EW, e, h, hr, y, att), d in zip(cache, emb.dims):
        denc = vx * dp[:, None]
        datt = denc @ EW.T
        gx = y * (datt * e).reshape(-1)
        sm = gx.reshape(B, d).sum(1)
        dz = (gx - y * sm[np.arange(B * d) % B]).reshape(B, d)
        dh = (dz @ H.T) * (h > 0)
        grads += [(hr.T @ dz).reshape(-1), (e.T @ dh).reshape(-1), dh.sum(0), (att.T @ denc).reshape(-1), denc.sum(0)]
    return loss, np.concatenate(grads)


def _sgd_grads(nf, k, tr, te, emb, p0, bs, lr=0.5):
    """one SGD step without decay: (p0 - p1) / lr is the gradient the restatement formed"""
    p1, _, _ = fm_oracle.fit(nf, 4, tr, te, p0, n_factors=k, n_epochs=1, lr=lr, reg=0.0, optimizer=1, batch_size=bs, max_steps=1, emb=emb)
    return ((p0.astype(np.float64) - p1.astype(np.float64)) / lr)[1 + nf * k + nf:]


@pytest.mark.parametrize("dims,bs", [((5,), 13), ((24,), 7), ((16, 5), 4), ((5, 3, 8), 13), ((40,), 1)])
def test_slot_gradients_equal_the_float64_statement(dims, bs):
    nf, k, tr, te, emb, p0 = _problem(3, dims=dims)
    D = max(4, int(np.diff(tr[0]).max()))
    _, want = _f64_step_grads(nf, k, tr, emb, p0, D, list(range(min(bs, 13))))
    got = _sgd_grads(nf, k, tr, te, emb, p0, bs)
    assert np.allclose(got, want, rtol=2e-3, atol=2e-6), np.abs(got - want).max()
    assert np.abs(want).max() > 1e-4


def test_gradient_is_the_numerical_one_where_a_row_couples_with_itself():
    """With one row per batch the partner of every element is its own row, the softmax is the textbook one and the
    reference's backward is the true gradient; with more rows it is not (the forward mixes rows, the backward's formula
    does not differentiate that)."""
    nf, k, tr, te, emb, p0 = _problem(5, dims=(6,), p_absent=0.0, p_no_item=0.0)
    D = max(4, int(np.diff(tr[0]).max()))
    _, g = _f64_step_grads(nf, k, tr, emb, p0, D, [0])
    base = 1 + nf * k + nf
    rng = np.random.default_rng(0)
    for j in rng.choice(g.size, 25, replace=False):
        q = p0.astype(np.float64)
        q[base + j] += 1e-5
        up = _f64_step_grads(nf, k, tr, emb, q, D, [0])[0]
        q[base + j] -= 2e-5
        dn = _f64_step_grads(nf, k, tr, emb, q, D, [0])[0]
        assert abs((up - dn) / 2e-5 - g[j]) < 1e-6 + 1e-4 * abs(g[j]), j


def test_vx_gradient_order_changes_the_parameters():
    nf, k, tr, te, emb, p0 = _problem(9, dims=(5, 8, 3))
    kw = dict(n_factors=k, n_epochs=2, batch_size=5, emb=emb)
    ref = fm_oracle.fit(nf, 4, tr, te, p0, **kw)[0]
    changed = 0
    try:
        for other in ([0, 1, 2, 3], [3, 2, 1, 0], [2, 1, 3, 0]):
            fm_oracle.set_vx_grad_order(other)
            changed += fm_oracle.fit(nf, 4, tr, te, p0, **kw)[0].tobytes() != ref.tobytes()
    finally:
        fm_oracle.set_vx_grad_order(None)
    assert changed >= 2 and fm_oracle.fit(nf, 4, tr, te, p0, **kw)[0].tobytes() == ref.tobytes()


def test_no_slots_equals_the_slot_free_restatement():
    nf, k, tr, te, _, _ = _problem(11)
    p0 = fm_oracle.init_params(np.random.default_rng(1), nf, k)
    none = fm_oracle.Embeddings((), [], None, np.zeros(13, np.int32), np.zeros(9, np.int32))
    for opt in (0, 1):
        a = fm_oracle.fit(nf, 4, tr, te, p0, n_factors=k, n_epochs=3, batch_size=5, optimizer=opt, verbose=1)
        b = fm_oracle.fit(nf, 4, tr, te, p0, n_factors=k, n_epochs=3, batch_size=5, optimizer=opt, verbose=1, emb=none)
        assert a[0].tobytes() == b[0].tobytes() and a[2].tobytes() == b[2].tobytes() and a[1] == b[1]


@pytest.mark.parametrize("alt", ["softmax_rowwise", "contraction_reversed", "bias_reversed"])
def test_alternative_rule_changes_the_parameters(alt):
    """The softmax backward with each row's own sum, the x0^T dy products walking the batch last to first, and the biases'
    sums walking it last to first: each gives other parameters than the pinned rule."""
    nf, k, tr, te, emb, p0 = _problem(19, dims=(24, 5), n_train=40)
    kw = dict(n_factors=k, n_epochs=2, batch_size=13, lr=0.01, emb=emb)
    ref = fm_oracle.fit(nf, 4, tr, te, p0, **kw)[0]
    try:
        fm_oracle.set_alternative(alt)
        other = fm_oracle.fit(nf, 4, tr, te, p0, **kw)[0]
    finally:
        fm_oracle.set_alternative(None)
    base = 1 + nf * k + nf
    assert other[base:].tobytes() != ref[base:].tobytes()
    if alt != "softmax_rowwise":                              # the same mathematics in another order: only roundings differ
        assert np.allclose(other, ref, rtol=1e-3, atol=1e-5)
    assert fm_oracle.fit(nf, 4, tr, te, p0, **kw)[0].tobytes() == ref.tobytes()


def test_optimiser_uses_each_slot_tensors_own_index():
    """With V = 0 every vx is 0 and every slot gradient is exactly zero, so one SGD step with weight decay is
    p + (-lr) (wd p + 0) through MulConstAddTo and MulConstAdd, whose 8-lane block rounds twice where the rest fuses.
    k = 8, dim = 3: H, AW and EW have 24 elements (block at 16..23), the biases 8 (all block).  The fitted tensors equal the
    two kernels applied per tensor bit for bit, and differ from them applied to the slot's parameters as one vector."""
    nf, k, tr, te, emb, p0 = _problem(13, dims=(3,))
    p0 = p0.copy()
    p0[1:1 + nf * k] = 0
    wd, lr = 0.9, 0.7      # a large step, so that the product's own rounding shows in the sum
    p1 = fm_oracle.fit(nf, 4, tr, te, p0, n_factors=k, n_epochs=1, lr=lr, reg=wd, optimizer=1, batch_size=13, max_steps=1, emb=emb)[0]
    base = 1 + nf * k + nf

    def step(w):
        return fm_oracle.mul_const_add(fm_oracle.mul_const_add_to(w, wd, np.zeros_like(w)), -lr, w)

    o, per_tensor = base, []
    for n in (24, 24, 8, 24, 8):
        per_tensor.append(step(p0[o:o + n]))
        o += n
    assert o == p0.size
    assert np.concatenate(per_tensor).tobytes() == p1[base:].tobytes()
    assert step(p0[base:]).tobytes() != p1[base:].tobytes()


def test_fitted_model_ranks_and_evaluates_in_chunks():
    """Evaluation predicts each list in chunks of batch_size with the coupled softmax: the result's AUC is that of
    fm_oracle.Model's chunked batch_predict on the fitted parameters, and differs from one big chunk."""
    nf, k, tr, te, emb, p0 = _problem(17, dims=(5,), n_test=40)
    p1, res, _ = fm_oracle.fit(nf, 4, tr, te, p0, n_factors=k, n_epochs=2, batch_size=4, verbose=1, emb=emb)
    off, idx, val, tgt = te

    def preds(bs, positive):
        sel = [i for i in range(40) if (tgt[i] > 0) == positive]
        rows = [(idx[off[i]:off[i + 1]], val[off[i]:off[i + 1]]) for i in sel]
        e = np.zeros((len(sel), 5), np.float32)
        for j, i in enumerate(sel):
            t = emb.test_rows[i]
            if t >= 0 and emb.mask[t, 0]:
                e[j] = (emb.table[0][t].astype(np.uint32) << 16).view(np.float32)
        return fm_oracle.Model(nf, k, 4, bs, (5,), p1).batch_predict(rows, [e])

    m = fm_oracle.metrics(preds(4, True), preds(4, False))
    assert np.float32(m[3]).tobytes() == np.float32(res["auc"]).tobytes() and np.float32(m[0]).tobytes() == np.float32(res["precision"]).tobytes()
    assert preds(4, True).tobytes() != preds(1024, True).tobytes()
