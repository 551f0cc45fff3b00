"""The ops of the FM training restatement (fm_oracle/fm_fit_oracle.c, fmf_op_*) pinned on the known answers of the
reference's common/nn/op_test.go: forward values and the gradients Tensor.Backward seeds with ones.  The restatement's
training step uses the same per-element rules, so these tie its graph to the reference's ops.  Where op_test.go checks a
gradient against a numerical derivative, so does this file, with the same step and tolerances (:24-57)."""
import numpy as np

import fm_oracle

EPS, RTOL, ATOL = 1e-4, 1e-2, 5e-3
X6 = np.array([1, 2, 3, 4, 5, 6], np.float32).reshape(2, 3)
Y6 = np.array([2, 3, 4, 5, 6, 7], np.float32).reshape(2, 3)


def numerical(f, x):
    """op_test.go numericalDiff: the sum over outputs of the central difference"""
    x = np.array(x, np.float32)
    dx = np.zeros(x.size, np.float32)
    for i in range(x.size):
        x0, x1 = x.copy().reshape(-1), x.copy().reshape(-1)
        x0[i] -= np.float32(EPS)
        x1[i] += np.float32(EPS)
        y0, y1 = f(x0.reshape(x.shape)), f(x1.reshape(x.shape))
        dx[i] = np.sum((y1.astype(np.float64) - y0) / (2 * EPS))
    return dx.reshape(x.shape)


def all_close(a, b):
    assert a.shape == b.shape
    assert np.all(np.abs(a - b) <= ATOL + RTOL * np.abs(b)), (a, b)


def rand(rng, *shape):
    return rng.random(shape).astype(np.float32)


def test_add():
    y, _, _ = fm_oracle.op_binary("add", X6, Y6)
    assert y.reshape(-1).tolist() == [3, 5, 7, 9, 11, 13]
    rng = np.random.default_rng(0)
    x, yy = rand(rng, 2, 3), rand(rng, 2, 3)
    _, gx, gy = fm_oracle.op_binary("add", x, yy)
    all_close(gx, numerical(lambda v: fm_oracle.op_binary("add", v, yy)[0], x))
    all_close(gy, numerical(lambda v: fm_oracle.op_binary("add", x, v)[0], yy))
    y, gx, gy = fm_oracle.op_binary("add", X6, [2])
    assert y.reshape(-1).tolist() == [3, 4, 5, 6, 7, 8] and gx.reshape(-1).tolist() == [1] * 6 and gy.tolist() == [6]
    y, gx, gy = fm_oracle.op_binary("add", X6, [2, 3, 4])
    assert y.reshape(-1).tolist() == [3, 5, 7, 6, 8, 10] and gx.reshape(-1).tolist() == [1] * 6 and gy.tolist() == [2, 2, 2]


def test_sub():
    y, _, _ = fm_oracle.op_binary("sub", X6, Y6)
    assert y.reshape(-1).tolist() == [-1] * 6
    rng = np.random.default_rng(1)
    x, yy = rand(rng, 2, 3), rand(rng, 2, 3)
    _, gx, gy = fm_oracle.op_binary("sub", x, yy)
    all_close(gx, numerical(lambda v: fm_oracle.op_binary("sub", v, yy)[0], x))
    all_close(gy, numerical(lambda v: fm_oracle.op_binary("sub", x, v)[0], yy))
    y, gx, gy = fm_oracle.op_binary("sub", X6, [2])
    assert y.reshape(-1).tolist() == [-1, 0, 1, 2, 3, 4] and gx.reshape(-1).tolist() == [1] * 6 and gy.tolist() == [-6]
    y, gx, gy = fm_oracle.op_binary("sub", X6, [2, 3, 4])
    assert y.reshape(-1).tolist() == [-1, -1, -1, 2, 2, 2] and gx.reshape(-1).tolist() == [1] * 6 and gy.tolist() == [-2, -2, -2]


def test_mul():
    y, _, _ = fm_oracle.op_binary("mul", X6, Y6)
    assert y.reshape(-1).tolist() == [2, 6, 12, 20, 30, 42]
    rng = np.random.default_rng(2)
    x, yy = rand(rng, 2, 3), rand(rng, 2, 3)
    _, gx, gy = fm_oracle.op_binary("mul", x, yy)
    all_close(gx, numerical(lambda v: fm_oracle.op_binary("mul", v, yy)[0], x))
    all_close(gy, numerical(lambda v: fm_oracle.op_binary("mul", x, v)[0], yy))
    y, gx, gy = fm_oracle.op_binary("mul", X6, [2])
    assert y.reshape(-1).tolist() == [2, 4, 6, 8, 10, 12] and gx.reshape(-1).tolist() == [2] * 6 and gy.tolist() == [21]
    y, gx, gy = fm_oracle.op_binary("mul", X6, [2, 3, 4])
    assert y.reshape(-1).tolist() == [2, 6, 12, 8, 15, 24] and gx.reshape(-1).tolist() == [2, 3, 4, 2, 3, 4] and gy.tolist() == [5, 7, 9]


def test_div():
    y, gx, gy = fm_oracle.op_binary("div", X6, Y6)
    assert np.allclose(y.reshape(-1), [0.5, 2 / 3, 0.75, 4 / 5, 5 / 6, 6 / 7], rtol=0, atol=1e-6)
    all_close(gx, numerical(lambda v: fm_oracle.op_binary("div", v, Y6)[0], X6))
    all_close(gy, numerical(lambda v: fm_oracle.op_binary("div", X6, v)[0], Y6))
    y, gx, gy = fm_oracle.op_binary("div", X6, [2])
    assert np.allclose(y.reshape(-1), [0.5, 1, 1.5, 2, 2.5, 3], rtol=0, atol=1e-6)
    assert np.allclose(gx, 0.5, rtol=0, atol=1e-6) and np.allclose(gy, [-21 / 4], rtol=0, atol=1e-6)
    y, gx, gy = fm_oracle.op_binary("div", X6, [2, 3, 4])
    assert np.allclose(y.reshape(-1), [0.5, 2 / 3, 3 / 4, 2, 5 / 3, 1.5], rtol=0, atol=1e-6)
    assert np.allclose(gx.reshape(-1), [1 / 2, 1 / 3, 1 / 4, 1 / 2, 1 / 3, 1 / 4], rtol=0, atol=1e-6)
    assert np.allclose(gy, [-5 / 4, -7 / 9, -9 / 16], rtol=0, atol=1e-6)


def test_square():
    assert fm_oracle.op_unary("square", X6)[0].reshape(-1).tolist() == [1, 4, 9, 16, 25, 36]
    x = rand(np.random.default_rng(3), 2, 3)
    all_close(fm_oracle.op_unary("square", x)[1], numerical(lambda v: fm_oracle.op_unary("square", v)[0], x))


def test_exp():
    y, _ = fm_oracle.op_unary("exp", np.arange(6, dtype=np.float32).reshape(2, 3))
    assert np.allclose(y.reshape(-1), np.exp(np.arange(6, dtype=np.float64)).astype(np.float32), rtol=0, atol=1e-5)
    x = rand(np.random.default_rng(4), 2, 3)
    all_close(fm_oracle.op_unary("exp", x)[1], numerical(lambda v: fm_oracle.op_unary("exp", v)[0], x))


def test_log():
    y, _ = fm_oracle.op_unary("log", X6)
    assert np.allclose(y.reshape(-1), np.log(np.arange(1, 7, dtype=np.float64)).astype(np.float32), rtol=0, atol=1e-6)
    x = (1 + rand(np.random.default_rng(5), 2, 3)).astype(np.float32)   # Uniform(1, 2)
    all_close(fm_oracle.op_unary("log", x)[1], numerical(lambda v: fm_oracle.op_unary("log", v)[0], x))


def test_abs():
    assert fm_oracle.op_unary("abs", [[1, -2, 3], [-4, 5, -6]])[0].reshape(-1).tolist() == [1, 2, 3, 4, 5, 6]
    x = np.array([[-0.9, -0.5, -0.1], [0.1, 0.5, 0.9]], np.float32)   # away from 0, where Abs is not differentiable
    _, g = fm_oracle.op_unary("abs", x)
    all_close(g, numerical(lambda v: fm_oracle.op_unary("abs", v)[0], x))
    # at 0 the reference keeps dy (x < 0 is false), also for -0
    assert fm_oracle.op_unary("abs", [0.0, -0.0], dy=[3.0, 3.0])[1].tolist() == [3.0, 3.0]


def test_relu():
    assert fm_oracle.op_unary("relu", [[-1, 0, 1], [2, 3, 4]])[0].reshape(-1).tolist() == [0, 0, 1, 2, 3, 4]
    x = rand(np.random.default_rng(6), 2, 3)
    all_close(fm_oracle.op_unary("relu", x)[1], numerical(lambda v: fm_oracle.op_unary("relu", v)[0], x))


def test_neg():
    y, g = fm_oracle.op_unary("neg", X6, dy=Y6)
    assert y.tolist() == (-X6).tolist() and g.tolist() == (-Y6).tolist()


def test_sum():
    y, g = fm_oracle.op_sum(X6)
    assert y.tolist() == [21] and g.reshape(-1).tolist() == [1] * 6
    x = np.array([1, 2, 3, 4, 5, 6, 1, 2, 3, 4, 5, 6], np.float32).reshape(2, 3, 2)
    y, g = fm_oracle.op_sum_axis(x, 1)
    assert y.shape == (2, 2) and y.reshape(-1).tolist() == [9, 12, 9, 12]
    assert g.shape == (2, 3, 2) and g.reshape(-1).tolist() == [1] * 12


def test_mean():
    y, g = fm_oracle.op_sum(X6, mean=True)
    assert y.tolist() == [3.5]
    assert g.reshape(-1).tolist() == [np.float32(1.0 / 6)] * 6


def test_bmm():
    x = np.array([1, 2, 3, 4, 5, 6, 1, 2, 3, 4, 5, 6], np.float32).reshape(2, 2, 3)
    y = np.tile(np.arange(1, 13, dtype=np.float32), 2).reshape(2, 3, 4)
    z, gx, gy = fm_oracle.op_bmm(x, y)
    assert z.shape == (2, 2, 4) and z.reshape(-1).tolist() == [38, 44, 50, 56, 83, 98, 113, 128] * 2
    assert gx.reshape(-1).tolist() == [10, 26, 42, 10, 26, 42] * 2
    assert gy.reshape(-1).tolist() == [5, 5, 5, 5, 7, 7, 7, 7, 9, 9, 9, 9] * 2
    rng = np.random.default_rng(7)
    for t1, t2, xs, ys in ((True, False, (2, 3, 2), (2, 3, 4)), (False, True, (2, 2, 3), (2, 4, 3)), (True, True, (2, 3, 2), (2, 4, 3))):
        a, b = rand(rng, *xs), rand(rng, *ys)
        z, ga, gb = fm_oracle.op_bmm(a, b, t1, t2)
        assert z.shape == (2, 2, 4) and ga.shape == xs and gb.shape == ys
        all_close(ga, numerical(lambda v: fm_oracle.op_bmm(v, b, t1, t2)[0], a))
        all_close(gb, numerical(lambda v: fm_oracle.op_bmm(a, v, t1, t2)[0], b))


def test_broadcast():
    y, g = fm_oracle.op_broadcast([1, 2], 3)
    assert y.reshape(-1).tolist() == [1, 1, 1, 2, 2, 2] and g.tolist() == [3, 3]


def test_embedding():
    idx = np.array([0, 1, 0, 3, 0, 5], np.float32).reshape(2, 3)
    for shape in ((6, 2), (6, 1, 2)):
        w = np.arange(12, dtype=np.float32).reshape(shape)
        y, gw = fm_oracle.op_embedding(w, idx)
        assert y.shape == (2, 3) + shape[1:]
        assert y.reshape(-1).tolist() == [0, 1, 2, 3, 0, 1, 6, 7, 0, 1, 10, 11]
        assert gw.reshape(-1).tolist() == [3, 3, 1, 1, 0, 0, 1, 1, 0, 0, 1, 1]
