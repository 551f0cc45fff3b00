"""ctypes view of the CPU restatement of the reference's factorization-machine inference (fm_oracle/libfm_oracle.so).

TEST INFRASTRUCTURE ONLY: importable from tests/, __graft_entry__.smoke() and tools/.  The product package (gorse_b200)
never imports this.  It lives beside the general oracle (oracle/) and checks gorse_b200_fm_rank; see fm_oracle.c.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libfm_oracle.so")
_SRC = [os.path.join(_HERE, "fm_oracle.c"), os.path.join(_HERE, "fm_fit_oracle.c"), os.path.join(_HERE, "..", "gorse_b200", "csrc", "fm_exp.h"),
        os.path.join(_HERE, "..", "gorse_b200", "csrc", "fm_fit_math.h")]


def build(force=False):
    if force or not os.path.exists(_SO) or any(os.path.getmtime(_SO) < os.path.getmtime(s) for s in _SRC):
        # -ffp-contract=off: only the explicit fmaf() calls fuse, as in the reference's floats.MM
        subprocess.check_call(["gcc", "-O2", "-std=gnu11", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-mfma",
                               "-o", _SO, _SRC[0], _SRC[1], "-lm"])


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_SO)
        VP = C.c_void_p
        L.fmo_mm.argtypes = [C.c_int, C.c_int, C.c_int64, C.c_int64, C.c_int64, VP, C.c_int64, VP, C.c_int64, VP, C.c_int64]
        L.fmo_mul_to.argtypes = [VP, VP, VP, C.c_int64]
        L.fmo_add_const.argtypes = [VP, C.c_float, C.c_int64]
        L.fmo_exp.restype = C.c_float
        L.fmo_exp.argtypes = [C.c_float]
        L.fmo_softmax.argtypes = [VP, C.c_int64, C.c_int64, C.c_int]
        L.fmo_batch_predict.restype = C.c_int32
        L.fmo_batch_predict.argtypes = [C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32, VP, VP, C.c_int64, VP, VP, VP, VP,
                                        C.c_int32, VP]
        L.fmo_rank.restype = C.c_int32
        L.fmo_rank.argtypes = [C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32, VP, VP, C.c_int64, VP, VP, VP, VP, C.c_int64, VP,
                               VP, VP, VP, VP, VP, VP, VP, C.c_int32, VP, VP]
        L.fmf_logf.restype = C.c_float
        L.fmf_logf.argtypes = [C.c_float]
        L.fmf_pow_steps.restype = C.c_float
        L.fmf_pow_steps.argtypes = [C.c_float, C.c_int64]
        L.fmf_p_order.restype = C.c_int32
        L.fmf_p_order.argtypes = [VP]
        L.fmf_set_p_order.argtypes = [VP]
        L.fmf_backward_order.restype = C.c_int32
        L.fmf_backward_order.argtypes = [C.c_int32, VP, VP]
        L.fmf_set_vx_order.argtypes = [VP, C.c_int32]
        L.fmf_set_alternative.argtypes = [C.c_int32]
        L.fmf_heap_order.restype = C.c_int32
        L.fmf_heap_order.argtypes = [C.c_int32, VP, VP]
        L.fmf_op_softmax.argtypes = [VP, C.c_int64, C.c_int64, VP, C.c_int32, VP, VP]
        L.fmo_dot.restype = C.c_float
        L.fmo_dot.argtypes = [VP, VP, C.c_int64]
        L.fmf_mul_const_add_to.argtypes = [VP, C.c_float, VP, VP, C.c_int64]
        L.fmf_mul_const_add.argtypes = [VP, C.c_float, VP, C.c_int64]
        L.fmf_metrics.argtypes = [C.c_int64, VP, C.c_int64, VP, VP]
        L.fmf_evaluate.argtypes = [C.c_int64, C.c_int32, C.c_int32, VP, C.c_int64, VP, VP, VP, VP, VP]
        L.fmf_op_binary.argtypes = [C.c_int32, VP, C.c_int64, VP, C.c_int64, VP, VP, VP, VP]
        L.fmf_op_unary.argtypes = [C.c_int32, VP, C.c_int64, VP, VP, VP]
        L.fmf_op_sum.argtypes = [C.c_int32, VP, C.c_int64, C.c_float, VP, VP]
        L.fmf_op_sum_axis.argtypes = [VP, C.c_int64, C.c_int64, C.c_int64, VP, VP, VP]
        L.fmf_op_bmm.argtypes = [C.c_int32, C.c_int32, C.c_int64, C.c_int64, C.c_int64, C.c_int64, C.c_int64, VP, VP, VP, VP, VP, VP]
        L.fmf_op_embedding.argtypes = [VP, C.c_int64, C.c_int64, VP, C.c_int64, VP, VP, VP]
        L.fmf_op_broadcast.argtypes = [VP, C.c_int64, C.c_int64, VP, VP, VP]
        L.fmf_fit.restype = C.c_int32
        L.fmf_fit.argtypes = [C.c_int64, C.c_int32, VP, VP, C.c_int64, C.c_int64, VP, VP, VP, VP, C.c_int64, VP, VP, VP, VP, VP, VP, VP, VP, VP]
        L.fmf_fit_emb.restype = C.c_int32
        L.fmf_fit_emb.argtypes = [C.c_int64, C.c_int32, VP, VP, C.c_int64, C.c_int64, VP, VP, VP, VP, C.c_int64, VP, VP, VP, VP, C.c_int32, VP, VP,
                                  VP, VP, VP, VP, VP, VP, VP, VP]
        _lib = L
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _c(a, dt):
    return np.ascontiguousarray(a, dt)


def mm(transA, transB, m, n, k, a, lda, b, ldb, c, ldc):
    """floats.MM restated (c += op(a) op(b), a fused chain over the contracted index); c updated in place"""
    assert a.dtype == b.dtype == c.dtype == np.float32 and c.flags.c_contiguous
    lib().fmo_mm(int(transA), int(transB), m, n, k, _p(_c(a, np.float32)), lda, _p(_c(b, np.float32)), ldb, _p(c), ldc)


def dot(a, b):
    """floats.Dot restated: what floats.MM's transB path assigns to every output element"""
    a, b = _c(a, np.float32), _c(b, np.float32)
    return np.float32(lib().fmo_dot(_p(a), _p(b), a.size))


def mul_to(a, b):
    a, b = _c(a, np.float32), _c(b, np.float32)
    c = np.empty_like(a)
    lib().fmo_mul_to(_p(a), _p(b), _p(c), a.size)
    return c


def add_const(a, c):
    a = _c(a, np.float32).copy()
    lib().fmo_add_const(_p(a), float(c), a.size)
    return a


def exp(x):
    return np.float32(lib().fmo_exp(float(x)))


def softmax(x, coupled=True):
    """Softmax(x, 1) of a [B, dim] tensor: the reference's (coupled) or the row-wise one"""
    y = _c(x, np.float32).copy()
    lib().fmo_softmax(_p(y), y.shape[0], y.shape[1], int(coupled))
    return y


class Model:
    """The parameters of an AFM as gorse_b200_fm_create takes them (fm.Parameters() concatenated)."""

    def __init__(self, n_features, n_factors, num_dimension, batch_size, emb_dims, params):
        self.n_features, self.k, self.num_dimension, self.batch_size = int(n_features), int(n_factors), int(num_dimension), int(batch_size)
        self.emb_dims = _c(list(emb_dims), np.int32)
        self.params = _c(params, np.float32)

    def _head(self):
        return (self.n_features, self.k, self.num_dimension, self.batch_size, self.emb_dims.size, _p(self.emb_dims), _p(self.params))

    def batch_predict(self, rows, emb=(), coupled=True):
        """BatchInternalPredict on built rows: rows = [(indices, values)], emb[s] = float32 [n, dim_s]"""
        n = len(rows)
        off = np.zeros(n + 1, np.int64)
        np.cumsum([len(r[0]) for r in rows], out=off[1:])
        idx = _c(np.concatenate([np.asarray(r[0], np.int32) for r in rows] + [np.zeros(1, np.int32)]), np.int32)
        val = _c(np.concatenate([np.asarray(r[1], np.float32) for r in rows] + [np.zeros(1, np.float32)]), np.float32)
        es = [_c(e, np.float32) for e in emb]
        arr = (C.c_void_p * max(len(es), 1))(*[_p(e) for e in es])
        out = np.zeros(max(n, 1), np.float32)
        assert lib().fmo_batch_predict(*self._head(), n, _p(off), _p(idx), _p(val), arr, int(coupled), _p(out)) == 0
        return out[:n]

    def rank(self, inp, coupled=True):
        """gorse_b200_fm_rank restated; inp is an FMInput-like object (see gorse_b200.FMRanker.rank) -> (scores, order)"""
        n_emb = self.emb_dims.size
        embs = [_c(e, np.uint16) for e in inp.item_emb]
        arr = (C.c_void_p * max(n_emb, 1))(*[_p(e) for e in embs])
        total = int(inp.cand_off[-1])
        scores, order = np.zeros(max(total, 1), np.float32), np.zeros(max(total, 1), np.int32)
        assert lib().fmo_rank(*self._head(), inp.n_users, _p(inp.user_feat), _p(inp.user_lab_off), _p(inp.user_lab_idx), _p(inp.user_lab_val),
                              inp.n_items, _p(inp.item_feat), _p(inp.item_lab_off), _p(inp.item_lab_idx), _p(inp.item_lab_val), arr,
                              _p(inp.item_emb_mask), _p(inp.cand_off), _p(inp.cand_items), int(coupled), _p(scores), _p(order)) == 0
        return scores[:total], order[:total]


# ---- FM training (fm_fit_oracle.c) -------------------------------------------------------------------------------------
P_GRAD_NAMES = ("ReLU", "Mul", "Abs")


def logf(x):
    return np.float32(lib().fmf_logf(float(x)))


def pow_steps(beta, t):
    return np.float32(lib().fmf_pow_steps(float(beta), int(t)))


def p_grad_order():
    """the order in which ReLU (0), Mul (1) and Abs (2) hand their gradients to the logit, from the replayed backward heap"""
    out = np.zeros(3, np.int32)
    assert lib().fmf_p_order(_p(out)) == 0
    return out.tolist()


def set_p_grad_order(order=None):
    """tests only: make fit() add the logit's gradients in another order (None: the replayed one)"""
    lib().fmf_set_p_order(None if order is None else _p(_c(order, np.int32)))


VX_GRAD_NAMES = ("Square", "BMM slot 0", "BMM slot 1", "BMM slot 2", "BMM slot 3", "BMM slot 4", "BMM slot 5", "BMM slot 6", "BMM slot 7")


def backward_order(n_emb):
    """-> (the order of p's gradients as p_grad_order gives it, the order in which Square (0) and slot s's BMM (1 + s) hand
    their gradients to vx), from the backward heap replayed on the graph with n_emb slots"""
    p, vx = np.zeros(3, np.int32), np.zeros(1 + n_emb, np.int32)
    assert lib().fmf_backward_order(int(n_emb), _p(p), _p(vx)) == 0
    return p.tolist(), vx.tolist()


def set_vx_grad_order(order=None):
    """tests only: make fit() add vx's gradients in another order (None: the replayed one)"""
    lib().fmf_set_vx_order(None if order is None else _p(_c(order, np.int32)), 0 if order is None else len(order))


ALTERNATIVES = {"softmax_rowwise": 1, "contraction_reversed": 2, "bias_reversed": 4}


def set_alternative(name=None):
    """tests only: make fit() use the alternative to one pinned rule of the slots' backward (None: the pinned rules)"""
    lib().fmf_set_alternative(0 if name is None else ALTERNATIVES[name])


def heap_order(inputs):
    """Tensor.Backward's pop order on a graph: inputs[o] = the (up to two) ops producing op o's inputs, -1 for a leaf, in
    creation order; the last op is the one Backward is called on"""
    a = _c([(list(i) + [-1, -1])[:2] for i in inputs], np.int32)
    out = np.zeros(len(inputs), np.int32)
    n = lib().fmf_heap_order(len(inputs), _p(a), _p(out))
    assert n >= 0
    return out[:n].tolist()


def op_softmax(x, dy=None, coupled=True):
    """Softmax(x, 1) of a [B, dim] tensor -> (y, dx)"""
    x = _c(x, np.float32)
    dy = np.ones(x.shape, np.float32) if dy is None else _c(dy, np.float32)
    y, g = np.empty_like(x), np.empty_like(x)
    lib().fmf_op_softmax(_p(x), x.shape[0], x.shape[1], _p(dy), int(coupled), _p(y), _p(g))
    return y, g


# the ops of the training graph as the restatement forms them (fmf_op_*): forward and gradients for an output gradient dy
# (default: ones, what Tensor.Backward seeds)
_BINARY = {"add": 0, "sub": 1, "mul": 2, "div": 3}
_UNARY = {"square": 0, "exp": 1, "log": 2, "abs": 3, "relu": 4, "neg": 5}


def op_binary(name, x0, x1, dy=None):
    """-> (y, dx0, dx1); x1 broadcasts over x0 as a suffix"""
    x0, x1 = _c(x0, np.float32), _c(x1, np.float32)
    dy = np.ones(x0.shape, np.float32) if dy is None else _c(dy, np.float32)
    y, g0, g1 = np.empty_like(x0), np.empty_like(x0), np.empty_like(x1)
    lib().fmf_op_binary(_BINARY[name], _p(x0), x0.size, _p(x1), x1.size, _p(dy), _p(y), _p(g0), _p(g1))
    return y, g0, g1


def op_unary(name, x, dy=None):
    x = _c(x, np.float32)
    dy = np.ones(x.shape, np.float32) if dy is None else _c(dy, np.float32)
    y, g = np.empty_like(x), np.empty_like(x)
    lib().fmf_op_unary(_UNARY[name], _p(x), x.size, _p(dy), _p(y), _p(g))
    return y, g


def op_sum(x, mean=False, dy=1.0):
    x = _c(x, np.float32)
    y, g = np.zeros(1, np.float32), np.empty_like(x)
    lib().fmf_op_sum(int(mean), _p(x), x.size, float(dy), _p(y), _p(g))
    return y, g


def op_sum_axis(x, axis, dy=None):
    x = _c(x, np.float32)
    s1, s2, s3 = int(np.prod(x.shape[:axis])), x.shape[axis], int(np.prod(x.shape[axis + 1:]))
    oshape = x.shape[:axis] + x.shape[axis + 1:]
    dy = np.ones(oshape, np.float32) if dy is None else _c(dy, np.float32)
    y, g = np.empty(oshape, np.float32), np.empty_like(x)
    lib().fmf_op_sum_axis(_p(x), s1, s2, s3, _p(dy), _p(y), _p(g))
    return y, g


def op_bmm(x, y, t1=False, t2=False, dz=None):
    """BMM of x [b, xr, xc] and y [b, yr, yc] -> (z, dx, dy)"""
    x, y = _c(x, np.float32), _c(y, np.float32)
    b, xr, xc = x.shape
    _, yr, yc = y.shape
    m, n = (xc if t1 else xr), (yr if t2 else yc)
    dz = np.ones((b, m, n), np.float32) if dz is None else _c(dz, np.float32)
    z, gx, gy = np.empty((b, m, n), np.float32), np.empty_like(x), np.empty_like(y)
    lib().fmf_op_bmm(int(t1), int(t2), b, xr, xc, yr, yc, _p(x), _p(y), _p(dz), _p(z), _p(gx), _p(gy))
    return z, gx, gy


def op_embedding(w, idx, dy=None):
    w, idx = _c(w, np.float32), _c(idx, np.float32)
    rows, dim = w.shape[0], int(np.prod(w.shape[1:]))
    dy = np.ones(idx.shape + w.shape[1:], np.float32) if dy is None else _c(dy, np.float32)
    y, gw = np.empty(idx.shape + w.shape[1:], np.float32), np.empty_like(w)
    lib().fmf_op_embedding(_p(w), rows, dim, _p(idx), idx.size, _p(dy), _p(y), _p(gw))
    return y, gw


def op_broadcast(x, w, dy=None):
    x = _c(x, np.float32)
    dy = np.ones(x.shape + (w,), np.float32) if dy is None else _c(dy, np.float32)
    y, g = np.empty(x.shape + (w,), np.float32), np.empty_like(x)
    lib().fmf_op_broadcast(_p(x), x.size, w, _p(dy), _p(y), _p(g))
    return y, g


def mul_const_add_to(a, c, b):
    a, b = _c(a, np.float32), _c(b, np.float32)
    d = np.empty_like(a)
    lib().fmf_mul_const_add_to(_p(a), float(c), _p(b), _p(d), a.size)
    return d


def mul_const_add(a, c, dst):
    a, d = _c(a, np.float32), _c(dst, np.float32).copy()
    lib().fmf_mul_const_add(_p(a), float(c), _p(d), a.size)
    return d


def metrics(pos_pred, neg_pred):
    """Precision, Recall, Accuracy, AUC of two prediction lists (evaluator.go:85-153)"""
    p, n = _c(pos_pred, np.float32).copy(), _c(neg_pred, np.float32).copy()
    out = np.zeros(4, np.float32)
    lib().fmf_metrics(p.size, _p(p), n.size, _p(n), _p(out))
    return out


def _rows(r):
    off, idx, val, tgt = r
    return (len(off) - 1, _c(off, np.int64), _c(np.concatenate([np.asarray(idx, np.int32), [0]]), np.int32),
            _c(np.concatenate([np.asarray(val, np.float32), [0]]), np.float32), _c(np.concatenate([np.asarray(tgt, np.float32), [0]]), np.float32))


def evaluate(n_features, k, num_dimension, params, test):
    n, off, idx, val, tgt = _rows(test)
    out = np.zeros(4, np.float32)
    lib().fmf_evaluate(int(n_features), int(k), int(num_dimension), _p(_c(params, np.float32)), n, _p(off), _p(idx), _p(val), _p(tgt), _p(out))
    return out


class Embeddings:
    """The item-embedding side of a fit: dims [n_emb], table[s] = bf16 bits [n_rows, dim_s], mask [n_rows, n_emb] uint8 or
    None (every embedding present), and the table row (-1: none) of every training and test sample."""

    def __init__(self, dims, table, mask, train_rows, test_rows):
        self.dims = _c(list(dims), np.int32)
        self.table = [_c(t, np.uint16) for t in table]
        self.n_rows = self.table[0].shape[0] if self.table else 0
        self.mask = None if mask is None else _c(mask, np.uint8)
        self.train_rows, self.test_rows = _c(np.append(train_rows, 0), np.int32)[:-1], _c(np.append(test_rows, 0), np.int32)[:-1]

    def n_slot_params(self, k):
        return int(sum(3 * k * int(d) + 2 * k for d in self.dims))


def fit(n_features, num_dimension, train, test, params_in, n_factors=16, n_epochs=50, lr=0.001, reg=0.0002, optimizer=0, batch_size=1024,
        verbose=10, patience=10, max_steps=0, cancel_epoch=-1, emb=None):
    """AFM.Fit restated (see fm_fit_oracle.c); train / test = (off, idx, val, target); emb = Embeddings for a model with slots.
    -> (params, result dict with gorse_b200_fm_fit_result's fields, moments [2, n_params])"""
    tr, te = _rows(train), _rows(test)
    pin = _c(params_in, np.float32)
    pout, mom = np.zeros(pin.size, np.float32), np.zeros((2, pin.size), np.float32)
    ip = _c([n_factors, n_epochs, optimizer, batch_size, verbose, patience, cancel_epoch], np.int32)
    fp = _c([lr, reg], np.float32)
    rf, ri = np.zeros(5, np.float32), np.zeros(6, np.int64)
    head = (int(n_features), int(num_dimension), _p(ip), _p(fp), int(max_steps), tr[0], _p(tr[1]), _p(tr[2]), _p(tr[3]), _p(tr[4]),
            te[0], _p(te[1]), _p(te[2]), _p(te[3]), _p(te[4]))
    if emb is None:
        assert lib().fmf_fit(*head, _p(pin), _p(pout), _p(mom), _p(rf), _p(ri)) == 0
    else:
        arr = (C.c_void_p * max(len(emb.table), 1))(*[_p(t) for t in emb.table])
        tr_row, te_row = np.append(emb.train_rows, 0).astype(np.int32), np.append(emb.test_rows, 0).astype(np.int32)
        assert lib().fmf_fit_emb(*head, emb.dims.size, _p(emb.dims), arr, _p(emb.mask), _p(tr_row), _p(te_row), _p(pin), _p(pout), _p(mom),
                                 _p(rf), _p(ri)) == 0
    res = dict(zip(("auc", "precision", "recall", "accuracy", "cost"), (np.float32(x) for x in rf)))
    res.update(zip(("epochs_run", "best_epoch", "early_stopped", "diverged", "cancelled", "steps"), (int(x) for x in ri)))
    return pout, res, mom


def random_ctr(rng, n_features, n_rows, labels=4, p_num=0.3, n_ids=None):
    """CTR rows shaped like the reference's: a user id, an item id and 0 .. labels label features (numerical with
    probability p_num), target +1 or -1.  -> (off, idx, val, target)"""
    n_ids = n_ids or n_features
    lens = 2 + rng.integers(0, labels + 1, n_rows)
    off = np.zeros(n_rows + 1, np.int64)
    np.cumsum(lens, out=off[1:])
    idx = rng.integers(0, n_features, int(off[-1])).astype(np.int32)
    idx[off[:-1]] = rng.integers(0, n_ids, n_rows)
    val = np.where(rng.random(int(off[-1])) < p_num, rng.standard_normal(int(off[-1])), 1.0).astype(np.float32)
    val[off[:-1]] = 1.0
    tgt = np.where(rng.random(n_rows) < 0.5, 1.0, -1.0).astype(np.float32)
    return off, idx, val, tgt


def init_params(rng, n_features, k, std=0.01, emb_dims=()):
    """B = 0, V and W ~ N(0, std) as AFM.Init draws them (fm.go:254-256, nn.NewEmbedding); per slot H ~ N(0, std), AW and EW
    uniform in +-1/sqrt(dim), Ab = Eb = 0 (NewAttention, NewLinear, layers.go:42-48, 166-171)"""
    parts = [[0.0], rng.standard_normal(n_features * k) * std, rng.standard_normal(n_features) * std]
    for d in emb_dims:
        b = 1 / np.sqrt(d)
        parts += [rng.standard_normal(k * d) * std, rng.uniform(-b, b, d * k), np.zeros(k), rng.uniform(-b, b, d * k), np.zeros(k)]
    return np.concatenate(parts).astype(np.float32)


def random_embeddings(rng, n_rows, dims, n_train, n_test, p_absent=0.15, p_no_item=0.1):
    """A seeded Embeddings: a bf16 table, slots absent with probability p_absent, samples without an item with p_no_item"""
    table = [to_bf16(rng.standard_normal((n_rows, d), dtype=np.float32)) for d in dims]
    mask = (rng.random((n_rows, len(dims))) >= p_absent).astype(np.uint8)
    rows = [np.where(rng.random(n) < p_no_item, -1, rng.integers(0, n_rows, n)).astype(np.int32) for n in (n_train, n_test)]
    return Embeddings(dims, table, mask, rows[0], rows[1])


# ---- seeded models and inputs (tests and tools/fm_rank_bench.py) ---------------------------------------------------------
def random_params(rng, n_features, k, emb_dims=()):
    """fm.Parameters() of a model with the shapes of NewAFM / Init (values scaled so that the softmax is not flat)"""
    f32 = np.float32
    parts = [rng.standard_normal(1, dtype=f32) * f32(0.1), rng.standard_normal(n_features * k, dtype=f32) * f32(0.3),
             rng.standard_normal(n_features, dtype=f32) * f32(0.3)]
    for d in emb_dims:
        b = f32(1 / np.sqrt(d))
        parts += [rng.standard_normal(k * d, dtype=f32), rng.uniform(-b, b, d * k).astype(f32) * f32(4),
                  rng.standard_normal(k, dtype=f32) * f32(0.1), rng.uniform(-b, b, d * k).astype(f32),
                  rng.standard_normal(k, dtype=f32) * f32(0.1)]
    return np.concatenate(parts).astype(np.float32)


def to_bf16(a):
    """float32 -> bf16 bits (truncation)"""
    return (np.ascontiguousarray(a, np.float32).view(np.uint32) >> 16).astype(np.uint16)


def random_input(rng, n_features, cand_counts, n_items, emb_dims=(), labels=5, p_unknown=0.2, p_no_emb=0.2):
    """An FMInput-compatible namespace: ids unknown with probability p_unknown, 0 .. 2*labels labels per user and item,
    embeddings missing with probability p_no_emb, candidates drawn with repeats."""
    import types

    def feats(n):
        feat = np.where(rng.random(n) < p_unknown, -1, rng.integers(0, n_features, n)).astype(np.int32)
        cnt = rng.integers(0, 2 * labels + 1, n)
        off = np.zeros(n + 1, np.int64)
        np.cumsum(cnt, out=off[1:])
        idx = rng.integers(0, n_features, int(off[-1]) + 1).astype(np.int32)
        val = np.where(rng.random(int(off[-1]) + 1) < 0.5, 1.0, rng.standard_normal(int(off[-1]) + 1)).astype(np.float32)
        return feat, off, idx, val

    ns = types.SimpleNamespace()
    ns.n_users, ns.n_items = len(cand_counts), n_items
    ns.user_feat, ns.user_lab_off, ns.user_lab_idx, ns.user_lab_val = feats(ns.n_users)
    ns.item_feat, ns.item_lab_off, ns.item_lab_idx, ns.item_lab_val = feats(n_items)
    ns.cand_off = np.zeros(ns.n_users + 1, np.int64)
    np.cumsum(cand_counts, out=ns.cand_off[1:])
    ns.cand_items = rng.integers(0, n_items, int(ns.cand_off[-1]) + 1).astype(np.int32)
    ns.item_emb = [to_bf16(rng.standard_normal((n_items, d), dtype=np.float32)) for d in emb_dims]
    ns.item_emb_mask = (rng.random((n_items, len(emb_dims))) >= p_no_emb).astype(np.uint8) if len(emb_dims) else None
    return ns
