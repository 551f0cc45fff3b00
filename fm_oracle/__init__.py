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
_SRC = [os.path.join(_HERE, "fm_oracle.c"), os.path.join(_HERE, "..", "gorse_b200", "csrc", "fm_exp.h")]


def build(force=False):
    if force or not os.path.exists(_SO) or any(os.path.getmtime(_SO) < os.path.getmtime(s) for s in _SRC):
        # -ffp-contract=off: only the explicit fmaf() calls fuse, as in the reference's floats.MM
        subprocess.check_call(["gcc", "-O2", "-std=gnu11", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-mfma",
                               "-o", _SO, _SRC[0], "-lm"])


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
