"""ctypes view of the CPU oracle (oracle/libgorse_oracle.so).

TEST INFRASTRUCTURE ONLY: importable from tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs.  The product package (gorse_b200) never imports this.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libgorse_oracle.so")
REF_SO = os.path.join(_HERE, "_ref", "libfloats_ref.so")

METRIC_EUCLIDEAN = 0
METRIC_NEG_DOT = 1


REF_KERNELS = os.path.join("common", "floats", "src", "floats_avx512.c")


def reference_dir():
    """The checkout of the reference project whose C kernels oracle/_ref is built from: $GORSE_REFERENCE_DIR, else a
    directory named `reference` next to this repository or next to any directory above it; None when there is none."""
    env = os.environ.get("GORSE_REFERENCE_DIR")
    if env:
        return env if os.path.isfile(os.path.join(env, REF_KERNELS)) else None
    d = os.path.dirname(os.path.dirname(_HERE))   # the directory holding the repository
    while True:
        cand = os.path.join(d, "reference")
        if os.path.isfile(os.path.join(cand, REF_KERNELS)):
            return cand
        up = os.path.dirname(d)
        if up == d:
            return None
        d = up


def build(force=False):
    """Compile the oracle and, whenever the reference project is found (reference_dir()), oracle/_ref from its own C
    kernels.  Without the reference a prebuilt oracle/_ref is kept; a missing one is reported on stderr, because the CPU
    baseline then times the oracle port and the reference-comparison tests fall back to stored outputs."""
    src_newer = (not os.path.exists(_SO)) or os.path.getmtime(_SO) < os.path.getmtime(
        os.path.join(_HERE, "gorse_oracle.c"))
    ref = reference_dir()
    if force or src_newer or (ref and not os.path.exists(REF_SO)):
        env = dict(os.environ, GORSE_REFERENCE_DIR=ref or "")
        subprocess.check_call(["make", "-C", _HERE, "--no-print-directory"], stdout=subprocess.DEVNULL, env=env)
    if not os.path.exists(REF_SO):
        print("oracle: the reference project was not found (set GORSE_REFERENCE_DIR to its checkout); oracle/_ref is not "
              "built: CPU baselines time the oracle port and the reference-comparison tests use stored outputs",
              file=sys.stderr)


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_SO):
            build()
        _lib = C.CDLL(_SO)
        _sig(_lib)
    return _lib


def _p(dt):
    return np.ctypeslib.ndpointer(dtype=dt, flags="C_CONTIGUOUS")


F32, I32, I64 = _p(np.float32), _p(np.int32), _p(np.int64)


def _sig(L):
    L.gbo_dot.restype = C.c_float
    L.gbo_dot.argtypes = [F32, F32, C.c_int64]
    L.gbo_euclidean.restype = C.c_float
    L.gbo_euclidean.argtypes = [F32, F32, C.c_int64]
    L.gbo_dot_scalar.restype = C.c_float
    L.gbo_dot_scalar.argtypes = [F32, F32, C.c_int64]
    L.gbo_euclidean_scalar.restype = C.c_float
    L.gbo_euclidean_scalar.argtypes = [F32, F32, C.c_int64]
    L.gbo_mul_const_to.argtypes = [F32, C.c_float, F32, C.c_int64]
    L.gbo_mul_const_add.argtypes = [F32, C.c_float, F32, C.c_int64]
    L.gbo_mul_const_add_to.argtypes = [F32, C.c_float, F32, F32, C.c_int64]
    L.gbo_mul_const.argtypes = [F32, C.c_float, C.c_int64]
    L.gbo_sub_to.argtypes = [F32, F32, F32, C.c_int64]
    L.gbo_exp.restype = C.c_float
    L.gbo_exp.argtypes = [C.c_float]
    L.gbo_log2.restype = C.c_float
    L.gbo_log2.argtypes = [C.c_float]
    L.gbo_topk_filter.restype = C.c_int32
    L.gbo_topk_filter.argtypes = [I32, F32, C.c_int64, C.c_int32, I32, F32]
    L.gbo_pq_push_pop_all.restype = C.c_int32
    L.gbo_pq_push_pop_all.argtypes = [I32, F32, C.c_int64, C.c_int32, C.c_int32, I32, F32]
    L.gbo_bpr_step.argtypes = [F32, F32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_float, C.c_float]
    L.gbo_bpr_apply_triples.argtypes = [F32, F32, C.c_int32, I32, C.c_int64, C.c_float, C.c_float]
    L.gbo_bpr_sample_triples.argtypes = [C.c_int32, I64, I32, I32, C.c_int32, C.c_uint64, C.c_int64, C.c_int64, I32]
    L.gbo_sample_user_negatives.argtypes = [C.c_int32, C.c_int32, C.c_int32, I64, I32, I64, I32, C.c_int32, C.c_uint64, I64, C.c_void_p]
    L.gbo_fill_normal_interleaved.argtypes = [F32, C.c_int64, C.c_float, C.c_uint64, C.c_int32]
    L.gbo_bpr_epoch_threads.restype = C.c_double
    L.gbo_bpr_epoch_threads.argtypes = [F32, F32, C.c_int32, C.c_int32, I64, I32, I32, C.c_int32, C.c_uint64,
                                        C.c_int64, C.c_float, C.c_float, C.c_int32, C.c_int32]
    L.gbo_als_epoch.argtypes = [F32, F32, C.c_int32, C.c_int32, C.c_int32, I64, I32, I64, I32, C.c_float, C.c_float]
    L.gbo_als_epoch_threads.restype = C.c_double
    L.gbo_als_epoch_threads.argtypes = [F32, F32, C.c_int32, C.c_int32, C.c_int32, I64, I32, I64, I32, C.c_float,
                                        C.c_float, C.c_int32]
    L.gbo_bruteforce_search.restype = C.c_int32
    L.gbo_bruteforce_search.argtypes = [F32, C.c_int64, C.c_int32, F32, C.c_int64, C.c_int32, C.c_int32, C.c_int32,
                                        I32, F32]
    L.gbo_bruteforce_all.restype = C.c_double
    L.gbo_bruteforce_all.argtypes = [F32, C.c_int64, C.c_int32, C.c_int64, C.c_int64, C.c_int32, C.c_int32,
                                     C.c_int32, C.c_int32, I32, F32, I32]
    for name in ("ndcg", "precision", "recall", "hr", "map", "mrr"):
        f = getattr(L, "gbo_" + name)
        f.restype = C.c_float
        f.argtypes = [I32, C.c_int32, I32, C.c_int32]
    L.gbo_evaluate.argtypes = [F32, F32, C.c_int32, C.c_int32, I64, I32, I64, I32, C.c_int32, F32]
    L.gbo_ref_bind.restype = C.c_int32
    L.gbo_ref_bind.argtypes = [C.c_char_p]
    L.gbo_bf16_truncate.argtypes = [F32, C.c_int64, F32]
    L.gbo_sparse_vector.restype = C.c_int32
    L.gbo_sparse_vector.argtypes = [I32, C.c_int32, F32, C.c_int32, C.c_uint32, _p(np.uint32), F32]
    L.gbo_als_observed_loss.restype = C.c_double
    L.gbo_als_observed_loss.argtypes = [F32, F32, C.c_int32, C.c_int32, I64, I32, C.c_double, C.c_int32]
    U32 = _p(np.uint32)
    L.gbo_sparse_dot.restype = C.c_float
    L.gbo_sparse_dot.argtypes = [U32, F32, C.c_int32, U32, F32, C.c_int32]
    L.gbo_sparse_bruteforce_search.restype = C.c_int32
    L.gbo_sparse_bruteforce_search.argtypes = [I64, U32, F32, C.c_int64, U32, F32, C.c_int32, C.c_int64, C.c_int32, I32, F32]
    L.gbo_similar_scores.restype = C.c_int32
    L.gbo_similar_scores.argtypes = [C.c_int32, C.c_double, C.c_int32, C.c_int32, I32, F32, C.c_int32, I32, _p(np.float64)]


def f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def i32(a):
    return np.ascontiguousarray(a, dtype=np.int32)


def i64(a):
    return np.ascontiguousarray(a, dtype=np.int64)


# ---- thin helpers -------------------------------------------------------------------------
def dot(a, b):
    a, b = f32(a), f32(b)
    return np.float32(lib().gbo_dot(a, b, a.size))


def euclidean(a, b):
    a, b = f32(a), f32(b)
    return np.float32(lib().gbo_euclidean(a, b, a.size))


def exp(x):
    return np.float32(lib().gbo_exp(np.float32(x)))


def topk_filter(values, weights, k):
    values, weights = i32(values), f32(weights)
    ov = np.zeros(max(k, 1), np.int32)
    ow = np.zeros(max(k, 1), np.float32)
    m = lib().gbo_topk_filter(values, weights, values.size, k, ov, ow)
    return ov[:m].copy(), ow[:m].copy()


def pq_push_pop_all(values, weights, desc, reverse_first=False):
    values, weights = i32(values), f32(weights)
    ov = np.zeros(max(values.size, 1), np.int32)
    ow = np.zeros(max(values.size, 1), np.float32)
    m = lib().gbo_pq_push_pop_all(values, weights, values.size, int(desc), int(reverse_first), ov, ow)
    return ov[:m].copy(), ow[:m].copy()


def bpr_apply_triples(P, Q, uij, lr, reg):
    """Sequential application (reference with Jobs=1 on this triple stream); P, Q updated in place."""
    assert P.dtype == np.float32 and Q.dtype == np.float32 and P.flags.c_contiguous and Q.flags.c_contiguous
    uij = i32(uij).reshape(-1, 3)
    lib().gbo_bpr_apply_triples(P, Q, P.shape[1], uij, uij.shape[0], lr, reg)


def bpr_sample_triples(n_items, user_off, user_items, active, seed, first_step, n):
    out = np.zeros((n, 3), np.int32)
    lib().gbo_bpr_sample_triples(n_items, i64(user_off), i32(user_items), i32(active), len(active), seed,
                                 first_step, n, out)
    return out


def sample_user_negatives(n_items, train_off, train_items, test_off, test_items, n_cand, seed=0, u_base=0):
    """dataset.SampleUserNegatives with the library's counter RNG; train rows sorted ascending."""
    U = len(train_off) - 1
    off = np.zeros(U + 1, np.int64)
    a = (n_items, U, u_base, i64(train_off), i32(train_items), i64(test_off), i32(test_items), n_cand, seed)
    lib().gbo_sample_user_negatives(*a, off, None)
    items = np.zeros(int(off[-1]), np.int32)
    lib().gbo_sample_user_negatives(*a, off, items.ctypes.data_as(C.c_void_p))
    return off, items


def fill_normal_interleaved(shape, std, seed, n_threads):
    """N(0, std) table whose pages are first touched round-robin by the pinned worker threads (NUMA-interleaved)."""
    a = np.empty(shape, np.float32)
    lib().gbo_fill_normal_interleaved(a.reshape(-1), a.size, std, seed, n_threads)
    return a


def bpr_epoch_threads(P, Q, user_off, user_items, active, seed, n_steps, lr, reg, n_threads, use_ref=False):
    return lib().gbo_bpr_epoch_threads(P, Q, Q.shape[0], P.shape[1], i64(user_off), i32(user_items), i32(active),
                                       len(active), seed, n_steps, lr, reg, n_threads, int(use_ref))


def als_epoch(P, Q, user_off, user_items, item_off, item_users, reg, alpha):
    assert P.dtype == np.float32 and Q.dtype == np.float32
    lib().gbo_als_epoch(P, Q, P.shape[0], Q.shape[0], P.shape[1], i64(user_off), i32(user_items), i64(item_off),
                        i32(item_users), reg, alpha)


def als_epoch_threads(P, Q, user_off, user_items, item_off, item_users, reg, alpha, n_threads):
    return lib().gbo_als_epoch_threads(P, Q, P.shape[0], Q.shape[0], P.shape[1], i64(user_off), i32(user_items),
                                       i64(item_off), i32(item_users), reg, alpha, n_threads)


def als_observed_loss(P, Q, user_off, user_items, w, n_threads=0):
    """sum over observed (u,i) of (1 - p.q)^2 - w (p.q)^2 in double (test helper for the eALS objective)."""
    import os
    n_threads = n_threads or len(os.sched_getaffinity(0))
    return lib().gbo_als_observed_loss(f32(P), f32(Q), P.shape[0], P.shape[1], i64(user_off), i32(user_items), float(w), n_threads)


def bruteforce_search(X, q, k, prune0=False, metric=METRIC_NEG_DOT, self_index=-1):
    X = f32(X)
    q = f32(q)
    oi = np.zeros(max(k, 1), np.int32)
    os_ = np.zeros(max(k, 1), np.float32)
    m = lib().gbo_bruteforce_search(X, X.shape[0], X.shape[1], q, self_index, k, int(prune0), metric, oi, os_)
    return oi[:m].copy(), os_[:m].copy()


def bruteforce_all(X, q0, q1, k, prune0=False, metric=METRIC_NEG_DOT, n_threads=1):
    X = f32(X)
    nq = q1 - q0
    oi = np.full((nq, k), -1, np.int32)
    os_ = np.zeros((nq, k), np.float32)
    oc = np.zeros(nq, np.int32)
    sec = lib().gbo_bruteforce_all(X, X.shape[0], X.shape[1], q0, q1, k, int(prune0), metric, n_threads, oi, os_, oc)
    return oi, os_, oc, sec


def bf16_truncate(a):
    a = f32(a)
    out = np.empty_like(a)
    lib().gbo_bf16_truncate(a.reshape(-1), a.size, out.reshape(-1))
    return out


def sparse_vector(ids, idf, offset=0):
    ids, idf = i32(ids), f32(idf)
    ind, val = np.zeros(len(ids), np.uint32), np.zeros(len(ids), np.float32)
    m = lib().gbo_sparse_vector(ids, len(ids), idf, len(idf), offset, ind, val)
    return ind[:m], val[:m]


def sparse_dot(ia, va, ib, vb):
    """merge-join dot of two sparse vectors in ascending index order (what the flat sparse index of the reference's vector
    store computes; restated, see gorse_oracle.h)"""
    ia, ib = np.ascontiguousarray(ia, np.uint32), np.ascontiguousarray(ib, np.uint32)
    va, vb = f32(va), f32(vb)
    return np.float32(lib().gbo_sparse_dot(ia, va, len(ia), ib, vb, len(ib)))


def sparse_bruteforce_search(off, indices, values, self_index, k):
    """k best neighbours (ids, dots) of stored sparse vector `self_index` among the CSR-packed vectors."""
    off = i64(off)
    indices = np.ascontiguousarray(indices, np.uint32)
    values = f32(values)
    a, b = int(off[self_index]), int(off[self_index + 1])
    oi, od = np.zeros(max(k, 1), np.int32), np.zeros(max(k, 1), np.float32)
    m = lib().gbo_sparse_bruteforce_search(off, indices, values, len(off) - 1, indices[a:b].copy(), values[a:b].copy(), b - a,
                                           self_index, k, oi, od)
    return oi[:m].copy(), od[:m].copy()


def similar_scores(euclidean, score_scale, self_id, n, nbr_ids, nbr_score):
    """logics.QueryItemToItem post-processing; nbr_score is the vector store's "higher is closer" score."""
    nbr_ids, nbr_score = i32(nbr_ids), f32(nbr_score)
    ids, sc = np.zeros(max(n, 1), np.int32), np.zeros(max(n, 1), np.float64)
    m = lib().gbo_similar_scores(int(euclidean), float(score_scale), int(self_id), int(n), nbr_ids, nbr_score, len(nbr_ids), ids, sc)
    return ids[:m], sc[:m]


def evaluate(P, Q, test_off, test_items, neg_off, neg_items, topk):
    out = np.zeros(3, np.float32)
    lib().gbo_evaluate(f32(P), f32(Q), P.shape[0], P.shape[1], i64(test_off), i32(test_items), i64(neg_off),
                       i32(neg_items), topk, out)
    return out


def metric(name, target, rank):
    target, rank = i32(target), i32(rank)
    return np.float32(getattr(lib(), "gbo_" + name)(target, target.size, rank, rank.size))


def ref_available():
    return os.path.exists(REF_SO)


def ref_bind():
    return lib().gbo_ref_bind(REF_SO.encode()) == 0


class RefFloats:
    """The reference's own compiled kernels (oracle/_ref/libfloats_ref.so), when present."""

    def __init__(self):
        self.L = C.CDLL(REF_SO)
        fp = C.POINTER(C.c_float)
        for pre in ("_mm512_", "_mm256_"):
            for n in ("dot", "euclidean"):
                f = getattr(self.L, pre + n)
                f.restype = C.c_float
                f.argtypes = [fp, fp, C.c_int64]
            for n in ("mul_const_to", "mul_const_add", "sub_to"):
                getattr(self.L, pre + n).argtypes = [fp, fp, fp, C.c_int64]
            getattr(self.L, pre + "mul_const").argtypes = [fp, fp, C.c_int64]
            getattr(self.L, pre + "mul_const_add_to").argtypes = [fp, fp, fp, fp, C.c_int64]

    @staticmethod
    def _fp(a):
        return a.ctypes.data_as(C.POINTER(C.c_float))

    def call2(self, name, a, b):
        return np.float32(getattr(self.L, name)(self._fp(a), self._fp(b), a.size))

    def mul_const_to(self, a, c, pre="_mm512_"):
        dst = np.zeros_like(a)
        cc = np.array([c], np.float32)
        getattr(self.L, pre + "mul_const_to")(self._fp(a), self._fp(cc), self._fp(dst), a.size)
        return dst

    def mul_const_add(self, a, c, dst, pre="_mm512_"):
        dst = dst.copy()
        cc = np.array([c], np.float32)
        getattr(self.L, pre + "mul_const_add")(self._fp(a), self._fp(cc), self._fp(dst), a.size)
        return dst

    def mul_const_add_to(self, a, b, c, pre="_mm512_"):
        dst = np.zeros_like(a)
        bb = np.array([b], np.float32)
        getattr(self.L, pre + "mul_const_add_to")(self._fp(a), self._fp(bb), self._fp(c), self._fp(dst), a.size)
        return dst

    def mul_const(self, a, c, pre="_mm512_"):
        a = a.copy()
        cc = np.array([c], np.float32)
        getattr(self.L, pre + "mul_const")(self._fp(a), self._fp(cc), a.size)
        return a

    def sub_to(self, a, b, pre="_mm512_"):
        dst = np.zeros_like(a)
        getattr(self.L, pre + "sub_to")(self._fp(a), self._fp(b), self._fp(dst), a.size)
        return dst
