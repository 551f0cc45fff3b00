"""gorse_b200 -- H100 (sm_90a) implementation of Gorse's collaborative-filtering training and
brute-force top-k hot path.

The product is the C-ABI shared library (include/gorse_b200.h, gorse_b200/libgorse_b200.so).  This
package is the thin Python binding over that ABI used by the tests and by bench.py; it holds no
compute of its own and has no CPU fallback (importing it without the built library fails).
"""
import ctypes as C

import numpy as np

from . import _lib
from ._lib import (DISTANCE_COSINE, DISTANCE_DOT, DISTANCE_EUCLIDEAN, GorseB200Error, METRIC_COSINE, METRIC_EUCLIDEAN,  # noqa: F401
                   METRIC_NEG_DOT, ORDER_HOGWILD, ORDER_SEQUENTIAL,
                   SCATTER_ATOMIC, SCATTER_STORE, check, lib, ptr)

__all__ = ["Context", "CFModel", "BruteforceIndex", "GorseB200Error", "csr_from_lists", "device_count"]


def device_count():
    n = C.c_int32(0)
    check(lib.gorse_b200_device_count(C.byref(n)))
    return n.value


def nccl_unique_id():
    buf = C.create_string_buffer(_lib.NCCL_ID_BYTES)
    check(lib.gorse_b200_nccl_unique_id(buf))
    return buf.raw


class PinnedArray:
    """numpy view of page-locked host memory from gorse_b200_host_alloc (the shim's flat factor mirror)."""

    def __init__(self, shape, dtype=np.float32):
        self.nbytes = int(np.prod(shape)) * np.dtype(dtype).itemsize
        p = C.c_void_p()
        check(lib.gorse_b200_host_alloc(self.nbytes, C.byref(p)))
        self._p = p
        buf = (C.c_char * self.nbytes).from_address(p.value) if self.nbytes else (C.c_char * 0)()
        self.array = np.frombuffer(buf, dtype=dtype).reshape(shape)

    def free(self):
        if self._p:
            self.array = None
            lib.gorse_b200_host_free(self._p)
            self._p = None


def csr_from_lists(rows):
    """[][]int32 (dataset.CFSplit.GetUserFeedback, dataset/dataset.go:40-60) -> (offsets int64, indices int32)."""
    off = np.zeros(len(rows) + 1, np.int64)
    for r, row in enumerate(rows):
        off[r + 1] = off[r] + len(row)
    idx = np.zeros(int(off[-1]), np.int32)
    for r, row in enumerate(rows):
        idx[off[r]:off[r + 1]] = row
    return off, idx


def transpose_csr(off, idx, n_cols):
    """user CSR -> item CSR preserving the reference's append order (dataset.go:231-240: users ascending)."""
    n_rows = len(off) - 1
    counts = np.bincount(idx, minlength=n_cols).astype(np.int64)
    toff = np.zeros(n_cols + 1, np.int64)
    np.cumsum(counts, out=toff[1:])
    rows = np.repeat(np.arange(n_rows, dtype=np.int32), np.diff(off))
    order = np.argsort(idx, kind="stable")
    return toff, rows[order].astype(np.int32)


class Context:
    """One GPU (+ optionally one NCCL rank)."""

    def __init__(self, device=0, rank=0, world=1, nccl_id=None):
        h = C.c_void_p()
        if world > 1:
            check(lib.gorse_b200_ctx_create_dist(device, rank, world, nccl_id, C.byref(h)))
        else:
            check(lib.gorse_b200_ctx_create(device, C.byref(h)))
        self.h = h
        self.rank, self.world = rank, world

    def close(self):
        if self.h:
            lib.gorse_b200_ctx_destroy(self.h)
            self.h = None

    def sync(self):
        check(lib.gorse_b200_ctx_sync(self.h))

    def barrier(self):
        check(lib.gorse_b200_ctx_barrier(self.h))

    def flush_l2(self):
        check(lib.gorse_b200_ctx_flush_l2(self.h))

    def timer_begin(self):
        check(lib.gorse_b200_ctx_timer_begin(self.h))

    def timer_end(self):
        ms = C.c_float(0)
        check(lib.gorse_b200_ctx_timer_end(self.h, C.byref(ms)))
        return ms.value

    def launch_count(self):
        n = C.c_int64(0)
        check(lib.gorse_b200_ctx_launch_count(self.h, C.byref(n)))
        return n.value

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()


class CFModel:
    """Device-resident factor tables + feedback CSR (cf.BaseMatrixFactorization state)."""

    def __init__(self, ctx, n_users, n_items, n_factors, user_off, user_items, item_off=None, item_users=None):
        self.ctx = ctx
        self.n_users, self.n_items, self.d = n_users, n_items, n_factors
        user_off = np.ascontiguousarray(user_off, np.int64)
        user_items = np.ascontiguousarray(user_items, np.int32)
        if item_off is not None:
            item_off = np.ascontiguousarray(item_off, np.int64)
            item_users = np.ascontiguousarray(item_users, np.int32)
        h = C.c_void_p()
        check(lib.gorse_b200_cf_create(ctx.h, n_users, n_items, n_factors, ptr(user_off), ptr(user_items),
                                       ptr(item_off), ptr(item_users), C.byref(h)))
        self.h = h

    def close(self):
        if self.h:
            lib.gorse_b200_cf_destroy(self.h)
            self.h = None

    def set_factors(self, P, Q):
        P = np.ascontiguousarray(P, np.float32)
        Q = np.ascontiguousarray(Q, np.float32)
        assert P.shape == (self.n_users, self.d) and Q.shape == (self.n_items, self.d)
        check(lib.gorse_b200_cf_set_factors(self.h, ptr(P), ptr(Q)))

    def init_normal(self, mean, std, seed):
        check(lib.gorse_b200_cf_init_normal(self.h, mean, std, seed))

    def get_factors(self, P=None, Q=None):
        if P is None:
            P = np.zeros((self.n_users, self.d), np.float32)
        if Q is None:
            Q = np.zeros((self.n_items, self.d), np.float32)
        check(lib.gorse_b200_cf_get_factors(self.h, ptr(P), ptr(Q)))
        return P, Q

    def predict(self, users, items):
        users = np.ascontiguousarray(users, np.int32)
        items = np.ascontiguousarray(items, np.int32)
        out = np.zeros(users.size, np.float32)
        check(lib.gorse_b200_cf_predict(self.h, ptr(users), ptr(items), users.size, ptr(out)))
        return out

    def bpr_apply_triples(self, uij, lr, reg, scatter=SCATTER_STORE, order=ORDER_HOGWILD):
        uij = np.ascontiguousarray(uij, np.int32).reshape(-1, 3)
        check(lib.gorse_b200_bpr_apply_triples(self.h, ptr(uij), uij.shape[0], lr, reg, scatter, order))

    def bpr_sample_triples(self, seed, first_step, n):
        out = np.zeros((n, 3), np.int32)
        check(lib.gorse_b200_bpr_sample_triples(self.h, seed, first_step, n, ptr(out)))
        return out

    def bpr_epoch(self, lr, reg, n_steps, seed, scatter=SCATTER_ATOMIC):
        check(lib.gorse_b200_bpr_epoch(self.h, lr, reg, n_steps, seed, scatter))

    def als_epoch(self, reg, alpha):
        check(lib.gorse_b200_als_epoch(self.h, reg, alpha))

    def fit(self, kind, test_off, test_items, neg_off, neg_items, progress=None, **params):
        """cf.BPR.Fit / cf.ALS.Fit through gorse_b200_{bpr,als}_fit; params override the reference defaults."""
        fp = _lib.FitParams()
        check(lib.gorse_b200_fit_params_default(1 if kind == "als" else 0, C.byref(fp)))
        fp.n_factors = self.d
        for k, v in params.items():
            setattr(fp, k, v)
        res = _lib.FitResult()
        test_off = np.ascontiguousarray(test_off, np.int64)
        test_items = np.ascontiguousarray(test_items, np.int32)
        if neg_off is not None:   # None: the negatives are sampled on the device (params: candidates)
            neg_off = np.ascontiguousarray(neg_off, np.int64)
            neg_items = np.ascontiguousarray(neg_items, np.int32)
        cb = _lib.PROGRESS_FN(lambda user, ep, n, ndcg: int(bool(progress(ep, n, ndcg)))) if progress else None
        fn = lib.gorse_b200_als_fit if kind == "als" else lib.gorse_b200_bpr_fit
        check(fn(self.h, C.byref(fp), ptr(test_off), ptr(test_items), ptr(neg_off), ptr(neg_items),
                 C.cast(cb, C.c_void_p) if cb else None, None, C.byref(res)))
        return res

    def eval_plan(self, test_off, test_items, neg_off=None, neg_items=None, n_candidates=100, seed=0, topk=10):
        return EvalPlan(self, test_off, test_items, neg_off, neg_items, n_candidates, seed, topk)

    def evaluate(self, test_off, test_items, neg_off, neg_items, topk=10):
        test_off = np.ascontiguousarray(test_off, np.int64)
        test_items = np.ascontiguousarray(test_items, np.int32)
        neg_off = np.ascontiguousarray(neg_off, np.int64)
        neg_items = np.ascontiguousarray(neg_items, np.int32)
        out = np.zeros(3, np.float32)
        check(lib.gorse_b200_cf_evaluate(self.h, ptr(test_off), ptr(test_items), ptr(neg_off), ptr(neg_items), topk,
                                         ptr(out)))
        return out

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()


class EvalPlan:
    """cf.Evaluate's inputs resident on the device (gorse_b200_eval_*): test rows + negatives, sampled there when
    neg_off is None (dataset.SampleUserNegatives, dataset/dataset.go:242-253)."""

    def __init__(self, model, test_off, test_items, neg_off, neg_items, n_candidates, seed, topk):
        self.model = model
        test_off = np.ascontiguousarray(test_off, np.int64)
        test_items = np.ascontiguousarray(test_items, np.int32)
        if neg_off is not None:
            neg_off = np.ascontiguousarray(neg_off, np.int64)
            neg_items = np.ascontiguousarray(neg_items, np.int32)
        self.rows = len(test_off) - 1
        h = C.c_void_p()
        check(lib.gorse_b200_eval_create(model.h, ptr(test_off), ptr(test_items), ptr(neg_off), ptr(neg_items), n_candidates, seed,
                                         topk, C.byref(h)))
        self.h = h

    def run(self):
        out = np.zeros(3, np.float32)
        check(lib.gorse_b200_eval_run(self.h, ptr(out)))
        return out

    def negatives(self):
        off = np.zeros(self.rows + 1, np.int64)
        check(lib.gorse_b200_eval_negatives(self.h, ptr(off), None))
        items = np.zeros(int(off[-1]), np.int32)
        check(lib.gorse_b200_eval_negatives(self.h, ptr(off), ptr(items)))
        return off, items

    def close(self):
        if self.h:
            lib.gorse_b200_eval_destroy(self.h)
            self.h = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()


class BruteforceIndex:
    """ann.Index backed by the GPU (common/ann/ann.go:21-25, bruteforce.go:24-83)."""

    def __init__(self, ctx, dim, metric=METRIC_NEG_DOT):
        self.ctx, self.dim, self.metric = ctx, dim, metric
        h = C.c_void_p()
        check(lib.gorse_b200_index_create(ctx.h, dim, metric, C.byref(h)))
        self.h = h

    def close(self):
        if self.h:
            lib.gorse_b200_index_destroy(self.h)
            self.h = None

    def add(self, vectors):
        """Bruteforce.Add for a batch; returns len after append (bruteforce.go:33-37)."""
        v = np.ascontiguousarray(vectors, np.float32).reshape(-1, self.dim)
        n = C.c_int64(0)
        check(lib.gorse_b200_index_add(self.h, ptr(v), v.shape[0], C.byref(n)))
        return n.value

    def __len__(self):
        n = C.c_int64(0)
        check(lib.gorse_b200_index_len(self.h, C.byref(n)))
        return n.value

    def stage1_stats(self):
        """(device ms, algorithmic flop, fallback rows) of the tensor-core candidate sweep since the last call."""
        ms, fl, fb = C.c_double(0), C.c_double(0), C.c_int64(0)
        check(lib.gorse_b200_index_stats(self.h, C.byref(ms), C.byref(fl), C.byref(fb)))
        return ms.value, fl.value, fb.value

    def stage1_scores(self, q0, q1):
        out = np.zeros((q1 - q0, len(self)), np.float32)
        check(lib.gorse_b200_index_stage1_scores(self.h, q0, q1, ptr(out)))
        return out

    def _out(self, nq, k):
        return (np.full((nq, max(k, 1)), -1, np.int32), np.zeros((nq, max(k, 1)), np.float32), np.zeros(nq, np.int32))

    def search_vectors(self, queries, k, prune0=False):
        q = np.ascontiguousarray(queries, np.float32).reshape(-1, self.dim)
        idx, dist, cnt = self._out(q.shape[0], k)
        check(lib.gorse_b200_index_search_vectors(self.h, ptr(q), q.shape[0], k, int(prune0), ptr(idx), ptr(dist), ptr(cnt)))
        return idx, dist, cnt

    def search_indices(self, q_idx, k, prune0=False):
        q = np.ascontiguousarray(q_idx, np.int64)
        idx, dist, cnt = self._out(q.size, k)
        check(lib.gorse_b200_index_search_indices(self.h, ptr(q), q.size, k, int(prune0), ptr(idx), ptr(dist), ptr(cnt)))
        return idx, dist, cnt

    def search_range(self, q0, q1, k, prune0=False, out=None):
        """out = (idx int32 [nq,k], dist float32 [nq,k], cnt int32 [nq]) to reuse (e.g. pinned) result buffers."""
        idx, dist, cnt = out if out is not None else self._out(max(q1 - q0, 0), k)
        check(lib.gorse_b200_index_search_range(self.h, q0, q1, k, int(prune0), ptr(idx), ptr(dist), ptr(cnt)))
        return idx, dist, cnt

    def query_similar(self, q0, q1, n, score_scale=1.0):
        """logics.QueryItemToItem / QueryUserToUser for stored vectors [q0, q1) (logics/item_to_item.go:50-86):
        (ids int32 [nq,n] padded with -1, scores float64 [nq,n], cnt int32 [nq])."""
        nq = max(q1 - q0, 0)
        ids, sc, cnt = np.full((nq, n), -1, np.int32), np.zeros((nq, n), np.float64), np.zeros(nq, np.int32)
        check(lib.gorse_b200_index_query_similar(self.h, q0, q1, n, float(score_scale), ptr(ids), ptr(sc), ptr(cnt)))
        return ids, sc, cnt

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()


class SparseIndex:
    """Brute-force Dot search over sparse vectors, the store side of the
    tags / users / auto similarity types (storage/vectors/xvec.go:244-248)."""

    def __init__(self, ctx):
        self.ctx = ctx
        h = C.c_void_p()
        check(lib.gorse_b200_sparse_index_create(ctx.h, C.byref(h)))
        self.h = h

    def close(self):
        if self.h:
            lib.gorse_b200_sparse_index_destroy(self.h)
            self.h = None

    def add(self, off, indices, values):
        """CSR batch: off int64 [n+1] from 0, indices uint32 strictly ascending per vector, values float32."""
        off = np.ascontiguousarray(off, np.int64)
        indices = np.ascontiguousarray(indices, np.uint32)
        values = np.ascontiguousarray(values, np.float32)
        n = C.c_int64(0)
        check(lib.gorse_b200_sparse_index_add(self.h, ptr(off), ptr(indices), ptr(values), len(off) - 1, C.byref(n)))
        return n.value

    def __len__(self):
        n = C.c_int64(0)
        check(lib.gorse_b200_sparse_index_len(self.h, C.byref(n)))
        return n.value

    def search_range(self, q0, q1, k):
        nq = max(q1 - q0, 0)
        idx, dot, cnt = np.full((nq, k), -1, np.int32), np.zeros((nq, k), np.float32), np.zeros(nq, np.int32)
        check(lib.gorse_b200_sparse_index_search_range(self.h, q0, q1, k, ptr(idx), ptr(dot), ptr(cnt)))
        return idx, dot, cnt

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()


class VectorCollection:
    """One collection of a vectors.Database on the GPU (gorse_b200_vecdb_*; storage/vectors/database.go:107-120).  Works on
    slots and int category ids; the Go shim keeps the id / category string maps."""

    def __init__(self, ctx, dim, distance):
        self.ctx, self.dim, self.distance = ctx, dim, distance
        h = C.c_void_p()
        check(lib.gorse_b200_vecdb_create(ctx.h, dim, distance, C.byref(h)))
        self.h = h

    def close(self):
        if self.h:
            lib.gorse_b200_vecdb_destroy(self.h)
            self.h = None

    def count(self):
        live, slots = C.c_int64(0), C.c_int64(0)
        check(lib.gorse_b200_vecdb_count(self.h, C.byref(live), C.byref(slots)))
        return live.value, slots.value

    def add(self, values=None, sparse=None, hidden=None, timestamps=None, categories=None, replace=None):
        """dense: values [n, dim]; sparse: list of (indices, values).  categories: list of int lists.  Returns the first slot."""
        sp_off = sp_ind = None
        if self.dim > 0:
            values = np.ascontiguousarray(values, np.float32).reshape(-1, self.dim)
            n = values.shape[0]
        else:
            n = len(sparse)
            sp_off = np.concatenate([[0], np.cumsum([len(v[0]) for v in sparse])]).astype(np.int64)
            sp_ind = np.ascontiguousarray(np.concatenate([np.asarray(v[0], np.uint32) for v in sparse]) if n else np.zeros(0), np.uint32)
            values = np.ascontiguousarray(np.concatenate([np.asarray(v[1], np.float32) for v in sparse]) if n else np.zeros(0), np.float32)
        hid = None if hidden is None else np.ascontiguousarray(hidden, np.uint8)
        ts = None if timestamps is None else np.ascontiguousarray(timestamps, np.int64)
        co = cv = None
        if categories is not None:
            co = np.concatenate([[0], np.cumsum([len(c) for c in categories])]).astype(np.int64)
            cv = np.ascontiguousarray([x for c in categories for x in c], np.int32)
        rep = None if replace is None else np.ascontiguousarray(replace, np.int64)
        first = C.c_int64(0)
        check(lib.gorse_b200_vecdb_add(self.h, n, ptr(values), ptr(sp_off), ptr(sp_ind), ptr(hid), ptr(ts), ptr(co), ptr(cv), ptr(rep), C.byref(first)))
        return first.value

    def get(self, slots):
        slots = np.ascontiguousarray(slots, np.int64)
        n = slots.size
        vals = np.zeros((n, max(self.dim, 1)), np.float32)
        hid, ts, live = np.zeros(n, np.uint8), np.zeros(n, np.int64), np.zeros(n, np.uint8)
        check(lib.gorse_b200_vecdb_get(self.h, ptr(slots), n, ptr(vals) if self.dim > 0 else None, ptr(hid), ptr(ts), ptr(live)))
        return vals, hid, ts, live

    def get_sparse(self, slot, cap=4096):
        ind, val, nnz = np.zeros(cap, np.uint32), np.zeros(cap, np.float32), C.c_int32(0)
        check(lib.gorse_b200_vecdb_get_sparse(self.h, slot, ptr(ind), ptr(val), cap, C.byref(nnz)))
        return ind[:nnz.value], val[:nnz.value]

    def delete_before(self, timestamp_ms, cap=1 << 20):
        out, cnt = np.zeros(cap, np.int64), C.c_int64(0)
        check(lib.gorse_b200_vecdb_delete_before(self.h, timestamp_ms, ptr(out), cap, C.byref(cnt)))
        return out[:min(cnt.value, cap)]

    def query(self, q, categories=(), topk=10):
        """q: dense [nq, dim] array, or a list of (indices, values) for a sparse collection.
        -> (slots int64 [nq, topk], scores float32 [nq, topk], count int32 [nq])"""
        sp_off = sp_ind = None
        if self.dim > 0:
            qv = np.ascontiguousarray(q, np.float32).reshape(-1, self.dim)
            nq = qv.shape[0]
        else:
            nq = len(q)
            sp_off = np.concatenate([[0], np.cumsum([len(v[0]) for v in q])]).astype(np.int64)
            sp_ind = np.ascontiguousarray(np.concatenate([np.asarray(v[0], np.uint32) for v in q]), np.uint32)
            qv = np.ascontiguousarray(np.concatenate([np.asarray(v[1], np.float32) for v in q]), np.float32)
        cats = np.ascontiguousarray(list(categories), np.int32)
        k = max(topk, 1)
        slots, scores, cnt = np.full((nq, k), -1, np.int64), np.zeros((nq, k), np.float32), np.zeros(nq, np.int32)
        check(lib.gorse_b200_vecdb_query(self.h, nq, ptr(qv), ptr(sp_off), ptr(sp_ind), ptr(cats) if cats.size else None, cats.size, topk,
                                         ptr(slots), ptr(scores), ptr(cnt)))
        return slots, scores, cnt

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()


def load_ncf(train_path, test_path=None):
    """dataset.LoadDataFromBuiltIn's NCF parsers (dataset/dataset.go:398-490) ->
    (n_users, n_items, (train_off, train_items), (test_off, test_items), (neg_off, neg_items))."""
    h = C.c_void_p()
    check(lib.gorse_b200_ncf_load(str(train_path).encode(), str(test_path).encode() if test_path else None, C.byref(h)))
    try:
        U, I = C.c_int32(0), C.c_int32(0)
        a, b, c = C.c_int64(0), C.c_int64(0), C.c_int64(0)
        check(lib.gorse_b200_ncf_shape(h, C.byref(U), C.byref(I), C.byref(a), C.byref(b), C.byref(c)))
        offs = [np.zeros(U.value + 1, np.int64) for _ in range(3)]
        idx = [np.zeros(n.value, np.int32) for n in (a, b, c)]
        check(lib.gorse_b200_ncf_get(h, ptr(offs[0]), ptr(idx[0]), ptr(offs[1]), ptr(idx[1]), ptr(offs[2]), ptr(idx[2])))
    finally:
        lib.gorse_b200_ncf_free(h)
    return U.value, I.value, (offs[0], idx[0]), (offs[1], idx[1]), (offs[2], idx[2])


# ---- logics: similarity vectors and scores (host functions; SURVEY 8a row J) ---------------------------------
def bf16_truncate(a):
    """bfloats.FromFloat32 + ToFloat32 (common/bfloats/bfloats.go:23-37): how the reference stores dense embeddings."""
    a = np.ascontiguousarray(a, np.float32)
    out = np.empty_like(a)
    check(lib.gorse_b200_bf16_truncate(ptr(a), a.size, ptr(out)))
    return out


def sparse_vector(ids, idf, offset=0):
    """appendSparseVector (logics/vector_writer.go:200-209) -> (indices uint32, values float32)."""
    ids, idf = np.ascontiguousarray(ids, np.int32), np.ascontiguousarray(idf, np.float32)
    ind, val = np.zeros(max(len(ids), 1), np.uint32), np.zeros(max(len(ids), 1), np.float32)
    m = C.c_int32(0)
    check(lib.gorse_b200_sparse_vector(ptr(ids), len(ids), ptr(idf), len(idf), int(offset), ptr(ind), ptr(val), C.byref(m)))
    return ind[:m.value], val[:m.value]


def similar_scores(metric, score_scale, self_id, n, nbr_ids, nbr_dist):
    """QueryItemToItem post-processing (logics/item_to_item.go:63-85) of one result row of BruteforceIndex."""
    nbr_ids, nbr_dist = np.ascontiguousarray(nbr_ids, np.int32), np.ascontiguousarray(nbr_dist, np.float32)
    ids, sc = np.zeros(max(n, 1), np.int32), np.zeros(max(n, 1), np.float64)
    m = C.c_int32(0)
    check(lib.gorse_b200_similar_scores(int(metric), float(score_scale), int(self_id), int(n), ptr(nbr_ids), ptr(nbr_dist),
                                        len(nbr_ids), ptr(ids), ptr(sc), C.byref(m)))
    return ids[:m.value], sc[:m.value]
