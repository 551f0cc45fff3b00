"""gorse_b200 -- H100 (sm_90a) implementation of Gorse's collaborative-filtering training and
brute-force top-k hot path.

The product is the C-ABI shared library (include/gorse_b200.h, gorse_b200/libgorse_b200.so).  This
package is the thin Python binding over that ABI used by the tests and by bench.py; it holds no
compute of its own and has no CPU fallback (importing it without the built library fails).
"""
import ctypes as C

import numpy as np

from . import _lib
from ._lib import (DISTANCE_COSINE, DISTANCE_DOT, DISTANCE_EUCLIDEAN, FM_ADAM, FM_SGD, GorseB200Error, METRIC_COSINE, METRIC_EUCLIDEAN,  # noqa: F401
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

    def fit_trials(self, trials, test_off, test_items, neg_off, neg_items, progress=None, factors=False):
        """ModelSearch's trials in one gorse_b200_cf_fit_trials call.  trials: a list of (kind, params) with kind "bpr" or
        "als" and params overriding that kind's defaults as in fit(); the fields the trials share (seed, verbose, candidates,
        topk, patience) must be equal.  progress(epoch, states), states a list of (epochs_run, ndcg or -1, finished) per
        trial, returns True to cancel.  Returns the list of FitResult, and with factors=True also a list of (P, Q)."""
        n = len(trials)
        als = np.array([1 if kind == "als" else 0 for kind, _ in trials], np.int32)
        fps = (_lib.FitParams * n)()
        for k, (kind, params) in enumerate(trials):
            check(lib.gorse_b200_fit_params_default(int(als[k]), C.byref(fps[k])))
            fps[k].n_factors = self.d
            for key, v in params.items():
                setattr(fps[k], key, v)
        res = (_lib.FitResult * n)()
        test_off = np.ascontiguousarray(test_off, np.int64)
        test_items = np.ascontiguousarray(test_items, np.int32)
        if neg_off is not None:   # None: the negatives are sampled on the device (params: candidates)
            neg_off = np.ascontiguousarray(neg_off, np.int64)
            neg_items = np.ascontiguousarray(neg_items, np.int32)
        out = None
        p_ptrs = q_ptrs = None
        if factors:
            out = [(np.zeros((self.n_users, self.d), np.float32), np.zeros((self.n_items, self.d), np.float32)) for _ in range(n)]
            p_ptrs = (C.c_void_p * n)(*[P.ctypes.data for P, _ in out])
            q_ptrs = (C.c_void_p * n)(*[Q.ctypes.data for _, Q in out])

        def on_epoch(user, epoch, n_trials, states):
            return int(bool(progress(epoch, [(states[k].epochs_run, states[k].ndcg, bool(states[k].finished)) for k in range(n_trials)])))

        cb = _lib.TRIALS_PROGRESS_FN(on_epoch) if progress else None
        check(lib.gorse_b200_cf_fit_trials(self.h, n, ptr(als), C.cast(fps, C.c_void_p), ptr(test_off), ptr(test_items), ptr(neg_off),
                                           ptr(neg_items), C.cast(cb, C.c_void_p) if cb else None, None, C.cast(res, C.c_void_p),
                                           C.cast(p_ptrs, C.c_void_p) if factors else None, C.cast(q_ptrs, C.c_void_p) if factors else None))
        res = list(res)
        return (res, out) if factors else res

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

    def stage1_scores(self, q0, q1, with_eps=False):
        """dense tensor-core scores of stored rows [q0, q1) against every vector [nq, N]; with_eps: (scores, each row's eps
        [nq]), the margin the sweep relies on: |score - exact score| <= eps."""
        out = np.zeros((q1 - q0, len(self)), np.float32)
        eps = np.zeros(q1 - q0, np.float32) if with_eps else None
        check(lib.gorse_b200_index_stage1_scores(self.h, q0, q1, ptr(out), ptr(eps)))
        return (out, eps) if with_eps else out

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

    def query_excluding(self, q, exclude_lists, n, categories=()):
        """Batched CF recall (gorse_b200_vecdb_query_excluding; worker/pipeline.go:403-449): row i is the first
        n + len(exclude_lists[i]) results of query(q[i], categories) minus the slots in exclude_lists[i] (-1 = an excluded id
        the collection does not hold).  -> ([(slots int64, scores float32) per row], rows answered by the exact scan)"""
        qv = np.ascontiguousarray(q, np.float32).reshape(-1, self.dim)
        nq = qv.shape[0]
        if len(exclude_lists) != nq:
            raise ValueError(f"{len(exclude_lists)} exclude lists for {nq} queries")
        off = np.zeros(nq + 1, np.int64)
        np.cumsum([len(e) for e in exclude_lists], out=off[1:])
        ex = np.ascontiguousarray(np.concatenate([np.asarray(e, np.int64).reshape(-1) for e in exclude_lists]) if nq else [], np.int64)
        cats = np.ascontiguousarray(list(categories), np.int32)
        total = nq * max(n, 0) + int(off[-1])
        slots, scores, cnt = np.full(max(total, 1), -1, np.int64), np.zeros(max(total, 1), np.float32), np.zeros(nq, np.int32)
        exact = C.c_int64(0)
        check(lib.gorse_b200_vecdb_query_excluding(self.h, nq, ptr(qv), ptr(cats) if cats.size else None, cats.size, n, ptr(off),
                                                   ptr(ex) if ex.size else None, ptr(slots), ptr(scores), ptr(cnt), C.byref(exact)))
        starts = np.arange(nq, dtype=np.int64) * max(n, 0) + off[:-1]
        return [(slots[s:s + c].copy(), scores[s:s + c].copy()) for s, c in zip(starts, cnt)], exact.value

    def item_to_item(self, context_lists, exclude_lists, n, categories=(), score_scale=1.0):
        """Batched item-to-item recommendation (gorse_b200_vecdb_item_to_item; logics/recommend.go:244-283): for user i, the
        neighbours of every slot of context_lists[i] in order (-1 = an id without a vector), their scores summed per slot in
        float64 without the slots of exclude_lists[i], the best n.  score_scale: 0.5 for type "auto", else 1.
        -> ([(slots int64, scores float64) per user], stats {context_items, exact_rows, shared_users, global_users})"""
        nu = len(context_lists)
        if len(exclude_lists) != nu:
            raise ValueError(f"{len(exclude_lists)} exclude lists for {nu} users")

        def csr(lists):
            off = np.zeros(nu + 1, np.int64)
            np.cumsum([len(x) for x in lists], out=off[1:])
            flat = np.ascontiguousarray(np.concatenate([np.asarray(x, np.int64).reshape(-1) for x in lists]) if nu else [], np.int64)
            return off, flat

        coff, cs = csr(context_lists)
        eoff, es = csr(exclude_lists)
        cats = np.ascontiguousarray(list(categories), np.int32)
        m = max(n, 0)
        slots, scores, cnt = np.full(max(nu * m, 1), -1, np.int64), np.zeros(max(nu * m, 1), np.float64), np.zeros(max(nu, 1), np.int32)
        stats = np.zeros(4, np.int64)
        check(lib.gorse_b200_vecdb_item_to_item(self.h, nu, ptr(coff), ptr(cs) if cs.size else None, ptr(eoff), ptr(es) if es.size else None,
                                                ptr(cats) if cats.size else None, cats.size, n, float(score_scale), ptr(slots), ptr(scores),
                                                ptr(cnt), ptr(stats)))
        rows = [(slots[u * m:u * m + c].copy(), scores[u * m:u * m + c].copy()) for u, c in zip(range(nu), cnt)]
        return rows, dict(zip(("context_items", "exact_rows", "shared_users", "global_users"), (int(x) for x in stats)))

    def user_to_user(self, user_slots, feedback_lists, exclude_lists, n, n_items, item_ok=None, score_scale=1.0):
        """Batched user-to-user recommendation (gorse_b200_vecdb_user_to_user; logics/recommend.go:285-348): for user i, the
        first n neighbours of slot user_slots[i] (-1 = a user without a vector), each neighbour v's score added to every item
        of feedback_lists[v] (item indices in [0, n_items); slots past the list have no feedback) not in exclude_lists[i]
        (-1 = an id outside the dictionary), summed in float64; the best n, then only the items with item_ok[item] != 0 (None:
        all).  score_scale: 0.5 for type "auto", else 1.
        -> ([(items int64, scores float64) per user], stats {query_users, exact_rows, shared_users, global_users})"""
        slots = np.ascontiguousarray(user_slots, np.int64).reshape(-1)
        nu = slots.size
        if len(exclude_lists) != nu:
            raise ValueError(f"{len(exclude_lists)} exclude lists for {nu} users")
        nf = len(feedback_lists)
        foff = np.zeros(nf + 1, np.int64)
        np.cumsum([len(x) for x in feedback_lists], out=foff[1:])
        fitems = np.ascontiguousarray(np.concatenate([np.asarray(x, np.int32).reshape(-1) for x in feedback_lists]) if nf else [], np.int32)
        eoff = np.zeros(nu + 1, np.int64)
        np.cumsum([len(x) for x in exclude_lists], out=eoff[1:])
        es = np.ascontiguousarray(np.concatenate([np.asarray(x, np.int64).reshape(-1) for x in exclude_lists]) if nu else [], np.int64)
        ok = None if item_ok is None else np.ascontiguousarray(item_ok, np.uint8)
        if ok is not None and ok.size != n_items:
            raise ValueError(f"item_ok has {ok.size} entries for {n_items} items")
        m = max(n, 0)
        items, scores, cnt = np.full(max(nu * m, 1), -1, np.int64), np.zeros(max(nu * m, 1), np.float64), np.zeros(max(nu, 1), np.int32)
        stats = np.zeros(4, np.int64)
        check(lib.gorse_b200_vecdb_user_to_user(self.h, nu, ptr(slots), nf, ptr(foff), ptr(fitems) if fitems.size else None, int(n_items),
                                                ptr(ok) if ok is not None and ok.size else None, ptr(eoff), ptr(es) if es.size else None, n,
                                                float(score_scale), ptr(items), ptr(scores), ptr(cnt), ptr(stats)))
        rows = [(items[u * m:u * m + c].copy(), scores[u * m:u * m + c].copy()) for u, c in zip(range(nu), cnt)]
        return rows, dict(zip(("query_users", "exact_rows", "shared_users", "global_users"), (int(x) for x in stats)))

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()


class FMInput:
    """The factored input of gorse_b200_fm_rank, packed from Python lists.
    user_feat[u]: the user-id feature or -1; user_labels[u]: [(feature, scaled value)] in label order.
    item_feat / item_labels: the same per row of the call's item table.  item_emb[s]: uint16 (bf16 bits) [n_items, dim_s];
    item_emb_mask: uint8 [n_items, n_emb] (None: all present).  candidates[u]: item-table rows of user u."""

    def __init__(self, user_feat, user_labels, item_feat, item_labels, candidates, item_emb=(), item_emb_mask=None):
        def csr(rows):
            off = np.zeros(len(rows) + 1, np.int64)
            np.cumsum([len(r) for r in rows], out=off[1:])
            idx = np.ascontiguousarray([f for r in rows for f, _ in r] or [0], np.int32)
            val = np.ascontiguousarray([v for r in rows for _, v in r] or [0], np.float32)
            return off, idx, val

        self.user_feat = np.ascontiguousarray(user_feat, np.int32).reshape(-1)
        self.item_feat = np.ascontiguousarray(item_feat, np.int32).reshape(-1)
        self.n_users, self.n_items = self.user_feat.size, self.item_feat.size
        if len(user_labels) != self.n_users or len(candidates) != self.n_users or len(item_labels) != self.n_items:
            raise ValueError("one label list per user / item and one candidate list per user")
        self.user_lab_off, self.user_lab_idx, self.user_lab_val = csr(user_labels)
        self.item_lab_off, self.item_lab_idx, self.item_lab_val = csr(item_labels)
        self.cand_off = np.zeros(self.n_users + 1, np.int64)
        np.cumsum([len(c) for c in candidates], out=self.cand_off[1:])
        self.cand_items = np.ascontiguousarray(np.concatenate([np.asarray(c, np.int32).reshape(-1) for c in candidates] + [np.zeros(1, np.int32)]),
                                               np.int32)
        self.item_emb = [np.ascontiguousarray(e, np.uint16) for e in item_emb]
        self.item_emb_mask = None if item_emb_mask is None else np.ascontiguousarray(item_emb_mask, np.uint8)

    def split(self, scores, order):
        """per-user lists of (scores, order) from flat outputs"""
        return [(scores[a:b], order[a:b]) for a, b in zip(self.cand_off[:-1], self.cand_off[1:])]


class FMRanker:
    """A trained factorization machine on the GPU (gorse_b200_fm_*; model/ctr/fm.go AFM inference).  params: fm.Parameters()
    concatenated (B, V, W, then H, AW, Ab, EW, Eb per embedding slot)."""

    def __init__(self, ctx, n_features, n_factors, num_dimension, batch_size=1024, emb_dims=(), params=None):
        self.ctx, self.n_factors = ctx, int(n_factors)
        dims = np.ascontiguousarray(list(emb_dims) or [0], np.int32)
        self.n_emb = len(list(emb_dims))
        p = np.ascontiguousarray(params, np.float32).reshape(-1)
        h = C.c_void_p()
        check(lib.gorse_b200_fm_create(ctx.h, int(n_features), int(n_factors), int(num_dimension), int(batch_size), self.n_emb, ptr(dims),
                                       ptr(p), p.size, C.byref(h)))
        self.h = h

    def close(self):
        if self.h:
            lib.gorse_b200_fm_destroy(self.h)
            self.h = None

    def rank(self, inp):
        """-> (scores float32 [pairs] in candidate order, order int32 [pairs]: each user's candidate positions by score
        descending, ties by position, NaN last; stats {pairs, chunks, passes, global_sorts})"""
        total = int(inp.cand_off[-1])
        scores, order, stats = np.zeros(max(total, 1), np.float32), np.zeros(max(total, 1), np.int32), np.zeros(4, np.int64)
        embs = (C.c_void_p * max(self.n_emb, 1))(*[ptr(e) for e in inp.item_emb])
        check(lib.gorse_b200_fm_rank(self.h, inp.n_users, ptr(inp.user_feat), ptr(inp.user_lab_off), ptr(inp.user_lab_idx), ptr(inp.user_lab_val),
                                     inp.n_items, ptr(inp.item_feat), ptr(inp.item_lab_off), ptr(inp.item_lab_idx), ptr(inp.item_lab_val),
                                     C.cast(embs, C.c_void_p) if inp.item_emb else None, ptr(inp.item_emb_mask), ptr(inp.cand_off),
                                     ptr(inp.cand_items), ptr(scores), ptr(order), ptr(stats)))
        return scores[:total], order[:total], dict(zip(("pairs", "chunks", "passes", "global_sorts"), (int(x) for x in stats)))

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()


def _flat(lists, dtype):
    off = np.zeros(len(lists) + 1, np.int64)
    np.cumsum([len(x) for x in lists], out=off[1:])
    flat = np.ascontiguousarray(np.concatenate([np.asarray(x, dtype).reshape(-1) for x in lists] + [np.zeros(0, dtype)]), dtype)
    return off, flat


class ListStage:
    """A list recommender of gorse_b200_recommend: non-personalized or latest (items / scores: one list for every user) or
    external (per_user: one (items, scores) pair per user).  Items are dictionary indices."""

    def __init__(self, items=None, scores=None, per_user=None):
        self.items, self.scores, self.per_user = items, scores, per_user


class CollaborativeStage:
    """The collaborative recommender: the CF recall row (the `cf` argument of recommend) as the cache would serve it."""


class ItemToItemStage:
    """An item-to-item recommender on `collection`: context_lists[u] are item indices, newest first (-1 = outside the
    dictionary); slot_of_item [n_items] / item_of_slot [slots] map between the dictionary and the collection."""

    def __init__(self, collection, n, context_lists, slot_of_item, item_of_slot, categories=(), score_scale=1.0):
        self.collection, self.n, self.context_lists, self.categories, self.score_scale = collection, n, context_lists, categories, score_scale
        self.slot_of_item, self.item_of_slot = slot_of_item, item_of_slot


class UserToUserStage:
    """A user-to-user recommender on `collection`: user_slots[u] (-1 = no vector), feedback_lists[slot] as item indices,
    item_ok [n_items] (None: every item passes)."""

    def __init__(self, collection, n, user_slots, feedback_lists, item_ok=None, score_scale=1.0):
        self.collection, self.n, self.user_slots, self.feedback_lists, self.item_ok, self.score_scale = collection, n, user_slots, feedback_lists, item_ok, score_scale


def recommend(ctx, exclude_lists, n_items, item_live, stages, cf=None, ranker=None, replacement=None, positive_decay=1.0, read_decay=1.0):
    """Batched offline recommendation (gorse_b200_recommend; worker/pipeline.go:124-319): for user u, E0 = exclude_lists[u]
    (dictionary indices, -1 = an id outside it), the stages in order with one growing exclude set, the live candidates,
    then with a ranker the replacement items and the FM ranking with the decay.
    cf: (collection, user_vectors [n_users, dim], slot_of_item, item_of_slot, n) for a CollaborativeStage.
    ranker: (FMRanker, FMInput of the users and the dictionary's item table; its candidates are ignored).
    replacement: per user a list of (item, positive) pairs.
    -> ([(items int32, scores float64) per user], stats {chunks, candidates, table_rows, exact_rows})"""
    nu = len(exclude_lists)
    keep = []

    def p(a):
        if a is None:
            return None
        keep.append(a)
        return a.ctypes.data

    eoff, eitems = _flat(exclude_lists, np.int32)
    live = np.ascontiguousarray(item_live, np.uint8)
    arr = (_lib.RecommendStage * max(len(stages), 1))()
    for i, s in enumerate(stages):
        d = arr[i]
        if isinstance(s, ListStage):
            d.kind = _lib.STAGE_LIST
            if s.per_user is not None:
                loff, li = _flat([x[0] for x in s.per_user], np.int32)
                _, ls = _flat([x[1] for x in s.per_user], np.float64)
                d.list_off = p(loff)
            else:
                li, ls = np.ascontiguousarray(s.items, np.int32), np.ascontiguousarray(s.scores, np.float64)
                d.list_len = li.size
            d.list_items, d.list_scores = p(li), p(ls)
        elif isinstance(s, CollaborativeStage):
            d.kind = _lib.STAGE_COLLABORATIVE
        elif isinstance(s, ItemToItemStage):
            d.kind = _lib.STAGE_ITEM_TO_ITEM
            d.db, d.n, d.score_scale = s.collection.h.value, int(s.n), float(s.score_scale)
            coff, citems = _flat(s.context_lists, np.int32)
            d.ctx_off, d.ctx_items = p(coff), p(citems)
            d.slot_of_item = p(np.ascontiguousarray(s.slot_of_item, np.int64))
            d.item_of_slot = p(np.ascontiguousarray(s.item_of_slot, np.int32))
            cats = np.ascontiguousarray(list(s.categories), np.int32)
            d.categories, d.n_categories = (p(cats) if cats.size else None), cats.size
        elif isinstance(s, UserToUserStage):
            d.kind = _lib.STAGE_USER_TO_USER
            d.db, d.n, d.score_scale = s.collection.h.value, int(s.n), float(s.score_scale)
            d.user_slots = p(np.ascontiguousarray(s.user_slots, np.int64))
            foff, fitems = _flat(s.feedback_lists, np.int32)
            d.n_fb_rows, d.fb_off, d.fb_items = len(s.feedback_lists), p(foff), p(fitems)
            d.item_ok = None if s.item_ok is None else p(np.ascontiguousarray(s.item_ok, np.uint8))
        else:
            raise TypeError(f"unknown stage {s!r}")
    cfs = None
    if cf is not None:
        coll, vecs, soi, ios, n = cf
        cfs = _lib.RecommendCF(coll.h.value, p(np.ascontiguousarray(vecs, np.float32)), p(np.ascontiguousarray(soi, np.int64)),
                               p(np.ascontiguousarray(ios, np.int32)), int(n))
    rk = None
    if ranker is not None:
        fm, inp = ranker
        i32, i64, f32 = (lambda a: p(np.ascontiguousarray(a, np.int32))), (lambda a: p(np.ascontiguousarray(a, np.int64))), \
            (lambda a: p(np.ascontiguousarray(a, np.float32)))
        emb = [np.ascontiguousarray(e, np.uint16) for e in inp.item_emb]
        keep.extend(emb)
        embs = (C.c_void_p * max(fm.n_emb, 1))(*[ptr(e) for e in emb])
        keep.append(embs)
        mask = None if inp.item_emb_mask is None else np.ascontiguousarray(inp.item_emb_mask, np.uint8)
        rk = _lib.RecommendRanker(fm.h.value, i32(inp.user_feat), i64(inp.user_lab_off), i32(inp.user_lab_idx), f32(inp.user_lab_val),
                                  i32(inp.item_feat), i64(inp.item_lab_off), i32(inp.item_lab_idx), f32(inp.item_lab_val),
                                  C.cast(embs, C.c_void_p).value if emb else None, p(mask))
    roff = ritems = rpos = None
    if replacement is not None:
        roff, ritems = _flat([[it for it, _ in r] for r in replacement], np.int32)
        _, rpos = _flat([[1 if pos else 0 for _, pos in r] for r in replacement], np.uint8)
    bound = recommend_bounds(nu, stages, cf, replacement if ranker is not None else None)
    out_at = np.zeros(nu + 1, np.int64)
    np.cumsum(bound, out=out_at[1:])
    total = int(out_at[-1])
    items, scores, cnt, stats = np.zeros(max(total, 1), np.int32), np.zeros(max(total, 1), np.float64), np.zeros(max(nu, 1), np.int32), np.zeros(4, np.int64)
    check(lib.gorse_b200_recommend(ctx.h if ctx is not None else None, nu, ptr(eoff), ptr(eitems) if eitems.size else None, int(n_items), ptr(live) if live.size else None,
                                   len(stages), C.cast(arr, C.c_void_p), C.byref(cfs) if cfs is not None else None,
                                   C.byref(rk) if rk is not None else None, ptr(roff), ptr(ritems) if ritems is not None and ritems.size else None,
                                   ptr(rpos) if rpos is not None and rpos.size else None, float(positive_decay), float(read_decay), ptr(items), ptr(scores),
                                   ptr(cnt), ptr(stats)))
    rows = [(items[a:a + c].copy(), scores[a:a + c].copy()) for a, c in zip(out_at[:-1], cnt[:nu])]
    return rows, dict(zip(("chunks", "candidates", "table_rows", "exact_rows"), (int(x) for x in stats)))


def recommend_bounds(n_users, stages, cf=None, replacement=None):
    """B_u of gorse_b200_recommend: the stage bounds (list length, or n) plus the replacement count (ranked calls only)."""
    b = np.zeros(n_users, np.int64)
    for s in stages:
        if isinstance(s, ListStage):
            b += np.array([len(x[0]) for x in s.per_user], np.int64) if s.per_user is not None else len(s.items)
        elif isinstance(s, CollaborativeStage):
            b += max(int(cf[4]), 0) if cf is not None else 0
        else:
            b += max(int(s.n), 0)
    if replacement is not None:
        b += np.array([len(r) for r in replacement], np.int64)
    return b


class FMTrainer:
    """AFM.Fit (model/ctr/fm.go:307-417) on the GPU: fit() for a model without embedding slots (gorse_b200_fm_fit), fit_emb()
    for one with them (gorse_b200_fm_fit_emb).  The rows are CSRs (off int64 [n + 1], idx int32, val float32, already
    through fm.Scalers) with float32 targets; params_in is fm.Parameters() after Init, the layout FMRanker takes."""

    def __init__(self, ctx, n_features, num_dimension, n_factors=16, n_epochs=50, lr=0.001, reg=0.0002, optimizer=FM_ADAM,
                 batch_size=1024, verbose=10, patience=10, max_steps=0, n_emb=0):
        self.ctx, self.n_features, self.num_dimension, self.n_emb = ctx, int(n_features), int(num_dimension), int(n_emb)
        self.params = _lib.FMFitParams(int(n_factors), int(n_epochs), float(lr), float(reg), int(optimizer), int(batch_size), int(verbose),
                                       int(patience), int(max_steps))

    def n_params(self):
        return 1 + self.n_features * self.params.n_factors + self.n_features

    def fit_emb(self, train, test, params_in, emb_dims, item_emb, item_emb_mask, train_emb_row, test_emb_row, progress=None,
                moments=False):
        """fit() for a model with item-embedding slots: emb_dims [n_emb]; item_emb[s] = bf16 bits uint16 [n_rows, dim_s];
        item_emb_mask uint8 [n_rows, n_emb] or None (all present); train_emb_row / test_emb_row int32: the table row of
        every sample, -1 for none.  params_in holds B, V, W, then per slot H, AW, Ab, EW, Eb."""
        return self._fit(train, test, params_in, progress, moments, (emb_dims, item_emb, item_emb_mask, train_emb_row, test_emb_row))

    def fit(self, train, test, params_in, progress=None, moments=False):
        """train / test = (off, idx, val, target); progress(epoch, n_epochs, auc) -> truthy to cancel.
        -> (params float32 [n_params], result dict, moments float32 [2, n_params] or None)"""
        return self._fit(train, test, params_in, progress, moments, None)

    def _fit(self, train, test, params_in, progress, moments, _emb):
        def rows(r):
            off, idx, val, tgt = r
            off = np.ascontiguousarray(off, np.int64)
            return (off.size - 1, off, np.ascontiguousarray(idx, np.int32), np.ascontiguousarray(val, np.float32),
                    np.ascontiguousarray(tgt, np.float32))

        tr, te = rows(train), rows(test)
        pin = np.ascontiguousarray(params_in, np.float32).reshape(-1)
        want = self.n_params() + (sum(self.params.n_factors * (3 * int(d) + 2) for d in _emb[0]) if _emb else 0)
        if pin.size != want:
            raise ValueError(f"params_in holds {pin.size} floats, the model has {want}")
        pout = np.zeros(max(pin.size, 1), np.float32)
        mom = np.zeros((2, pin.size), np.float32) if moments else None
        res = _lib.FMFitResult()
        cb = _lib.PROGRESS_FN(lambda user, ep, n, auc: int(bool(progress(ep, n, auc)))) if progress else None
        if _emb is None:
            check(lib.gorse_b200_fm_fit(self.ctx.h, self.n_features, self.num_dimension, self.n_emb, C.byref(self.params), tr[0], ptr(tr[1]),
                                        ptr(tr[2]), ptr(tr[3]), ptr(tr[4]), te[0], ptr(te[1]), ptr(te[2]), ptr(te[3]), ptr(te[4]), ptr(pin),
                                        pin.size, ptr(pout), ptr(mom), cb, None, C.byref(res)))
        else:
            dims = np.ascontiguousarray(list(_emb[0]), np.int32)
            tabs = [np.ascontiguousarray(t, np.uint16) for t in _emb[1]]
            if len(tabs) != dims.size or any(t.ndim != 2 or t.shape[1] != d or t.shape[0] != tabs[0].shape[0] for t, d in zip(tabs, dims)):
                raise ValueError("item_emb needs one [n_rows, dim] table per slot")
            n_rows = tabs[0].shape[0] if tabs else 0
            mask = None if _emb[2] is None else np.ascontiguousarray(_emb[2], np.uint8)
            if mask is not None and mask.shape != (n_rows, dims.size):
                raise ValueError("item_emb_mask must be [n_rows, n_emb]")
            er = [np.ascontiguousarray(r, np.int32).reshape(-1) for r in _emb[3:5]]
            if er[0].size != tr[0] or er[1].size != te[0]:
                raise ValueError("one table row per training and per test sample")
            arr = (C.c_void_p * max(len(tabs), 1))(*[ptr(t) for t in tabs])
            check(lib.gorse_b200_fm_fit_emb(self.ctx.h, self.n_features, self.num_dimension, C.byref(self.params), tr[0], ptr(tr[1]), ptr(tr[2]),
                                            ptr(tr[3]), ptr(tr[4]), ptr(er[0]), te[0], ptr(te[1]), ptr(te[2]), ptr(te[3]), ptr(te[4]),
                                            ptr(er[1]), dims.size, ptr(dims), n_rows, arr, ptr(mask), ptr(pin), pin.size, ptr(pout), ptr(mom),
                                            cb, None, C.byref(res)))
        out = {f: getattr(res, f) for f, _ in _lib.FMFitResult._fields_}
        return pout[:pin.size], out, mom

    def fit_trials(self, trials, train, test, params_in_list, emb=None, progress=None, moments=False):
        """AFM's ModelSearch trials in one gorse_b200_fm_fit_trials call.  trials: one dict per trial overriding this trainer's
        params (lr, reg, optimizer and n_epochs may differ; n_factors, batch_size, verbose, patience and max_steps are
        shared); params_in_list: each trial's fm.Parameters() after its own Init.  emb: None, or (emb_dims, item_emb,
        item_emb_mask, train_emb_row, test_emb_row) as fit_emb takes them.  progress(epoch, states), states a list of
        (epochs_run, auc or -1, finished) per trial, returns True to cancel.
        -> one (params, result dict, moments or None) per trial, each equal to that trial's solo fit bit for bit"""
        n = len(trials)
        if n != len(params_in_list):
            raise ValueError("one params_in per trial")
        tr, te = self._rows(train), self._rows(test)
        fps = (_lib.FMFitParams * max(n, 1))()
        for i, over in enumerate(trials):
            C.memmove(C.byref(fps[i]), C.byref(self.params), C.sizeof(_lib.FMFitParams))
            for key, v in over.items():
                setattr(fps[i], key, v)
        dims, tabs, mask, er = self._emb(emb, tr, te)
        k = self.params.n_factors
        want = self.n_params() + sum(k * (3 * int(d) + 2) for d in dims)
        pins = [np.ascontiguousarray(p, np.float32).reshape(-1) for p in params_in_list]
        if any(p.size != want for p in pins):
            raise ValueError(f"every params_in must hold the model's {want} floats")
        pouts = [np.zeros(max(want, 1), np.float32) for _ in range(n)]
        moms = [np.zeros((2, want), np.float32) for _ in range(n)] if moments else None
        pin_arr = (C.c_void_p * max(n, 1))(*[ptr(p) for p in pins])
        pout_arr = (C.c_void_p * max(n, 1))(*[ptr(p) for p in pouts])
        mom_arr = (C.c_void_p * max(n, 1))(*[ptr(m) for m in moms]) if moments else None
        res = (_lib.FMFitResult * max(n, 1))()

        def on_epoch(user, epoch, n_trials, states):
            return int(bool(progress(epoch, [(states[i].epochs_run, states[i].auc, bool(states[i].finished)) for i in range(n_trials)])))

        cb = _lib.FM_TRIALS_PROGRESS_FN(on_epoch) if progress else None
        arr = (C.c_void_p * max(len(tabs), 1))(*[ptr(t) for t in tabs])
        n_rows = tabs[0].shape[0] if tabs else 0
        check(lib.gorse_b200_fm_fit_trials(self.ctx.h, self.n_features, self.num_dimension, n, C.cast(fps, C.c_void_p), tr[0], ptr(tr[1]),
                                           ptr(tr[2]), ptr(tr[3]), ptr(tr[4]), ptr(er[0]), te[0], ptr(te[1]), ptr(te[2]), ptr(te[3]),
                                           ptr(te[4]), ptr(er[1]), dims.size, ptr(dims), n_rows, arr if tabs else None, ptr(mask),
                                           C.cast(pin_arr, C.c_void_p), want, C.cast(pout_arr, C.c_void_p),
                                           C.cast(mom_arr, C.c_void_p) if moments else None, C.cast(cb, C.c_void_p) if cb else None, None,
                                           C.cast(res, C.c_void_p)))
        return [(pouts[i][:want], {f: getattr(res[i], f) for f, _ in _lib.FMFitResult._fields_}, moms[i] if moments else None)
                for i in range(n)]

    @staticmethod
    def _rows(r):
        off, idx, val, tgt = r
        off = np.ascontiguousarray(off, np.int64)
        return (off.size - 1, off, np.ascontiguousarray(idx, np.int32), np.ascontiguousarray(val, np.float32), np.ascontiguousarray(tgt, np.float32))

    @staticmethod
    def _emb(emb, tr, te):
        """(dims, tables, mask, (train rows, test rows)) of fit_trials' emb argument; None: no slots"""
        if emb is None:
            return np.zeros(0, np.int32), [], None, (None, None)
        dims = np.ascontiguousarray(list(emb[0]), np.int32)
        tabs = [np.ascontiguousarray(t, np.uint16) for t in emb[1]]
        if len(tabs) != dims.size or any(t.ndim != 2 or t.shape[1] != d or t.shape[0] != tabs[0].shape[0] for t, d in zip(tabs, dims)):
            raise ValueError("item_emb needs one [n_rows, dim] table per slot")
        n_rows = tabs[0].shape[0] if tabs else 0
        mask = None if emb[2] is None else np.ascontiguousarray(emb[2], np.uint8)
        if mask is not None and mask.shape != (n_rows, dims.size):
            raise ValueError("item_emb_mask must be [n_rows, n_emb]")
        er = [np.ascontiguousarray(r, np.int32).reshape(-1) for r in emb[3:5]]
        if er[0].size != tr[0] or er[1].size != te[0]:
            raise ValueError("one table row per training and per test sample")
        return dims, tabs, mask, er


def user_feedback_counts(train, n_users):
    """feedbackCount of `gorse-bench reranker` (cmd/gorse-bench/main.go:133-140): per user, the training rows with target > 0
    whose first index is the user.  train = (off, idx, val, target) -> int64 [n_users]"""
    off, idx, _, tgt = train
    off = np.asarray(off, np.int64)
    first = np.asarray(idx, np.int64)[off[:-1][np.diff(off) > 0]]
    pos = np.asarray(tgt, np.float32)[np.diff(off) > 0] > 0
    return np.bincount(first[pos], minlength=n_users).astype(np.int64)


def ranker_gauc(ctx, n_features, n_factors, num_dimension, params, test, n_users, feedback_count, context_size=100, batch_size=1024,
                emb=None, predictions=False):
    """The AFM half of `gorse-bench reranker` after the fit (gorse_b200_fm_gauc): every test row predicted as one list in test
    order, then per user (the first index of its rows) the AUC of its positives against its negatives, and GAUC.
    params: fm.Parameters() as FMRanker takes them; test = (off, idx, val, target) with values through fm.Scalers;
    feedback_count [n_users] (user_feedback_counts); emb: None, or (emb_dims, item_emb, item_emb_mask, test_emb_row) as
    FMTrainer.fit_emb takes them.
    -> dict: gauc (float), users, feedback, candidates, auc (one entry per scored user, ascending user), stats {rows,
    users, scored, chained, nan} and predictions (float32 [n_test] when asked for, else None)"""
    n, off, idx, val, tgt = FMTrainer._rows(test)
    p = np.ascontiguousarray(params, np.float32).reshape(-1)
    dims, tabs, mask, er = FMTrainer._emb(None if emb is None else (emb[0], emb[1], emb[2], np.zeros(0, np.int32), emb[3]), (0,), (n,))
    fb = np.ascontiguousarray(feedback_count, np.int64).reshape(-1)
    if fb.size != n_users:
        raise ValueError("one feedback count per user")
    m = max(int(n_users), 1)
    users, feedback, cand, auc = np.zeros(m, np.int32), np.zeros(m, np.int64), np.zeros(m, np.int64), np.zeros(m, np.float32)
    pred = np.zeros(max(n, 1), np.float32) if predictions else None
    stats, ns, g = np.zeros(5, np.int64), C.c_int64(0), C.c_double(0)
    arr = (C.c_void_p * max(len(tabs), 1))(*[ptr(t) for t in tabs])
    check(lib.gorse_b200_fm_gauc(ctx.h, int(n_features), int(n_factors), int(num_dimension), int(batch_size), dims.size, ptr(dims), ptr(p), p.size,
                                 n, ptr(off), ptr(idx), ptr(val), ptr(tgt), ptr(er[1]), tabs[0].shape[0] if tabs else 0, arr if tabs else None,
                                 ptr(mask), int(n_users), ptr(fb), int(context_size), ptr(pred), ptr(users), ptr(feedback), ptr(cand), ptr(auc),
                                 C.byref(ns), C.byref(g), ptr(stats)))
    k = ns.value
    return dict(gauc=g.value, users=users[:k], feedback=feedback[:k], candidates=cand[:k], auc=auc[:k],
                stats=dict(zip(("rows", "users", "scored", "chained", "nan"), (int(x) for x in stats))),
                predictions=None if pred is None else pred[:n])


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


def evaluate_embeddings(ctx, emb, mask, shots, test, excl, negatives=None, n_candidates=99, seed=0, topk=10):
    """`gorse-bench embedding`'s scoring (gorse_b200_embedding_eval) for every user at once.  emb [n_items, dim] float32, mask
    [n_items] (None: every item has an embedding); shots, test, excl and negatives are (off, items) CSRs over the users; with
    negatives None they are sampled on the device under seed, excluding test(u) and excl(u).
    -> (ndcg, precision, recall, users scored)"""
    emb = np.ascontiguousarray(emb, np.float32)
    if emb.ndim != 2:
        raise ValueError("emb must be [n_items, dim]")
    mask = None if mask is None else np.ascontiguousarray(mask, np.uint8)
    if mask is not None and mask.shape != (emb.shape[0],):
        raise ValueError("mask must be [n_items]")

    def csr(pair):
        if pair is None:
            return None, None
        off = np.ascontiguousarray(pair[0], np.int64)
        return off, np.ascontiguousarray(pair[1], np.int32)

    (so, si), (to, ti), (xo, xi), (no, ni) = csr(shots), csr(test), csr(excl), csr(negatives)
    out, users = np.zeros(3, np.float32), C.c_int64(0)
    check(lib.gorse_b200_embedding_eval(ctx.h, emb.shape[0], emb.shape[1], ptr(emb), ptr(mask), len(so) - 1, ptr(so), ptr(si), ptr(to), ptr(ti),
                                        ptr(xo), ptr(xi), ptr(no), ptr(ni), int(n_candidates), int(seed), int(topk), ptr(out), C.byref(users)))
    return np.float32(out[0]), np.float32(out[1]), np.float32(out[2]), users.value


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
