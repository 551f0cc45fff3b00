"""The CPU restatement of `gorse-bench reranker`'s per-user AUC and GAUC (fmo_gauc in fm_oracle/fm_fit_oracle.c) on
hand-built predictions, and gorse_b200_fm_gauc's argument errors with a NULL context (no device needed)."""
import ctypes as C

import numpy as np

import fm_oracle

f32 = np.float32


def rows(users, preds, targets):
    return np.array(preds, f32), np.array(users, np.int32), np.array(targets, f32)


def test_ties_are_not_counted():
    # user 0: positives 1, 2 against negatives 1, 0.5 -> 1 counts 0.5 only, 2 counts both: 3 / 4
    p, u, t = rows([0, 0, 0, 0], [1.0, 2.0, 1.0, 0.5], [1, 1, -1, -1])
    g, users, cand, auc = fm_oracle.gauc(p, u, t, 1, [1])
    assert users.tolist() == [0] and cand.tolist() == [4] and auc.tolist() == [0.75] and g == 0.75


def test_negative_zero_ties_positive_zero():
    p, u, t = rows([0, 0, 1, 1], [-0.0, 0.0, 0.0, -0.0], [1, -1, 1, -1])
    g, users, _, auc = fm_oracle.gauc(p, u, t, 2, [1, 1])
    assert users.tolist() == [0, 1] and auc.tolist() == [0.0, 0.0] and g == 0.0


def test_skip_rules():
    # users 0..5: feedback 0 (skipped), == context (kept), context + 1 (skipped), only positives, only negatives, no rows
    ctx = 3
    p, u, t = rows([0, 0, 1, 1, 2, 2, 3, 4], [1, 0, 1, 0, 1, 0, 1, 0], [1, -1, 1, -1, 1, -1, 1, -1])
    g, users, cand, auc = fm_oracle.gauc(p, u, t, 6, [0, ctx, ctx + 1, 1, 1, 1], context_size=ctx)
    assert users.tolist() == [1] and cand.tolist() == [2] and auc.tolist() == [1.0] and g == 1.0
    g, users, _, _ = fm_oracle.gauc(p, u, t, 6, [0, 0, 0, 1, 1, 1], context_size=ctx)
    assert users.size == 0 and g == 0.0


def test_weighted_sum_in_float32():
    # AUC 1/3 weighted by 4 candidates, AUC 1 by 2: sum and count in float32, unfused, in user order
    p, u, t = rows([0, 0, 0, 0, 1, 1], [0.5, 0.1, 0.9, 0.7, 1, 0], [1, -1, -1, -1, 1, -1])
    g, _, cand, auc = fm_oracle.gauc(p, u, t, 2, [1, 1])
    assert auc[0] == f32(1) / f32(3) and cand.tolist() == [4, 2]
    s = f32(auc[0]) * f32(4) + f32(1) * f32(2)
    assert g == float(s / f32(6))


def test_count_rounds_in_float32():
    # user 0: one positive above 2^24 negatives (2^24 + 1 candidates, float32 2^24); user 1: 1 + 2 candidates
    n0 = (1 << 24) + 1
    p = np.full(n0 + 3, -1.0, f32)
    p[0] = 1.0
    p[n0], p[n0 + 1] = 0.0, 0.5
    u = np.zeros(n0 + 3, np.int32)
    u[n0:] = 1
    t = np.full(n0 + 3, -1.0, f32)
    t[0] = t[n0] = 1.0
    g, _, cand, auc = fm_oracle.gauc(p, u, t, 2, [1, 1])
    assert cand.tolist() == [n0, 3] and auc[0] == 1.0 and auc[1] == f32(0.5)
    c0, c1 = f32(n0), f32(3)
    assert c0 == f32(1 << 24) and c0 + c1 == f32((1 << 24) + 4)   # the count rounds twice
    want = float((auc[0] * c0 + auc[1] * c1) / (c0 + c1))
    exact = (n0 + 0.5 * 3) / (n0 + 3)
    assert g == want and g != exact


def test_chain_above_2_24_pairs_is_sequential():
    # every positive above every negative: counts of N = 4999, P = 5000; past 2^24 the float32 chain drops the odd sums' 1s
    P, N = 5000, 4999
    p = np.concatenate([np.ones(P, f32), np.zeros(N, f32)])
    t = np.concatenate([np.ones(P, f32), -np.ones(N, f32)])
    _, _, _, auc = fm_oracle.gauc(p, np.zeros(P + N, np.int32), t, 1, [1])
    s = f32(0)
    for _ in range(P):
        s = f32(s + f32(N))
    assert int(s) != P * N
    assert auc[0] == s / f32(P * N)


def test_nan_prediction_gives_nan():
    p, u, t = rows([0, 0, 1, 1], [np.nan, 0, 1, 0], [1, -1, 1, -1])
    g, users, _, auc = fm_oracle.gauc(p, u, t, 2, [1, 1])
    assert users.tolist() == [0, 1] and np.isnan(auc[0]) and auc[1] == 1.0 and np.isnan(g)


# ---- argument checks with a NULL context ------------------------------------------------------------------------------
def ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def call(_lib, nf=10, k=4, bs=8, n_params=None, off=None, idx=None, n_users=3, fb=None, n_emb=0, dims=None, emb_rows=None, n_test=None,
         out=True, tgt=True):
    off = np.array([0, 2, 4, 5], np.int64) if off is None else np.asarray(off, np.int64)
    idx = np.array([0, 5, 1, 6, 2], np.int32) if idx is None else np.asarray(idx, np.int32)
    val = np.ones(max(idx.size, 1), np.float32)
    target = np.array([1, -1, 1], np.float32)
    n = off.size - 1 if n_test is None else n_test
    dims = np.array(dims or [0], np.int32)
    want = 1 + nf * k + nf + sum(3 * k * int(d) + 2 * k for d in dims[:n_emb])
    params = np.zeros(want if n_params is None else n_params, np.float32)
    fb = np.ones(max(n_users, 1), np.int64) if fb is None else np.asarray(fb, np.int64)
    er = None if emb_rows is None else np.asarray(emb_rows, np.int32)
    table = np.zeros(int(dims.max()) or 1, np.uint16)
    tabs = (C.c_void_p * 1)(ptr(table))
    ns, g = C.c_int64(0), C.c_double(0)
    return _lib.lib.gorse_b200_fm_gauc(None, nf, k, 4, bs, n_emb, ptr(dims), ptr(params), params.size, n, ptr(off), ptr(idx), ptr(val),
                                       ptr(target) if tgt else None, ptr(er), 1, tabs if n_emb else None, None, n_users, ptr(fb), 100, None, None, None, None,
                                       None, C.byref(ns) if out else None, C.byref(g), None)


def test_argument_errors_without_a_device(gb):
    from gorse_b200 import _lib

    def err(**kw):
        st = call(_lib, **kw)
        return st, _lib.lib.gorse_b200_last_error().decode()

    assert err() == (_lib.ERR_ARG, "ctx is NULL")   # every argument is valid: the context is checked last
    for kw, word in [(dict(bs=0), "batch_size"), (dict(n_params=5), "n_params"), (dict(n_users=-1), "n_users"),
                     (dict(n_users=2), "user 2"), (dict(idx=[0, 5, 1, 6, 10]), "feature"), (dict(off=[0, 2, 2, 5]), "no features"),
                     (dict(fb=[1, -1, 1]), "negative feedback"), (dict(off=[0, 2, 1, 5]), "decrease"), (dict(out=False), "n_scored_out"),
                     (dict(tgt=False), "targets"), (dict(n_emb=1, dims=[16]), "test_emb_row"),
                     (dict(n_emb=1, dims=[16], emb_rows=[0, -1, 1]), "table row"),
                     (dict(nf=(1 << 24) + 4, n_params=1, idx=[0, 5, 1, 6, (1 << 24) + 3]), "float32")]:
        st, msg = err(**kw)
        assert st == _lib.ERR_ARG and word in msg, (kw, msg)
    for kw, word in [(dict(k=33), "n_factors"), (dict(n_emb=1, dims=[1025], emb_rows=[-1, -1, -1]), "dim"), (dict(n_test=1 << 31), "test rows")]:
        st, msg = err(**kw)
        assert st == _lib.ERR_UNSUPPORTED and word in msg, (kw, msg)
    # no rows: nothing to check but the context
    assert err(off=[0], idx=[], n_users=0) == (_lib.ERR_ARG, "ctx is NULL")
