"""ctypes view of the CPU restatement of `gorse-bench embedding`'s scoring (embedding_oracle/libembedding_oracle.so), plus the
dataset split and the seeded data its checks use.

TEST INFRASTRUCTURE ONLY: importable from tests/ and tools/.  The product package (gorse_b200) never imports this.  It lives
beside the general oracle (oracle/), whose primitives it links, and checks gorse_b200_embedding_eval; see
embedding_oracle.c.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libembedding_oracle.so")
_SRC = os.path.join(_HERE, "embedding_oracle.c")
_ORACLE_DIR = os.path.join(_HERE, "..", "oracle")


def build(force=False):
    import oracle

    oracle.build()
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(_SRC):
        subprocess.check_call(["gcc", "-O2", "-std=gnu11", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-o", _SO, _SRC,
                               "-L" + _ORACLE_DIR, "-l:libgorse_oracle.so", "-Wl,-rpath,$ORIGIN/../oracle"])


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_SO)
        VP = C.c_void_p
        L.gbo_evaluate_embedding.restype = C.c_int64
        L.gbo_evaluate_embedding.argtypes = [C.c_int32, C.c_int32, VP, VP, C.c_int32, VP, VP, VP, VP, VP, VP, C.c_int32, VP]
        _lib = L
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _c(a, dt):
    return np.ascontiguousarray(a, dt)


def _csr(pair):
    off, items = pair
    off = _c(off, np.int64)
    return off - off[0], _c(np.append(np.asarray(items, np.int32)[:int(off[-1] - off[0])], 0), np.int32)


def evaluate(emb, mask, shots, test, negatives, topk=10):
    """EvaluateEmbedding with jobs = 1 on (off, items) CSRs -> (ndcg, precision, recall, users)"""
    emb = _c(emb, np.float32)
    n_items, dim = emb.shape
    mask = None if mask is None else _c(mask, np.uint8)
    (so, si), (to, ti), (no, ni) = _csr(shots), _csr(test), _csr(negatives)
    out = np.zeros(3, np.float32)
    users = lib().gbo_evaluate_embedding(n_items, dim, _p(emb), _p(mask), len(so) - 1, _p(so), _p(si), _p(to), _p(ti), _p(no), _p(ni),
                                         int(topk), _p(out))
    return np.float32(out[0]), np.float32(out[1]), np.float32(out[2]), int(users)


def sample_negatives(n_items, excl, test, n_cand, seed=0):
    """the negatives gorse_b200_embedding_eval samples when none are passed: SampleUserNegatives excluding test(u) and the
    user's dataset feedback excl(u), with the library's counter RNG"""
    import oracle

    xo, xi = _csr(excl)
    xi = xi[:-1].copy()
    for u in range(len(xo) - 1):
        xi[xo[u]:xo[u + 1]].sort()
    to, ti = _csr(test)
    return oracle.sample_user_negatives(n_items, xo, xi, to, ti[:-1], n_cand, seed=seed)


def split_latest(off, items, ts, shots):
    """dataset.SplitLatest(shots) (dataset/dataset.go:321-351) on a feedback CSR with timestamps: per user with feedback the
    newest item is the test row and the next min(shots, len - 1) items, newest first, the train row.  Equal timestamps keep
    their CSR order (the reference's sort.Slice leaves them unpinned).  -> ((train_off, train_items), (test_off, test_items))"""
    off, items, ts = np.asarray(off, np.int64), np.asarray(items, np.int32), np.asarray(ts)
    n = len(off) - 1
    lens = np.diff(off)
    user = np.repeat(np.arange(n), lens)
    order = np.lexsort((np.arange(len(items)), -ts.astype(np.float64), user))   # by user, newest first, then position
    srt = items[order]
    pos = np.arange(len(items)) - np.repeat(off[:-1], lens)
    te_mask = pos == 0
    tr_mask = (pos >= 1) & (pos <= shots)
    te_off, tr_off = np.zeros(n + 1, np.int64), np.zeros(n + 1, np.int64)
    np.cumsum(np.bincount(user[te_mask], minlength=n), out=te_off[1:])
    np.cumsum(np.bincount(user[tr_mask], minlength=n), out=tr_off[1:])
    return (tr_off, srt[tr_mask].astype(np.int32)), (te_off, srt[te_mask].astype(np.int32))
