"""`gorse-bench embedding`'s scoring without a GPU: the oracle's known answer on hand-built points, the dataset split, and
gorse_b200_embedding_eval's argument checks, which run on the host before the device is touched (the context last)."""
import ctypes as C

import numpy as np
import pytest

import embedding_oracle as eo

# 2-D integer points whose distances are 3-4-5 triangles; item 4 has no embedding
POINTS = np.array([[0, 0], [3, 4], [6, 8], [0, 5], [9, 9], [-3, -4]], np.float32)
MASK = np.array([1, 1, 1, 1, 0, 1], np.uint8)


def csr(rows):
    off = np.zeros(len(rows) + 1, np.int64)
    np.cumsum([len(r) for r in rows], out=off[1:])
    return off, np.array([i for r in rows for i in r], np.int32)


def known_case():
    shots = csr([[0], [4], [0, 5], [0], []])
    test = csr([[1], [1], [3], [], [2]])
    negs = csr([[2, 4, 3], [2], [1, 2], [1], [1]])
    return shots, test, negs


def embed(points, dim):
    """the points in `dim` dimensions: x at element 0, y at the last element (the d % 16 tail when dim = 17)"""
    e = np.zeros((len(points), dim), np.float32)
    e[:, 0], e[:, dim - 1] = points[:, 0], points[:, 1]
    return e


@pytest.mark.parametrize("dim", [2, 17])
def test_oracle_known_answer(dim):
    # user 0: totals 1 -> -5, 2 -> -10, 3 -> -5 (item 4 has no embedding); with topk = 1 the tie at the cut keeps item 3, the
    #         later push: container/heap pops the root (item 1) when the filter overflows.  NDCG = Precision = Recall = 0.
    # user 1: its only shot has no embedding: no candidate enters the filter, the user is skipped.
    # user 2: two shots in order; 2 -> -10 - 15 = -25, 1 -> -5 - 10 = -15, 3 -> -5 - sqrt(90) = -14.49: item 3, the test
    #         item, ranks first: 1, 1, 1.
    # user 3: no test item; user 4: no shot.  Both skipped.
    shots, test, negs = known_case()
    nd, pr, rc, users = eo.evaluate(embed(POINTS, dim), MASK, shots, test, negs, topk=1)
    assert users == 2
    assert (nd, pr, rc) == (np.float32(0.5), np.float32(0.5), np.float32(0.5))


def test_oracle_known_answer_top2():
    # topk = 2: user 0 ranks [1, 3] (the tie pops in push order) -> NDCG 1, Precision 1/2, Recall 1; user 2 ranks [3, 1]
    shots, test, negs = known_case()
    nd, pr, rc, users = eo.evaluate(embed(POINTS, 17), MASK, shots, test, negs, topk=2)
    assert users == 2
    assert nd == np.float32(1.0) and pr == np.float32(0.5) and rc == np.float32(1.0)


def test_oracle_no_user_scored_is_zero():
    shots, test, negs = csr([[4]]), csr([[1]]), csr([[2]])
    assert eo.evaluate(embed(POINTS, 2), MASK, shots, test, negs, topk=5) == (0.0, 0.0, 0.0, 0)


def test_split_latest():
    off, items = csr([[5, 6, 7, 8], [9], [], [1, 2, 3]])
    ts = np.array([10, 40, 20, 30, 5, 3, 1, 2])
    (tro, tri), (teo, tei) = eo.split_latest(off, items, ts, shots=2)
    assert teo.tolist() == [0, 1, 2, 2, 3] and tei.tolist() == [6, 9, 1]
    assert tro.tolist() == [0, 2, 2, 2, 4] and tri.tolist() == [8, 7, 3, 2]
    (tro, tri), _ = eo.split_latest(off, items, ts, shots=1 << 62)
    assert tri.tolist() == [8, 7, 5, 3, 2]


# ---- argument checks with a NULL context ------------------------------------------------------------------------------
def ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def call(_lib, dim=4, n_items=6, topk=10, shots=None, test=None, excl=None, negs=None, n_cand=3, emb=None, out=True):
    shots = shots or csr([[0, 1], [2]])
    test = test or csr([[3], [4]])
    excl = excl if excl is not None else csr([[0, 1, 3], [2, 4]])
    emb = np.zeros((max(n_items, 1), max(dim, 1)), np.float32) if emb is None else emb
    o, users = np.zeros(3, np.float32), C.c_int64(0)
    ex = (None, None) if excl is False else excl
    ng = (None, None) if negs is None else negs
    return _lib.lib.gorse_b200_embedding_eval(None, n_items, dim, ptr(emb), None, len(shots[0]) - 1, ptr(shots[0]), ptr(shots[1]),
                                              ptr(test[0]), ptr(test[1]), ptr(ex[0]), ptr(ex[1]), ptr(ng[0]), ptr(ng[1]), n_cand, 0, topk,
                                              ptr(o) if out else None, C.byref(users))


def test_argument_errors_without_a_device(gb):
    from gorse_b200 import _lib

    def err(**kw):
        st = call(_lib, **kw)
        return st, _lib.lib.gorse_b200_last_error().decode()

    assert err() == (_lib.ERR_ARG, "NULL ctx")   # every argument is valid: the context is checked last
    for kw, word in [(dict(dim=0), "dim"), (dict(dim=16385), "dim"), (dict(topk=0), "topk"), (dict(topk=129), "topk"),
                     (dict(shots=csr([[0, 6], [2]])), "shot item"), (dict(test=csr([[-1], [4]])), "test item"),
                     (dict(excl=csr([[0, 9], []])), "excl item"), (dict(negs=csr([[1], [7]])), "neg item"),
                     (dict(n_cand=-1), "n_candidates"), (dict(excl=False), "excl_off"), (dict(out=False), "out")]:
        st, msg = err(**kw)
        assert st == _lib.ERR_ARG and word in msg, (kw, msg)
    off = np.array([0, 2, 1], np.int64)
    st, msg = err(test=(off, np.array([3, 4], np.int32)))
    assert st == _lib.ERR_ARG and "non-decreasing" in msg
    # the per-user bound: (candidates) x (shots with an embedding) above 2^28 distances
    many = csr([list(range(5)) * 200, [2]])
    st, msg = err(shots=many, n_cand=(1 << 28) // 1000 + 1)
    assert st == _lib.ERR_UNSUPPORTED and "distances" in msg
    assert err(shots=many, n_cand=(1 << 28) // 1000 - 1) == (_lib.ERR_ARG, "NULL ctx")
