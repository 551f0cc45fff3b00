"""The session recommendation restatement (session_model.py) on hand-built neighbour lists, and
gorse_b200_vecdb_session_recommend's argument errors with a NULL collection (no device needed)."""
import numpy as np

import session_model as sm

# the reference's TestSessionRecommend (server/rest_test.go:1803-1886) on a tags collection: slots 0..8 = ids "1".."9",
# slot 9 = "100" (hidden, never a neighbour); every vector is a set of tags with weight 1, so a neighbour's score is the
# number of shared tags.  Items "1".."5" exist only as vectors, "100" is hidden in the data store.
TAGS = [{0}, {1}, {2}, {3}, {4}, {3}, {2, 3}, {1, 2, 3}, {0, 1, 2, 3}]


def tags_neighbours(c):
    scored = [(j, len(TAGS[c] & TAGS[j])) for j in range(len(TAGS)) if j != c and TAGS[c] & TAGS[j]]
    scored.sort(key=lambda t: (-t[1], t[0]))
    return [j for j, _ in scored], [float(s) for _, s in scored]


def rows_as_lists(rows):
    return [(s.tolist(), v.tolist()) for s, v in rows]


def test_reference_known_answer():
    ok = np.zeros(10, np.uint8)
    ok[5:9] = 1                                      # "6", "7", "8", "9"
    ctx, ex = [[0, 1, 2, 3, 4]], [[0, 1, 2, 3, 4]]   # newest first; the session's items are its exclude set
    assert rows_as_lists(sm.session_rows(tags_neighbours, ctx, ex, 4, 3, ok)) == [([8, 7, 6], [4.0, 3.0, 2.0])]
    # category "*": "7" and "9"
    ok_star = np.zeros(10, np.uint8)
    ok_star[[6, 8]] = 1
    assert rows_as_lists(sm.session_rows(tags_neighbours, ctx, ex, 4, 3, ok_star)) == [([8, 6], [4.0, 2.0])]


def lists(table):
    return lambda c: table.get(c, ((), ()))


def test_a_list_emptied_by_item_ok_does_not_count():
    nb = lists({0: ([5], [1.0]), 1: ([6], [2.0]), 2: ([7], [3.0])})
    ok = np.ones(8, np.uint8)
    ok[5] = 0
    # context_size 1: entry 0's list is empty after the filter, so entry 1 is the one that counts
    assert rows_as_lists(sm.session_rows(nb, [[0, 1, 2]], [[]], 1, 10, ok)) == [([6], [2.0])]
    assert rows_as_lists(sm.session_rows(nb, [[0, 1, 2]], [[]], 1, 10)) == [([5], [1.0])]


def test_a_list_of_excluded_items_still_counts():
    nb = lists({0: ([5], [1.0]), 1: ([6], [2.0])})
    assert rows_as_lists(sm.session_rows(nb, [[0, 1]], [[5]], 1, 10)) == [([], [])]
    assert rows_as_lists(sm.session_rows(nb, [[0, 1]], [[5]], 2, 10)) == [([6], [2.0])]


def test_missing_items_and_repeats():
    nb = lists({0: ([5, 6], [0.5, 0.25])})
    # -1 and an item without neighbours give empty lists and do not count; the repeat of 0 counts and adds again
    assert rows_as_lists(sm.session_rows(nb, [[-1, 3, 0, 0, 0]], [[]], 2, 10)) == [([5, 6], [1.0, 0.5])]
    # context_size <= 0 stops after the first entry that counts, as the handler's `used >= ContextSize`
    assert rows_as_lists(sm.session_rows(nb, [[0, 0]], [[]], 0, 10)) == [([5, 6], [0.5, 0.25])]


def test_float64_sums_in_context_order():
    a, b, c = 0.1, 0.2, 0.3
    nb = lists({0: ([5], [a]), 1: ([5], [b]), 2: ([5], [c])})
    fwd = sm.session_rows(nb, [[0, 1, 2]], [[]], 10, 1)[0][1][0]
    rev = sm.session_rows(nb, [[2, 1, 0]], [[]], 10, 1)[0][1][0]
    assert fwd == (a + b) + c and rev == (c + b) + a and fwd != rev


def test_top_cut_and_tie_order():
    nb = lists({0: ([9, 4, 7, 2], [1.0, 2.0, 1.0, 3.0])})
    assert rows_as_lists(sm.session_rows(nb, [[0]], [[]], 1, 3)) == [([2, 4, 7], [3.0, 2.0, 1.0])]
    assert rows_as_lists(sm.session_rows(nb, [[0]], [[]], 1, 10)) == [([2, 4, 7, 9], [3.0, 2.0, 1.0, 1.0])]
    assert rows_as_lists(sm.session_rows(nb, [[0]], [[]], 1, 0)) == [([], [])]


# ---- argument checks with a NULL collection ---------------------------------------------------------------------------
def raw_call(gb, h, ctx_lists, ex_lists, n=10, context_size=100, top=10, scale=1.0, ctx_off=None, null_ctx_off=False, null_out=False):
    from gorse_b200 import _lib

    ns = len(ctx_lists)
    co = np.concatenate([[0], np.cumsum([len(x) for x in ctx_lists])]).astype(np.int64) if ctx_off is None else np.asarray(ctx_off, np.int64)
    cs = np.asarray([x for l in ctx_lists for x in l], np.int64)
    eo = np.concatenate([[0], np.cumsum([len(x) for x in ex_lists])]).astype(np.int64)
    es = np.asarray([x for l in ex_lists for x in l], np.int64)
    m = max(top, 1)
    slots, scores, cnt = np.zeros(ns * m + 1, np.int64), np.zeros(ns * m + 1, np.float64), np.zeros(ns + 1, np.int32)
    return _lib.lib.gorse_b200_vecdb_session_recommend(h, ns, None if null_ctx_off else gb.ptr(co), gb.ptr(cs) if cs.size else None, gb.ptr(eo),
                                                       gb.ptr(es) if es.size else None, None, n, context_size, top, scale,
                                                       None if null_out else gb.ptr(slots), gb.ptr(scores), gb.ptr(cnt), None)


def test_argument_errors_without_a_device(gb):
    from gorse_b200 import _lib

    def err(*a, **kw):
        return raw_call(gb, None, *a, **kw), _lib.lib.gorse_b200_last_error().decode()

    ok_args = ([[1, 2], [3]], [[1, 2], [3, -1]])
    assert err(*ok_args) == (_lib.ERR_ARG, "collection is NULL")   # every argument is valid: the collection is checked last
    for kw, word in [(dict(null_ctx_off=True), "NULL"), (dict(null_out=True), "NULL"), (dict(ctx_off=[0, 2, 1]), "decreases"),
                     (dict(scale=float("nan")), "NaN")]:
        st, msg = err(*ok_args, **kw)
        assert st == _lib.ERR_ARG and word in msg, (kw, msg)
    for a, word in [(([[1], [2]], [[5, 5], []]), "twice"), (([[1, -2]], [[]]), "not a slot"), (([[1]], [[-3]]), "not a slot")]:
        st, msg = err(*a)
        assert st == _lib.ERR_ARG and word in msg, (a, msg)
    assert err([[1], [2]], [[5, -1, -1], []]) == (_lib.ERR_ARG, "collection is NULL")   # -1 may repeat
    st, msg = err(*ok_args, top=1025)
    assert st == _lib.ERR_UNSUPPORTED and "top" in msg
    assert err([], [])[1] == "collection is NULL"
