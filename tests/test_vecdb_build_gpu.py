"""Sparse similarity collections built on the device (gorse_b200_vecdb_add_idf_vectors): every added vector equals
appendSparseVector of its row's sorted, de-duplicated ids (oracle.sparse_vector, A then B for "auto") bit for bit, empty vectors
are not added, and a collection built this way answers every search exactly as the same vectors added with vecdb_add do --
after a rewrite cycle (a second build with replace, delete_before, compact) and when host adds and device builds are mixed.
Errors that need the ids leave the collection exactly as it was."""
import types

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

TILE = 8192
N = 3 * TILE + 517          # rows: four tiles of the sparse search
N_FEAT = 6000               # feedback ids of a part
N_TAGS = 300                # tag ids of "auto"
LONG = 1234                 # the row of more than 100K ids
KINDS = ("users", "auto")


@pytest.fixture(scope="module")
def ctx(gb):
    c = gb.Context(0)
    yield c
    c.close()


def make_idf(rng, n):
    idf = (rng.random(n) * 4 + 0.01).astype(np.float32)
    idf[rng.random(n) < 0.03] = 0
    idf[rng.random(n) < 0.02] *= -1
    return idf


def make_rows(rng, n, n_ids, long_row=None):
    """n rows of ids in any order: most 0..30 ids from a popular range, repeats, negative ids, ids >= n_ids, every 17th row empty,
    every 23rd row only ids that are skipped; row long_row holds 120,000 ids"""
    rows = []
    for r in range(n):
        if r == long_row:
            ids = rng.integers(-5, n_ids + 5, 120_000)
        elif r % 17 == 0:
            ids = np.zeros(0, np.int64)
        elif r % 23 == 0:
            ids = np.array([-1, n_ids, n_ids + 7, -3])[: int(rng.integers(1, 5))]
        else:
            k = int(rng.integers(1, 31))
            ids = np.where(rng.random(k) < 0.8, rng.integers(0, min(n_ids, 400), k), rng.integers(0, n_ids, k))
            if rng.random() < 0.3:
                ids = np.concatenate([ids, ids[: int(rng.integers(1, 4))]])   # the same id from two feedback types
            if rng.random() < 0.1:
                ids = np.concatenate([ids, [-2, n_ids + 1]])
            ids = rng.permutation(ids)
        rows.append(np.asarray(ids, np.int32))
    return rows


def expected(orc, a_rows, a_idf, b_rows=None, b_idf=None):
    """appendSparseVector of the sorted, de-duplicated ids: part A at offset 0, then part B at offset len(a_idf)"""
    out = []
    for i, a in enumerate(a_rows):
        ind, val = orc.sparse_vector(np.unique(a), a_idf, 0)
        if b_rows is not None:
            bi, bv = orc.sparse_vector(np.unique(b_rows[i]), b_idf, len(a_idf))
            ind, val = np.concatenate([ind, bi]), np.concatenate([val, bv])
        out.append((ind.astype(np.uint32), val.astype(np.float32)))
    return out


def build_data(rng, kind):
    d = types.SimpleNamespace()
    if kind == "users":
        d.a_idf, d.b_idf = make_idf(rng, N_FEAT), None
        d.a_rows, d.b_rows = make_rows(rng, N, N_FEAT, LONG), None
    else:
        d.a_idf, d.b_idf = make_idf(rng, N_TAGS), make_idf(rng, N_FEAT)
        d.a_rows = make_rows(rng, N, N_TAGS)
        d.b_rows = make_rows(rng, N, N_FEAT, LONG)
    d.hidden = (rng.random(N) < 0.05).astype(np.uint8)
    d.cats = [list(rng.choice(4, int(rng.integers(0, 3)), replace=False)) for _ in range(N)]
    return d


def add_both(gb, orc, pair, d, ts, replace_dev=None, replace_host=None):
    """d's rows into the device-built collection, their expected vectors with vecdb_add into the host one; -> (slot_out, vectors)"""
    vecs = expected(orc, d.a_rows, d.a_idf, d.b_rows, d.b_idf)
    slot_out = pair.dev.add_idf_vectors(d.a_rows, d.a_idf, 0, d.b_rows, d.b_idf, len(d.a_idf), hidden=d.hidden, timestamp_ms=ts,
                                        categories=d.cats, replace=replace_dev)
    keep = [i for i, v in enumerate(vecs) if len(v[0])]
    first = pair.host.add(sparse=[vecs[i] for i in keep], hidden=d.hidden[keep], timestamps=np.full(len(keep), ts, np.int64),
                          categories=[d.cats[i] for i in keep], replace=None if replace_host is None else np.asarray(replace_host)[keep])
    want = np.full(len(vecs), -1, np.int64)
    want[keep] = first + np.arange(len(keep))
    assert slot_out.tolist() == want.tolist()
    return slot_out, vecs


def answers(gb, ctx, col, rng_seed, queries):
    """every search of the collection on a seeded workload over its current slots"""
    rng = np.random.default_rng(rng_seed)
    slots = col.count()[1]
    out = {}
    for k in (100, 129):
        s, sc, cnt = col.query(queries, (), k)
        out[f"query{k}"] = (s.tobytes(), sc.tobytes(), cnt.tobytes())
        s, sc, cnt = col.query(queries, (1,), k)
        out[f"query{k}_cat"] = (s.tobytes(), sc.tobytes(), cnt.tobytes())

    def pick(k):
        s = rng.integers(0, slots, k)
        s[rng.random(k) > 0.9] = -1
        return s

    nu = 150
    ctxs = [pick(int(rng.integers(1, 6))) for _ in range(nu)]
    exs = [np.unique(pick(int(rng.integers(0, 6)))) for _ in range(nu)]
    user_slots = pick(nu)
    fb = [rng.integers(0, slots, int(rng.integers(0, 5))) for _ in range(slots)]
    ok = (rng.random(slots) > 0.1).astype(np.uint8)

    def flat(rows):
        return [(a.tobytes(), b.tobytes()) for a, b in rows]

    out["item_to_item"] = flat(col.item_to_item(ctxs, exs, 20, categories=(0,))[0])
    out["user_to_user"] = flat(col.user_to_user(user_slots, fb, exs, 20, slots, ok)[0])
    out["session"] = flat(col.session_recommend(ctxs, exs, 20, 3, 25, item_ok=ok)[0])
    ident = np.arange(slots, dtype=np.int64)
    stages = [gb.ItemToItemStage(col, 15, ctxs, ident, ident.astype(np.int32), score_scale=0.5), gb.UserToUserStage(col, 15, user_slots, fb, ok)]
    out["recommend"] = flat(gb.recommend(ctx, [e[e >= 0] for e in exs], slots, np.ones(slots, np.uint8), stages)[0])
    return out


def assert_same(a, b):
    assert a.keys() == b.keys()
    for k in a:
        assert a[k] == b[k], k


@pytest.fixture(scope="module", params=KINDS)
def built(request, gb, orc, ctx):
    kind = request.param
    rng = np.random.default_rng(7 if kind == "users" else 8)
    pair = types.SimpleNamespace(kind=kind, dev=gb.VectorCollection(ctx, 0, gb.DISTANCE_DOT), host=gb.VectorCollection(ctx, 0, gb.DISTANCE_DOT))
    pair.d = build_data(rng, kind)
    pair.slot_out, pair.vecs = add_both(gb, orc, pair, pair.d, 1000)
    pair.queries = [v for v in pair.vecs[::97] if len(v[0])][:60]
    yield pair
    pair.dev.close()
    pair.host.close()


def test_contents(built):
    d, dev = built.d, built.dev
    empty = [i for i, v in enumerate(built.vecs) if len(v[0]) == 0]
    assert len(empty) > N // 20
    assert (built.slot_out[empty] == -1).all()
    added = built.slot_out[built.slot_out >= 0]
    assert added.tolist() == list(range(added.size))
    assert dev.count() == (added.size, added.size)
    for i, s in enumerate(built.slot_out):
        if s < 0:
            continue
        ind, val = dev.get_sparse(int(s), cap=len(built.vecs[i][0]) + 1)
        assert ind.tobytes() == built.vecs[i][0].tobytes() and val.tobytes() == built.vecs[i][1].tobytes(), i
    # the data hit every case: repeats, skipped ids, rows that became empty, a row of more than 100K ids over several tiles
    rows = d.a_rows if d.b_rows is None else d.b_rows
    assert any(len(np.unique(r)) < len(r) for r in rows) and any((r < 0).any() for r in rows)
    assert any(len(r) and len(built.vecs[i][0]) == 0 for i, r in enumerate(rows))
    assert len(rows[LONG]) > 100_000 and built.slot_out[LONG] >= 0 and added.size > 2 * TILE


def test_same_answers_as_host_add(gb, ctx, built):
    assert built.dev.count() == built.host.count()
    assert_same(answers(gb, ctx, built.dev, 1, built.queries), answers(gb, ctx, built.host, 1, built.queries))


def test_rewrite_cycle(gb, orc, ctx, built):
    """the master's hourly rewrite: every row again with replace, then delete_before and compact"""
    rng = np.random.default_rng(11)
    d2 = build_data(rng, built.kind)
    rep = built.slot_out.copy()   # the slot holding row i's id, -1 when it has none
    add_both(gb, orc, built, d2, 2000, replace_dev=rep, replace_host=rep)
    assert built.dev.count() == built.host.count()
    assert_same(answers(gb, ctx, built.dev, 2, built.queries), answers(gb, ctx, built.host, 2, built.queries))
    a, b = built.dev.delete_before(2000), built.host.delete_before(2000)
    assert a.tolist() == b.tolist()
    sa, sb = built.dev.compact()[0], built.host.compact()[0]
    assert sa.tolist() == sb.tolist()
    assert_same(answers(gb, ctx, built.dev, 3, built.queries), answers(gb, ctx, built.host, 3, built.queries))
    # a host add after a device build
    extra = [v for v in built.vecs[::5] if len(v[0])]
    for col in (built.dev, built.host):
        col.add(sparse=extra, timestamps=np.full(len(extra), 3000, np.int64))
    assert_same(answers(gb, ctx, built.dev, 4, built.queries), answers(gb, ctx, built.host, 4, built.queries))


def test_device_build_after_unsearched_host_add(gb, orc, ctx):
    rng = np.random.default_rng(21)
    pair = types.SimpleNamespace(dev=gb.VectorCollection(ctx, 0, gb.DISTANCE_DOT), host=gb.VectorCollection(ctx, 0, gb.DISTANCE_DOT))
    try:
        d = build_data(rng, "users")
        first = [v for v in expected(orc, d.a_rows[:3000], d.a_idf) if len(v[0])]
        for col in (pair.dev, pair.host):
            col.add(sparse=first, timestamps=np.full(len(first), 5, np.int64))   # never searched before the device build
        d.a_rows, d.hidden, d.cats = d.a_rows[3000:], d.hidden[3000:], d.cats[3000:]
        _, vecs = add_both(gb, orc, pair, d, 6)
        queries = [v for v in vecs[::131] if len(v[0])][:40]
        assert_same(answers(gb, ctx, pair.dev, 5, queries), answers(gb, ctx, pair.host, 5, queries))
    finally:
        pair.dev.close()
        pair.host.close()


def snapshot(col, queries):
    live, slots = col.count()
    return (live, slots, [col.get_sparse(s, cap=1 << 18) for s in range(0, slots, 53)], col.query(queries, (), 100))


def same_snapshot(a, b):
    assert a[:2] == b[:2]
    assert all(x[0].tobytes() == y[0].tobytes() and x[1].tobytes() == y[1].tobytes() for x, y in zip(a[2], b[2]))
    assert all(x.tobytes() == y.tobytes() for x, y in zip(a[3], b[3]))


def test_errors_leave_the_collection_unchanged(gb, ctx):
    from gorse_b200 import _lib

    rng = np.random.default_rng(31)
    col = gb.VectorCollection(ctx, 0, gb.DISTANCE_DOT)
    try:
        idf = make_idf(rng, 500)
        idf[idf <= 0] = 1.0
        rows = make_rows(rng, 3000, 500)
        col.add_idf_vectors(rows, idf, timestamp_ms=1)
        queries = [(np.array([1, 2, 3], np.uint32), np.ones(3, np.float32)), (np.array([7, 40], np.uint32), np.ones(2, np.float32))]
        before = snapshot(col, queries)

        def refused(*args, **kw):
            with pytest.raises(gb.GorseB200Error) as ei:
                col.add_idf_vectors(*args, **kw)
            assert ei.value.status == _lib.ERR_ARG
            same_snapshot(before, snapshot(col, queries))
            return ei.value.message

        nan = idf.copy()
        nan[3] = np.nan
        assert "NaN" in refused([[5, 4], [3, 9, 3]], nan)
        nan_unused = idf.copy()
        nan_unused[499] = np.nan   # a NaN idf no row uses is not an error (and the rows are added)
        assert "too large" in refused([[1, 2], [3]], idf, a_offset=0x7fffffff - 2)
        assert "ascending" in refused([[1, 2], [4]], idf, 0, [[0], [7]], idf, 2)   # B at offset 2 collides with A
        assert "ascending" in refused([[10], [4]], idf, 0, [[0], [7]], idf, 5)     # B below A
        # decreasing offsets, through the C entry
        off, ids, slot = np.array([0, 3, 2], np.int64), np.array([1, 2, 3], np.int32), np.zeros(2, np.int64)
        st = _lib.lib.gorse_b200_vecdb_add_idf_vectors(col.h, 2, _lib.ptr(off), _lib.ptr(ids), _lib.ptr(idf), idf.size, 0, None, None, None, 0, 0,
                                                       None, 0, None, None, None, _lib.ptr(slot))
        assert st == _lib.ERR_ARG
        same_snapshot(before, snapshot(col, queries))
        got = col.add_idf_vectors([[1, 2], [600]], nan_unused, timestamp_ms=2)
        assert got.tolist() == [before[1], -1]
    finally:
        col.close()
    with gb.VectorCollection(ctx, 8, gb.DISTANCE_DOT) as dense:
        with pytest.raises(gb.GorseB200Error) as ei:
            dense.add_idf_vectors([[1, 2]], np.ones(4, np.float32))
        assert ei.value.status == _lib.ERR_ARG
        assert dense.count() == (0, 0)
