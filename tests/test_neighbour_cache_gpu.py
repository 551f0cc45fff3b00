"""The neighbour cache of a collection (gorse_b200_vecdb_neighbour_cache): every neighbour entry answers with the cache on
exactly what it answers with it off.  Each check gives the same writes to two collections, one with the cache and one
without, and requires the same slots, float64 score bits and counts from item_to_item, session_recommend, user_to_user and
gorse_b200_recommend's item-to-item and user-to-user stages -- on dense Dot and Euclidean collections in bf16 and fp32 and on
sparse Dot collections, over tie-heavy grid data (as in test_ties_gpu.py), along call sequences that go from all misses to
all hits, across stage-B chunks, across the tensor-core sweep / exact-scan boundary, past a full pool, and after each change
of the collection, where the data makes the stale answer differ from the fresh one."""
import io

import numpy as np
import pytest

gpu = pytest.mark.gpu

GRID = np.array([-7, -5, -3, -1, 1, 3, 5, 7], np.float32) / 4
N, D, K = 2000, 16, 10   # stored vectors, dense dimension, neighbours per row
KINDS = ("dot-bf16", "dot-fp32", "euclid-bf16", "euclid-fp32", "sparse")


@pytest.fixture(scope="module")
def ctx(gb):
    c = gb.Context(0)
    yield c
    c.close()


# ---- data -------------------------------------------------------------------------------------------------------------------
def dense_rows(rng, n, d=D):
    return GRID[rng.integers(0, GRID.size, (n, d))]


def sparse_rows(rng, n):
    """3 .. 8 indices of 64 with values 1 or 2: exact dots, many ties"""
    out = []
    for _ in range(n):
        ind = np.sort(rng.choice(64, int(rng.integers(3, 9)), replace=False)).astype(np.uint32)
        out.append((ind, rng.integers(1, 3, ind.size).astype(np.float32)))
    return out


class Twins:
    """a collection with the cache (`on`) and one without (`off`), given the same writes"""

    def __init__(self, gb, ctx, kind, n=N, seed=0, cache_rows=1 << 20, categories=None, timestamps=None):
        self.gb, self.kind = gb, kind
        self.rng = np.random.default_rng(seed)
        self.sparse = kind == "sparse"
        dist = gb.DISTANCE_EUCLIDEAN if kind.startswith("euclid") else gb.DISTANCE_DOT
        dim = 0 if self.sparse else D
        self.on, self.off = gb.VectorCollection(ctx, dim, dist), gb.VectorCollection(ctx, dim, dist)
        if self.sparse:
            self.data = sparse_rows(self.rng, n)
            self.add(sparse=self.data, categories=categories, timestamps=timestamps)
        else:
            self.data = dense_rows(self.rng, n)
            if kind.endswith("fp32"):   # one value that is not bf16-exact: the collection is stored in fp32
                self.data[-1, 0] = 0.1
            self.add(values=self.data, categories=categories, timestamps=timestamps)
            assert self.on.storage()[0] == (4 if kind.endswith("fp32") else 2)
        self.on.neighbour_cache(K, cache_rows)

    def add(self, **kw):
        a, b = self.on.add(**kw), self.off.add(**kw)
        assert a == b
        return a

    def both(self, name, *args, **kw):
        return getattr(self.on, name)(*args, **kw), getattr(self.off, name)(*args, **kw)

    def stats(self):
        return self.on.neighbour_cache_stats()

    def slots(self):
        return self.on.count()[1]

    def close(self):
        self.on.close()
        self.off.close()


def same_rows(a, b):
    assert len(a) == len(b)
    for u, ((s1, v1), (s2, v2)) in enumerate(zip(a, b)):
        assert np.array_equal(s1, s2), f"row {u}: slots {s1} != {s2}"
        assert np.array_equal(np.asarray(v1, np.float64).view(np.uint64), np.asarray(v2, np.float64).view(np.uint64)), f"row {u}: score bits"


def contexts(rng, users, pool, lo=1, hi=6):
    return [rng.choice(pool, int(rng.integers(lo, hi + 1))).astype(np.int64).tolist() for _ in range(users)]


def exclusions(rng, users, slots):
    return [np.unique(rng.integers(0, slots, int(rng.integers(0, 4)))).tolist() for _ in range(users)]


# ---- the entries on both collections ----------------------------------------------------------------------------------------
def item_to_item(t, ctxs, excl, n=K, categories=()):
    (a, sa), (b, sb) = t.both("item_to_item", ctxs, excl, n, categories=categories)
    same_rows(a, b)
    assert sa["context_items"] == sb["context_items"]
    return a, sa, sb


def session(t, ctxs, excl, n=K):
    ok = (np.arange(t.slots()) % 3 != 0).astype(np.uint8)
    (a, sa), (b, sb) = t.both("session_recommend", ctxs, excl, n, 2, n + 3, item_ok=ok)
    same_rows(a, b)
    return a, sa, sb


def user_to_user(t, users, n=K):
    S = t.slots()
    n_items = 300
    fb = [t.rng.integers(0, n_items, int(t.rng.integers(0, 5))).tolist() for _ in range(S)]
    ok = (np.arange(n_items) % 5 != 0).astype(np.uint8)
    excl = [np.unique(t.rng.integers(0, n_items, 2)).tolist() for _ in users]
    (a, sa), (b, sb) = t.both("user_to_user", users, fb, excl, n, n_items, item_ok=ok)
    same_rows(a, b)
    return a, sa, sb


def recommend(gb, ctx, t, ctxs, users, n=K):
    """gorse_b200_recommend with an item-to-item and a user-to-user stage on the collection (items = slots)"""
    S = t.slots()
    ident = np.arange(S, dtype=np.int64)
    fb = [t.rng.integers(0, S, int(t.rng.integers(0, 4))).tolist() for _ in range(S)]
    excl = exclusions(t.rng, len(users), S)
    live = np.ones(S, np.uint8)
    out = []
    for col in (t.on, t.off):
        stages = [gb.ItemToItemStage(col, n, ctxs, ident, ident.astype(np.int32)), gb.UserToUserStage(col, n, users, fb)]
        out.append(gb.recommend(ctx, excl, S, live, stages))
    same_rows(out[0][0], out[1][0])
    assert out[0][1]["table_rows"] == out[1][1]["table_rows"]
    return out


def distinct_rows(ctxs):
    return len({s for c in ctxs for s in c if s >= 0})


# ---- every entry, every storage kind, a call sequence -------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("kind", KINDS)
def test_every_entry_equals_the_uncached_twin(gb, ctx, kind):
    t = Twins(gb, ctx, kind, seed=KINDS.index(kind))
    try:
        rng = t.rng
        first = rng.permutation(N)[:400]
        ctxs = contexts(rng, 300, first)
        excl = exclusions(rng, 300, N)
        R = distinct_rows(ctxs)
        # the first call: every row is a miss
        _, sa, sb = item_to_item(t, ctxs, excl)
        st = t.stats()
        assert (st["n"], st["rows"], st["served"], st["computed"], st["emptied"]) == (K, R, 0, R, 0)
        assert sa["exact_rows"] == sb["exact_rows"]
        # the same call again: nothing computed, and no row is scanned
        _, sa, _ = item_to_item(t, ctxs, excl)
        st = t.stats()
        assert (st["served"], st["computed"], sa["exact_rows"]) == (R, R, 0)
        # a batch mixing held rows and new ones
        mixed = contexts(rng, 300, np.concatenate([first[:200], rng.permutation(N)[:300]]))
        new = len({s for c in mixed for s in c} - {s for c in ctxs for s in c})
        assert new > 0
        item_to_item(t, mixed, exclusions(rng, 300, N))
        st2 = t.stats()
        assert st2["computed"] == R + new and st2["served"] == R + distinct_rows(mixed) - new
        # the other entries on the same cache
        session(t, mixed, exclusions(rng, 300, N))
        users = rng.integers(-1, N, 500)
        user_to_user(t, users)
        rctx = mixed + mixed[:200]   # one context list per user of the call
        recommend(gb, ctx, t, rctx, users)
        st3 = t.stats()
        assert st3["computed"] == st3["rows"] and st3["emptied"] == 0   # the pool has room for every row: each is computed once
        # everything again: all hits
        before = t.stats()["computed"]
        session(t, mixed, exclusions(rng, 300, N))
        user_to_user(t, users)
        recommend(gb, ctx, t, rctx, users)
        assert t.stats()["computed"] == before
    finally:
        t.close()


@gpu
def test_more_than_one_stage_b_chunk(gb, ctx):
    """more users than one chunk of stage B (sm_count * 1024), cold and then warm"""
    t = Twins(gb, ctx, "dot-bf16", seed=11)
    try:
        rng = t.rng
        users = 140_000
        ctxs = contexts(rng, users, np.arange(N), 1, 2)
        excl = [[] for _ in range(users)]
        item_to_item(t, ctxs, excl)
        computed = t.stats()["computed"]
        item_to_item(t, ctxs, excl)
        assert t.stats()["computed"] == computed
    finally:
        t.close()


@gpu
@pytest.mark.parametrize("exact", [False, True])
def test_rows_from_the_sweep_serve_a_call_the_exact_scan_answers(gb, ctx, monkeypatch, exact):
    """a 33,000-vector collection: the first call's rows go through the tensor-core sweep (>= 64 rows), the second call has
    fewer than 64 misses, which the exact kernel answers, while the twin computes every row of it in the sweep"""
    if exact:
        monkeypatch.setenv("GORSE_B200_TOPK_EXACT", "1")
    t = Twins(gb, ctx, "dot-bf16", n=33_000, seed=21)
    try:
        rng = t.rng
        pool = rng.permutation(33_000)
        first = [[int(s)] for s in pool[:200]]
        _, sa, sb = item_to_item(t, first, [[] for _ in first])
        if exact:
            assert sa["exact_rows"] == 200
        else:
            assert sa["exact_rows"] < 200, "the sweep answered none of the first call's rows"
        second = [[int(s)] for s in pool[:220]]   # 20 misses
        _, sa, sb = item_to_item(t, second, [[] for _ in second])
        assert t.stats()["computed"] == 220
        assert sa["exact_rows"] == 20
        if not exact:
            assert sb["exact_rows"] < 220
    finally:
        t.close()


# ---- what does not use the cache, and a pool that fills ---------------------------------------------------------------------
@gpu
def test_category_filter_and_other_n_bypass_the_cache(gb, ctx):
    cats = [[int(c) for c in np.nonzero(np.random.default_rng(s).integers(0, 2, 3))[0]] for s in range(N)]
    t = Twins(gb, ctx, "euclid-bf16", seed=31, categories=cats)
    try:
        ctxs = contexts(t.rng, 200, np.arange(N))
        excl = exclusions(t.rng, 200, N)
        item_to_item(t, ctxs, excl)
        st = t.stats()
        item_to_item(t, ctxs, excl, categories=(1,))
        item_to_item(t, ctxs, excl, n=K - 3)
        session(t, ctxs, excl, n=K + 2)
        assert t.stats() == st
    finally:
        t.close()


@gpu
def test_a_pool_smaller_than_the_rows(gb, ctx):
    t = Twins(gb, ctx, "sparse", seed=41, cache_rows=50)
    try:
        ctxs = contexts(t.rng, 300, np.arange(N))
        excl = exclusions(t.rng, 300, N)
        R = distinct_rows(ctxs)
        assert R > 50
        item_to_item(t, ctxs, excl)
        st = t.stats()
        assert (st["capacity"], st["rows"], st["computed"], st["served"]) == (50, 50, R, 0)
        item_to_item(t, ctxs, excl)
        st = t.stats()
        assert (st["rows"], st["computed"], st["served"]) == (50, 2 * R - 50, 50)
    finally:
        t.close()


@gpu
def test_sizing_accounting_and_turning_off(gb, ctx):
    from gorse_b200 import _lib

    t = Twins(gb, ctx, "dot-bf16", seed=51, cache_rows=0)
    try:
        ctxs = contexts(t.rng, 200, np.arange(N))
        excl = exclusions(t.rng, 200, N)
        item_to_item(t, ctxs, excl)   # the work buffers of this call exist before the cache does
        base, store = gb.device_bytes(), t.on.storage()[1]
        assert t.stats() == dict(n=0, capacity=0, rows=0, device_bytes=0, served=0, computed=0, emptied=0)
        t.on.neighbour_cache(K, 1000)
        assert t.stats()["device_bytes"] == 1000 * (8 * K + 4)
        item_to_item(t, ctxs, excl)
        st = t.stats()
        assert t.on.storage()[1] == store + st["device_bytes"] and gb.device_bytes() == base + st["device_bytes"]
        t.on.neighbour_cache(K, 1000)   # the same size again keeps the rows
        assert t.stats() == st
        t.on.neighbour_cache(K, 999)    # another size drops them
        assert t.stats()["rows"] == 0 and t.stats()["capacity"] == 999
        t.on.neighbour_cache(K, 0)
        assert gb.device_bytes() == base and t.on.storage()[1] == store
        item_to_item(t, ctxs, excl)
        assert t.stats()["computed"] == 0
        with pytest.raises(gb.GorseB200Error):
            t.on.neighbour_cache(1025, 10)
    finally:
        t.close()
    with gb.VectorCollection(ctx, 8, gb.DISTANCE_COSINE) as c:
        assert _lib.lib.gorse_b200_vecdb_neighbour_cache(c.h, K, 10) == _lib.ERR_UNSUPPORTED
    with gb.VectorCollection(ctx, 0, gb.DISTANCE_DOT) as c:
        assert _lib.lib.gorse_b200_vecdb_neighbour_cache(c.h, 129, 10) == _lib.ERR_UNSUPPORTED
        assert _lib.lib.gorse_b200_vecdb_neighbour_cache(c.h, 128, 10) == _lib.OK


# ---- every change of the collection empties the cache -----------------------------------------------------------------------
def differs(a, b):
    return len(a) != len(b) or any(not np.array_equal(x[0], y[0]) or not np.array_equal(x[1], y[1]) for x, y in zip(a, b))


def strongest(t, s):
    """a dense vector that scores above every grid row against row s: itself (Euclidean) or 7/4 sign(x) (Dot)"""
    x = t.data[s]
    return x.copy() if t.kind.startswith("euclid") else (np.where(x > 0, 1.75, -1.75)).astype(np.float32)


MUTATORS = ("add", "upsert", "hidden", "delete_before", "compact", "promotion", "add_idf_vectors", "add_item_factors")


@gpu
@pytest.mark.parametrize("mutator", MUTATORS)
def test_a_change_of_the_collection_empties_the_cache(gb, ctx, mutator):
    from gorse_b200 import _lib, synth

    kind = "sparse" if mutator == "add_idf_vectors" else "euclid-bf16" if mutator == "hidden" else "dot-bf16"
    ts = np.full(N, 1000, np.int64)
    t = Twins(gb, ctx, kind, seed=61 + MUTATORS.index(mutator), timestamps=ts)
    try:
        rng = t.rng
        ctxs = contexts(rng, 100, rng.permutation(N)[:150])
        excl = [[] for _ in ctxs]
        stale, _, _ = item_to_item(t, ctxs, excl)
        assert t.stats()["rows"] > 0
        top = int(stale[0][0][0])   # the best neighbour sum of user 0
        if mutator == "add":
            t.add(values=np.stack([strongest(t, s) for s in ctxs[0]]))
        elif mutator == "upsert":   # the id of `top` gets the opposite vector
            t.add(values=-t.data[top][None], replace=np.array([top]))
        elif mutator == "hidden":
            t.add(values=t.data[top][None], hidden=np.array([1], np.uint8), replace=np.array([top]))
        elif mutator in ("delete_before", "compact"):
            # `top` again with an old timestamp; each change below follows a call that refilled the cache
            t.add(values=t.data[top][None], timestamps=np.array([0]), replace=np.array([top]))
            stale = item_to_item(t, ctxs, excl)[0]
            a, b = t.both("delete_before", 1)
            assert a.size == b.size == 1
            if mutator == "compact":
                stale = item_to_item(t, ctxs, excl)[0]
                (m1, _, _), (m2, _, _) = t.both("compact")
                assert np.array_equal(m1, m2)
                ctxs = [[int(m1[s]) for s in c] for c in ctxs]
        elif mutator == "promotion":
            v = strongest(t, ctxs[0][0]) * np.float32(1.0009765625 + 2.0 ** -12)   # not bf16-exact
            t.add(values=v[None])
            assert t.on.storage()[0] == 4
        elif mutator == "add_idf_vectors":
            ind = t.data[ctxs[0][0]][0]
            idf = np.full(64, 100.0, np.float32)
            a, b = t.both("add_idf_vectors", [ind.astype(np.int32).tolist()], idf)
            assert np.array_equal(a, b) and a[0] >= 0
        elif mutator == "add_item_factors":
            U, I = 50, 40
            off, items = synth.make_feedback(U, I, 400, seed=5)
            with gb.CFModel(ctx, U, I, D, off, items) as m:
                Q = np.tile(strongest(t, ctxs[0][0]), (I, 1))   # every item with feedback becomes a vector
                m.set_factors(dense_rows(rng, U), Q)
                for col in (t.on, t.off):
                    slot = np.zeros(I, np.int64)
                    gb.check(_lib.lib.gorse_b200_vecdb_add_item_factors(col.h, m.h, None, 0, None, None, gb.ptr(slot)))
        emptied = t.stats()["emptied"]
        fresh, _, _ = item_to_item(t, ctxs, excl)
        assert differs(fresh, stale), "the data does not tell a stale cache from a fresh one"
        assert t.stats()["emptied"] == emptied + 1
    finally:
        t.close()


@gpu
@pytest.mark.parametrize("kind", ("dot-bf16", "sparse"))
def test_snapshots_do_not_contain_the_cache(gb, ctx, kind):
    t = Twins(gb, ctx, kind, seed=71)
    try:
        ctxs = contexts(t.rng, 200, np.arange(N))
        item_to_item(t, ctxs, [[] for _ in ctxs])
        assert t.stats()["rows"] > 0
        a, b = io.BytesIO(), io.BytesIO()
        t.on.save(a)
        t.off.save(b)
        assert a.getvalue() == b.getvalue()
    finally:
        t.close()
