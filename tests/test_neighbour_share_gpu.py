"""Neighbour caches shared between processes: gorse_b200_vecdb_neighbour_cache_fill, _save and _load.

After a fill every neighbour entry answers from the cache alone, with the same slots, float64 score bits and counts as a twin
collection without a cache -- dense Dot and Euclidean in bf16 and fp32 and sparse, on both sides of the tensor-core routing.
A filled cache saved beside its collection's snapshot loads into the collection restored on a fresh context (also from a
collection with deleted slots) and serves every row.  Streams do not depend on how the rows were computed, a bf16 collection
and its fp32 twin give the same stream, and every bad stream or changed collection is refused with the cache untouched."""
import io
import struct

import numpy as np
import pytest

gpu = pytest.mark.gpu

GRID = np.array([-7, -5, -3, -1, 1, 3, 5, 7], np.float32) / 4
N, D, K = 2000, 16, 10
BIG = 33_000   # N >= 32,768: calls of >= 64 rows go through the tensor-core sweep
KINDS = ("dot-bf16", "dot-fp32", "euclid-bf16", "euclid-fp32", "sparse")
HEADER = 48


@pytest.fixture(scope="module")
def ctx(gb):
    c = gb.Context(0)
    yield c
    c.close()


def dense_rows(rng, n, d=D):
    return GRID[rng.integers(0, GRID.size, (n, d))]


def sparse_rows(rng, n):
    out = []
    for _ in range(n):
        ind = np.sort(rng.choice(64, int(rng.integers(3, 9)), replace=False)).astype(np.uint32)
        out.append((ind, rng.integers(1, 3, ind.size).astype(np.float32)))
    return out


def make(gb, ctx, kind, data, **kw):
    dist = gb.DISTANCE_EUCLIDEAN if kind.startswith("euclid") else gb.DISTANCE_DOT
    col = gb.VectorCollection(ctx, 0 if kind == "sparse" else D, dist)
    if kind == "sparse":
        col.add(sparse=data, **kw)
    else:
        col.add(values=data, **kw)
    return col


def data_of(kind, n, seed):
    rng = np.random.default_rng(seed)
    if kind == "sparse":
        return sparse_rows(rng, n)
    x = dense_rows(rng, n)
    if kind.endswith("fp32"):   # one value that is not bf16-exact: the collection is stored in fp32
        x[-1, 0] = 0.1
    return x


def same_rows(a, b, slot_map=None):
    assert len(a) == len(b)
    for u, ((s1, v1), (s2, v2)) in enumerate(zip(a, b)):
        s1 = np.asarray(s1) if slot_map is None else slot_map[np.asarray(s1, np.int64)]
        assert np.array_equal(s1, s2), f"row {u}: slots {s1} != {s2}"
        assert np.array_equal(np.asarray(v1, np.float64).view(np.uint64), np.asarray(v2, np.float64).view(np.uint64)), f"row {u}: score bits"


def contexts(rng, users, pool, lo=1, hi=6):
    return [rng.choice(pool, int(rng.integers(lo, hi + 1))).astype(np.int64).tolist() for _ in range(users)]


def exclusions(rng, users, slots):
    return [np.unique(rng.integers(0, slots, int(rng.integers(0, 4)))).tolist() for _ in range(users)]


def stream(col):
    b = io.BytesIO()
    n = col.save_neighbour_cache(b)
    assert n == len(b.getvalue())
    return b.getvalue()


def held_ranks(s):
    """the row ranks of a stream, parsed by the documented format"""
    rows = struct.unpack_from("<q", s, 40)[0]
    at, out = HEADER, []
    for _ in range(rows):
        r, c = struct.unpack_from("<ii", s, at)
        out.append(r)
        at += 8 + 8 * c
    assert at == len(s)
    return out


def all_entries(gb, ctx, on, off, rng, live_slots, n_users=300):
    """item-to-item, session, user-to-user and both recommend stages on `on` and `off`: the same answers"""
    S = on.count()[1]
    ctxs = contexts(rng, n_users, live_slots)
    excl = exclusions(rng, n_users, S)
    (a, _), (b, _) = on.item_to_item(ctxs, excl, K), off.item_to_item(ctxs, excl, K)
    same_rows(a, b)
    ok = (np.arange(S) % 3 != 0).astype(np.uint8)
    (a, _), (b, _) = (c.session_recommend(ctxs, excl, K, 2, K + 3, item_ok=ok) for c in (on, off))
    same_rows(a, b)
    n_items = 300
    fb = [rng.integers(0, n_items, int(rng.integers(0, 5))).tolist() for _ in range(S)]
    users = rng.choice(np.concatenate([live_slots, [-1]]), n_users).astype(np.int64)
    iok = (np.arange(n_items) % 5 != 0).astype(np.uint8)
    uex = [np.unique(rng.integers(0, n_items, 2)).tolist() for _ in users]
    (a, _), (b, _) = (c.user_to_user(users, fb, uex, K, n_items, item_ok=iok) for c in (on, off))
    same_rows(a, b)
    ident = np.arange(S, dtype=np.int64)
    live = np.ones(S, np.uint8)
    out = []
    for col in (on, off):
        stages = [gb.ItemToItemStage(col, K, ctxs, ident, ident.astype(np.int32)), gb.UserToUserStage(col, K, users, fb)]
        out.append(gb.recommend(ctx, excl, S, live, stages))
    same_rows(out[0][0], out[1][0])


# ---- answers after a fill -----------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("size", [N, BIG])
@pytest.mark.parametrize("kind", KINDS)
def test_every_entry_after_a_fill_is_served_from_the_cache(gb, ctx, kind, size):
    data = data_of(kind, size, KINDS.index(kind) + size)
    on, off = make(gb, ctx, kind, data), make(gb, ctx, kind, data)
    try:
        on.neighbour_cache(K, 1 << 20)
        st = on.neighbour_cache_fill()
        assert (st["computed"], st["rows"], st["left_out"]) == (size, size, 0) and st["device_us"] > 0
        assert on.neighbour_cache_fill()["computed"] == 0, "a second fill computes nothing"
        before = on.neighbour_cache_stats()
        assert (before["rows"], before["computed"], before["served"]) == (size, size, 0)
        rng = np.random.default_rng(size)
        all_entries(gb, ctx, on, off, rng, np.arange(size))
        after = on.neighbour_cache_stats()
        assert after["computed"] == size and after["served"] > 0, "every context row is served, none computed"
    finally:
        on.close()
        off.close()


@gpu
@pytest.mark.parametrize("kind", ("dot-bf16", "sparse"))
def test_fill_with_deleted_and_hidden_slots(gb, ctx, kind):
    data = data_of(kind, N, 7)
    ts = np.where(np.arange(N) % 7 == 0, 0, 1000).astype(np.int64)
    hidden = (np.arange(N) % 5 == 0).astype(np.uint8)
    on, off = (make(gb, ctx, kind, data, timestamps=ts, hidden=hidden) for _ in range(2))
    try:
        for c in (on, off):
            c.delete_before(1)
        live = np.nonzero(ts > 0)[0]
        on.neighbour_cache(K, 1 << 20)
        st = on.neighbour_cache_fill()
        assert (st["computed"], st["rows"], st["left_out"]) == (live.size, live.size, 0), "hidden vectors are filled, deleted ones not"
        all_entries(gb, ctx, on, off, np.random.default_rng(1), live)
        assert on.neighbour_cache_stats()["computed"] == live.size
    finally:
        on.close()
        off.close()


@gpu
def test_a_pool_smaller_than_the_live_count(gb, ctx):
    data = data_of("euclid-bf16", N, 8)
    on, off = make(gb, ctx, "euclid-bf16", data), make(gb, ctx, "euclid-bf16", data)
    try:
        on.neighbour_cache(K, 50)
        st = on.neighbour_cache_fill()
        assert (st["computed"], st["rows"], st["left_out"]) == (50, 50, N - 50)
        assert held_ranks(stream(on)) == list(range(50)), "the lowest slots are held"
        assert on.neighbour_cache_fill()["computed"] == 0
        all_entries(gb, ctx, on, off, np.random.default_rng(2), np.arange(N))
    finally:
        on.close()
        off.close()


@gpu
def test_fill_needs_the_cache_and_refuses_cosine(gb, ctx):
    from gorse_b200 import _lib

    with gb.VectorCollection(ctx, D, gb.DISTANCE_DOT) as c:
        c.add(values=dense_rows(np.random.default_rng(0), 100))
        assert _lib.lib.gorse_b200_vecdb_neighbour_cache_fill(c.h, None) == _lib.ERR_STATE
        assert _lib.lib.gorse_b200_vecdb_neighbour_cache_save(c.h, _lib.WRITE_FN(lambda u, b, n: 0), None, None) == _lib.ERR_STATE
    with gb.VectorCollection(ctx, D, gb.DISTANCE_COSINE) as c:
        c.add(values=dense_rows(np.random.default_rng(0), 100))
        assert _lib.lib.gorse_b200_vecdb_neighbour_cache_fill(c.h, None) == _lib.ERR_UNSUPPORTED


# ---- round trip -----------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("kind, dead", [("dot-bf16", False), ("euclid-fp32", True), ("sparse", True), ("dot-bf16", True)])
def test_round_trip_on_a_fresh_context(gb, ctx, kind, dead):
    size = BIG if kind == "dot-bf16" and dead else N
    data = data_of(kind, size, 9)
    ts = np.where((np.arange(size) % 9 == 0) & dead, 0, 1000).astype(np.int64)
    src = make(gb, ctx, kind, data, timestamps=ts)
    try:
        src.delete_before(1)
        src.neighbour_cache(K, 1 << 20)
        src.neighbour_cache_fill()
        nbr = stream(src)
        snap = io.BytesIO()
        new_slot = src.save(snap)
        live = np.nonzero(new_slot >= 0)[0]
        with gb.Context(0) as ctx2:
            dst = gb.VectorCollection.load(ctx2, io.BytesIO(snap.getvalue()))
            try:
                dst.neighbour_cache(K, 1 << 20)
                st = dst.load_neighbour_cache(io.BytesIO(nbr))
                assert st == dict(loaded=live.size, dropped=0, bytes=len(nbr))
                assert stream(dst) == nbr
                rng = np.random.default_rng(3)
                ctxs = contexts(rng, 300, live)
                excl = exclusions(rng, 300, size)
                excl = [[s for s in e if new_slot[s] >= 0] for e in excl]
                m = lambda rows: [[int(new_slot[s]) for s in r] for r in rows]
                (a, _), (b, _) = src.item_to_item(ctxs, excl, K), dst.item_to_item(m(ctxs), m(excl), K)
                same_rows(a, b, new_slot)
                ok = (np.arange(size) % 3 != 0).astype(np.uint8)
                (a, _) = src.session_recommend(ctxs, excl, K, 2, K + 3, item_ok=ok)
                (b, _) = dst.session_recommend(m(ctxs), m(excl), K, 2, K + 3, item_ok=ok[live])
                same_rows(a, b, new_slot)
                st = dst.neighbour_cache_stats()
                assert st["computed"] == 0 and st["served"] > 0, "every row came from the stream"
            finally:
                dst.close()
    finally:
        src.close()


# ---- stream determinism -------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("kind", ("dot-fp32", "sparse"))
def test_lazy_and_filled_caches_save_the_same_stream(gb, ctx, kind):
    data = data_of(kind, N, 10)
    lazy, filled = make(gb, ctx, kind, data), make(gb, ctx, kind, data)
    try:
        for c in (lazy, filled):
            c.neighbour_cache(K, 1 << 20)
        rng = np.random.default_rng(4)
        order = rng.permutation(N)
        for i in range(0, N, 500):   # every slot in a random order, over several calls
            lazy.item_to_item([[int(s)] for s in order[i:i + 500]], [[] for _ in order[i:i + 500]], K)
        filled.neighbour_cache_fill()
        assert lazy.neighbour_cache_stats()["rows"] == N
        assert stream(lazy) == stream(filled)
    finally:
        lazy.close()
        filled.close()


@gpu
def test_a_bf16_collection_and_its_fp32_twin_give_the_same_stream(gb, ctx):
    x = dense_rows(np.random.default_rng(11), N)
    ts = np.full(N + 1, 1000, np.int64)
    ts[-1] = 0
    a = make(gb, ctx, "dot-bf16", x)
    b = make(gb, ctx, "dot-fp32", np.vstack([x, np.full((1, D), 0.1, np.float32)]), timestamps=ts)
    try:
        b.delete_before(1)   # the value that made it fp32 is gone; the live vectors are a's
        assert a.storage()[0] == 2 and b.storage()[0] == 4
        for c in (a, b):
            c.neighbour_cache(K, 1 << 20)
            c.neighbour_cache_fill()
        sa, sb = stream(a), stream(b)
        assert sa[32:40] == sb[32:40], "fingerprints"
        assert sa == sb
    finally:
        a.close()
        b.close()


# ---- refusals -----------------------------------------------------------------------------------------------------------------
def refused(gb, col, data, status):
    """loading `data` fails with `status` and leaves the held rows and the stats as they were"""
    st, s = col.neighbour_cache_stats(), stream(col)
    with pytest.raises(gb.GorseB200Error) as ei:
        col.load_neighbour_cache(io.BytesIO(data))
    assert ei.value.status == status, ei.value.message
    assert col.neighbour_cache_stats() == st and stream(col) == s
    return ei.value.message


@pytest.fixture(scope="module")
def saved(gb, ctx):
    """a Dot collection with hidden and deleted slots, its cache filled, and its stream"""
    rng = np.random.default_rng(12)
    x = dense_rows(rng, N)
    ts = np.where(np.arange(N) % 11 == 0, 0, 1000).astype(np.int64)
    c = make(gb, ctx, "dot-bf16", x, timestamps=ts, hidden=(np.arange(N) % 13 == 0).astype(np.uint8))
    c.delete_before(1)
    c.neighbour_cache(K, 1 << 20)
    c.neighbour_cache_fill()
    yield c, stream(c), x, ts
    c.close()


@gpu
def test_refused_streams_leave_the_cache_as_it_was(gb, ctx, saved):
    from gorse_b200 import _lib

    col, s, _, _ = saved
    live = struct.unpack_from("<q", s, 24)[0]
    refused(gb, col, b"GB200NBX" + s[8:], _lib.ERR_ARG)
    refused(gb, col, s[:8] + struct.pack("<I", 2) + s[12:], _lib.ERR_ARG)
    # truncation at every section boundary (each header field, each of the first rows' fields) and at 40 seeded offsets
    cuts = [0, 8, 12, 16, 20, 24, 32, 40, 47]
    at = HEADER
    for _ in range(5):
        c = struct.unpack_from("<i", s, at + 4)[0]
        cuts += [at, at + 4, at + 8, at + 8 + 8 * c - 4]
        at += 8 + 8 * c
    cuts += np.random.default_rng(13).integers(1, len(s), 40).tolist() + [len(s) - 1]
    for k in cuts:
        assert "ends at byte" in refused(gb, col, s[:k], _lib.ERR_ARG)
    # a row rank out of range, repeated, descending; an entry count above n; an entry rank out of range
    b = bytearray(s)
    r1 = HEADER + 8 + 8 * struct.unpack_from("<i", s, HEADER + 4)[0]
    r2 = r1 + 8 + 8 * struct.unpack_from("<i", s, r1 + 4)[0]
    rank0 = struct.unpack_from("<i", s, HEADER)[0]
    for name, off, val in (("row rank", HEADER, live), ("row rank", HEADER, -1), ("row rank", r1, rank0), ("row rank", r2, rank0),
                           ("entry count", HEADER + 4, K + 1), ("entry rank", HEADER + 8, live), ("entry rank", HEADER + 8, -1)):
        bad = bytearray(b)
        struct.pack_into("<i", bad, off, val)
        assert name in refused(gb, col, bytes(bad), _lib.ERR_ARG)
    struct.pack_into("<q", b, 40, live + 1)
    refused(gb, col, bytes(b), _lib.ERR_ARG)


@gpu
def test_another_n_or_the_cache_off_is_a_state_error(gb, ctx, saved):
    from gorse_b200 import _lib

    _, s, x, ts = saved
    other = make(gb, ctx, "dot-bf16", x, timestamps=ts, hidden=(np.arange(N) % 13 == 0).astype(np.uint8))
    try:
        other.delete_before(1)
        with pytest.raises(gb.GorseB200Error) as ei:
            other.load_neighbour_cache(io.BytesIO(s))
        assert ei.value.status == _lib.ERR_STATE
        assert other.neighbour_cache_stats()["n"] == 0
        other.neighbour_cache(K + 1, 1 << 20)
        other.neighbour_cache_fill()
        refused(gb, other, s, _lib.ERR_STATE)
        other.neighbour_cache(K, 1 << 20)
        assert other.load_neighbour_cache(io.BytesIO(s))["loaded"] == N - len(range(0, N, 11))
        assert stream(other) == s
    finally:
        other.close()


MUTATORS = ("add", "upsert", "hidden", "delete", "delete_compact", "other_collection")


@gpu
@pytest.mark.parametrize("mutator", MUTATORS)
def test_a_stream_of_another_state_is_refused(gb, ctx, mutator):
    from gorse_b200 import _lib

    x = dense_rows(np.random.default_rng(14), N)
    ts = np.full(N, 1000, np.int64)
    ts[5] = 0
    col = make(gb, ctx, "dot-bf16", x, timestamps=ts)
    try:
        col.neighbour_cache(K, 1 << 20)
        col.neighbour_cache_fill()
        s = stream(col)
        if mutator == "add":
            col.add(values=x[:1])
        elif mutator == "upsert":
            col.add(values=-x[7:8], replace=np.array([7]))
        elif mutator == "hidden":
            col.add(values=x[7:8], hidden=np.array([1], np.uint8), replace=np.array([7]))
        elif mutator in ("delete", "delete_compact"):
            assert col.delete_before(1).size == 1
            if mutator == "delete_compact":
                col.compact()
        else:   # the same counts, other values
            col.close()
            col = make(gb, ctx, "dot-bf16", dense_rows(np.random.default_rng(15), N), timestamps=ts)
            col.neighbour_cache(K, 1 << 20)
        col.neighbour_cache_fill()
        msg = refused(gb, col, s, _lib.ERR_ARG)
        assert "fingerprint" in msg or "live count" in msg
    finally:
        col.close()


@gpu
def test_a_compaction_alone_keeps_the_stream_valid(gb, ctx, saved):
    """compaction renames slots but not live ranks: the stream of a collection with deleted slots loads after its compaction,
    as it loads into the collection its snapshot restores"""
    _, s, x, ts = saved
    col = make(gb, ctx, "dot-bf16", x, timestamps=ts, hidden=(np.arange(N) % 13 == 0).astype(np.uint8))
    try:
        col.delete_before(1)
        col.compact()
        col.neighbour_cache(K, 1 << 20)
        assert col.load_neighbour_cache(io.BytesIO(s))["dropped"] == 0
        assert stream(col) == s
        assert col.neighbour_cache_fill()["computed"] == 0
    finally:
        col.close()


class Failing(io.BytesIO):
    def __init__(self, data=b"", after=0):
        super().__init__(data)
        self.after = after

    def write(self, b):
        raise OSError("disk full")

    def readinto(self, b):
        if self.tell() >= self.after:
            raise OSError("read error")
        return super().readinto(memoryview(b)[:max(1, self.after - self.tell())])


@gpu
def test_write_and_read_failures_are_io_errors(gb, ctx, saved):
    from gorse_b200 import _lib

    col, s, _, _ = saved
    st = col.neighbour_cache_stats()
    with pytest.raises(gb.GorseB200Error) as ei:
        col.save_neighbour_cache(Failing())
    assert ei.value.status == _lib.ERR_IO
    assert col.neighbour_cache_stats() == st and stream(col) == s
    for after in (0, 20, HEADER + 100):
        with pytest.raises(gb.GorseB200Error) as ei:
            col.load_neighbour_cache(Failing(s, after))
        assert ei.value.status == _lib.ERR_IO
        assert col.neighbour_cache_stats() == st and stream(col) == s
