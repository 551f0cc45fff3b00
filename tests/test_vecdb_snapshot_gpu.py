"""Snapshots of a vector collection (gorse_b200_vecdb_save / gorse_b200_vecdb_load): a collection rebuilt from its stream
answers every entry exactly as the saved collection answers after compaction -- the same slots, score bits and tie order --
and lives on identically through later adds, deletes and compactions.  Also: streams read a few bytes at a time, a failing
write, malformed streams (each refused with no handle created), another device, and the NULL-argument errors, which need no
device."""
import ctypes as C
import io
import struct
import types

import numpy as np
import pytest

# name -> (dim, distance, ids written per cycle).  dot1024 writes 40 000 ids and keeps 34 799 live vectors: 143 MB of rows,
# more than two 64 MB staging buffers, and enough for the tensor-core sweep.
KINDS = {f"{d[:3].lower()}{dim}": (dim, d, 2500) for d in ("DOT", "EUCLIDEAN", "COSINE") for dim in (8, 64, 130, 1024)}
KINDS["dot1024"] = (1024, "DOT", 40000)
KINDS["sparse"] = (0, "DOT", 4000)
N_Q = 80
N_USERS = 96
HEADER = struct.Struct("<8sIiiIqqq")


def test_null_arguments_need_no_device(gb):
    from gorse_b200 import _lib

    lib = _lib.lib
    h, n = C.c_void_p(), C.c_int64(0)
    write = _lib.WRITE_FN(lambda user, buf, k: 0)
    read = _lib.READ_FN(lambda user, buf, k: 0)
    assert lib.gorse_b200_vecdb_save(None, write, None, None, C.byref(n)) == _lib.ERR_ARG
    assert b"NULL" in lib.gorse_b200_last_error()
    assert lib.gorse_b200_vecdb_save(None, None, None, None, None) == _lib.ERR_ARG
    assert lib.gorse_b200_vecdb_load(None, read, None, C.byref(h), C.byref(n)) == _lib.ERR_ARG
    assert b"NULL" in lib.gorse_b200_last_error() and not h.value
    assert lib.gorse_b200_vecdb_load(None, None, None, None, None) == _lib.ERR_ARG
    assert _lib.ERR_IO == -8


@pytest.fixture(scope="module")
def ctx(gb):
    c = gb.Context(0)
    yield c
    c.close()


class Twins:
    """one or two collections written alike, and the id <-> slot map a shim keeps (the same for both)"""

    def __init__(self, cols, dim, seed):
        self.cols, self.dim, self.rng = cols, dim, np.random.default_rng(seed)
        self.slot_of, self.id_of = {}, []

    def vectors(self, n):
        """tie-heavy: small integers (dense) or a few values on few features (sparse), and repeated rows"""
        rng = self.rng
        if self.dim > 0:
            v = rng.integers(-2, 3, (n, self.dim)).astype(np.float32)
            dup = rng.random(n) < 0.2
            v[dup] = v[rng.integers(0, n, int(dup.sum()))]
            v[np.all(v == 0, axis=1), 0] = 1.0   # no zero rows (Cosine)
            return dict(values=v)
        out = []
        for _ in range(n):
            k = int(rng.integers(1, 9))
            out.append((np.sort(rng.choice(64, k, replace=False)).astype(np.uint32), rng.choice([0.5, 1.0, 2.0], k).astype(np.float32)))
        return dict(sparse=out)

    def upsert(self, ids, ts, batch=10000):
        for a in range(0, len(ids), batch):
            part = [int(i) for i in ids[a:a + batch]]
            n = len(part)
            kw = dict(hidden=self.rng.random(n) < 0.05, timestamps=np.full(n, ts),
                      categories=[np.flatnonzero(self.rng.random(3) < 0.5).tolist() for _ in range(n)],
                      replace=[self.slot_of.get(i, -1) for i in part], **self.vectors(n))
            firsts = {c.add(**kw) for c in self.cols}
            assert len(firsts) == 1
            first = firsts.pop()
            for j, i in enumerate(part):
                self.slot_of[i] = first + j
            self.id_of += part

    def delete_before(self, ts):
        gone = [c.delete_before(ts) for c in self.cols]
        assert all(np.array_equal(g, gone[0]) for g in gone)
        for s in gone[0]:
            del self.slot_of[self.id_of[s]]

    def compact(self):
        maps = [c.compact()[0] for c in self.cols]
        assert all(np.array_equal(m, maps[0]) for m in maps)
        self.slot_of = {i: int(maps[0][s]) for i, s in self.slot_of.items()}
        self.id_of = [self.id_of[s] for s in np.flatnonzero(maps[0] >= 0)]
        return maps[0]


def history(gb, ctx, kind):
    dim, dist, m = KINDS[kind]
    t = Twins([gb.VectorCollection(ctx, dim, getattr(gb, "DISTANCE_" + dist))], dim, seed=5)
    t.upsert(np.arange(m), 1000)
    t.upsert(t.rng.choice(m, m // 2, replace=False), 2000)   # upserts tombstone the previous versions
    t.upsert(t.rng.choice(m, m * 7 // 10, replace=False), 3000)
    t.delete_before(2000)                                     # delete_before tombstones the rest of the first cycle
    t.upsert(np.arange(m, m + m // 50), 4000)
    t.n_ids = m + m // 50
    return t


def workload(t, seed):
    """slot-valued inputs over the (compacted, shared) slot space, -1 entries included"""
    rng = np.random.default_rng(seed)
    slots = t.cols[0].count()[1]
    live = np.array(sorted(t.slot_of.values()), np.int64)

    def pick(k):
        s = rng.choice(live, k)
        s[rng.random(k) > 0.93] = -1
        return s

    def ids(k):
        s = rng.integers(0, t.n_ids, k)
        s[rng.random(k) > 0.9] = -1
        return s

    w = types.SimpleNamespace()
    if t.dim > 0:
        w.q = rng.integers(-2, 3, (N_Q, t.dim)).astype(np.float32)
        # stored rows that have a copy as queries: exact ties near the top of their answers
        vals = t.cols[0].get(live)[0]
        _, first, cnt = np.unique(vals.astype(np.float64) @ rng.standard_normal(t.dim), return_index=True, return_counts=True)
        copied = first[cnt >= 2]
        w.q[:min(8, copied.size)] = vals[copied[:8]]
    else:
        w.q = t.vectors(N_Q)["sparse"]
    w.excl = [np.unique(pick(int(rng.integers(0, 12)))) for _ in range(N_Q)]
    w.ctx = [pick(int(rng.integers(1, 8))) for _ in range(N_USERS)]
    w.ex = [np.unique(pick(int(rng.integers(0, 10)))) for _ in range(N_USERS)]
    w.user_slots = pick(N_USERS)
    w.fb = [rng.integers(0, t.n_ids, int(rng.integers(0, 6))) for _ in range(slots)]
    w.ex_items = [np.unique(ids(int(rng.integers(0, 8)))) for _ in range(N_USERS)]
    w.item_ok = (rng.random(t.n_ids) > 0.1).astype(np.uint8)
    w.slot_ok = (rng.random(slots) > 0.1).astype(np.uint8)
    w.ctx_items = [ids(int(rng.integers(1, 8))) for _ in range(N_USERS)]
    w.item_live = (rng.random(t.n_ids) > 0.05).astype(np.uint8)
    w.soi = np.full(t.n_ids, -1, np.int64)
    w.ios = np.full(slots, -1, np.int32)
    for i, s in t.slot_of.items():
        w.soi[i], w.ios[s] = s, i
    return w


def rows_of(slots, scores, cnt):
    return [(slots[q, :c].copy(), scores[q, :c].copy()) for q, c in enumerate(cnt)]


def answers(gb, ctx, col, t, w):
    out = {}
    out["query"] = rows_of(*col.query(w.q, (), 20))
    out["query_categories"] = rows_of(*col.query(w.q, (1,), 20))
    if t.dim == 0:
        out["query_wide"] = rows_of(*col.query(w.q[:16], (), 200))   # the sparse path past 128 neighbours
    if t.dim > 0:
        out["query_excluding"] = col.query_excluding(w.q, w.excl, 15)[0]
    if col.distance == gb.DISTANCE_COSINE:   # the batched recommenders refuse Cosine
        return out
    out["item_to_item"] = col.item_to_item(w.ctx, w.ex, 10, categories=(0,))[0]
    out["session_recommend"] = col.session_recommend(w.ctx, w.ex, 10, 3, 15, item_ok=w.slot_ok)[0]
    out["user_to_user"] = col.user_to_user(w.user_slots, w.fb, w.ex_items, 10, t.n_ids, w.item_ok)[0]
    stages = [gb.ItemToItemStage(col, 10, w.ctx_items, w.soi, w.ios, score_scale=0.5), gb.UserToUserStage(col, 10, w.user_slots, w.fb, w.item_ok)]
    out["recommend"] = gb.recommend(ctx, w.ex_items, t.n_ids, w.item_live, stages)[0]
    return out


def stored(col, dim):
    live, slots = col.count()
    s = np.arange(slots, dtype=np.int64)
    vals, hid, ts, alive = col.get(s)
    sp = [col.get_sparse(int(i)) for i in s] if dim == 0 else None
    return (live, slots), vals, hid, ts, alive, sp


def assert_same(a, b):
    assert a.keys() == b.keys()
    for name in a:
        assert len(a[name]) == len(b[name]), name
        for (s0, v0), (s1, v1) in zip(a[name], b[name]):
            assert np.array_equal(s0, s1), name   # the same slots in the same (tie) order
            assert v0.tobytes() == v1.tobytes(), name   # the same score bits


def assert_same_stored(a, b):
    assert a[0] == b[0]
    for x, y in zip(a[1:5], b[1:5]):
        assert x.tobytes() == y.tobytes()
    if a[5] is not None:
        for (i0, x0), (i1, x1) in zip(a[5], b[5]):
            assert np.array_equal(i0, i1) and x0.tobytes() == x1.tobytes()


def ties(rows):
    """adjacent equal scores: entries whose order only the tie rule decides"""
    return sum(int(np.sum(v[1:] == v[:-1])) for _, v in rows)


@pytest.fixture(scope="module", params=list(KINDS))
def restored(request, gb, ctx):
    kind = request.param
    t = history(gb, ctx, kind)
    col = t.cols[0]
    r = types.SimpleNamespace(kind=kind, t=t, count_saved=col.count())
    before = stored(col, t.dim)
    buf = io.BytesIO()
    r.new_slot = col.save(buf)
    r.stream = buf.getvalue()
    assert_same_stored(before, stored(col, t.dim))   # save changes nothing
    assert np.array_equal(t.compact(), r.new_slot)   # save's map is compaction's
    src = io.BytesIO(r.stream + b"trailing bytes of the caller")
    r.loaded = gb.VectorCollection.load(ctx, src)
    r.read = src.tell()
    t.cols.append(r.loaded)
    yield r
    for c in t.cols:
        c.close()


@pytest.mark.gpu
def test_stream_layout(restored):
    r = restored
    dim, dist, _ = KINDS[r.kind]
    magic, version, d, distance, reserved, n, nnz, ncat = HEADER.unpack_from(r.stream)
    assert (magic, version, d, reserved) == (b"GB200VDB", 1, dim, 0)
    assert n == r.count_saved[0] and n < r.count_saved[1]
    values = 4 * n * dim if dim else 8 * (n + 1) + 8 * nnz
    assert len(r.stream) == 48 + 17 * n + 8 + 4 * ncat + values
    assert r.read == len(r.stream)   # exactly the stream is read
    assert r.loaded.dim == dim and r.loaded.distance == distance
    if r.kind == "dot1024":
        assert 4 * n * dim > 2 * (64 << 20)


@pytest.mark.gpu
def test_same_answers(gb, ctx, restored):
    r = restored
    t = r.t
    w = workload(t, 11)
    a, b = answers(gb, ctx, t.cols[0], t, w), answers(gb, ctx, r.loaded, t, w)
    assert_same(a, b)
    assert sum(len(s) for s, _ in a["query"]) > 0 and ties(a["query"]) > 0
    assert_same_stored(stored(t.cols[0], t.dim), stored(r.loaded, t.dim))
    assert r.loaded.count() == t.cols[0].count() == (r.count_saved[0], r.count_saved[0])


@pytest.mark.gpu
def test_same_life_afterwards(gb, ctx, restored):
    """the same adds, deletes and compaction on both, then every entry again"""
    r = restored
    t = r.t
    m = KINDS[r.kind][2]
    t.upsert(np.concatenate([t.rng.choice(t.n_ids, m // 5, replace=False), np.arange(t.n_ids, t.n_ids + 40)]), 5000)
    t.n_ids += 40
    t.delete_before(3000)
    w = workload(t, 12)
    assert_same(answers(gb, ctx, t.cols[0], t, w), answers(gb, ctx, r.loaded, t, w))
    t.compact()
    w = workload(t, 13)
    assert_same(answers(gb, ctx, t.cols[0], t, w), answers(gb, ctx, r.loaded, t, w))
    assert_same_stored(stored(t.cols[0], t.dim), stored(r.loaded, t.dim))


class Trickle(io.RawIOBase):
    """a source that hands out 1 .. 7 bytes per read"""

    def __init__(self, data, seed=0):
        self.data, self.pos, self.rng = data, 0, np.random.default_rng(seed)

    def readable(self):
        return True

    def readinto(self, b):
        k = min(len(b), int(self.rng.integers(1, 8)), len(self.data) - self.pos)
        b[:k] = self.data[self.pos:self.pos + k]
        self.pos += k
        return k


class FailingSink(io.RawIOBase):
    def __init__(self, after):
        self.after, self.n = after, 0

    def writable(self):
        return True

    def write(self, b):
        if self.n + len(b) > self.after:
            raise OSError("disk full")
        self.n += len(b)
        return len(b)


def small(gb, ctx, dim, n=60, seed=9):
    t = Twins([gb.VectorCollection(ctx, dim, gb.DISTANCE_DOT)], dim, seed)
    t.upsert(np.arange(n), 1000)
    t.upsert(np.arange(0, n, 4), 2000)
    t.n_ids = n
    return t


@pytest.mark.gpu
@pytest.mark.parametrize("dim", [0, 130])
def test_odd_read_boundaries(gb, ctx, dim):
    t = small(gb, ctx, dim)
    buf = io.BytesIO()
    t.cols[0].save(buf)
    loaded = gb.VectorCollection.load(ctx, Trickle(buf.getvalue()))
    t.compact()
    t.cols.append(loaded)
    assert_same_stored(stored(t.cols[0], dim), stored(loaded, dim))
    w = workload(t, 3)
    assert_same(answers(gb, ctx, t.cols[0], t, w), answers(gb, ctx, loaded, t, w))
    for c in t.cols:
        c.close()


@pytest.mark.gpu
@pytest.mark.parametrize("dim", [0, 64])
def test_write_failure_leaves_the_collection(gb, ctx, dim):
    t = small(gb, ctx, dim)
    col = t.cols[0]
    before = stored(col, dim)
    full = io.BytesIO()
    col.save(full)
    for after in (0, 47, 48 + 30, len(full.getvalue()) - 1):
        with pytest.raises(gb.GorseB200Error) as ei:
            col.save(FailingSink(after))
        assert ei.value.status == -8 and isinstance(ei.value.__cause__, OSError)
        assert b"write callback" in ei.value.message.encode()
        assert_same_stored(before, stored(col, dim))
    again = io.BytesIO()
    col.save(again)
    assert again.getvalue() == full.getvalue()
    col.close()


@pytest.mark.gpu
def test_write_failure_inside_the_dense_chunks(gb, ctx):
    """a failure while the next chunk is gathered and downloaded: 40,000 live rows of 1024 (164 MB, three 64 MB chunks)
    over 50,000 slots, the write failing in each chunk"""
    t = small(gb, ctx, 1024, n=40000)
    col = t.cols[0]
    live, slots = col.count()
    assert (live, slots) == (40000, 50000)
    q = t.vectors(70)["values"]
    before = col.query(q, (), 25)
    full = io.BytesIO()
    col.save(full)
    good = full.getvalue()
    dense = 4 * live * 1024
    assert dense > 2 * (64 << 20)
    meta = len(good) - dense
    for after in (meta + 10, meta + (64 << 20) + 10, meta + (128 << 20) + 10):
        with pytest.raises(gb.GorseB200Error) as ei:
            col.save(FailingSink(after))
        assert ei.value.status == -8 and isinstance(ei.value.__cause__, OSError)
        assert col.count() == (live, slots)
        assert all(np.array_equal(a, b) for a, b in zip(before, col.query(q, (), 25)))
    again = io.BytesIO()
    col.save(again)
    assert again.getvalue() == good
    col.close()


def raw_load(gb, ctx, data):
    """gorse_b200_vecdb_load over bytes: (status, handle, bytes read, message)"""
    from gorse_b200 import _lib

    src = io.BytesIO(data)
    read = _lib.READ_FN(lambda user, buf, n: src.readinto(memoryview((C.c_char * n).from_address(buf)).cast("B")))
    h, nb = C.c_void_p(), C.c_int64(0)
    st = _lib.lib.gorse_b200_vecdb_load(ctx.h, read, None, C.byref(h), C.byref(nb))
    msg = _lib.lib.gorse_b200_last_error().decode()
    if h.value:
        _lib.lib.gorse_b200_vecdb_destroy(h)
    return st, h.value, nb.value, msg


def sections(stream):
    """the byte offset where each section starts, by the documented format"""
    _, _, dim, _, _, n, nnz, ncat = HEADER.unpack_from(stream)
    out, at = {"hidden": 48}, 48 + n
    for name, size in (("timestamp_ms", 8 * n), ("cat_off", 8 * (n + 1)), ("cats", 4 * ncat)):
        out[name] = at
        at += size
    if dim:
        out["values"] = at
        at += 4 * n * dim
    else:
        for name, size in (("off", 8 * (n + 1)), ("ind", 4 * nnz), ("val", 4 * nnz)):
            out[name] = at
            at += size
    assert at == len(stream)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("dim", [0, 64])
def test_malformed_streams(gb, ctx, dim):
    from gorse_b200 import _lib

    t = small(gb, ctx, dim, n=200)
    buf = io.BytesIO()
    t.cols[0].save(buf)
    good = buf.getvalue()
    t.cols[0].close()
    assert raw_load(gb, ctx, good)[:3:2] == (0, len(good))
    sec = sections(good)

    def refused(data, want=_lib.ERR_ARG, field=None):
        st, h, _, msg = raw_load(gb, ctx, bytes(data))
        assert st == want and h is None, (st, msg)
        if field:
            assert field in msg, msg
        return msg

    # truncation at every section boundary (and inside the header), and at seeded random offsets
    rng = np.random.default_rng(1)
    for cut in sorted(set([0, 7, 20, 47] + list(sec.values()) + rng.integers(0, len(good), 40).tolist())):
        msg = refused(good[:cut])
        assert f"at byte {cut}" in msg, msg
    # wrong magic, version, dim / distance, reserved
    for off, fmt, val, field in ((0, "<8s", b"GB200VDX", "magic"), (8, "<I", 2, "version"), (12, "<i", 16385, "dim"),
                                 (16, "<i", 7, "distance"), (20, "<I", 1, "reserved")):
        bad = bytearray(good)
        struct.pack_into(fmt, bad, off, val)
        refused(bad, field=f"{field} at byte {off}")
    if dim:
        bad = bytearray(good)
        struct.pack_into("<i", bad, 12, 0)   # a sparse Dot header over dense sections
        refused(bad)
    else:
        bad = bytearray(good)
        struct.pack_into("<i", bad, 16, 1)   # a sparse Euclidean collection
        refused(bad, field="distance")
    # counts that disagree with their sections, or overflow
    n = HEADER.unpack_from(good)[5]
    for off, val, field in ((40, HEADER.unpack_from(good)[7] + 1, "cat_off"), (24, -1, "n"), (24, 1 << 61, "n"), (40, -5, "category count")):
        bad = bytearray(good)
        struct.pack_into("<q", bad, off, val)
        refused(bad, field=field)
    bad = bytearray(good)
    struct.pack_into("<q", bad, sec["cat_off"], 1)   # cat_off[0] != 0
    refused(bad, field=f"cat_off at byte {sec['cat_off']}")
    bad = bytearray(good)
    bad[sec["hidden"] + 3] = 2
    refused(bad, field=f"hidden at byte {sec['hidden'] + 3}")
    if dim == 0:
        nnz = HEADER.unpack_from(good)[6]
        bad = bytearray(good)
        struct.pack_into("<q", bad, 32, nnz - 1)   # nnz disagrees with off[n]
        refused(bad, field="off")
        off = np.frombuffer(good, "<i8", n + 1, sec["off"])
        r = int(np.flatnonzero(np.diff(off) >= 2)[0])
        t0 = int(off[r])
        bad = bytearray(good)   # an unsorted row: its first two indices swapped
        a, b = struct.unpack_from("<II", bad, sec["ind"] + 4 * t0)
        struct.pack_into("<II", bad, sec["ind"] + 4 * t0, b, a)
        refused(bad, field=f"ind at byte {sec['ind'] + 4 * (t0 + 1)}")
        bad = bytearray(good)
        struct.pack_into("<I", bad, sec["ind"] + 4 * (int(off[-1]) - 1), 0x7fffffff)
        refused(bad, field="ind")
        bad = bytearray(good)
        struct.pack_into("<f", bad, sec["val"] + 4 * 5, float("nan"))
        refused(bad, field=f"val at byte {sec['val'] + 20}")
        bad = bytearray(good)
        struct.pack_into("<q", bad, sec["off"] + 8 * 3, int(off[2]) - 1 if off[2] > 0 else -1)   # decreasing offsets
        refused(bad, field="off")
    # a read failure is GORSE_B200_ERR_IO
    src = io.BytesIO(good)

    def read(user, buf, k):
        if src.tell() > 100:
            return -1
        return src.readinto(memoryview((C.c_char * min(k, 64)).from_address(buf)).cast("B"))

    h = C.c_void_p()
    assert _lib.lib.gorse_b200_vecdb_load(ctx.h, _lib.READ_FN(read), None, C.byref(h), None) == _lib.ERR_IO and not h.value
    assert b"read callback" in _lib.lib.gorse_b200_last_error()
    # a header that claims far more than the stream holds fails at the end of the stream, not in an allocation
    bad = bytearray(good[:48])
    struct.pack_into("<q", bad, 24, 1 << 40 if dim == 0 else (1 << 40) // dim)
    msg = refused(bad)
    assert "ends at byte 48" in msg or "n at byte 24" in msg, msg


@pytest.mark.gpu
@pytest.mark.parametrize("dim", [0, 8, 1024])
def test_empty_collections(gb, ctx, dim):
    for deleted in (False, True):
        col = gb.VectorCollection(ctx, dim, gb.DISTANCE_DOT)
        if deleted:   # every vector tombstoned: an empty stream too
            t = Twins([col], dim, 4)
            t.upsert(np.arange(30), 1000)
            t.delete_before(5000)
        buf = io.BytesIO()
        ns = col.save(buf)
        assert np.all(ns == -1) and len(buf.getvalue()) == 48 + 8 + (0 if dim else 8)
        loaded = gb.VectorCollection.load(ctx, io.BytesIO(buf.getvalue()))
        assert loaded.count() == (0, 0)
        t = Twins([loaded], dim, 6)
        q = t.vectors(3)["values" if dim else "sparse"]
        assert loaded.query(q, (), 5)[2].tolist() == [0, 0, 0]
        t.upsert(np.arange(20), 2000)
        assert loaded.count() == (20, 20) and loaded.query(q, (), 5)[2].max() > 0
        loaded.close()
        col.close()


@pytest.mark.gpu
def test_load_on_another_device(gb, ctx):
    if gb.device_count() < 2:
        pytest.skip("one GPU")
    for kind in ("dot64", "sparse"):
        t = history(gb, ctx, kind)
        buf = io.BytesIO()
        t.cols[0].save(buf)
        t.compact()
        with gb.Context(1) as ctx1:
            other = gb.VectorCollection.load(ctx1, io.BytesIO(buf.getvalue()))
            w = workload(t, 21)
            a = {k: v for k, v in answers(gb, ctx, t.cols[0], t, w).items() if k != "recommend"}
            b = {k: v for k, v in answers(gb, ctx1, other, t, w).items() if k != "recommend"}
            assert_same(a, b)
            assert_same_stored(stored(t.cols[0], t.dim), stored(other, t.dim))
            other.close()
        t.cols[0].close()
