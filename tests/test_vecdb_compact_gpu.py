"""Compaction of a vector collection (gorse_b200_vecdb_compact) after master-style write cycles: upserts that replace the
previous version of an id, hidden vectors, categories, timestamps and delete_before.  Every entry answers afterwards what it
answered before, with every slot-valued input and output renamed through the returned map and the same score bits; the map,
the counts and the stored vectors; the edge cases; and the device bytes of a collection compacted every cycle stay bounded."""
import types

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

# name -> (dim, distance, ids).  dot64 keeps >= 32768 live vectors, so the tensor-core sweep answers before and after;
# euc48 has >= 32768 slots before and < 32768 live vectors after (sweep before, exact scan after); cos30 (d % 4 != 0: the
# scalar row copy) answers query only; sparse upserts change features, so dead rows sit in posting lists.
KINDS = {"dot64": (64, "DOT", 40000), "euc48": (48, "EUCLIDEAN", 24000), "cos30": (30, "COSINE", 3000), "sparse": (0, "DOT", 4000)}
N_Q = 80   # query rows: >= 64 for the sweep
N_USERS = 96


@pytest.fixture(scope="module")
def ctx(gb):
    c = gb.Context(0)
    yield c
    c.close()


class History:
    """a collection and the id <-> slot map a shim keeps for it"""

    def __init__(self, gb, ctx, dim, distance, seed):
        self.col = gb.VectorCollection(ctx, dim, getattr(gb, "DISTANCE_" + distance))
        self.dim, self.rng = dim, np.random.default_rng(seed)
        self.slot_of, self.id_of = {}, []

    def vectors(self, n):
        if self.dim > 0:
            return dict(values=self.rng.standard_normal((n, self.dim)).astype(np.float32))
        out = []
        for _ in range(n):
            k = int(self.rng.integers(2, 16))
            out.append((np.sort(self.rng.choice(300, k, replace=False)).astype(np.uint32), self.rng.uniform(0.1, 1.0, k).astype(np.float32)))
        return dict(sparse=out)

    def upsert(self, ids, ts, batch=10000):
        for a in range(0, len(ids), batch):
            part = [int(i) for i in ids[a:a + batch]]
            n = len(part)
            cats = [np.flatnonzero(self.rng.random(3) < 0.5).tolist() for _ in range(n)]
            first = self.col.add(hidden=self.rng.random(n) < 0.05, timestamps=np.full(n, ts), categories=cats,
                                 replace=[self.slot_of.get(i, -1) for i in part], **self.vectors(n))
            for j, i in enumerate(part):
                self.slot_of[i] = first + j
            self.id_of += part

    def delete_before(self, ts):
        gone = self.col.delete_before(ts)
        for s in gone:
            del self.slot_of[self.id_of[s]]
        return gone

    def compact(self):
        new_slot, b0, b1 = self.col.compact()
        self.slot_of = {i: int(new_slot[s]) for i, s in self.slot_of.items()}
        self.id_of = [self.id_of[s] for s in np.flatnonzero(new_slot >= 0)]
        return new_slot, b0, b1


def history(gb, ctx, kind):
    dim, dist, m = KINDS[kind]
    h = History(gb, ctx, dim, dist, seed=7)
    h.upsert(np.arange(m), 1000)
    h.upsert(h.rng.choice(m, m * 6 // 10, replace=False), 2000)
    h.upsert(h.rng.choice(m, m * 8 // 10, replace=False), 3000)
    assert len(h.delete_before(2000)) > 0   # the ids last written by the first cycle
    h.upsert(np.arange(m, m + m // 50), 4000)
    h.n_ids = m + m // 50
    return h


def workload(h):
    """slot-valued inputs of every entry, drawn from the slots before compaction: live ones, deleted ones and -1"""
    rng = np.random.default_rng(11)
    slots = h.col.count()[1]
    live = np.array(sorted(h.slot_of.values()), np.int64)
    dead = np.setdiff1d(np.arange(slots), live)

    def pick(k):
        s = rng.choice(live, k)
        r = rng.random(k)
        s[r < 0.15] = rng.choice(dead, int((r < 0.15).sum()))
        s[r > 0.93] = -1
        return s

    def ids(k):   # dictionary items (= ids), some of them deleted, some -1
        s = rng.integers(0, h.n_ids, k)
        s[rng.random(k) > 0.9] = -1
        return s

    w = types.SimpleNamespace()
    w.q = rng.standard_normal((N_Q, h.dim)).astype(np.float32) if h.dim > 0 else h.vectors(N_Q)["sparse"]
    w.excl = [np.unique(pick(int(rng.integers(0, 12)))) for _ in range(N_Q)]
    w.ctx = [pick(int(rng.integers(1, 8))) for _ in range(N_USERS)]
    w.ex = [np.unique(pick(int(rng.integers(0, 10)))) for _ in range(N_USERS)]
    w.user_slots = pick(N_USERS)
    w.fb = [rng.integers(0, h.n_ids, int(rng.integers(0, 6))) for _ in range(slots)]   # per slot, item indices
    w.ex_items = [np.unique(ids(int(rng.integers(0, 8)))) for _ in range(N_USERS)]
    w.item_ok = (rng.random(h.n_ids) > 0.1).astype(np.uint8)
    w.slot_ok = (rng.random(slots) > 0.1).astype(np.uint8)
    w.ctx_items = [ids(int(rng.integers(1, 8))) for _ in range(N_USERS)]
    w.item_live = (rng.random(h.n_ids) > 0.05).astype(np.uint8)
    w.soi = np.full(h.n_ids, -1, np.int64)
    w.ios = np.full(slots, -1, np.int32)
    for i, s in h.slot_of.items():
        w.soi[i], w.ios[s] = s, i
    return w


def renamed(w, new_slot):
    """the same workload in the compacted slot space"""
    keep = new_slot >= 0

    def ren(a):
        a = np.asarray(a, np.int64)
        return np.where(a >= 0, new_slot[np.maximum(a, 0)], -1)

    r = types.SimpleNamespace(**vars(w))
    r.excl, r.ctx, r.ex = [ren(e) for e in w.excl], [ren(c) for c in w.ctx], [ren(e) for e in w.ex]
    r.user_slots, r.soi = ren(w.user_slots), ren(w.soi)
    r.fb = [f for f, k in zip(w.fb, keep) if k]
    r.slot_ok, r.ios = w.slot_ok[keep], w.ios[keep]
    return r


def rows_of(slots, scores, cnt):
    return [(slots[q, :c].copy(), scores[q, :c].copy()) for q, c in enumerate(cnt)]


def answers(gb, ctx, h, w):
    col, out = h.col, {}
    out["query"] = rows_of(*col.query(w.q, (), 20))
    out["query_categories"] = rows_of(*col.query(w.q, (1,), 20))
    if h.col.distance == gb.DISTANCE_COSINE:
        return out, None
    exact = None
    if h.dim > 0:
        out["query_excluding"], exact = col.query_excluding(w.q, w.excl, 15)
    out["item_to_item"] = col.item_to_item(w.ctx, w.ex, 10, categories=(0,))[0]
    out["session_recommend"] = col.session_recommend(w.ctx, w.ex, 10, 3, 15, item_ok=w.slot_ok)[0]
    items = {}   # item-valued answers: compared without renaming
    items["user_to_user"] = col.user_to_user(w.user_slots, w.fb, w.ex_items, 10, h.n_ids, w.item_ok)[0]
    stages = [gb.ItemToItemStage(col, 10, w.ctx_items, w.soi, w.ios, score_scale=0.5),
              gb.UserToUserStage(col, 10, w.user_slots, w.fb, w.item_ok)]
    items["recommend"] = gb.recommend(ctx, w.ex_items, h.n_ids, w.item_live, stages)[0]
    out["items"] = items
    return out, exact


def stored(h, slots):
    vals, hid, ts, live = h.col.get(slots)
    sp = [h.col.get_sparse(int(s)) for s in slots[::37]] if h.dim == 0 else None
    return vals, hid, ts, live, sp


@pytest.fixture(scope="module", params=list(KINDS))
def compacted(request, gb, ctx):
    kind = request.param
    h = history(gb, ctx, kind)
    w = workload(h)
    r = types.SimpleNamespace(kind=kind, h=h, count_before=h.col.count())
    r.live_before = np.array(sorted(h.slot_of.values()), np.int64)
    r.stored_before = stored(h, r.live_before)
    r.before, r.exact_before = answers(gb, ctx, h, w)
    r.new_slot, r.bytes_before, r.bytes_after = h.compact()
    r.count_after = h.col.count()
    r.stored_after = stored(h, r.new_slot[r.live_before])
    r.after, r.exact_after = answers(gb, ctx, h, renamed(w, r.new_slot))
    yield r
    h.col.close()


def same_rows(a, b, rename=None):
    assert len(a) == len(b)
    for (s0, v0), (s1, v1) in zip(a, b):
        s0 = np.asarray(s0, np.int64)
        if rename is not None:
            s0 = rename[s0]
        assert np.array_equal(s0, s1)
        assert v0.tobytes() == v1.tobytes()   # the same score bits


def test_same_answers(compacted):
    r = compacted
    assert r.before.keys() == r.after.keys()
    for name in r.before:
        if name == "items":
            for entry in r.before["items"]:
                same_rows(r.before["items"][entry], r.after["items"][entry])
        else:
            same_rows(r.before[name], r.after[name], r.new_slot)
    assert sum(len(s) for s, _ in r.before["query"]) > 0
    if "item_to_item" in r.before:
        assert sum(len(s) for s, _ in r.before["item_to_item"]) > 0 and sum(len(s) for s, _ in r.before["items"]["recommend"]) > 0


def test_both_dense_paths(compacted):
    r = compacted
    if r.kind not in ("dot64", "euc48"):
        pytest.skip("dense Dot / Euclidean only")
    assert r.count_before[1] >= 32768 and r.exact_before < N_Q   # the sweep answered before
    if r.kind == "dot64":
        assert r.count_after[0] >= 32768 and r.exact_after < N_Q
    else:
        assert r.count_after[0] < 32768 and r.exact_after == N_Q


def test_the_map(compacted):
    r = compacted
    live, slots = r.count_before
    ns = r.new_slot
    assert ns.size == slots and r.count_after == (live, live)
    assert np.array_equal(np.flatnonzero(ns >= 0), r.live_before)
    assert np.array_equal(ns[r.live_before], np.arange(live))   # strictly increasing over the live slots
    assert np.all(ns[np.setdiff1d(np.arange(slots), r.live_before)] == -1)
    assert r.bytes_after < r.bytes_before
    (v0, h0, t0, l0, sp0), (v1, h1, t1, l1, sp1) = r.stored_before, r.stored_after
    assert l0.all() and l1.all()
    assert np.array_equal(v0, v1) and np.array_equal(h0, h1) and np.array_equal(t0, t1)
    assert h0.any() and len(set(t0.tolist())) > 1
    if sp0 is not None:
        for (i0, x0), (i1, x1) in zip(sp0, sp1):
            assert np.array_equal(i0, i1) and x0.tobytes() == x1.tobytes()


def small(gb, ctx, sparse, n, ts=1000):
    h = History(gb, ctx, 0 if sparse else 24, "DOT", seed=3)
    h.upsert(np.arange(n), ts)
    return h


@pytest.mark.parametrize("sparse", [False, True])
def test_second_compaction_is_identity(gb, ctx, sparse):
    h = small(gb, ctx, sparse, 500)
    h.upsert(np.arange(0, 500, 3), 2000)
    h.col.query(h.vectors(4)["values"] if not sparse else h.vectors(4)["sparse"], (), 5)
    ns, b0, b1 = h.compact()
    assert (ns == -1).sum() == len(range(0, 500, 3))
    ns2, c0, c1 = h.compact()
    assert np.array_equal(ns2, np.arange(500)) and c0 == c1 == b1
    h.col.close()


@pytest.mark.parametrize("sparse", [False, True])
def test_all_dead_collection_becomes_empty(gb, ctx, sparse):
    h = small(gb, ctx, sparse, 300)
    q = h.vectors(3)["values"] if not sparse else h.vectors(3)["sparse"]
    h.col.query(q, (), 5)
    assert len(h.delete_before(5000)) == 300
    ns, b0, b1 = h.compact()
    assert np.all(ns == -1) and h.col.count() == (0, 0) and b1 < b0
    assert h.col.query(q, (), 5)[2].tolist() == [0, 0, 0]
    h.upsert(np.arange(300, 340), 6000)
    assert h.col.count() == (40, 40) and sorted(h.slot_of.values()) == list(range(40))
    s, _, cnt = h.col.query(q, (), 5)
    assert cnt.max() > 0 and s[0, :cnt[0]].max() < 40
    h.col.close()


@pytest.mark.parametrize("sparse", [False, True])
def test_add_and_delete_after_compaction(gb, ctx, sparse):
    h = small(gb, ctx, sparse, 400)
    h.upsert(np.arange(100), 2000)     # slots 0 .. 99 die
    h.compact()
    assert h.col.count() == (400, 400)
    first = h.col.add(**h.vectors(1), timestamps=[3000], replace=[h.slot_of[7]])
    assert first == 400 and h.col.count() == (400, 401)
    # the ids last written at 1000 sit in the new slots 0 .. 299
    gone = h.col.delete_before(2000)
    assert np.array_equal(gone, np.arange(300)) and h.col.count() == (100, 401)
    _, hid, ts, live = h.col.get(np.array([300, 307, 400]))
    assert live.tolist() == [1, 0, 1] and ts.tolist() == [2000, 0, 3000]
    h.col.close()


@pytest.mark.parametrize("sparse", [False, True])
def test_bounded_memory(gb, ctx, sparse):
    """five master cycles -- upsert every vector in batches of 10 000 with a new timestamp, delete_before, a few queries --
    with compaction end at no more device bytes than after the first; without it the slots grow by the collection per cycle"""
    m = 4000 if sparse else 20000
    arms = {True: small(gb, ctx, sparse, 0), False: small(gb, ctx, sparse, 0)}
    q = arms[True].vectors(32)["sparse" if sparse else "values"]   # < 64 rows: the same search path every cycle
    nbytes = []
    for cycle in range(1, 6):
        for compact, h in arms.items():
            h.upsert(np.arange(m), 1000 * cycle)
            h.delete_before(1000 * cycle)
            h.col.query(q, (), 10)
            if compact:
                nbytes.append(h.compact()[2])
            assert h.col.count() == (m, m if compact else m * cycle)
    assert max(nbytes) <= nbytes[0], nbytes
    for h in arms.values():
        h.col.close()
