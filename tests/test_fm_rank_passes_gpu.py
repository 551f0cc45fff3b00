"""gorse_b200_fm_rank past one device pass, and the ranked gorse_b200_recommend past one chunk, at the ranker's production
sizes.  A call to fm_rank runs in passes of at most 2^22 pairs (or one user), each with a pair_base that the pair and
attention kernels subtract to index the pass's vx / row-sum buffers, and sorts users of more than 2,048 candidates in
per-CTA global buffers that each CTA reuses for every user it sorts.  Every case here asserts the pass, chunk and
global-sort counters it is built for, checks the order of every user against the spec over the device's own scores
(exact numpy), and restates a sample of users -- the first and last users of every pass, the users at the planted
boundaries and seeded others -- with fm_oracle: scores bit-identical (NaN as one value) and order equal.  A user's
answer depends only on its own row, candidates and the item table, so the sample is restated as a call of its own.
The recommend cases compare a call of more than one chunk with the same users in two calls, and a sample around every
chunk boundary with the composed path (the single-stage entries and the restated ranker)."""
import types

import numpy as np
import pytest

import fm_oracle
import recommend_model as rm
from test_fm_rank_gpu import same
from test_fm_rank_passes import (GROUP_PAIRS, SORT_SMEM, check_order, device_passes, expected_stats, gather, pass_layout,
                                 pow2_at_least, sample_users, sort_grid, take_users)
from test_recommend_gpu import check_same, fm_rank_fn

pytestmark = pytest.mark.gpu

NF, N_ITEMS = 3000, 5000


@pytest.fixture(scope="module")
def ctx(gb):
    with gb.Context(0) as c:
        yield c


@pytest.fixture(scope="module")
def sms():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def layout():
    """about 3.5 passes of 300-candidate users (pass_layout) with 0 to 6 labels per user and per item; the users at the
    planted boundaries and their neighbours"""
    counts, marks = pass_layout(50)
    inp = fm_oracle.random_input(np.random.default_rng(51), NF, counts, N_ITEMS, labels=3)
    edges = sorted({m + d for m in marks for d in (-3, -2, -1, 0, 1, 2, 3)})
    return inp, edges


def with_slots(inp, dims, seed):
    """inp with bf16 item embeddings of `dims` and a presence mask (a fifth of them absent)"""
    rng = np.random.default_rng(seed)
    s = types.SimpleNamespace(**vars(inp))
    s.item_emb = [fm_oracle.to_bf16(rng.standard_normal((inp.n_items, d), dtype=np.float32)) for d in dims]
    s.item_emb_mask = (rng.random((inp.n_items, len(dims))) >= 0.2).astype(np.uint8)
    return s


def check_sample(model, inp, sg, og, users):
    """the users' scores bit-identical to the restatement of those users alone (NaN as one value), their order equal"""
    sub = take_users(inp, users)
    so, oo = model.rank(sub)
    _, s_dev, o_dev = gather(inp.cand_off, users, sg, og)
    if not (same(s_dev, so) and o_dev.tolist() == oo.tolist()):
        bad = [int(u) for j, u in enumerate(users) if not same(s_dev[sub.cand_off[j]:sub.cand_off[j + 1]], so[sub.cand_off[j]:sub.cand_off[j + 1]])
               or o_dev[sub.cand_off[j]:sub.cand_off[j + 1]].tolist() != oo[sub.cand_off[j]:sub.cand_off[j + 1]].tolist()]
        pytest.fail(f"{len(bad)} of {len(users)} sampled users differ from the restatement, first {bad[:8]}")


def rank_and_check(gb, ctx, inp, k, num_dim, bs, dims, params, users, name):
    with gb.FMRanker(ctx, NF, k, num_dim, bs, dims, params) as fm:
        sg, og, stats = fm.rank(inp)
    print(f"{name}: {stats}")
    assert stats == expected_stats(inp.cand_off, bs if dims else None)
    check_order(inp.cand_off, sg, og)
    check_sample(fm_oracle.Model(NF, k, num_dim, bs, dims, params), inp, sg, og, users)
    return sg, og, stats


@pytest.mark.parametrize("k", [8, 16, 32])
def test_passes_without_slots(gb, ctx, layout, k):
    inp, edges = layout
    P = device_passes(inp.cand_off)
    users = np.union1d(sample_users(inp.cand_off, P, 50, k), edges)
    params = fm_oracle.random_params(np.random.default_rng(52 + k), NF, k)
    _, _, stats = rank_and_check(gb, ctx, inp, k, 3, 1024, (), params, users, f"k = {k}")
    assert stats["passes"] >= 3


@pytest.mark.parametrize("dims,bs", [((16,), 7), ((16,), 1024), ((16, 7), 7)], ids=["16-bs7", "16-bs1024", "16+7-bs7"])
def test_passes_with_slots(gb, ctx, layout, dims, bs):
    """the attention reads each pair's vx and its chunk's row sums at pair - pair_base: on passes 1 to 3 a slip to the
    absolute pair reads another pair's values; the users at every boundary end inside an attention chunk"""
    inp, edges = layout
    inp = with_slots(inp, dims, 53 + bs)
    P = device_passes(inp.cand_off)
    n = np.diff(inp.cand_off)
    assert all(n[u] % bs for u0, u1 in P for u in (u0, u1 - 1) if n[u])
    users = np.union1d(sample_users(inp.cand_off, P, 50, bs + len(dims)), edges)
    params = fm_oracle.random_params(np.random.default_rng(54 + len(dims)), NF, 16, dims)
    _, _, stats = rank_and_check(gb, ctx, inp, 16, 3, bs, dims, params, users, f"slots {dims}, batch {bs}")
    assert stats["passes"] >= 3 and stats["chunks"] > 0


def test_one_user_above_a_pass(gb, ctx):
    """a user of 2^22 + 1 candidates between two small users: a pass of its own and a global sort at p = 2^23, over
    repeated candidates (exact ties) and items with a NaN label (NaN scores)"""
    rng = np.random.default_rng(60)
    counts = [700, GROUP_PAIRS + 1, 300]
    ni, k = 3000, 8
    inp = fm_oracle.random_input(rng, NF, counts, ni, labels=1)
    inp.user_lab_off[:] = 0   # the users' rows are their ids: short rows keep the restatement of the big user in seconds
    labelled = np.nonzero(np.diff(inp.item_lab_off))[0]
    inp.item_lab_val[inp.item_lab_off[rng.choice(labelled, 40, replace=False)]] = np.nan
    assert pow2_at_least(counts[1]) == 1 << 23 and device_passes(inp.cand_off) == [(0, 1), (1, 2), (2, 3)]
    params = fm_oracle.random_params(rng, NF, k)
    sg, og, stats = rank_and_check(gb, ctx, inp, k, 3, 1024, (), params, [0, 1, 2], "one user above a pass")
    assert stats["passes"] == 3 and stats["global_sorts"] == 1
    big = sg[counts[0]:counts[0] + counts[1]]
    assert np.isnan(big).sum() > 10000 and np.unique(big[~np.isnan(big)]).size < ni   # NaN and exact ties at this size


def test_many_global_sorted_users_per_cta(gb, ctx, sms):
    """one pass of 270 users above 2,048 candidates (up to 40,000) among 400 below and one of 1.1M, whose 2^21-entry sort
    buffers cap the grid at 10 CTAs: each CTA sorts many users in turn in its reused buffer"""
    rng = np.random.default_rng(70)
    glob = np.concatenate([[2049, 4096, 4097, 8193], rng.integers(2049, 12000, 256), rng.integers(20000, 40001, 10)])
    small = np.concatenate([[2048, 0, 1, 2047], rng.integers(0, 2049, 396)])
    counts = np.concatenate([glob, small, [1_100_000]])
    rng.shuffle(counts)
    nu, n_global = counts.size, int((counts > SORT_SMEM).sum())
    inp = fm_oracle.random_input(rng, NF, counts, N_ITEMS, labels=3)
    assert inp.cand_off[-1] <= GROUP_PAIRS and device_passes(inp.cand_off) == [(0, nu)]
    grid = sort_grid(inp.cand_off, 0, nu, sms)
    assert grid == 10 and n_global > 20 * grid
    # the users each CTA sorts second and third, its first global-sorted user after the first, the big user and seeded others
    later = np.arange(grid, 3 * grid)
    second_global = [np.nonzero(counts[b::grid] > SORT_SMEM)[0][1] * grid + b for b in range(grid)]
    users = np.unique(np.concatenate([later, second_global, [int(np.argmax(counts))], rng.choice(nu, 20, replace=False)]))
    params = fm_oracle.random_params(rng, NF, 16)
    _, _, stats = rank_and_check(gb, ctx, inp, 16, 3, 1024, (), params, users, "many global sorts")
    assert stats["passes"] == 1 and stats["global_sorts"] == n_global


@pytest.mark.parametrize("dims,bs", [((), 1024), ((16,), 7)], ids=["no-slot", "16-bs7"])
def test_split_and_repeated_calls_give_the_same_bits(gb, ctx, layout, dims, bs):
    """the whole input twice, then in three calls cut inside passes 1 and 2, on the buffers the whole call grew"""
    inp, _ = layout
    if dims:
        inp = with_slots(inp, dims, 55)
    P = device_passes(inp.cand_off)
    cuts = [0, P[1][0] + (P[1][1] - P[1][0]) // 3, P[2][0] + (P[2][1] - P[2][0]) // 2, inp.n_users]
    assert not {u0 for u0, _ in P} & set(cuts[1:-1])
    params = fm_oracle.random_params(np.random.default_rng(56), NF, 16, dims)
    with gb.FMRanker(ctx, NF, 16, 3, bs, dims, params) as fm:
        s1, o1, st = fm.rank(inp)
        s2, o2, _ = fm.rank(inp)
        parts = [fm.rank(take_users(inp, np.arange(a, b))) for a, b in zip(cuts[:-1], cuts[1:])]
    print(f"whole call {st}; parts {[p[2] for p in parts]}")
    assert st["passes"] >= 3
    assert s1.tobytes() == s2.tobytes() and o1.tobytes() == o2.tobytes()
    assert np.concatenate([p[0] for p in parts]).tobytes() == s1.tobytes()
    assert np.concatenate([p[1] for p in parts]).tobytes() == o1.tobytes()


# ---- gorse_b200_recommend with a ranker past one chunk ---------------------------------------------------------------------------
CHUNK_ENTRIES = 1 << 26   # candidate / exclude-set entries of one chunk of gorse_b200_recommend (recommend.cu); a 16th with slots


def recommend_chunks(bound, cap, sms, lim):
    """the first user of every chunk of gorse_b200_recommend (plan in recommend.cu): at most sm_count * 1024 users, and at
    most lim bound and exclude-set entries, or one user"""
    at, b, c = [0], 0, 0
    for u in range(len(bound)):
        if u > at[-1] and (u - at[-1] == sms * 1024 or b + bound[u] > lim or c + cap[u] > lim):
            at.append(u)
            b = c = 0
        b += int(bound[u])
        c += int(cap[u])
    return at


@pytest.fixture(scope="module")
def rec_world(gb, ctx, sms):
    rng = np.random.default_rng(80)
    w = types.SimpleNamespace()
    w.nu, w.ni = max(140000, sms * 1024 + 4000), 3000
    w.live = (rng.random(w.ni) > 0.1).astype(np.uint8)
    w.E0 = [rng.choice(w.ni, size=int(rng.integers(0, 6)), replace=False).tolist() for _ in range(w.nu)]
    w.coll = gb.VectorCollection(ctx, 16, gb.DISTANCE_DOT)
    w.coll.add(values=rng.standard_normal((2000, 16)).astype(np.float32))
    w.fb = [rng.choice(w.ni, size=int(rng.integers(0, 9))).tolist() for _ in range(2000)]
    w.slots = rng.integers(-1, 2000, w.nu)
    w.pop = (rng.choice(w.ni, 60, replace=False).astype(np.int32), rng.standard_normal(60))
    w.n = 12
    w.inp = fm_oracle.random_input(rng, 500, [0] * w.nu, w.ni, (32,))
    yield w
    w.coll.close()


@pytest.mark.parametrize("ranker", ["fm", "fm_slot"])
def test_recommend_ranked_past_one_chunk(gb, ctx, sms, rec_world, ranker):
    """a list stage and a user-to-user stage, ranked by the FM (no slot, or one 32-dim slot in attention chunks of 7 that
    cross user ends), over more users than one chunk: equal to the same users in two calls cut inside a chunk, and around
    every chunk boundary equal to the composed path with the restated ranker"""
    w = rec_world
    dims, bs = ((32,), 7) if ranker == "fm_slot" else ((), 1024)
    nf, k, nd = 500, 8, 6
    params = fm_oracle.random_params(np.random.default_rng(81), nf, k, dims)
    inp = w.inp if dims else types.SimpleNamespace(**{**vars(w.inp), "item_emb": [], "item_emb_mask": None})

    def stages(a, b):
        return [gb.ListStage(*w.pop), gb.UserToUserStage(w.coll, w.n, w.slots[a:b], w.fb)]

    bound = gb.recommend_bounds(w.nu, stages(0, w.nu))
    cap = np.array([len(set(e)) for e in w.E0], np.int64) + len(w.pop[0])   # E0 and every stage but the last
    at = recommend_chunks(bound, cap, sms, CHUNK_ENTRIES // 16 if dims else CHUNK_ENTRIES)
    with gb.FMRanker(ctx, nf, k, nd, bs, dims, params) as fm:
        fm.oracle = fm_oracle.Model(nf, k, nd, bs, dims, params)
        big, stats = gb.recommend(ctx, w.E0, w.ni, w.live, stages(0, w.nu), ranker=(fm, inp))
        print(f"recommend, ranker {ranker}: {stats}, chunks start at users {at}")
        assert stats["chunks"] == len(at) >= 2
        cut = 70001
        assert cut not in at
        small = []
        for a, b in ((0, cut), (cut, w.nu)):
            small += gb.recommend(ctx, w.E0[a:b], w.ni, w.live, stages(a, b), ranker=(fm, take_users(inp, np.arange(a, b))))[0]
        assert len(small) == len(big)
        for u, ((a, b), (c, d)) in enumerate(zip(big, small)):
            assert a.tobytes() == c.tobytes() and b.tobytes() == d.tobytes(), u
        lens = np.array([len(r[0]) for r in big])
        assert np.unique(lens).size > 10 and (lens % bs != 0).any()
        # around every chunk boundary, the first and last users, and seeded others from the first, a middle and the last chunk
        rng = np.random.default_rng(82)
        users = {0, 1, w.nu - 2, w.nu - 1}
        for a in at[1:]:
            users.update(range(a - 3, a + 3))
        for c in {0, len(at) // 2, len(at) - 1}:
            lo, hi = at[c], (at + [w.nu])[c + 1]
            users.update(rng.integers(lo, hi, 10).tolist())
        users = np.array(sorted(users), np.int64)

        def u2u(E):
            rows, _ = w.coll.user_to_user(w.slots[users], w.fb, [sorted(e) for e in E], w.n, w.ni)
            return [[(int(i), float(v)) for i, v in zip(*r)] for r in rows]

        want = rm.chain([w.E0[u] for u in users], w.live, [rm.list_stage(*w.pop), u2u],
                        rank=fm_rank_fn(fm, take_users(inp, users), oracle=True))
    assert sum(len(r) for r in want) > 0
    check_same([big[u] for u in users], want)
