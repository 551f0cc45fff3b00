"""The helpers of tests/test_fm_rank_passes_gpu.py, checked without a device: cutting an FM ranking input down to some of
its users (the restatement of the cut users equals their rows in the restatement of the whole input), the device passes
and sort grid of gorse_b200_fm_rank restated from fm.cu, the order spec checked over every user, and the layouts the GPU
tests are built on, which must reach the pass and global-sort boundaries they are meant to reach."""
import types

import numpy as np
import pytest

import fm_oracle

# restated from csrc/fm.cuh and csrc/fm.cu
GROUP_PAIRS = 1 << 22              # pairs of one device pass, unless one user has more
SORT_SMEM = 2048                   # candidates a CTA sorts in shared memory; more sort in a per-CTA global buffer
SORT_BUFFER_BYTES = 256 << 20      # the per-CTA global sort buffers of one pass together (8-byte key + 4-byte position each)


def pow2_at_least(n):
    p = 1
    while p < n:
        p <<= 1
    return p


def gather(off, users, *cols):
    """the rows of `users` (in that order) of the CSR columns `cols` over offsets `off` -> (rebased offsets, *columns)"""
    users = np.asarray(users, np.int64)
    lo, n = off[users], off[users + 1] - off[users]
    new = np.zeros(users.size + 1, np.int64)
    np.cumsum(n, out=new[1:])
    at = np.repeat(lo - new[:-1], n) + np.arange(new[-1])
    return (new,) + tuple(c[at] for c in cols)


def take_users(inp, users):
    """the FM ranking input of `users` alone, in that order: their user rows and candidate lists with the offsets rebased;
    the item table and its embeddings shared with `inp`"""
    users = np.asarray(users, np.int64)
    s = types.SimpleNamespace(**vars(inp))
    s.n_users = users.size
    s.user_feat = np.ascontiguousarray(inp.user_feat[users])

    def rows(off, *cols):   # with one entry past the end, as every FMInput array has, so that no pointer is NULL
        new, *got = gather(off, users, *cols)
        return (new,) + tuple(np.ascontiguousarray(np.append(g, np.zeros(1, g.dtype))) for g in got)

    s.user_lab_off, s.user_lab_idx, s.user_lab_val = rows(inp.user_lab_off, inp.user_lab_idx, inp.user_lab_val)
    s.cand_off, s.cand_items = rows(inp.cand_off, inp.cand_items)
    return s


def device_passes(cand_off):
    """gorse_b200_fm_rank's device passes [(u0, u1)]: consecutive users of at most GROUP_PAIRS pairs, or one user; a pass
    without pairs is skipped and not counted"""
    n, out, u0 = len(cand_off) - 1, [], 0
    while u0 < n:
        u1 = u0 + 1
        while u1 < n and cand_off[u1 + 1] - cand_off[u0] <= GROUP_PAIRS:
            u1 += 1
        if cand_off[u1] > cand_off[u0]:
            out.append((u0, u1))
        u0 = u1
    return out


def sort_grid(cand_off, u0, u1, sm_count):
    """the CTAs of fm_sort_kernel on pass [u0, u1): CTA b sorts users u0 + b, u0 + b + grid, ...; with a user above
    SORT_SMEM the per-CTA global buffers of pow2_at_least(largest) entries are capped at SORT_BUFFER_BYTES together"""
    sg = min(u1 - u0, sm_count * 8)
    max_p = pow2_at_least(max(int(np.diff(cand_off[u0:u1 + 1]).max()), 1))
    if max_p > SORT_SMEM:
        sg = max(1, min(sg, SORT_BUFFER_BYTES // (max_p * 12)))
    return sg


def expected_stats(cand_off, batch_size=None):
    """the stats gorse_b200_fm_rank reports for cand_off; batch_size with embedding slots, None without"""
    n = np.diff(np.asarray(cand_off, np.int64))
    return {"pairs": int(n.sum()), "chunks": int((-(-n // batch_size)).sum()) if batch_size else 0,
            "passes": len(device_passes(cand_off)), "global_sorts": int((n > SORT_SMEM).sum())}


def check_order(cand_off, scores, order):
    """every user's order is a permutation of its positions by (score descending, position ascending), -0 == +0, NaN
    last: exact, over the device's own scores, every user"""
    cand_off = np.asarray(cand_off, np.int64)
    n = np.diff(cand_off)
    total = int(cand_off[-1])
    assert scores.shape == order.shape == (total,)
    user = np.repeat(np.arange(n.size), n)
    assert (order >= 0).all() and (order < n[user]).all(), "a position outside its user's list"
    g = cand_off[user] + order                       # the pair each rank names
    seen = np.zeros(total, bool)
    seen[g] = True
    assert seen.all(), "a user's order repeats a position"
    s, same_user = scores[g], user[1:] == user[:-1]
    a, b, pa, pb = s[:-1], s[1:], order[:-1], order[1:]
    na, nb = np.isnan(a), np.isnan(b)
    with np.errstate(invalid="ignore"):
        ok = np.where(na, nb & (pa < pb), nb | (a > b) | ((a == b) & (pa < pb)))
    bad = np.nonzero(same_user & ~ok)[0]
    assert bad.size == 0, f"user {user[bad[0]]}: ranks {order[bad[0]]} ({a[bad[0]]}) then {order[bad[0] + 1]} ({b[bad[0]]})"


def pass_layout(seed):
    """candidate counts over about 3.5 device passes, each count not a multiple of 7 or 1024 (so that a slot's attention
    chunk of 7 or 1024 candidates ends inside a user at every boundary).  Pass 0 opens with a user without candidates and
    ends with a user that fills it to exactly GROUP_PAIRS, then two users without candidates.  Pass 1 ends with two users
    without candidates; the next user overflows it by one pair and opens pass 2, followed by two users without candidates.
    Pass 2 ends the same way, and pass 3 holds about half a pass and ends with a user without candidates.
    -> (counts int64, the users at the planted boundaries)"""
    rng = np.random.default_rng(seed)

    def draw(room):   # counts in [1, 600) with a sum in (room - 1600, room - 1000]
        c = rng.integers(1, 600, room // 300 + 200)
        c += (c % 7 == 0)
        c = c[:np.searchsorted(np.cumsum(c), room - 1000, side="right")]
        return c.tolist()

    def last(need):   # `need` candidates, or more users before it when `need` is a multiple of 7 or 1024
        out = []
        while need % 7 == 0 or need % 1024 == 0:
            out.append(1)
            need -= 1
        return out + [need]

    counts, marks = [0], []
    body = draw(GROUP_PAIRS)
    counts += body + last(GROUP_PAIRS - sum(body))
    marks.append(len(counts) - 1)                  # fills pass 0 to exactly GROUP_PAIRS
    counts += [0, 0]
    opened = 0                                     # the pairs of the user that opened the pass
    for _ in range(2):
        body = draw(GROUP_PAIRS - opened)
        need = GROUP_PAIRS - opened - sum(body) + 1
        while need % 7 == 0 or need % 1024 == 0:
            body.append(1)
            need -= 1
        counts += body + [0, 0, need]
        marks.append(len(counts) - 1)              # overflows the pass before it by one pair
        counts += [0, 0]
        opened = need
    counts += draw(GROUP_PAIRS // 2) + [0]
    return np.array(counts, np.int64), marks


def sample_users(cand_off, passes, n_random, seed):
    """the first two and the last two users with candidates of every pass, and n_random seeded others"""
    n = np.diff(cand_off)
    users = set()
    for u0, u1 in passes:
        nz = np.nonzero(n[u0:u1])[0] + u0
        users.update(nz[:2].tolist() + nz[-2:].tolist())
    users.update(np.random.default_rng(seed).choice(n.size, n_random, replace=False).tolist())
    return np.array(sorted(users), np.int64)


def offsets(counts):
    off = np.zeros(len(counts) + 1, np.int64)
    np.cumsum(counts, out=off[1:])
    return off


# ---- the helpers ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dims", [(), (16,), (16, 7)])
def test_take_users_restates_as_the_whole(dims):
    rng = np.random.default_rng(40 + len(dims))
    nf, k, bs = 120, 8, 7
    counts = [5, 0, 13, 1, 0, 30, 8, 22, 0, 3]
    params = fm_oracle.random_params(rng, nf, k, dims)
    inp = fm_oracle.random_input(rng, nf, counts, 60, dims)
    model = fm_oracle.Model(nf, k, 4, bs, dims, params)
    s_all, o_all = model.rank(inp)
    for users in ([0, 2, 5, 9], [7, 1, 3, 5, 5], [4], list(range(len(counts)))):
        sub = take_users(inp, users)
        assert sub.n_users == len(users) and sub.cand_off[-1] == sum(counts[u] for u in users)
        s_sub, o_sub = model.rank(sub)
        off, s_want, o_want = gather(inp.cand_off, users, s_all, o_all)
        assert off.tolist() == sub.cand_off.tolist()
        assert s_sub.tobytes() == s_want.tobytes() and o_sub.tolist() == o_want.tolist()


def test_check_order_is_the_restatement_order():
    """the restatement's order passes; a swapped tie, a NaN ahead of a number, -0 ahead of an earlier +0 and a repeated
    position do not"""
    rng = np.random.default_rng(41)
    nf, k = 50, 8
    params = fm_oracle.random_params(rng, nf, k)
    inp = fm_oracle.random_input(rng, nf, [40, 0, 25, 60], 8)   # 8 items: repeated candidates tie exactly
    s, o = fm_oracle.Model(nf, k, 3, 1024, (), params).rank(inp)
    check_order(inp.cand_off, s, o)
    u0 = o[:40].copy()
    t = next(i for i in range(39) if s[u0[i]] == s[u0[i + 1]])
    for bad in (np.r_[u0[:t], u0[t + 1], u0[t], u0[t + 2:]], np.r_[u0[:1], u0[:39]]):
        with pytest.raises(AssertionError):
            check_order(inp.cand_off, s, np.r_[bad, o[40:]].astype(np.int32))
    s2 = np.array([1.0, np.nan, 0.0, -0.0, 0.0, 2.0], np.float32)
    off = np.array([0, 6], np.int64)
    check_order(off, s2, np.array([5, 0, 2, 3, 4, 1], np.int32))
    for bad in ([5, 0, 3, 2, 4, 1], [1, 5, 0, 2, 3, 4], [5, 0, 2, 3, 1, 4]):
        with pytest.raises(AssertionError):
            check_order(off, s2, np.array(bad, np.int32))


def test_device_passes_and_sort_grid():
    G = GROUP_PAIRS
    assert device_passes(offsets([G])) == [(0, 1)]
    assert device_passes(offsets([0, 0])) == []
    assert device_passes(offsets([G - 5, 5, 0, 1])) == [(0, 3), (3, 4)]
    assert device_passes(offsets([3, G + 1, 0, 2])) == [(0, 1), (1, 2), (2, 4)]
    assert sort_grid(offsets([10] * 5), 0, 5, 132) == 5
    assert sort_grid(offsets([2048] * 2000), 0, 2000, 132) == 1056
    assert sort_grid(offsets([2049, 5]), 0, 2, 132) == 2
    assert sort_grid(offsets([1 << 21] + [3000] * 50), 0, 51, 132) == 10   # 256 MB / (2^21 * 12 bytes)
    assert sort_grid(offsets([G + 1]), 0, 1, 132) == 1
    assert expected_stats(offsets([3, 0, 2049, 7]), 7) == {"pairs": 2059, "chunks": 1 + 293 + 1, "passes": 1, "global_sorts": 1}


def test_pass_layout_reaches_its_boundaries():
    counts, marks = pass_layout(50)
    off = offsets(counts)
    P = device_passes(off)
    assert len(P) == 4 and 3.3 * GROUP_PAIRS < off[-1] < 3.7 * GROUP_PAIRS
    assert [u1 for _, u1 in P[:3]] == [marks[0] + 3, marks[1], marks[2]]
    assert off[marks[0] + 1] == GROUP_PAIRS and counts[marks[0] + 1:marks[0] + 3].tolist() == [0, 0]
    for (u0, u1), m in zip(P[1:3], marks[1:]):
        assert u0 < m == u1 and off[u1 + 1] - off[u0] == GROUP_PAIRS + 1     # the user that opens the next pass
        assert counts[m - 2:m].tolist() == [0, 0] and counts[m + 1:m + 3].tolist() == [0, 0]
    assert counts[0] == 0 and counts[-1] == 0
    nz = counts[counts > 0]
    assert (nz % 7 != 0).all() and (nz % 1024 != 0).all() and counts.max() <= SORT_SMEM
