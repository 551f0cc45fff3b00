"""The stage-1 error bound of the tensor-core sweep (csrc/topk_mma.cu) on inputs built to round adversarially.

The index search and the batched recall are exact only if, for every query row and every column, the bf16 stage-1 score is
within the row's eps of the exact score: the sample threshold, the certification and the re-rank window all assume it.
Gaussian data never comes near the bound, because rounding errors cancel.  Here they do not:

  q   = 1 + 2^-8 - 2^-20 on its first half (bf16 rounds it down, to 1) and 1 + 2^-8 + 2^-20 on its second half (rounds up)
  A   = q's round-down entries on the first half, 0 elsewhere: stage 1 UNDER-estimates q.A by about d 2^-8
  B   = q's round-up entries on the second half with one entry lowered to 1 - 2^-7: stage 1 OVER-estimates q.B by about as
        much, although q.B < q.A exactly

so a bound that covers the rounding of one operand only (1.02 2^-8 |q| max|x|) is exceeded about 1.4 times, and the A
columns, the true top 3, can fall out of the re-rank window of a certified row.  The CPU test checks these premises on the
very data sets the GPU tests use, in a numpy model of stage 1."""
import math

import numpy as np
import pytest

gpu = pytest.mark.gpu

N = 33000                      # >= 32768: the tensor path is eligible
U32 = np.float32(1 + 2**-8 + 2**-20)   # bf16 rounds it up, to 1 + 2^-7
D32 = np.float32(1 + 2**-8 - 2**-20)   # bf16 rounds it down, to 1
W32 = np.float32(1 - 2**-7)            # exact in bf16


@pytest.fixture(scope="module")
def ctx(gb):
    c = gb.Context(0)
    yield c
    c.close()


# ---- numpy model of stage 1 ------------------------------------------------------------------------------------------------
def bf16_round(x):
    u = np.asarray(x, np.float32).view(np.uint32).astype(np.uint64)
    u = (u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000
    return u.astype(np.uint32).view(np.float32)


def kp_of(d, euclid):
    return (d + 2 * euclid + 63) // 64 * 64


def approx(Q, X, euclid):
    """stage 1 in exact arithmetic: bf16 operands, exact sum (and the exact -|x|^2/2 for Euclidean)"""
    s = bf16_round(Q).astype(np.float64) @ bf16_round(X).astype(np.float64).T
    return s - 0.5 * (X.astype(np.float64) ** 2).sum(1)[None, :] if euclid else s


def exact(Q, X, euclid):
    s = Q.astype(np.float64) @ X.astype(np.float64).T
    return s - 0.5 * (X.astype(np.float64) ** 2).sum(1)[None, :] if euclid else s


def eps_old(Q, X, euclid):
    """the bound of the parent commit: one operand's bf16 rounding"""
    Q, X = Q.astype(np.float64), X.astype(np.float64)
    qn, M = np.linalg.norm(Q, axis=1), np.linalg.norm(X, axis=1).max()
    e = 1.02 * 2**-8 * qn * M
    return e + 6.2e-5 * (qn**2 + M**2) if euclid else e


def eps_new(Q, X, euclid):
    """build_queries_kernel's bound: |q^| max|x^ - x| + |q^ - q| max|x| + accumulation [+ Euclidean terms], padded"""
    Qh, Xh = bf16_round(Q).astype(np.float64), bf16_round(X).astype(np.float64)
    Q, X = Q.astype(np.float64), X.astype(np.float64)
    qh, dq = np.linalg.norm(Qh, axis=1), np.linalg.norm(Qh - Q, axis=1)
    M, dx = np.linalg.norm(X, axis=1).max(), np.linalg.norm(Xh - X, axis=1).max()
    kp = kp_of(X.shape[1], euclid)
    e = qh * dx + dq * M + kp * 2.0**-21 * qh * (M + dx)
    if euclid:
        e = e + (6 * kp + 64) * 2.0**-24 * ((Q**2).sum(1) + M**2)
    return 1.001 * e


# ---- the adversarial data sets -------------------------------------------------------------------------------------------
def pattern(d):
    h = d // 2
    q = np.full(d, U32, np.float32)
    q[:h] = D32
    a = np.zeros(d, np.float32)
    a[:h] = D32
    b = np.zeros(d, np.float32)
    b[h:] = U32
    b[h] = W32
    return q, a, b


def stage1_set(metric, d):
    """rows [0, 64): the query pattern at four power-of-two scales (a power of two keeps the rounding pattern); [64, 128):
    random rows; [128, 136) A, [136, 144) B; the rest random.  NEG_DOT: queries at 2^-10, so they cannot set max|x|.
    Euclidean: queries at 1 and A / B at 2, so that the dot term, not the norm term, dominates eps."""
    rng = np.random.default_rng(d + 7 * (metric == "euclid"))
    sq, sx = (1.0, 2.0) if metric == "euclid" else (2.0**-10, 1.0)
    q, a, b = pattern(d)
    X = (rng.standard_normal((N, d)) * 0.25).astype(np.float32)
    X[:64] = q[None, :] * (sq * 2.0 ** -(np.arange(64) % 4))[:, None]
    X[128:136] = a * sx
    X[136:144] = b * sx
    return X


def search_set(metric, d, k, n_b, stored_queries=False, seed=0):
    """3 A columns, n_b B columns (>= k: the k-th best approximate score is a B), 3000 filler columns spread over scores well
    below B (the sample's 16th best lands among them, so certification has room: fewer than 16 of A and B fall in the sample),
    the rest noise of norm 0.05.  Queries: the pattern at a few power-of-two scales (x4 for Euclidean, so that q.x and not the
    norm differences separates A from B).  stored_queries: rows [0, 64) hold them at 2^-10 (the all-pairs form)."""
    rng = np.random.default_rng(1000 * d + k + seed)
    q, a, b = pattern(d)
    X = rng.standard_normal((N, d)).astype(np.float32)
    X *= (0.05 / np.linalg.norm(X, axis=1, keepdims=True)).astype(np.float32)
    pos = rng.permutation(np.arange(64 if stored_queries else 0, N))
    a_idx, b_idx, f_idx = pos[:3], pos[3:3 + n_b], pos[3 + n_b:3 + n_b + 3000]
    X[a_idx] = a
    X[b_idx] = b
    # distinct B scores, 2^-13 apart (bf16-exact, 32 fp32 ulps): no exact ties for an exclusion list to split at the cut
    X[b_idx, 0] = -np.arange(n_b, dtype=np.float32) * np.float32(2.0**-13)
    X[f_idx] = rng.uniform(0.25, 0.4, (3000, 1)).astype(np.float32) * np.ones(d, np.float32)
    scales = np.full(64, 4.0) if metric == "euclid" else 2.0 ** -(np.arange(64) % 4 - 1.0)
    Q = (q[None, :] * scales[:, None]).astype(np.float32)
    if stored_queries:
        Q = (Q * np.float32(2.0**-10)).astype(np.float32)
        X[:64] = Q
    return X, Q, a_idx, b_idx


SEARCH_CASES = [(m, k) for m in ("negdot", "euclid") for k in (10, 100, 128)]


def n_b_for(k):
    return k + max(7, k // 10)


def recall_set(metric):
    X, Q, a_idx, b_idx = search_set(metric, 64, 270, 270, seed=1)
    return X, Q, a_idx, b_idx


def recall_rows(rng, nq, a_idx, b_idx, N_):
    """k = 100 + |E| in each class (<= 128, <= 256, <= 270 of 512); some rows exclude B slots, some an A slot"""
    rest = np.setdiff1d(np.arange(N_), np.concatenate([a_idx, b_idx]))
    excl = []
    for r in range(nq):
        m = [r % 29, 29 + (7 * r) % 127, 157 + r % 14][r % 3]
        e = []
        if r % 4 == 1:
            e.append(int(a_idx[r % 3]))
        if r % 4 >= 2:
            e.extend(int(s) for s in rng.choice(b_idx, size=min(m - len(e), 40), replace=False))
        e.extend(int(s) for s in rng.choice(rest, size=m - len(e), replace=False))
        excl.append(rng.permutation(np.array(e, np.int64)))
    return excl


def orc_metric(orc, metric):
    return orc.METRIC_EUCLIDEAN if metric == "euclid" else orc.METRIC_NEG_DOT


# ---- CPU: the premises ---------------------------------------------------------------------------------------------------
def check_gap(X, Q, a_idx, b_idx, k, euclid):
    """the k-th best B clears every A by more than 2 old eps (A leaves the parent's window) and by less than 2 new eps"""
    sa, sb = approx(Q, X[a_idx], euclid), approx(Q, X[b_idx], euclid)
    kth_b = -np.sort(-sb, axis=1)[:, k - 1]
    gap = kth_b - sa.max(1)
    eo, en = eps_old(Q, X, euclid), eps_new(Q, X, euclid)
    assert (gap > 2 * eo).all(), (gap / (2 * eo)).min()
    assert (gap < 2 * en).all(), (gap / (2 * en)).max()
    assert (exact(Q, X[b_idx], euclid).max(1) < exact(Q, X[a_idx], euclid).min(1)).all()


def test_premises_of_the_adversarial_sets(orc):
    # per column: A's stage-1 error exceeds the old eps and stays within the new one
    for metric, d in [("negdot", dd) for dd in (16, 40, 64, 128, 192)] + [("euclid", dd) for dd in (16, 64, 128, 190)]:
        eu = metric == "euclid"
        X = stage1_set(metric, d)
        Q = X[:64]
        err = np.abs(approx(Q, X[128:144], eu) - exact(Q, X[128:144], eu)).max(1)
        assert (err > eps_old(Q, X, eu)).all(), (metric, d, (err / eps_old(Q, X, eu)).min())
        assert (err < eps_new(Q, X, eu)).all(), (metric, d, (err / eps_new(Q, X, eu)).max())
    # end to end: A is the oracle's true top 3, and only the new eps keeps it in the window
    sets = [(m, search_set(m, 64, k, n_b_for(k)), k) for m, k in SEARCH_CASES]
    sets.append(("negdot", search_set("negdot", 64, 10, n_b_for(10), stored_queries=True), 10))
    sets += [(m, recall_set(m), k) for m in ("negdot", "euclid") for k in (100, 200, 270)]
    for metric, (X, Q, a_idx, b_idx), k in sets:
        eu = metric == "euclid"
        check_gap(X, Q, a_idx, b_idx, k, eu)
        for r in (0, 1, 2, 3):
            oi, _ = orc.bruteforce_search(X, Q[r], k, metric=orc_metric(orc, metric))
            assert set(a_idx.tolist()) <= set(oi[:3].tolist()), (metric, k, r)


# ---- GPU: the per-column bound -------------------------------------------------------------------------------------------
def report(msg):
    print(msg)


@gpu
@pytest.mark.parametrize("metric,d", [("negdot", d) for d in (16, 40, 64, 128, 192)] + [("euclid", d) for d in (16, 64, 128, 190)])
def test_stage1_error_within_eps_per_column(gb, ctx, metric, d):
    eu = metric == "euclid"
    X = stage1_set(metric, d)
    with gb.BruteforceIndex(ctx, d, gb.METRIC_EUCLIDEAN if eu else gb.METRIC_NEG_DOT) as ix:
        ix.add(X)
        got, eps = ix.stage1_scores(0, 128, with_eps=True)
    S = exact(X[:128], X, eu)
    ratio = np.abs(got.astype(np.float64) - S) / eps[:, None].astype(np.float64)
    rnd_cols = np.r_[64:128, 144:N]
    report(f"{metric} d={d}: max |stage1 - S| / eps = {ratio[:64].max():.3f} adversarial rows, "
           f"{ratio[64:128][:, rnd_cols].max():.3f} random rows x random columns")
    worst = np.unravel_index(np.argmax(ratio), ratio.shape)
    assert ratio.max() <= 1.0, f"row {worst[0]}, column {worst[1]}: |stage1 - S| = {ratio.max():.3f} eps"
    # the eps the kernel used is the bound derived in build_queries_kernel (what the CPU premises assume)
    np.testing.assert_allclose(eps, eps_new(X[:128], X, eu), rtol=1e-4)


# ---- GPU: the tensor core's fp32 accumulation ----------------------------------------------------------------------------
def cancelling_set(d, rng):
    """rows [0, 64): queries, [64, 128): one column per query with |x_i| ~ |q_i| (so sum|q^ x^| ~ |q^| |x^|) and exponents
    over 2^+-10 (products over 2^+-20).  Every product appears twice, with opposite signs, at random coordinates: the exact
    sum is 0 while the partial sums the tensor core forms are large.  The entries are bf16-exact, so every product is exact
    in fp32 and only the accumulation can err.  The rest: small noise."""
    X = (rng.standard_normal((N, d)) * 2.0**-12).astype(np.float32)
    h = d // 2
    for r in range(64):
        ex = rng.integers(-10, 11, h)
        q = (1 + rng.integers(0, 128, h) / 128.0) * 2.0**ex * rng.choice([-1.0, 1.0], h)
        x = (1 + rng.integers(0, 128, h) / 128.0) * 2.0**ex
        p = rng.permutation(d)
        X[r] = np.concatenate([q, q])[p]
        X[64 + r] = np.concatenate([x, -x])[p]
    return X


@gpu
@pytest.mark.parametrize("d", [64, 128, 192])
def test_tensor_core_accumulation_within_its_share(gb, ctx, d):
    rng = np.random.default_rng(d)
    X = cancelling_set(d, rng)
    assert (bf16_round(X[:128]) == X[:128]).all()
    with gb.BruteforceIndex(ctx, d, gb.METRIC_NEG_DOT) as ix:
        ix.add(X)
        got, eps = ix.stage1_scores(0, 64, with_eps=True)
    Xh = bf16_round(X).astype(np.float64)   # (the noise rows are not bf16-exact)
    want = Xh[:64] @ Xh.T                 # the exact products summed in float64 (off by ~2^-53 sum|q^ x^|)
    matched = np.arange(64)
    assert all(math.fsum(Xh[r] * Xh[64 + r]) == 0.0 for r in matched)   # they do cancel, exactly
    want[matched, 64 + matched] = 0.0
    absum = np.abs(Xh[:64]) @ np.abs(Xh).T
    err = np.abs(got.astype(np.float64) - want)
    # the share eps reserves for accumulation is Kp 2^-21 |q^| max|x^| >= Kp 2^-21 sum|q^_i x^_i|: assert the smaller one
    share = d * 2.0**-21 * absum
    report(f"Kp={d}: max accumulation error = {(err / (2.0**-24 * absum)).max():.2f} x 2^-24 sum|q^x^| "
           f"({(err / share).max():.4f} of the share); matched pairs {(err[matched, 64 + matched] / (2.0**-24 * absum[matched, 64 + matched])).max():.2f}")
    assert (err <= share).all(), (err / share).max()
    assert (err <= eps[:, None]).all()


# ---- GPU: end to end, index search ---------------------------------------------------------------------------------------
def assert_same_neighbours(idx, dist, oi, od):
    """as in test_topk_mma_gpu.py: distances bit-exact; ids identical except for the order of exact fp32 ties"""
    assert dist.tobytes() == od.tobytes()
    if idx.tolist() == oi.tolist():
        return
    last = od[-1]
    for v in np.unique(od):
        ours, theirs = set(idx[dist == v].tolist()), set(oi[od == v].tolist())
        if v < last:
            assert ours == theirs, (v, ours, theirs)
        else:
            assert len(ours) == len(theirs)


def assert_a_found(idx, a_idx):
    miss = [(r, sorted(set(a_idx.tolist()) - set(idx[r].tolist()))) for r in range(idx.shape[0])]
    miss = [(r, m) for r, m in miss if m]
    assert not miss, f"{len(miss)} of {idx.shape[0]} rows miss true top-3 columns, e.g. row {miss[0][0]} misses {miss[0][1]}"


@gpu
@pytest.mark.parametrize("metric,k", SEARCH_CASES)
def test_search_vectors_on_adversarial_rounding(gb, orc, ctx, metric, k):
    X, Q, a_idx, b_idx = search_set(metric, 64, k, n_b_for(k))
    with gb.BruteforceIndex(ctx, 64, gb.METRIC_EUCLIDEAN if metric == "euclid" else gb.METRIC_NEG_DOT) as ix:
        ix.add(X)
        idx, dist, cnt = ix.search_vectors(Q, k)
        fb = ix.stage1_stats()[2]
    assert fb == 0, f"{fb} of {len(Q)} rows fell back to the exact scan: no tensor-path row was checked"
    assert_a_found(idx, a_idx)
    for r in range(len(Q)):
        oi, od = orc.bruteforce_search(X, Q[r], k, metric=orc_metric(orc, metric))
        assert cnt[r] == len(oi)
        assert_same_neighbours(idx[r, :cnt[r]], dist[r, :cnt[r]], oi, od)


@gpu
def test_search_range_on_adversarial_rounding(gb, orc, ctx):
    k = 10
    X, Q, a_idx, b_idx = search_set("negdot", 64, k, n_b_for(k), stored_queries=True)
    with gb.BruteforceIndex(ctx, 64, gb.METRIC_NEG_DOT) as ix:
        ix.add(X)
        idx, dist, cnt = ix.search_range(0, 64, k)
        fb = ix.stage1_stats()[2]
    assert fb == 0, f"{fb} of 64 rows fell back to the exact scan"
    assert_a_found(idx, a_idx)
    oi, od, oc, _ = orc.bruteforce_all(X, 0, 64, k, metric=orc.METRIC_NEG_DOT, n_threads=8)
    assert cnt.tolist() == oc.tolist()
    for r in range(64):
        assert_same_neighbours(idx[r, :cnt[r]], dist[r, :cnt[r]], oi[r, :oc[r]], od[r, :oc[r]])


# ---- GPU: end to end, batched recall -------------------------------------------------------------------------------------
def expected(orc, X, allow, Q, excl, n, metric):
    """as in test_recall_gpu.py: the oracle's top n + |E_q| over the allowed rows, mapped back to slots, minus E_q"""
    ids = np.nonzero(allow)[0]
    Xa = np.ascontiguousarray(X[ids])
    out = []
    for q in range(Q.shape[0]):
        oi, od = orc.bruteforce_search(Xa, Q[q], n + len(excl[q]), metric=metric)
        drop = set(int(s) for s in excl[q])
        keep = np.array([int(ids[i]) not in drop for i in oi], bool)
        out.append((ids[oi][keep].astype(np.int64), (-od[keep]).astype(np.float32)))
    return out


def assert_rows_equal(got, want):
    """as in test_recall_gpu.py: scores bit-identical; slots identical except for the order of exact fp32 ties"""
    assert len(got) == len(want)
    for r, ((gs, gv), (ws, wv)) in enumerate(zip(got, want)):
        assert gv.tobytes() == wv.tobytes(), f"row {r}: scores differ"
        if gs.tolist() != ws.tolist():
            vals = np.unique(wv)
            for v in vals[1:]:
                assert set(gs[gv == v].tolist()) == set(ws[wv == v].tolist()), f"row {r}"


@gpu
@pytest.mark.parametrize("metric", ["negdot", "euclid"])
def test_recall_on_adversarial_rounding(gb, orc, ctx, metric):
    n, nq = 100, 96
    X, Q, a_idx, b_idx = recall_set(metric)
    Q = np.concatenate([Q, Q[:nq - len(Q)]])
    excl = recall_rows(np.random.default_rng(5), nq, a_idx, b_idx, N)
    ks = np.array([n + len(e) for e in excl])
    assert (ks <= 128).any() and ((ks > 128) & (ks <= 256)).any() and ((ks > 256) & (ks <= 512)).any() and ks.max() <= len(b_idx)
    with gb.VectorCollection(ctx, 64, gb.DISTANCE_EUCLIDEAN if metric == "euclid" else gb.DISTANCE_DOT) as col:
        col.add(X)
        rows, exact_rows = col.query_excluding(Q, excl, n)
    assert exact_rows == 0, f"{exact_rows} of {nq} rows went to the exact scan"
    a = set(a_idx.tolist())
    miss = [(r, sorted(a - set(s.tolist()) - set(excl[r].tolist()))) for r, (s, _) in enumerate(rows)]
    miss = [(r, m) for r, m in miss if m]
    assert not miss, f"{len(miss)} of {nq} rows miss true top-3 slots, e.g. row {miss[0][0]} (k = {ks[miss[0][0]]}) misses {miss[0][1]}"
    assert_rows_equal(rows, expected(orc, X, np.ones(N, bool), Q, excl, n, orc_metric(orc, metric)))
