"""The tensor-core sweep at embedding widths (192 < Kp <= 4096, csrc/topk_mma.cu, the WIDE kernel): every dense entry gives the
same slots and score bits as the exact kernel alone (GORSE_B200_TOPK_EXACT=1), the sweep really answers the rows, the
(score desc, slot asc) order holds at the cut on tie-heavy data, the stage-1 scores stay within eps column by column on
inputs built to round adversarially, and a mirror that cannot be allocated leaves the answers unchanged.  Above Kp = 4096
every row takes the exact kernel."""
import numpy as np
import pytest

from test_ties_gpu import GRID, dense_data, dense_scores, first_k
from test_topk_bound_gpu import bf16_round, cancelling_set, eps_new, exact, stage1_set

pytestmark = pytest.mark.gpu

N = 33000                                 # >= 32768 vectors: the sweep is eligible
NQ, NU = 96, 96                           # query rows and users: >= 64 rows per call
DIMS = (200, 256, 768, 1024, 1536, 3072, 4096)
ABOVE = 4160                              # d > 4096: the exact scan
CLASS_EXCL = (9, 120, 350, 480)           # with n = 40: k = n + |E| in each class (<= 128, <= 256, <= 512, above)


@pytest.fixture(scope="module")
def ctx(gb):
    c = gb.Context(0)
    yield c
    c.close()


def truncate(x):
    """bf16-exact values: the low 16 bits cleared"""
    return (np.ascontiguousarray(x, np.float32).view(np.uint32) & np.uint32(0xFFFF0000)).view(np.float32)


def make_data(dim, bf16, seed):
    """clustered rows (so that top scores sit close together) scaled to norm ~1; bf16: truncated to bf16-exact values"""
    rng = np.random.default_rng(seed)
    centres = rng.standard_normal((256, dim)).astype(np.float32)
    X = centres[rng.integers(0, 256, N)] + rng.standard_normal((N, dim)).astype(np.float32)
    X *= np.float32(1.0 / np.sqrt(2.0 * dim))
    X = truncate(X) if bf16 else X
    Q = X[rng.integers(0, N, NQ)] + np.float32(0.3 / np.sqrt(dim)) * rng.standard_normal((NQ, dim)).astype(np.float32)
    return np.ascontiguousarray(X), np.ascontiguousarray(Q.astype(np.float32))


def pick(rng, k, hi):
    s = rng.integers(0, hi, k)
    s[rng.random(k) > 0.95] = -1
    return s


def workload(rng, n_items):
    w = {}
    w["excl"] = [np.unique(rng.choice(N, CLASS_EXCL[r % 4], replace=False)) for r in range(NQ)]
    w["ctx"] = [pick(rng, int(rng.integers(1, 6)), N) for _ in range(NU)]
    w["ex"] = [np.unique(pick(rng, int(rng.integers(0, 8)), N)) for _ in range(NU)]
    w["users"] = rng.choice(N, NU, replace=False)
    w["fb"] = [rng.integers(0, n_items, int(rng.integers(0, 5))) for _ in range(N)]
    w["ex_items"] = [np.unique(pick(rng, int(rng.integers(0, 6)), n_items)) for _ in range(NU)]
    w["item_ok"] = (rng.random(n_items) > 0.1).astype(np.uint8)
    w["ctx_items"] = [pick(rng, int(rng.integers(1, 6)), n_items) for _ in range(NU)]
    w["soi"] = np.where(np.arange(n_items) < N, np.arange(n_items), -1).astype(np.int64)   # items past the slots have no vector
    w["ios"] = np.arange(N, dtype=np.int32)
    w["live"] = np.ones(n_items, np.uint8)
    return w


def rows_of(slots, scores, cnt):
    return [(slots[q, :c].copy(), scores[q, :c].copy()) for q, c in enumerate(cnt)]


def collection_answers(gb, ctx, col, Q, w, exact_rows):
    """every dense entry of a collection; exact_rows[name] = the rows its stats report the exact kernel answered"""
    out = {"query": rows_of(*col.query(Q, (), 20)), "query_categories": rows_of(*col.query(Q, (1,), 20))}
    out["query_excluding"], exact_rows["query_excluding"] = col.query_excluding(Q, w["excl"], 40)
    out["item_to_item"], st = col.item_to_item(w["ctx"], w["ex"], 10, categories=(0,))
    exact_rows["item_to_item"] = (st["exact_rows"], st["context_items"])
    out["session_recommend"], st = col.session_recommend(w["ctx"], w["ex"], 10, 3, 15)
    exact_rows["session_recommend"] = (st["exact_rows"], st["context_items"])
    out["user_to_user"], st = col.user_to_user(w["users"], w["fb"], w["ex_items"], 10, len(w["soi"]), w["item_ok"])
    exact_rows["user_to_user"] = (st["exact_rows"], st["query_users"])
    stages = [gb.ItemToItemStage(col, 10, w["ctx_items"], w["soi"], w["ios"]), gb.UserToUserStage(col, 10, w["users"], w["fb"], w["item_ok"])]
    out["recommend"], st = gb.recommend(ctx, w["ex_items"], len(w["soi"]), w["live"], stages)
    exact_rows["recommend"] = st["exact_rows"]
    return out


def index_answers(ix, Q):
    ix.stage1_stats()   # reset the counters
    out = {"search_vectors": ix.search_vectors(Q, 30), "search_indices": ix.search_indices(np.arange(5, 5 + NQ) * 311, 30),
           "search_range": ix.search_range(1000, 1000 + NQ, 30)}
    _, flop, fb = ix.stage1_stats()
    return out, flop, fb


def assert_same(a, b):
    assert a.keys() == b.keys()
    for name in a:
        if isinstance(a[name], tuple):   # the index's (ids, distances, counts)
            for x, y in zip(a[name], b[name]):
                assert x.tobytes() == y.tobytes(), name
            continue
        assert len(a[name]) == len(b[name]), name
        for r, ((s0, v0), (s1, v1)) in enumerate(zip(a[name], b[name])):
            assert np.array_equal(s0, s1), (name, r)   # the same slots in the same (tie) order
            assert np.asarray(v0).tobytes() == np.asarray(v1).tobytes(), (name, r)   # the same score bits


@pytest.mark.parametrize("bf16", [False, True], ids=["fp32", "bf16"])
@pytest.mark.parametrize("dist", ["DOT", "EUCLIDEAN"])
@pytest.mark.parametrize("dim", DIMS + (ABOVE,))
def test_every_dense_entry_same_on_both_paths(gb, orc, ctx, monkeypatch, dim, dist, bf16):
    euclid = dist == "EUCLIDEAN"
    swept = dim <= 4096
    X, Q = make_data(dim, bf16, seed=dim * 4 + 2 * euclid + bf16)
    rng = np.random.default_rng(dim)
    w = workload(rng, N + 20)
    meta = dict(hidden=rng.random(N) < 0.03, categories=[[c for c in range(3) if rng.random() < 0.5] for _ in range(N)])
    with gb.VectorCollection(ctx, dim, getattr(gb, "DISTANCE_" + dist)) as col, \
            gb.BruteforceIndex(ctx, dim, gb.METRIC_EUCLIDEAN if euclid else gb.METRIC_NEG_DOT) as ix:
        col.add(X, **meta)
        assert col.storage()[0] == (2 if bf16 else 4)
        ix.add(X)
        sweep_stats, exact_stats = {}, {}
        got = collection_answers(gb, ctx, col, Q, w, sweep_stats)
        got_ix, flop, fb = index_answers(ix, Q)
        monkeypatch.setenv("GORSE_B200_TOPK_EXACT", "1")
        want = collection_answers(gb, ctx, col, Q, w, exact_stats)
        want_ix, flop_exact, _ = index_answers(ix, Q)
        monkeypatch.delenv("GORSE_B200_TOPK_EXACT")
    assert_same(got, want)
    assert_same(got_ix, want_ix)
    assert flop_exact == 0
    assert exact_stats["query_excluding"] == NQ
    report = dict(sweep_stats, index_fallback=fb)
    print(f"d={dim} {dist} {'bf16' if bf16 else 'fp32'}: {report}")
    if swept:
        # the sweep answered the rows of small k.  query_excluding's rows of the 256 and 512 classes fail certification more
        # often as d grows (eps grows with Kp while these unit rows' scores crowd together; DESIGN 5.3), so there only some
        # row must have been swept.
        assert flop > 0 and fb <= NQ // 4, (flop, fb)
        assert sweep_stats["query_excluding"] < NQ
        for name in ("item_to_item", "session_recommend", "user_to_user"):
            ex, rows = sweep_stats[name]
            assert rows >= 64 and ex <= rows // 4, (name, ex, rows)
    else:
        assert flop == 0 and sweep_stats["query_excluding"] == NQ
        for name in ("item_to_item", "session_recommend", "user_to_user"):
            assert sweep_stats[name][0] == sweep_stats[name][1], name
    # a seeded sample against the oracle: distances bit-exact, ids equal up to the order of exact ties
    ids, dist_, cnt = got_ix["search_vectors"]
    for r in np.random.default_rng(dim + 1).choice(NQ, 3, replace=False):
        oi, od = orc.bruteforce_search(X, Q[r], 30, metric=orc.METRIC_EUCLIDEAN if euclid else orc.METRIC_NEG_DOT)
        assert cnt[r] == len(oi) and dist_[r, :cnt[r]].tobytes() == od.tobytes()
        for v in np.unique(od):
            assert sorted(ids[r, :cnt[r]][dist_[r, :cnt[r]] == v]) == sorted(oi[od == v]) or v == od[-1]


# ---- ties at the cut ------------------------------------------------------------------------------------------------------
TIE_K = (100, 128, 129, 256, 257, 512)


@pytest.mark.parametrize("euclid", [False, True], ids=["dot", "euclid"])
@pytest.mark.parametrize("dim", [1024, 4096])
def test_tie_order_at_the_cut(gb, ctx, dim, euclid):
    """grid-valued rows (every score exact, many ties) in copies; 2 100 copies of the queries' own best row make the first
    rows' top k one tie group wider than a candidate list (CAP = 2048), which the sweep hands to the exact kernel"""
    X, Q = dense_data(seed=11, n_base=8500, copies=4, d=dim, nq=64)
    X, Q = X.copy(), Q.copy()
    hot = np.full(dim, GRID[-1], np.float32)
    X[np.random.default_rng(12).choice(len(X), 2100, replace=False)] = hot
    Q[:8] = hot
    assert len(X) >= 32768
    S = dense_scores(Q, X, euclid)
    slots, allow = np.arange(len(X)), np.ones(len(X), bool)
    with gb.BruteforceIndex(ctx, dim, gb.METRIC_EUCLIDEAN if euclid else gb.METRIC_NEG_DOT) as ix:
        ix.add(X)
        for k in TIE_K:
            ids, dist, cnt = ix.search_vectors(Q, k)
            _, flop, fb = ix.stage1_stats()
            assert flop > 0   # the sweep ran (at d = 4096 the Euclidean rows' eps sends them on to the exact kernel)
            print(f"d={dim} {'euclid' if euclid else 'dot'} k={k}: {fb} of {len(Q)} rows to the exact kernel")
            ties = 0
            for r in range(len(Q)):
                ws, wv = first_k(S[r], slots, allow, (), -1, k)
                ties += len(wv) > 1 and wv[-1] == wv[-2]
                assert cnt[r] == k and np.array_equal(ids[r, :k], ws), (k, r)
                assert np.array_equal(-dist[r, :k], wv), (k, r)
            assert ties > 0, k   # the data does tie at the cut


# ---- the stage-1 bound -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("metric,d", [(m, d) for m in ("negdot", "euclid") for d in (256, 1024, 4096)])
def test_stage1_error_within_eps_per_column(gb, ctx, metric, d):
    """test_topk_bound_gpu.py's adversarial rounding pattern at the wide sweep's widths"""
    eu = metric == "euclid"
    X = stage1_set(metric, d)
    with gb.BruteforceIndex(ctx, d, gb.METRIC_EUCLIDEAN if eu else gb.METRIC_NEG_DOT) as ix:
        ix.add(X)
        got, eps = ix.stage1_scores(0, 128, with_eps=True)
    S = exact(X[:128], X, eu)
    ratio = np.abs(got.astype(np.float64) - S) / eps[:, None].astype(np.float64)
    print(f"{metric} d={d}: max |stage1 - S| / eps = {ratio[:64].max():.3f} adversarial rows, {ratio[64:128].max():.3f} random rows")
    worst = np.unravel_index(np.argmax(ratio), ratio.shape)
    assert ratio.max() <= 1.0, f"row {worst[0]}, column {worst[1]}: |stage1 - S| = {ratio.max():.3f} eps"
    np.testing.assert_allclose(eps, eps_new(X[:128], X, eu), rtol=1e-4)


@pytest.mark.parametrize("d", [256, 1024, 4096])
def test_tensor_core_accumulation_within_its_share(gb, ctx, d):
    """the accumulation share of eps (Kp 2^-21 |q^| max|x^|) over all Kp / 64 k-blocks of a tile, on sums that cancel"""
    rng = np.random.default_rng(d)
    X = cancelling_set(d, rng)
    with gb.BruteforceIndex(ctx, d, gb.METRIC_NEG_DOT) as ix:
        ix.add(X)
        got, eps = ix.stage1_scores(0, 64, with_eps=True)
    Xh = bf16_round(X).astype(np.float64)
    want = Xh[:64] @ Xh.T
    matched = np.arange(64)
    want[matched, 64 + matched] = 0.0
    absum = np.abs(Xh[:64]) @ np.abs(Xh).T
    err = np.abs(got.astype(np.float64) - want)
    share = d * 2.0**-21 * absum
    print(f"Kp={d}: max accumulation error = {(err / (2.0**-24 * absum)).max():.2f} x 2^-24 sum|q^x^|")
    assert (err <= share).all(), (err / share).max()
    assert (err <= eps[:, None]).all()


# ---- a mirror that cannot be allocated -------------------------------------------------------------------------------------
def test_mirror_allocation_failure_answers_exactly(gb, ctx, monkeypatch):
    dim = 1024
    X, Q = make_data(dim, True, seed=5)
    excl = [np.arange(r % 7, dtype=np.int64) for r in range(NQ)]
    with gb.VectorCollection(ctx, dim, gb.DISTANCE_DOT) as col, gb.BruteforceIndex(ctx, dim, gb.METRIC_NEG_DOT) as ix:
        col.add(X)
        ix.add(X)
        rows, ex = col.query_excluding(Q, excl, 30)
        ans = ix.search_vectors(Q, 30)
        assert ex < NQ and ix.stage1_stats()[1] > 0   # the sweep answered
        col2 = gb.VectorCollection(ctx, dim, gb.DISTANCE_DOT)
        ix2 = gb.BruteforceIndex(ctx, dim, gb.METRIC_NEG_DOT)
        try:
            col2.add(X)
            ix2.add(X)
            before = gb.device_bytes()
            monkeypatch.setenv("GORSE_B200_TOPK_MAX_MIRROR_BYTES", str(2 * N * dim - 1))   # one byte short
            rows2, ex2 = col2.query_excluding(Q, excl, 30)
            ans2 = ix2.search_vectors(Q, 30)
            assert ex2 == NQ and ix2.stage1_stats()[1] == 0   # every row took the exact kernel
            # no mirror is held (the exact path's own buffers grew)
            assert gb.device_bytes() - before < 2 * N * dim
            assert_same({"q": rows}, {"q": rows2})
            assert_same({"s": ans}, {"s": ans2})
            monkeypatch.delenv("GORSE_B200_TOPK_MAX_MIRROR_BYTES")
            rows3, ex3 = col2.query_excluding(Q, excl, 30)   # the next call builds the mirror
            assert ex3 < NQ
            assert_same({"q": rows}, {"q": rows3})
        finally:
            col2.close()
            ix2.close()
