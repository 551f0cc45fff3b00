"""gorse_b200_fm_gauc against the CPU restatement: the predictions of the whole test list (fmo_batch_predict), then the
per-user AUC and GAUC (fmo_gauc), bit for bit -- without slots and with one and two, chunks that straddle users, rows
longer than num_dimension, tied predictions, a user above 2^24 pairs, empty and fully skipped inputs, NaN predictions, the
chunk coupling in test order, and repeated calls."""
import numpy as np
import pytest

import fm_oracle

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx(gb):
    with gb.Context(0) as c:
        yield c


def same(a, b):
    """bitwise, every NaN counting as one value"""
    a, b = np.array(a, np.float32), np.array(b, np.float32)
    a[np.isnan(a)] = np.nan
    b[np.isnan(b)] = np.nan
    return a.tobytes() == b.tobytes()


def gather(emb, rows):
    """per slot, the float32 embedding of every sample (zeros when it has none), as BatchInternalPredict receives them"""
    out = []
    for s, (t, d) in enumerate(zip(emb.table, emb.dims)):
        e = np.zeros((rows.size, d), np.float32)
        ok = rows >= 0
        if emb.mask is not None:
            ok &= emb.mask[np.maximum(rows, 0), s] > 0
        e[ok] = (t[rows[ok]].astype(np.uint32) << 16).view(np.float32)
        out.append(e)
    return out


def oracle_predict(nf, k, nd, bs, emb, params, te, which=None):
    off, idx, val, _ = te
    which = np.arange(off.size - 1) if which is None else which
    rows = [(idx[off[i]:off[i + 1]], val[off[i]:off[i + 1]]) for i in which]
    dims = () if emb is None else tuple(int(d) for d in emb.dims)
    es = gather(emb, emb.test_rows[which]) if emb is not None else ()
    return fm_oracle.Model(nf, k, nd, bs, dims, params).batch_predict(rows, es)


def problem(seed, n_users=40, nf=300, n_test=600, dims=(), ties=False, fb_max=5):
    rng = np.random.default_rng(seed)
    te = fm_oracle.random_ctr(rng, nf, n_test, n_ids=n_users)
    if ties:   # items and labels from three features with value 1: a user's rows repeat
        rest = np.ones(te[1].size, bool)
        rest[te[0][:-1]] = False
        te[1][rest] %= 3
        te[2][rest] = 1.0
    emb = fm_oracle.random_embeddings(rng, 30, dims, 0, n_test) if dims else None
    params = fm_oracle.random_params(rng, nf, 8, dims)
    fb = rng.integers(0, fb_max + 1, n_users).astype(np.int64)
    return te, emb, params, fb


def run(gb, ctx, nf, nd, bs, te, emb, params, n_users, fb, context_size=4, k=8):
    e = None if emb is None else (emb.dims, emb.table, emb.mask, emb.test_rows)
    return gb.ranker_gauc(ctx, nf, k, nd, params, te, n_users, fb, context_size, bs, e, predictions=True)


def check(gb, ctx, te, emb, params, fb, nf=300, nd=3, bs=1024, n_users=40, context_size=4):
    got = run(gb, ctx, nf, nd, bs, te, emb, params, n_users, fb, context_size)
    pred = oracle_predict(nf, 8, nd, bs, emb, params, te)
    assert same(got["predictions"], pred), "predictions"
    off, idx, _, tgt = te
    users = idx[off[:-1]]
    g, uo, co, ao = fm_oracle.gauc(pred, users, tgt, n_users, fb, context_size)
    assert got["users"].tolist() == uo.tolist() and got["candidates"].tolist() == co.tolist()
    assert got["feedback"].tolist() == fb[uo].tolist()
    assert same(got["auc"], ao), "per-user AUC"
    assert np.float64(got["gauc"]).tobytes() == np.float64(g).tobytes() or (np.isnan(g) and np.isnan(got["gauc"])), (got["gauc"], g)
    st = got["stats"]
    assert st["rows"] == off.size - 1 and st["users"] == np.unique(users).size and st["scored"] == uo.size
    assert st["nan"] == int(np.isnan(ao).sum())
    return got


@pytest.mark.parametrize("dims,bs", [((), 1024), ((), 5), ((16,), 5), ((16,), 64), ((16, 7), 5), ((16, 7), 64), ((7,), 1024)])
@pytest.mark.parametrize("ties", [False, True])
def test_matches_oracle(gb, ctx, dims, bs, ties):
    te, emb, params, fb = problem(1, dims=dims, ties=ties)
    got = check(gb, ctx, te, emb, params, fb, bs=bs)
    assert got["stats"]["scored"] > 5
    assert np.diff(te[0]).max() > 3   # rows longer than num_dimension
    if ties and not dims:   # slot-free rows that repeat predict the same value (with slots the chunk softmax may part them)
        off, idx, _, tgt = te
        u, p = idx[off[:-1]], got["predictions"]
        assert any(np.intersect1d(p[(u == x) & (tgt > 0)], p[(u == x) & (tgt <= 0)]).size for x in got["users"]), "no tie between a positive and a negative"


def test_user_above_2_24_pairs(gb, ctx):
    rng = np.random.default_rng(2)
    n_users, nf, P, N = 3, 50, 5000, 4999
    rows = [(u, t) for u, t in [(0, 1)] * P + [(0, -1)] * N + [(1, 1), (1, -1), (2, 1), (2, -1), (2, -1)]]
    order = rng.permutation(len(rows))
    rows = [rows[i] for i in order]
    off = np.arange(0, 2 * len(rows) + 1, 2, dtype=np.int64)
    idx = np.array([[u, n_users + rng.integers(0, nf - n_users)] for u, _ in rows], np.int32).reshape(-1)
    val = np.ones(idx.size, np.float32)
    te = (off, idx, val, np.array([t for _, t in rows], np.float32))
    params = fm_oracle.random_params(rng, nf, 8)
    got = check(gb, ctx, te, None, params, np.array([1, 1, 1], np.int64), nf=nf, n_users=n_users)
    assert got["stats"]["chained"] == 1 and got["users"].tolist() == [0, 1, 2]


def test_no_rows_and_every_user_skipped(gb, ctx):
    te, emb, params, fb = problem(3, dims=(16,))
    empty = (np.zeros(1, np.int64), np.zeros(0, np.int32), np.zeros(0, np.float32), np.zeros(0, np.float32))
    e0 = fm_oracle.Embeddings(emb.dims, emb.table, emb.mask, np.zeros(0, np.int32), np.zeros(0, np.int32))
    got = run(gb, ctx, 300, 3, 5, empty, e0, params, 40, fb)
    assert got["gauc"] == 0.0 and got["users"].size == 0 and got["predictions"].size == 0
    assert got["stats"] == dict(rows=0, users=0, scored=0, chained=0, nan=0)
    got = check(gb, ctx, te, emb, params, np.zeros(40, np.int64), bs=5)
    assert got["gauc"] == 0.0 and got["stats"]["scored"] == 0 and got["stats"]["users"] > 0


def test_nan_prediction(gb, ctx):
    te, _, params, fb = problem(4)
    off, idx, _, tgt = te
    fb[:] = 1
    bad = int(idx[off[0] + 1])   # the second feature of row 0: every row holding it predicts NaN
    params = params.copy()
    params[1 + 300 * 8 + bad] = np.nan
    got = check(gb, ctx, te, None, params, fb)
    assert got["stats"]["nan"] >= 1 and np.isnan(got["gauc"])


def test_slot_predictions_follow_test_order(gb, ctx):
    # the chunk softmax couples the rows of a chunk: the whole list in test order predicts other values than the fit's
    # evaluation, which predicts the positives and the negatives as two lists
    te, emb, params, fb = problem(5, dims=(16,))
    got = check(gb, ctx, te, emb, params, fb, bs=64)
    tgt = te[3]
    split = np.zeros(tgt.size, np.float32)
    for m in (tgt > 0, tgt <= 0):
        split[m] = oracle_predict(300, 8, 3, 64, emb, params, te, np.flatnonzero(m))
    assert not same(got["predictions"], split)


def test_repeated_calls_identical(gb, ctx):
    te, emb, params, fb = problem(6, dims=(16, 7))
    a = run(gb, ctx, 300, 3, 64, te, emb, params, 40, fb)
    b = run(gb, ctx, 300, 3, 64, te, emb, params, 40, fb)
    assert a["predictions"].tobytes() == b["predictions"].tobytes() and a["auc"].tobytes() == b["auc"].tobytes() and a["gauc"] == b["gauc"]
