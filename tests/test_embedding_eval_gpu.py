"""gorse_b200_embedding_eval on the device against the CPU restatement of `gorse-bench embedding`'s scoring
(embedding_oracle): the three averages and the number of users scored, bit for bit."""
import os

import numpy as np
import pytest

import embedding_oracle as eo

pytestmark = pytest.mark.gpu

ALL = 1 << 62


@pytest.fixture(scope="module")
def ctx(gb):
    c = gb.Context(0)
    yield c
    c.close()


def feedback(rng, n_users, n_items, mean_len, heavy=()):
    """a feedback CSR (distinct items per user, some users without feedback or with one item) and distinct timestamps"""
    lens = rng.poisson(mean_len, n_users)
    lens[rng.random(n_users) < 0.05] = 0
    lens[rng.random(n_users) < 0.05] = 1
    for u, n in heavy:
        lens[u] = n
    lens = np.minimum(lens, n_items)
    off = np.zeros(n_users + 1, np.int64)
    np.cumsum(lens, out=off[1:])
    items = np.concatenate([rng.choice(n_items, int(n), replace=False) for n in lens] + [np.zeros(0, np.int64)]).astype(np.int32)
    ts = rng.permutation(len(items))
    return (off, items), ts


def embeddings(rng, n_items, dim, p_missing=0.15):
    emb = rng.standard_normal((n_items, dim), dtype=np.float32)
    mask = (rng.random(n_items) >= p_missing).astype(np.uint8)
    return emb, mask


def problem(seed, n_users, n_items, dim, shots, mean_len=8, heavy=(), p_missing=0.15):
    rng = np.random.default_rng(seed)
    fb, ts = feedback(rng, n_users, n_items, mean_len, heavy)
    tr, te = eo.split_latest(fb[0], fb[1], ts, shots)
    emb, mask = embeddings(rng, n_items, dim, p_missing)
    return emb, mask, tr, te, fb


def check(gb, ctx, emb, mask, tr, te, fb, topk=10, seed=0, n_cand=99):
    got = gb.evaluate_embeddings(ctx, emb, mask, tr, te, fb, None, n_candidates=n_cand, seed=seed, topk=topk)
    negs = eo.sample_negatives(emb.shape[0], fb, te, n_cand, seed=seed)
    want = eo.evaluate(emb, mask, tr, te, negs, topk=topk)
    assert got[3] == want[3] and got[3] > 0
    assert [np.float32(x).tobytes() for x in got[:3]] == [np.float32(x).tobytes() for x in want[:3]], (got, want)
    return got


@pytest.mark.parametrize("shots", [1, 10, ALL])
@pytest.mark.parametrize("dim", [1, 15, 16, 17, 100, 768, 1536, 3072])
def test_matches_oracle(gb, ctx, dim, shots):
    n_users, n_items = (400, 1500) if dim <= 768 else (150, 800)
    check(gb, ctx, *problem(dim * 7 + (shots % 97), n_users, n_items, dim, shots, mean_len=12))


def test_heavy_users_span_many_ctas(gb, ctx):
    # users with more than 4,096 shots: their distances come from hundreds of CTAs, the totals still in shot order
    emb, mask, tr, te, fb = problem(5, 60, 9000, 64, ALL, heavy=[(3, 6000), (17, 4500)])
    assert np.diff(tr[0]).max() > 4096
    check(gb, ctx, emb, mask, tr, te, fb, topk=20)


def test_every_shot_quad_count(gb, ctx):
    # users with 1 .. 90 shots: 1 .. 23 shot quads, so a CTA's 16 micro-tiles span from 16 candidate quads and one shot quad
    # to two candidate quads and 16 shot quads; 0 .. 30 missing negatives move the candidate quads' padding
    rng = np.random.default_rng(12)
    n_items, dim = 3000, 20
    lens = np.arange(2, 92)
    off = np.zeros(len(lens) + 1, np.int64)
    np.cumsum(lens, out=off[1:])
    items = np.concatenate([rng.choice(n_items, n, replace=False) for n in lens]).astype(np.int32)
    fb = (off, items)
    tr, te = eo.split_latest(off, items, rng.permutation(len(items)), ALL)
    emb, mask = embeddings(rng, n_items, dim, p_missing=0.1)
    check(gb, ctx, emb, mask, tr, te, fb)
    check(gb, ctx, emb, None, tr, te, fb, topk=128)


def test_missing_embeddings_on_both_sides(gb, ctx):
    emb, mask, tr, te, fb = problem(6, 500, 400, 33, ALL, p_missing=0.6)
    check(gb, ctx, emb, mask, tr, te, fb)
    check(gb, ctx, emb, None, tr, te, fb)


def test_duplicate_shots(gb, ctx):
    emb, mask, tr, te, fb = problem(7, 300, 500, 48, 10)
    off, items = tr
    rng = np.random.default_rng(1)
    rows = [list(items[off[u]:off[u + 1]]) for u in range(len(off) - 1)]
    rows = [r + [r[i] for i in rng.integers(0, len(r), 3)] if r else r for r in rows]   # repeats inside the shot lists
    noff = np.zeros(len(rows) + 1, np.int64)
    np.cumsum([len(r) for r in rows], out=noff[1:])
    check(gb, ctx, emb, mask, (noff, np.array(sum(rows, []), np.int32)), te, fb)


@pytest.mark.parametrize("seed", range(6))
def test_ties_single_user(gb, ctx, seed):
    # one user per dataset, so the averages expose its ranked list; the items share a handful of embeddings, so totals tie
    rng = np.random.default_rng(100 + seed)
    n_items, dim = 60, 19
    base = rng.integers(-3, 4, (4, dim)).astype(np.float32)
    emb = base[rng.integers(0, 4, n_items)]
    items = rng.choice(n_items, 12, replace=False).astype(np.int32)
    fb = (np.array([0, 12], np.int64), items)
    tr, te = eo.split_latest(fb[0], fb[1], np.arange(12)[::-1], ALL)
    for topk in (1, 3, 10):
        check(gb, ctx, emb, None, tr, te, fb, topk=topk, n_cand=30)


def test_device_negatives_equal_the_oracle_sampler(gb, ctx):
    emb, mask, tr, te, fb = problem(8, 700, 300, 24, ALL, mean_len=40)   # dense rows: some users keep fewer than 99 items
    for seed in (0, 3):
        got = check(gb, ctx, emb, mask, tr, te, fb, seed=seed)
        negs = eo.sample_negatives(emb.shape[0], fb, te, 99, seed=seed)
        assert gb.evaluate_embeddings(ctx, emb, mask, tr, te, None, negs) == got


def test_chunks_and_split_calls(gb, ctx, monkeypatch):
    emb, mask, tr, te, fb = problem(9, 800, 1000, 40, ALL)
    one = gb.evaluate_embeddings(ctx, emb, mask, tr, te, fb)
    again = gb.evaluate_embeddings(ctx, emb, mask, tr, te, fb)
    assert [np.float32(x).tobytes() for x in one] == [np.float32(x).tobytes() for x in again]
    for cap in ("1", "5000"):
        monkeypatch.setenv("GORSE_B200_EMBEDDING_EVAL_CHUNK_PAIRS", cap)
        assert gb.evaluate_embeddings(ctx, emb, mask, tr, te, fb) == one
    monkeypatch.delenv("GORSE_B200_EMBEDDING_EVAL_CHUNK_PAIRS")
    # the same users over two calls (explicit negatives: each call draws its own streams): each half is the oracle's answer
    # on that half, and the halves' users add up
    negs = eo.sample_negatives(emb.shape[0], fb, te, 99)

    def part(c, a, b):
        off, items = c
        return off[a:b + 1] - off[a], items[off[a]:off[b]]

    users = 0
    for a, b in ((0, 350), (350, 800)):
        got = gb.evaluate_embeddings(ctx, emb, mask, part(tr, a, b), part(te, a, b), None, part(negs, a, b))
        want = eo.evaluate(emb, mask, part(tr, a, b), part(te, a, b), part(negs, a, b))
        assert got == want
        users += got[3]
    assert users == one[3]


def test_nan_embedding_is_an_argument_error(gb, ctx):
    emb, mask, tr, te, fb = problem(10, 50, 100, 16, ALL)
    bad = emb.copy()
    absent = int(np.flatnonzero(mask == 0)[0])
    bad[absent, 3] = np.nan   # a row without an embedding is never read
    gb.evaluate_embeddings(ctx, bad, mask, tr, te, fb)
    bad[int(np.flatnonzero(mask)[0]), 5] = np.nan
    with pytest.raises(gb.GorseB200Error) as ei:
        gb.evaluate_embeddings(ctx, bad, mask, tr, te, fb)
    assert ei.value.status == -1 and "non-finite" in ei.value.message
    bad[:, :] = emb
    bad[7, 0] = np.inf
    with pytest.raises(gb.GorseB200Error):
        gb.evaluate_embeddings(ctx, bad, None, tr, te, fb)


def test_planted_embeddings_beat_shuffled(gb, ctx):
    # each user's items come from one of 20 clusters and the embeddings sit near their cluster's centre
    rng = np.random.default_rng(11)
    n_users, n_items, dim, k = 600, 2000, 64, 20
    cluster = rng.integers(0, k, n_items)
    centres = rng.standard_normal((k, dim)).astype(np.float32) * 3
    emb = (centres[cluster] + rng.standard_normal((n_items, dim)).astype(np.float32)).astype(np.float32)
    members = [np.flatnonzero(cluster == c) for c in range(k)]
    rows = [rng.choice(members[rng.integers(0, k)], 8, replace=False) for _ in range(n_users)]
    off = np.arange(n_users + 1, dtype=np.int64) * 8
    fb = (off, np.concatenate(rows).astype(np.int32))
    tr, te = eo.split_latest(off, fb[1], rng.permutation(8 * n_users), ALL)
    planted = check(gb, ctx, emb, None, tr, te, fb)
    shuffled = check(gb, ctx, emb[rng.permutation(n_items)], None, tr, te, fb)
    assert planted[0] > shuffled[0] + 0.2
    assert os.environ.get("GORSE_B200_EMBEDDING_EVAL_CHUNK_PAIRS") is None
