"""gorse_b200_fm_rank against the CPU restatement of the reference's FM inference (fm_oracle): bit-identical scores and
identical order, the chunk coupling of the softmax, padding, float32 indices, call splitting and argument errors."""
import ctypes as C

import numpy as np
import pytest

import fm_oracle

pytestmark = pytest.mark.gpu

COUNTS = [0, 1, 1023, 1024, 1025, 2500, 3, 40]


@pytest.fixture(scope="module")
def ctx(gb):
    with gb.Context(0) as c:
        yield c


def same(a, b):
    """bitwise, every NaN counting as one value (the device and the CPU propagate different NaN payloads)"""
    a, b = np.array(a, np.float32), np.array(b, np.float32)
    a[np.isnan(a)] = np.nan
    b[np.isnan(b)] = np.nan
    return a.tobytes() == b.tobytes()


def run_both(gb, ctx, nf, k, nd, bs, dims, params, inp):
    with gb.FMRanker(ctx, nf, k, nd, bs, dims, params) as fm:
        sg, og, stats = fm.rank(inp)
    so, oo = fm_oracle.Model(nf, k, nd, bs, dims, params).rank(inp)
    return sg, og, so, oo, stats


@pytest.mark.parametrize("k", [8, 16, 32])
@pytest.mark.parametrize("dims", [(), (32,), (64, 768)])
@pytest.mark.parametrize("bs", [1024, 7])
def test_matches_oracle(gb, ctx, k, dims, bs):
    rng = np.random.default_rng(k * 100 + len(dims) * 10 + (bs == 7))
    nf = 300
    params = fm_oracle.random_params(rng, nf, k, dims)
    inp = fm_oracle.random_input(rng, nf, COUNTS, 200, dims)
    nd = 3 if bs == 7 else 40   # below and above the longest row (at most 2 + 10 + 10 features)
    sg, og, so, oo, stats = run_both(gb, ctx, nf, k, nd, bs, dims, params, inp)
    assert same(sg, so)
    assert og.tolist() == oo.tolist()
    assert stats["pairs"] == sum(COUNTS)
    if dims:
        assert stats["chunks"] == sum(-(-c // bs) for c in COUNTS)
        rowwise, _ = fm_oracle.Model(nf, k, nd, bs, dims, params).rank(inp, coupled=False)
        assert not same(sg, rowwise), "the coupled softmax should be detectable"


def test_unknown_ids_no_labels_missing_embeddings_and_ties(gb, ctx):
    rng = np.random.default_rng(9)
    nf, k, dims = 50, 16, (32,)
    params = fm_oracle.random_params(rng, nf, k, dims)
    inp = fm_oracle.random_input(rng, nf, [30, 30, 12], 5, dims, labels=0, p_unknown=0.5, p_no_emb=0.6)
    inp.user_feat[:] = -1
    inp.item_feat[:2] = -1
    sg, og, so, oo, _ = run_both(gb, ctx, nf, k, 3, 1024, dims, params, inp)
    assert same(sg, so) and og.tolist() == oo.tolist()
    # without embeddings a repeated candidate is an exact tie, ordered by position
    params0 = fm_oracle.random_params(rng, nf, k)
    inp0 = fm_oracle.random_input(rng, nf, [60], 4)
    sg, og, so, oo, _ = run_both(gb, ctx, nf, k, 3, 1024, (), params0, inp0)
    assert same(sg, so) and og.tolist() == oo.tolist()
    assert len(set(sg.tolist())) < 60
    assert og.tolist() == sorted(range(60), key=lambda t: (-sg[t], t))


def test_index_above_2_24_rounds_through_float32(gb, ctx):
    rng = np.random.default_rng(7)
    nf, k = (1 << 24) + 8, 8
    params = fm_oracle.random_params(rng, nf, k)
    inp = fm_oracle.random_input(rng, 100, [5, 4], 3)
    big = np.array([(1 << 24) + 1, (1 << 24) + 3, (1 << 24) + 5, (1 << 24) + 6], np.int32)   # -> 2^24, +4, +4, +6
    inp.user_lab_idx[:inp.user_lab_off[-1]] = rng.choice(big, int(inp.user_lab_off[-1]))
    inp.item_feat[:] = big[:3]
    sg, og, so, oo, _ = run_both(gb, ctx, nf, k, 3, 1024, (), params, inp)
    assert same(sg, so) and og.tolist() == oo.tolist()
    # an index that rounds to n_features leaves the table
    inp.item_feat[0] = (1 << 24) + 7
    with gb.FMRanker(ctx, nf, k, 3, 1024, (), params) as fm:
        with pytest.raises(gb.GorseB200Error) as ei:
            fm.rank(inp)
    assert ei.value.status == gb._lib.ERR_ARG


def test_split_calls_and_repeats_give_the_same_bits(gb, ctx):
    rng = np.random.default_rng(12)
    nf, k, dims = 200, 16, (32,)
    params = fm_oracle.random_params(rng, nf, k, dims)
    counts = [int(c) for c in rng.integers(0, 300, 40)]
    inp = fm_oracle.random_input(rng, nf, counts, 150, dims)
    with gb.FMRanker(ctx, nf, k, 3, 64, dims, params) as fm:
        s1, o1, _ = fm.rank(inp)
        s2, o2, _ = fm.rank(inp)
        assert s1.tobytes() == s2.tobytes() and o1.tolist() == o2.tolist()
        parts = []
        for a, b in ((0, 13), (13, 14), (14, 40)):
            sub = fm_oracle.random_input(np.random.default_rng(0), nf, counts[a:b], 150, dims)
            for name in ("item_feat", "item_lab_off", "item_lab_idx", "item_lab_val", "item_emb", "item_emb_mask"):
                setattr(sub, name, getattr(inp, name))
            sub.user_feat = inp.user_feat[a:b].copy()
            lo, hi = inp.user_lab_off[a], inp.user_lab_off[b]
            sub.user_lab_off = (inp.user_lab_off[a:b + 1] - lo).astype(np.int64)
            sub.user_lab_idx = np.concatenate([inp.user_lab_idx[lo:hi], [0]]).astype(np.int32)
            sub.user_lab_val = np.concatenate([inp.user_lab_val[lo:hi], [0]]).astype(np.float32)
            c0, c1 = inp.cand_off[a], inp.cand_off[b]
            sub.cand_off = (inp.cand_off[a:b + 1] - c0).astype(np.int64)
            sub.cand_items = np.concatenate([inp.cand_items[c0:c1], [0]]).astype(np.int32)
            parts.append(fm.rank(sub)[:2])
    assert np.concatenate([p[0] for p in parts]).tobytes() == s1.tobytes()
    assert np.concatenate([p[1] for p in parts]).tolist() == o1.tolist()


def test_argument_errors(gb, ctx):
    from gorse_b200 import _lib

    rng = np.random.default_rng(13)
    nf, k, dims = 20, 8, (16,)
    params = fm_oracle.random_params(rng, nf, k, dims)
    h = C.c_void_p()
    dd = np.array(dims, np.int32)
    P = params.ctypes.data_as(C.c_void_p)
    create = _lib.lib.gorse_b200_fm_create
    assert create(ctx.h, nf, k, 3, 1024, 1, dd.ctypes.data_as(C.c_void_p), P, params.size - 1, C.byref(h)) == _lib.ERR_ARG   # n_params
    assert create(ctx.h, nf, k, 3, 0, 1, dd.ctypes.data_as(C.c_void_p), P, params.size, C.byref(h)) == _lib.ERR_ARG          # batch_size
    big = fm_oracle.random_params(rng, nf, 33)
    assert create(ctx.h, nf, 33, 3, 1024, 0, None, big.ctypes.data_as(C.c_void_p), big.size, C.byref(h)) == _lib.ERR_UNSUPPORTED
    wide = fm_oracle.random_params(rng, nf, k, (1025,))
    d2 = np.array([1025], np.int32)
    assert create(ctx.h, nf, k, 3, 1024, 1, d2.ctypes.data_as(C.c_void_p), wide.ctypes.data_as(C.c_void_p), wide.size,
                  C.byref(h)) == _lib.ERR_UNSUPPORTED
    with gb.FMRanker(ctx, nf, k, 3, 1024, dims, params) as fm:
        def bad(mutate):
            inp = fm_oracle.random_input(np.random.default_rng(1), nf, [4, 3], 6, dims)
            mutate(inp)
            with pytest.raises(gb.GorseB200Error) as ei:
                fm.rank(inp)
            assert ei.value.status == gb._lib.ERR_ARG

        bad(lambda i: i.user_feat.__setitem__(0, nf))
        bad(lambda i: i.user_feat.__setitem__(0, -2))
        bad(lambda i: i.item_feat.__setitem__(1, nf))
        bad(lambda i: i.user_lab_idx.__setitem__(slice(None), -1) if i.user_lab_off[-1] else i.item_lab_idx.__setitem__(slice(None), -1))
        bad(lambda i: i.item_lab_idx.__setitem__(slice(None), nf + 5))
        bad(lambda i: i.cand_items.__setitem__(0, 6))
        bad(lambda i: i.cand_items.__setitem__(0, -1))
        bad(lambda i: setattr(i, "cand_off", np.array([0, 5, 4], np.int64)))
        bad(lambda i: setattr(i, "user_lab_off", np.array([1] * 3, np.int64)))
        bad(lambda i: setattr(i, "item_emb", []))
        # the handle still answers after the rejected calls
        inp = fm_oracle.random_input(np.random.default_rng(1), nf, [4, 3], 6, dims)
        s, o, st = fm.rank(inp)
        assert st["pairs"] == 7
