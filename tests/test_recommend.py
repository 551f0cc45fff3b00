"""The chaining rules of the worker's offline recommendation, pinned on hand-built lists with the Python restatement
(recommend_model.chain) -- each rule shown to change the answer -- and gorse_b200_recommend's host-side argument checks,
which run before the device is touched."""
import numpy as np
import pytest

import recommend_model as rm

LIVE = np.ones(20, np.uint8)


def topn_stage(pool, n):
    """a recommender that ranks a fixed pool and keeps the first n outside E_u (as item-to-item / user-to-user do)"""
    return lambda E: [[(i, s) for i, s in pool if i not in e][:n] for e in E]


def test_exclude_set_grows_after_the_stage():
    ext = rm.external_stage([([5, 5, 6], [0.0, 0.0, 0.0])])
    out = rm.chain([[]], LIVE, [ext, rm.list_stage([5, 7], [1.0, 2.0])])
    assert [i for i, _ in out[0]] == [5, 5, 6, 7]   # the duplicate survives its stage, the later list drops 5
    ranked = rm.chain([[]], LIVE, [ext], rank=lambda c: [np.float32([0.1, 0.3, 0.2])])
    assert [i for i, _ in ranked[0]] == [5, 6, 5]   # ranked twice


def test_earlier_stage_moves_the_later_cut():
    pool = [(1, 0.9), (2, 0.8), (3, 0.7)]
    alone = rm.chain([[]], LIVE, [topn_stage(pool, 2)])
    after = rm.chain([[]], LIVE, [rm.list_stage([1], [5.0]), topn_stage(pool, 2)])
    assert [i for i, _ in alone[0]] == [1, 2]
    assert [i for i, _ in after[0]] == [1, 2, 3]   # the row's 2nd entry is now 3


def test_cf_row_is_cut_before_the_filter():
    row = [(np.array([2, 3, 4]), np.array([0.9, 0.8, 0.7]))]
    out = rm.chain([[]], LIVE, [rm.list_stage([2], [1.0]), rm.collaborative_stage(row, LIVE, 2)])
    assert [i for i, _ in out[0]] == [2, 3]   # the CF stage returns one item, not n = 2
    live = LIVE.copy()
    live[3] = 0
    out = rm.chain([[]], live, [rm.collaborative_stage(row, live, 2)])
    assert [i for i, _ in out[0]] == [2, 4]   # hidden items are skipped before the cut


def test_non_live_item_is_dropped_but_excludes():
    live = LIVE.copy()
    live[8] = 0
    out = rm.chain([[]], live, [rm.list_stage([8, 9], [1.0, 1.0]), rm.list_stage([8, 10], [2.0, 2.0])])
    assert [i for i, _ in out[0]] == [9, 10]
    both_live = rm.chain([[]], LIVE, [rm.list_stage([9], [1.0]), rm.list_stage([8, 10], [2.0, 2.0])])
    assert [i for i, _ in both_live[0]] == [9, 8, 10]


def test_replacement_only_when_live_and_new():
    live = LIVE.copy()
    live[4] = 0
    seen = []

    def rank(cands):
        seen.extend(cands)
        return [np.zeros(len(c), np.float32) for c in cands]

    rm.chain([[1, 2, 4]], live, [rm.list_stage([3], [1.0])], rank=rank, replacement=[[(3, 1), (4, 1), (2, 0)]])
    assert seen == [[3, 2]]   # 3 is a candidate already, 4 is not live


def test_decay_after_ranking_then_resort():
    rank = lambda c: [np.float32([0.5, 0.4, 0.3])]
    plain = rm.chain([[]], LIVE, [rm.list_stage([1, 2, 3], [0, 0, 0])], rank=rank)
    decayed = rm.chain([[]], LIVE, [rm.list_stage([1, 2, 3], [0, 0, 0])], rank=rank, replacement=[[(1, 1)]], positive_decay=0.5)
    assert [i for i, _ in plain[0]] == [1, 2, 3]
    assert [i for i, _ in decayed[0]] == [2, 3, 1]
    assert decayed[0][2][1] == float(np.float32(0.5)) * 0.5


def test_no_ranker_keeps_merged_order_without_replacement():
    out = rm.chain([[]], LIVE, [rm.list_stage([3, 1], [0.1, 0.9]), rm.list_stage([2], [5.0])])
    assert out == [[(3, 0.1), (1, 0.9), (2, 5.0)]]


def test_ties_by_position_and_nan_last():
    rank = lambda c: [np.float32([1.0, np.nan, 1.0, -0.0, 0.0])]
    out = rm.chain([[]], LIVE, [rm.list_stage([1, 2, 3, 4, 5], [0] * 5)], rank=rank)
    assert [i for i, _ in out[0]] == [1, 3, 4, 5, 2]


# ---- host-side argument checks: the context is checked last, so every case below fails with a NULL context before any
# pointer it would need is read, and names its own problem ------------------------------------------------------------------
@pytest.mark.parametrize("case,status,words", [("item_range", -1, "excluded item"), ("item_twice", -1, "excluded twice"),
                                               ("list_item", -1, "list entry"), ("list_nan", -1, "NaN"),
                                               ("cf_missing", -1, "CF inputs"), ("list_too_long", -7, "at most 4096"),
                                               ("valid", -1, "ctx is NULL")])
def test_argument_errors(gb, case, status, words):
    E0, stages = [[1, 2], [3]], [gb.ListStage(np.array([1, 4], np.int32), np.zeros(2))]
    if case == "item_range":
        E0 = [[1, 20], [3]]
    elif case == "item_twice":
        E0 = [[1, 1], [3]]
    elif case == "list_item":
        stages = [gb.ListStage(np.array([-1], np.int32), np.zeros(1))]
    elif case == "list_nan":
        stages = [gb.ListStage(np.array([1], np.int32), np.array([np.nan]))]
    elif case == "cf_missing":
        stages = [gb.CollaborativeStage()]
    elif case == "list_too_long":
        stages = [gb.ListStage(np.zeros(5000, np.int32), np.zeros(5000))]
    with pytest.raises(gb.GorseB200Error) as e:
        gb.recommend(None, E0, 20, LIVE, stages)
    assert e.value.status == status
    assert words in e.value.message, e.value.message


def test_no_cpu_fallback_without_a_device(gb):
    """Without a device no context can be made (GORSE_B200_ERR_CUDA), and the entry answers nothing without one: a
    well-formed call with a NULL context is refused rather than computed on the host."""
    import torch

    if torch.cuda.is_available():
        pytest.skip("a GPU is present; the loud-failure path is exercised on the CPU box")
    with pytest.raises(gb.GorseB200Error) as e:
        gb.Context(0)
    assert e.value.status == -2
    with pytest.raises(gb.GorseB200Error) as e:
        gb.recommend(None, [[1], [2]], 20, LIVE, [gb.ListStage(np.array([3], np.int32), np.ones(1))])
    assert e.value.status == -1 and "ctx is NULL" in e.value.message
