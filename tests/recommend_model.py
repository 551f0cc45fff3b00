"""A per-user restatement of the worker's offline chaining (Pipeline.Recommend, worker/pipeline.go:124-319 with
Recommender.RecommendSequential, logics/recommend.go:135-156) in Python sets and lists, independent of the device.  The
stages are callables, so the same chaining runs over hand-built lists (test_recommend.py) and over the library's
single-stage entries (test_recommend_gpu.py)."""
import math

import numpy as np


def list_stage(items, scores):
    """non-personalized / latest: one list for every user, entries in E_u dropped"""
    return lambda E: [[(int(i), float(s)) for i, s in zip(items, scores) if int(i) not in e] for e in E]


def external_stage(rows):
    """external: one (items, scores) list per user, entries in E_u dropped"""
    return lambda E: [[(int(i), float(s)) for i, s in zip(*rows[u]) if int(i) not in e] for u, e in enumerate(E)]


def collaborative_stage(cf_rows, live, n):
    """the cached CF row: the non-hidden items, the first n (SearchScores(0, CacheSize)), then the filter"""
    def run(E):
        out = []
        for u, e in enumerate(E):
            shown = [(int(i), float(s)) for i, s in zip(*cf_rows[u]) if live[int(i)]][:n]
            out.append([(i, s) for i, s in shown if i not in e])
        return out
    return run


def score_key(s):
    """(descending score, NaN last, -0 == +0) as a sort key"""
    return (1, 0.0) if math.isnan(s) else (0, -s)


def chain(E0, live, stages, rank=None, replacement=None, positive_decay=1.0, read_decay=1.0):
    """-> per user [(item, score)].  E0[u]: item indices, -1 = outside the dictionary.  rank(cands) -> per user float32
    scores in candidate order (None: Ranker.Type = "none").  replacement[u]: [(item, positive)]."""
    E = [set(int(x) for x in e if x >= 0) for e in E0]
    merged = [[] for _ in E0]
    for st in stages:
        rows = st(E)
        for u, r in enumerate(rows):
            merged[u] += r
        for u, r in enumerate(rows):   # the exclude set grows only after the whole stage
            E[u] |= {i for i, _ in r}
    cands = [[(i, s) for i, s in m if live[i]] for m in merged]
    if rank is None:
        return cands
    flags = [{} for _ in E0]
    if replacement is not None:
        for u, rep in enumerate(replacement):
            have = {i for i, _ in cands[u]}
            for i, pos in rep:
                if live[i]:
                    flags[u][i] = bool(pos)
                    if i not in have:
                        cands[u].append((i, 0.0))
                        have.add(i)
    scores = rank([[i for i, _ in c] for c in cands])
    out = []
    for u, c in enumerate(cands):
        sc = []
        for p, (i, _) in enumerate(c):
            s = float(np.float32(scores[u][p]))
            if i in flags[u]:
                s = s * (positive_decay if flags[u][i] else read_decay)
            sc.append(s)
        order = sorted(range(len(c)), key=lambda p: (score_key(sc[p]), p))
        out.append([(c[p][0], sc[p]) for p in order])
    return out
