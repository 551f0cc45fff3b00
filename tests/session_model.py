"""The REST server's session recommendation (RestServer.sessionRecommend, server/rest.go:1069-1173) restated per session in
Python, independent of the device.  The neighbour query is a callable, so the same handler runs over hand-built lists
(test_session.py) and over the oracle's QueryItemToItem restatement of tests/test_item_to_item_gpu.py (test_session_gpu.py)."""
import numpy as np

from test_item_to_item_gpu import allow_mask


def session_rows(neighbours, contexts, excludes, context_size, top, item_ok=None):
    """neighbours(c) -> (slots, scores): QueryItemToItem(c, nil, n), empty for -1 and deleted slots.  Per session: visit the
    context in order, keep the neighbours with item_ok (FilterVisibleItemsByCategories), add the kept ones not in the
    exclude set in float64 (each sum starting at 0 + s), count the entry when its kept list is not empty and stop once the
    count reaches context_size; the first `top` sums by (score desc, slot asc)."""
    out = []
    for ctx, ex in zip(contexts, excludes):
        drop = set(int(x) for x in ex)
        acc, used = {}, 0
        for c in ctx:
            ids, scores = neighbours(int(c))
            kept = [(int(j), float(s)) for j, s in zip(ids, scores) if item_ok is None or item_ok[int(j)]]
            for j, s in kept:
                if j not in drop:
                    acc[j] = acc.get(j, 0.0) + s
            if kept:
                used += 1
                if used >= context_size:
                    break
        best = sorted(acc.items(), key=lambda t: (-t[1], t[0]))[:max(top, 0)]
        out.append((np.array([b[0] for b in best], np.int64), np.array([b[1] for b in best], np.float64)))
    return out


def oracle_neighbours(orc, store, hidden, dead, n, scale):
    """QueryItemToItem(c, nil, n) over the oracle's brute force (test_item_to_item_gpu's Dense / Sparse), memoised"""
    allow = allow_mask(hidden, dead, [()] * len(hidden))
    cache = {}

    def query(c):
        if c < 0 or dead[c]:
            return (), ()   # GetVectors finds nothing
        if c not in cache:
            cache[c] = store.neighbours(orc, c, allow, n, scale)
        return cache[c]
    return query
