#!/usr/bin/env python
"""tools/recommend_bench.py -- batched offline recommendation (gorse_b200_recommend) against the composed path.

  python tools/recommend_bench.py [--users N] [--composed-users M]

Data: synth.make_feedback(users, 100K items, 11 feedback per user, seed=1000) -- C2's shape when --users is 1M.  Factors
are seeded normals (not trained), the item-to-item collection holds them truncated to bf16 (Euclidean), the user-to-user
collection the user factors (Euclidean), the CF collection the item factors (Dot).  Stages: a 100-entry non-personalized
list, item-to-item (n = 100), user-to-user (n = 100), collaborative (n = 100), a 100-entry latest list; FM ranker k = 16
without slots; about 8 % of the items not live.  Users go in batches of --batch.

The first --composed-users users are run both ways -- the pipeline, and the four single-stage entries with the exclude sets
grown and the candidates merged and ranked in Python between them (tests/recommend_model.chain) -- and must agree bit for bit.
One JSON line: card (name, power limit, SM clock, read in the same run), pipeline wall time for all users (host in to host
out, median of 3), and both wall times on the composed subset (median of 3, after one warm-up call of the pipeline).  Both
include Python: the binding's packing of lists for the pipeline, and the set and list work of recommend_model.chain between
the entries for the composed path -- the composed figure is what a Python caller pays, not a bound on a Go worker.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from user_to_user_bench import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--users", type=int, default=1_000_000)
    ap.add_argument("--items", type=int, default=100_000)
    ap.add_argument("--batch", type=int, default=131072)
    ap.add_argument("--composed-users", type=int, default=4096)
    args = ap.parse_args()
    import fm_oracle
    import gorse_b200 as gb
    import recommend_model as rm
    from gorse_b200 import synth
    import types

    rng = np.random.default_rng(1000)
    U, I, d, n = args.users, args.items, 16, 100
    off, items = synth.make_feedback(U, I, 11 * U, seed=1000)
    E0 = [items[a:b].tolist() for a, b in zip(off[:-1], off[1:])]
    live = (rng.random(I) > 0.08).astype(np.uint8)
    P = rng.standard_normal((U, d)).astype(np.float32) * 0.3
    Q = rng.standard_normal((I, d)).astype(np.float32) * 0.3
    ident = np.arange(I, dtype=np.int64)
    with gb.Context(0) as ctx:
        cfc, i2c, u2c = gb.VectorCollection(ctx, d, gb.DISTANCE_DOT), gb.VectorCollection(ctx, d, gb.DISTANCE_EUCLIDEAN), gb.VectorCollection(ctx, d, gb.DISTANCE_EUCLIDEAN)
        cfc.add(values=Q)
        i2c.add(values=gb.bf16_truncate(Q))
        u2c.add(values=P)
        pop = (rng.choice(I, n, replace=False).astype(np.int32), np.sort(rng.random(n))[::-1].copy())
        latest = (rng.choice(I, n, replace=False).astype(np.int32), np.arange(n, 0, -1).astype(np.float64))
        fb = E0
        nf = U + I + 10
        params = fm_oracle.random_params(rng, nf, 16)
        inp = types.SimpleNamespace(n_users=U, n_items=I, user_feat=np.arange(U, dtype=np.int32), user_lab_off=np.zeros(U + 1, np.int64),
                                    user_lab_idx=np.zeros(1, np.int32), user_lab_val=np.zeros(1, np.float32),
                                    item_feat=np.arange(U, U + I, dtype=np.int32), item_lab_off=np.zeros(I + 1, np.int64),
                                    item_lab_idx=np.zeros(1, np.int32), item_lab_val=np.zeros(1, np.float32), item_emb=[], item_emb_mask=None)
        fm = gb.FMRanker(ctx, nf, 16, 2, 1024, (), params)

        def stages(a, b):
            ctxs = [E0[u][::-1] for u in range(a, b)]
            return [gb.ListStage(*pop), gb.ItemToItemStage(i2c, n, ctxs, ident, ident.astype(np.int32)),
                    gb.UserToUserStage(u2c, n, np.arange(a, b), fb), gb.CollaborativeStage(), gb.ListStage(*latest)]

        def sub(a, b):
            s = types.SimpleNamespace(**vars(inp))
            s.n_users, s.user_feat, s.user_lab_off = b - a, inp.user_feat[a:b].copy(), np.zeros(b - a + 1, np.int64)
            return s

        def run(a, b):
            return gb.recommend(ctx, E0[a:b], I, live, stages(a, b), cf=(cfc, P[a:b], ident, ident.astype(np.int32), n), ranker=(fm, sub(a, b)))

        # the composed subset: both ways, compared bit for bit
        m = min(args.composed_users, U)
        run(0, m)   # warm-up: the context's buffers and the library's first launches
        ts = []
        for _ in range(3):
            t0 = time.perf_counter()
            got, _ = run(0, m)
            ts.append(time.perf_counter() - t0)
        t_pipe_sub = float(np.median(ts))
        ctxs = [E0[u][::-1] for u in range(m)]

        def i2i(E):
            rows, _ = i2c.item_to_item(ctxs, [sorted(e) for e in E], n)
            return [[(int(s), float(v)) for s, v in zip(*r)] for r in rows]

        def u2u(E):
            rows, _ = u2c.user_to_user(np.arange(m), fb, [sorted(e) for e in E], n, I)
            return [[(int(i), float(v)) for i, v in zip(*r)] for r in rows]
        sin = sub(0, m)

        def rank(cands):
            s = types.SimpleNamespace(**vars(sin))
            s.cand_off = np.zeros(m + 1, np.int64)
            np.cumsum([len(c) for c in cands], out=s.cand_off[1:])
            s.cand_items = np.ascontiguousarray(np.concatenate([np.asarray(c, np.int32) for c in cands] + [np.zeros(1, np.int32)]))
            sc, _, _ = fm.rank(s)
            return [sc[a:b] for a, b in zip(s.cand_off[:-1], s.cand_off[1:])]
        ts = []
        for _ in range(3):
            t0 = time.perf_counter()
            cf_rows, _ = cfc.query_excluding(P[:m], [E0[u] for u in range(m)], n)
            cf_rows = [(s, sc.astype(np.float64)) for s, sc in cf_rows]
            want = rm.chain(E0[:m], live, [rm.list_stage(*pop), i2i, u2u, rm.collaborative_stage(cf_rows, live, n), rm.list_stage(*latest)],
                            rank=rank)
            ts.append(time.perf_counter() - t0)
        t_comp_sub = float(np.median(ts))
        for u, ((gi, gs), w) in enumerate(zip(got, want)):
            assert gi.tolist() == [i for i, _ in w] and gs.tobytes() == np.array([s for _, s in w], np.float64).tobytes(), f"user {u} differs"
        # every user, in batches, median of 3
        walls = []
        for _ in range(3):
            t0 = time.perf_counter()
            for a in range(0, U, args.batch):
                run(a, min(U, a + args.batch))
            walls.append(time.perf_counter() - t0)
        fm.close()
        for c in (cfc, i2c, u2c):
            c.close()
    print(json.dumps({"bench": "recommend", "card": card(), "users": U, "items": I, "batch": args.batch,
                      "pipeline_wall_s": float(np.median(walls)), "composed_check_users": m, "composed_subset_pipeline_s": t_pipe_sub,
                      "composed_subset_composed_s": t_comp_sub}))


if __name__ == "__main__":
    main()
