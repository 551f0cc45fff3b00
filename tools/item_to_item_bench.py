#!/usr/bin/env python
"""tools/item_to_item_bench.py -- batched item-to-item recommendation (gorse_b200_vecdb_item_to_item) at C2 shapes.

  python tools/item_to_item_bench.py [--small]

Data: bench.py's c2 (synth.make_feedback(1M, 100K, 11M, seed=1000, exact=True) + leave_one_out(seed=1001)).  Two
item-to-item collections over the items, slot = item id:
  users      sparse Dot: each item's users with weights sqrt(log(1 + I / freq(u))) through gb.sparse_vector, as the "users"
             type builds them (logics/item_to_item.go, appendSparseVector)
  embedding  dense Euclidean: the item factors of 20 BPR epochs truncated to bf16 -- a stand-in for an embedding column
Context = each user's training row in a seeded order (the reference visits feedback newest first), exclusions = the same row,
n = 100, users in batches of 131,072 as a worker would send its shard.  Before timing, a seeded sample of users is checked
against a restatement of recommendItemToItem over the oracle's brute force (for the sparse collection, users whose context
items have at most 2,000 users each: the restatement's cost grows with the longest vector).

One JSON line, with per collection:
  card                 name, power limit and SM clock (nvidia-smi --query-gpu, read in the same run)
  wall_s / users_per_s all users, host in to host out, median of 3
  device_ms            stage A (neighbour table) and stage B (aggregation) device time in one profiled pass (torch.profiler)
  stats                distinct context items over all batches, neighbour rows answered by the exact scan, users per accumulator
  per_item             today's path: one gorse_b200_vecdb_query(topK = n + 1) per context item of the first 1,024 users (fewer
                       if they take more than a minute), per user, and the all-user time it implies -- a LOWER BOUND: it
                       leaves out the shim's map and heap
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={q}", "--format=csv,noheader,nounits"], capture_output=True, text=True,
                         timeout=60).stdout.strip()
    name, power, sm, sm_max = [x.strip() for x in out.split(",")]
    return {"name": name, "power_limit_w": float(power), "sm_mhz": float(sm), "sm_max_mhz": float(sm_max)}


def log(msg):
    print(f"[item_to_item_bench] {msg}", file=sys.stderr, flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--small", action="store_true", help="20K users x 5K items (a rehearsal, not a measurement)")
    ap.add_argument("--n", type=int, default=100)
    ap.add_argument("--batch", type=int, default=131072)
    ap.add_argument("--epochs", type=int, default=20)
    ap.add_argument("--check", type=int, default=64, help="users checked against the oracle (about a minute on the host)")
    ap.add_argument("--per-item-users", type=int, default=1024)
    args = ap.parse_args()

    import gorse_b200 as gb
    import oracle
    from gorse_b200 import _lib, synth

    U, I, R, d = (20_000, 5_000, 200_000, 64) if args.small else (1_000_000, 100_000, 10_000_000, 64)
    n = args.n
    off0, items0 = synth.make_feedback(U, I, R + U, seed=1000, zipf_s=1.0, exact=True)
    (off, items), _ = synth.leave_one_out(off0, items0, seed=1001)
    lib = _lib.lib
    rng = np.random.default_rng(7)
    # context: each training row in a seeded order
    ctx_items = items.astype(np.int64).copy()
    for u in range(U):
        a, b = off[u], off[u + 1]
        ctx_items[a:b] = ctx_items[a:b][rng.permutation(b - a)]
    batches = [(b, min(b + args.batch, U)) for b in range(0, U, args.batch)]
    records = {}
    log(f"data: {U} users, {I} items, {int(off[-1])} training rows")
    with gb.Context(0) as ctx:
        # ---- the collections
        with gb.CFModel(ctx, U, I, d, off, items) as m:
            m.init_normal(0.0, 0.001, 0)
            for e in range(args.epochs):
                m.bpr_epoch(0.05, 0.01, int(off[-1]), 1000 + e)
            _, Q = m.get_factors()
        X = gb.bf16_truncate(Q)
        log("model trained")
        ioff, iusers = gb.transpose_csr(off, items, I)
        freq = np.diff(off).astype(np.float64)
        idf = np.log(1 + I / np.maximum(freq, 1)).astype(np.float32)
        sp = [gb.sparse_vector(iusers[ioff[i]:ioff[i + 1]], idf) for i in range(I)]
        sp_off = np.concatenate([[0], np.cumsum([len(v[0]) for v in sp])]).astype(np.int64)
        sp_ind = np.concatenate([v[0] for v in sp]).astype(np.uint32)
        sp_val = np.concatenate([v[1] for v in sp]).astype(np.float32)

        for name in ("users", "embedding"):
            dense = name == "embedding"
            col = gb.VectorCollection(ctx, d if dense else 0, gb.DISTANCE_EUCLIDEAN if dense else gb.DISTANCE_DOT)
            with col:
                col.add(X) if dense else col.add(sparse=sp)
                log(f"{name}: collection built")
                cap = max(u1 - u0 for u0, u1 in batches) * n
                out = (np.zeros(cap, np.int64), np.zeros(cap, np.float64), np.zeros(U, np.int32))
                stats = np.zeros(4, np.int64)

                def run(u0, u1):
                    co = off[u0:u1 + 1] - off[u0]
                    cs = np.ascontiguousarray(ctx_items[off[u0]:off[u1]])
                    gb.check(lib.gorse_b200_vecdb_item_to_item(col.h, u1 - u0, gb.ptr(co), gb.ptr(cs), gb.ptr(co), gb.ptr(cs), None, 0, n, 1.0,
                                                               gb.ptr(out[0]), gb.ptr(out[1]), gb.ptr(out[2][u0:u1]), gb.ptr(stats)))
                    return stats.copy()

                # ---- correctness first: seeded users against the restated recommender
                # the sparse restatement merge-joins every stored vector per context item, which is prohibitive for the most
                # popular items (hundreds of thousands of users): the sample is drawn from users whose context items have at
                # most 2,000 users each
                light = np.ones(U, bool) if dense else np.array([np.diff(sp_off)[ctx_items[off[u]:off[u + 1]]].max(initial=0) <= 2000 for u in range(U)])
                sel = np.sort(np.random.default_rng(0).choice(np.nonzero(light)[0], size=min(args.check, int(light.sum())), replace=False))
                # The neighbour lists are fetched 4n deep and ordered (score desc, slot asc), the library's documented order
                # of exact ties (the reference's is its heap's); a user whose cut falls inside a tie group that reaches the
                # end of a fetched list cannot be restated this way and is skipped.
                rows, _ = col.item_to_item([ctx_items[off[u]:off[u + 1]] for u in sel], [ctx_items[off[u]:off[u + 1]] for u in sel], n)
                kk, checked = 4 * n + 1, 0
                for (gs, gv), u in zip(rows, sel):
                    acc, drop, ok = {}, set(ctx_items[off[u]:off[u + 1]].tolist()), True
                    for c in ctx_items[off[u]:off[u + 1]].tolist():
                        if dense:
                            oi, od = oracle.bruteforce_search(X, X[c], kk, metric=oracle.METRIC_EUCLIDEAN)
                            sc = -od
                        else:
                            oi, sc = oracle.sparse_bruteforce_search(sp_off, sp_ind, sp_val, c, kk)
                        o = np.lexsort((oi, -sc))
                        oi, sc = oi[o], sc[o]
                        ok &= len(oi) < kk or sc[min(n, len(sc) - 1)] != sc[-1] or (not dense and sc[min(n, len(sc) - 1)] <= 0)
                        ids, ss = oracle.similar_scores(dense, 1.0, c, n, oi, sc)
                        for j, s in zip(ids.tolist(), ss.tolist()):
                            if j not in drop:
                                acc[j] = acc.get(j, 0.0) + s
                    if not ok:
                        continue
                    checked += 1
                    best = sorted(acc.items(), key=lambda t: (-t[1], t[0]))[:n]
                    want = np.array([b[1] for b in best], np.float64)
                    assert gv.tobytes() == want.tobytes(), f"{name} user {u}: scores differ from the oracle"
                    assert gs.tolist() == [b[0] for b in best] or len(set(want.tolist())) < len(want), f"{name} user {u}: slots differ"

                log(f"{name}: {checked} of {len(sel)} sampled users match the oracle")
                # ---- all users, host in to host out
                run(*batches[0])   # warm-up: mirror, work buffers, modules
                walls, totals = [], np.zeros(4, np.int64)
                for rep in range(3):
                    t0 = time.perf_counter()
                    totals = sum(run(u0, u1) for u0, u1 in batches)
                    walls.append(time.perf_counter() - t0)
                wall = float(np.median(walls))

                log(f"{name}: all users in {walls} s")
                # ---- device time per stage in a separate, profiled pass
                import torch
                from torch.profiler import ProfilerActivity, profile

                torch.cuda.init()
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for u0, u1 in batches:
                        run(u0, u1)
                dev = {}
                for e in prof.key_averages():
                    t = getattr(e, "device_time_total", 0.0) or getattr(e, "cuda_time_total", 0.0)
                    if "Memcpy" in e.key or "Memset" in e.key or not t:
                        continue
                    stage = "B" if "i2i_aggregate_kernel" in e.key else "A"
                    dev[stage] = dev.get(stage, 0.0) + t / 1e3

                # ---- today's path: one vecdb_query per context item, lower bound
                nu = min(args.per_item_users, U)
                s_, v_, c_ = np.zeros(n + 1, np.int64), np.zeros(n + 1, np.float32), np.zeros(1, np.int32)

                def query(c):
                    if dense:
                        st = lib.gorse_b200_vecdb_query(col.h, 1, gb.ptr(X[c]), None, None, None, 0, n + 1, gb.ptr(s_), gb.ptr(v_), gb.ptr(c_))
                    else:
                        qo = np.array([0, sp_off[c + 1] - sp_off[c]], np.int64)
                        st = lib.gorse_b200_vecdb_query(col.h, 1, gb.ptr(sp_val[sp_off[c]:sp_off[c + 1]]), gb.ptr(qo),
                                                        gb.ptr(sp_ind[sp_off[c]:sp_off[c + 1]]), None, 0, n + 1, gb.ptr(s_), gb.ptr(v_), gb.ptr(c_))
                    gb.check(st)

                query(int(ctx_items[0]))   # warm-up
                t0 = time.perf_counter()
                for u in range(nu):   # the first nu users, or as many as 60 s allow
                    for c in ctx_items[off[u]:off[u + 1]].tolist():
                        query(c)
                    if time.perf_counter() - t0 > 60:
                        nu = u + 1
                        break
                per_user_s = (time.perf_counter() - t0) / nu
                log(f"{name}: per-item path {per_user_s * 1e3:.2f} ms per user over {nu} users")

            records[name] = {
                "d": d if dense else 0,
                "checked_users": checked, "sampled_users": int(len(sel)),
                "wall_s": wall, "wall_s_all": walls, "users_per_s": U / wall,
                "device_ms": {"stage_a": dev.get("A", 0.0), "stage_b": dev.get("B", 0.0)},
                "stats": {"context_items_over_batches": int(totals[0]), "exact_rows": int(totals[1]), "shared_users": int(totals[2]),
                          "global_users": int(totals[3])},
                "per_item_lower_bound": {"users_timed": nu, "queries": int(off[nu]), "ms_per_user": per_user_s * 1e3,
                                         "implied_all_users_s": per_user_s * U, "batched_speedup_at_least": per_user_s * U / wall},
            }
    print(json.dumps({"metric": "batched item-to-item recommendation, users/s (host in to host out)", "card": card(),
                      "shape": {"users": U, "items": I, "n": n, "batch": args.batch, "context_entries": int(off[-1]), "bpr_epochs": args.epochs,
                                "small": args.small},
                      "collections": records}))


if __name__ == "__main__":
    main()
