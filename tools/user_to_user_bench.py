#!/usr/bin/env python
"""tools/user_to_user_bench.py -- batched user-to-user recommendation (gorse_b200_vecdb_user_to_user) at C2 shapes.

  python tools/user_to_user_bench.py [--small]

Data: bench.py's c2 (synth.make_feedback(1M, 100K, 11M, seed=1000, exact=True) + leave_one_out(seed=1001)).  Two
user-to-user collections over the users, slot = user id:
  embedding  dense Euclidean, all 1M users: the user factors of 20 BPR epochs truncated to bf16 -- a stand-in for an
             embedding column
  items      sparse Dot, all users (--sparse-users takes the first ones): each user's training items with weights
             sqrt(log(1 + U / freq(i))) through gb.sparse_vector, as the "items" type builds them (logics/user_to_user.go,
             appendSparseVector).
Feedback = the training rows (item indices), exclusions = the user's own training row, about 8 % of the items have
item_ok = 0 (seeded), n = 100, users in batches of 131,072 as a worker would send its shard.  Before timing, a seeded sample
of users is checked against a restatement of recommendUserToUser over the oracle's brute force.

One JSON line, with per collection:
  card                 name, power limit and SM clock (nvidia-smi --query-gpu, read in the same run)
  wall_s / users_per_s all users, host in to host out, median of 3
  device_ms            stage A (neighbour table), routing and stage B (aggregation) device time, and the host-to-device
                       copies (the feedback rows are most of them), in one profiled pass (torch.profiler)
  stats                distinct query users over all batches, neighbour rows answered by the exact scan, users per accumulator
  per_user             today's path: one gorse_b200_vecdb_query(topK = n + 1) per user for the first 1,024 users (fewer if
                       they take more than a minute), and the all-user time it implies -- a LOWER BOUND: it leaves out the
                       feedback lookups, the shim's map and heap
"""
import argparse
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
    print(f"[user_to_user_bench] {msg}", file=sys.stderr, flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--small", action="store_true", help="20K users x 5K items (a rehearsal, not a measurement)")
    ap.add_argument("--n", type=int, default=100)
    ap.add_argument("--batch", type=int, default=131072)
    ap.add_argument("--epochs", type=int, default=20)
    ap.add_argument("--check", type=int, default=32, help="users per collection checked against the oracle")
    ap.add_argument("--per-user-users", type=int, default=1024)
    ap.add_argument("--sparse-users", type=int, default=None, help="the first users in the sparse collection (default: all)")
    args = ap.parse_args()

    import gorse_b200 as gb
    import oracle
    from gorse_b200 import _lib, synth

    U, I, R, d = (20_000, 5_000, 200_000, 64) if args.small else (1_000_000, 100_000, 10_000_000, 64)
    n = args.n
    off0, items0 = synth.make_feedback(U, I, R + U, seed=1000, zipf_s=1.0, exact=True)
    (off, items), _ = synth.leave_one_out(off0, items0, seed=1001)
    items = items.astype(np.int32)
    ex_all = items.astype(np.int64)
    item_ok = (np.random.default_rng(8).random(I) >= 0.08).astype(np.uint8)
    lib = _lib.lib
    records = {}
    log(f"data: {U} users, {I} items, {int(off[-1])} training rows")
    with gb.Context(0) as ctx:
        with gb.CFModel(ctx, U, I, d, off, items) as m:
            m.init_normal(0.0, 0.001, 0)
            for e in range(args.epochs):
                m.bpr_epoch(0.05, 0.01, int(off[-1]), 1000 + e)
            P, _ = m.get_factors()
        X = gb.bf16_truncate(P)
        log("model trained")
        Us = U if args.sparse_users is None else min(args.sparse_users, U)
        freq = np.bincount(items, minlength=I).astype(np.float64)
        idf = np.log(1 + U / np.maximum(freq, 1)).astype(np.float32)
        sp = [gb.sparse_vector(items[off[u]:off[u + 1]], idf) for u in range(Us)]
        sp_off = np.concatenate([[0], np.cumsum([len(v[0]) for v in sp])]).astype(np.int64)
        sp_ind = np.concatenate([v[0] for v in sp]).astype(np.uint32)
        sp_val = np.concatenate([v[1] for v in sp]).astype(np.float32)

        for name in ("embedding", "items"):
            dense = name == "embedding"
            NU = U if dense else Us
            batches = [(b, min(b + args.batch, NU)) for b in range(0, NU, args.batch)]
            col = gb.VectorCollection(ctx, d if dense else 0, gb.DISTANCE_EUCLIDEAN if dense else gb.DISTANCE_DOT)
            with col:
                col.add(X) if dense else col.add(sparse=sp)
                log(f"{name}: collection built ({NU} users)")
                cap = max(u1 - u0 for u0, u1 in batches) * n
                out = (np.zeros(cap, np.int64), np.zeros(cap, np.float64), np.zeros(NU, np.int32))
                stats = np.zeros(4, np.int64)
                fb_off = np.ascontiguousarray(off[:NU + 1], np.int64)
                fb_items = np.ascontiguousarray(items[:off[NU]])

                def run(u0, u1):
                    sl = np.arange(u0, u1, dtype=np.int64)
                    eo = off[u0:u1 + 1] - off[u0]
                    es = np.ascontiguousarray(ex_all[off[u0]:off[u1]])
                    gb.check(lib.gorse_b200_vecdb_user_to_user(col.h, u1 - u0, gb.ptr(sl), NU, gb.ptr(fb_off), gb.ptr(fb_items), I, gb.ptr(item_ok),
                                                               gb.ptr(eo), gb.ptr(es), n, 1.0, gb.ptr(out[0]), gb.ptr(out[1]),
                                                               gb.ptr(out[2][u0:u1]), gb.ptr(stats)))
                    return stats.copy()

                # ---- correctness first: seeded users against the restated recommender.  Neighbour lists are fetched
                # 4n deep and ordered (score desc, slot asc), the library's documented order of exact ties; a user whose cut
                # falls inside a tie group reaching the end of a fetched list cannot be restated this way and is skipped.
                sel = np.sort(np.random.default_rng(0).choice(NU, size=min(args.check, NU), replace=False))
                rows, _ = col.user_to_user(sel, [items[off[v]:off[v + 1]] for v in range(NU)], [ex_all[off[u]:off[u + 1]] for u in sel], n, I,
                                           item_ok=item_ok)
                kk, checked = 4 * n + 1, 0
                for (gs, gv), u in zip(rows, sel.tolist()):
                    if dense:
                        oi, od = oracle.bruteforce_search(X, X[u], kk, metric=oracle.METRIC_EUCLIDEAN)
                        sc = -od
                    else:
                        oi, sc = oracle.sparse_bruteforce_search(sp_off, sp_ind, sp_val, u, kk)
                    o = np.lexsort((oi, -sc))
                    oi, sc = oi[o], sc[o]
                    if not (len(oi) < kk or sc[min(n, len(sc) - 1)] != sc[-1] or (not dense and sc[min(n, len(sc) - 1)] <= 0)):
                        continue
                    ids, ss = oracle.similar_scores(dense, 1.0, u, n, oi, sc)
                    acc, drop = {}, set(ex_all[off[u]:off[u + 1]].tolist())
                    for v, s in zip(ids.tolist(), ss.tolist()):
                        for it in items[off[v]:off[v + 1]].tolist():
                            if it not in drop:
                                acc[it] = acc.get(it, 0.0) + s
                    best = [b for b in sorted(acc.items(), key=lambda t: (-t[1], t[0]))[:n] if item_ok[b[0]]]
                    want = np.array([b[1] for b in best], np.float64)
                    assert gv.tobytes() == want.tobytes(), f"{name} user {u}: scores differ from the oracle"
                    assert gs.tolist() == [b[0] for b in best] or len(set(want.tolist())) < len(want), f"{name} user {u}: items differ"
                    checked += 1
                log(f"{name}: {checked} of {len(sel)} sampled users match the oracle")

                # ---- all users, host in to host out
                t0 = time.perf_counter()
                run(*batches[0])   # warm-up: mirror, work buffers, modules
                log(f"{name}: warm-up batch in {time.perf_counter() - t0:.2f} s")
                walls, totals = [], np.zeros(4, np.int64)
                for rep in range(3):
                    t0, totals = time.perf_counter(), np.zeros(4, np.int64)
                    for b, (u0, u1) in enumerate(batches):
                        totals += run(u0, u1)
                        log(f"{name}: pass {rep}, batch {b} done at {time.perf_counter() - t0:.2f} s, stats so far {totals.tolist()}")
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
                log(f"{name}: profiled pass done")
                dev = {}
                for e in prof.key_averages():
                    t = getattr(e, "device_time_total", 0.0) or getattr(e, "cuda_time_total", 0.0)
                    if not t or "Memset" in e.key or "DtoH" in e.key:
                        continue
                    stage = ("htod" if "HtoD" in e.key else "route" if "u2u_route_kernel" in e.key else "B" if "u2u_aggregate_kernel" in e.key
                             else "A")
                    dev[stage] = dev.get(stage, 0.0) + t / 1e3

                # ---- today's path: one vecdb_query per user, lower bound
                nu = min(args.per_user_users, NU)
                s_, v_, c_ = np.zeros(n + 1, np.int64), np.zeros(n + 1, np.float32), np.zeros(1, np.int32)

                def query(u):
                    if dense:
                        st = lib.gorse_b200_vecdb_query(col.h, 1, gb.ptr(X[u]), None, None, None, 0, n + 1, gb.ptr(s_), gb.ptr(v_), gb.ptr(c_))
                    else:
                        qo = np.array([0, sp_off[u + 1] - sp_off[u]], np.int64)
                        st = lib.gorse_b200_vecdb_query(col.h, 1, gb.ptr(sp_val[sp_off[u]:sp_off[u + 1]]), gb.ptr(qo),
                                                        gb.ptr(sp_ind[sp_off[u]:sp_off[u + 1]]), None, 0, n + 1, gb.ptr(s_), gb.ptr(v_), gb.ptr(c_))
                    gb.check(st)

                query(0)   # warm-up
                t0 = time.perf_counter()
                for u in range(nu):   # the first nu users, or as many as 60 s allow
                    query(u)
                    if time.perf_counter() - t0 > 60:
                        nu = u + 1
                        break
                per_user_s = (time.perf_counter() - t0) / nu
                log(f"{name}: per-user path {per_user_s * 1e3:.2f} ms per user over {nu} users")

            records[name] = {
                "d": d if dense else 0, "users": NU,
                "checked_users": checked, "sampled_users": int(len(sel)),
                "wall_s": wall, "wall_s_all": walls, "users_per_s": NU / wall,
                "device_ms": {"stage_a": dev.get("A", 0.0), "routing": dev.get("route", 0.0), "stage_b": dev.get("B", 0.0),
                              "htod_copies": dev.get("htod", 0.0)},
                "feedback_bytes_per_call": int(fb_off.nbytes + fb_items.nbytes), "calls": len(batches),
                "stats": {"query_users_over_batches": int(totals[0]), "exact_rows": int(totals[1]), "shared_users": int(totals[2]),
                          "global_users": int(totals[3])},
                "per_user_lower_bound": {"users_timed": nu, "ms_per_user": per_user_s * 1e3, "implied_all_users_s": per_user_s * NU,
                                         "batched_speedup_at_least": per_user_s * NU / wall},
            }
    print(json.dumps({"metric": "batched user-to-user recommendation, users/s (host in to host out)", "card": card(),
                      "shape": {"users": U, "items": I, "n": n, "batch": args.batch, "feedback_entries": int(off[-1]), "bpr_epochs": args.epochs,
                                "small": args.small},
                      "collections": records}))


if __name__ == "__main__":
    main()
