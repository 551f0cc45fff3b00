#!/usr/bin/env python
"""tools/recall_bench.py -- batched collaborative-filtering recall (gorse_b200_vecdb_query_excluding) at C2 shapes.

  python tools/recall_bench.py [--small]

Data: bench.py's c2 (synth.make_feedback(1M, 100K, 11M, seed=1000, exact=True) + leave_one_out(seed=1001)); model: 20 BPR
epochs through the library, so that seen items rank high as they do in production; collection: the hand-off
gorse_b200_vecdb_add_item_factors.  Queries are the user factors, exclusions the users' training rows as slots, n = 100, users
in batches of 131,072 as a worker would send its shard.  Before timing, 2,000 seeded users are checked against the oracle.

One JSON line:
  card                 name, power limit and SM clock (nvidia-smi --query-gpu, read in the same run)
  wall_s / users_per_s all users, host in to host out, median of 3
  stage1               device time of the tensor-core sweep kernels in one pass (torch.profiler), 2 * rows * N * d flop, and
                       the share of the H100 SXM data-sheet dense bf16 peak (989 TFLOP/s)
  rows                 users per k class (k = n + |E_u| <= 128 / 256 / 512, above) and rows answered by the exact scan
  per_user             gorse_b200_vecdb_query with nq = 1 and topK = n + |E_u| (the worker's path today) on the first 4,096
                       users, per user, and the whole-population time it implies
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

BF16_PEAK_TFLOPS = 989.0   # H100 SXM data sheet, dense


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={q}", "--format=csv,noheader,nounits"], capture_output=True, text=True,
                         timeout=60).stdout.strip()
    name, power, sm, sm_max = [x.strip() for x in out.split(",")]
    return {"name": name, "power_limit_w": float(power), "sm_mhz": float(sm), "sm_max_mhz": float(sm_max)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--small", action="store_true", help="50K users x 40K items (a rehearsal, not a measurement)")
    ap.add_argument("--n", type=int, default=100)
    ap.add_argument("--batch", type=int, default=131072)
    ap.add_argument("--epochs", type=int, default=20)
    ap.add_argument("--check", type=int, default=2000)
    ap.add_argument("--per-user", type=int, default=4096)
    args = ap.parse_args()

    import gorse_b200 as gb
    import oracle
    from gorse_b200 import _lib, synth

    U, I, R, d = (50_000, 40_000, 500_000, 64) if args.small else (1_000_000, 100_000, 10_000_000, 64)
    n = args.n
    off0, items0 = synth.make_feedback(U, I, R + U, seed=1000, zipf_s=1.0, exact=True)
    (off, items), _ = synth.leave_one_out(off0, items0, seed=1001)
    lib = _lib.lib
    with gb.Context(0) as ctx, gb.CFModel(ctx, U, I, d, off, items) as m, gb.VectorCollection(ctx, d, gb.DISTANCE_DOT) as col:
        m.init_normal(0.0, 0.001, 0)
        for e in range(args.epochs):
            m.bpr_epoch(0.05, 0.01, int(off[-1]), 1000 + e)
        slot = np.zeros(I, np.int64)
        gb.check(lib.gorse_b200_vecdb_add_item_factors(col.h, m.h, None, 0, None, None, gb.ptr(slot)))
        P, Q = m.get_factors()
        N = int((slot >= 0).sum())
        ex_all = slot[items]                     # every training item has feedback: all are slots
        k = n + np.diff(off)

        def recall(u0, u1, out):
            eo = off[u0:u1 + 1] - off[u0]
            ex = np.ascontiguousarray(ex_all[off[u0]:off[u1]])
            slots, scores, cnt = out
            exact = C.c_int64(0)
            gb.check(lib.gorse_b200_vecdb_query_excluding(col.h, u1 - u0, gb.ptr(P[u0:u1]), None, 0, n, gb.ptr(eo), gb.ptr(ex), gb.ptr(slots),
                                                          gb.ptr(scores), gb.ptr(cnt[u0:u1]), C.byref(exact)))
            return exact.value

        batches = [(b, min(b + args.batch, U)) for b in range(0, U, args.batch)]
        cap = max((u1 - u0) * n + int(off[u1] - off[u0]) for u0, u1 in batches)   # rows * n + |E| of the largest batch
        out = (np.zeros(cap, np.int64), np.zeros(cap, np.float32), np.zeros(U, np.int32))

        # ---- correctness first: seeded users against the oracle over the downloaded factors
        rng = np.random.default_rng(0)
        sel = np.sort(rng.choice(U, size=min(args.check, U), replace=False))
        X = np.zeros((N, d), np.float32)
        X[slot[slot >= 0]] = Q[slot >= 0]
        rows, _ = col.query_excluding(P[sel], [ex_all[off[u]:off[u + 1]] for u in sel], n)
        for (gs, gv), u in zip(rows, sel):
            oi, od = oracle.bruteforce_search(X, P[u], int(k[u]), metric=oracle.METRIC_NEG_DOT)
            keep = ~np.isin(oi, ex_all[off[u]:off[u + 1]])
            assert gv.tobytes() == (-od[keep]).astype(np.float32).tobytes(), f"user {u}: scores differ from the oracle"
            assert gs.tolist() == oi[keep].tolist() or len(set(od.tolist())) < len(od), f"user {u}: slots differ from the oracle"

        # ---- all users, host in to host out
        recall(*batches[0], out)   # warm-up: mirror, work buffers, modules
        walls, exact_rows = [], 0
        for rep in range(3):
            t0 = time.perf_counter()
            exact_rows = sum(recall(u0, u1, out) for u0, u1 in batches)
            walls.append(time.perf_counter() - t0)
        wall = float(np.median(walls))

        # ---- stage-1 device time in a separate, profiled pass
        import torch
        from torch.profiler import ProfilerActivity, profile

        torch.cuda.init()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for u0, u1 in batches:
                recall(u0, u1, out)
        s1_us = sum(getattr(e, "device_time_total", 0.0) or getattr(e, "cuda_time_total", 0.0)
                    for e in prof.key_averages() if "topk_mma_kernel" in e.key)
        swept = int((k <= 512).sum())
        flop = 2.0 * swept * N * d
        s1_ms = s1_us / 1e3

        # ---- the per-user path the worker takes today
        nu = min(args.per_user, U)
        kmax = int(k[:nu].max())
        s_, v_, c_ = np.zeros(kmax, np.int64), np.zeros(kmax, np.float32), np.zeros(1, np.int32)
        lib.gorse_b200_vecdb_query(col.h, 1, gb.ptr(P[0]), None, None, None, 0, int(k[0]), gb.ptr(s_), gb.ptr(v_), gb.ptr(c_))   # warm-up
        t0 = time.perf_counter()
        for u in range(nu):
            gb.check(lib.gorse_b200_vecdb_query(col.h, 1, gb.ptr(P[u]), None, None, None, 0, int(k[u]), gb.ptr(s_), gb.ptr(v_), gb.ptr(c_)))
        per_user_s = (time.perf_counter() - t0) / nu

    rec = {
        "metric": "batched CF recall, users/s (host in to host out)",
        "card": card(),
        "shape": {"users": U, "items_in_collection": N, "d": d, "n": n, "batch": args.batch, "bpr_epochs": args.epochs, "small": args.small},
        "checked_users": int(len(sel)),
        "wall_s": wall, "wall_s_all": walls, "users_per_s": U / wall,
        "stage1": {"device_ms": s1_ms, "flop": flop, "tflops": flop / (s1_ms * 1e-3) / 1e12 if s1_ms else None,
                   "bf16_peak_share": flop / (s1_ms * 1e-3) / 1e12 / BF16_PEAK_TFLOPS if s1_ms else None},
        "rows": {"k<=128": int((k <= 128).sum()), "k<=256": int(((k > 128) & (k <= 256)).sum()), "k<=512": int(((k > 256) & (k <= 512)).sum()),
                 "k>512": int((k > 512).sum()), "exact_path": int(exact_rows)},
        "per_user": {"users_timed": nu, "ms_per_user": per_user_s * 1e3, "implied_all_users_s": per_user_s * U,
                     "batched_speedup": per_user_s * U / wall},
    }
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
