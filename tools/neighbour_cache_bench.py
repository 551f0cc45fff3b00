#!/usr/bin/env python
"""tools/neighbour_cache_bench.py -- the neighbour cache of a collection (gorse_b200_vecdb_neighbour_cache) on the worker's
item-to-item pass and on one-session server calls, cache off against cache on, alternating in one process.

  python tools/neighbour_cache_bench.py [--small] [--session-calls-dense 1000] [--session-calls-sparse 200]
  python tools/neighbour_cache_bench.py --sha-only [--root TREE]   (cache off: SHA-256 of a seeded 50,000-user batch on the
                                                                   embedding collection, its vectors seeded normals in bf16)

Data: item_to_item_bench.py's C2 (synth.make_feedback(1M, 100K, 11M, seed=1000, exact=True) + leave_one_out(seed=1001)), its
two collections over the items ("users": sparse Dot, "embedding": dense Euclidean over 20 BPR epochs' item factors truncated to
bf16), context = each user's training row in a seeded order, exclusions = the same row, n = 100.

  worker    every user in batches of 131,072, one pass per arm, the arms alternating 3 times; the "on" arm sizes a fresh cache
            (rows = every item) before its pass, so each pass starts cold and later batches reuse the rows earlier ones
            computed.  wall_s: median and spread of the 3 passes; rows_computed_per_batch from the cache's counters;
            stage_a_device_ms from one torch.profiler pass per arm (every kernel but the stage-B aggregation); sha256 of
            each arm's answers (slots, score bits, counts of every user).
  sessions  one session per call (a REST request), drawn from the C2 rows (the first 20 items of a seeded user's row, no
            exclusions, context_size 100), per-call host latency: off, cold (the first pass with a fresh cache) and warm
            (the same calls again); p50 / p99.  The sparse collection takes ~0.3 s per uncached call, so it runs fewer calls.
The card's name and power limit are read in the same run, and per collection "clocks" holds the SM clock (median of
nvidia-smi samples every 50 ms) and any throttle reasons during the timed worker passes and the session passes (bench.py's
ClockSampler).  One JSON line on stdout.
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench import ClockSampler  # noqa: E402  (nvidia-smi sampled during the timed region)


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={q}", "--format=csv,noheader,nounits"], capture_output=True, text=True,
                         timeout=60).stdout.strip()
    name, power, sm, sm_max = [x.strip() for x in out.split(",")]
    return {"name": name, "power_limit_w": float(power), "sm_mhz": float(sm), "sm_max_mhz": float(sm_max)}


def log(msg):
    print(f"[neighbour_cache_bench] {msg}", file=sys.stderr, flush=True)


def spread(xs):
    return {"median": float(np.median(xs)), "min": float(np.min(xs)), "max": float(np.max(xs)), "samples": [float(x) for x in xs]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--small", action="store_true", help="20K users x 5K items (a rehearsal, not a measurement)")
    ap.add_argument("--n", type=int, default=100)
    ap.add_argument("--batch", type=int, default=131072)
    ap.add_argument("--epochs", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--session-calls-dense", type=int, default=1000)
    ap.add_argument("--session-calls-sparse", type=int, default=200)
    ap.add_argument("--sha-only", action="store_true", help="print the SHA-256 of a seeded 50,000-user batch, cache off, and stop")
    ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))), help="the tree whose package is timed")
    args = ap.parse_args()
    sys.path.insert(0, args.root)

    import gorse_b200 as gb
    from gorse_b200 import _lib, synth

    U, I, R, d = (20_000, 5_000, 200_000, 64) if args.small else (1_000_000, 100_000, 10_000_000, 64)
    n = args.n
    off0, items0 = synth.make_feedback(U, I, R + U, seed=1000, zipf_s=1.0, exact=True)
    (off, items), _ = synth.leave_one_out(off0, items0, seed=1001)
    lib = _lib.lib
    rng = np.random.default_rng(7)
    ctx_items = items.astype(np.int64).copy()
    for u in range(U):
        a, b = off[u], off[u + 1]
        ctx_items[a:b] = ctx_items[a:b][rng.permutation(b - a)]
    batches = [(b, min(b + args.batch, U)) for b in range(0, U, args.batch)]
    log(f"data: {U} users, {I} items, {int(off[-1])} training rows")
    result = {"metric": "neighbour cache: worker item-to-item pass and one-session calls, cache off vs on", "card": card(),
              "shape": {"users": U, "items": I, "n": n, "batch": args.batch, "context_entries": int(off[-1])}}
    with gb.Context(0) as ctx:
        if args.sha_only:   # seeded vectors: BPR's atomic epochs are not bit-reproducible from run to run
            Q = (np.random.default_rng(5).standard_normal((I, d)) * 0.1).astype(np.float32)
        else:
            with gb.CFModel(ctx, U, I, d, off, items) as m:
                m.init_normal(0.0, 0.001, 0)
                for e in range(args.epochs):
                    m.bpr_epoch(0.05, 0.01, int(off[-1]), 1000 + e)
                _, Q = m.get_factors()
        X = gb.bf16_truncate(Q)
        names = ("embedding",) if args.sha_only else ("embedding", "users")
        if "users" in names:
            ioff, iusers = gb.transpose_csr(off, items, I)
            freq = np.diff(off).astype(np.float64)
            idf = np.log(1 + I / np.maximum(freq, 1)).astype(np.float32)
            sp = [gb.sparse_vector(iusers[ioff[i]:ioff[i + 1]], idf) for i in range(I)]
        log("collections' data built")
        for name in names:
            dense = name == "embedding"
            with gb.VectorCollection(ctx, d if dense else 0, gb.DISTANCE_EUCLIDEAN if dense else gb.DISTANCE_DOT) as col:
                col.add(X) if dense else col.add(sparse=sp)
                cap = max(u1 - u0 for u0, u1 in batches) * n
                out = (np.zeros(cap, np.int64), np.zeros(cap, np.float64), np.zeros(U, np.int32))
                stats = np.zeros(4, np.int64)

                def run(u0, u1, h=None):
                    co = off[u0:u1 + 1] - off[u0]
                    cs = np.ascontiguousarray(ctx_items[off[u0]:off[u1]])
                    gb.check(lib.gorse_b200_vecdb_item_to_item(col.h, u1 - u0, gb.ptr(co), gb.ptr(cs), gb.ptr(co), gb.ptr(cs), None, 0, n, 1.0,
                                                               gb.ptr(out[0]), gb.ptr(out[1]), gb.ptr(out[2][u0:u1]), gb.ptr(stats)))
                    if h is not None:   # the answer: each row's first count entries (the rest of a row is unspecified)
                        cnt = out[2][u0:u1]
                        keep = np.arange(n)[None, :] < cnt[:, None]
                        k = (u1 - u0) * n
                        h.update(out[0][:k].reshape(-1, n)[keep].tobytes()); h.update(out[1][:k].reshape(-1, n)[keep].tobytes())
                        h.update(cnt.tobytes())

                if args.sha_only:
                    h = hashlib.sha256()
                    run(0, min(50_000, U), h)
                    print(json.dumps({"sha256_item_to_item_50000_users_cache_off": h.hexdigest(), "root": args.root}))
                    return

                def arm(on, h=None):
                    col.neighbour_cache(n, I if on else 0)
                    per_batch = []
                    t0 = time.perf_counter()
                    for u0, u1 in batches:
                        c0 = col.neighbour_cache_stats()["computed"]
                        run(u0, u1, h)
                        per_batch.append(col.neighbour_cache_stats()["computed"] - c0 if on else int(stats[0]))
                    return time.perf_counter() - t0, per_batch

                run(*batches[0])   # warm-up: mirror, work buffers, modules
                walls = {"off": [], "on": []}
                sha, computed = {}, {}
                clk = ClockSampler()
                t_w0 = time.time()
                for rep in range(args.reps):
                    for a in ("off", "on"):
                        h = hashlib.sha256() if rep == 0 else None
                        w, pb = arm(a == "on", h)
                        walls[a].append(w)
                        if h is not None:
                            sha[a], computed[a] = h.hexdigest(), pb
                    log(f"{name}: rep {rep}: off {walls['off'][-1]:.3f} s, on {walls['on'][-1]:.3f} s")
                clocks = {"worker": clk.stop(t_w0, time.time())}
                # stage A device time, one profiled pass per arm
                import torch
                from torch.profiler import ProfilerActivity, profile

                torch.cuda.init()
                dev = {}
                for a in ("off", "on"):
                    col.neighbour_cache(n, I if a == "on" else 0)
                    with profile(activities=[ProfilerActivity.CUDA]) as prof:
                        for u0, u1 in batches:
                            run(u0, u1)
                    t_a = 0.0
                    for e in prof.key_averages():
                        t = getattr(e, "device_time_total", 0.0) or getattr(e, "cuda_time_total", 0.0)
                        if "Memcpy" in e.key or "Memset" in e.key or not t or "i2i_aggregate_kernel" in e.key:
                            continue
                        t_a += t / 1e3
                    dev[a] = t_a
                # sessions: one per call
                calls = args.session_calls_dense if dense else args.session_calls_sparse
                srng = np.random.default_rng(11)
                sess = [ctx_items[off[u]:off[u + 1]][:20].tolist() for u in srng.choice(U, calls, replace=False)]
                lat = {}

                def session_pass(key):
                    ts = []
                    for s in sess:
                        t0 = time.perf_counter()
                        col.session_recommend([s], [[]], n, 100, n)
                        ts.append(time.perf_counter() - t0)
                    lat[key] = {"p50_ms": float(np.percentile(ts, 50) * 1e3), "p99_ms": float(np.percentile(ts, 99) * 1e3), "calls": len(ts)}

                col.neighbour_cache(n, 0)
                col.session_recommend([sess[0]], [[]], n, 100, n)   # warm-up
                clk = ClockSampler()
                t_s0 = time.time()
                session_pass("off")
                col.neighbour_cache(n, I)
                session_pass("cold")
                session_pass("warm")
                clocks["sessions"] = clk.stop(t_s0, time.time())
                result[name] = {
                    "wall_s": {a: spread(walls[a]) for a in walls},
                    "rows_computed_per_batch": computed,
                    "stage_a_device_ms": dev,
                    "sha256": sha, "answers_equal": sha["off"] == sha["on"],
                    "sessions": lat,
                    "clocks": clocks,
                    "cache": col.neighbour_cache_stats(),
                }
                log(f"{name}: {json.dumps(result[name])}")
    print(json.dumps(result))


if __name__ == "__main__":
    main()
