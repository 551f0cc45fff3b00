#!/usr/bin/env python
"""tools/neighbour_share_bench.py -- neighbour caches shared between processes (gorse_b200_vecdb_neighbour_cache_fill,
_save and _load): what a fill, a save and a load cost, and what a loaded cache saves a worker and a server.

  python tools/neighbour_share_bench.py [--small] [--reps 3] [--n 100]

Collections (n = 100 neighbours per list):
  embedding   C2's dense Euclidean item collection: 100,000 x 64 seeded normals * 0.1, truncated to bf16 (stored in bf16)
  users       C2's sparse Dot item collection: each item's users with idf weights (synth.make_feedback(1M, 100K, 11M,
              seed=1000) + leave_one_out(seed=1001), as tools/neighbour_cache_bench.py)
  wide        200,000 x 1024 bf16 (seeded unit normals, truncated to bf16), Dot
  million     1,000,000 x 128 fp32 (seeded normals), Dot
Per collection, each median over --reps runs with min / max:
  fill        a freshly sized cache (rows = every vector) filled in one call: wall time and the call's device time
  stream      the saved stream's bytes; save into memory and load from memory into a freshly sized cache (wall times)
  sha256      of the stream of every rep: equal when fills are deterministic
C2 collections also:
  worker      the item-to-item pass over every user in batches of 131,072 (context = each user's training row in a seeded
              order, exclusions = the same row): cold (a freshly sized cache) against loaded (the same, then the saved
              stream loaded), the arms alternating; sha256 of each arm's answers from one more pass per arm, not timed
  session     the first one-session call after a reload: the collection restored from its snapshot, the cache sized, then
              one session call of 20 context items, cold or after the stream is loaded (the load timed apart); the same
              session in every rep; sha256 of each arm's answers
The card's name, power limit and SM clock are read in the same run.  One JSON line on stdout.
"""
import argparse
import hashlib
import io
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={q}", "--format=csv,noheader,nounits"], capture_output=True, text=True,
                         timeout=60).stdout.strip()
    name, power, sm, sm_max = [x.strip() for x in out.split(",")]
    return {"name": name, "power_limit_w": float(power), "sm_mhz": float(sm), "sm_max_mhz": float(sm_max)}


def log(msg):
    print(f"[neighbour_share_bench] {msg}", file=sys.stderr, flush=True)


def spread(xs):
    return {"median": float(np.median(xs)), "min": float(np.min(xs)), "max": float(np.max(xs)), "samples": [float(x) for x in xs]}


def timed(f):
    t0 = time.perf_counter()
    r = f()
    return time.perf_counter() - t0, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--small", action="store_true", help="small shapes (a rehearsal, not a measurement)")
    ap.add_argument("--n", type=int, default=100)
    ap.add_argument("--batch", type=int, default=131072)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()

    import gorse_b200 as gb
    from gorse_b200 import _lib, synth

    lib = _lib.lib
    n = args.n
    U, I, R = (20_000, 5_000, 200_000) if args.small else (1_000_000, 100_000, 10_000_000)
    wide_rows, million_rows = (5_000, 40_000) if args.small else (200_000, 1_000_000)
    off0, items0 = synth.make_feedback(U, I, R + U, seed=1000, zipf_s=1.0, exact=True)
    (off, items), _ = synth.leave_one_out(off0, items0, seed=1001)
    rng = np.random.default_rng(7)
    ctx_items = items.astype(np.int64).copy()
    for u in range(U):
        a, b = off[u], off[u + 1]
        ctx_items[a:b] = ctx_items[a:b][rng.permutation(b - a)]
    batches = [(b, min(b + args.batch, U)) for b in range(0, U, args.batch)]
    result = {"metric": "neighbour caches shared between processes: fill, save, load, and a loaded cache against a cold one",
              "card": card(), "n": n, "shape": {"users": U, "items": I, "context_entries": int(off[-1]), "batch": args.batch}}

    def collections(ctx):
        yield "embedding", (lambda c: c.add(gb.bf16_truncate((np.random.default_rng(5).standard_normal((I, 64)) * 0.1).astype(np.float32)))), \
            64, gb.DISTANCE_EUCLIDEAN
        ioff, iusers = gb.transpose_csr(off, items, I)
        idf = np.log(1 + I / np.maximum(np.diff(off).astype(np.float64), 1)).astype(np.float32)
        sp = [gb.sparse_vector(iusers[ioff[i]:ioff[i + 1]], idf) for i in range(I)]
        yield "users", (lambda c: c.add(sparse=sp)), 0, gb.DISTANCE_DOT

        def wide(c):
            for i in range(0, wide_rows, 20_000):
                x = np.random.default_rng(100 + i).standard_normal((min(20_000, wide_rows - i), 1024)).astype(np.float32)
                c.add(gb.bf16_truncate(x / np.linalg.norm(x, axis=1, keepdims=True)))
        yield "wide", wide, 1024, gb.DISTANCE_DOT

        def million(c):
            for i in range(0, million_rows, 100_000):
                c.add(np.random.default_rng(200 + i).standard_normal((min(100_000, million_rows - i), 128)).astype(np.float32))
        yield "million", million, 128, gb.DISTANCE_DOT

    with gb.Context(0) as ctx:
        for name, fill_data, dim, dist in collections(ctx):
            with gb.VectorCollection(ctx, dim, dist) as col:
                fill_data(col)
                rows = col.count()[0]
                log(f"{name}: {rows} vectors, storage {col.storage()}")
                res = {"vectors": rows, "value_bytes": col.storage()[0]}
                fill_wall, fill_dev, save_s, load_s, shas = [], [], [], [], []
                data = b""
                for rep in range(args.reps):
                    col.neighbour_cache(n, 0)
                    col.neighbour_cache(n, rows)
                    w, st = timed(col.neighbour_cache_fill)
                    assert st["computed"] == rows and st["left_out"] == 0, st
                    fill_wall.append(w)
                    fill_dev.append(st["device_us"] / 1e6)
                    buf = io.BytesIO()
                    w, nbytes = timed(lambda: col.save_neighbour_cache(buf))
                    save_s.append(w)
                    data = buf.getvalue()
                    shas.append(hashlib.sha256(data).hexdigest())
                    col.neighbour_cache(n, 0)
                    col.neighbour_cache(n, rows)
                    w, ld = timed(lambda: col.load_neighbour_cache(io.BytesIO(data)))
                    assert ld == {"loaded": rows, "dropped": 0, "bytes": len(data)}, ld
                    load_s.append(w)
                    log(f"{name}: rep {rep}: fill {fill_wall[-1]:.3f} s (device {fill_dev[-1]:.3f} s), {len(data)} bytes, "
                        f"save {save_s[-1]:.3f} s, load {load_s[-1]:.3f} s")
                res.update({"fill_wall_s": spread(fill_wall), "fill_device_s": spread(fill_dev), "stream_bytes": len(data),
                            "save_s": spread(save_s), "load_s": spread(load_s), "stream_sha256": shas,
                            "streams_equal": len(set(shas)) == 1})
                if name in ("embedding", "users"):
                    cap = max(u1 - u0 for u0, u1 in batches) * n
                    out = (np.zeros(cap, np.int64), np.zeros(cap, np.float64), np.zeros(U, np.int32))
                    stats = np.zeros(4, np.int64)

                    def run(u0, u1, h):
                        co = off[u0:u1 + 1] - off[u0]
                        cs = np.ascontiguousarray(ctx_items[off[u0]:off[u1]])
                        gb.check(lib.gorse_b200_vecdb_item_to_item(col.h, u1 - u0, gb.ptr(co), gb.ptr(cs), gb.ptr(co), gb.ptr(cs), None, 0, n, 1.0,
                                                                   gb.ptr(out[0]), gb.ptr(out[1]), gb.ptr(out[2][u0:u1]), gb.ptr(stats)))
                        if h is None:
                            return
                        cnt = out[2][u0:u1]
                        keep = np.arange(n)[None, :] < cnt[:, None]
                        k = (u1 - u0) * n
                        h.update(out[0][:k].reshape(-1, n)[keep].tobytes()); h.update(out[1][:k].reshape(-1, n)[keep].tobytes())
                        h.update(cnt.tobytes())

                    def worker(loaded, h=None):
                        col.neighbour_cache(n, 0)
                        col.neighbour_cache(n, rows)
                        if loaded:
                            col.load_neighbour_cache(io.BytesIO(data))
                        c0 = col.neighbour_cache_stats()["computed"]
                        t0 = time.perf_counter()
                        for u0, u1 in batches:
                            run(u0, u1, h)
                        return time.perf_counter() - t0, col.neighbour_cache_stats()["computed"] - c0

                    worker(False)   # warm-up: mirror, work buffers, modules
                    walls, wsha, wcomp = {"cold": [], "loaded": []}, {}, {}
                    for rep in range(args.reps):
                        for arm in ("cold", "loaded"):
                            w, wcomp[arm] = worker(arm == "loaded")
                            walls[arm].append(w)
                        log(f"{name}: worker rep {rep}: cold {walls['cold'][-1]:.3f} s, loaded {walls['loaded'][-1]:.3f} s")
                    for arm in ("cold", "loaded"):   # the answers, hashed in a pass of their own
                        h = hashlib.sha256()
                        worker(arm == "loaded", h)
                        wsha[arm] = h.hexdigest()
                    res["worker"] = {"wall_s": {a: spread(walls[a]) for a in walls}, "rows_computed": wcomp,
                                     "sha256": wsha, "answers_equal": wsha["cold"] == wsha["loaded"]}
                    snap = io.BytesIO()
                    col.save(snap)
                    # one session of 20 context items (the first seeded user with that many), the same in every rep: each
                    # rep restores a fresh collection, so each call is a first call
                    srng = np.random.default_rng(11)
                    u = next(int(u) for u in srng.permutation(U) if off[u + 1] - off[u] >= 20)
                    sess = ctx_items[off[u]:off[u] + 20].tolist()
                    first, load_first, ssha = {"cold": [], "loaded": []}, [], {"cold": [], "loaded": []}
                    for rep in range(args.reps):
                        for arm in ("cold", "loaded"):
                            # the kernels are loaded on this context already; the restored collection's work buffers
                            # are part of its first call
                            with gb.VectorCollection.load(ctx, io.BytesIO(snap.getvalue())) as rc:
                                rc.neighbour_cache(n, rows)
                                if arm == "loaded":
                                    w, _ = timed(lambda: rc.load_neighbour_cache(io.BytesIO(data)))
                                    load_first.append(w)
                                w, (ans, _) = timed(lambda: rc.session_recommend([sess], [[]], n, 100, n))
                                first[arm].append(w * 1e3)
                                assert len(ans[0][0]) > 0
                                ssha[arm].append(hashlib.sha256(np.asarray(ans[0][0]).tobytes() + np.asarray(ans[0][1]).tobytes()).hexdigest())
                    res["session"] = {"first_call_ms": {a: spread(first[a]) for a in first}, "stream_load_s": spread(load_first),
                                      "answers_equal": ssha["cold"] == ssha["loaded"], "sha256": ssha}
                result[name] = res
                log(f"{name}: {json.dumps(res)}")
    result["card_after"] = card()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
