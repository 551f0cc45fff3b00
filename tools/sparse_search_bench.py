#!/usr/bin/env python
"""tools/sparse_search_bench.py -- the tiled sparse search (gorse_b200_sparse_index_search_range) at C2 shapes.

  python tools/sparse_search_bench.py [--small] [--collections items,users] [--k 100]

Data: bench.py's c2 (synth.make_feedback(1M, 100K, 11M, seed=1000, exact=True) + leave_one_out(seed=1001)), as the sparse
similarity types build their vectors through gb.sparse_vector:
  items  one vector per user (1M): the user's training items with weights log(1 + U / freq(i)), what the "items" user-to-user
         type stores.  Few features per query, long posting lists: the push path's side.
  users  one vector per item (100K): the item's users with weights log(1 + I / freq(u)), what the "users" item-to-item type
         stores.  A Zipf(1) head item has hundreds of thousands of features: the pull path's side.
Each collection answers the all-pairs search_range(0, N, k) once after a warm-up on its first rows.

One JSON line:
  card          name, power limit and SM clock (nvidia-smi --query-gpu, read in the same run)
  per collection
    rows / nnz  vectors and stored entries
    wall_s      the all-pairs search, host in to host out
    device_ms   the searches' device time (gorse_b200_sparse_index_stats)
    push / pull work items by path, and tiles walked
    sha256      of the answers (idx int32, dot float32, count int32 bytes, in that order)
"""
import argparse
import hashlib
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
    print(f"[sparse_search_bench] {msg}", file=sys.stderr, flush=True)


def vectors(gb, rows_off, rows_ind, n_other):
    """one sparse vector per row of the CSR (rows_off, rows_ind), weights log(1 + n_other / freq) through gb.sparse_vector"""
    n_rows = len(rows_off) - 1
    freq = np.bincount(rows_ind, minlength=n_other).astype(np.float64)
    idf = np.log(1 + n_rows / np.maximum(freq, 1)).astype(np.float32)
    sp = [gb.sparse_vector(rows_ind[rows_off[r]:rows_off[r + 1]], idf) for r in range(n_rows)]
    off = np.concatenate([[0], np.cumsum([len(v[0]) for v in sp])]).astype(np.int64)
    ind = np.concatenate([v[0] for v in sp]).astype(np.uint32)
    val = np.concatenate([v[1] for v in sp]).astype(np.float32)
    return off, ind, val


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--small", action="store_true", help="20K users x 5K items (a rehearsal, not a measurement)")
    ap.add_argument("--collections", default="items,users")
    ap.add_argument("--k", type=int, default=100)
    args = ap.parse_args()

    import gorse_b200 as gb
    from gorse_b200 import synth

    U, I, R = (20_000, 5_000, 200_000) if args.small else (1_000_000, 100_000, 10_000_000)
    off0, items0 = synth.make_feedback(U, I, R + U, seed=1000, zipf_s=1.0, exact=True)
    (off, items), _ = synth.leave_one_out(off0, items0, seed=1001)
    items = items.astype(np.int32)
    log(f"data: {U} users, {I} items, {int(off[-1])} training rows")
    records = {}
    with gb.Context(0) as ctx:
        for name in args.collections.split(","):
            if name == "items":
                v_off, v_ind, v_val = vectors(gb, off, items, I)
            else:
                ioff, iusers = gb.transpose_csr(off, items, I)
                v_off, v_ind, v_val = vectors(gb, ioff, iusers.astype(np.int32), U)
            N = len(v_off) - 1
            log(f"{name}: {N} vectors, {int(v_off[-1])} entries")
            with gb.SparseIndex(ctx) as ix:
                ix.add(v_off, v_ind, v_val)
                ix.search_range(0, min(N, 4096), args.k)   # warm-up: device layouts, modules, work buffers
                ix.stats()
                t0 = time.perf_counter()
                idx, dot, cnt = ix.search_range(0, N, args.k)
                wall = time.perf_counter() - t0
                st = ix.stats()
            h = hashlib.sha256()
            for a in (idx, dot, cnt):
                h.update(np.ascontiguousarray(a).tobytes())
            records[name] = {"rows": N, "nnz": int(v_off[-1]), "k": args.k, "wall_s": round(wall, 3), "device_ms": round(st["search_ms"], 2),
                             "push": st["push"], "pull": st["pull"], "tiles": st["tiles"], "sha256": h.hexdigest()}
            log(f"{name}: {records[name]}")
    print(json.dumps({"metric": "sparse all-pairs search_range, s", "card": card(),
                      "shape": {"users": U, "items": I, "training_rows": int(off[-1])}, "collections": records}))


if __name__ == "__main__":
    main()
