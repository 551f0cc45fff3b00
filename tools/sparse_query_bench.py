#!/usr/bin/env python
"""tools/sparse_query_bench.py -- sparse neighbour queries past 128 neighbours (the wide path of the tiled sparse search) at C2
shapes, next to the list path at k <= 128.

  python tools/sparse_query_bench.py [--small] [--collections users,items] [--calls 1000] [--check 8]

Data: bench.py's c2 (synth.make_feedback(1M, 100K, 11M, seed=1000, exact=True) + leave_one_out(seed=1001)), as
tools/sparse_search_bench.py builds its collections:
  users  one vector per item (100K): the item's users with weights log(1 + I / freq(u)) ("users" item-to-item type).
  items  one vector per user (1M): the user's training items with weights log(1 + U / freq(i)) ("items" user-to-user type).

Before anything is timed, `--check` seeded stored vectors per collection are queried at every topK and their answers are
compared with the oracle's sparse brute force bit for bit (rows, dot bits, order (dot desc, row asc)).

Measured, host in to host out:
  query         `--calls` single-vector VectorCollection.query calls (the REST neighbour endpoints' shape: one vector, no
                category) at topK 101 (list path) and 129 / 500 / 2000 (wide path), the query vectors a seeded sample of
                stored ones; after one warm-up call per topK
  search_range  SparseIndex.search_range over all rows at k = 500 on `users`, and over rows [0, 10000) on `items`

One JSON line: the card (name, power limit and SM clock, read in the same run), and per collection the rows, the checked
answers, per topK the query calls' total s, ms per call and mean answer length, and the search_range wall s, device ms
(gorse_b200_sparse_index_stats), work items by path, tiles walked and the sha256 of its answers.
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

TOPKS = (101, 129, 500, 2000)


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={q}", "--format=csv,noheader,nounits"], capture_output=True, text=True,
                         timeout=60).stdout.strip()
    name, power, sm, sm_max = [x.strip() for x in out.split(",")]
    return {"name": name, "power_limit_w": float(power), "sm_mhz": float(sm), "sm_max_mhz": float(sm_max)}


def log(msg):
    print(f"[sparse_query_bench] {msg}", file=sys.stderr, flush=True)


def vectors(gb, rows_off, rows_ind, n_other):
    """one sparse vector per row of the CSR (rows_off, rows_ind), weights log(1 + n_other / freq) through gb.sparse_vector"""
    n_rows = len(rows_off) - 1
    freq = np.bincount(rows_ind, minlength=n_other).astype(np.float64)
    idf = np.log(1 + n_rows / np.maximum(freq, 1)).astype(np.float32)
    return [gb.sparse_vector(rows_ind[rows_off[r]:rows_off[r + 1]], idf) for r in range(n_rows)]


def oracle_order(oracle, off, ind, val, vec):
    """the oracle's positive dots of every stored vector with the external vector vec, in (dot desc, row asc) order"""
    n = len(off) - 1
    qi, qv = np.ascontiguousarray(vec[0], np.uint32), np.ascontiguousarray(vec[1], np.float32)
    oi, od = np.zeros(n, np.int32), np.zeros(n, np.float32)
    m = oracle.lib().gbo_sparse_bruteforce_search(off, ind, val, n, qi, qv, len(qi), -1, n, oi, od)
    oi, od = oi[:m], od[:m]
    keep = od > 0
    oi, od = oi[keep], od[keep]
    o = np.lexsort((oi, -od.astype(np.float64)))
    return oi[o], od[o]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--small", action="store_true", help="20K users x 5K items (a rehearsal, not a measurement)")
    ap.add_argument("--collections", default="users,items")
    ap.add_argument("--calls", type=int, default=1000)
    ap.add_argument("--check", type=int, default=8, help="stored vectors per collection checked against the oracle")
    args = ap.parse_args()

    import gorse_b200 as gb
    import oracle
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
                sp = vectors(gb, off, items, I)
                slice_rows = 10_000
            else:
                ioff, iusers = gb.transpose_csr(off, items, I)
                sp = vectors(gb, ioff, iusers.astype(np.int32), U)
                slice_rows = None
            N = len(sp)
            v_off = np.concatenate([[0], np.cumsum([len(v[0]) for v in sp])]).astype(np.int64)
            v_ind = np.concatenate([v[0] for v in sp]).astype(np.uint32)
            v_val = np.concatenate([v[1] for v in sp]).astype(np.float32)
            log(f"{name}: {N} vectors, {int(v_off[-1])} entries")
            rng = np.random.default_rng(17)
            rec = {"rows": N, "nnz": int(v_off[-1])}
            col = gb.VectorCollection(ctx, 0, gb.DISTANCE_DOT)
            try:
                col.add(sparse=sp, timestamps=np.full(N, 1000))
                # the check: seeded stored vectors as external queries, every topK, bit for bit
                check = rng.choice(N, size=min(args.check, N), replace=False)
                want = [oracle_order(oracle, v_off, v_ind, v_val, sp[q]) for q in check]
                for k in TOPKS:
                    slots, scores, cnt = col.query([sp[q] for q in check], (), k)
                    for j, q in enumerate(check):
                        wi, wd = want[j][0][:k], want[j][1][:k]
                        c = int(cnt[j])
                        if not (c == len(wi) and slots[j, :c].tolist() == wi.tolist() and scores[j, :c].tobytes() == wd.tobytes()):
                            raise SystemExit(f"{name}: query of stored vector {q} at topK {k} differs from the oracle")
                rec["checked_queries"] = int(len(check) * len(TOPKS))
                log(f"{name}: {rec['checked_queries']} answers match the oracle")
                calls = rng.integers(0, N, args.calls)
                rec["query"] = {}
                for k in TOPKS:
                    col.query([sp[int(calls[0])]], (), k)   # warm-up
                    t0 = time.perf_counter()
                    got = 0
                    for q in calls:
                        got += int(col.query([sp[int(q)]], (), k)[2][0])
                    wall = time.perf_counter() - t0
                    rec["query"][str(k)] = {"calls": int(args.calls), "total_s": round(wall, 4), "ms_per_call": round(1e3 * wall / args.calls, 4),
                                            "mean_count": round(got / args.calls, 1)}
                    log(f"{name}: query topK {k}: {rec['query'][str(k)]}")
            finally:
                col.close()
            with gb.SparseIndex(ctx) as ix:
                ix.add(v_off, v_ind, v_val)
                q1 = N if slice_rows is None else min(N, slice_rows)
                ix.search_range(0, min(q1, 256), 500)   # warm-up: device layouts, modules, work buffers
                ix.stats()
                t0 = time.perf_counter()
                idx, dot, cnt = ix.search_range(0, q1, 500)
                wall = time.perf_counter() - t0
                st = ix.stats()
            h = hashlib.sha256()
            for a in (idx, dot, cnt):
                h.update(np.ascontiguousarray(a).tobytes())
            rec["search_range"] = {"rows": [0, q1], "k": 500, "wall_s": round(wall, 3), "device_ms": round(st["search_ms"], 2), "push": st["push"],
                                   "pull": st["pull"], "tiles": st["tiles"], "mean_count": round(float(cnt.mean()), 1), "sha256": h.hexdigest()}
            log(f"{name}: search_range {rec['search_range']}")
            records[name] = rec
    print(json.dumps({"metric": "sparse neighbour queries past 128, ms per call / s", "card": card(),
                      "shape": {"users": U, "items": I, "training_rows": int(off[-1]), "small": args.small}, "collections": records}))


if __name__ == "__main__":
    main()
