#!/usr/bin/env python
"""tools/vecdb_build_bench.py -- building a sparse similarity collection: rows built on the host and added with
gorse_b200_vecdb_add, against the rows' ids handed to gorse_b200_vecdb_add_idf_vectors.

  python tools/vecdb_build_bench.py [--small] [--c5] [--reps 3] [--batch 10000]

Workloads (rows = items, ids = the users with positive feedback on the item, a "users" item-to-item collection):
  c2  bench.py's c2 data, synth.make_feedback(1M users, 100K items, 11M, seed=1000, zipf 1.0, exact=True) + leave_one_out
      (seed=1001): 100,000 rows, 10M ids, sorted and without repeats
  c5  (--c5) the C5 shape: 1,000,000 rows, 200M ids drawn uniformly from 10M users with seeded Zipf(1.0) row lengths, in
      drawn order, repeats included
  IDF: log(1 + rows / freq(user)), computed on the host as the master does, with every 1000th user's entry set to 0.
Two arms, each from a fresh collection, one after the other:
  device  the id rows in batches of --batch rows through gorse_b200_vecdb_add_idf_vectors
  host    the rows built with numpy (row-wise sort, skip rule, de-duplication, (float)sqrt((double)idf)) and added in the
          same batches with gorse_b200_vecdb_add; rows whose vector is empty are not added
Each arm times, with host clocks around calls that end synchronised:
  build_s     host arm: numpy rows + adds; device arm: the calls
  query_s     gorse_b200_vecdb_query of the vectors of 1,000 seeded rows, topK 100 (host arm: the first query after the adds
              builds the device layouts)
  rewrite_s   the master's next cycle: every row again with replace and a later timestamp, delete_before, compact, the query
              (rewrite_build_s, delete_s, compact_s, rewrite_query_s are its parts)
Medians of --reps repetitions.  Both arms must give the same slots, counts and score bits for both queries; the run fails
otherwise.  One JSON line with the card's name, power limit and SM clock read in the same run.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from item_to_item_bench import card  # noqa: E402


def log(msg):
    print(f"[vecdb_build_bench] {msg}", file=sys.stderr, flush=True)


def host_rows(off, ids, idf):
    """appendSparseVector of every row's sorted, de-duplicated ids, vectorised -> (per-row nnz, indices, values)"""
    n = off.size - 1
    row = np.repeat(np.arange(n, dtype=np.int64), np.diff(off))
    order = np.lexsort((ids, row))
    s, r = ids[order], row[order]
    valid = (s >= 0) & (s < idf.size)
    valid[valid] = ~(idf[s[valid]] <= 0)
    valid[1:] &= (s[1:] != s[:-1]) | (r[1:] != r[:-1])
    s, r = s[valid], r[valid]
    return np.bincount(r, minlength=n), s.astype(np.uint32), np.sqrt(idf[s].astype(np.float64)).astype(np.float32)


def workload(name, small):
    from gorse_b200 import synth, transpose_csr

    if name == "c2":
        U, I, R = (20_000, 5_000, 200_000) if small else (1_000_000, 100_000, 10_000_000)
        off0, items0 = synth.make_feedback(U, I, R + U, seed=1000, zipf_s=1.0, exact=True)
        (off, items), _ = synth.leave_one_out(off0, items0, seed=1001)
        roff, rids = transpose_csr(off, items.astype(np.int32), I)
    else:
        U, I, R = (100_000, 10_000, 2_000_000) if small else (10_000_000, 1_000_000, 200_000_000)
        rng = np.random.default_rng(5000)
        w = 1.0 / np.arange(1, I + 1)
        cnt = rng.multinomial(R, w / w.sum())
        roff = np.concatenate([[0], np.cumsum(cnt)]).astype(np.int64)
        rids = rng.integers(0, U, R, dtype=np.int32)
    freq = np.bincount(rids, minlength=U).astype(np.float64)
    idf = np.log(1 + I / np.maximum(freq, 1)).astype(np.float32)
    idf[::1000] = 0
    return roff.astype(np.int64), np.ascontiguousarray(rids, np.int32), idf


def run_arm(gb, ctx, arm, off, ids, idf, batch, nq):
    import ctypes as C

    from gorse_b200 import _lib

    lib, n = _lib.lib, off.size - 1
    rec = {}
    col = gb.VectorCollection(ctx, 0, gb.DISTANCE_DOT)
    slot_of = np.full(n, -1, np.int64)

    def build(ts):
        t0 = time.perf_counter()
        if arm == "host":
            cnt, ind, val = host_rows(off, ids, idf)
            vo = np.concatenate([[0], np.cumsum(cnt)]).astype(np.int64)
        for a in range(0, n, batch):
            b = min(a + batch, n)
            rep = np.ascontiguousarray(slot_of[a:b])
            if arm == "host":
                keep = np.flatnonzero(cnt[a:b]) + a
                so = np.concatenate([[0], np.cumsum(cnt[keep])]).astype(np.int64)
                first = C.c_int64(0)
                gb.check(lib.gorse_b200_vecdb_add(col.h, keep.size, gb.ptr(val[vo[a]:vo[b]]), gb.ptr(so), gb.ptr(ind[vo[a]:vo[b]]), None,
                                                  gb.ptr(np.full(keep.size, ts, np.int64)), None, None, gb.ptr(np.ascontiguousarray(rep[keep - a])),
                                                  C.byref(first)))
                slot_of[keep] = first.value + np.arange(keep.size)
            else:
                o = np.ascontiguousarray(off[a:b + 1] - off[a])
                out = np.zeros(b - a, np.int64)
                gb.check(lib.gorse_b200_vecdb_add_idf_vectors(col.h, b - a, gb.ptr(o), gb.ptr(ids[off[a]:off[b]]), gb.ptr(idf), idf.size, 0, None, None,
                                                              None, 0, 0, None, ts, None, None, gb.ptr(rep), gb.ptr(out)))
                slot_of[a:b] = np.where(out >= 0, out, slot_of[a:b])
        return time.perf_counter() - t0

    rows_q = np.sort(np.random.default_rng(77).choice(n, min(nq, n), replace=False))   # the queries: these rows' vectors

    def vector(s):
        nnz = C.c_int32(0)
        gb.check(lib.gorse_b200_vecdb_get_sparse(col.h, int(s), None, None, 0, C.byref(nnz)))
        return col.get_sparse(int(s), cap=max(nnz.value, 1))

    def query():
        qs = [vector(s) for s in slot_of[rows_q] if s >= 0]
        t0 = time.perf_counter()
        s, sc, c = col.query(qs, (), 100)
        return time.perf_counter() - t0, (s.tobytes(), sc.tobytes(), c.tobytes())

    with col:
        rec["build_s"] = build(1000)
        rec["query_s"], a1 = query()
        rec["slots"] = col.count()[1]
        rec["rewrite_build_s"] = build(2000)
        t1 = time.perf_counter()
        col.delete_before(2000)
        t2 = time.perf_counter()
        new_slot, _, _ = col.compact()
        t3 = time.perf_counter()
        slot_of[:] = np.where(slot_of >= 0, new_slot[np.maximum(slot_of, 0)], -1)
        rec["rewrite_query_s"], a2 = query()
        rec["delete_s"], rec["compact_s"] = t2 - t1, t3 - t2
        rec["rewrite_s"] = rec["rewrite_build_s"] + rec["delete_s"] + rec["compact_s"] + rec["rewrite_query_s"]
        rec["live"] = col.count()[0]
    return rec, (a1, a2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--small", action="store_true", help="small shapes (a rehearsal, not a measurement)")
    ap.add_argument("--c5", action="store_true", help="also the C5 shape (1M rows, 200M ids)")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--batch", type=int, default=10_000)
    ap.add_argument("--queries", type=int, default=1_000)
    args = ap.parse_args()

    import gorse_b200 as gb

    out = {}
    with gb.Context(0) as ctx:
        for name in ["c2"] + (["c5"] if args.c5 else []):
            off, ids, idf = workload(name, args.small)
            log(f"{name}: {off.size - 1} rows, {ids.size} ids")
            reps = {"device": [], "host": []}
            for r in range(args.reps):
                got = {}
                for arm in ("device", "host"):
                    rec, got[arm] = run_arm(gb, ctx, arm, off, ids, idf, args.batch, args.queries)
                    log(f"{name} rep {r} {arm}: {rec}")
                    reps[arm].append(rec)
                assert got["host"] == got["device"], f"{name}: the two arms answer differently"
            med = {arm: {k: float(np.median([x[k] for x in v])) for k in v[0]} for arm, v in reps.items()}
            out[name] = {"rows": off.size - 1, "ids": int(ids.size), "median": med, "reps": reps}
    print(json.dumps({"metric": "sparse collection build: host rows + vecdb_add vs vecdb_add_idf_vectors", "card": card(),
                      "batch": args.batch, "queries": args.queries, "small": args.small, "workloads": out}))


if __name__ == "__main__":
    main()
