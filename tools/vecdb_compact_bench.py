#!/usr/bin/env python
"""tools/vecdb_compact_bench.py -- vector collections under the master's hourly rewrite, with and without compaction
(gorse_b200_vecdb_compact).

  python tools/vecdb_compact_bench.py [--small] [--cycles 8]

Data: bench.py's c2 (synth.make_feedback(1M, 100K, 11M, seed=1000, exact=True) + leave_one_out(seed=1001)) and the three
collections the other tools build from it, slot order = id order on the first write:
  embedding  dense Euclidean user-to-user, all 1M users, d = 64: the user factors of 20 BPR epochs truncated to bf16
  items      sparse Dot user-to-user, the first 100,000 users: their training items with weights sqrt(log(1 + U / freq(i)))
  users      sparse Dot item-to-item, all 100,000 items: their users with weights sqrt(log(1 + I / freq(u)))
A cycle is what runLoadDatasetTask does to a collection (master/tasks.go:783-877): every vector upserted by id in batches of
10,000 with the cycle's timestamp, then DeleteVectors(timestamp).  Arm A compacts after each cycle, arm B does not; the arms
run one after the other on fresh collections.  After each cycle:
  slots, live            gorse_b200_vecdb_count
  library_bytes          arm A: the device bytes gorse_b200_vecdb_compact reports after compacting
  device_used_bytes      both arms: device memory in use (cudaMemGetInfo) minus its value before the arm's collection existed
  compact_s              arm A: host clock around the call, which ends synchronised
  query_s                a fixed workload, host clock around the call: embedding -- gorse_b200_vecdb_query_excluding for the
                         first 4,096 users, each user's own vector excluded, n = 100; users -- gorse_b200_vecdb_session_recommend
                         for 1,000 seeded sessions (training rows in seeded order), n = 100, context_size = 100, top = 10;
                         items -- gorse_b200_vecdb_query of the first 1,000 users' vectors, topK = 100 (a sparse collection
                         builds its device mirrors at the first query after a write, so without one arm B would hold none)
  digest                sha256 of the workload's answers with slots written as ids, and the score bits
Every cycle's digests of arm A and arm B must match (arm A's slots renamed through new_slot are arm B's); the run fails
otherwise.  One JSON line with the card's name, power limit and SM clock read in the same run.
"""
import argparse
import ctypes as C
import hashlib
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
    print(f"[vecdb_compact_bench] {msg}", file=sys.stderr, flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--small", action="store_true", help="20K users x 5K items (a rehearsal, not a measurement)")
    ap.add_argument("--cycles", type=int, default=8)
    ap.add_argument("--epochs", type=int, default=20)
    ap.add_argument("--batch", type=int, default=10_000)
    ap.add_argument("--query-users", type=int, default=4_096)
    ap.add_argument("--sessions", type=int, default=1_000)
    ap.add_argument("--sparse-users", type=int, default=100_000)
    args = ap.parse_args()

    import torch

    import gorse_b200 as gb
    from gorse_b200 import _lib, synth

    U, I, R, d = (20_000, 5_000, 200_000, 64) if args.small else (1_000_000, 100_000, 10_000_000, 64)
    n, cs, top = 100, 100, 10
    off0, items0 = synth.make_feedback(U, I, R + U, seed=1000, zipf_s=1.0, exact=True)
    (off, items), _ = synth.leave_one_out(off0, items0, seed=1001)
    items = items.astype(np.int32)
    lib = _lib.lib
    torch.cuda.init()

    def used():
        free, total = torch.cuda.mem_get_info(0)
        return total - free

    rng = np.random.default_rng(1000)
    rows_of = rng.integers(0, U, args.sessions)
    s_off = np.concatenate([[0], np.cumsum(np.diff(off)[rows_of])]).astype(np.int64)
    s_items = np.concatenate([items[off[u]:off[u + 1]][rng.permutation(off[u + 1] - off[u])] for u in rows_of]).astype(np.int64)
    records = {}
    with gb.Context(0) as ctx:
        with gb.CFModel(ctx, U, I, d, off, items) as m:
            m.init_normal(0.0, 0.001, 0)
            for e in range(args.epochs):
                m.bpr_epoch(0.05, 0.01, int(off[-1]), 1000 + e)
            P, _ = m.get_factors()
        X = np.ascontiguousarray(gb.bf16_truncate(P), np.float32)
        log("model trained")
        Us = min(args.sparse_users, U)
        freq = np.bincount(items, minlength=I).astype(np.float64)
        idf_i = np.log(1 + U / np.maximum(freq, 1)).astype(np.float32)
        ioff, iusers = gb.transpose_csr(off, items, I)
        idf_u = np.log(1 + I / np.maximum(np.diff(off).astype(np.float64), 1)).astype(np.float32)

        def csr(vecs):
            sp_off = np.concatenate([[0], np.cumsum([len(v[0]) for v in vecs])]).astype(np.int64)
            return sp_off, np.concatenate([v[0] for v in vecs]).astype(np.uint32), np.concatenate([v[1] for v in vecs]).astype(np.float32)

        data = {"embedding": (U, None), "items": (Us, csr([gb.sparse_vector(items[off[u]:off[u + 1]], idf_i) for u in range(Us)])),
                "users": (I, csr([gb.sparse_vector(iusers[ioff[i]:ioff[i + 1]], idf_u) for i in range(I)]))}
        log("sparse vectors built")

        for name, (N, sp) in data.items():
            dense = sp is None
            arms = {}
            for arm in ("A", "B"):
                base = used()
                col = gb.VectorCollection(ctx, d if dense else 0, gb.DISTANCE_EUCLIDEAN if dense else gb.DISTANCE_DOT)
                slot_of = np.full(N, -1, np.int64)     # id -> live slot
                id_of = np.zeros(0, np.int64)          # slot -> id
                cycles = []
                with col:
                    for k in range(1, args.cycles + 1):
                        t0 = time.perf_counter()
                        for a in range(0, N, args.batch):
                            b = min(a + args.batch, N)
                            ts = np.full(b - a, 1000 * k, np.int64)
                            rep = np.ascontiguousarray(slot_of[a:b])
                            first = C.c_int64(0)
                            if dense:
                                gb.check(lib.gorse_b200_vecdb_add(col.h, b - a, gb.ptr(X[a:b]), None, None, None, gb.ptr(ts), None, None, gb.ptr(rep),
                                                                  C.byref(first)))
                            else:
                                so, si, sv = sp
                                o = np.ascontiguousarray(so[a:b + 1] - so[a])
                                gb.check(lib.gorse_b200_vecdb_add(col.h, b - a, gb.ptr(sv[so[a]:so[b]]), gb.ptr(o), gb.ptr(si[so[a]:so[b]]), None,
                                                                  gb.ptr(ts), None, None, gb.ptr(rep), C.byref(first)))
                            slot_of[a:b] = first.value + np.arange(b - a)
                        id_of = np.concatenate([id_of, np.arange(N)])   # the batches write the ids in order
                        col.delete_before(1000 * k)
                        rec = {"cycle": k, "write_s": time.perf_counter() - t0}
                        if arm == "A":
                            t0 = time.perf_counter()
                            new_slot, _, after = col.compact()
                            rec["compact_s"] = time.perf_counter() - t0
                            rec["library_bytes"] = after
                            slot_of = new_slot[slot_of]
                            id_of = id_of[new_slot >= 0]
                        rec["live"], rec["slots"] = col.count()
                        h = hashlib.sha256()
                        if name == "embedding":
                            nq = min(args.query_users, N)
                            eo, ex = np.arange(nq + 1, dtype=np.int64), np.ascontiguousarray(slot_of[:nq])
                            sl, sc, ct, ez = np.zeros(nq * (n + 1), np.int64), np.zeros(nq * (n + 1), np.float32), np.zeros(nq, np.int32), C.c_int64(0)
                            call = lambda: gb.check(lib.gorse_b200_vecdb_query_excluding(  # noqa: E731
                                col.h, nq, gb.ptr(X[:nq]), None, 0, n, gb.ptr(eo), gb.ptr(ex), gb.ptr(sl), gb.ptr(sc), gb.ptr(ct), C.byref(ez)))
                            stride = n + 1
                        elif name == "users":
                            S = args.sessions
                            ci = np.ascontiguousarray(slot_of[s_items])
                            sl, sc, ct, st = np.zeros(S * top, np.int64), np.zeros(S * top, np.float64), np.zeros(S, np.int32), np.zeros(4, np.int64)
                            call = lambda: gb.check(lib.gorse_b200_vecdb_session_recommend(  # noqa: E731
                                col.h, S, gb.ptr(s_off), gb.ptr(ci), gb.ptr(s_off), gb.ptr(ci), None, n, cs, top, 1.0, gb.ptr(sl), gb.ptr(sc),
                                gb.ptr(ct), gb.ptr(st)))
                            stride = top
                        else:
                            so, si, sv = sp
                            nq = min(args.sessions, N)
                            sl, sc, ct = np.zeros(nq * n, np.int64), np.zeros(nq * n, np.float32), np.zeros(nq, np.int32)
                            call = lambda: gb.check(lib.gorse_b200_vecdb_query(  # noqa: E731
                                col.h, nq, gb.ptr(sv), gb.ptr(so), gb.ptr(si), None, 0, n, gb.ptr(sl), gb.ptr(sc), gb.ptr(ct)))
                            stride = n
                        t0 = time.perf_counter()   # no warm-up: the first query after a write rebuilds the mirrors, a cost of the cycle
                        call()
                        rec["query_s"] = time.perf_counter() - t0
                        for q, c in enumerate(ct):
                            h.update(id_of[sl[q * stride:q * stride + c]].tobytes())
                            h.update(sc[q * stride:q * stride + c].tobytes())
                        rec["digest"] = h.hexdigest()
                        rec["device_used_bytes"] = used() - base
                        log(f"{name} arm {arm}: {rec}")
                        cycles.append(rec)
                arms[arm] = cycles
            for a, b in zip(arms["A"], arms["B"]):
                assert a.get("digest") == b.get("digest"), f"{name} cycle {a['cycle']}: compacted answers differ"
            records[name] = {"vectors": N, "dim": d if dense else 0, "arms": arms}
    print(json.dumps({"metric": "vector collections over master cycles, compacted (A) and not (B)", "card": card(),
                      "shape": {"users": U, "items": I, "cycles": args.cycles, "batch": args.batch, "query_users": args.query_users,
                                "sessions": args.sessions, "bpr_epochs": args.epochs, "small": args.small},
                      "collections": records}))


if __name__ == "__main__":
    main()
