#!/usr/bin/env python
"""tools/session_bench.py -- batched session recommendation (gorse_b200_vecdb_session_recommend) at C2 shapes.

  python tools/session_bench.py [--small]

Data: bench.py's c2 (synth.make_feedback(1M, 100K, 11M, seed=1000, exact=True) + leave_one_out(seed=1001)), and the two
item-to-item collections of tools/item_to_item_bench.py over its 100,000 items, slot = item id:
  users      sparse Dot: each item's users with weights sqrt(log(1 + I / freq(u))) (gb.sparse_vector), the "users" type
  embedding  dense Euclidean, d = 64: the item factors of 20 BPR epochs truncated to bf16
Sessions: 100,000 seeded draws of a training row (so their lengths follow the C2 rows), each row in a seeded order as the
session's positive feedback, newest first; the exclude set is the same row (every item of the session).  n = 100 (CacheSize),
context_size = 100, top = 10 (n + offset of the request), an item_ok that drops a seeded 8 % of the items.  Before timing,
64 seeded sessions are checked against the handler's restatement (tests/session_model.py) over the oracle's brute force (for
the sparse collection, sessions whose items have at most 2,000 users each: the restatement's cost grows with the longest
vector).

One JSON line, with per collection:
  card                 name, power limit and SM clock (nvidia-smi --query-gpu, read in the same run)
  wall_s               all sessions in one call, host in to host out, median of 3
  device_ms            stage A (neighbour table) and stage B (i2i_aggregate_kernel) device time in one profiled call
  single_session_ms    n_sessions = 1, median over 100 seeded sessions
  stats                distinct context items, neighbour rows answered by the exact scan, sessions per accumulator
  per_item             the handler's path: one gorse_b200_vecdb_query(topK = n + 1) per context item up to the handler's cut,
                       for the first 1,024 sessions (fewer if they take more than a minute), per session, and the all-session
                       time it implies -- a LOWER BOUND: it leaves out the data store's BatchGetItems per item and the map
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

from item_to_item_bench import card  # noqa: E402


def log(msg):
    print(f"[session_bench] {msg}", file=sys.stderr, flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--small", action="store_true", help="20K users x 5K items, 5K sessions (a rehearsal, not a measurement)")
    ap.add_argument("--n", type=int, default=100)
    ap.add_argument("--context-size", type=int, default=100)
    ap.add_argument("--top", type=int, default=10)
    ap.add_argument("--sessions", type=int, default=100_000)
    ap.add_argument("--epochs", type=int, default=20)
    ap.add_argument("--check", type=int, default=64)
    ap.add_argument("--per-item-sessions", type=int, default=1024)
    args = ap.parse_args()

    import gorse_b200 as gb
    import oracle
    import session_model as sm
    from gorse_b200 import _lib, synth

    U, I, R, d = (20_000, 5_000, 200_000, 64) if args.small else (1_000_000, 100_000, 10_000_000, 64)
    S = min(args.sessions, 5_000) if args.small else args.sessions
    n, cs, top = args.n, args.context_size, args.top
    off0, items0 = synth.make_feedback(U, I, R + U, seed=1000, zipf_s=1.0, exact=True)
    (off, items), _ = synth.leave_one_out(off0, items0, seed=1001)
    lib = _lib.lib
    rng = np.random.default_rng(1000)
    # sessions: seeded training rows, each in a seeded order
    rows_of = rng.integers(0, U, S)
    lens = np.diff(off)[rows_of]
    s_off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    s_items = np.concatenate([items[off[u]:off[u + 1]][rng.permutation(off[u + 1] - off[u])] for u in rows_of]).astype(np.int64)
    item_ok = (rng.random(I) >= 0.08).astype(np.uint8)
    session = lambda s: s_items[s_off[s]:s_off[s + 1]]   # noqa: E731
    log(f"data: {U} users, {I} items; {S} sessions, {int(s_off[-1])} session items (mean {lens.mean():.1f}, max {lens.max()})")
    records = {}
    with gb.Context(0) as ctx:
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
                out = (np.zeros(S * top, np.int64), np.zeros(S * top, np.float64), np.zeros(S, np.int32))
                stats = np.zeros(4, np.int64)

                def run(s0, s1):
                    co = s_off[s0:s1 + 1] - s_off[s0]
                    ci = np.ascontiguousarray(s_items[s_off[s0]:s_off[s1]])
                    gb.check(lib.gorse_b200_vecdb_session_recommend(col.h, s1 - s0, gb.ptr(co), gb.ptr(ci), gb.ptr(co), gb.ptr(ci), gb.ptr(item_ok), n,
                                                                    cs, top, 1.0, gb.ptr(out[0]), gb.ptr(out[1]), gb.ptr(out[2]), gb.ptr(stats)))
                    return stats.copy()

                # ---- correctness first: seeded sessions against the restated handler.  The neighbour lists are fetched 4n
                # deep and ordered (score desc, slot asc), the library's documented order of exact ties; a session whose
                # neighbour cut falls inside a tie group that reaches the end of a fetched list cannot be restated this way
                # and is skipped.
                light = np.ones(S, bool) if dense else np.array([np.diff(sp_off)[session(s)].max(initial=0) <= 2000 for s in range(S)])
                sel = np.sort(np.random.default_rng(0).choice(np.nonzero(light)[0], size=min(args.check, int(light.sum())), replace=False))
                got, _ = col.session_recommend([session(s) for s in sel], [session(s) for s in sel], n, cs, top, item_ok=item_ok)
                kk, checked, clear = 4 * n + 1, 0, [True]

                def neighbours(c):
                    if dense:
                        oi, od = oracle.bruteforce_search(X, X[c], kk, metric=oracle.METRIC_EUCLIDEAN)
                        sc = -od
                    else:
                        oi, sc = oracle.sparse_bruteforce_search(sp_off, sp_ind, sp_val, c, kk)
                    o = np.lexsort((oi, -sc))
                    oi, sc = oi[o], sc[o]
                    clear[0] &= len(oi) < kk or sc[min(n, len(sc) - 1)] != sc[-1] or (not dense and sc[min(n, len(sc) - 1)] <= 0)
                    return oracle.similar_scores(dense, 1.0, c, n, oi, sc)

                for (gs, gv), s in zip(got, sel):
                    clear[0] = True
                    (ws, wv), = sm.session_rows(neighbours, [session(s)], [session(s)], cs, top, item_ok)
                    if not clear[0]:
                        continue
                    checked += 1
                    assert gv.tobytes() == wv.tobytes(), f"{name} session {s}: scores differ from the restatement"
                    assert gs.tolist() == ws.tolist() or len(set(wv.tolist())) < len(wv), f"{name} session {s}: slots differ"
                log(f"{name}: {checked} of {len(sel)} sampled sessions match the restatement")

                # ---- all sessions in one call, host in to host out
                run(0, S)   # warm-up: mirror, work buffers, modules
                walls = []
                for _ in range(3):
                    t0 = time.perf_counter()
                    totals = run(0, S)
                    walls.append(time.perf_counter() - t0)
                wall = float(np.median(walls))
                log(f"{name}: all sessions in {walls} s")

                # ---- one session per call
                one = []
                for s in np.random.default_rng(1).choice(S, 100, replace=False):
                    t0 = time.perf_counter()
                    run(int(s), int(s) + 1)
                    one.append(time.perf_counter() - t0)
                single_ms = float(np.median(one)) * 1e3

                # ---- device time per stage in a separate, profiled call
                import torch
                from torch.profiler import ProfilerActivity, profile

                torch.cuda.init()
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    run(0, S)
                dev = {}
                for e in prof.key_averages():
                    t = getattr(e, "device_time_total", 0.0) or getattr(e, "cuda_time_total", 0.0)
                    if "Memcpy" in e.key or "Memset" in e.key or not t:
                        continue
                    stage = "B" if "i2i_aggregate_kernel" in e.key else "A"
                    dev[stage] = dev.get(stage, 0.0) + t / 1e3

                # ---- the handler's path: one vecdb_query per context item up to its cut, lower bound
                ns = min(args.per_item_sessions, S)
                s_, v_, c_ = np.zeros(n + 1, np.int64), np.zeros(n + 1, np.float32), np.zeros(1, np.int32)

                def query(c):
                    if dense:
                        st = lib.gorse_b200_vecdb_query(col.h, 1, gb.ptr(X[c]), None, None, None, 0, n + 1, gb.ptr(s_), gb.ptr(v_), gb.ptr(c_))
                    else:
                        qo = np.array([0, sp_off[c + 1] - sp_off[c]], np.int64)
                        st = lib.gorse_b200_vecdb_query(col.h, 1, gb.ptr(sp_val[sp_off[c]:sp_off[c + 1]]), gb.ptr(qo),
                                                        gb.ptr(sp_ind[sp_off[c]:sp_off[c + 1]]), None, 0, n + 1, gb.ptr(s_), gb.ptr(v_), gb.ptr(c_))
                    gb.check(st)
                    return any(item_ok[j] for j in s_[:c_[0]].tolist() if j != c)

                query(int(s_items[0]))   # warm-up
                queries = 0
                t0 = time.perf_counter()
                for s in range(ns):
                    used = 0
                    for c in session(s).tolist():
                        queries += 1
                        used += query(c)
                        if used >= cs:
                            break
                    if time.perf_counter() - t0 > 60:
                        ns = s + 1
                        break
                per_session_s = (time.perf_counter() - t0) / ns
                log(f"{name}: per-item path {per_session_s * 1e3:.2f} ms per session over {ns} sessions")

            records[name] = {
                "d": d if dense else 0,
                "checked_sessions": checked, "sampled_sessions": int(len(sel)),
                "wall_s": wall, "wall_s_all": walls, "sessions_per_s": S / wall,
                "device_ms": {"stage_a": dev.get("A", 0.0), "stage_b": dev.get("B", 0.0)},
                "single_session_ms": single_ms,
                "stats": {"context_items": int(totals[0]), "exact_rows": int(totals[1]), "shared_sessions": int(totals[2]),
                          "global_sessions": int(totals[3])},
                "per_item_lower_bound": {"sessions_timed": ns, "queries": queries, "ms_per_session": per_session_s * 1e3,
                                         "implied_all_sessions_s": per_session_s * S, "batched_speedup_at_least": per_session_s * S / wall},
            }
    print(json.dumps({"metric": "batched session recommendation, sessions/s (host in to host out)", "card": card(),
                      "shape": {"users": U, "items": I, "sessions": S, "session_items": int(s_off[-1]), "n": n, "context_size": cs, "top": top,
                                "item_ok_share": float(item_ok.mean()), "bpr_epochs": args.epochs, "small": args.small},
                      "collections": records}))


if __name__ == "__main__":
    main()
