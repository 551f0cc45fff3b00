"""Batched FM ranking on the H100: gorse_b200_fm_rank for many users (the worker's "fm" ranker, rankByClickTroughRate).

Shape: --users users, --cands candidates each drawn from --items items with C2's seed (1000), k = --k, about 5 labels per
user and per item, no embedding slot or one --emb-dim slot.  Before timing, a seeded sample of users is checked against the
CPU restatement (fm_oracle) bit for bit; the same sample gives the restatement's single-thread throughput (the C
restatement, not Go).  Reports users/s from host arrays in to host arrays out, and the device time per kernel from
torch.profiler in a separate call.  Prints one JSON line, and also writes it to a file under --out if given.

  python tools/fm_rank_bench.py --users 1000000 --emb-dim 0
  python tools/fm_rank_bench.py --users 20000 --emb-dim 768
"""
import argparse
import json
import os
import subprocess
import sys
import time
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={q}", "--format=csv,noheader,nounits"], capture_output=True, text=True,
                         check=True).stdout.strip()
    name, power, sm, sm_max = [x.strip() for x in out.split(",")]
    return {"name": name, "power_limit_w": float(power), "sm_mhz": float(sm), "sm_max_mhz": float(sm_max)}


def make_input(args, rng):
    import fm_oracle

    dims = (args.emb_dim,) if args.emb_dim else ()
    ns = fm_oracle.random_input(rng, args.features, [0], args.items, dims)   # the item table and one placeholder user
    U = args.users
    ns.n_users = U
    ns.user_feat = rng.integers(0, args.features, U).astype(np.int32)
    cnt = rng.integers(0, 11, U)
    ns.user_lab_off = np.zeros(U + 1, np.int64)
    np.cumsum(cnt, out=ns.user_lab_off[1:])
    ns.user_lab_idx = rng.integers(0, args.features, int(ns.user_lab_off[-1]) + 1).astype(np.int32)
    ns.user_lab_val = rng.standard_normal(int(ns.user_lab_off[-1]) + 1).astype(np.float32)
    ns.cand_off = np.arange(U + 1, dtype=np.int64) * args.cands
    ns.cand_items = np.random.default_rng(1000).integers(0, args.items, U * args.cands + 1).astype(np.int32)
    return ns, dims


def subset(ns, users):
    s = types.SimpleNamespace(**vars(ns))
    s.n_users = len(users)
    s.user_feat = ns.user_feat[users].copy()
    lo, hi = ns.user_lab_off[users], ns.user_lab_off[users + 1]
    s.user_lab_off = np.concatenate([[0], np.cumsum(hi - lo)]).astype(np.int64)
    s.user_lab_idx = np.concatenate([ns.user_lab_idx[a:b] for a, b in zip(lo, hi)] + [[0]]).astype(np.int32)
    s.user_lab_val = np.concatenate([ns.user_lab_val[a:b] for a, b in zip(lo, hi)] + [[0]]).astype(np.float32)
    c0, c1 = ns.cand_off[users], ns.cand_off[users + 1]
    s.cand_off = np.concatenate([[0], np.cumsum(c1 - c0)]).astype(np.int64)
    s.cand_items = np.concatenate([ns.cand_items[a:b] for a, b in zip(c0, c1)] + [[0]]).astype(np.int32)
    return s


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--users", type=int, default=1000000)
    ap.add_argument("--cands", type=int, default=300)
    ap.add_argument("--items", type=int, default=100000)
    ap.add_argument("--features", type=int, default=200000)
    ap.add_argument("--k", type=int, default=16)
    ap.add_argument("--emb-dim", type=int, default=0)
    ap.add_argument("--batch-size", type=int, default=1024)
    ap.add_argument("--check", type=int, default=64)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import gorse_b200 as gb
    import fm_oracle

    info = {"card": card(), "args": vars(args)}
    rng = np.random.default_rng(0)
    t = time.perf_counter()
    inp, dims = make_input(args, rng)
    params = fm_oracle.random_params(rng, args.features, args.k, dims)
    info["input_build_s"] = round(time.perf_counter() - t, 2)
    with gb.Context(0) as ctx, gb.FMRanker(ctx, args.features, args.k, 12, args.batch_size, dims, params) as fm:
        # seeded sample against the restatement
        users = np.sort(np.random.default_rng(5).choice(args.users, min(args.check, args.users), replace=False))
        sub = subset(inp, users)
        sg, og, _ = fm.rank(sub)
        model = fm_oracle.Model(args.features, args.k, 12, args.batch_size, dims, params)
        t = time.perf_counter()
        so, oo = model.rank(sub)
        info["oracle_users_per_s_single_thread_C"] = round(len(users) / (time.perf_counter() - t), 1)
        info["sample_bit_identical"] = bool(sg.tobytes() == so.tobytes() and og.tolist() == oo.tolist())
        if not info["sample_bit_identical"]:
            print(json.dumps(info))
            sys.exit("sample differs from the restatement")
        fm.rank(subset(inp, np.arange(min(1000, args.users))))   # warm-up of every kernel
        times = []
        for _ in range(args.repeats):
            t = time.perf_counter()
            scores, order, stats = fm.rank(inp)
            times.append(time.perf_counter() - t)
        info["call_s"] = [round(x, 3) for x in times]
        info["users_per_s"] = round(args.users / min(times), 1)
        info["stats"] = stats
        # device time per kernel, on a separate call
        import torch
        from torch.profiler import ProfilerActivity, profile

        prof_users = np.arange(min(args.users, 100000))
        psub = subset(inp, prof_users)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fm.rank(psub)
        kern = {}
        for e in prof.key_averages():
            if e.device_type is not None and "fm_" in e.key:
                kern[e.key.split("(")[0][-60:]] = round(e.device_time_total / 1e3, 3)
        info["profiled_users"] = int(prof_users.size)
        info["kernel_ms"] = kern
        del torch
    line = json.dumps(info)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, f"fm_rank_bench_emb{args.emb_dim}.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
