"""`gorse-bench embedding`'s scoring on the H100: gorse_b200_embedding_eval on a C2-shaped dataset.

Data: --users users, --items items, --feedback feedback with Zipf(1) item popularity (gorse_b200.synth.make_feedback) and
distinct timestamps, split with embedding_oracle.split_latest (a restatement of dataset.SplitLatest) at each --shots value
("all" = every earlier item); seeded N(0, 1) fp32 embeddings at each --dims; 99 negatives sampled on the device.
Before timing, the first --check users are scored by the library and by the CPU restatement (embedding_oracle), which
must agree bit for bit; the restatement's single-thread milliseconds per user are reported as the CPU reference point.
Reported per (d, shots): host-in to host-out seconds (median of --repeat), the scoring kernels' device time from a separate
torch.profiler run, distance pairs, algorithmic flop (3 d per pair: sub, mul, add) and the bytes the CTAs stage, each per
second, with the card's name, power limit and SM clock read in the same run.  Prints one JSON line.

  python tools/embedding_eval_bench.py [--dims 768,1536,3072] [--shots all,10]
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

ALL = 1 << 62
MT = 16   # 4 x 4 micro-tiles per CTA of the scoring kernel (csrc/embedding_eval.cu)


def staged_rows(m, k):
    """rows the CTAs of one user with m candidates and k shots stage: per CTA, the candidate quads and the shot quads its
    MT consecutive micro-tiles (candidate quad major) touch"""
    nq_s, total = (k + 3) // 4, ((m + 3) // 4) * ((k + 3) // 4)
    rows = 0
    for t0 in range(0, total, MT):
        nt = min(MT, total - t0)
        rows += 4 * ((t0 + nt - 1) // nq_s - t0 // nq_s + 1) + 4 * min(nt, nq_s)
    return rows


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={q}", "--format=csv,noheader,nounits"], capture_output=True, text=True,
                         check=True).stdout.strip()
    name, power, sm, sm_max = [x.strip() for x in out.split(",")]
    return {"name": name, "power_limit_w": float(power), "sm_mhz": float(sm), "sm_max_mhz": float(sm_max)}


def head(c, n):
    off, items = c
    return off[:n + 1].copy(), items[:off[n]].copy()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--users", type=int, default=1_000_000)
    ap.add_argument("--items", type=int, default=100_000)
    ap.add_argument("--feedback", type=int, default=10_000_000)
    ap.add_argument("--dims", default="768,1536,3072")
    ap.add_argument("--shots", default="all,10")
    ap.add_argument("--check", type=int, default=2000)
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()

    import torch

    import embedding_oracle as eo
    import gorse_b200 as gb
    from gorse_b200 import synth

    rng = np.random.default_rng(a.seed)
    fb = synth.make_feedback(a.users, a.items, a.feedback, seed=a.seed)
    ts = rng.permutation(int(fb[0][-1]))
    rows = []
    with gb.Context(0) as ctx:
        for dim in [int(x) for x in a.dims.split(",")]:
            emb = rng.standard_normal((a.items, dim), dtype=np.float32)
            for sv in a.shots.split(","):
                shots = ALL if sv == "all" else int(sv)
                tr, te = eo.split_latest(fb[0], fb[1], ts, shots)
                # the first users, against the restatement
                n = min(a.check, a.users)
                trc, tec, fbc = head(tr, n), head(te, n), head(fb, n)
                got = gb.evaluate_embeddings(ctx, emb, None, trc, tec, fbc)
                negs = eo.sample_negatives(a.items, fbc, tec, 99)
                t0 = time.perf_counter()
                want = eo.evaluate(emb, None, trc, tec, negs)
                cpu_ms_per_user = (time.perf_counter() - t0) * 1e3 / max(want[3], 1)
                assert got == want, (got, want)
                times = []
                for _ in range(a.repeat):
                    t0 = time.perf_counter()
                    res = gb.evaluate_embeddings(ctx, emb, None, tr, te, fb)
                    times.append(time.perf_counter() - t0)
                with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                    gb.evaluate_embeddings(ctx, emb, None, tr, te, fb)
                dev = {}
                for ev in prof.events():
                    if ev.device_type == torch.autograd.DeviceType.CUDA:
                        dev[ev.name] = dev.get(ev.name, 0.0) + ev.device_time_total / 1e3
                dist_ms = sum(v for k, v in dev.items() if "emb_dist_kernel" in k)
                total_ms = sum(v for k, v in dev.items() if "emb_total_kernel" in k)
                # every item has an embedding: users with a test item and a shot score 1 + 99 candidates over all their shots
                k = np.diff(tr[0])
                scored = (k > 0) & (np.diff(te[0]) > 0)
                pairs = int(100 * k[scored].sum())
                ks, counts = np.unique(k[scored], return_counts=True)
                staged = sum(staged_rows(100, int(kk)) * int(c) for kk, c in zip(ks, counts)) * dim * 4
                rows.append({"dim": dim, "shots": sv, "users_scored": res[3], "ndcg": float(res[0]), "host_s_median": float(np.median(times)),
                             "host_s_spread": float(max(times) - min(times)), "dist_kernel_ms": dist_ms, "total_kernel_ms": total_ms,
                             "device_ms_all_kernels": sum(dev.values()), "pairs": pairs, "pairs_per_s": pairs / (dist_ms / 1e3),
                             "tflop_per_s": 3 * dim * pairs / (dist_ms / 1e3) / 1e12, "staged_tb_per_s": staged / (dist_ms / 1e3) / 1e12,
                             "checked_users": want[3], "cpu_oracle_single_thread_ms_per_user": cpu_ms_per_user})
                print(json.dumps(rows[-1]), file=sys.stderr, flush=True)
    print(json.dumps({"bench": "embedding_eval", "card": card(), "users": a.users, "items": a.items, "feedback": int(fb[0][-1]),
                      "datasheet": {"fp32_tflop_per_s_fma_counted_as_2": 67.0, "hbm_tb_per_s": 3.35}, "rows": rows}))


if __name__ == "__main__":
    main()
