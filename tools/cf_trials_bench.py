#!/usr/bin/env python
"""tools/cf_trials_bench.py -- the CF model search: ten trials as ten solo fits, or in one gorse_b200_cf_fit_trials call.

  python tools/cf_trials_bench.py [--sizes c1,c2] [--epochs 100] [--als-epochs 50] [--reps 3] [--small]

Data at d = 16 (the search's NFactors):
  c1  943 users x 1,682 items x 100K feedback (the MovieLens 100K shape), synth.make_feedback(seed=1000, Zipf 1)
  c2  bench.py's C2: 1M users x 100K items, 10M training triples after leave_one_out
Trials: ten draws at seed 0, log-uniform over SuggestParams' ranges (model/cf/model.go:397-405, 588-596): Lr, Reg and
InitStdDev in [0.001, 0.1] for BPR; Reg, Alpha and InitStdDev in [0.001, 0.1] for ALS.  FitConfig: Verbose 10,
Candidates 100 (negatives drawn on the device), TopK 10, no patience.

Timed with a host clock around calls that end in a device synchronise, after one warm-up of each, alternating the ways,
median of --reps:
  a  one solo BPR epoch (device events, median of 10)
  b  ten gorse_b200_bpr_fit calls one after the other
  c  one gorse_b200_cf_fit_trials call with the same ten BPR trials
  d  five BPR and five ALS trials, as ten solo fits and as one call
Then, untimed: the largest factor difference of each BPR trial between (b) and (c), relative to the largest factor of (b);
and in a separate run with torch.profiler (CUDA activities), the device time per round of bpr_trials_round_kernel for 1, 2,
5 and 10 models and of bpr_round_kernel.  One JSON line; the card's name, power limit and SM clock come from the same run.
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ROUND = 8192


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={q}", "--format=csv,noheader,nounits"], capture_output=True, text=True,
                         timeout=60).stdout.strip()
    name, power, sm, sm_max = [x.strip() for x in out.split(",")]
    return {"name": name, "power_limit_w": float(power), "sm_mhz": float(sm), "sm_max_mhz": float(sm_max)}


def draw_trials(kind, n, rng, epochs):
    def log_uniform():
        return float(math.exp(rng.uniform(math.log(0.001), math.log(0.1))))

    out = []
    for _ in range(n):
        if kind == "bpr":
            kw = dict(lr=log_uniform(), reg=log_uniform(), init_stddev=log_uniform())
        else:
            kw = dict(init_stddev=log_uniform(), reg=log_uniform(), alpha=log_uniform())
        kw.update(n_epochs=epochs, verbose=10, candidates=100, topk=10, seed=0)
        out.append((kind, kw))
    return out


def data(size, small):
    from gorse_b200 import synth

    if size == "c1":
        U, I, R = 943, 1682, 100_000
    else:
        U, I, R = (50_000, 10_000, 500_000) if small else (1_000_000, 100_000, 10_000_000)
    off0, items0 = synth.make_feedback(U, I, R + U if size == "c2" else R, seed=1000, zipf_s=1.0, exact=True)
    train, test = synth.leave_one_out(off0, items0, seed=1001)
    return U, I, train, test


def timed(ctx, fn):
    ctx.sync()
    t0 = time.perf_counter()
    fn()
    ctx.sync()
    return time.perf_counter() - t0


def run_size(gb, size, args, rec):
    U, I, train, test = data(size, args.small)
    ioff, iusers = gb.transpose_csr(train[0], train[1], I)
    rng = np.random.default_rng(0)
    bpr = draw_trials("bpr", 10, rng, args.epochs)
    mix = bpr[:5] + draw_trials("als", 5, rng, args.als_epochs)
    out = {"shape": {"users": U, "items": I, "steps": int(train[0][-1])}, "trials": {"bpr": [kw for _, kw in bpr], "mix": [kw for _, kw in mix]}}
    with gb.Context(0) as ctx, gb.CFModel(ctx, U, I, 16, train[0], train[1], ioff, iusers) as m:
        n = int(train[0][-1])
        # (a) the solo d = 16 epoch
        m.init_normal(0.0, 0.001, 0)
        for e in range(2):
            m.bpr_epoch(0.05, 0.01, n, 900 + e)
        ms = []
        for e in range(10):
            ctx.timer_begin()
            m.bpr_epoch(0.05, 0.01, n, 1000 + e)
            ms.append(ctx.timer_end())
        out["a_epoch_ms"] = {"median": float(np.median(ms)), "min": float(min(ms)), "max": float(max(ms))}

        def seq(trials):
            for kind, kw in trials:
                m.fit(kind, test[0], test[1], None, None, **kw)

        def one(trials):
            m.fit_trials(trials, test[0], test[1], None, None)

        ways = {"b_sequential_s": lambda: seq(bpr), "c_batched_s": lambda: one(bpr),
                "d_mix_sequential_s": lambda: seq(mix), "d_mix_batched_s": lambda: one(mix)}
        for f in ways.values():   # warm-up
            f()
        times = {k: [] for k in ways}
        for _ in range(args.reps):
            for k, f in ways.items():
                times[k].append(timed(ctx, f))
        for k, v in times.items():
            out[k] = {"median": float(np.median(v)), "all": [float(x) for x in v]}
        out["speedup_bpr"] = out["b_sequential_s"]["median"] / out["c_batched_s"]["median"]
        out["speedup_mix"] = out["d_mix_sequential_s"]["median"] / out["d_mix_batched_s"]["median"]

        # the factors of (b) and (c), trial by trial
        _, fac = m.fit_trials(bpr, test[0], test[1], None, None, factors=True)
        rel = []
        for (kind, kw), (P, Q) in zip(bpr, fac):
            m.fit(kind, test[0], test[1], None, None, **kw)
            Ps, Qs = m.get_factors()
            big = max(np.abs(Ps).max(), np.abs(Qs).max())
            rel.append(float(max(np.abs(P.astype(np.float64) - Ps).max(), np.abs(Q.astype(np.float64) - Qs).max()) / big))
            del P, Q
        out["max_rel_factor_diff_b_vs_c"] = rel
        del fac

        # per-round device time, profiler on (a separate run: its numbers are not the timings above)
        if not args.no_profile:
            from torch.profiler import ProfilerActivity, profile

            rounds = (n + ROUND - 1) // ROUND
            prof_out = {}
            short = [(k, dict(kw, n_epochs=2)) for k, kw in bpr]
            for K in (1, 2, 5, 10):
                with profile(activities=[ProfilerActivity.CUDA]) as p:
                    m.fit_trials(short[:K], test[0], test[1], None, None)
                    if K == 1:
                        m.fit("bpr", test[0], test[1], None, None, **short[0][1])
                    ctx.sync()
                for ev in p.events():
                    if ev.device_type.name != "CUDA":
                        continue
                    for name in ("bpr_trials_round_kernel", "bpr_round_kernel"):
                        if name in ev.name and (name != "bpr_round_kernel" or "trials" not in ev.name):
                            key = f"{name}[{K}]" if name == "bpr_trials_round_kernel" else name
                            prof_out.setdefault(key, []).append(ev.device_time / rounds)
            out["us_per_round"] = {k: {"median": float(np.median(v)), "launches": len(v)} for k, v in prof_out.items()}
    rec[size] = out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="c1,c2")
    ap.add_argument("--epochs", type=int, default=100, help="BPR NEpochs of every trial (the reference's default)")
    ap.add_argument("--als-epochs", type=int, default=50, help="ALS NEpochs (the reference's default)")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--small", action="store_true", help="c2 at 50K users x 10K items (a rehearsal, not a measurement)")
    ap.add_argument("--no-profile", action="store_true")
    args = ap.parse_args()

    import gorse_b200 as gb

    rec = {"metric": "CF model search, 10 trials at d = 16", "card": card(), "epochs": args.epochs, "als_epochs": args.als_epochs,
           "reps": args.reps, "small": args.small}
    for size in args.sizes.split(","):
        run_size(gb, size, args, rec)
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
