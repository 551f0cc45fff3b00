#!/usr/bin/env python
"""tools/bpr_any_d_bench.py -- one atomic-scatter BPR epoch at d outside 16/32/64/128, on C2-shaped data.

  python tools/bpr_any_d_bench.py [--root DIR] [--small] [--dims 8,48] [--epochs 10]

--root imports gorse_b200 from another checkout (built with its own `make -C gorse_b200/csrc`), so that two versions of
the library can be timed on the same card in one session, alternating.  Data: bench.py's C2 (synth.make_feedback(1M,
100K, 11M, seed=1000, zipf_s=1, exact=True) + leave_one_out(seed=1001), 10M training triples); factors from
init_normal(0, 0.001).  Two warm-up epochs, then each timed epoch between device events (gorse_b200_ctx_timer_*).

One JSON line:
  card          name, power limit and SM clocks (nvidia-smi --query-gpu, read in the same run)
  ms_per_epoch  per d: median, min and max over the timed epochs
  launches      per d: kernel launches of one epoch
  repeat        per d: max |run 1 - run 2| / max |run 1| after 3 epochs from the same factors and seeds
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={q}", "--format=csv,noheader,nounits"], capture_output=True, text=True,
                         timeout=60).stdout.strip()
    name, power, sm, sm_max = [x.strip() for x in out.split(",")]
    return {"name": name, "power_limit_w": float(power), "sm_mhz": float(sm), "sm_max_mhz": float(sm_max)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--root", default=ROOT, help="checkout whose gorse_b200 is imported")
    ap.add_argument("--small", action="store_true", help="50K users x 10K items (a rehearsal, not a measurement)")
    ap.add_argument("--dims", default="8,48")
    ap.add_argument("--epochs", type=int, default=10)
    args = ap.parse_args()
    sys.path.insert(0, os.path.abspath(args.root))

    import gorse_b200 as gb
    from gorse_b200 import synth

    U, I, R = (50_000, 10_000, 500_000) if args.small else (1_000_000, 100_000, 10_000_000)
    off0, items0 = synth.make_feedback(U, I, R + U, seed=1000, zipf_s=1.0, exact=True)
    (off, items), _ = synth.leave_one_out(off0, items0, seed=1001)
    n = int(off[-1])
    lr, reg = 0.05, 0.01
    rec = {"metric": "atomic-scatter BPR epoch, ms", "root": os.path.abspath(args.root), "card": card(),
           "shape": {"users": U, "items": I, "steps": n, "small": args.small},
           "ms_per_epoch": {}, "launches": {}, "repeat": {}}
    with gb.Context(0) as ctx:
        for d in [int(x) for x in args.dims.split(",")]:
            with gb.CFModel(ctx, U, I, d, off, items) as m:
                m.init_normal(0.0, 0.001, 0)
                P0, Q0 = m.get_factors()
                for e in range(2):
                    m.bpr_epoch(lr, reg, n, 900 + e)
                ms = []
                for e in range(args.epochs):
                    l0 = ctx.launch_count()
                    ctx.timer_begin()
                    m.bpr_epoch(lr, reg, n, 1000 + e)
                    ms.append(ctx.timer_end())
                    launches = ctx.launch_count() - l0
                runs = []
                for _ in range(2):
                    m.set_factors(P0, Q0)
                    for e in range(3):
                        m.bpr_epoch(lr, reg, n, 500 + e)
                    runs.append(m.get_factors())
            (P1, Q1), (P2, Q2) = runs
            big = max(np.abs(P1).max(), np.abs(Q1).max())
            diff = max(np.abs(P1.astype(np.float64) - P2).max(), np.abs(Q1.astype(np.float64) - Q2).max())
            rec["ms_per_epoch"][d] = {"median": float(np.median(ms)), "min": float(min(ms)), "max": float(max(ms))}
            rec["launches"][d] = int(launches)
            rec["repeat"][d] = float(diff / big)
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
