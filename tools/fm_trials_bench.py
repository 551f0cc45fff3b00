"""FM model search on the H100: ten trials of AFM's ModelSearch as ten solo fits (gorse_b200_fm_fit / _fit_emb) and as one
gorse_b200_fm_fit_trials call.

The trials are drawn as AFM.SuggestParams draws them (model/ctr/fm.go:79-87): Lr, Reg and InitStdDev log-uniform in
[0.001, 0.1] from --seed, NFactors 16, Adam, batch 1024, --epochs epochs evaluated at 0 and on the last.  Shapes:
  large  tools/fm_fit_bench.py's rows: 2M training rows, 1.1M features (DESIGN §8.5's shape)
  small  a ranker dataset with --small-features features and --small-rows rows, where launches dominate
  slot   tools/fm_fit_emb_bench.py's shape with one 768-dim item-embedding slot
Before timing, every trial of the batched call is compared bit for bit with its solo fit.  Each way is timed --repeat
times, alternating, host in to host out; the medians and the spreads (max - min) are reported with the card's name,
power limit and SM clock read in the same run.  Prints one JSON line.

  python tools/fm_trials_bench.py [--shapes large,small,slot]
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
sys.path.insert(0, os.path.join(ROOT, "tools"))


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={q}", "--format=csv,noheader,nounits"], capture_output=True, text=True,
                         check=True).stdout.strip()
    name, power, sm, sm_max = [x.strip() for x in out.split(",")]
    return {"name": name, "power_limit_w": float(power), "sm_mhz": float(sm), "sm_max_mhz": float(sm_max)}


def suggest(rng, n):
    """SuggestLogFloat(0.001, 0.1) for Lr, Reg and InitStdDev, n times"""
    draw = lambda: float(np.exp(rng.uniform(np.log(0.001), np.log(0.1))))   # noqa: E731
    return [(draw(), draw(), draw()) for _ in range(n)]


def shape(name, a):
    import fm_oracle

    rng = np.random.default_rng(a.seed)
    if name == "large":
        import fm_fit_bench

        nf, tr, te = fm_fit_bench.make_rows(argparse.Namespace(positives=1_000_000, test=200_000, labels=1000))
        return nf, int(np.max(np.diff(tr[0]))), tr, te, None
    if name == "small":
        nf = a.small_features
        tr, te = fm_oracle.random_ctr(rng, nf, a.small_rows, labels=10), fm_oracle.random_ctr(rng, nf, a.small_rows // 10, labels=10)
        return nf, 12, tr, te, None
    nf, rows, test_rows = 200_000, 200_000, 20_000
    tr, te = fm_oracle.random_ctr(rng, nf, rows, labels=10), fm_oracle.random_ctr(rng, nf, test_rows, labels=10)
    return nf, 12, tr, te, fm_oracle.random_embeddings(rng, 100_000, (768,), rows, test_rows)


def run_shape(gb, ctx, name, a):
    import fm_oracle

    nf, nd, tr, te, emb = shape(name, a)
    dims = () if emb is None else tuple(int(d) for d in emb.dims)
    rng = np.random.default_rng(a.seed + 1)
    draws = suggest(rng, a.trials)
    pins = [fm_oracle.init_params(rng, nf, 16, std, dims) for _, _, std in draws]
    trials = [dict(lr=lr, reg=reg) for lr, reg, _ in draws]
    base = dict(n_factors=16, n_epochs=a.epochs, batch_size=1024, verbose=a.epochs, patience=0)
    e = None if emb is None else (emb.dims, emb.table, emb.mask, emb.train_rows, emb.test_rows)

    def solo(i):
        t = gb.FMTrainer(ctx, nf, nd, **{**base, **trials[i]})
        if emb is None:
            return t.fit(tr, te, pins[i])
        return t.fit_emb(tr, te, pins[i], emb.dims, emb.table, emb.mask, emb.train_rows, emb.test_rows)

    def batched():
        return gb.FMTrainer(ctx, nf, nd, **base).fit_trials(trials, tr, te, pins, emb=e)

    out = batched()   # also the warm-up of both ways
    for i in range(a.trials):
        ps, rs, _ = solo(i)
        assert out[i][0].tobytes() == ps.tobytes() and out[i][1] == rs, f"{name}: trial {i} differs from its solo fit"
    times = {"solo": [], "batched": []}
    for _ in range(a.repeat):
        t = time.perf_counter()
        for i in range(a.trials):
            solo(i)
        times["solo"].append(time.perf_counter() - t)
        t = time.perf_counter()
        batched()
        times["batched"].append(time.perf_counter() - t)
    r = {"rows": len(tr[0]) - 1, "n_features": nf, "dims": list(dims), "epochs": a.epochs, "trials": a.trials, "bit_identical": True}
    for k, v in times.items():
        r[f"{k}_s_median"] = round(float(np.median(v)), 3)
        r[f"{k}_s_spread"] = round(float(np.max(v) - np.min(v)), 3)
    r["speedup"] = round(r["solo_s_median"] / r["batched_s_median"], 2)
    r["auc"] = [round(float(o[1]["auc"]), 4) for o in out]
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="large,small,slot")
    ap.add_argument("--trials", type=int, default=10)
    ap.add_argument("--epochs", type=int, default=3)
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--seed", type=int, default=5)
    ap.add_argument("--small-features", type=int, default=3000)
    ap.add_argument("--small-rows", type=int, default=20_000)
    a = ap.parse_args()

    import gorse_b200 as gb

    res = {"card": card()}
    with gb.Context(0) as ctx:
        for name in a.shapes.split(","):
            res[name] = run_shape(gb, ctx, name, a)
    res["card_after"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
