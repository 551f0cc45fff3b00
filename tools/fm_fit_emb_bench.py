#!/usr/bin/env python3
"""Times gorse_b200_fm_fit_emb: a CTR training set with one item-embedding slot (default 768 wide over 100K items, k = 16,
Adam, batches of 1024).  The first 3 steps are checked bit for bit against the CPU restatement; then whole epochs are timed
with the epoch as one CUDA graph and with plain launches, one evaluation of the test rows, every kernel of an epoch through
torch.profiler (a run of its own), and the slot-free model through the new entry against gorse_b200_fm_fit, alternating,
with the spread of both.  Prints one JSON line with the card's name, power limit, its maximum SM clock and the SM clock
read right after the timed runs.  Needs a GPU."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import fm_oracle  # noqa: E402
import gorse_b200 as gb  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=200_000)
    ap.add_argument("--test-rows", type=int, default=20_000)
    ap.add_argument("--features", type=int, default=200_000)
    ap.add_argument("--items", type=int, default=100_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--factors", type=int, default=16)
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--epochs", type=int, default=3)
    a = ap.parse_args()
    def smi(q):
        return subprocess.check_output(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], text=True).strip()

    card = smi("name,power.limit,clocks.max.sm")
    rng = np.random.default_rng(2)
    nf, k, dims = a.features, a.factors, (a.dim,)
    tr, te = fm_oracle.random_ctr(rng, nf, a.rows, labels=10), fm_oracle.random_ctr(rng, nf, a.test_rows, labels=10)
    emb = fm_oracle.random_embeddings(rng, a.items, dims, a.rows, a.test_rows)
    p0 = fm_oracle.init_params(rng, nf, k, emb_dims=dims)
    out = {"card_name_power_limit_max_sm_clock": card, "rows": a.rows, "dim": a.dim, "k": k, "batch": a.batch, "steps_per_epoch": -(-a.rows // a.batch)}
    with gb.Context(0) as ctx:
        def fit(emb_, p, epochs, verbose=1000, **kw):
            t = gb.FMTrainer(ctx, nf, 12, n_factors=k, n_epochs=epochs, batch_size=a.batch, verbose=verbose, patience=0, **kw)
            t0 = time.perf_counter()
            r = t.fit_emb(tr, te, p, emb_.dims, emb_.table, emb_.mask, emb_.train_rows, emb_.test_rows, moments=True)
            return r, time.perf_counter() - t0   # the call ends with a device synchronise and the copy of the parameters

        (pg, _, mg), _ = fit(emb, p0, 1, max_steps=3)
        po, _, mo = fm_oracle.fit(nf, 12, tr, te, p0, n_factors=k, n_epochs=1, batch_size=a.batch, verbose=1000, patience=0, max_steps=3, emb=emb)
        assert pg.tobytes() == po.tobytes() and mg.tobytes() == mo.tobytes(), "the first 3 steps differ from the restatement"
        out["checked_steps"] = 3

        def per_epoch(emb_, p, **kw):   # the time E epochs add over 1: set-up and the evaluations cancel
            fit(emb_, p, 1, **kw)
            one = min(fit(emb_, p, 1, **kw)[1] for _ in range(2))
            many = min(fit(emb_, p, 1 + a.epochs, **kw)[1] for _ in range(2))
            return (many - one) / a.epochs

        out["epoch_s_graph"] = per_epoch(emb, p0)
        os.environ["GORSE_B200_FM_FIT_NO_GRAPH"] = "1"
        out["epoch_s_plain_launches"] = per_epoch(emb, p0)
        del os.environ["GORSE_B200_FM_FIT_NO_GRAPH"]
        out["step_ms_graph"] = 1e3 * out["epoch_s_graph"] / out["steps_per_epoch"]
        # one evaluation of the test rows: what evaluating after every epoch adds, per epoch
        n_ev = 1 + a.epochs
        every = min(fit(emb, p0, n_ev, verbose=1)[1] for _ in range(2))
        last = min(fit(emb, p0, n_ev)[1] for _ in range(2))
        out["test_rows"], out["evaluation_s"] = a.test_rows, (every - last) / (n_ev - 1)
        out["sm_clock_after_timed_runs"] = smi("clocks.sm")
        # every kernel of one fit of 1 epoch (2 evaluations), in a run of its own: tracing slows the host
        import torch
        from torch.profiler import ProfilerActivity, profile

        torch.cuda.init()
        os.environ["GORSE_B200_FM_FIT_NO_GRAPH"] = "1"
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fit(emb, p0, 1)
        del os.environ["GORSE_B200_FM_FIT_NO_GRAPH"]
        kern = {}
        for ev in prof.key_averages():
            if "fm_fit" in ev.key:
                us = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
                kern[ev.key.split("(")[0].split("::")[-1]] = {"launches": ev.count, "mean_us": round(us / max(ev.count, 1), 2)}
        out["kernels_one_epoch_two_evaluations"] = kern
        # the slot-free model: the new entry against gorse_b200_fm_fit, alternating, 20 epochs a call
        none = fm_oracle.Embeddings((), [], None, np.zeros(a.rows, np.int32), np.zeros(a.test_rows, np.int32))
        q0 = p0[:1 + nf * k + nf]
        t_new, t_old = [], []
        for _ in range(5):
            t_new.append(fit(none, q0, 20)[1])
            t = gb.FMTrainer(ctx, nf, 12, n_factors=k, n_epochs=20, batch_size=a.batch, verbose=1000, patience=0)
            t0 = time.perf_counter()
            t.fit(tr, te, q0)
            t_old.append(time.perf_counter() - t0)
        out["slot_free_20_epochs_s_new_entry_min_max"] = [min(t_new), max(t_new)]
        out["slot_free_20_epochs_s_fm_fit_min_max"] = [min(t_old), max(t_old)]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
