"""FM training on the H100: gorse_b200_fm_fit (AFM.Fit without embedding slots) on a synthetic CTR set shaped like C2.

Rows: the first --positives of C2's training feedback (1M users, 100K items, Zipf items, seed 1000) as positives (target +1),
as many negatives (a uniform item for the same user, target -1), each row a user id, an item id, and 0-10 labels of the
user and 0-10 of the item from --labels label features (1 / 0.5 / 0.25-scaled values), in a fixed shuffled order.  The test
set is --test further rows built the same way.  k = --k, Adam, batch 1024.
Reports ms per epoch and per step for the CUDA-graph epoch and for plain launches, ms per evaluation, and the C
restatement on one thread (fm_oracle, not Go) on --cpu-rows rows as the CPU figure.  Before timing, --check steps are
compared bit for bit with the restatement on a slice.  Prints one JSON line.

  python tools/fm_fit_bench.py
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


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={q}", "--format=csv,noheader,nounits"], capture_output=True, text=True,
                         check=True).stdout.strip()
    name, power, sm, sm_max = [x.strip() for x in out.split(",")]
    return {"name": name, "power_limit_w": float(power), "sm_mhz": float(sm), "sm_max_mhz": float(sm_max)}


def make_rows(args):
    from gorse_b200 import synth

    U, I, L = 1_000_000, 100_000, args.labels
    n_pos = args.positives + args.test // 2
    off, items = synth.make_feedback(U, I, max(n_pos, U) + U // 10, seed=1000, zipf_s=1.0, exact=True)
    users = np.repeat(np.arange(U, dtype=np.int64), np.diff(off))
    rng = np.random.default_rng(1001)
    pick = rng.permutation(users.size)[:n_pos]
    pu, pi = users[pick], items[pick].astype(np.int64)
    nu, ni = pu, rng.integers(0, I, n_pos)
    u = np.concatenate([pu, nu])
    it = np.concatenate([pi, ni])
    tgt = np.concatenate([np.ones(n_pos, np.float32), -np.ones(n_pos, np.float32)])
    order = rng.permutation(u.size)
    u, it, tgt = u[order], it[order], tgt[order]
    # labels of a user / item: 0-10 fixed features per id (features U + I .. U + I + L)
    ucnt, icnt = rng.integers(0, 11, U), rng.integers(0, 11, I)
    n = u.size
    lens = 2 + ucnt[u] + icnt[it]
    roff = np.zeros(n + 1, np.int64)
    np.cumsum(lens, out=roff[1:])
    idx = np.empty(int(roff[-1]), np.int32)
    val = np.empty(int(roff[-1]), np.float32)
    idx[roff[:-1]] = u
    idx[roff[:-1] + 1] = U + it
    val[roff[:-1]] = 1.0
    val[roff[:-1] + 1] = 1.0
    lab_pos = np.ones(idx.size, bool)
    lab_pos[roff[:-1]] = False
    lab_pos[roff[:-1] + 1] = False
    m = int(lab_pos.sum())
    idx[lab_pos] = U + I + rng.integers(0, L, m)
    val[lab_pos] = rng.choice(np.array([1.0, 0.5, 0.25], np.float32), m)
    nf = U + I + L
    te_n = args.test
    tr_n = n - te_n

    def part(a, b):
        o = roff[a:b + 1] - roff[a]
        return o, idx[roff[a]:roff[b]], val[roff[a]:roff[b]], tgt[a:b]

    return nf, part(0, tr_n), part(tr_n, n)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--positives", type=int, default=1_000_000)
    ap.add_argument("--test", type=int, default=200_000)
    ap.add_argument("--labels", type=int, default=1000)
    ap.add_argument("--k", type=int, default=16)
    ap.add_argument("--epochs", type=int, default=3)
    ap.add_argument("--cpu-rows", type=int, default=20_000)
    ap.add_argument("--check", type=int, default=3)
    args = ap.parse_args()

    import fm_oracle
    import gorse_b200 as gb

    t0 = time.time()
    nf, tr, te = make_rows(args)
    n_train = len(tr[0]) - 1
    D = int(np.max(np.diff(tr[0])))
    rng = np.random.default_rng(7)
    p0 = fm_oracle.init_params(rng, nf, args.k)
    prep_s = time.time() - t0
    kw = dict(n_factors=args.k, lr=0.001, reg=0.0002, batch_size=1024, patience=0)
    res = {"rows": n_train, "test_rows": len(te[0]) - 1, "n_features": nf, "D": D, "k": args.k, "prep_s": round(prep_s, 1)}
    with gb.Context(0) as ctx:
        # bit-for-bit check of the first steps on a slice (the restatement walks every parameter each step)
        sl = min(n_train, 1024 * args.check)
        sub = (tr[0][:sl + 1], tr[1][:tr[0][sl]], tr[2][:tr[0][sl]], tr[3][:sl])
        tsub = (te[0][:1001], te[1][:te[0][1000]], te[2][:te[0][1000]], te[3][:1000])
        pg, _, mg = gb.FMTrainer(ctx, nf, D, n_epochs=1, verbose=1, **kw).fit(sub, tsub, p0, moments=True)
        po, _, mo = fm_oracle.fit(nf, D, sub, tsub, p0, n_epochs=1, verbose=1, **kw)
        res["checked_steps"] = args.check
        res["check_bit_identical"] = bool(pg.tobytes() == po.tobytes() and mg.tobytes() == mo.tobytes())
        n_batches = (n_train + 1023) // 1024
        for mode in ("graph", "launches"):
            if mode == "launches":
                os.environ["GORSE_B200_FM_FIT_NO_GRAPH"] = "1"
            # one epoch, then E + 1 epochs evaluated only on the last: the difference is E epochs
            t = time.time()
            gb.FMTrainer(ctx, nf, D, n_epochs=1, verbose=1, **kw).fit(tr, te, p0)
            one = time.time() - t
            t = time.time()
            _, r, _ = gb.FMTrainer(ctx, nf, D, n_epochs=args.epochs + 1, verbose=1000, **kw).fit(tr, te, p0)
            many = time.time() - t
            epoch_ms = (many - one) / args.epochs * 1e3
            res[f"{mode}_ms_per_epoch"] = round(epoch_ms, 2)
            res[f"{mode}_ms_per_step"] = round(epoch_ms / n_batches, 4)
            res[f"{mode}_auc_after_{args.epochs + 1}"] = float(r["auc"])
            if mode == "graph":   # the same E + 1 epochs evaluated after every one: E more evaluations
                t = time.time()
                gb.FMTrainer(ctx, nf, D, n_epochs=args.epochs + 1, verbose=1, **kw).fit(tr, te, p0)
                res["ms_per_eval"] = round(((time.time() - t) - many) / args.epochs * 1e3, 2)
                t = time.time()
                gb.FMTrainer(ctx, nf, D, n_epochs=0, verbose=1, **kw).fit(tr, te, p0)
                res["ms_upload_and_first_eval"] = round((time.time() - t) * 1e3, 1)
            os.environ.pop("GORSE_B200_FM_FIT_NO_GRAPH", None)
    # CPU figure: the C restatement on one thread, one epoch over --cpu-rows rows (every step walks all parameters)
    c = min(args.cpu_rows, n_train)
    csub = (tr[0][:c + 1], tr[1][:tr[0][c]], tr[2][:tr[0][c]], tr[3][:c])
    t = time.time()
    fm_oracle.fit(nf, D, csub, tsub, p0, n_epochs=1, verbose=1000, **kw)
    cpu = time.time() - t
    res["cpu_restatement_ms_per_step"] = round(cpu / ((c + 1023) // 1024) * 1e3, 2)
    try:
        res["card"] = card()
    except Exception as e:  # noqa: BLE001
        res["card"] = str(e)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
