"""`gorse-bench reranker`'s AFM scoring on the H100: gorse_b200_fm_gauc on a synthetic CTR dataset at the C2 shape.

Data: --users users and --items items; --positives positive feedback with Zipf(1) item popularity and --reads read
(negative) feedback drawn the same way (gorse_b200.synth.make_feedback), seeded distinct timestamps, and per user the
newest 20 % as the test side.  A row is [user, item, the user's labels, the item's labels]: 0 .. 4 labels per user and per
item from --labels label features, value 1 or N(0, 1) as fm_oracle.random_ctr draws them.  feedback_count comes from the
train side's positives, context_size = 100.
Models: k = 16 without slots, and with one 768-dim slot (a bf16 table row per item); Init's parameters
(fm_oracle.init_params); num_dimension = the longest row.
Before timing, the --check seeded users are scored by the CPU restatement (fmo_batch_predict on the chunks of
batch_size rows that hold their rows, then fmo_gauc) and must agree bit for bit.  The restatement's single-thread
milliseconds per user over those chunks are reported (the CPU restatement's, not Go's).
Reported per model: host-in to host-out seconds (median of --repeat after a warm-up), every kernel's device time from a
separate torch.profiler run, and the card's name, power limit and SM clock read in the same run.  Prints one JSON line.

  python tools/fm_gauc_bench.py [--users 1000000] [--check 64]
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


def expand(counts):
    """(group of every element, its place in the group) for groups of the given sizes"""
    counts = np.asarray(counts, np.int64)
    g = np.repeat(np.arange(counts.size), counts)
    start = np.cumsum(counts) - counts
    return g, np.arange(int(counts.sum())) - start[g]


def labels(rng, n, first, n_labels):
    cnt = rng.integers(0, 5, n)
    off = np.zeros(n + 1, np.int64)
    np.cumsum(cnt, out=off[1:])
    idx = (first + rng.integers(0, n_labels, int(off[-1]))).astype(np.int32)
    val = np.where(rng.random(int(off[-1])) < 0.3, rng.standard_normal(int(off[-1])), 1.0).astype(np.float32)
    return off, idx, val


def dataset(a):
    from gorse_b200 import synth

    rng = np.random.default_rng(a.seed)
    U, I = a.users, a.items
    parts = []
    for n, seed, t in ((a.positives, a.seed, 1.0), (a.reads, a.seed + 1, -1.0)):
        off, items = synth.make_feedback(U, I, n, seed=seed)
        parts.append((np.repeat(np.arange(U), np.diff(off)), items, np.full(items.size, t, np.float32)))
    user, item, tgt = (np.concatenate(x) for x in zip(*parts))
    order = np.lexsort((rng.permutation(user.size), user))   # per user, oldest first
    user, item, tgt = user[order], item[order], tgt[order]
    deg = np.bincount(user, minlength=U)
    _, place = expand(deg)
    test = place >= deg[user] - (deg[user] // 5)
    fb = np.bincount(user[~test & (tgt > 0)], minlength=U).astype(np.int64)
    user, item, tgt = user[test], item[test], tgt[test]
    ul, il = labels(rng, U, U + I, a.labels), labels(rng, I, U + I, a.labels)
    uc, ic = np.diff(ul[0])[user], np.diff(il[0])[item]
    lens = 2 + uc + ic
    off = np.zeros(user.size + 1, np.int64)
    np.cumsum(lens, out=off[1:])
    idx, val = np.zeros(int(off[-1]), np.int32), np.ones(int(off[-1]), np.float32)
    idx[off[:-1]], idx[off[:-1] + 1] = user, U + item
    for c, (lo, li, lv), who, at in ((uc, ul, user, 2), (ic, il, item, None)):
        r, k = expand(c)
        pos = off[:-1][r] + (2 if at else 2 + uc[r]) + k
        src = lo[who[r]] + k
        idx[pos], val[pos] = li[src], lv[src]
    return (off, idx, val, tgt), item.astype(np.int32), fb, U + I + a.labels


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--users", type=int, default=1_000_000)
    ap.add_argument("--items", type=int, default=100_000)
    ap.add_argument("--positives", type=int, default=10_000_000)
    ap.add_argument("--reads", type=int, default=10_000_000)
    ap.add_argument("--labels", type=int, default=1000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--batch-size", type=int, default=1024)
    ap.add_argument("--check", type=int, default=64)
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()

    import torch

    import fm_oracle
    import gorse_b200 as gb

    t0 = time.perf_counter()
    te, item, fb, nf = dataset(a)
    off, idx, val, tgt = te
    n = off.size - 1
    nd, k, bs = int(np.diff(off).max()), 16, a.batch_size
    users = idx[off[:-1]]
    print(f"dataset: {n} test rows, {nf} features, {time.perf_counter() - t0:.1f} s", file=sys.stderr, flush=True)
    rng = np.random.default_rng(a.seed + 7)
    sample = rng.choice(np.unique(users), size=min(a.check, a.users), replace=False)
    table = fm_oracle.to_bf16(rng.standard_normal((a.items, a.dim), dtype=np.float32))
    rows = []
    with gb.Context(0) as ctx:
        for dims in ((), (a.dim,)):
            params = fm_oracle.init_params(rng, nf, k, 0.01, dims)
            emb = (dims, [table] if dims else [], None, item) if dims else None
            # the restatement on the chunks that hold the sampled users' rows
            got = gb.ranker_gauc(ctx, nf, k, nd, params, te, a.users, fb, 100, bs, emb, predictions=True)
            chunks = np.unique(np.flatnonzero(np.isin(users, sample)) // bs)
            t0 = time.perf_counter()
            model = fm_oracle.Model(nf, k, nd, bs, dims, params)
            for c in chunks:
                r = np.arange(c * bs, min((c + 1) * bs, n))
                es = [(table[item[r]].astype(np.uint32) << 16).view(np.float32)] if dims else ()
                p = model.batch_predict([(idx[off[i]:off[i + 1]], val[off[i]:off[i + 1]]) for i in r], es)
                assert p.tobytes() == got["predictions"][r].tobytes(), ("predictions", dims, int(c))
            r = np.flatnonzero(np.isin(users, sample))
            g, uo, co, ao = fm_oracle.gauc(got["predictions"][r], users[r], tgt[r], a.users, fb, 100)
            cpu_ms = (time.perf_counter() - t0) * 1e3
            in_chunks = np.unique(users[np.concatenate([np.arange(c * bs, min((c + 1) * bs, n)) for c in chunks])]).size
            mine = np.isin(got["users"], uo)
            assert got["users"][mine].tolist() == uo.tolist() and got["auc"][mine].tobytes() == ao.tobytes(), ("per-user AUC", dims)
            times = []
            for _ in range(a.repeat + 1):
                t1 = time.perf_counter()
                res = gb.ranker_gauc(ctx, nf, k, nd, params, te, a.users, fb, 100, bs, emb)
                times.append(time.perf_counter() - t1)
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                gb.ranker_gauc(ctx, nf, k, nd, params, te, a.users, fb, 100, bs, emb)
            dev = {}
            for ev in prof.events():
                if ev.device_type == torch.autograd.DeviceType.CUDA:
                    name = ev.name.split("(")[0].split("<")[0].replace("gb::fmfit::", "")
                    dev[name] = dev.get(name, 0.0) + ev.device_time_total / 1e3
            rows.append({"slots": list(dims), "gauc": res["gauc"], "stats": res["stats"], "host_s_median": float(np.median(times[1:])),
                         "host_s_spread": float(max(times[1:]) - min(times[1:])), "device_ms_by_kernel": {kk: round(v, 3) for kk, v in dev.items()},
                         "device_ms_all_kernels": sum(dev.values()), "checked_users": int(uo.size), "checked_chunks": int(chunks.size),
                         "cpu_restatement_single_thread_ms_per_user": cpu_ms / max(in_chunks, 1)})
            print(json.dumps(rows[-1]), file=sys.stderr, flush=True)
    print(json.dumps({"bench": "fm_gauc", "card": card(), "users": a.users, "items": a.items, "test_rows": n, "features": nf,
                      "num_dimension": nd, "n_factors": k, "batch_size": bs, "rows": rows}))


if __name__ == "__main__":
    main()
