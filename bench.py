#!/usr/bin/env python
"""bench.py -- BASELINE.json's headline metric ("BPR-MF triples/sec and item-to-item top-k vectors/sec at 1/2/4/8 GPUs").

  python bench.py [--gpus N] [--steps K] [--warmup W] [--impl ours|reference] [--workload c2|c3|c4|c5|c1|small]
                  [--dump-outputs DIR]

Default: BASELINE configs[1] ("c2": BPR, 1M users x 100K items x 10M feedback, d=64).  A "step" is
one BPR epoch = |R| fused sample-gather-dot-sigmoid-scatter triples.  For N > 1 (torchrun, one rank per GPU) the workload
is weak-scaled: every rank owns 1M users / 10M feedback and hands the C ABI ONLY ITS OWN ROWS; the item table is replicated
and its deltas are exchanged (NCCL) once per epoch.

One JSON line on rank 0 (DESIGN.md "measurement" explains every key):
  value      triples/s, device-timed (CUDA events on the library's stream, max over ranks), inputs resident in HBM
  e2e        the same metric through the reference-facing call: cf_create from HOST buffers (CSR H2D) + gorse_b200_bpr_fit
             (Init, NEpochs epochs, Evaluate every Verbose epochs like cf.BPR.Fit) + get_factors (D2H), wall clock
  roofline   algorithmic bytes / epoch duration against the measured HBM copy peak
  also       at N = 1: compact records of BASELINE configs[2] (eALS, "c3") and configs[3] (all-pairs top-k, "c4"), each
             with its own value / e2e / roofline / cpu_baseline / clocks, so that the default line carries the second half
             of the metric too (--no-also skips them)
`--dump-outputs DIR` writes what the timed path computed in its last timed step as DIR/<name>.npy (float32 / float64; fixed,
seeded row samples of the large tables, under 64 MB in all), so that two builds can be compared output for output: the
inputs depend only on the arguments.
`--impl reference` times the reference's CPU path for the same workload (oracle/_ref = the reference's own C kernels
compiled here; threads pinned, median of the samples).
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

WORKLOADS = {
    # name: (users per rank, items, TRAIN feedback per rank, d, description)
    "c2": (1_000_000, 100_000, 10_000_000, 64, "BPR 1M users x 100K items x 10M feedback, d=64 (BASELINE configs[1])"),
    "c5": (1_250_000, 1_000_000, 25_000_000, 128, "BPR 10M users x 1M items x 200M feedback, d=128, user rows sharded over 8 ranks (BASELINE configs[4]); per rank 1.25M users / 25M feedback"),
    "c1": (943, 1_682, 100_000, 16, "BPR ml-100k-shaped surrogate 943 x 1682 x 100K, d=16 (BASELINE configs[0])"),
    "small": (50_000, 10_000, 500_000, 64, "reduced smoke size (NOT a bench number)"),
}
LR, REG = 0.05, 0.01            # BPR defaults, model/cf/model.go:391-392
INIT_STD = 0.001                # :394
ALS_REG, ALS_ALPHA, ALS_STD = 0.06, 0.001, 0.1   # ALS defaults, :582-585
ZIPF_S = 1.0                    # item popularity skew of the synthetic feedback (SURVEY 8d)


def bytes_per_triple(d):
    return 6 * d * 4 + 12       # SURVEY 8(d): 3 rows read + 3 rows written + 3 ids


def read_peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    hbm, tf, src = 3350.0, 989.0, "H100 SXM data sheet (HBM3 bandwidth, dense bf16), not measured"
    if os.path.exists(p):
        try:
            j = json.load(open(p))
            hbm, tf, src = float(j["hbm_gbs"]), float(j.get("bf16_tflops_sustained", tf)), "measured (MEASURED_PEAKS.json)"
        except Exception:
            pass
    return hbm, tf, src


def bpr_config(wl, world):
    """The `config` object of the JSON line -- ONE function for both arms so that their dicts are key- and value-identical."""
    upr, n_items, fpr, d, desc = WORKLOADS[wl]
    return {"workload": desc, "users_per_rank": upr, "items": n_items, "train_feedback_per_rank": fpr, "d": d, "lr": LR, "reg": REG,
            "item_popularity": f"zipf({ZIPF_S})", "split": "leave-one-out (dataset.SplitCF(0, seed)): one test item per user beside the train rows",
            "cache": "inputs larger than L2: the user table (256 MB per rank at c2) exceeds the 50 MB L2; no flush between steps"}


class ClockSampler:
    """nvidia-smi clocks / throttle reasons sampled DURING the timed region."""
    Q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, index=0):
        self.rows, self.proc = [], None
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--id={index}", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits",
                                          "-lms", "50"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.t = threading.Thread(target=self._read, daemon=True)
            self.t.start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append((time.time(), [x.strip() for x in line.split(",")]))

    def stop(self, t0, t1):
        if not self.proc:
            return None
        time.sleep(0.12)
        for _ in range(20):                      # nvidia-smi needs 0.1-0.3 s for its first line: never return without one
            if self.rows:
                break
            time.sleep(0.05)
        self.proc.terminate()
        # samples inside the timed region; a region shorter than the 50 ms period takes the samples next to it
        rows = ([r for (t, r) in self.rows if t0 - 0.05 <= t <= t1 + 0.12 and len(r) >= 7]
                or [r for (t, r) in sorted(self.rows, key=lambda x: abs(x[0] - 0.5 * (t0 + t1)))[:2] if len(r) >= 7])
        if not rows:
            return None
        sm = sorted(float(r[0]) for r in rows)
        reasons = [n for k, n in ((3, "hw_slowdown"), (4, "hw_thermal_slowdown"), (5, "sw_thermal_slowdown"), (6, "sw_power_cap"))
                   if any(r[k].lower().startswith("active") for r in rows)]
        return {"sm_mhz": sm[len(sm) // 2], "sm_max_mhz": float(rows[0][1]), "reasons": reasons, "samples": len(rows)}


DUMP_ROWS = 16384   # rows of a table --dump-outputs keeps (a fixed, seeded sample of the larger ones)


def dump_outputs(args, name, arrays):
    """DIR/<name>_<key>.npy for every array; tables with more than DUMP_ROWS rows are sampled with a fixed seed"""
    if not args.dump_outputs:
        return
    os.makedirs(args.dump_outputs, exist_ok=True)
    for key, a in arrays.items():
        a = np.asarray(a)
        if a.shape[0] > DUMP_ROWS:
            a = a[np.sort(np.random.default_rng(20261015).choice(a.shape[0], DUMP_ROWS, replace=False))]
        a = a.astype(np.float32 if a.dtype in (np.float32, np.float16) else np.float64)
        np.save(os.path.join(args.dump_outputs, f"{name}_{key}.npy"), a)


def dist_env():
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", str(rank)))
    return rank, world, local


_DATA_CACHE = {}


def get_data(wl, seed):
    """(train CSR, test CSR) of one rank's users: |train| = the workload's feedback count, one held-out item per user."""
    from gorse_b200 import synth

    if (wl, seed) not in _DATA_CACHE:
        upr, n_items, fpr, d, _ = WORKLOADS[wl]
        off, items = synth.make_feedback(upr, n_items, fpr + upr, seed=seed, zipf_s=ZIPF_S, exact=True)
        _DATA_CACHE[(wl, seed)] = synth.leave_one_out(off, items, seed=seed + 1)
    return _DATA_CACHE[(wl, seed)]


def make_shard(wl, rank, world):
    """This rank's rows of the global user CSR (the C ABI takes ONLY the rank's own rows in a distributed context):
    users [rank*upr, (rank+1)*upr) of n_users = upr*world, seeded per rank."""
    upr, n_items, fpr, d, _ = WORKLOADS[wl]
    (off_l, items), _ = get_data(wl, 1000 + rank)
    return upr * world, n_items, d, off_l, items


# ---------------------------------------------------------------------------------------------------------------------
# CPU arms (the only places that touch oracle/: `cpu_baseline` and `--impl reference`)
# ---------------------------------------------------------------------------------------------------------------------
_CPU_CACHE = {}


def cpu_bpr(wl, seconds_budget=2.0, samples=5):
    """The reference's CPU path for the same step on this box's host cores: per triple the reference's own call sequence
    (2x dot, exp, 3 row copies, 10 vector ops, model/cf/model.go:469-488) through the reference's C kernels (oracle/_ref,
    compiled from the reference's common/floats/src) when present and the CPU has AVX-512, else through the oracle port;
    Hogwild over all host cores, worker t pinned to the t-th allowed CPU, tables first-touched page-interleaved over the
    workers; `samples` bounded samples of one epoch, MEDIAN reported."""
    import oracle

    upr, n_items, fpr, d, _ = WORKLOADS[wl]
    cores = len(os.sched_getaffinity(0))
    if wl not in _CPU_CACHE:
        (off, items), _ = get_data(wl, 1000)
        P = oracle.fill_normal_interleaved((upr, d), INIT_STD, 1, cores)
        Q = oracle.fill_normal_interleaved((n_items, d), INIT_STD, 2, cores)
        _CPU_CACHE[wl] = (off, items, P, Q, np.nonzero(np.diff(off) > 0)[0].astype(np.int32))
    off, items, P, Q, active = _CPU_CACHE[wl]
    kind, use_ref = "port", False
    if oracle.ref_available() and "avx512f" in open("/proc/cpuinfo").read() and oracle.ref_bind():
        kind, use_ref = "reference", True
    probe = 400_000
    sec = oracle.bpr_epoch_threads(P, Q, off, items, active, 1, probe, LR, REG, cores, use_ref)   # warms caches, sizes the sample
    n = int(min(off[-1] * 4, max(probe, probe * seconds_budget / max(sec, 1e-6))))
    secs = sorted(oracle.bpr_epoch_threads(P, Q, off, items, active, 2 + s, n, LR, REG, cores, use_ref) for s in range(samples))
    med = secs[len(secs) // 2]
    return {"value": n / med, "unit": "triples/s", "cores": cores, "kind": kind,
            "sample": f"median of {samples} samples of {n} sampled triples of the step (min {n / secs[-1]:.3g}, max {n / secs[0]:.3g} triples/s), "
                      f"Hogwild over {cores} pinned threads, tables page-interleaved"}, n, med


def run_reference(args):
    rank, world, _ = dist_env()
    if rank != 0:
        return
    wl = args.workload if args.workload in WORKLOADS else "c2"
    vals, times, last = [], [], None
    for s in range(args.warmup + args.steps):
        cb, n, sec = cpu_bpr(wl, seconds_budget=1.0, samples=1)
        if s >= args.warmup:
            times.append(sec)
            vals.append(cb["value"])
        last = cb
    v = float(np.median(vals))
    last["value"] = v
    last["sample"] = f"median over {args.steps} steps; each step = " + last["sample"]
    line = {"impl": "reference", "metric": "BPR-MF triples/sec", "value": v, "unit": "triples/s", "n_gpus": args.gpus,
            "steps": args.steps, "warmup": args.warmup, "ms_per_step": 1e3 * float(np.median(times)), "higher_is_better": True,
            "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic", "config": bpr_config(wl, 1),
            "cpu_baseline": last,
            "e2e": {"value": v, "unit": "triples/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
            "gpu_launches": 0}
    print(json.dumps(line), flush=True)


# ---------------------------------------------------------------------------------------------------------------------
# BPR (c2 / c5 / c1)
# ---------------------------------------------------------------------------------------------------------------------
def run_bpr(args):
    rank, world, local = dist_env()
    assert world == args.gpus or world == 1, f"WORLD_SIZE {world} != --gpus {args.gpus}"
    dist = None
    if world > 1:
        import torch  # control plane only: rendezvous, id broadcast, max-over-ranks
        import torch.distributed as dist

        dist.init_process_group("gloo", rank=rank, world_size=world)
    import gorse_b200 as gb

    wl = args.workload
    upr, n_items_w, fpr, d, desc = WORKLOADS[wl]
    n_users, n_items, d, off, items = make_shard(wl, rank, world)
    _, (test_off, test_items) = get_data(wl, 1000 + rank)
    n_local = int(off[-1])
    if world > 1:
        import torch

        idbuf = torch.zeros(128, dtype=torch.uint8)
        if rank == 0:
            idbuf = torch.frombuffer(bytearray(gb.nccl_unique_id()), dtype=torch.uint8).clone()
        dist.broadcast(idbuf, 0)
        ctx = gb.Context(local, rank, world, bytes(idbuf.numpy().tobytes()))
    else:
        ctx = gb.Context(local)
    steps_per_epoch = n_local * world       # exact=True data: every rank holds the same count

    def max_over_ranks(x):
        if world == 1:
            return x
        import torch

        t = torch.tensor([x], dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    model = gb.CFModel(ctx, n_users, n_items, d, off, items)
    model.init_normal(0.0, INIT_STD, 0)
    ctx.sync()

    # ---- device-resident timing: K epochs, CUDA events on the library's own stream, max over ranks ----
    sampler = ClockSampler(local) if rank == 0 else None   # started before the warm-up so that it is already printing
    for w in range(args.warmup):
        model.bpr_epoch(LR, REG, steps_per_epoch, 100 + w)
    ctx.barrier()
    if dist:
        dist.barrier()
    l0 = ctx.launch_count()
    t0 = time.time()
    ctx.timer_begin()
    for s in range(args.steps):
        model.bpr_epoch(LR, REG, steps_per_epoch, 1000 + s)
    ctx.barrier() if world > 1 else None
    ms_total = ctx.timer_end()
    t1 = time.time()
    launches = ctx.launch_count() - l0
    clocks = sampler.stop(t0, t1) if sampler else None
    if rank == 0:
        P_, Q_ = model.get_factors()
        dump_outputs(args, "bpr", {"user_factors": P_, "item_factors": Q_})
        del P_, Q_
    ms_total = max_over_ranks(ms_total)
    ms_per_step = ms_total / args.steps
    value = steps_per_epoch / (ms_per_step * 1e-3)

    # ---- one epoch per event pair, for the roofline ----
    kms = []
    for s in range(min(args.steps, 5)):
        ctx.timer_begin()
        model.bpr_epoch(LR, REG, steps_per_epoch, 2000 + s)   # N > 1: includes the delta exchange
        kms.append(ctx.timer_end())
    k_ms = float(np.mean(kms))
    hbm, _, peak_src = read_peaks()
    achieved = bytes_per_triple(d) * n_local / (k_ms * 1e-3) / 1e9
    traffic = None   # measured DRAM bytes per epoch: not available without a profiler
    roofline = {"bound": "hbm", "achieved": achieved, "peak": hbm, "unit": "GB/s", "frac": achieved / hbm, "traffic": traffic,
                "kernel": f"one epoch on one rank = bpr_round_kernel<{d // 16 if d % 16 == 0 else 0}> (rounds of 8192 triples)" + (" + item-delta exchange" if world > 1 else ""),
                "kernel_ms": k_ms, "algorithmic_bytes_per_launch": bytes_per_triple(d) * n_local,
                "dram_frac": (traffic / (k_ms * 1e-3) / 1e9 / hbm) if traffic else None, "peak_source": peak_src}
    model.close()

    # ---- end to end through the plugin call with HOST buffers: what cf.BPR.Fit does per call ----
    e2e, e2e_error = None, None
    if not args.no_e2e:
        hp = hq = m2 = None
        try:
            hp = gb.PinnedArray((upr, d))            # the shim's flat pinned mirror: this rank's user rows + the item table
            hq = gb.PinnedArray((n_items, d))
            p_base = C.c_void_p(hp.array.ctypes.data - rank * upr * d * 4)   # the ABI takes the base of the FULL user table
            e_epochs = max(1, args.e2e_epochs)
            # three complete, independent calls; the MEDIAN wall time is reported (one call is ~0.4 s of device work plus
            # host work -- CSR validation/sort on 16 threads, plan set-up -- that moved 0.62 -> 1.31 s between boxes and runs)
            walls = []
            for _rep in range(3):
                if dist:
                    dist.barrier()
                w0 = time.time()
                m2 = gb.CFModel(ctx, n_users, n_items, d, off, items)
                r_ = m2.fit("bpr", test_off, test_items, None, None, n_epochs=e_epochs, verbose=10, seed=0)
                gb.check(gb.lib.gorse_b200_cf_get_factors(m2.h, p_base, gb.ptr(hq.array)))
                w1 = time.time()
                m2.close()
                m2 = None
                walls.append((max_over_ranks(w1 - w0), float(r_.ndcg), int(r_.epochs_run)))
            e_sec, e_ndcg, e_run = sorted(walls)[1]
            finite = bool(np.isfinite(hq.array).all() and np.isfinite(hp.array).all())
            if max_over_ranks(0.0 if finite else 1.0) > 0.5:
                raise FloatingPointError("non-finite factors after the end-to-end leg")
            h2d = off.nbytes + items.nbytes + test_off.nbytes + test_items.nbytes
            n_eval = 1 + e_epochs // 10 + (1 if e_epochs % 10 else 0)
            d2h = upr * d * 4 + n_items * d * 4 + n_eval * upr * 16
            e2e = {"value": e_epochs * steps_per_epoch / e_sec, "unit": "triples/s",
                   "h2d_bytes_per_step": h2d / e_epochs, "d2h_bytes_per_step": d2h / e_epochs,
                   "what": f"per rank: cf_create (own CSR rows, host -> device) + gorse_b200_bpr_fit (Init, {e_epochs} epochs = reference default NEpochs, "
                           f"Evaluate at epoch 0 and every 10 epochs over all test users x 101 candidates with negatives sampled on the device, {n_eval} evaluations) "
                           f"+ get_factors into the pinned mirror; bytes are per rank and per epoch, amortised over the call",
                   "wall_s": e_sec, "wall_s_all": [w for w, _, _ in walls], "ndcg_at_10": e_ndcg, "epochs_run": e_run}
        except Exception as ex:  # keep the contract line even if the end-to-end leg fails
            e2e_error = f"{type(ex).__name__}: {ex}"
        finally:
            if m2 is not None:
                m2.close()
            for b in (hp, hq):
                if b is not None:
                    b.free()

    line = None
    if rank == 0:
        cb = None
        if world == 1 and not args.no_cpu:
            cb, _, _ = cpu_bpr(wl)
        cfg = bpr_config(wl, world)
        line = {"metric": "BPR-MF triples/sec", "value": value, "unit": "triples/s", "n_gpus": world, "steps": args.steps,
                "warmup": args.warmup, "ms_per_step": ms_per_step, "higher_is_better": True, "scaling": "weak",
                "vs_baseline": None, "dtype": "f32", "data": "synthetic", "config": cfg,
                "parallelism": (f"{world} ranks: users row-sharded (each rank passes only its rows), item table replicated, per-epoch NCCL exchange of item deltas"
                                if world > 1 else "1 GPU"),
                "feedback_per_epoch": steps_per_epoch,
                "roofline": roofline, "cpu_baseline": cb, "e2e": e2e, "gpu_launches": int(launches), "clocks": clocks}
        if e2e_error:
            line["e2e_error"] = e2e_error
    ctx.close()
    if dist:
        dist.barrier()
        dist.destroy_process_group()
    return line


# ---------------------------------------------------------------------------------------------------------------------
# eALS (c3)
# ---------------------------------------------------------------------------------------------------------------------
def run_als(args):
    """BASELINE configs[2]: eALS ("CCD") on the C2 data at d = 128; one step = one epoch (both half-sweeps + 2 Grams)."""
    import gorse_b200 as gb
    from gorse_b200 import synth

    small = args.small
    U, I, R, d = (1_000_000, 100_000, 10_000_000, 128) if not small else (50_000, 10_000, 500_000, 128)
    if small:
        off0, items0 = synth.make_feedback(U, I, R + U, seed=1000, zipf_s=ZIPF_S, exact=True)
        (off, items), (test_off, test_items) = synth.leave_one_out(off0, items0, seed=1001)
    else:
        (off, items), (test_off, test_items) = get_data("c2", 1000)
    ioff, iusers = gb.transpose_csr(off, items, I)
    steps, warm = args.steps, args.warmup
    with gb.Context(0) as ctx:
        with gb.CFModel(ctx, U, I, d, off, items, ioff, iusers) as m:
            m.init_normal(0.0, ALS_STD, 0)
            sampler = ClockSampler(0)
            for _ in range(warm):
                m.als_epoch(ALS_REG, ALS_ALPHA)
            l0, t0 = ctx.launch_count(), time.time()
            ctx.timer_begin()
            for _ in range(steps):
                m.als_epoch(ALS_REG, ALS_ALPHA)
            ms = ctx.timer_end() / steps
            t1 = time.time()
            launches = ctx.launch_count() - l0
            clocks = sampler.stop(t0, t1)
            P_, Q_ = m.get_factors()
            dump_outputs(args, "als", {"user_factors": P_, "item_factors": Q_})
            del P_, Q_
        e2e = None
        if not args.no_e2e:
            hp, hq = gb.PinnedArray((U, d)), gb.PinnedArray((I, d))
            e_epochs = 50 if not small else 5      # ALS default NEpochs, model.go:581
            w0 = time.time()
            with gb.CFModel(ctx, U, I, d, off, items, ioff, iusers) as m2:
                res = m2.fit("als", test_off, test_items, None, None, n_epochs=e_epochs, verbose=10, seed=0)
                gb.check(gb.lib.gorse_b200_cf_get_factors(m2.h, gb.ptr(hp.array), gb.ptr(hq.array)))
            w1 = time.time()
            n_eval = 1 + e_epochs // 10 + (1 if e_epochs % 10 else 0)
            e2e = {"value": e_epochs * 2 * int(off[-1]) / (w1 - w0), "unit": "feedback visits/s",
                   "h2d_bytes_per_step": (off.nbytes + items.nbytes + ioff.nbytes + iusers.nbytes + test_off.nbytes + test_items.nbytes) / e_epochs,
                   "d2h_bytes_per_step": ((U + I) * d * 4 + n_eval * U * 16) / e_epochs, "wall_s": w1 - w0, "ndcg_at_10": float(res.ndcg),
                   "what": f"cf_create (both CSRs from host) + gorse_b200_als_fit ({e_epochs} epochs = reference default, Evaluate every 10) + get_factors"}
            hp.free()
            hq.free()
    hbm, _, src = read_peaks()
    R_ = int(off[-1])
    nbytes = 2 * R_ * (4 * d + 4) + 3 * (U + I) * 4 * d
    cb = None
    if not args.no_cpu:
        import oracle

        cores = len(os.sched_getaffinity(0))
        Us, Is, Rs = 50_000, 10_000, 500_000
        o2, i2 = synth.make_feedback(Us, Is, Rs, seed=1000, zipf_s=ZIPF_S, exact=True)
        io2, iu2 = gb.transpose_csr(o2, i2, Is)
        rng = np.random.default_rng(0)
        P = (rng.standard_normal((Us, d)) * 0.1).astype(np.float32)
        Q = (rng.standard_normal((Is, d)) * 0.1).astype(np.float32)
        sec = oracle.als_epoch_threads(P, Q, o2, i2, io2, iu2, ALS_REG, ALS_ALPHA, cores)
        cb = {"value": 2 * Rs / sec, "unit": "feedback visits/s", "cores": cores, "kind": "port",
              "sample": f"one epoch at {Us} x {Is} x {Rs}, d={d}: rows over {cores} threads, serial Gram as in the reference, {sec:.2f} s"}
    return {"metric": "eALS (CCD) feedback visits/sec", "value": 2 * R_ / (ms * 1e-3), "unit": "feedback visits/s", "n_gpus": 1,
            "steps": steps, "warmup": warm, "ms_per_step": ms, "higher_is_better": True, "scaling": "weak",
            "vs_baseline": None, "dtype": "f32", "data": "synthetic",
            "config": {"workload": f"eALS {U} users x {I} items x {R_} feedback, d={d} (BASELINE configs[2])", "reg": ALS_REG, "alpha": ALS_ALPHA,
                       "item_popularity": f"zipf({ZIPF_S})"},
            "roofline": {"bound": "hbm", "achieved": nbytes / (ms * 1e-3) / 1e9, "peak": hbm, "unit": "GB/s",
                         "frac": nbytes / (ms * 1e-3) / 1e9 / hbm, "traffic": None, "algorithmic_bytes_per_epoch": nbytes,
                         "kernel": "one epoch = 2 Grams + user sweep + item sweep", "peak_source": src},
            "cpu_baseline": cb, "e2e": e2e, "gpu_launches": int(launches), "clocks": clocks}


# ---------------------------------------------------------------------------------------------------------------------
# all-pairs top-k (c4)
# ---------------------------------------------------------------------------------------------------------------------
def run_topk(args):
    """BASELINE configs[3]: all-pairs top-100 over 1M x 128 unit vectors (cosine via -dot); value = query vectors/s."""
    import gorse_b200 as gb

    N, d, k = (1_000_000, 128, 100) if not args.small else (100_000, 128, 100)
    nq = min(N, args.queries)
    # N > 1: the vectors are replicated, rank r answers its own nq query rows, no collective (SURVEY 8e; weak scaling)
    rank, world, local = dist_env()
    assert world == args.gpus or world == 1, f"WORLD_SIZE {world} != --gpus {args.gpus}"
    dist = None
    if world > 1:
        import torch
        import torch.distributed as dist

        dist.init_process_group("gloo", rank=rank, world_size=world)
    q_lo = (rank * nq) % max(1, N - nq + 1)
    rng = np.random.default_rng(0)
    X = rng.standard_normal((N, d), dtype=np.float32)
    X /= np.linalg.norm(X, axis=1, keepdims=True)
    steps = args.steps
    with gb.Context(local) as ctx:
        with gb.BruteforceIndex(ctx, d, gb.METRIC_NEG_DOT) as ix:
            ix.add(X)
            ix.search_range(0, 512, k)  # builds the bf16 mirror
            # results land in page-locked host buffers, like the shim's pinned mirror (gorse_b200_host_alloc)
            pin = (gb.PinnedArray((nq, k), np.int32), gb.PinnedArray((nq, k), np.float32), gb.PinnedArray((nq,), np.int32))
            out = (pin[0].array, pin[1].array, pin[2].array)
            for _ in range(max(1, args.warmup - 1)):
                ix.search_range(q_lo, q_lo + nq, k, out=out)
            if dist:
                dist.barrier()
            sampler = ClockSampler(local) if rank == 0 else None
            ix.stage1_stats()
            l0, t0 = ctx.launch_count(), time.time()
            ms_list = []
            for s in range(steps):
                ctx.timer_begin()
                idx, dist_, cnt = ix.search_range(q_lo, q_lo + nq, k, out=out)   # host buffers out
                ms_list.append(ctx.timer_end())
            t1 = time.time()
            launches = ctx.launch_count() - l0
            s1_ms, s1_flop, fb = ix.stage1_stats()
            clocks = sampler.stop(t0, t1) if sampler else None
            assert cnt.min() == k
            if rank == 0:
                dump_outputs(args, "topk", {"indices": idx, "distances": dist_})
        # end to end from host buffers: build the index (vectors H2D + mirror) and answer nq queries into host memory
        e2e = None
        if not args.no_e2e:
            w0 = time.time()
            with gb.BruteforceIndex(ctx, d, gb.METRIC_NEG_DOT) as ix2:
                ix2.add(X)
                ix2.search_range(q_lo, q_lo + nq, k, out=out)
            w1 = time.time()
            e2e = {"value": nq * world / (w1 - w0), "unit": "vectors/s", "h2d_bytes_per_step": X.nbytes, "d2h_bytes_per_step": nq * k * 8 + nq * 4,
                   "wall_s": w1 - w0, "what": "index_create + index_add (1M vectors host -> device, bf16 mirror) + one search_range call into host buffers"}
        for p_ in pin:
            p_.free()
    ms = float(np.mean(ms_list))
    if dist:
        import torch

        t = torch.tensor([ms], dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)   # device-timed, max over ranks
        ms = float(t.item())
        dist.barrier()
        dist.destroy_process_group()
        if rank != 0:
            return None
    nq_all = nq * world
    flop = 2.0 * nq_all * N * d
    _, peak, src = read_peaks()
    cb = None
    if not args.no_cpu and world == 1:
        import oracle

        cores = len(os.sched_getaffinity(0))
        sample = 4 * cores
        _, _, _, sec = oracle.bruteforce_all(X, 0, sample, k, metric=oracle.METRIC_NEG_DOT, n_threads=cores)
        cb = {"value": sample / sec, "unit": "vectors/s", "cores": cores, "kind": "port",
              "sample": f"{sample} queries of the same set: reference-order dot + Go heap per query, {cores} threads, {sec:.2f} s"}
    return {"metric": "item-to-item top-k vectors/sec", "value": nq_all / (ms * 1e-3), "unit": "vectors/s", "n_gpus": world, "steps": steps,
            "warmup": args.warmup, "ms_per_step": ms, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
            "dtype": "bf16 tensor-core candidate generation + f32 exact re-rank", "data": "synthetic",
            "config": {"workload": f"all-pairs top-{k} over {N} x {d} unit vectors, {nq} query rows per step and rank (BASELINE configs[3])"
                                   + (f" x {world} ranks, vectors replicated, queries sharded, no collective" if world > 1 else ""),
                       "metric": "-dot (cosine on unit vectors)", "fallback_rows": int(fb)},
            "roofline": {"bound": "tensor", "achieved": s1_flop / (s1_ms * 1e-3) / 1e12, "peak": peak, "unit": "TFLOP/s",
                         "frac": s1_flop / (s1_ms * 1e-3) / 1e12 / peak, "traffic": None, "kernel": "mma::topk_mma_kernel (wgmma sweep)",
                         "kernel_ms": s1_ms / steps, "algorithmic_flop_per_launch": s1_flop / steps,
                         "whole_call_tflops": flop / (ms * 1e-3) / 1e12, "peak_source": src + " sustained bf16"},
            "cpu_baseline": cb, "e2e": e2e, "gpu_launches": int(launches), "clocks": clocks}


def build_parser():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--workload", default="c2", choices=sorted(WORKLOADS) + ["c3", "c4"])
    ap.add_argument("--small", action="store_true", help="c3/c4 at reduced size (not a bench number)")
    ap.add_argument("--queries", type=int, default=151552, help="c4: query rows per step (on 132 SMs one 135168-row chunk plus a 16384-row tail, DESIGN 5.3)")
    ap.add_argument("--e2e-epochs", type=int, default=100, help="BPR default NEpochs, model/cf/model.go:390")
    ap.add_argument("--zipf", type=float, default=None, help="item popularity exponent of the synthetic data (default 1.0; 0 = uniform)")
    ap.add_argument("--no-e2e", action="store_true")
    ap.add_argument("--no-cpu", action="store_true")
    ap.add_argument("--no-also", action="store_true", help="default run: skip the c3 / c4 sub-records")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write the last timed step's outputs as DIR/<name>.npy (seeded row samples of large tables)")
    return ap


def compact(rec):
    keep = ("metric", "value", "unit", "ms_per_step", "steps", "dtype", "config", "roofline", "cpu_baseline", "e2e", "gpu_launches", "clocks")
    return {k: rec[k] for k in keep if k in rec}


def main():
    args = build_parser().parse_args()
    if args.zipf is not None:
        global ZIPF_S
        ZIPF_S = args.zipf
    if args.impl == "reference":
        run_reference(args)
        return
    args.warmup = max(args.warmup, 3)
    rank, world, _ = dist_env()
    if args.workload == "c3":
        line = run_als(args)
    elif args.workload == "c4":
        line = run_topk(args)
    else:
        line = run_bpr(args)
        if line is not None and world == 1 and args.workload == "c2" and not args.no_also:
            also = []
            for fn in (run_als, run_topk):
                try:
                    also.append(compact(fn(args)))
                except Exception as ex:
                    also.append({"metric": fn.__name__, "error": f"{type(ex).__name__}: {ex}"})
            line["also"] = also
    if line is not None and rank == 0:
        print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
