#!/usr/bin/env python
"""tools/vecdb_snapshot_bench.py -- saving a vector collection to a stream and loading it back (gorse_b200_vecdb_save /
gorse_b200_vecdb_load), host in to host out.

  python tools/vecdb_snapshot_bench.py [--small] [--reps 3] [--shapes dense,c5]

Shapes:
  dense  a Euclidean collection of 1,000,000 x 1024 fp32 (4 GB; the "embedding" item-to-item type at the default
         openai.embedding_dimensions), seeded normal rows added in batches of 50,000
  c5     the sparse C5 collection of tools/vecdb_build_bench.py: 1,000,000 rows built from 200M ids with
         gorse_b200_vecdb_add_idf_vectors
Sinks, each timed for save and for load:
  memory  a preallocated host buffer of the stream's size: the callbacks copy into and out of it, so the rate is the
          library's (the device copies over PCIe, the gather, the validation) plus one host memcpy
  file    a file in the system's temporary directory, written unbuffered and fsync'd before the clock stops; loaded back
          through readinto (the page cache may still hold it, so this is the write path to disk and the read path from cache)
Every timed call ends with the device synchronised (save synchronises before it returns; after a load the context is
synchronised).  Medians of --reps.  Each load is checked against the saved collection (counts and a sample of rows, bit for
bit).  The card's pinned copy rates (256 MB, host to device and device to host, CUDA events) are measured in the same run.
One JSON line with the card's name and power limit.
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from item_to_item_bench import card  # noqa: E402


def log(msg):
    print(f"[vecdb_snapshot_bench] {msg}", file=sys.stderr, flush=True)


class MemorySink:
    """a preallocated host buffer, written and read like a binary file"""

    def __init__(self, size):
        self.buf, self.pos = np.empty(size, np.uint8), 0

    def write(self, b):
        n = len(b)
        self.buf[self.pos:self.pos + n] = np.frombuffer(b, np.uint8)
        self.pos += n
        return n

    def readinto(self, b):
        n = min(len(b), self.buf.size - self.pos)
        np.frombuffer(b, np.uint8, n)[:] = self.buf[self.pos:self.pos + n]
        self.pos += n
        return n


def copy_rates():
    """pinned host <-> device copy rates of 256 MB, GB/s"""
    import torch

    h = torch.empty(256 << 20, dtype=torch.uint8).pin_memory()
    d = torch.empty(256 << 20, dtype=torch.uint8, device="cuda:0")
    out = {}
    for name, dst, src in (("h2d_gbps", d, h), ("d2h_gbps", h, d)):
        dst.copy_(src, non_blocking=True)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(5):
            dst.copy_(src, non_blocking=True)
        e1.record()
        torch.cuda.synchronize()
        out[name] = 5 * (256 << 20) / (e0.elapsed_time(e1) * 1e-3) / 1e9
    return out


def build(gb, ctx, shape, small):
    if shape == "dense":
        n, dim, batch = (20_000, 1024, 5_000) if small else (1_000_000, 1024, 50_000)
        col = gb.VectorCollection(ctx, dim, gb.DISTANCE_EUCLIDEAN)
        rng = np.random.default_rng(1)
        for a in range(0, n, batch):
            col.add(rng.standard_normal((min(batch, n - a), dim), dtype=np.float32), timestamps=np.full(min(batch, n - a), 1000))
        return col
    from vecdb_build_bench import workload

    off, ids, idf = workload("c5", small)
    col = gb.VectorCollection(ctx, 0, gb.DISTANCE_DOT)
    n, batch = off.size - 1, 10_000
    for a in range(0, n, batch):   # the batches of vecdb_build_bench's device arm
        b = min(a + batch, n)
        o, slots = np.ascontiguousarray(off[a:b + 1] - off[a]), np.zeros(b - a, np.int64)
        gb.check(gb.lib.gorse_b200_vecdb_add_idf_vectors(col.h, b - a, gb.ptr(o), gb.ptr(ids[off[a]:off[b]]), gb.ptr(idf), idf.size, 0, None, None,
                                                         None, 0, 0, None, 1000, None, None, None, gb.ptr(slots)))
    return col


def sample(col, slots):
    vals, hid, ts, live = col.get(slots)
    sp = [col.get_sparse(int(s)) for s in slots] if col.dim == 0 else []
    return vals.tobytes(), hid.tobytes(), ts.tobytes(), live.tobytes(), [(i.tobytes(), v.tobytes()) for i, v in sp]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--small", action="store_true", help="small shapes (a rehearsal, not a measurement)")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--shapes", default="dense,c5")
    args = ap.parse_args()

    import gorse_b200 as gb

    out = {"card": card(), "copy": copy_rates(), "small": args.small, "shapes": {}}
    with gb.Context(0) as ctx, tempfile.TemporaryDirectory() as tmp:
        for shape in args.shapes.split(","):
            col = build(gb, ctx, shape, args.small)
            live = col.count()[0]
            check = np.sort(np.random.default_rng(2).choice(live, min(live, 200), replace=False)).astype(np.int64)
            want = sample(col, check)
            size = [0]

            class Counter:
                def write(self, b):
                    size[0] += len(b)
                    return len(b)

            col.save(Counter())
            nbytes = size[0]
            log(f"{shape}: {live} vectors, stream {nbytes / 1e9:.3f} GB")
            rec = {}
            for sink in ("memory", "file"):
                times = {"save_s": [], "load_s": []}
                for r in range(args.reps):
                    path = os.path.join(tmp, f"{shape}.b200vec")
                    if sink == "memory":
                        dst = MemorySink(nbytes)
                        t0 = time.perf_counter()
                        col.save(dst)
                        times["save_s"].append(time.perf_counter() - t0)
                        dst.pos = 0
                        t0 = time.perf_counter()
                        got = gb.VectorCollection.load(ctx, dst)
                        ctx.sync()
                        times["load_s"].append(time.perf_counter() - t0)
                    else:
                        t0 = time.perf_counter()
                        with open(path, "wb", buffering=0) as f:
                            col.save(f)
                            os.fsync(f.fileno())
                        times["save_s"].append(time.perf_counter() - t0)
                        t0 = time.perf_counter()
                        with open(path, "rb", buffering=0) as f:
                            got = gb.VectorCollection.load(ctx, f)
                        ctx.sync()
                        times["load_s"].append(time.perf_counter() - t0)
                        os.remove(path)
                    assert got.count() == (live, live) and sample(got, check) == want, f"{shape} {sink}: the loaded collection differs"
                    got.close()
                    log(f"{shape} {sink} rep {r}: save {times['save_s'][-1]:.3f} s, load {times['load_s'][-1]:.3f} s")
                med = {k: float(np.median(v)) for k, v in times.items()}
                med["save_gbps"], med["load_gbps"] = nbytes / med["save_s"] / 1e9, nbytes / med["load_s"] / 1e9
                rec[sink] = {"median": med, "reps": times}
            out["shapes"][shape] = {"vectors": live, "stream_bytes": nbytes, **rec}
            col.close()
    print(json.dumps({"metric": "vector collection snapshot: save and load, host in to host out", **out}))


if __name__ == "__main__":
    main()
