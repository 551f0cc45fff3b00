"""Times the dense top-k entry points at the shapes a shim or worker calls them with, and hashes their answers.

  python tools/topk_probe.py [--reps R]

Prints one JSON line: the card (name, power limit, SM clock), then per shape the median and minimum wall time of one call
(host clock around a call that returns host results), and a hash of the answers (ids, distance or score bits, counts; the
collection query's entries past count[q] are not part of its answer and are left out).  The package is imported from
PYTHONPATH when it is set there, else from this checkout, so two builds can be compared on the same card.  "c4" also reports
the device memory the index holds after the call (bench.py's all-pairs workload)."""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.append(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import gorse_b200 as gb  # noqa: E402


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True).stdout
    return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))


def digest(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()[:16]


def timed(fn, reps):
    fn()   # warm-up: buffers, modules, the bf16 mirror
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        out = fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return {"ms_median": float(np.median(ts)), "ms_min": float(np.min(ts))}, out


def unit_rows(rng, n, d):
    X = rng.standard_normal((n, d), dtype=np.float32)
    return X / np.linalg.norm(X, axis=1, keepdims=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    import torch   # device memory before / after (the library shares the primary context)

    rng = np.random.default_rng(0)
    res = {"card": card(), "package": os.path.dirname(gb.__file__)}
    with gb.Context(0) as ctx:
        X = unit_rows(rng, 1_000_000, 128)
        Q = unit_rows(rng, 1, 128)
        free0 = torch.cuda.mem_get_info()[0]
        with gb.BruteforceIndex(ctx, 128, gb.METRIC_NEG_DOT) as ix:
            ix.add(X)
            shapes = {
                "index_vectors_nq1_N1M_k100": lambda: ix.search_vectors(Q, 100),
                "index_indices_nq1_N1M_k100": lambda: ix.search_indices(np.array([12345], np.int64), 100),
                "index_range_nq32_N1M_k100": lambda: ix.search_range(5000, 5032, 100),
                "index_range_nq4096_N1M_k300": lambda: ix.search_range(0, 4096, 300),
                "c4_index_range_nq151552_N1M_k100": lambda: ix.search_range(0, 151552, 100),
            }
            for name, fn in shapes.items():
                t, out = timed(fn, args.reps if "c4" not in name else 3)
                res[name] = dict(t, hash=digest(*out))
            res["c4_index_range_nq151552_N1M_k100"]["device_mb_held"] = (free0 - torch.cuda.mem_get_info()[0]) / 2**20
        X = unit_rows(rng, 20000, 64)
        with gb.BruteforceIndex(ctx, 64, gb.METRIC_NEG_DOT) as ix:
            ix.add(X)
            t, out = timed(lambda: ix.search_range(0, 4096, 10), args.reps)
            res["index_range_nq4096_N20000_d64_k10"] = dict(t, hash=digest(*out))
        X = unit_rows(rng, 100_000, 64)
        with gb.VectorCollection(ctx, 64, gb.DISTANCE_DOT) as col:
            col.add(X)
            for nq in (1, 256):
                Qv = unit_rows(rng, nq, 64)
                t, (s, v, c) = timed(lambda: col.query(Qv, [], 100), args.reps)
                live = np.arange(100)[None, :] < c[:, None]
                res[f"vecdb_query_nq{nq}_N100K_d64_k100"] = dict(t, hash=digest(s[live], v[live], c))
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
