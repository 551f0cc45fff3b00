#!/usr/bin/env python
"""tools/vecdb_bf16_bench.py -- dense vector collections in bf16 storage against their fp32 twins, host in to host out.

  python tools/vecdb_bf16_bench.py [--small] [--reps 3] [--shapes d1024,d3072,d128]

Shapes (seeded normal rows truncated to bf16, Euclidean):
  d1024  200,000 x 1024   the exact scan (d > 192 takes no tensor-core sweep)
  d3072  200,000 x 3072   the exact scan
  d128   1,000,000 x 128  the tensor-core sweep
Each shape builds a bf16 collection and its fp32 twin from the same rows.  The twin is made fp32 first by one vector that is
not bf16-exact (added first, with an older timestamp; the bf16 collection gets a bf16-exact one), so its rows go in through
the fp32 add path; both first vectors are then deleted and compacted away, so both collections hold the same vectors in the
same slots at a capacity of exactly their count.
Reported per shape, bf16 and twin:
  device_bytes  gorse_b200_vecdb_storage after the build and a compaction (which releases the bf16 upload staging)
  add_s         the add of all rows in batches of 50,000, host in (the call returns after the device has the rows), summed
                over the batches; each rep builds both collections again
  load_s        gorse_b200_vecdb_load of the collection's stream from host memory, ended by a context synchronise.  Both
                streams are bf16-exact, so the twin's load reads its stream with the first value made inexact: the load
                promotes at its first chunk and takes the fp32 path from there, as a load of fp32 data does
  query_s       1,024 query rows, top 20, host in to host out
  i2i_s         item-to-item for 1,024 users with 5 context slots each, top 20, host in to host out
Times are medians of --reps with their spread (max - min); the bf16 collection and the twin alternate within each rep.  The
outputs of both (query and item-to-item answers, the saved streams) are hashed with SHA-256 and must match.  The card's
name, power limit and SM clock are read in the same run.  One JSON line.
"""
import argparse
import hashlib
import io
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from item_to_item_bench import card  # noqa: E402

SHAPES = {"d1024": (200_000, 1024), "d3072": (200_000, 3072), "d128": (1_000_000, 128)}
BATCH = 50_000


def log(msg):
    print(f"[vecdb_bf16_bench] {msg}", file=sys.stderr, flush=True)


def exact(x):
    return (x.view(np.uint32) & np.uint32(0xFFFF0000)).view(np.float32)


def rows(seed, n, dim):
    return exact(np.random.default_rng(seed).standard_normal((n, dim), dtype=np.float32))


def timed(f):
    t0 = time.perf_counter()
    r = f()
    return time.perf_counter() - t0, r


def stat(v):
    return {"median": float(np.median(v)), "spread": float(np.max(v) - np.min(v)), "reps": [float(x) for x in v]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--small", action="store_true", help="tiny shapes (a rehearsal, not a measurement)")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--shapes", default="d1024,d3072,d128")
    args = ap.parse_args()

    import gorse_b200 as gb

    out = {"card": card(), "small": args.small, "shapes": {}}
    with gb.Context(0) as ctx:
        for shape in args.shapes.split(","):
            n, dim = SHAPES[shape]
            if args.small:
                n //= 100
            X = rows(1, n, dim)
            rng = np.random.default_rng(2)
            q = exact(rng.standard_normal((1024, dim), dtype=np.float32))
            ctx_lists = [rng.integers(0, n, 5) for _ in range(1024)]
            ex_lists = [np.zeros(0, np.int64)] * 1024
            add = {"bf16": [], "twin": []}
            cols = None
            for r in range(args.reps):   # each rep builds both collections afresh; the last build is measured further
                if cols:
                    for c in cols.values():
                        c.close()
                cols = {"bf16": gb.VectorCollection(ctx, dim, gb.DISTANCE_EUCLIDEAN), "twin": gb.VectorCollection(ctx, dim, gb.DISTANCE_EUCLIDEAN)}
                # a first vector, deleted and compacted away after the adds: bf16-exact in the bf16 collection, not in the
                # twin, so both end with the same slots and a capacity of n
                cols["bf16"].add(np.ones((1, dim), np.float32), timestamps=[1])
                cols["twin"].add(np.full((1, dim), 1.0 + 2.0 ** -20, np.float32), timestamps=[1])
                t = {k: 0.0 for k in cols}
                for a in range(0, n, BATCH):   # the two alternate batch by batch, each going first every other batch
                    part = X[a:a + BATCH]
                    for k in (("bf16", "twin") if (a // BATCH + r) % 2 == 0 else ("twin", "bf16")):
                        t[k] += timed(lambda: cols[k].add(part, timestamps=np.full(len(part), 1000)))[0]
                for k in cols:
                    add[k].append(t[k])
                log(f"{shape} rep {r}: add bf16 {t['bf16']:.3f} s, twin {t['twin']:.3f} s")
            for c in cols.values():
                c.delete_before(2)
                c.compact()
            rec = {k: {"add_s": stat(add[k])} for k in cols}
            streams = {}
            for k, c in cols.items():
                rec[k]["value_bytes"], rec[k]["device_bytes"] = c.storage()
                buf = io.BytesIO()
                c.save(buf)
                streams[k] = buf.getvalue()
                rec[k]["stream_sha256"] = hashlib.sha256(streams[k]).hexdigest()
            values = len(streams["twin"]) - 4 * n * dim
            loads = {"bf16": streams["bf16"], "twin": bytearray(streams["twin"])}
            loads["twin"][values:values + 4] = np.array([1.0 + 2.0 ** -20], np.float32).tobytes()
            loads["twin"] = bytes(loads["twin"])
            log(f"{shape}: {n} x {dim}, bf16 {rec['bf16']['device_bytes'] / 1e9:.3f} GB, twin {rec['twin']['device_bytes'] / 1e9:.3f} GB")
            # warm-up: every shape the timed calls use
            for c in cols.values():
                c.query(q, (), 20)
                c.item_to_item(ctx_lists, ex_lists, 20)
            times = {k: {"query_s": [], "i2i_s": [], "load_s": []} for k in cols}
            hashes = {}
            for r in range(args.reps):
                for k, c in cols.items():
                    t, res = timed(lambda: c.query(q, (), 20))
                    times[k]["query_s"].append(t)
                    h = hashlib.sha256(b"".join(np.ascontiguousarray(x).tobytes() for x in res))
                    t, (i2i, _) = timed(lambda: c.item_to_item(ctx_lists, ex_lists, 20))
                    times[k]["i2i_s"].append(t)
                    for s, v in i2i:
                        h.update(s.tobytes())
                        h.update(v.tobytes())
                    hashes.setdefault(k, h.hexdigest())
                    assert hashes[k] == h.hexdigest(), f"{shape} {k}: answers changed between reps"

                    def load():
                        got = gb.VectorCollection.load(ctx, io.BytesIO(loads[k]))
                        ctx.sync()
                        return got

                    t, got = timed(load)
                    times[k]["load_s"].append(t)
                    assert got.storage()[0] == rec[k]["value_bytes"]
                    got.close()
                log(f"{shape} rep {r}: " + ", ".join(f"{k} query {times[k]['query_s'][-1]:.4f} s i2i {times[k]['i2i_s'][-1]:.4f} s "
                                                    f"load {times[k]['load_s'][-1]:.3f} s" for k in cols))
            for k in cols:
                rec[k].update({name: stat(v) for name, v in times[k].items()})
                rec[k]["answers_sha256"] = hashes[k]
            same = hashes["bf16"] == hashes["twin"] and streams["bf16"] == streams["twin"]
            out["shapes"][shape] = {"vectors": n, "dim": dim, "outputs_identical": same, **rec}
            for c in cols.values():
                c.close()
            assert same, f"{shape}: the bf16 collection and its twin answer differently"
    out["card_after"] = card()
    print(json.dumps({"metric": "dense vector collections: bf16 storage against the fp32 twin, host in to host out", **out}))


if __name__ == "__main__":
    main()
