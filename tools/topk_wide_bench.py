#!/usr/bin/env python
"""tools/topk_wide_bench.py -- dense collections at embedding widths: the wide tensor-core sweep against the exact kernel alone
(GORSE_B200_TOPK_EXACT=1), host in to host out.

  python tools/topk_wide_bench.py [--small] [--reps 3] [--shapes 200k_1024,200k_3072,1m_1024] [--types bf16,fp32]

Shapes (Dot, seeded normal rows; bf16: truncated to bf16-exact values, so the collection stores two bytes a value):
  200k_1024  200,000 x 1024
  200k_3072  200,000 x 3072
  1m_1024    1,000,000 x 1024
Timed per shape and type, the two arms alternating within each rep (each goes first every other rep):
  query_1024_s / query_8192_s   query with 1,024 / 8,192 rows, top 20
  i2i_s                         item-to-item for 1,024 users with 5 context slots each, top 20
Reported besides: medians of --reps with their spread (max - min); the rows the exact kernel answered per call on the sweep
arm (query_excluding of the 8,192 rows with empty exclusions: the same pipeline as query, which reports them; item-to-item's
stats); the stage-1 rate (a BruteforceIndex over the same rows, search_vectors of the 8,192 rows: device time of the sweep
kernels and 2 nq N d flop from gorse_b200_index_stats); SHA-256 of each arm's answers, which must be equal; the card's name,
power limit and SM clock before and after.
--text: the fallback rate on unit-normalised, clustered vectors standing in for text embeddings (200,000 x 1024, bf16, 1,024
query rows near stored rows, top 20 and top 100).  One JSON line.
"""
import argparse
import hashlib
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from item_to_item_bench import card  # noqa: E402

SHAPES = {"200k_1024": (200_000, 1024), "200k_3072": (200_000, 3072), "1m_1024": (1_000_000, 1024)}
BATCH = 50_000
ARMS = ("sweep", "exact")


def log(msg):
    print(f"[topk_wide_bench] {msg}", file=sys.stderr, flush=True)


def truncate(x):
    return (x.view(np.uint32) & np.uint32(0xFFFF0000)).view(np.float32)


def timed(f):
    t0 = time.perf_counter()
    r = f()
    return time.perf_counter() - t0, r


def stat(v):
    return {"median": float(np.median(v)), "spread": float(np.max(v) - np.min(v)), "reps": [float(x) for x in v]}


def arm(name):
    if name == "exact":
        os.environ["GORSE_B200_TOPK_EXACT"] = "1"
    else:
        os.environ.pop("GORSE_B200_TOPK_EXACT", None)


def rows(seed, n, dim, bf16):
    X = np.empty((n, dim), np.float32)
    rng = np.random.default_rng(seed)
    for a in range(0, n, BATCH):
        X[a:a + BATCH] = rng.standard_normal((min(BATCH, n - a), dim), dtype=np.float32)
    return truncate(X) if bf16 else X


def text_like(seed, n, dim):
    """unit rows around 2,000 unit centres (angle ~ 40 degrees to their centre): close top scores, as sentence embeddings"""
    rng = np.random.default_rng(seed)
    C = rng.standard_normal((2000, dim), dtype=np.float32)
    C /= np.linalg.norm(C, axis=1, keepdims=True)
    X = np.empty((n, dim), np.float32)
    for a in range(0, n, BATCH):
        m = min(BATCH, n - a)
        v = C[rng.integers(0, 2000, m)] + np.float32(0.8 / np.sqrt(dim)) * rng.standard_normal((m, dim), dtype=np.float32)
        X[a:a + m] = v / np.linalg.norm(v, axis=1, keepdims=True)
    return truncate(X)


def build(gb, ctx, X, distance):
    col = gb.VectorCollection(ctx, X.shape[1], distance)
    for a in range(0, len(X), BATCH):
        col.add(X[a:a + BATCH])
    return col


def digest(h, res):
    for x in res:
        if isinstance(x, list):
            for s, v in x:
                h.update(np.ascontiguousarray(s).tobytes())
                h.update(np.ascontiguousarray(v).tobytes())
        elif isinstance(x, np.ndarray):
            h.update(np.ascontiguousarray(x).tobytes())


def measure(gb, ctx, X, reps, rng):
    n, dim = X.shape
    q8 = X[rng.integers(0, n, 8192)] + np.float32(0.5) * rng.standard_normal((8192, dim), dtype=np.float32)
    q1 = np.ascontiguousarray(q8[:1024])
    ctx_lists = [rng.integers(0, n, 5) for _ in range(1024)]
    ex_lists = [np.zeros(0, np.int64)] * 1024
    col = build(gb, ctx, X, gb.DISTANCE_DOT)
    rec = {"value_bytes": col.storage()[0], "device_bytes_before_sweep": gb.device_bytes()}
    calls = {"query_1024_s": lambda: col.query(q1, (), 20), "query_8192_s": lambda: col.query(q8, (), 20),
             "i2i_s": lambda: col.item_to_item(ctx_lists, ex_lists, 20)}
    for a in ARMS:   # warm-up: the mirror, the work buffers and every launch shape of the timed calls
        arm(a)
        for f in calls.values():
            f()
    rec["device_bytes_after_sweep"] = gb.device_bytes()
    times = {a: {k: [] for k in calls} for a in ARMS}
    hashes = {}
    for r in range(reps):
        for a in (ARMS if r % 2 == 0 else ARMS[::-1]):
            arm(a)
            h = hashlib.sha256()
            for k, f in calls.items():
                t, res = timed(f)
                times[a][k].append(t)
                digest(h, res if isinstance(res, tuple) and not isinstance(res[0], list) else res[:1])
            assert hashes.setdefault(a, h.hexdigest()) == h.hexdigest(), f"{a}: answers changed between reps"
        log(f"rep {r}: " + ", ".join(f"{a} " + " ".join(f"{k} {v[-1]:.4f}" for k, v in times[a].items()) for a in ARMS))
    arm("sweep")
    _, exact_q = col.query_excluding(q8, [np.zeros(0, np.int64)] * len(q8), 20)
    _, st = col.item_to_item(ctx_lists, ex_lists, 20)
    col.close()
    ix = gb.BruteforceIndex(ctx, dim, gb.METRIC_NEG_DOT)
    for a in range(0, n, BATCH):
        ix.add(X[a:a + BATCH])
    ix.search_vectors(q8, 20)
    ix.stage1_stats()
    ix.search_vectors(q8, 20)
    ms, flop, fb = ix.stage1_stats()
    ix.close()
    rec.update({a: {k: stat(v) for k, v in times[a].items()} for a in ARMS})
    for a in ARMS:
        rec[a]["answers_sha256"] = hashes[a]
    rec["outputs_identical"] = hashes["sweep"] == hashes["exact"]
    rec["fallback_rows"] = {"query_8192": int(exact_q), "i2i": st["exact_rows"], "i2i_context_items": st["context_items"],
                            "index_search_8192": int(fb)}
    rec["stage1"] = {"ms": ms, "flop": flop, "tflops": flop / (ms * 1e-3) / 1e12 if ms > 0 else None}
    return rec


def text_fallback(gb, ctx, small):
    n, dim = (2_000, 1024) if small else (200_000, 1024)
    X = text_like(7, max(n, 40_000), dim)
    rng = np.random.default_rng(8)
    q = X[rng.integers(0, len(X), 1024)] + np.float32(0.3 / np.sqrt(dim)) * rng.standard_normal((1024, dim), dtype=np.float32)
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    out = {"vectors": len(X), "dim": dim, "query_rows": len(q)}
    col = build(gb, ctx, X, gb.DISTANCE_DOT)
    arm("sweep")
    for k in (20, 100):
        _, ex = col.query_excluding(q, [np.zeros(0, np.int64)] * len(q), k)
        out[f"exact_rows_top{k}"] = int(ex)
    col.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--small", action="store_true", help="shapes / 100 (a rehearsal, not a measurement)")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--shapes", default="200k_1024,200k_3072,1m_1024")
    ap.add_argument("--types", default="bf16,fp32")
    ap.add_argument("--text", action="store_true", help="also the fallback rate on text-embedding-like rows")
    args = ap.parse_args()

    import gorse_b200 as gb

    out = {"card_before": card(), "small": args.small, "shapes": {}}
    with gb.Context(0) as ctx:
        for shape in args.shapes.split(","):
            n, dim = SHAPES[shape]
            n = max(n // 100, 40_000) if args.small else n
            for ty in args.types.split(","):
                log(f"{shape} {ty}: {n} x {dim}")
                X = rows(1, n, dim, ty == "bf16")
                rec = measure(gb, ctx, X, args.reps, np.random.default_rng(2))
                del X
                out["shapes"][f"{shape}_{ty}"] = {"vectors": n, "dim": dim, **rec}
                log(json.dumps(out["shapes"][f"{shape}_{ty}"]))
                assert rec["outputs_identical"], f"{shape} {ty}: the sweep and the exact kernel answer differently"
        if args.text:
            out["text_like"] = text_fallback(gb, ctx, args.small)
            log(json.dumps(out["text_like"]))
    out["card_after"] = card()
    print(json.dumps({"metric": "dense top-k at embedding widths: wide tensor-core sweep against the exact kernel, host in to host out", **out}))


if __name__ == "__main__":
    main()
