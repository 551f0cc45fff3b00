"""Generates tests/golden/ref_kernels_golden.npz by RUNNING THE REFERENCE's own C kernels (common/floats/src/floats_avx512.c +
floats_avx.c of the reference project, compiled by oracle/Makefile into oracle/_ref/libfloats_ref.so) on the exact inputs of
tests/test_oracle_floats.py's two live checks:

  * live_n<n>_*: _mm512_dot, _mm512_euclidean and (where the check uses it) _mm512_mul_const_add on seeded vectors of
    length n
  * bpr_d<d>_P_sha256 / _Q_sha256: SHA-256 of the bytes of the factors after BPR.Fit's per-triple call sequence ran through
    those kernels (one thread, 20000 sampled triples); the check is bit equality, so the digests keep the fixture small

so that both checks also run where the reference is not available.  Needs a CPU with AVX-512 and a checkout of the
reference project:

    GORSE_REFERENCE_DIR=<reference checkout> python tests/golden/make_ref_kernels_golden.py
"""
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import oracle  # noqa: E402
from test_oracle_floats import BPR_DIMS, LIVE_LENGTHS, bpr_problem, live_inputs  # noqa: E402


def main():
    oracle.build(force=True)
    assert oracle.ref_available() and oracle.ref_bind(), "oracle/_ref is not built"
    ref = oracle.RefFloats()
    out = {}
    for n, a, b, c in live_inputs():
        out[f"live_n{n}_dot"] = np.array([ref.call2("_mm512_dot", a, b)], np.float32)
        out[f"live_n{n}_euc"] = np.array([ref.call2("_mm512_euclidean", a, b)], np.float32)
        if n % 16 < 8:
            out[f"live_n{n}_mca"] = ref.mul_const_add(a, c, b)
    for d in BPR_DIMS:
        P, Q, off, items, act = bpr_problem(d)
        oracle.bpr_epoch_threads(P, Q, off, items, act, 42, 20000, 0.05, 0.01, 1, use_ref=True)
        out[f"bpr_d{d}_P_sha256"] = np.frombuffer(hashlib.sha256(P.tobytes()).digest(), np.uint8)
        out[f"bpr_d{d}_Q_sha256"] = np.frombuffer(hashlib.sha256(Q.tobytes()).digest(), np.uint8)
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "ref_kernels_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
