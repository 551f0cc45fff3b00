"""Generates tests/golden/floats_golden.npz by RUNNING THE REFERENCE's own C kernels
(common/floats/src/floats_avx512.c + floats_avx.c of the reference project, compiled by oracle/Makefile into
oracle/_ref/libfloats_ref.so) on seeded random inputs.  Needs a CPU with AVX-512 and a checkout of the reference:

    GORSE_REFERENCE_DIR=<reference checkout> python tests/golden/make_floats_golden.py

The fixture pins the oracle restatement (tests/test_oracle_floats.py) on machines without the reference.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import oracle  # noqa: E402

LENGTHS = [1, 2, 3, 7, 8, 9, 15, 16, 17, 20, 23, 24, 25, 31, 32, 33, 40, 47, 48, 63, 64, 65, 100, 128, 256]


def main():
    oracle.build(force=True)
    ref = oracle.RefFloats()
    rng = np.random.default_rng(20260922)
    out = {}
    for n in LENGTHS:
        for rep in range(3):
            a = rng.standard_normal(n).astype(np.float32)
            b = rng.standard_normal(n).astype(np.float32)
            c = np.float32(rng.standard_normal())
            key = f"n{n}_r{rep}"
            out[key + "_a"] = a
            out[key + "_b"] = b
            out[key + "_c"] = np.array([c], np.float32)
            for pre, tag in (("_mm512_", "512"), ("_mm256_", "256")):
                out[f"{key}_dot{tag}"] = np.array([ref.call2(pre + "dot", a, b)], np.float32)
                out[f"{key}_euc{tag}"] = np.array([ref.call2(pre + "euclidean", a, b)], np.float32)
                out[f"{key}_mct{tag}"] = ref.mul_const_to(a, c, pre)
                out[f"{key}_mca{tag}"] = ref.mul_const_add(a, c, b, pre)
                out[f"{key}_mcat{tag}"] = ref.mul_const_add_to(a, c, b, pre)
                out[f"{key}_mc{tag}"] = ref.mul_const(a, c, pre)
                out[f"{key}_sub{tag}"] = ref.sub_to(a, b, pre)
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "floats_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
