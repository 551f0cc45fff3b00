"""Regenerates tests/golden/fm_mm_golden.npz: the outputs of the reference's compiled _mm512_mm (all four transpose cases)
and _mm512_dot (oracle/_ref) on the seeded operands of tests/test_oracle_fm_fit_emb.py.  Run from the repository root where
the reference project is available:  python tests/golden/make_fm_mm_golden.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import test_oracle_fm_fit_emb as t  # noqa: E402

out = t.reference_outputs()
assert out is not None, "oracle/_ref is not built: the reference project was not found"
np.savez(t.GOLDEN, **out)
print("wrote", t.GOLDEN)
