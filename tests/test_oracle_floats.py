"""Pins the oracle's common/floats restatement:
  * known answers lifted (values only) from common/floats/floats_test.go
  * bit-equality against golden vectors produced by the reference's own C kernels
    (tests/golden/make_floats_golden.py, tests/golden/make_ref_kernels_golden.py) and, when oracle/_ref is present on a
    CPU with AVX-512, against them live.
"""
import hashlib
import os

import numpy as np
import pytest

GOLD = os.path.join(os.path.dirname(__file__), "golden", "floats_golden.npz")
REF_GOLD = os.path.join(os.path.dirname(__file__), "golden", "ref_kernels_golden.npz")
LIVE_LENGTHS = list(range(1, 70)) + [96, 128, 200, 256]
BPR_DIMS = [16, 32, 64, 128]


def live_inputs():
    """(n, a, b, c) of the live comparison, in the order the seeded generator yields them"""
    rng = np.random.default_rng(7)
    for n in LIVE_LENGTHS:
        a = rng.standard_normal(n).astype(np.float32)
        b = rng.standard_normal(n).astype(np.float32)
        c = np.float32(rng.standard_normal())
        yield n, a, b, c


def bpr_problem(d):
    """(P, Q, user_off, user_items, active users) of the BPR step comparison"""
    from gorse_b200 import synth

    U, I = 300, 120
    off, items = synth.make_feedback(U, I, 4000, seed=d)
    act = np.nonzero(np.diff(off) > 0)[0].astype(np.int32)
    rng = np.random.default_rng(d)
    P0 = (rng.standard_normal((U, d)) * 0.3).astype(np.float32)   # large enough that the sigmoid gradient is not ~0.5
    Q0 = (rng.standard_normal((I, d)) * 0.3).astype(np.float32)
    return P0, Q0, off, items, act


def ref_runs(orc):
    """the reference's own kernels can be called here (oracle/_ref built, CPU with AVX-512)"""
    return orc.ref_available() and "avx512f" in open("/proc/cpuinfo").read()


def ramp(n, step=1):
    return (np.arange(n) * step).astype(np.float32)


def test_known_answers_floats_test_go(orc):
    L = orc.lib()
    a, b = ramp(11), ramp(11, 2)
    # floats_test.go:167-172 TestDot, :174-179 TestEuclidean
    assert orc.dot(a, b) == np.float32(770)
    assert orc.euclidean(a, b) == np.float32(19.621416)
    assert np.float32(L.gbo_dot_scalar(a, b, 11)) == np.float32(770)
    assert np.float32(L.gbo_euclidean_scalar(a, b, 11)) == np.float32(19.621416)
    # :91-98 TestMulConstTo
    dst = np.zeros(11, np.float32)
    L.gbo_mul_const_to(a, 2.0, dst, 11)
    assert dst.tolist() == (2 * np.arange(11)).tolist()
    # :100-107 TestMulConstAdd
    dst = ramp(11)
    L.gbo_mul_const_add(a, 2.0, dst, 11)
    assert dst.tolist() == (3 * np.arange(11)).tolist()
    # :109-116 TestMulConstAddTo
    dst = np.zeros(11, np.float32)
    L.gbo_mul_const_add_to(a, 3.0, b, dst, 11)
    assert dst.tolist() == (5 * np.arange(11)).tolist()
    # :59-66 TestSubTo, :77-81 TestMulConst
    c = np.zeros(4, np.float32)
    L.gbo_sub_to(np.array([1, 2, 3, 4], np.float32), np.array([5, 6, 7, 8], np.float32), c, 4)
    assert c.tolist() == [-4, -4, -4, -4]
    m = np.array([1, 2, 3, 4], np.float32)
    L.gbo_mul_const(m, 2.0, 4)
    assert m.tolist() == [2, 4, 6, 8]


def test_simd_suite_equals_scalar_on_ramps(orc):
    # floats_test.go:318-423 SIMDTestSuite: each ISA variant == scalar Go loop on 20-element ramps
    L = orc.lib()
    a = np.arange(1, 21).astype(np.float32)
    b = (10 * np.arange(1, 21)).astype(np.float32)
    assert orc.dot(a, b) == np.float32(L.gbo_dot_scalar(a, b, 20))
    assert orc.euclidean(a, b) == np.float32(L.gbo_euclidean_scalar(a, b, 20))
    dst = b.copy()
    L.gbo_mul_const_add(a, 2.0, dst, 20)
    assert dst.tolist() == (b + 2 * a).tolist()


def _check_against(get, orc, key, a, b, c, tag):
    L = orc.lib()
    n = a.size
    if tag == "512":
        assert orc.dot(a, b).tobytes() == get(f"{key}_dot512").tobytes(), key
        assert orc.euclidean(a, b).tobytes() == get(f"{key}_euc512").tobytes(), key
        # The committed Go assembly (clang) keeps the 8-lane block of mul_const_add[_to] as vmulps+vaddps
        # (floats_avx512.s:160-161) while gcc 13 -- the only compiler here -- contracts those intrinsics
        # into an FMA whenever tail fusion is enabled.  The oracle follows the assembly; the gcc-built
        # golden is therefore only comparable when no 8-lane block exists (n % 16 < 8; every BASELINE
        # config has d % 16 == 0).
        if n % 16 < 8:
            d = b.copy()
            L.gbo_mul_const_add(a, c, d, n)
            assert d.tobytes() == get(f"{key}_mca512").tobytes(), key
            d = np.zeros_like(a)
            L.gbo_mul_const_add_to(a, c, b, d, n)
            assert d.tobytes() == get(f"{key}_mcat512").tobytes(), key
    d = np.zeros_like(a)
    L.gbo_mul_const_to(a, c, d, n)
    assert d.tobytes() == get(f"{key}_mct{tag}").tobytes(), key
    d = a.copy()
    L.gbo_mul_const(d, c, n)
    assert d.tobytes() == get(f"{key}_mc{tag}").tobytes(), key
    d = np.zeros_like(a)
    L.gbo_sub_to(a, b, d, n)
    assert d.tobytes() == get(f"{key}_sub{tag}").tobytes(), key


def test_bit_equal_to_reference_golden(orc):
    g = np.load(GOLD)
    keys = sorted({k.rsplit("_", 1)[0] for k in g.files if k.endswith("_a")})
    assert len(keys) >= 60
    for key in keys:
        a, b, c = g[key + "_a"], g[key + "_b"], float(g[key + "_c"][0])
        _check_against(lambda k: np.asarray(g[k]).reshape(-1)[0] if g[k].size == 1 and ("dot" in k or "euc" in k)
                       else g[k], orc, key, a, b, np.float32(c), "512")
        # element-wise ops have no reduction order: the AVX (256) variant must agree too
        _check_against(lambda k: g[k], orc, key, a, b, np.float32(c), "256")


def test_bit_equal_to_reference_live(orc):
    """The reference's kernels run live where they can; elsewhere their stored outputs for the same inputs stand in."""
    ref = orc.RefFloats() if ref_runs(orc) else None
    g = np.load(REF_GOLD)
    for n, a, b, c in live_inputs():
        dot = ref.call2("_mm512_dot", a, b) if ref else np.float32(g[f"live_n{n}_dot"][0])
        euc = ref.call2("_mm512_euclidean", a, b) if ref else np.float32(g[f"live_n{n}_euc"][0])
        assert orc.dot(a, b).tobytes() == dot.tobytes(), n
        assert orc.euclidean(a, b).tobytes() == euc.tobytes(), n
        if n % 16 < 8:  # see _check_against
            d = b.copy()
            orc.lib().gbo_mul_const_add(a, c, d, n)
            assert d.tobytes() == (ref.mul_const_add(a, c, b) if ref else g[f"live_n{n}_mca"]).tobytes(), n


def test_exp_accuracy(orc):
    # math32.Exp restatement (parity unpinned): must be a faithful exp to <= 2 ulp on the BPR range
    xs = np.concatenate([np.linspace(-20, 20, 4001), np.linspace(-1e-3, 1e-3, 201)]).astype(np.float32)
    got = np.array([orc.exp(x) for x in xs], np.float32)
    want = np.exp(xs.astype(np.float64))
    ulp = np.abs(got.astype(np.float64) - want) / np.spacing(want.astype(np.float32)).astype(np.float64)
    assert ulp.max() <= 2.0, ulp.max()
    assert orc.exp(np.float32(0)) == np.float32(1)
    assert np.isinf(orc.exp(np.float32(89.0)))       # SURVEY F11: overflow -> +Inf -> NaN gradient
    assert orc.exp(np.float32(-200.0)) == np.float32(0)


@pytest.mark.parametrize("d", BPR_DIMS)
def test_bpr_step_through_the_reference_kernels(orc, d):
    """BPR.Fit's per-triple call sequence (model/cf/model.go:469-488) executed with the REFERENCE'S OWN compiled
    kernels (oracle/_ref: _mm512_dot, _mm512_mul_const_to, _mm512_mul_const_add, _mm512_sub_to, _mm512_mul_const) against
    the oracle's restatement of the same step, one thread, same triple stream: factors must agree bit for bit.  Where the
    reference's kernels cannot run, the stored digests of their result (tests/golden/ref_kernels_golden.npz) stand in."""
    P0, Q0, off, items, act = bpr_problem(d)
    Pa, Qa = P0.copy(), Q0.copy()
    orc.bpr_epoch_threads(Pa, Qa, off, items, act, 42, 20000, 0.05, 0.01, 1, use_ref=False)
    assert not np.array_equal(Pa, P0)
    if ref_runs(orc):
        assert orc.ref_bind()
        Pb, Qb = P0.copy(), Q0.copy()
        orc.bpr_epoch_threads(Pb, Qb, off, items, act, 42, 20000, 0.05, 0.01, 1, use_ref=True)
        assert Pa.tobytes() == Pb.tobytes() and Qa.tobytes() == Qb.tobytes()
    else:
        g = np.load(REF_GOLD)
        assert hashlib.sha256(Pa.tobytes()).digest() == g[f"bpr_d{d}_P_sha256"].tobytes()
        assert hashlib.sha256(Qa.tobytes()).digest() == g[f"bpr_d{d}_Q_sha256"].tobytes()
