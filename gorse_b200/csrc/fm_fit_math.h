/* fm_fit_math.h -- the two scalar functions of FM training that the project restates itself, shared by the kernel
 * (csrc/fm_fit.cu) and the CPU restatement (fm_fit_oracle.c of the test suite) so that both give the same bits.
 *
 * fmx_logf: the loss's Log (common/nn/tensor.go:421-426) is math32.Log.  Restated here as the FreeBSD e_logf.c
 *   algorithm that Go's math.Log follows, in float32 with e_logf.c's constants: x = 2^k (1 + f) with 1 + f in
 *   [sqrt(2)/2, sqrt(2)), s = f / (2 + f), a degree-7 odd polynomial in s, then k ln2 split in two parts.  Every float
 *   operation is explicit and rounds once (no contraction; the device side uses __fadd_rn / __fmul_rn / __fdiv_rn).
 *   On amd64 math32 may run its own assembly, which this project does not hold, so agreement with it is not pinned.
 * fmx_pow_steps: Adam's bias corrections (common/nn/optimizers.go:121-122) use math32.Pow(beta, t) with a whole t.
 *   Restated as exponentiation by squaring in double, rounded once to float32.  The host computes it once per step;
 *   agreement with math32.Pow is not pinned either.
 * Plain C99 and CUDA. */
#ifndef GORSE_B200_FM_FIT_MATH_H
#define GORSE_B200_FM_FIT_MATH_H

#include <stdint.h>
#include <string.h>

#if defined(__CUDACC__)
#define FMF_FN static __host__ __device__ __forceinline__
#else
#define FMF_FN static inline
#endif

#if defined(__CUDA_ARCH__)
#define FMF_ADD(a, b) __fadd_rn((a), (b))
#define FMF_SUB(a, b) __fsub_rn((a), (b))
#define FMF_MUL(a, b) __fmul_rn((a), (b))
#define FMF_DIV(a, b) __fdiv_rn((a), (b))
#else
#define FMF_ADD(a, b) ((a) + (b))
#define FMF_SUB(a, b) ((a) - (b))
#define FMF_MUL(a, b) ((a) * (b))
#define FMF_DIV(a, b) ((a) / (b))
#endif

FMF_FN uint32_t fmf_bits(float x)
{
#if defined(__CUDA_ARCH__)
    return __float_as_uint(x);
#else
    uint32_t b;
    memcpy(&b, &x, 4);
    return b;
#endif
}

FMF_FN float fmf_from_bits(uint32_t b)
{
#if defined(__CUDA_ARCH__)
    return __uint_as_float(b);
#else
    float x;
    memcpy(&x, &b, 4);
    return x;
#endif
}

/* natural log in float32 */
FMF_FN float fmx_logf(float x)
{
    const float LN2_HI = 6.9313812256e-01f, LN2_LO = 9.0580006145e-06f;
    const float L1 = 6.6666668653e-01f, L2 = 4.0000000596e-01f, L3 = 2.8571429849e-01f, L4 = 2.2222198546e-01f,
                L5 = 1.8183572590e-01f, L6 = 1.5313838422e-01f, L7 = 1.4798198640e-01f;
    const float SQRT2_2 = 7.0710677e-01f;
    const uint32_t b0 = fmf_bits(x);
    if (x != x || b0 == 0x7f800000u) return x;       /* NaN, +Inf */
    if (x < 0.0f) return fmf_from_bits(0x7fc00000u); /* NaN */
    if (x == 0.0f) return fmf_from_bits(0xff800000u); /* -Inf */
    /* Frexp: x = f1 2^ki with f1 in [0.5, 1) */
    int ki = 0;
    uint32_t b = b0;
    if ((b & 0x7f800000u) == 0) { /* subnormal: scale by 2^23 first */
        b = fmf_bits(FMF_MUL(x, 8388608.0f));
        ki = -23;
    }
    ki += (int)((b >> 23) & 0xffu) - 126;
    float f1 = fmf_from_bits((b & 0x807fffffu) | (126u << 23));
    if (f1 < SQRT2_2) {
        f1 = FMF_MUL(f1, 2.0f);
        ki--;
    }
    const float f = FMF_SUB(f1, 1.0f);
    const float k = (float)ki;
    const float s = FMF_DIV(f, FMF_ADD(2.0f, f));
    const float s2 = FMF_MUL(s, s);
    const float s4 = FMF_MUL(s2, s2);
    const float t1 = FMF_MUL(s2, FMF_ADD(L1, FMF_MUL(s4, FMF_ADD(L3, FMF_MUL(s4, FMF_ADD(L5, FMF_MUL(s4, L7)))))));
    const float t2 = FMF_MUL(s4, FMF_ADD(L2, FMF_MUL(s4, FMF_ADD(L4, FMF_MUL(s4, L6)))));
    const float R = FMF_ADD(t1, t2);
    const float hfsq = FMF_MUL(FMF_MUL(0.5f, f), f);
    return FMF_SUB(FMF_MUL(k, LN2_HI), FMF_SUB(FMF_SUB(hfsq, FMF_ADD(FMF_MUL(s, FMF_ADD(hfsq, R)), FMF_MUL(k, LN2_LO))), f));
}

/* beta^t for a whole t >= 0 */
FMF_FN float fmx_pow_steps(float beta, int64_t t)
{
    double r = 1.0, b = (double)beta;
    for (; t > 0; t >>= 1) {
        if (t & 1) r *= b;
        b *= b;
    }
    return (float)r;
}

#endif /* GORSE_B200_FM_FIT_MATH_H */
