/* fm_exp.h -- the double exp of the FM ranker's softmax, as one restated algorithm shared by the kernel (csrc/fm.cu) and
 * the CPU restatement of the ranker, so that both give the same bits.
 *
 * The reference's softmax computes float32(math.Exp(float64(x))) (common/nn/tensor.go:414-419).  Go's portable
 * math.Exp is the FreeBSD e_exp.c algorithm: k = round(x / ln 2), r = (x - k ln2_hi) - k ln2_lo, a degree-5 rational
 * correction, then a scaling by 2^k.  It is restated here with every double operation explicit (no contraction; the
 * device side uses __dadd_rn / __dsub_rn / __dmul_rn / __ddiv_rn).  On amd64 Go runs its own assembly instead, which this
 * project does not hold, so whether every result agrees with it after rounding to float32 is not pinned.
 * Plain C99 (the CPU restatement compiles it with gcc -ffp-contract=off) and CUDA. */
#ifndef GORSE_B200_FM_EXP_H
#define GORSE_B200_FM_EXP_H

#include <stdint.h>
#include <string.h>

#if defined(__CUDACC__)
#define FMX_FN static __host__ __device__ __forceinline__
#else
#define FMX_FN static inline
#endif

#if defined(__CUDA_ARCH__)
#define FMX_ADD(a, b) __dadd_rn((a), (b))
#define FMX_SUB(a, b) __dsub_rn((a), (b))
#define FMX_MUL(a, b) __dmul_rn((a), (b))
#define FMX_DIV(a, b) __ddiv_rn((a), (b))
#else
#define FMX_ADD(a, b) ((a) + (b))
#define FMX_SUB(a, b) ((a) - (b))
#define FMX_MUL(a, b) ((a) * (b))
#define FMX_DIV(a, b) ((a) / (b))
#endif

FMX_FN double fmx_pow2(int k) /* 2^k for -1022 <= k <= 1023 */
{
    const uint64_t b = (uint64_t)(k + 1023) << 52;
    double d;
#if defined(__CUDA_ARCH__)
    d = __longlong_as_double((long long)b);
#else
    memcpy(&d, &b, sizeof d);
#endif
    return d;
}

/* exp(x) in double */
FMX_FN double fmx_exp64(double x)
{
    const double LN2_HI = 6.93147180369123816490e-01, LN2_LO = 1.90821492927058770002e-10, LOG2E = 1.44269504088896338700e+00;
    const double OVERFLOW_AT = 7.09782712893383973096e+02, UNDERFLOW_AT = -7.45133219101941108420e+02;
    const double NEAR_ZERO = 1.0 / (double)(1 << 28);
    const double P1 = 1.66666666666666657415e-01, P2 = -2.77777777770155933842e-03, P3 = 6.61375632143793436117e-05,
                 P4 = -1.65339022054652515390e-06, P5 = 4.13813679705723846039e-08;
    if (x != x) return x;
    if (x > OVERFLOW_AT) return 1.0 / 0.0; /* +Inf included */
    if (x < UNDERFLOW_AT) return 0.0;      /* -Inf included */
    if (-NEAR_ZERO < x && x < NEAR_ZERO) return FMX_ADD(1.0, x);
    int k = 0;
    if (x < 0) k = (int)FMX_SUB(FMX_MUL(LOG2E, x), 0.5);
    else if (x > 0) k = (int)FMX_ADD(FMX_MUL(LOG2E, x), 0.5);
    const double hi = FMX_SUB(x, FMX_MUL((double)k, LN2_HI));
    const double lo = FMX_MUL((double)k, LN2_LO);
    const double r = FMX_SUB(hi, lo);
    const double t = FMX_MUL(r, r);
    const double p = FMX_ADD(P4, FMX_MUL(t, P5));
    const double q = FMX_ADD(P3, FMX_MUL(t, p));
    const double s = FMX_ADD(P2, FMX_MUL(t, q));
    const double u = FMX_ADD(P1, FMX_MUL(t, s));
    const double c = FMX_SUB(r, FMX_MUL(t, u));
    const double y = FMX_SUB(1.0, FMX_SUB(FMX_SUB(lo, FMX_DIV(FMX_MUL(r, c), FMX_SUB(2.0, c))), hi));
    /* y * 2^k; k is in [-1075, 1024].  Outside [-1000, 1000] the scaling takes two exact steps and a last rounding, which
     * only changes results far outside float32's range. */
    if (k > 1000) return FMX_MUL(FMX_MUL(y, fmx_pow2(k - 1000)), fmx_pow2(1000));
    if (k < -1000) return FMX_MUL(FMX_MUL(y, fmx_pow2(k + 1000)), fmx_pow2(-1000));
    return FMX_MUL(y, fmx_pow2(k));
}

/* the softmax's exp: float32(exp(float64(x))) */
FMX_FN float fmx_expf(float x) { return (float)fmx_exp64((double)x); }

#endif /* GORSE_B200_FM_EXP_H */
