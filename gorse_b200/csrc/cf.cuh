// cf.cuh -- CF model state in HBM and the device primitives shared by the BPR / ALS / evaluate kernels.
//
// HBM layout (all row-major, natural element order so every kernel and the host mirror agree):
//   P        [n_local_users x d] fp32   user factors of this rank's user shard (all users when world = 1)
//   Q        [n_items x d]       fp32   item factors (replicated across ranks)
//   user_off [n_local_users + 1] int64, user_items [|R_local|] int32   R_u of the shard's users (row u at index u - u_lo,
//            offsets rebased to 0), each row sorted ascending;  user_meta likewise indexed by u - u_lo
//   item_off [n_local_items + 1] int64, item_users [...] int32         R_i of the shard's items (ALS only)
//   active   [n_active] int32    users of this shard with >= 1 feedback, ascending (global ids)
//
// Row -> lane mapping used by every d % 16 == 0 kernel ("quad" layout): 4 lanes own one row.  For the
// c-th 16-float chunk, lane l (0..3) holds the float4 at floats [16c + 4l, 16c + 4l + 4).  A quad
// therefore reads a row as d/16 fully-coalesced 64-byte segments with 128-bit loads, and lane l keeps
// accumulator lanes m = 4l..4l+3 of the reference's 16-lane AVX-512 accumulator
// (common/floats/src/floats_avx512.c:306-341), so the reduce tree below reproduces the reference's
// summation order bit for bit:  r8 = acc[m] + acc[m+8]  (partner lane l^2),  r4 = r8[m] + r8[m+4]
// (partner lane l^1),  result = (r4[0] + r4[2]) + (r4[1] + r4[3])  (inside the lane).
#pragma once
#include "common.cuh"

namespace gb {
// Per-user sampling record: one 16-byte load gives the row's offset and length and a 64-bit Bloom signature
// (one hash) used to answer "j is certainly not in R_u" without a binary search.
struct __align__(16) UserMeta {
    uint64_t off_len;  // offset in the low 38 bits, length in the high 26
    uint64_t bloom;
    __host__ __device__ int64_t off() const { return (int64_t)(off_len & ((1ull << 38) - 1)); }
    __host__ __device__ int64_t len() const { return (int64_t)(off_len >> 38); }
    __host__ __device__ static uint64_t bit(int32_t item) { return 1ull << (((uint32_t)item * 0x9E3779B1u) >> 26); }
    __host__ __device__ bool maybe_contains(int32_t item) const { return (bloom & bit(item)) != 0; }
};
}  // namespace gb

struct gorse_b200_cf {
    gorse_b200_ctx *ctx = nullptr;
    int32_t n_users = 0, n_items = 0, d = 0;
    int32_t u_lo = 0, u_hi = 0;  // user shard [u_lo, u_hi) owned by this rank
    int32_t i_lo = 0, i_hi = 0;  // item shard (the rows of the item CSR this rank holds and updates in the eALS item sweep)
    int64_t n_feedback = 0;         // entries of this rank's user rows
    int64_t n_feedback_global = 0;  // over all ranks (== n_feedback when world = 1)
    int64_t n_item_feedback = 0;    // entries of this rank's item rows
    int32_t n_active = 0;
    bool has_item_csr = false;
    gb::DevBuf<float> P, Q, Q0;
    // multi-rank item exchange (bpr.cu): expected updates of item i per local BPR step, and the [a | L | psq] buffer
    gb::DevBuf<float> item_rate, xchg;
    gb::DevBuf<float> P_all;   // multi-rank eALS: the full user table (every rank needs all of P for its item rows)
    gb::DevBuf<int64_t> user_off, item_off;
    gb::DevBuf<int32_t> user_items, item_users, active;
    gb::DevBuf<gb::UserMeta> user_meta;
    gb::DevBuf<uint32_t> bpr_barrier;  // arrival counter of the round epoch's grid barrier (bpr.cu), zeroed before each launch
    // the two-launch round epoch (bpr.cu, d outside 16/32/64/128): one round's row deltas, 3 * GB_BPR_ROUND rows of d
    // floats, and the rows they go to; allocated by the first such epoch
    gb::DevBuf<float> bpr_delta;
    gb::DevBuf<int32_t> bpr_rows;
    bool all_active = false;  // every user of the shard has feedback: active[k] == u_lo + k
    // ALS scratch
    gb::DevBuf<float> gram;      // d x d
    gb::DevBuf<float> als_pred;  // eALS scratch: one prediction per entry of the longer CSR side, kept across epochs
    gb::DevBuf<int32_t> als_rows[2][7];  // [side][class] row ids bucketed by length (built lazily; als.cu prepare_als)
    int32_t als_rows_n[2][7] = {{0, 0, 0, 0, 0, 0, 0}, {0, 0, 0, 0, 0, 0, 0}};
    bool als_ready = false;
    // long rows in Gram form (d <= 128): chunk work list per side
    int32_t als_n_chunks[2] = {0, 0};
    gb::DevBuf<int32_t> als_chunk_len[2], als_row_chunk0[2];
    gb::DevBuf<int64_t> als_chunk_begin[2];
    // one partial (G, h) per chunk, of a long row or of S, als_partial_stride(d) floats apart
    gb::DevBuf<float> als_partial;
    // rows with feedback, in chunks: what S = sum x x^T runs over
    int32_t als_s_chunks[2] = {0, 0};
    gb::DevBuf<int32_t> als_s_rows[2], als_s_len[2];
    gb::DevBuf<int64_t> als_s_begin[2];
    std::vector<int64_t> h_user_off, h_item_off;  // host copies of the offsets (bucketing, wave building)
};

namespace gb {

// ---- splitmix64-based counter RNG (our design; DESIGN.md "sampling") ---------------------------
__host__ __device__ __forceinline__ uint64_t mix64(uint64_t z)
{
    z ^= z >> 30;
    z *= 0xBF58476D1CE4E5B9ull;
    z ^= z >> 27;
    z *= 0x94D049BB133111EBull;
    z ^= z >> 31;
    return z;
}

struct SStream {
    uint64_t x;
    __host__ __device__ __forceinline__ uint32_t next32()
    {
        x += 0x9E3779B97F4A7C15ull;
        return (uint32_t)(mix64(x) >> 32);
    }
    // unbiased integer in [0, n) (Lemire's multiply-shift with rejection)
    __host__ __device__ __forceinline__ uint32_t bounded(uint32_t n)
    {
        uint64_t m = (uint64_t)next32() * n;
        uint32_t l = (uint32_t)m;
        if (l < n) {
            uint32_t t = (0u - n) % n;
            while (l < t) {
                m = (uint64_t)next32() * n;
                l = (uint32_t)m;
            }
        }
        return (uint32_t)(m >> 32);
    }
};

#ifdef __CUDACC__

__device__ __forceinline__ UserMeta ld_meta(const UserMeta *p)
{
    const uint4 r = __ldg(reinterpret_cast<const uint4 *>(p));
    UserMeta m;
    m.off_len = (uint64_t)r.x | ((uint64_t)r.y << 32);
    m.bloom = (uint64_t)r.z | ((uint64_t)r.w << 32);
    return m;
}

__device__ __forceinline__ unsigned quad_mask() { return 0xFu << (threadIdx.x & 28u); }

// chewxy/math32 Exp as restated in DESIGN.md: the FreeBSD e_expf.c algorithm, each operation rounded
// to fp32 (no contraction).  model/cf/model.go:470-471.
__device__ __forceinline__ float exp_math32(float x)
{
    const float Ln2Hi = 6.9313812256e-01f, Ln2Lo = 9.0580006145e-06f, Log2e = 1.4426950216e+00f;
    const float Overflow = 7.09782712893383973096e+02f, Underflow = -7.45133219101941108420e+02f;
    const float NearZero = 1.0f / (float)(1 << 28);
    const float P1 = 1.6666667163e-01f, P2 = -2.7777778450e-03f, P3 = 6.6137559770e-05f,
                P4 = -1.6533901999e-06f, P5 = 4.1381369442e-08f;
    if (isnan(x) || (isinf(x) && x > 0)) return x;
    if (isinf(x)) return 0.0f;
    if (x > Overflow) return __int_as_float(0x7f800000);
    if (x < Underflow) return 0.0f;
    if (-NearZero < x && x < NearZero) return __fadd_rn(1.0f, x);
    int k = 0;
    if (x < 0) k = (int)__fsub_rn(__fmul_rn(Log2e, x), 0.5f);
    else if (x > 0) k = (int)__fadd_rn(__fmul_rn(Log2e, x), 0.5f);
    float kf = (float)k;
    float hi = __fsub_rn(x, __fmul_rn(kf, Ln2Hi));
    float lo = __fmul_rn(kf, Ln2Lo);
    float r = __fsub_rn(hi, lo);
    float t = __fmul_rn(r, r);
    float c = __fmul_rn(t, P5);
    c = __fadd_rn(P4, c); c = __fmul_rn(t, c);
    c = __fadd_rn(P3, c); c = __fmul_rn(t, c);
    c = __fadd_rn(P2, c); c = __fmul_rn(t, c);
    c = __fadd_rn(P1, c); c = __fmul_rn(t, c);
    c = __fsub_rn(r, c);
    float y = __fdiv_rn(__fmul_rn(r, c), __fsub_rn(2.0f, c));
    y = __fsub_rn(lo, y);
    y = __fsub_rn(y, hi);
    y = __fsub_rn(1.0f, y);
    return ldexpf(y, k);
}

// one chunk of the quad dot: first chunk multiplies, later chunks fuse (floats_avx512.c:312-326)
__device__ __forceinline__ void dot_chunk(float4 &acc, const float4 a, const float4 b, bool first)
{
    if (first) {
        acc.x = __fmul_rn(a.x, b.x); acc.y = __fmul_rn(a.y, b.y);
        acc.z = __fmul_rn(a.z, b.z); acc.w = __fmul_rn(a.w, b.w);
    } else {
        acc.x = __fmaf_rn(a.x, b.x, acc.x); acc.y = __fmaf_rn(a.y, b.y, acc.y);
        acc.z = __fmaf_rn(a.z, b.z, acc.z); acc.w = __fmaf_rn(a.w, b.w, acc.w);
    }
}

// reduce tree of the 16-lane accumulator spread over a quad (floats_avx512.c:327-339); every lane of
// the quad ends up with the same bits
__device__ __forceinline__ float quad_tree(float4 acc, unsigned mask)
{
    acc.x = __fadd_rn(acc.x, __shfl_xor_sync(mask, acc.x, 2));
    acc.y = __fadd_rn(acc.y, __shfl_xor_sync(mask, acc.y, 2));
    acc.z = __fadd_rn(acc.z, __shfl_xor_sync(mask, acc.z, 2));
    acc.w = __fadd_rn(acc.w, __shfl_xor_sync(mask, acc.w, 2));
    acc.x = __fadd_rn(acc.x, __shfl_xor_sync(mask, acc.x, 1));
    acc.y = __fadd_rn(acc.y, __shfl_xor_sync(mask, acc.y, 1));
    acc.z = __fadd_rn(acc.z, __shfl_xor_sync(mask, acc.z, 1));
    acc.w = __fadd_rn(acc.w, __shfl_xor_sync(mask, acc.w, 1));
    return __fadd_rn(__fadd_rn(acc.x, acc.z), __fadd_rn(acc.y, acc.w));
}

// floats.Dot for d % 16 == 0 rows read straight from global memory by a quad
__device__ __forceinline__ float quad_dot_global(const float *a, const float *b, int chunks, int lane4, unsigned mask)
{
    const float4 *a4 = reinterpret_cast<const float4 *>(a) + lane4;
    const float4 *b4 = reinterpret_cast<const float4 *>(b) + lane4;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int c = 0; c < chunks; c++) dot_chunk(acc, a4[4 * c], b4[4 * c], c == 0);
    return quad_tree(acc, mask);
}

// value i of a row: fp32, or bf16 kept as the high 16 bits of the fp32 pattern (a vector collection's rows, topk.cuh), widened
// exactly by a shift
template <typename I>
__device__ __forceinline__ float row_val(const float *x, I i) { return x[i]; }
template <typename I>
__device__ __forceinline__ float row_val(const uint16_t *x, I i) { return __uint_as_float((uint32_t)__ldg(x + i) << 16); }

// floats.Dot for any d, one thread, the reference's order: 16-lane body, 8-lane block, fused scalar tail
// (common/floats/src/floats_avx512.c:306-367 and the committed assembly for which parts fuse).  TA, TB: float, or uint16_t for
// bf16 rows (row_val).
// values 0 .. 15 of a bf16 row chunk, widened: four 8-byte loads when the chunk is 8-byte aligned (d % 4 == 0), else 16
// 2-byte loads.  The one-thread scans (dot_any, dist_any) read bf16 rows through it, so that a value costs fewer load
// instructions than an fp32 value does.
__device__ __forceinline__ void row_chunk16(const uint16_t *p, float (&v)[16])
{
    if ((reinterpret_cast<uintptr_t>(p) & 7u) == 0) {
#pragma unroll
        for (int i = 0; i < 4; i++) {
            const uint2 u = __ldg(reinterpret_cast<const uint2 *>(p) + i);
            v[4 * i] = __uint_as_float(u.x << 16);
            v[4 * i + 1] = __uint_as_float(u.x & 0xffff0000u);
            v[4 * i + 2] = __uint_as_float(u.y << 16);
            v[4 * i + 3] = __uint_as_float(u.y & 0xffff0000u);
        }
    } else {
#pragma unroll
        for (int l = 0; l < 16; l++) v[l] = row_val(p, l);
    }
}

template <typename TA, typename TB>
__device__ inline float dot_any(const TA *a, const TB *b, int n)
{
    int epoch = n / 16, remain = n % 16;
    float s[16];
#pragma unroll
    for (int l = 0; l < 16; l++) s[l] = 0.f;
    if constexpr (std::is_same<TA, float>::value && std::is_same<TB, uint16_t>::value) {   // a bf16 row against an fp32 query
        float bv[16];
        if (epoch > 0) {
            row_chunk16(b, bv);
#pragma unroll
            for (int l = 0; l < 16; l++) s[l] = __fmul_rn(a[l], bv[l]);
        }
        for (int c = 1; c < epoch; c++) {
            row_chunk16(b + 16 * c, bv);
#pragma unroll
            for (int l = 0; l < 16; l++) s[l] = __fmaf_rn(a[16 * c + l], bv[l], s[l]);
        }
    } else {
        if (epoch > 0) {
#pragma unroll
            for (int l = 0; l < 16; l++) s[l] = __fmul_rn(row_val(a, l), row_val(b, l));
        }
        for (int c = 1; c < epoch; c++) {
#pragma unroll
            for (int l = 0; l < 16; l++) s[l] = __fmaf_rn(row_val(a, 16 * c + l), row_val(b, 16 * c + l), s[l]);
        }
    }
    float r4[4];
#pragma unroll
    for (int l = 0; l < 4; l++) r4[l] = __fadd_rn(__fadd_rn(s[l + 12], s[l + 4]), __fadd_rn(s[l + 8], s[l]));
    float sum = __fadd_rn(__fadd_rn(r4[0], r4[2]), __fadd_rn(r4[1], r4[3]));
    a += 16 * epoch;
    b += 16 * epoch;
    if (remain >= 8) {
        float q4[4];
#pragma unroll
        for (int l = 0; l < 4; l++) q4[l] = __fadd_rn(__fmul_rn(row_val(a, l + 4), row_val(b, l + 4)), __fmul_rn(row_val(a, l), row_val(b, l)));
        sum = __fadd_rn(sum, __fadd_rn(__fadd_rn(q4[0], q4[2]), __fadd_rn(q4[1], q4[3])));
        a += 8;
        b += 8;
        remain -= 8;
    }
    for (int i = 0; i < remain; i++) sum = __fmaf_rn(row_val(a, i), row_val(b, i), sum);
    return sum;
}

// dst[i] = fma(a[i], c, dst[i]) with the reference's per-index fusing rule (mul_const_add,
// floats_avx512.c:51-80): body and tail fuse, the 8-lane block rounds twice
__device__ __forceinline__ float axpy_elem(float a, float c, float dst, int idx, int n)
{
    int body = (n / 16) * 16;
    bool in_block8 = idx >= body && (n - body) >= 8 && idx < body + 8;
    return in_block8 ? __fadd_rn(__fmul_rn(a, c), dst) : __fmaf_rn(a, c, dst);
}

__device__ __forceinline__ bool row_contains(const int32_t *row, int64_t len, int32_t v)
{
    int64_t lo = 0, hi = len;
    while (lo < hi) {
        int64_t mid = (lo + hi) >> 1;
        if (row[mid] < v) lo = mid + 1;
        else hi = mid;
    }
    return lo < len && row[lo] == v;
}

#endif  // __CUDACC__

}  // namespace gb
