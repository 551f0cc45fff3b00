// als_gram_tc.cu -- the Gram form of long eALS rows on the Hopper tensor cores (d = 128).
//
// For a row with many entries the coordinate sweep of model/cf/model.go:664-686 is one Gauss-Seidel sweep on A x = h with
// A = (1-w) G + w S + reg I,  G = sum_t y_t y_t^T,  h = sum_t y_t  (als.cu, "Gram form").  G is |R_row| * d^2 multiply-adds,
// and most of the item side's feedback sits in long rows, so this one dense contraction of the eALS epoch goes to wgmma:
//
//   D[64 x 128] (fp32, registers) += A[64 x 8] * B[128 x 8]^T   per instruction, kind tf32, one warpgroup
//
// with A = rows 64 g .. 64 g + 63 (warpgroup g of two) and B = all 128 rows of the tile of gathered entries, transposed.
// wgmma takes 32-bit operands K-major only (K = entry contiguous), while the gathered data lie in memory as [entry][d]; the
// tile is therefore written transposed, [d][entry], one 4-byte store per value: thread = entry, so a warp's 32 stores of
// one d row land in 32 different banks.  A stage is KT = 32 entries = one 128-byte row per d, stored in the 128-byte swizzle
// (16-byte chunk index ^= d % 8) that the descriptor names; one K = 8 instruction advances 32 bytes along the row.
//
// fp32-grade accuracy from tf32 operands ("3xTF32"): y = hi + lo with hi = y rounded to tf32 and lo = (y - hi) rounded to tf32;
// G ~= hi hi^T + hi lo^T + lo hi^T, three MMAs per k-step into the same accumulator.  Dropped: lo lo^T and the rounding of
// lo, both <= 2^-22 relative per product and of random sign.
//
// One CTA = one chunk (<= GB_ALS_CHUNK entries of one row, or rows with feedback for S): 256 threads gather KT = 32 entries per stage into registers,
// split them into the hi and lo tiles of a 3-stage ring and issue the stage's 12 MMAs per warpgroup asynchronously; the
// gather of the next stage overlaps them.  Epilogue: each thread stores its accumulator fragment straight into the partial
// (G, h) buffer that gram_reduce_kernel (for S) or als_partial_reduce_kernel (for a long row) sums.
#include "als.cuh"
#include "wgmma.cuh"

namespace gb {

namespace {

constexpr int TC_D = 128, TC_KT = 32, TC_STAGES = 3, TC_THREADS = 256;
constexpr uint32_t TC_TILE_BYTES = TC_D * TC_KT * 4;          // one [128 d x 32 entries] tile = 16 KB

// fp32 -> tf32 with round-to-nearest (the tensor core itself TRUNCATES the low 13 mantissa bits of an fp32 word: splitting by
// truncation leaves |lo| < 2^-10 |y| with the sign of y, and the dropped lo*lo term and the truncation of lo then bias every
// entry of G by ~1e-6 relative in the same direction.  Rounded: |lo| <= 2^-11 |y| with random sign, and lo is exactly
// representable, so nothing is truncated.)
__device__ __forceinline__ float to_tf32(float x)
{
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return __uint_as_float(r);
}

__global__ void __launch_bounds__(TC_THREADS)
als_chunk_gram_tc_kernel(const float *Y, const int32_t *idx, const int64_t *chunk_begin, const int32_t *chunk_len, float *partial)
{
    using namespace mma;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t *tiles = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);   // [STAGES][hi, lo]

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2;
    const int64_t b0 = chunk_begin[blockIdx.x];
    const int len = chunk_len[blockIdx.x];
    const int n_stage = (len + TC_KT - 1) / TC_KT;
    // thread -> entry `lane` of a stage and the 16-byte chunks c = 4 warp + i (i < 4) of its row: d = 16 warp .. 16 warp + 15
    float4 pre[4], hsum[4];
#pragma unroll
    for (int i = 0; i < 4; i++) hsum[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    auto gather = [&](int st) {
        const int k = st * TC_KT + lane;
        const float4 *src = k < len ? reinterpret_cast<const float4 *>(Y + (int64_t)__ldg(idx + b0 + k) * TC_D) + 4 * warp : nullptr;
#pragma unroll
        for (int i = 0; i < 4; i++) pre[i] = src ? __ldg(src + i) : make_float4(0.f, 0.f, 0.f, 0.f);
    };
    float acc[64];   // written first by an MMA with the accumulate flag off (an explicit zeroing would serialise the MMAs)
    if (n_stage > 0) gather(0);
    for (int st = 0; st < n_stage; st++) {
        const int slot = st % TC_STAGES;
        // the MMAs that read this ring slot (stage st - STAGES) have retired: this warpgroup's by the wait, the other's by the barrier
        wgmma_wait<TC_STAGES - 1>();
        __syncthreads();
        uint8_t *hi = tiles + (size_t)slot * 2 * TC_TILE_BYTES, *lo = hi + TC_TILE_BYTES;
#pragma unroll
        for (int i = 0; i < 4; i++) {
            const float4 v = pre[i];
            hsum[i].x += v.x; hsum[i].y += v.y; hsum[i].z += v.z; hsum[i].w += v.w;
            const float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int q = 0; q < 4; q++) {
                const int m = 16 * warp + 4 * i + q;   // d index = tile row
                const uint32_t o = (uint32_t)m * 128u + ((((uint32_t)lane >> 2) ^ ((uint32_t)m & 7u)) << 4) + (((uint32_t)lane & 3u) << 2);
                const float h = to_tf32(vv[q]);
                *reinterpret_cast<float *>(hi + o) = h;
                *reinterpret_cast<float *>(lo + o) = to_tf32(vv[q] - h);
            }
        }
        if (st + 1 < n_stage) gather(st + 1);   // in flight while this stage's MMAs run
        // generic-proxy stores -> async-proxy (tensor core) reads
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncthreads();
        wgmma_fence();
        const uint32_t b_hi = s32(hi), b_lo = s32(lo), a_hi = b_hi + (uint32_t)wg * 64u * 128u, a_lo = b_lo + (uint32_t)wg * 64u * 128u;
#pragma unroll
        for (int ks = 0; ks < TC_KT / 8; ks++) {
            const uint32_t ko = (uint32_t)ks * 32u;   // 8 tf32 = 32 bytes along the row
            wgmma_m64n128k8_tf32(acc, wgmma_desc(a_hi + ko), wgmma_desc(b_hi + ko), (st | ks) != 0);
            wgmma_m64n128k8_tf32(acc, wgmma_desc(a_hi + ko), wgmma_desc(b_lo + ko), 1);
            wgmma_m64n128k8_tf32(acc, wgmma_desc(a_lo + ko), wgmma_desc(b_hi + ko), 1);
        }
        wgmma_commit();
    }
    wgmma_wait<0>();
    float *out = partial + (int64_t)blockIdx.x * als_partial_stride(TC_D);
    if (n_stage == 0) {
#pragma unroll
        for (int e = 0; e < 64; e++) acc[e] = 0.f;
    }
    {
        // accumulator fragment -> G rows 64 wg + 16 (warp % 4) + lane / 4 (+ 8), columns 8 j + 2 (lane % 4) + {0, 1}
        const int r = 64 * wg + 16 * (warp & 3) + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
        for (int j = 0; j < TC_D / 8; j++) {
            *reinterpret_cast<float2 *>(out + r * TC_D + 8 * j + c0) = make_float2(acc[4 * j], acc[4 * j + 1]);
            *reinterpret_cast<float2 *>(out + (r + 8) * TC_D + 8 * j + c0) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
        }
    }
    // column sums h: reduce the 32 entries (lanes) of every chunk
#pragma unroll
    for (int i = 0; i < 4; i++) {
#pragma unroll
        for (int o = 16; o; o >>= 1) {
            hsum[i].x += __shfl_xor_sync(0xffffffffu, hsum[i].x, o);
            hsum[i].y += __shfl_xor_sync(0xffffffffu, hsum[i].y, o);
            hsum[i].z += __shfl_xor_sync(0xffffffffu, hsum[i].z, o);
            hsum[i].w += __shfl_xor_sync(0xffffffffu, hsum[i].w, o);
        }
        if (lane == 0) *reinterpret_cast<float4 *>(out + TC_D * TC_D + 16 * warp + 4 * i) = hsum[i];
    }
}

}  // namespace

// partial[chunk] = (G, h) of every chunk; d must be 128
int32_t als_chunk_gram_tc(gorse_b200_ctx *c, const float *Y, const int32_t *idx, const int64_t *chunk_begin, const int32_t *chunk_len,
                          int32_t n_chunks, float *partial)
{
    const size_t sm = (size_t)TC_STAGES * 2 * TC_TILE_BYTES + 1024 /* alignment */;
    GB_CUDA(cudaFuncSetAttribute(als_chunk_gram_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
    als_chunk_gram_tc_kernel<<<n_chunks, TC_THREADS, sm, c->stream>>>(Y, idx, chunk_begin, chunk_len, partial);
    GB_LAUNCHED(c);
    return GORSE_B200_OK;
}

}  // namespace gb
