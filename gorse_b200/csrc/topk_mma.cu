// topk_mma.cu -- stage 1 of the brute-force search on the Hopper tensor cores.
//
//   scores[q][x] = <bf16(q'), bf16(x')>   (q', x' = vectors, for Euclidean augmented so that the score is
//                                          q.x - |x|^2/2, i.e. larger = closer for both metrics)
// computed by wgmma (m64n128k16, bf16 operands, fp32 accumulators in registers), operands staged by TMA
// (cp.async.bulk.tensor, 128-byte swizzle) through an mbarrier ring.  The N x N score matrix is never written: each consumer
// warpgroup keeps only the columns whose score clears a per-row threshold, appending (column, score) to a small per-row
// candidate list.  The window kernel (topk.cu) certifies each row and re-ranks its window exactly in the reference's fp32 order.
//
// Threshold without a second pass: the vectors are stored in a random column permutation, so the first m columns are a
// uniform sample.  For those the epilogue tracks each row's 16 best scores; theta = 16th best - 2*eps is then fixed,
// the sweep continues over all columns (the first m are revisited at the end) and pushes score >= theta.
//   * soundness: every true top-k element has score >= (k-th best approximate score) - 2*eps, because |score - reference|
//     <= eps for every column.  eps is an upper bound, not an estimate (build_queries_kernel derives it): |bf16(q)| max|bf16(x)
//     - x| + |bf16(q) - q| max|x| for the bf16 rounding of both operands, plus the fp32 accumulation here and in the
//     reference and, for Euclidean, the |x|^2/2 and distance roundings.  The window kernel verifies that at least k
//     candidates clear theta + 2*eps, which makes the candidate set a superset of the true top-k; rows that fail the check
//     (or overflow their list) go to the exact kernel.  With m = 4N/k and the 16th best, a row fails with probability ~1e-6.
//
// Roofline class: tensor pipe.  F = 2 * nq * N * Kp flop per sweep.
#include <cuda.h>

#include <algorithm>
#include <cmath>
#include <random>

#include "cf.cuh"
#include "topk.cuh"
#include "wgmma.cuh"

namespace gb {
namespace mma {

struct Params {
    int64_t n;            // real vectors
    int32_t n_tiles;      // ceil(n / 128)
    int32_t m_tiles;      // sample tiles (the sweep revisits them at the end)
    int32_t kb;           // k-blocks (Kp / 64)
    int64_t nq;           // real query rows of this launch
    int32_t n_groups;     // ceil(nq / GROUP_ROWS)
    const float *eps;     // [nq] error margin per query row
    int32_t *cand_col;    // [nq][CAP] permuted column index
    float *cand_val;      // [nq][CAP]
    int32_t *cand_cnt;    // [nq][PARTS] pushes per part (may exceed PART_CAP)
    float *theta;         // [nq][PARTS] threshold used by each part
    float *dbg;           // optional dense [nq][n_tiles*128] score dump (tests)
};

// One CTA: a producer warp streams the vector tiles through a STAGES-deep ring (and the group's query tiles once per group);
// each consumer warpgroup multiplies its 64 query rows with every tile (8 or fewer wgmma, K = 16 each, into one 64 x 128
// accumulator), waits, hands the ring slot back and examines the scores in registers.  The two consumers meet on the same
// slots, so the tensor core runs one warpgroup's MMAs while the other examines its scores.
// WIDE (Kp > BK * MAX_KB): the group's query rows no longer fit in shared memory beside the ring, so a ring slot holds ONE
// k-block of both operands (the two consumers' query k-blocks and the tile's vector k-block, WIDE_STAGE_BYTES) and a tile
// takes kb slots.  A consumer accumulates the tile's kb k-blocks, one wgmma group each, keeping one group in flight: the
// slot of k-block j - 1 goes back to the producer once group j is issued.  The epilogue is the same code for both.
// Accumulator fragment (wgmma.cuh): a thread holds 2 rows x 32 columns of a tile, and the 4 threads of a quad share their
// rows; a (row, quad lane) pair is a PART with its own sample, candidate list and push count.  The 4 parts of a row merge
// their 16 best into ONE threshold by shuffles.
template <int STAGES, bool DBG, bool WIDE = false>
__global__ void __launch_bounds__(THREADS, 1)
topk_mma_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, Params P)
{
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint8_t *smem_a = smem;                                                  // [CONSUMERS][kb] query tiles (WIDE: the ring)
    uint8_t *smem_b = smem_a + (size_t)CONSUMERS * P.kb * A_TILE_BYTES;      // [STAGES][kb] vector tiles (WIDE: unused)
    uint64_t *bars = reinterpret_cast<uint64_t *>(WIDE ? smem + (size_t)STAGES * WIDE_STAGE_BYTES
                                                       : smem_b + (size_t)STAGES * P.kb * B_TILE_BYTES);
    uint64_t *full = bars, *empty = bars + STAGES, *a_full = bars + 2 * STAGES, *a_empty = a_full + 1;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        // a slot / the query tiles are free again once every consumer WARP has waited for its MMAs
        for (int s = 0; s < STAGES; s++) { mbar_init(&full[s], 1); mbar_init(&empty[s], CONSUMERS * 4); }
        mbar_init(a_full, 1);
        mbar_init(a_empty, CONSUMERS * 4);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const int total_tiles = P.n_tiles + P.m_tiles;

    if (WIDE && warp == 0) {
        // ===== TMA producer of the k-block ring: slot `slot` of pass `phase`
        uint32_t slot = 0, phase = 0;
        for (int g = blockIdx.x; g < P.n_groups; g += gridDim.x)
            for (int t = 0; t < total_tiles; t++) {
                const int bt = t < P.n_tiles ? t : t - P.n_tiles;
                for (int kb = 0; kb < P.kb; kb++) {
                    mbar_wait_backoff(&empty[slot], phase ^ 1);
                    if (elect_one()) {
                        uint8_t *st = smem + (size_t)slot * WIDE_STAGE_BYTES;
                        mbar_expect_tx(&full[slot], WIDE_STAGE_BYTES);
                        for (int m = 0; m < CONSUMERS; m++)
                            tma_load_2d(st + m * A_TILE_BYTES, &map_a, kb * BK, (g * CONSUMERS + m) * BM, &full[slot]);
                        tma_load_2d(st + CONSUMERS * A_TILE_BYTES, &map_b, kb * BK, bt * BN, &full[slot]);
                    }
                    __syncwarp();
                    if (++slot == STAGES) { slot = 0; phase ^= 1; }
                }
            }
    } else if (warp == 0) {
        // ===== TMA producer: the warp waits together, one elected lane issues
        uint32_t it = 0, ag = 0;
        for (int g = blockIdx.x; g < P.n_groups; g += gridDim.x, ag++) {
            mbar_wait_backoff(a_empty, (ag & 1) ^ 1);  // MMAs of the previous group no longer read the query tiles
            if (elect_one()) {
                mbar_expect_tx(a_full, (uint32_t)CONSUMERS * P.kb * A_TILE_BYTES);
                for (int m = 0; m < CONSUMERS; m++)
                    for (int kb = 0; kb < P.kb; kb++)
                        tma_load_2d(smem_a + ((size_t)m * P.kb + kb) * A_TILE_BYTES, &map_a, kb * BK, (g * CONSUMERS + m) * BM, a_full);
            }
            __syncwarp();
            for (int t = 0; t < total_tiles; t++, it++) {
                const int s = it % STAGES;
                mbar_wait_backoff(&empty[s], ((it / STAGES) & 1) ^ 1);
                if (elect_one()) {
                    mbar_expect_tx(&full[s], (uint32_t)P.kb * B_TILE_BYTES);
                    const int bt = t < P.n_tiles ? t : t - P.n_tiles;
                    for (int kb = 0; kb < P.kb; kb++)
                        tma_load_2d(smem_b + ((size_t)s * P.kb + kb) * B_TILE_BYTES, &map_b, kb * BK, bt * BN, &full[s]);
                }
                __syncwarp();
            }
        }
    } else if (warp >= 4) {
        // ===== consumer warpgroup wg: query rows [(g * CONSUMERS + wg) * 64, +64)
        const int wg = (warp >> 2) - 1, quad = lane & 3;
        const uint32_t a_base = s32(smem_a) + (uint32_t)wg * (uint32_t)P.kb * A_TILE_BYTES, b_base = s32(smem_b);
        float acc[64];
        uint32_t slot = 0, phase = 0;   // WIDE: the k-block ring's position, as the producer's
        // the MMAs of tile `it` into acc; every ring slot it read goes back to the producer
        auto mma_tile = [&](uint32_t it) {
            if constexpr (WIDE) {
                uint32_t prev = 0;
                for (int kb = 0; kb < P.kb; kb++) {
                    mbar_wait(&full[slot], phase);
                    const uint32_t a_k = s32(smem) + slot * WIDE_STAGE_BYTES + (uint32_t)wg * A_TILE_BYTES;
                    const uint32_t b_k = s32(smem) + slot * WIDE_STAGE_BYTES + CONSUMERS * A_TILE_BYTES;
                    wgmma_fence();
#pragma unroll
                    for (int k = 0; k < BK / 16; k++)
                        wgmma_m64n128k16_bf16(acc, wgmma_desc(a_k + (uint32_t)k * 32u), wgmma_desc(b_k + (uint32_t)k * 32u), (kb | k) != 0);
                    wgmma_commit();
                    if (kb > 0) {   // k-block kb - 1's group is done: its slot is free
                        wgmma_wait<1>();
                        __syncwarp();
                        if (lane == 0) mbar_arrive(&empty[prev]);
                    }
                    prev = slot;
                    if (++slot == STAGES) { slot = 0; phase ^= 1; }
                }
                wgmma_wait<0>();
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty[prev]);
                return;
            }
            const uint32_t s = it % STAGES;
            mbar_wait(&full[s], (it / STAGES) & 1);
            const uint32_t b_slot = b_base + s * (uint32_t)P.kb * B_TILE_BYTES;
            wgmma_fence();
            for (int kb = 0; kb < P.kb; kb++) {
#pragma unroll
                for (int k = 0; k < BK / 16; k++) {   // 16 bf16 = 32 bytes along the 128-byte row
                    const uint32_t off = (uint32_t)k * 32u;
                    wgmma_m64n128k16_bf16(acc, wgmma_desc(a_base + (uint32_t)kb * A_TILE_BYTES + off),
                                          wgmma_desc(b_slot + (uint32_t)kb * B_TILE_BYTES + off), (kb | k) != 0);
                }
            }
            wgmma_commit();
            wgmma_wait<0>();
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[s]);
        };
        uint32_t it = 0, ag = 0;
        for (int g = blockIdx.x; g < P.n_groups; g += gridDim.x, ag++) {
            int64_t row[2];
            bool row_ok[2];
            row[0] = (int64_t)(g * CONSUMERS + wg) * BM + (warp & 3) * 16 + (lane >> 2);
            row[1] = row[0] + 8;
            row_ok[0] = row[0] < P.nq;
            row_ok[1] = row[1] < P.nq;
            [[maybe_unused]] auto dump = [&](int64_t col0) {
                if (P.dbg) {
                    const int64_t ld = (int64_t)P.n_tiles * BN;
#pragma unroll
                    for (int h = 0; h < 2; h++)
                        if (row_ok[h]) {
#pragma unroll
                            for (int j = 0; j < BN / 8; j++) {
                                P.dbg[row[h] * ld + col0 + 8 * j] = acc[4 * j + 2 * h];
                                P.dbg[row[h] * ld + col0 + 8 * j + 1] = acc[4 * j + 2 * h + 1];
                            }
                        }
                }
            };
            if constexpr (!WIDE) mbar_wait(a_full, ag & 1);
            float theta[2];
            {
                // ---- the sample: each part's R_TOP best scores of the first m_tiles tiles
                float top[2][R_TOP];
#pragma unroll
                for (int h = 0; h < 2; h++)
#pragma unroll
                    for (int r = 0; r < R_TOP; r++) top[h][r] = -INFINITY;
                auto insert = [&](int h, float cur) {   // into the sorted 16 best
#pragma unroll
                    for (int r = 0; r < R_TOP; r++) {
                        const float hi = fmaxf(top[h][r], cur);
                        cur = fminf(top[h][r], cur);
                        top[h][r] = hi;
                    }
                };
                for (int t = 0; t < P.m_tiles; t++, it++) {
                    mma_tile(it);
                    const int64_t col0 = (int64_t)t * BN + 2 * quad;
                    if constexpr (DBG) dump(col0);
#pragma unroll
                    for (int j = 0; j < BN / 8; j++)
#pragma unroll
                        for (int e = 0; e < 2; e++)
#pragma unroll
                            for (int h = 0; h < 2; h++) {
                                const float x = acc[4 * j + 2 * h + e];
                                if (x > top[h][R_TOP - 1] && col0 + 8 * j + e < P.n) insert(h, x);   // rare after the first columns
                            }
                }
                // ---- one threshold per row: merge the 16 best of the quad's 4 parts (butterfly over lane ^ 1, lane ^ 2;
                // every lane ends with the same 16 values).  Two sorted lists merge as a bitonic sequence: max(a[r], b[15-r])
                // holds the 16 best of both, and four half-cleaner steps sort it.
#pragma unroll
                for (int x = 1; x <= 2; x <<= 1)
#pragma unroll
                    for (int h = 0; h < 2; h++) {
                        float c[R_TOP];
#pragma unroll
                        for (int r = 0; r < R_TOP; r++) c[r] = fmaxf(top[h][r], __shfl_xor_sync(0xffffffffu, top[h][R_TOP - 1 - r], x));
#pragma unroll
                        for (int w = R_TOP / 2; w; w >>= 1)
#pragma unroll
                            for (int r = 0; r < R_TOP; r++)
                                if ((r & w) == 0) {
                                    const float hi = fmaxf(c[r], c[r + w]);
                                    c[r + w] = fminf(c[r], c[r + w]);
                                    c[r] = hi;
                                }
#pragma unroll
                        for (int r = 0; r < R_TOP; r++) top[h][r] = c[r];
                    }
#pragma unroll
                for (int h = 0; h < 2; h++) theta[h] = row_ok[h] ? top[h][R_TOP - 1] - 2.f * P.eps[row[h]] : INFINITY;   // padding rows never hit
            }
            // ---- the sweep: every column at or above theta goes to the part's list
            int cnt[2] = {0, 0};
            int32_t *ccol[2];
            float *cval[2];
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const int64_t base = (row_ok[h] ? row[h] : 0) * CAP + quad * PART_CAP;
                ccol[h] = P.cand_col + base;
                cval[h] = P.cand_val + base;
            }
            for (int t = P.m_tiles; t < total_tiles; t++, it++) {
                const int bt = t < P.n_tiles ? t : t - P.n_tiles;
                mma_tile(it);
                const int64_t col0 = (int64_t)bt * BN + 2 * quad;
                if constexpr (DBG) {
                    if (t < P.n_tiles) dump(col0);
                }
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    // a max tree over the part's 32 scores; only a part whose maximum clears theta (~1 % of them) walks the
                    // columns and pushes the ones that do
                    float m0 = -INFINITY, m1 = -INFINITY, m2 = -INFINITY, m3 = -INFINITY;   // 4 independent chains
#pragma unroll
                    for (int j = 0; j < BN / 8; j += 2) {
                        m0 = fmaxf(m0, acc[4 * j + 2 * h]);
                        m1 = fmaxf(m1, acc[4 * j + 2 * h + 1]);
                        m2 = fmaxf(m2, acc[4 * j + 4 + 2 * h]);
                        m3 = fmaxf(m3, acc[4 * j + 4 + 2 * h + 1]);
                    }
                    if (fmaxf(fmaxf(m0, m1), fmaxf(m2, m3)) >= theta[h]) {
#pragma unroll
                        for (int j = 0; j < BN / 8; j++)
#pragma unroll
                            for (int e = 0; e < 2; e++) {
                                const float x = acc[4 * j + 2 * h + e];
                                const int64_t col = col0 + 8 * j + e;
                                if (x >= theta[h] && col < P.n) {   // padding columns only in the last tile
                                    if (cnt[h] < PART_CAP) { ccol[h][cnt[h]] = (int32_t)col; cval[h][cnt[h]] = x; }
                                    cnt[h]++;
                                }
                            }
                    }
                }
            }
#pragma unroll
            for (int h = 0; h < 2; h++)
                if (row_ok[h]) { P.cand_cnt[PARTS * row[h] + quad] = cnt[h]; P.theta[PARTS * row[h] + quad] = theta[h]; }
            if constexpr (!WIDE) {
                __syncwarp();
                if (lane == 0) mbar_arrive(a_empty);   // this warp's MMAs of the group have all been waited for
            }
        }
    }
}

// ---- mirror construction ----------------------------------------------------------------------------
// row p of the mirror = bf16 of vector perm[p] (zero rows beyond n); Euclidean appends hi/lo of -|x|^2/2.
// max_dx: running max over the vectors of |bf16(x) - x| (the ints of non-negative floats order as the floats; NaN -> Inf).
// T = uint16_t: bf16 rows, every value exact, so the mirror holds the rows' own bits and max_dx stays 0.
template <typename T>
__global__ void build_mirror_kernel(const T *X, int64_t n, int d, const int32_t *perm, int64_t n_pad, int kp, int metric,
                                    __nv_bfloat16 *Xb, float *norm /* [n] |x| by original index */, float *max_dx)
{
    const int64_t p = blockIdx.x;
    __nv_bfloat16 *dst = Xb + p * kp;
    if (p >= n) {
        for (int k = threadIdx.x; k < kp; k += blockDim.x) dst[k] = __float2bfloat16(0.f);
        return;
    }
    const int64_t src = perm[p];
    const T *x = X + src * d;
    __shared__ float s_sum[32], s_dd[32];
    float ss = 0.f, dd = 0.f;
    for (int k = threadIdx.x; k < d; k += blockDim.x) {
        const float v = row_val(x, k);
        ss = __fmaf_rn(v, v, ss);
        if constexpr (std::is_same<T, float>::value) {
            const __nv_bfloat16 b = __float2bfloat16(v);
            const float r = __fsub_rn(__bfloat162float(b), v);   // exact: the bits bf16 drops
            dd = __fmaf_rn(r, r, dd);
            dst[k] = b;
        } else {
            dst[k] = __nv_bfloat16_raw{x[k]};
        }
    }
    for (int o = 16; o; o >>= 1) { ss += __shfl_xor_sync(0xffffffffu, ss, o); dd += __shfl_xor_sync(0xffffffffu, dd, o); }
    if ((threadIdx.x & 31) == 0) { s_sum[threadIdx.x >> 5] = ss; s_dd[threadIdx.x >> 5] = dd; }
    __syncthreads();
    if (threadIdx.x == 0) {
        float tot = 0.f, dtot = 0.f;
        for (int w = 0; w < (int)(blockDim.x >> 5); w++) { tot += s_sum[w]; dtot += s_dd[w]; }
        norm[src] = sqrtf(tot);
        if constexpr (std::is_same<T, float>::value) {
            const float dx = sqrtf(dtot);
            atomicMax(reinterpret_cast<int *>(max_dx), __float_as_int(dx == dx ? dx : INFINITY));
        }
        int k = d;
        if (metric == GORSE_B200_METRIC_EUCLIDEAN) {
            const float a = -0.5f * tot;
            const __nv_bfloat16 hi = __float2bfloat16(a);
            const __nv_bfloat16 lo = __float2bfloat16(a - __bfloat162float(hi));
            dst[k++] = hi;
            dst[k++] = lo;
        }
        for (; k < kp; k++) dst[k] = __float2bfloat16(0.f);
    }
    // (columns d.. are written by thread 0 only; columns < d by the loop above)
}

// query mirror rows + per-row eps; queries come from q_ptr, or from X rows (q_idx / q0 + i; T = uint16_t: bf16 rows, widened)
template <typename T>
__global__ void build_queries_kernel(const T *X, const float *q_ptr, const int64_t *q_idx, int64_t q0, int64_t nq, int64_t nq_pad,
                                     int d, int kp, int metric, float max_norm, float max_dx, __nv_bfloat16 *Qb, float *eps)
{
    const int64_t r = blockIdx.x;
    __nv_bfloat16 *dst = Qb + r * kp;
    if (r >= nq) {
        for (int k = threadIdx.x; k < kp; k += blockDim.x) dst[k] = __float2bfloat16(0.f);
        return;
    }
    constexpr bool f32 = std::is_same<T, float>::value;
    const float *q = nullptr;   // fp32 rows are read in place; bf16 rows (x) are widened value by value
    const T *x = nullptr;
    if constexpr (f32) q = q_ptr ? q_ptr + r * d : X + (q_idx ? q_idx[r] : q0 + r) * d;
    else if (q_ptr) q = q_ptr + r * d;
    else x = X + (q_idx ? q_idx[r] : q0 + r) * d;
    __shared__ float s_sum[3][32];
    float ss = 0.f, sh = 0.f, sd = 0.f;   // |q|^2, |bf16(q)|^2, |bf16(q) - q|^2
    for (int k = threadIdx.x; k < d; k += blockDim.x) {
        const float v = f32 || q ? q[k] : row_val(x, k);
        const __nv_bfloat16 b = __float2bfloat16(v);
        const float h = __bfloat162float(b), rd = __fsub_rn(h, v);
        ss = __fmaf_rn(v, v, ss);
        sh = __fmaf_rn(h, h, sh);
        sd = __fmaf_rn(rd, rd, sd);
        dst[k] = b;
    }
    for (int o = 16; o; o >>= 1) {
        ss += __shfl_xor_sync(0xffffffffu, ss, o);
        sh += __shfl_xor_sync(0xffffffffu, sh, o);
        sd += __shfl_xor_sync(0xffffffffu, sd, o);
    }
    if ((threadIdx.x & 31) == 0) { s_sum[0][threadIdx.x >> 5] = ss; s_sum[1][threadIdx.x >> 5] = sh; s_sum[2][threadIdx.x >> 5] = sd; }
    __syncthreads();
    if (threadIdx.x == 0) {
        float tot = 0.f, toth = 0.f, totd = 0.f;
        for (int w = 0; w < (int)(blockDim.x >> 5); w++) { tot += s_sum[0][w]; toth += s_sum[1][w]; totd += s_sum[2][w]; }
        const float qh = sqrtf(toth), dq = sqrtf(totd);
        int k = d;
        if (metric == GORSE_B200_METRIC_EUCLIDEAN) { dst[k++] = __float2bfloat16(1.f); dst[k++] = __float2bfloat16(1.f); }
        for (; k < kp; k++) dst[k] = __float2bfloat16(0.f);
        // |stage-1 score - reference score| <= eps, with q^ = bf16(q), x^ = bf16(x), M = max|x|, Dx = max|x^ - x|, u = 2^-24:
        //   bf16 rounding      q^.x^ - q.x = q^.(x^ - x) + (q^ - q).x, so by Cauchy-Schwarz |.| <= |q^| Dx + |q^ - q| M.
        //                      (Each operand moves by up to 2^-8 relative, so no single-operand bound like 2^-8 |q| M holds.)
        //   fp32 accumulation  the tensor core's sum of the Kp exact products, <= 6 Kp u sum|q^_i x^_i| for aligned, truncated
        //                      partial sums, plus the reference's own fp32 dot, <= 1.02 d u |q| |x|; both <= 8 Kp u |q^| (M + Dx).
        //   Euclidean          the score is q.x - |x|^2/2 with the last two columns (1, 1) x (hi, lo) of -|x|^2/2: the fp32 norm
        //                      (d u M^2 / 2), the hi/lo split (2^-19 M^2 = 32 u M^2), the tensor core's accumulation of hi and lo
        //                      (4.02 Kp u M^2) and the rounding of the reference's distance ((d + 5) u (|q|^2 + M^2), as a score)
        //                      sum to less than (6 Kp + 64) u (|q|^2 + M^2) for d <= Kp.
        //   fp32 evaluation    the norms here and in the mirror carry < (Kp + 2) u relative error each: a 1.001 pad covers them.
        // NaN/Inf inputs make eps NaN or Inf (Inf norms, Inf Dx) -> the certification compares fail -> exact fallback.
        float e = qh * max_dx + dq * max_norm + (float)kp * 0x1p-21f * qh * (max_norm + max_dx);
        if (metric == GORSE_B200_METRIC_EUCLIDEAN) e += (6.f * (float)kp + 64.f) * 0x1p-24f * (tot + max_norm * max_norm);
        eps[r] = 1.001f * e;
    }
}

__global__ void max_kernel(const float *v, int64_t n, float *out)
{
    float m = 0.f;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) m = fmaxf(m, v[i] == v[i] ? v[i] : INFINITY);
    for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) atomicMax(reinterpret_cast<int *>(out), __float_as_int(m));  // non-negative floats order as ints
}

}  // namespace mma

// ---- host side --------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                  const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn()
{
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult qr;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qr) == cudaSuccess && qr == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)p;
    }
    return fn;
}

static int32_t make_map(CUtensorMap *map, const void *base, int64_t rows, int kp, int box_rows)
{
    EncodeTiledFn fn = encode_fn();
    if (!fn) { set_error("cuTensorMapEncodeTiled is not available from the driver"); return GORSE_B200_ERR_CUDA; }
    cuuint64_t dims[2] = {(cuuint64_t)kp, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)kp * 2};
    cuuint32_t box[2] = {(cuuint32_t)mma::BK, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void *>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed with %d", (int)r); return GORSE_B200_ERR_CUDA; }
    return GORSE_B200_OK;
}

static int kp_of(const gorse_b200_index *ix)
{
    int d = ix->d + (ix->metric == GORSE_B200_METRIC_EUCLIDEAN ? 2 : 0);
    return (d + mma::BK - 1) / mma::BK * mma::BK;
}

bool mma_path_eligible(const gorse_b200_index *ix, int64_t nq)
{
    if (const char *e = getenv("GORSE_B200_TOPK_EXACT")) if (*e == '1') return false;
    // the sample needs >= 32 tiles to make theta tight; small problems are faster on the exact scan anyway.  Kp <= 192: the
    // kernel with the queries resident; up to d = 4096 the wide kernel; wider rows take the exact scan.
    if (ix->metric != GORSE_B200_METRIC_EUCLIDEAN && ix->metric != GORSE_B200_METRIC_NEG_DOT) return false;   // cosine (vecdb.cu): exact scan
    return ix->d <= mma::MAX_D && ix->n >= 32768 && nq >= 64 && ix->n < (1ll << 31);
}

static int32_t ensure_mirror(gorse_b200_index *ix)
{
    if (ix->mma_ready) return GORSE_B200_OK;
    gorse_b200_ctx *c = ix->ctx;
    const int kp = kp_of(ix);
    const int64_t n_pad = (ix->n + mma::BN - 1) / mma::BN * mma::BN;
    if (const char *e = getenv("GORSE_B200_TOPK_MAX_MIRROR_BYTES"))   // tests of the exact fallback: a mirror that does not fit
        if (2.0 * (double)n_pad * kp > atof(e)) { set_error("top-k mirror: %lld bytes over the limit", (long long)(2 * n_pad * kp)); return GORSE_B200_ERR_OOM; }
    GB_TRY(ix->Xb.alloc((size_t)n_pad * kp));
    GB_TRY(ix->norm.alloc((size_t)ix->n + 2));
    GB_TRY(ix->perm.alloc((size_t)ix->n));
    std::vector<int32_t> perm((size_t)ix->n);
    for (int64_t i = 0; i < ix->n; i++) perm[i] = (int32_t)i;
    std::mt19937_64 rng(0x9E3779B97F4A7C15ull ^ (uint64_t)ix->n);
    std::shuffle(perm.begin(), perm.end(), rng);
    GB_CUDA(cudaMemcpyAsync(ix->perm.p, perm.data(), sizeof(int32_t) * perm.size(), cudaMemcpyHostToDevice, c->stream));
    GB_CUDA(cudaMemsetAsync(ix->norm.p + ix->n, 0, 2 * sizeof(float), c->stream));   // max |x|, max |bf16(x) - x|
    with_rows(ix->rows(), [&](auto x) {
        mma::build_mirror_kernel<<<(unsigned)n_pad, 128, 0, c->stream>>>(x, ix->n, ix->d, ix->perm.p, n_pad, kp, ix->metric, ix->Xb.p, ix->norm.p,
                                                                         ix->norm.p + ix->n + 1);
    });
    GB_LAUNCHED(c);
    mma::max_kernel<<<c->sm_count * 2, 256, 0, c->stream>>>(ix->norm.p, ix->n, ix->norm.p + ix->n);
    GB_LAUNCHED(c);
    float maxes[2];
    GB_CUDA(cudaMemcpyAsync(maxes, ix->norm.p + ix->n, sizeof(maxes), cudaMemcpyDeviceToHost, c->stream));
    GB_CUDA(cudaStreamSynchronize(c->stream));  // perm (host) dies here
    ix->max_norm = maxes[0];
    ix->max_dx = maxes[1];
    ix->mma_ready = true;
    return GORSE_B200_OK;
}

static int32_t reserve(gorse_b200_index *ix, int64_t cq)
{
    GB_TRY(ensure_mirror(ix));
    const int kp = kp_of(ix);
    if (ix->w_cq >= cq && ix->w_kp == kp) return GORSE_B200_OK;   // reuse
    // work buffers live in the index and are reused by later searches (multi-GB cudaMalloc/cudaFree per call otherwise)
    ix->w_cq = 0;
    const int64_t cq_pad = (cq + mma::GROUP_ROWS - 1) / mma::GROUP_ROWS * mma::GROUP_ROWS;
    GB_TRY(ix->w_qb.alloc((size_t)cq_pad * kp));
    GB_TRY(ix->w_eps.alloc(cq));
    GB_TRY(ix->w_cval.alloc((size_t)cq * mma::CAP));
    GB_TRY(ix->w_theta.alloc(mma::PARTS * cq));
    GB_TRY(ix->w_ccol.alloc((size_t)cq * mma::CAP));
    GB_TRY(ix->w_ccnt.alloc(mma::PARTS * cq));
    ix->w_cq = cq;
    ix->w_kp = kp;
    return GORSE_B200_OK;
}

int32_t mma_reserve(gorse_b200_index *ix, int64_t cq)
{
    const int32_t st = reserve(ix, cq);
    if (st == GORSE_B200_ERR_OOM) {   // hold none of it: the exact kernel answers without it
        ix->Xb.free(); ix->norm.free(); ix->perm.free();
        ix->w_qb.free(); ix->w_eps.free(); ix->w_cval.free(); ix->w_theta.free(); ix->w_ccol.free(); ix->w_ccnt.free();
        ix->mma_ready = false;
        ix->w_cq = 0;
        cudaGetLastError();   // the failed cudaMalloc's error is not the caller's
    }
    return st;
}

// sample size: the R_TOP-th best of m random columns leaves on average R_TOP * N / m columns above it (Gamma(R_TOP) spread)
int mma_sample_tiles(const gorse_b200_index *ix, double cands)
{
    const int n_tiles = (int)((ix->n + mma::BN - 1) / mma::BN);
    const int m_tiles = (int)((double)mma::R_TOP * (double)ix->n / cands / mma::BN);
    return std::max(1, std::min(m_tiles, n_tiles));
}

int32_t mma_sweep(gorse_b200_index *ix, RowView q_base, const float *d_q, const int64_t *d_qidx, int64_t q0, int64_t nq, int m_tiles,
                  cudaEvent_t ev0, cudaEvent_t ev1)
{
    gorse_b200_ctx *c = ix->ctx;
    const int kp = kp_of(ix), kb = kp / mma::BK;
    const int64_t n_pad = (ix->n + mma::BN - 1) / mma::BN * mma::BN;
    // stages from the shared-memory budget (227 KB per block), at most 4: the epilogue's global traffic keeps some L1.
    // Kp > 192: the wide kernel's k-block ring (WIDE_STAGES slots of WIDE_STAGE_BYTES).
    const bool wide = kb > mma::MAX_KB;
    const size_t a_bytes = (size_t)mma::CONSUMERS * kb * mma::A_TILE_BYTES, b_stage = (size_t)kb * mma::B_TILE_BYTES;
    const int stages = wide ? mma::WIDE_STAGES : (int)std::min<size_t>(4, (227 * 1024 - 1280 - a_bytes) / b_stage);
    if (kb > mma::WIDE_MAX_KB || stages < 2) { set_error("mma_sweep: Kp = %d does not fit", kp); return GORSE_B200_ERR_UNSUPPORTED; }
    const size_t smem = (wide ? (size_t)mma::WIDE_STAGES * mma::WIDE_STAGE_BYTES : a_bytes + (size_t)stages * b_stage) + 1024 /*align*/ +
                        256 /*barriers*/;
    const bool dbg = ix->dbg_scores != nullptr;   // the dense score dump of the test hook is compiled out of the production kernel
    auto pick = [&](auto s4, auto s3, auto s2) { return stages >= 4 ? s4 : stages == 3 ? s3 : s2; };
    auto kern = wide ? (dbg ? mma::topk_mma_kernel<mma::WIDE_STAGES, true, true> : mma::topk_mma_kernel<mma::WIDE_STAGES, false, true>)
                : dbg ? pick(mma::topk_mma_kernel<4, true>, mma::topk_mma_kernel<3, true>, mma::topk_mma_kernel<2, true>)
                      : pick(mma::topk_mma_kernel<4, false>, mma::topk_mma_kernel<3, false>, mma::topk_mma_kernel<2, false>);
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { set_error("mma_sweep smem attr: %s", cudaGetErrorString(e)); return GORSE_B200_ERR_CUDA; }
    CUtensorMap map_a, map_b;
    GB_TRY(make_map(&map_b, ix->Xb.p, n_pad, kp, mma::BN));
    const int64_t nq_pad = (nq + mma::GROUP_ROWS - 1) / mma::GROUP_ROWS * mma::GROUP_ROWS;
    with_rows(q_base, [&](auto x) {
        mma::build_queries_kernel<<<(unsigned)nq_pad, 128, 0, c->stream>>>(x, d_q, d_qidx, q0, nq, nq_pad, ix->d, kp, ix->metric, ix->max_norm,
                                                                          ix->max_dx, ix->w_qb.p, ix->w_eps.p);
    });
    c->launches++;
    GB_TRY(make_map(&map_a, ix->w_qb.p, nq_pad, kp, mma::BM));
    mma::Params P;
    P.n = ix->n; P.n_tiles = (int)(n_pad / mma::BN); P.m_tiles = m_tiles; P.kb = kb; P.nq = nq; P.n_groups = (int)(nq_pad / mma::GROUP_ROWS);
    P.eps = ix->w_eps.p; P.cand_col = ix->w_ccol.p; P.cand_val = ix->w_cval.p; P.cand_cnt = ix->w_ccnt.p; P.theta = ix->w_theta.p; P.dbg = ix->dbg_scores;
    const int grid = std::min(P.n_groups, c->sm_count);
    if (ev0) cudaEventRecord(ev0, c->stream);
    kern<<<grid, mma::THREADS, smem, c->stream>>>(map_a, map_b, P);
    if (ev1) cudaEventRecord(ev1, c->stream);
    GB_LAUNCHED(c);
    return GORSE_B200_OK;
}

}  // namespace gb
