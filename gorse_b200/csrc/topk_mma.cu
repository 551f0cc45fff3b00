// topk_mma.cu -- stage 1 of the brute-force search on the Hopper tensor cores.
//
//   scores[q][x] = <bf16(q'), bf16(x')>   (q', x' = vectors, for Euclidean augmented so that the score is
//                                          q.x - |x|^2/2, i.e. larger = closer for both metrics)
// computed by wgmma (m64n128k16, bf16 operands, fp32 accumulators in registers), operands staged by TMA
// (cp.async.bulk.tensor, 128-byte swizzle) through an mbarrier ring.  The N x N score matrix is never written: each consumer
// warpgroup keeps only the columns whose score clears a per-row threshold, appending (column, score) to a small per-row
// candidate list.  Stage 2 (topk.cu) re-ranks the candidates exactly in the reference's fp32 order.
//
// Threshold without a second pass: the vectors are stored in a random column permutation, so the first m columns are a
// uniform sample.  For those the epilogue tracks each row's 16 best scores; theta = 16th best - 2*eps is then fixed,
// the sweep continues over all columns (the first m are revisited at the end) and pushes score >= theta.
//   * soundness: every true top-k element has score >= (k-th best approximate score) - 2*eps  (|score - exact| <= eps,
//     eps from bf16 rounding: 1.02 * 2^-8 * |q| * max|x| + ...).  Stage 2 verifies that at least k candidates clear
//     theta + 2*eps, which makes the candidate set a superset of the true top-k; rows that fail the check (or overflow
//     their list) are redone by the exact scan.  With m = 4N/k and the 16th best, a row fails with probability ~1e-6.
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

constexpr int BM = 64, BN = 128, BK = 64;      // rows per consumer warpgroup (queries), tile columns (vectors), k-block (bf16)
constexpr int CONSUMERS = 2;                   // consumer warpgroups per CTA; both multiply every B tile
constexpr int GROUP_ROWS = CONSUMERS * BM;     // query rows of one CTA pass over all vectors
constexpr int MAX_KB = 3;                      // k-blocks per tile: Kp <= 192
constexpr int CAP = 2048;                      // candidate slots per query row
constexpr int PARTS = 4;                       // a row's columns are split over the 4 threads of an accumulator quad
constexpr int PART_CAP = CAP / PARTS;          // candidate slots per (row, part)
constexpr int R_TOP = 16;                      // sample order statistic that fixes the threshold
constexpr int THREADS = 128 * (1 + CONSUMERS); // warpgroup 0: warp 0 = TMA producer, warps 1-3 idle; then the consumers
constexpr uint32_t A_TILE_BYTES = BM * BK * 2; // one [64 x 64] bf16 k-block of queries = 8 KB
constexpr uint32_t B_TILE_BYTES = BN * BK * 2; // one [128 x 64] bf16 k-block of vectors = 16 KB

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
// Accumulator fragment (wgmma.cuh): a thread holds 2 rows x 32 columns of a tile, and the 4 threads of a quad share their
// rows; a (row, quad lane) pair is a PART with its own sample, candidate list and push count.  The 4 parts of a row merge
// their 16 best into ONE threshold by shuffles.
template <int STAGES, bool DBG>
__global__ void __launch_bounds__(THREADS, 1)
topk_mma_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, Params P)
{
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint8_t *smem_a = smem;                                                  // [CONSUMERS][kb] query tiles
    uint8_t *smem_b = smem_a + (size_t)CONSUMERS * P.kb * A_TILE_BYTES;      // [STAGES][kb] vector tiles
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem_b + (size_t)STAGES * P.kb * B_TILE_BYTES);
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

    if (warp == 0) {
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
        // the MMAs of one ring slot into acc, then the slot goes back to the producer
        auto mma_tile = [&](uint32_t s) {
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
            mbar_wait(a_full, ag & 1);
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
                    const uint32_t s = it % STAGES;
                    mbar_wait(&full[s], (it / STAGES) & 1);
                    mma_tile(s);
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
                const uint32_t s = it % STAGES;
                const int bt = t < P.n_tiles ? t : t - P.n_tiles;
                mbar_wait(&full[s], (it / STAGES) & 1);
                mma_tile(s);
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
            __syncwarp();
            if (lane == 0) mbar_arrive(a_empty);   // this warp's MMAs of the group have all been waited for
        }
    }
}

// ---- mirror construction ----------------------------------------------------------------------------
// row p of the mirror = bf16 of vector perm[p] (zero rows beyond n); Euclidean appends hi/lo of -|x|^2/2
__global__ void build_mirror_kernel(const float *X, int64_t n, int d, const int32_t *perm, int64_t n_pad, int kp, int metric,
                                    __nv_bfloat16 *Xb, float *norm /* [n] |x| by original index */)
{
    const int64_t p = blockIdx.x;
    __nv_bfloat16 *dst = Xb + p * kp;
    if (p >= n) {
        for (int k = threadIdx.x; k < kp; k += blockDim.x) dst[k] = __float2bfloat16(0.f);
        return;
    }
    const int64_t src = perm[p];
    const float *x = X + src * d;
    __shared__ float s_sum[32];
    float ss = 0.f;
    for (int k = threadIdx.x; k < d; k += blockDim.x) { float v = x[k]; ss = __fmaf_rn(v, v, ss); dst[k] = __float2bfloat16(v); }
    for (int o = 16; o; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    if ((threadIdx.x & 31) == 0) s_sum[threadIdx.x >> 5] = ss;
    __syncthreads();
    if (threadIdx.x == 0) {
        float tot = 0.f;
        for (int w = 0; w < (int)(blockDim.x >> 5); w++) tot += s_sum[w];
        norm[src] = sqrtf(tot);
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

// query mirror rows + per-row eps; queries come from q_ptr, or from X rows (q_idx / q0 + i)
__global__ void build_queries_kernel(const float *X, const float *q_ptr, const int64_t *q_idx, int64_t q0, int64_t nq, int64_t nq_pad,
                                     int d, int kp, int metric, float max_norm, __nv_bfloat16 *Qb, float *eps)
{
    const int64_t r = blockIdx.x;
    __nv_bfloat16 *dst = Qb + r * kp;
    if (r >= nq) {
        for (int k = threadIdx.x; k < kp; k += blockDim.x) dst[k] = __float2bfloat16(0.f);
        return;
    }
    const float *q = q_ptr ? q_ptr + r * d : X + (q_idx ? q_idx[r] : q0 + r) * d;
    __shared__ float s_sum[32];
    float ss = 0.f;
    for (int k = threadIdx.x; k < d; k += blockDim.x) { float v = q[k]; ss = __fmaf_rn(v, v, ss); dst[k] = __float2bfloat16(v); }
    for (int o = 16; o; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    if ((threadIdx.x & 31) == 0) s_sum[threadIdx.x >> 5] = ss;
    __syncthreads();
    if (threadIdx.x == 0) {
        float tot = 0.f;
        for (int w = 0; w < (int)(blockDim.x >> 5); w++) tot += s_sum[w];
        const float qn = sqrtf(tot);
        int k = d;
        if (metric == GORSE_B200_METRIC_EUCLIDEAN) { dst[k++] = __float2bfloat16(1.f); dst[k++] = __float2bfloat16(1.f); }
        for (; k < kp; k++) dst[k] = __float2bfloat16(0.f);
        // |approx - exact| <= eps: bf16 rounding of both operands (2^-8 relative on each product, Cauchy-Schwarz), fp32
        // accumulation in the tensor core and in the reference, and for Euclidean the hi/lo split of |x|^2/2 plus the
        // rounding of the reference's own distance.  NaN/Inf inputs make eps NaN -> every compare fails -> exact fallback.
        float e = 1.02f * 0.00390625f * qn * max_norm;
        if (metric == GORSE_B200_METRIC_EUCLIDEAN) e += 6.2e-5f * (tot + max_norm * max_norm);
        eps[r] = e;
    }
}

__global__ void max_kernel(const float *v, int64_t n, float *out)
{
    float m = 0.f;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) m = fmaxf(m, v[i] == v[i] ? v[i] : INFINITY);
    for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) atomicMax(reinterpret_cast<int *>(out), __float_as_int(m));  // non-negative floats order as ints
}

// ---- stage 2a: prune each row's candidates to the rigorous window and translate to original ids -------------
// One warp per row.  The k-th largest approximate score is found WITHOUT sorting: the scores are mapped to order-preserving
// 32-bit keys and the key is built bit by bit from the top (32 counting passes over <= CAP values held in shared memory).
__device__ __forceinline__ uint32_t float_key(float v)
{
    const uint32_t u = __float_as_uint(v);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_float(uint32_t k)
{
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

__global__ void __launch_bounds__(128)
prune_kernel(const int32_t *cand_col, const float *cand_val, const int32_t *cand_cnt, const float *theta, const float *eps,
             const int32_t *perm, const int64_t *q_idx, int64_t q0, bool self_skip, int64_t nq, int k, int32_t *out_ids /* [nq][CAP] */,
             int32_t *out_cnt, int32_t *fallback_flag)
{
    extern __shared__ uint8_t sm[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    uint32_t *sk = reinterpret_cast<uint32_t *>(sm) + (size_t)warp * mma::CAP;                                          // keys
    int32_t *sc = reinterpret_cast<int32_t *>(reinterpret_cast<uint32_t *>(sm) + (size_t)nw * mma::CAP) + (size_t)warp * mma::CAP;  // ids
    for (int64_t row = (int64_t)blockIdx.x * nw + warp; row < nq; row += (int64_t)gridDim.x * nw) {
        // every column with score >= max over the parts' thresholds was pushed by one of the parts
        int np[mma::PARTS], n = 0;
        float th = -INFINITY;
        bool bad = !(eps[row] == eps[row]);
#pragma unroll
        for (int p = 0; p < mma::PARTS; p++) {
            const int raw = cand_cnt[mma::PARTS * row + p];
            bad |= raw > mma::PART_CAP;
            np[p] = min(raw, mma::PART_CAP);
            n += np[p];
            th = fmaxf(th, theta[mma::PARTS * row + p]);
        }
        if (!(th == th)) bad = true;
        int32_t *oi = out_ids + row * mma::CAP;
        const int64_t self = self_skip ? (q_idx ? q_idx[row] : q0 + row) : -1;
        int have = 0;
        for (int e = lane; e < n; e += 32) {
            int p = 0, r = e;   // entry e of the concatenated part lists
#pragma unroll
            for (int q = 0; q + 1 < mma::PARTS; q++)
                if (p == q && r >= np[q]) { r -= np[q]; p++; }
            const int64_t src = row * mma::CAP + p * mma::PART_CAP + r;
            const int32_t c = perm[cand_col[src]];  // original id
            const float v = cand_val[src];
            const bool keep = c != self && v == v;   // SearchIndex never returns the query itself
            sk[e] = keep ? float_key(v) : 0u;
            sc[e] = c;
            have += keep;
        }
        for (int o = 16; o; o >>= 1) have += __shfl_xor_sync(0xffffffffu, have, o);
        __syncwarp();
        if (have < k) bad = true;
        int w = 0;
        if (!bad) {
            uint32_t t = 0;
            for (int bit = 31; bit >= 0; bit--) {
                const uint32_t candk = t | (1u << bit);
                int cnt = 0;
                for (int e = lane; e < n; e += 32) cnt += sk[e] >= candk;
                for (int o = 16; o; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
                if (cnt >= k) t = candk;
            }
            const float kth = key_float(t);            // the k-th largest approximate score
            const float two_eps = 2.f * eps[row];
            // validity: at least k candidates clear theta + 2 eps, i.e. the k-th best approximate score is known exactly
            if (!(kth >= th + two_eps)) bad = true;
            else {
                const uint32_t lim = float_key(kth - two_eps);
                for (int e0 = 0; e0 < n; e0 += 32) {
                    const int e = e0 + lane;
                    const bool in = e < n && sk[e] >= lim && sk[e] != 0u;
                    const unsigned mk = __ballot_sync(0xffffffffu, in);
                    if (in) oi[w + __popc(mk & ((1u << lane) - 1))] = sc[e];
                    w += __popc(mk);
                }
            }
        }
        if (lane == 0) {
            out_cnt[row] = bad ? 0 : w;
            if (bad) fallback_flag[row] = 1;
        }
        __syncwarp();
    }
}

__global__ void compact_flags_kernel(const int32_t *flag, int64_t nq, int32_t *list, int32_t *n_list)
{
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r < nq && flag[r]) list[atomicAdd(n_list, 1)] = (int32_t)r;
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

bool mma_path_eligible(const gorse_b200_index *ix, int64_t nq, int k)
{
    if (const char *e = getenv("GORSE_B200_TOPK_EXACT")) if (*e == '1') return false;
    const int kp = kp_of(ix);
    // the sample needs >= 32 tiles to make theta tight; small problems are faster on the exact scan anyway
    if (ix->metric != GORSE_B200_METRIC_EUCLIDEAN && ix->metric != GORSE_B200_METRIC_NEG_DOT) return false;   // cosine (vecdb.cu): exact scan
    return kp <= mma::BK * mma::MAX_KB && k >= 1 && k <= 128 && ix->n >= 32768 && nq >= 64 && ix->n < (1ll << 31);
}

static int32_t ensure_mirror(gorse_b200_index *ix)
{
    if (ix->mma_ready) return GORSE_B200_OK;
    gorse_b200_ctx *c = ix->ctx;
    const int kp = kp_of(ix);
    const int64_t n_pad = (ix->n + mma::BN - 1) / mma::BN * mma::BN;
    GB_TRY(ix->Xb.alloc((size_t)n_pad * kp));
    GB_TRY(ix->norm.alloc((size_t)ix->n + 1));
    GB_TRY(ix->perm.alloc((size_t)ix->n));
    std::vector<int32_t> perm((size_t)ix->n);
    for (int64_t i = 0; i < ix->n; i++) perm[i] = (int32_t)i;
    std::mt19937_64 rng(0x9E3779B97F4A7C15ull ^ (uint64_t)ix->n);
    std::shuffle(perm.begin(), perm.end(), rng);
    GB_CUDA(cudaMemcpyAsync(ix->perm.p, perm.data(), sizeof(int32_t) * perm.size(), cudaMemcpyHostToDevice, c->stream));
    mma::build_mirror_kernel<<<(unsigned)n_pad, 128, 0, c->stream>>>(ix->X.p, ix->n, ix->d, ix->perm.p, n_pad, kp, ix->metric, ix->Xb.p, ix->norm.p);
    GB_LAUNCHED(c);
    GB_CUDA(cudaMemsetAsync(ix->norm.p + ix->n, 0, sizeof(float), c->stream));
    mma::max_kernel<<<c->sm_count * 2, 256, 0, c->stream>>>(ix->norm.p, ix->n, ix->norm.p + ix->n);
    GB_LAUNCHED(c);
    GB_CUDA(cudaMemcpyAsync(&ix->max_norm, ix->norm.p + ix->n, sizeof(float), cudaMemcpyDeviceToHost, c->stream));
    GB_CUDA(cudaStreamSynchronize(c->stream));  // perm (host) dies here
    ix->mma_ready = true;
    return GORSE_B200_OK;
}

int32_t search_mma(gorse_b200_index *ix, const float *d_q, const int64_t *d_qidx, int64_t q0, int64_t nq, int k, int prune0,
                   int32_t *d_idx, float *d_dist, int32_t *d_count, int *d_nan, int32_t *h_idx, float *h_dist, int32_t *h_count)
{
    gorse_b200_ctx *c = ix->ctx;
    GB_TRY(ensure_mirror(ix));
    const int kp = kp_of(ix), kb = kp / mma::BK;
    const int64_t n_pad = (ix->n + mma::BN - 1) / mma::BN * mma::BN;
    const int n_tiles = (int)(n_pad / mma::BN);
    // sample size: the R_TOP-th best of m random columns leaves on average R_TOP * N / m columns above it (Gamma(R_TOP)
    // spread).  The parts of a row share ONE threshold from the whole sample, aimed at 4k columns per row: the row has
    // fewer than k candidates when >= R_TOP of its true top k fell into the sample, Poisson(k m / N = R_TOP / 4): ~1e-6 per
    // row, and a part's PART_CAP-slot list holds 4x its expected k columns (k <= 128).
    int m_tiles = (int)((double)mma::R_TOP * (double)ix->n / (4.0 * k) / mma::BN);
    m_tiles = std::max(1, std::min(m_tiles, n_tiles));
    const bool self_skip = d_q == nullptr;
    // stages from the shared-memory budget (227 KB per block), at most 4: the epilogue's global traffic keeps some L1
    const size_t a_bytes = (size_t)mma::CONSUMERS * kb * mma::A_TILE_BYTES, b_stage = (size_t)kb * mma::B_TILE_BYTES;
    int stages = (int)std::min<size_t>(4, (227 * 1024 - 1280 - a_bytes) / b_stage);
    if (stages < 2) { set_error("search_mma: Kp = %d does not fit", kp); return GORSE_B200_ERR_UNSUPPORTED; }
    const size_t smem = a_bytes + (size_t)stages * b_stage + 1024 /*align*/ + 256 /*barriers*/;

    CUtensorMap map_b;
    GB_TRY(make_map(&map_b, ix->Xb.p, n_pad, kp, mma::BN));
    // queries are processed in chunks of 1024 rows per SM so that the candidate lists stay modest while every chunk's kernel
    // tail, host sync for the fallback count and fallback launches are amortised; a finished chunk is downloaded on the copy
    // stream while the next one computes
    const int64_t chunk = (int64_t)c->sm_count * mma::GROUP_ROWS * 8;
    // work buffers live in the index and are reused by later searches (multi-GB cudaMalloc/cudaFree per call otherwise)
    DevBuf<__nv_bfloat16> &Qb = ix->w_qb;
    DevBuf<float> &eps = ix->w_eps, &cval = ix->w_cval, &theta = ix->w_theta;
    DevBuf<int32_t> &ccol = ix->w_ccol, &ccnt = ix->w_ccnt, &ids = ix->w_ids, &idcnt = ix->w_idcnt, &flag = ix->w_flag, &flist = ix->w_flist;
    int32_t st = GORSE_B200_OK;
    auto done = [&](int32_t s) {
        cudaStreamSynchronize(c->stream);
        cudaStreamSynchronize(c->copy_stream);
        return s;
    };
    const int64_t cq = std::min(nq, chunk), cq_pad = (cq + mma::GROUP_ROWS - 1) / mma::GROUP_ROWS * mma::GROUP_ROWS;
    if (ix->w_cq >= cq && ix->w_kp == kp) {
        // reuse
    } else if ((ix->w_cq = 0, false) || (st = Qb.alloc((size_t)cq_pad * kp)) || (st = eps.alloc(cq)) || (st = cval.alloc((size_t)cq * mma::CAP)) || (st = theta.alloc(mma::PARTS * cq)) ||
        (st = ccol.alloc((size_t)cq * mma::CAP)) || (st = ccnt.alloc(mma::PARTS * cq)) || (st = ids.alloc((size_t)cq * mma::CAP)) || (st = idcnt.alloc(cq)) ||
        (st = flag.alloc(cq)) || (st = flist.alloc(cq + 1)))
        return done(st);
    else { ix->w_cq = cq; ix->w_kp = kp; }
    const int64_t fl_off = ix->w_cq;  // the fallback counter sits after the list
    const bool dbg = ix->dbg_scores != nullptr;   // the dense score dump of the test hook is compiled out of the production kernel
    auto pick = [&](auto s4, auto s3, auto s2) { return stages >= 4 ? s4 : stages == 3 ? s3 : s2; };
    auto kern = dbg ? pick(mma::topk_mma_kernel<4, true>, mma::topk_mma_kernel<3, true>, mma::topk_mma_kernel<2, true>)
                    : pick(mma::topk_mma_kernel<4, false>, mma::topk_mma_kernel<3, false>, mma::topk_mma_kernel<2, false>);
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { set_error("search_mma smem attr: %s", cudaGetErrorString(e)); return done(GORSE_B200_ERR_CUDA); }
    for (int64_t off = 0; off < nq; off += cq) {
        const int64_t n_this = std::min(cq, nq - off), n_this_pad = (n_this + mma::GROUP_ROWS - 1) / mma::GROUP_ROWS * mma::GROUP_ROWS;
        const float *qp = d_q ? d_q + off * ix->d : nullptr;
        const int64_t *qi = d_qidx ? d_qidx + off : nullptr;
        mma::build_queries_kernel<<<(unsigned)n_this_pad, 128, 0, c->stream>>>(ix->X.p, qp, qi, q0 + off, n_this, n_this_pad, ix->d, kp, ix->metric,
                                                                              ix->max_norm, Qb.p, eps.p);
        c->launches++;
        CUtensorMap map_a;
        if ((st = make_map(&map_a, Qb.p, n_this_pad, kp, mma::BM))) return done(st);
        mma::Params P;
        P.n = ix->n; P.n_tiles = n_tiles; P.m_tiles = m_tiles; P.kb = kb; P.nq = n_this; P.n_groups = (int)(n_this_pad / mma::GROUP_ROWS);
        P.eps = eps.p; P.cand_col = ccol.p; P.cand_val = cval.p; P.cand_cnt = ccnt.p; P.theta = theta.p; P.dbg = ix->dbg_scores;
        const int grid = std::min(P.n_groups, c->sm_count);
        if (!ix->ev0) { cudaEventCreate(&ix->ev0); cudaEventCreate(&ix->ev1); }
        cudaEventRecord(ix->ev0, c->stream);
        kern<<<grid, mma::THREADS, smem, c->stream>>>(map_a, map_b, P);
        cudaEventRecord(ix->ev1, c->stream);
        c->launches++;
        if ((e = cudaMemsetAsync(flag.p, 0, sizeof(int32_t) * n_this, c->stream)) != cudaSuccess ||
            (e = cudaMemsetAsync(flist.p + fl_off, 0, sizeof(int32_t), c->stream)) != cudaSuccess) {
            set_error("search_mma memset: %s", cudaGetErrorString(e));
            return done(GORSE_B200_ERR_CUDA);
        }
        const int pw = 4;
        const size_t psm = (size_t)pw * mma::CAP * 8;
        if ((e = cudaFuncSetAttribute(mma::prune_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)psm)) != cudaSuccess) {
            set_error("prune smem attr: %s", cudaGetErrorString(e));
            return done(GORSE_B200_ERR_CUDA);
        }
        mma::prune_kernel<<<(unsigned)std::min<int64_t>((n_this + pw - 1) / pw, (int64_t)c->sm_count * 8), 32 * pw, psm, c->stream>>>(
            ccol.p, cval.p, ccnt.p, theta.p, eps.p, ix->perm.p, qi, q0 + off, self_skip, n_this, k, ids.p, idcnt.p, flag.p);
        c->launches++;
        // stage 2: exact re-rank of the window, reference fp32 order
        if ((st = launch_exact(ix, qp, qi, q0 + off, n_this, k, ids.p, idcnt.p, mma::CAP, nullptr, d_idx + off * k, d_dist + off * k, d_count + off,
                               prune0, d_nan)))
            return done(st);
        // rows whose candidate set could not be certified: exact scan over everything
        mma::compact_flags_kernel<<<(unsigned)((n_this + 255) / 256), 256, 0, c->stream>>>(flag.p, n_this, flist.p, flist.p + fl_off);
        c->launches++;
        int32_t n_fb = 0;
        if ((e = cudaMemcpyAsync(&n_fb, flist.p + fl_off, sizeof(int32_t), cudaMemcpyDeviceToHost, c->stream)) != cudaSuccess ||
            (e = cudaStreamSynchronize(c->stream)) != cudaSuccess) {
            set_error("search_mma: %s", cudaGetErrorString(e));
            return done(GORSE_B200_ERR_CUDA);
        }
        ix->last_fallback_rows += n_fb;
        {
            float ms = 0.f;  // the stream was synchronised just above
            if (cudaEventElapsedTime(&ms, ix->ev0, ix->ev1) == cudaSuccess) { ix->stage1_ms += ms; ix->stage1_flop += 2.0 * (double)n_this * (double)ix->n * (double)ix->d; }
        }
        if (n_fb > 0) {
            if ((st = launch_exact_split(ix, qp, qi, q0 + off, n_fb, k, flist.p, d_idx + off * k, d_dist + off * k, d_count + off, prune0, d_nan)))
                return done(st);
        }
        if (h_idx) {
            // this chunk is final: download it on the copy stream while the next chunk computes
            if ((e = cudaEventRecord(c->copy_ev, c->stream)) != cudaSuccess || (e = cudaStreamWaitEvent(c->copy_stream, c->copy_ev, 0)) != cudaSuccess ||
                (e = cudaMemcpyAsync(h_idx + off * k, d_idx + off * k, sizeof(int32_t) * n_this * k, cudaMemcpyDeviceToHost, c->copy_stream)) != cudaSuccess ||
                (e = cudaMemcpyAsync(h_dist + off * k, d_dist + off * k, sizeof(float) * n_this * k, cudaMemcpyDeviceToHost, c->copy_stream)) != cudaSuccess ||
                (e = cudaMemcpyAsync(h_count + off, d_count + off, sizeof(int32_t) * n_this, cudaMemcpyDeviceToHost, c->copy_stream)) != cudaSuccess) {
                set_error("search_mma download: %s", cudaGetErrorString(e));
                return done(GORSE_B200_ERR_CUDA);
            }
        }
    }
    if ((e = cudaGetLastError()) != cudaSuccess) { set_error("search_mma: %s", cudaGetErrorString(e)); return done(GORSE_B200_ERR_CUDA); }
    return done(GORSE_B200_OK);
}

}  // namespace gb
