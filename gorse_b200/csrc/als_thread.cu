// als_thread.cu -- eALS row update, ONE THREAD PER ROW, for short rows (the bulk of every CF dataset: 96 % of the users
// of BASELINE configs[2] have <= 32 feedback entries).  Reference loop: model/cf/model.go:659-687 (users) / :707-735 (items).
//
// Why this shape (round 2; the lane-group kernel it replaces ran at sm__warps_active 12 %, 0.054 of the HBM roofline):
//   * the coordinate sweep over f is strictly sequential per row, but rows are independent: a thread owns a row, so the
//     sweep needs NO shuffle and NO reduction -- a warp advances 32 rows per instruction instead of 2-4;
//   * x (the row being solved, D floats) lives in REGISTERS, every x[k] a named register, and the S-term
//     b_f = w * sum_{k != f} x_k S_kf  is D FMAs whose second operand is a warp-uniform (broadcast) shared-memory read of
//     row f of S (S is symmetric).  The f loop is ROLLED (4 coordinates per iteration): the one dynamically indexed read /
//     write of x per coordinate goes through a local-memory copy, the register copy is refreshed by predicated moves;
//   * the gathered opposite-table rows Y[R_x] are needed one COLUMN at a time.  Each warp stages, for a block of BC
//     coordinates, the BC-float slice of every entry of its 32 rows into shared memory with warp-cooperative 128-bit
//     loads (BC/4 lanes per entry: whole 32..128-byte segments of a row, 1/8 .. 1/2 of the L1 wavefronts a thread-per-row
//     gather would cost) in the layout [t][c][row] with a padded stride, conflict-free both for the staging stores and for
//     the per-thread column reads.  Warps never synchronise with each other after S is loaded;
//   * two passes over the staged blocks per row batch: pred_t = x . y_t (model.go:661-663), then the sweep.
// Per row: D^2 + 5 n D FMAs, D^2/4 broadcast LDS.128, 2 n D scalar LDS; n D / 4 x 2 gathered float4.
// Differences from the reference: the S-dot and pred are FMA chains over 8 accumulators (the reference rounds every
// multiply and add); sums over the row's entries keep the reference's order.  Observed ~1e-6 relative, budget 1e-4.
#include "als.cuh"

namespace gb {

template <int BC>
struct StageGeom {
    static constexpr int LPE = BC / 4;          // lanes per entry (one float4 each)
    static constexpr int EPI = 32 / LPE;        // entries per warp instruction
    static constexpr int STR = 32 + 8 / LPE;    // floats between consecutive (t, c) planes: makes staging stores conflict-free
};

// stage coordinates [b*BC, (b+1)*BC) of entry t (t < nmax) of the warp's 32 rows
template <int D, int NMAX, int BC>
__device__ __forceinline__ void stage_block(float *ys, const float *Y, const int32_t (&ids)[NMAX], int n, int nmax, int b, int lane)
{
    using G = StageGeom<BC>;
    const int piece = lane % G::LPE, q = lane / G::LPE;
#pragma unroll
    for (int t = 0; t < NMAX; t++) {
        if (t >= nmax) break;   // warp-uniform
#pragma unroll
        for (int rg = 0; rg < 32 / G::EPI; rg++) {
            const int src = rg * G::EPI + q;
            const int32_t id = __shfl_sync(0xffffffffu, ids[t], src);
            const int nn = __shfl_sync(0xffffffffu, n, src);
            if (t < nn) {
                const float4 v = __ldg(reinterpret_cast<const float4 *>(Y + (int64_t)id * D + b * BC) + piece);
                float *dst = ys + (t * BC + piece * 4) * G::STR + src;
                dst[0] = v.x; dst[G::STR] = v.y; dst[2 * G::STR] = v.z; dst[3 * G::STR] = v.w;
            }
        }
    }
}

// BCU coordinates are unrolled inside the (rolled) sweep loop.  The first version unrolled all D coordinates (600 KB of
// straight-line code at D = 128, five minutes of ptxas) and was no faster.
#define GB_ALS_BCU 4

template <int D, int NMAX, int BC, int WARPS>
__global__ void __launch_bounds__(32 * WARPS, 1)
als_thread_kernel(float *X, const float *Y, const int64_t *off, const int32_t *idx, const float *S, float reg, float w,
                  const int32_t *row_ids, int32_t n_rows)
{
    using G = StageGeom<BC>;
    constexpr int YS = NMAX * BC * G::STR;   // staging floats per warp
    constexpr int BCU = GB_ALS_BCU;
    static_assert(BC % BCU == 0 && D % BC == 0, "block sizes");
    extern __shared__ __align__(16) float smem[];
    float *Ss = smem;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float *ys = smem + D * D + warp * YS;
    for (int e = threadIdx.x; e < D * D / 4; e += 32 * WARPS)
        reinterpret_cast<float4 *>(Ss)[e] = __ldg(reinterpret_cast<const float4 *>(S) + e);
    __syncthreads();
    const float omw = 1.0f - w;
    for (int32_t base = (blockIdx.x * WARPS + warp) * 32; base < n_rows; base += gridDim.x * WARPS * 32) {
        const int32_t slot = base + lane;
        const bool act = slot < n_rows;
        int32_t r = 0;
        int n = 0;
        int64_t o = 0;
        if (act) { r = row_ids[slot]; o = off[r]; n = (int)(off[r + 1] - o); }
        int32_t ids[NMAX];
#pragma unroll
        for (int t = 0; t < NMAX; t++) ids[t] = t < n ? __ldg(idx + o + t) : 0;
        // x twice: in registers (every x[k] a named register: the S-dot below) and in local memory (per-lane interleaved by
        // the hardware, i.e. coalesced) for the one dynamically indexed read and write per coordinate
        float x[D], xl[D];
#pragma unroll
        for (int k4 = 0; k4 < D / 4; k4++) {
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (act) v = *(reinterpret_cast<const float4 *>(X + (int64_t)r * D) + k4);
            x[4 * k4] = v.x; x[4 * k4 + 1] = v.y; x[4 * k4 + 2] = v.z; x[4 * k4 + 3] = v.w;
            xl[4 * k4] = v.x; xl[4 * k4 + 1] = v.y; xl[4 * k4 + 2] = v.z; xl[4 * k4 + 3] = v.w;
        }
        const int nmax = __reduce_max_sync(0xffffffffu, n);
        // ---- pass 1: pred_t = x . y_t (model.go:661-663) ----
        float pred[NMAX];
#pragma unroll
        for (int t = 0; t < NMAX; t++) pred[t] = 0.f;
#pragma unroll 1
        for (int b = 0; b < D / BC; b++) {
            __syncwarp();
            stage_block<D, NMAX, BC>(ys, Y, ids, n, nmax, b, lane);
            __syncwarp();
#pragma unroll 4
            for (int c = 0; c < BC; c++) {
                const float xf = xl[b * BC + c];
                const float *yc = ys + c * G::STR + lane;
#pragma unroll
                for (int t = 0; t < NMAX; t++) {
                    if (t >= nmax) break;
                    if (t < n) pred[t] = fmaf(xf, yc[t * BC * G::STR], pred[t]);
                }
            }
        }
        // ---- pass 2: the coordinate sweep (model.go:664-686) ----
#pragma unroll 1
        for (int b = 0; b < D / BC; b++) {
            __syncwarp();
            stage_block<D, NMAX, BC>(ys, Y, ids, n, nmax, b, lane);
            __syncwarp();
#pragma unroll 1
            for (int cb = 0; cb < BC / BCU; cb++) {
                const int fb = (b * BC) / BCU + cb;          // coordinates [fb*BCU, (fb+1)*BCU)
#pragma unroll
                for (int j = 0; j < BCU; j++) {
                    const int f = fb * BCU + j;
                    const float xf = xl[f];
                    const float *yc = ys + (cb * BCU + j) * G::STR + lane;
                    float a = 0.f, cc = 0.f, yv[NMAX];
#pragma unroll
                    for (int t = 0; t < NMAX; t++) {
                        yv[t] = 0.f;
                        if (t >= nmax) break;
                        const float y = t < n ? yc[t * BC * G::STR] : 0.f;
                        yv[t] = y;
                        const float res = pred[t] - xf * y;                 // :666-668
                        pred[t] = res;
                        a = a + (1.0f - omw * res) * y;                      // :672
                        cc = cc + (omw * y) * y;                             // :673
                    }
                    // :675-679   b = w * sum_{k != f} x_k S_kf.  S is symmetric: row f (contiguous, warp-uniform address) instead
                    // of column f; the k = f term is taken out afterwards (x_f S_ff is exactly what the dot added)
                    float acc[8];
#pragma unroll
                    for (int i = 0; i < 8; i++) acc[i] = 0.f;
                    const float4 *srow = reinterpret_cast<const float4 *>(Ss + f * D);
#pragma unroll
                    for (int k4 = 0; k4 < D / 4; k4++) {
                        const float4 s4 = srow[k4];
                        acc[(4 * k4) & 7] = fmaf(x[4 * k4], s4.x, acc[(4 * k4) & 7]);
                        acc[(4 * k4 + 1) & 7] = fmaf(x[4 * k4 + 1], s4.y, acc[(4 * k4 + 1) & 7]);
                        acc[(4 * k4 + 2) & 7] = fmaf(x[4 * k4 + 2], s4.z, acc[(4 * k4 + 2) & 7]);
                        acc[(4 * k4 + 3) & 7] = fmaf(x[4 * k4 + 3], s4.w, acc[(4 * k4 + 3) & 7]);
                    }
                    const float sff = Ss[f * D + f];
                    const float dot = ((acc[0] + acc[1]) + (acc[2] + acc[3])) + ((acc[4] + acc[5]) + (acc[6] + acc[7]));
                    const float bsum = fmaf(-xf, sff, dot);
                    const float xn = __fdiv_rn(a - w * bsum, (cc + w * sff) + reg);   // :680
                    xl[f] = xn;
                    // the register copy: one predicated move per block of BCU coordinates (fb is warp-uniform)
#pragma unroll
                    for (int B = 0; B < D / BCU; B++)
                        if (fb == B) x[B * BCU + j] = xn;
#pragma unroll
                    for (int t = 0; t < NMAX; t++) {
                        if (t >= nmax) break;
                        pred[t] = pred[t] + xn * yv[t];                      // :682-684
                    }
                }
            }
        }
        if (act) {
#pragma unroll
            for (int k4 = 0; k4 < D / 4; k4++)
                *(reinterpret_cast<float4 *>(X + (int64_t)r * D) + k4) = make_float4(x[4 * k4], x[4 * k4 + 1], x[4 * k4 + 2], x[4 * k4 + 3]);
        }
    }
}

template <int D, int NMAX, int BC>
static int32_t launch_thread_rows(gorse_b200_ctx *c, float *X, const float *Y, const int64_t *off, const int32_t *idx, const float *S,
                                  float reg, float w, const int32_t *rows, int32_t n_rows)
{
    using G = StageGeom<BC>;
    constexpr int WARPS = 8;
    constexpr size_t sm = sizeof(float) * ((size_t)D * D + (size_t)WARPS * NMAX * BC * G::STR);
    static_assert(sm <= 227 * 1024, "shared memory budget");
    auto *k = als_thread_kernel<D, NMAX, BC, WARPS>;
    GB_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
    const int grid = (int)std::max<int64_t>(1, std::min<int64_t>(((int64_t)n_rows + 32 * WARPS - 1) / (32 * WARPS), c->sm_count));
    k<<<grid, 32 * WARPS, sm, c->stream>>>(X, Y, off, idx, S, reg, w, rows, n_rows);
    GB_LAUNCHED(c);
    return GORSE_B200_OK;
}

// rows with at most 4 entries, d in {32, 64, 96, 128}.  Only the shortest class runs here: NMAX = 8 / 16 (staging blocks of
// 16 / 8 coordinates) lost to the lane-group kernels with blocked staging, 1.16 vs 0.80 and 1.99 vs 1.27 ms per half-sweep at C3.
int32_t als_thread_rows(gorse_b200_cf *cf, float *X, const float *Y, const int64_t *off, const int32_t *idx, float reg, float w,
                        const int32_t *rows, int32_t n_rows)
{
    gorse_b200_ctx *c = cf->ctx;
    const float *S = cf->gram.p;
    switch (cf->d) {
        case 32: return launch_thread_rows<32, 4, 32>(c, X, Y, off, idx, S, reg, w, rows, n_rows);
        case 64: return launch_thread_rows<64, 4, 32>(c, X, Y, off, idx, S, reg, w, rows, n_rows);
        case 96: return launch_thread_rows<96, 4, 32>(c, X, Y, off, idx, S, reg, w, rows, n_rows);
        case 128: return launch_thread_rows<128, 4, 32>(c, X, Y, off, idx, S, reg, w, rows, n_rows);
    }
    set_error("als_thread_rows: unsupported d = %d", cf->d);
    return GORSE_B200_ERR_UNSUPPORTED;
}

}  // namespace gb
