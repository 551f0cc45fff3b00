// als.cu -- eALS ("CCD") epoch: model/cf/model.go:641-738.
//   S^q = sum_{i: |R_i|>0} q_i q_i^T          (:645-658)   run_gram
//   user rows, coordinate descent over f      (:659-687)   run_rows
//   S^p = sum_{u: |R_u|>0} p_u p_u^T          (:693-706)
//   item rows                                 (:707-735)
// Roofline class: HBM bandwidth (one gather of the opposite table's rows per feedback + own row + one
// Gram pass): B_epoch = 2|R|(4d+4) + 3(U+I)4d bytes.
//
// Grams.  A Gram is taken over a list of rows cut into chunks of <= GB_ALS_CHUNK: every chunk becomes one partial (G, h)
// in cf->als_partial, als_partial_stride(d) floats apart.  The chunk kernel is als_chunk_gram_tc (tensor cores,
// als_gram_tc.cu) at d = 128, als_chunk_gram_kernel at other d <= 128 and als_chunk_gram_generic_kernel at d > 128.
// S runs it over the rows with feedback and sums the partials in chunk order (gram_reduce_kernel); a long row runs it
// over its own entries (d <= 128 only).
//
// Row updates, chosen per row by d and its length n (prepare_als, kRowClasses):
//   d % 32 == 0, d <= 128:  n <= 4            als_thread_kernel (als_thread.cu), one thread per row
//                           n <= 96           als_rows_group_blocked_kernel<G, E>, a group of 8/16/32 lanes per row, g = S x
//                                             kept current in registers, the gathered rows staged G coordinates at a time
//   other d:                n (d+1) <= 12288  als_rows_kernel, one warp per row with the reference's loop structure; the
//                                             gathered rows Y[R_x] staged once in shared memory ([n][d+1], the +1 makes the
//                                             per-f column walk conflict-free), the running predictions in registers
//   longer, d <= 128:       Gram form: chunk Grams, als_partial_reduce_kernel, als_solve_kernel (one Gauss-Seidel sweep
//                           on A x = h)
//   longer, d > 128:        als_rows_kernel gathering from L2 without staging
// In all forms sums over the row's feedback are taken lane-parallel, so results differ from the reference's serial
// order by reassociation only (parity budget 1e-4 relative, observed ~1e-6).
#include <cstdlib>

#include "als.cuh"
#include "tables.cuh"

namespace gb {

#define GB_ALS_PRED_REGS 4      // rows up to 128 entries keep pred in registers
#define GB_ALS_WARPS 4          // warps per CTA in the row kernel

__device__ __forceinline__ float warp_sum(float v)
{
    v += __shfl_xor_sync(0xffffffffu, v, 16);
    v += __shfl_xor_sync(0xffffffffu, v, 8);
    v += __shfl_xor_sync(0xffffffffu, v, 4);
    v += __shfl_xor_sync(0xffffffffu, v, 2);
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    return v;
}

// acc[x][y] += a[x] * b[y] over a TxT register tile
template <int T>
struct GramTile {
    float acc[T][T];
    __device__ __forceinline__ void zero()
    {
#pragma unroll
        for (int x = 0; x < T; x++)
#pragma unroll
            for (int y = 0; y < T; y++) acc[x][y] = 0.f;
    }
    __device__ __forceinline__ void mac(const float (&a)[T], const float (&b)[T])
    {
#pragma unroll
        for (int x = 0; x < T; x++)
#pragma unroll
            for (int y = 0; y < T; y++) acc[x][y] = __fmaf_rn(a[x], b[y], acc[x][y]);
    }
    __device__ __forceinline__ float get(int x, int y) const { return acc[x][y]; }
};

// fixed-order reduction of the chunk partials: deterministic run to run
__global__ void gram_reduce_kernel(const float *partial, int n_parts, int dd, int64_t stride, float *S)
{
    int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= dd) return;
    float s = 0.f;
    for (int p = 0; p < n_parts; p++) s += partial[(int64_t)p * stride + e];
    S[e] = s;
}

// One warp per row.  X: table being updated, Y: the opposite table.
// smem per warp: xrow[d] + (staged ? ys[cap_n][d+1] : 0)
__global__ void __launch_bounds__(32 * GB_ALS_WARPS)
als_rows_kernel(float *X, const float *Y, int d, const int64_t *off, const int32_t *idx, const float *S, float reg, float w,
                const int32_t *row_ids, int32_t n_rows, int stage_floats_per_warp, float *pred_scratch)
{
    extern __shared__ float smem[];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int per_warp = d + stage_floats_per_warp;
    float *xrow = smem + (size_t)wid * per_warp;
    float *ys = xrow + d;
    const int dp = d + 1;
    const float omw = 1.0f - w;
    int32_t slot = blockIdx.x * GB_ALS_WARPS + wid;
    const int32_t n_slots = gridDim.x * GB_ALS_WARPS;
    for (; slot < n_rows; slot += n_slots) {
        const int32_t r = row_ids[slot];
        const int64_t o = off[r];
        const int n = (int)(off[r + 1] - o);
        float *xg = X + (int64_t)r * d;
        for (int k = lane; k < d; k += 32) xrow[k] = xg[k];
        const bool staged = (int64_t)n * dp <= stage_floats_per_warp;
        const bool pred_in_regs = n <= 32 * GB_ALS_PRED_REGS;
        float *pg = pred_scratch + o;
        __syncwarp();
        if (staged) {
            // coalesced row copies: lane walks the row, one row at a time
            for (int t = 0; t < n; t++) {
                const float *yr = Y + (int64_t)idx[o + t] * d;
                for (int k = lane; k < d; k += 32) ys[t * dp + k] = yr[k];
            }
            __syncwarp();
        }
        // pred[t] = internalPredict = floats.Dot(x, y_t)   (:661-663)
        float pr[GB_ALS_PRED_REGS];
#pragma unroll
        for (int q = 0; q < GB_ALS_PRED_REGS; q++) pr[q] = 0.f;
        for (int t0 = 0; t0 < n; t0 += 32) {
            int t = t0 + lane;
            float v = 0.f;
            if (t < n) {
                if (staged) {
                    // same order as dot_any on the staged copy
                    const float *yr = ys + t * dp;
                    v = dot_any(xrow, yr, d);
                } else {
                    v = dot_any(xrow, Y + (int64_t)idx[o + t] * d, d);
                }
            }
            if (pred_in_regs) {
#pragma unroll
                for (int q = 0; q < GB_ALS_PRED_REGS; q++) if (t0 == 32 * q) pr[q] = v;
            } else if (t < n) pg[t] = v;
        }
        for (int f = 0; f < d; f++) {
            const float xf = xrow[f];
            float a = 0.f, c = 0.f, b = 0.f;
            // :666-674
            for (int t0 = 0, q = 0; t0 < n; t0 += 32, q++) {
                int t = t0 + lane;
                if (t < n) {
                    float y = staged ? ys[t * dp + f] : __ldg(Y + (int64_t)idx[o + t] * d + f);
                    float p;
                    if (pred_in_regs) {
                        p = pr[0];
#pragma unroll
                        for (int qq = 1; qq < GB_ALS_PRED_REGS; qq++) if (q == qq) p = pr[qq];
                    } else p = pg[t];
                    float res = p - xf * y;
                    a = a + (1.0f - omw * res) * y;
                    c = c + (omw * y) * y;
                }
            }
            // :675-679   S is bitwise symmetric, so read row f (contiguous) instead of column f
            for (int k = lane; k < d; k += 32)
                if (k != f) b = b + (w * xrow[k]) * __ldg(S + f * d + k);
            a = warp_sum(a);
            c = warp_sum(c);
            b = warp_sum(b);
            const float xn = (a - b) / ((c + w * __ldg(S + f * d + f)) + reg);  // :680
            // :682-684
            for (int t0 = 0, q = 0; t0 < n; t0 += 32, q++) {
                int t = t0 + lane;
                if (t < n) {
                    float y = staged ? ys[t * dp + f] : __ldg(Y + (int64_t)idx[o + t] * d + f);
                    if (pred_in_regs) {
#pragma unroll
                        for (int qq = 0; qq < GB_ALS_PRED_REGS; qq++)
                            if (q == qq) { float res = pr[qq] - xf * y; pr[qq] = res + xn * y; }
                    } else {
                        float res = pg[t] - xf * y;
                        pg[t] = res + xn * y;
                    }
                }
            }
            __syncwarp();
            if (lane == 0) xrow[f] = xn;
            __syncwarp();
        }
        for (int k = lane; k < d; k += 32) xg[k] = xrow[k];
        __syncwarp();
    }
}

// ---- short rows, lane-group form (d % 32 == 0, d <= 128) ---------------------------------------------------
// A group of G lanes (8, 16 or 32) owns one row; 32/G rows share a warp.  With h_f = sum_t y_tf, c_f = (1-w) sum_t y_tf^2
// and g = S x kept CURRENT (g += delta * S[f,:] after every coordinate), the reference's step (model.go:666-680) is
//     x_f <- ( h_f - (1-w) * sum_t pred_t y_tf + x_f * (c_f + w S_ff) - w * g_f ) / (c_f + w S_ff + reg)
// (a = h_f - (1-w) z_f + x_f c_f,  b = w (g_f - S_ff x_f)): the only reduction on the strictly sequential f chain is
// z_f over the row's entries (log2 G shuffles); h, c and the reciprocal denominators are computed up front, lane
// parallel, and the S-part of b needs no reduction at all.  Lane j of the group owns the factors k = i*G + j
// (i < KPL = d/G) of x, g, h, c in registers and the entries t = j + e*G (e < E) of pred; the gathered rows sit in
// shared memory as [t][d+1] (conflict-free both along a row and down a column) next to one copy of S per CTA.
// Differences from the reference are reassociation (lane-parallel sums, incremental g) and one reciprocal-multiply
// instead of a divide: observed ~1e-6 relative, budget 1e-4.
template <int G>
__device__ __forceinline__ float group_sum(float v)
{
#pragma unroll
    for (int o = G / 2; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// ---- lane-group form with BLOCKED staging ------------------------------------------------------------------------------
// The arithmetic above with the gathered rows staged one block of G coordinates at a time: n * (G+1) floats per row in
// shared memory instead of n * (D+1).  Staging whole rows holds 33 KB (rows up to 32 entries, two rows per warp) / 49.5 KB
// (rows up to 96 entries) per warp next to the 64 KB copy of S, i.e. 3-4 warps per SM, each running a dependent shuffle
// chain per coordinate: that measured 2.3 + 3.0 ms per half-sweep for 7 % of the rows.
// Lane j of the group owns coordinate i*G + j of block i, so a block is exactly what the group works on at a time:
//   pass A  per sub-range of G entries and per block: stage G x G floats, partial_tt += x_i * y (registers, one per entry of
//           the sub-range), h_i, c_i column sums; the partials are reduced across the group once per sub-range -> pred;
//   sweep   per block: stage all n entries of the block, then the G coordinates as before.
// Every entry is staged once per pass, as before (in G*4-byte pieces instead of whole rows).
template <int G, int E, int KPL>
__global__ void __launch_bounds__(G == 16 ? 1024 : 512)   // G = 16: 64 registers, 32 warps next to ONE copy of S
als_rows_group_blocked_kernel(float *X, const float *Y, const int64_t *off, const int32_t *idx, const float *S, float reg, float w,
                              const int32_t *row_ids, int32_t n_rows)
{
    constexpr int D = G * KPL, NG = 32 / G, GP = G + 1, G4 = G / 4;
    constexpr int YS = E * G * GP + (G < 32 ? G : 0);      // floats per lane group (padded so that groups start G banks apart)
    extern __shared__ float smem[];
    float *Ss = smem;                                   // [D][D]
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
    const int grp = lane / G, j = lane % G;
    float *ys = smem + D * D + (size_t)(wid * NG + grp) * YS;
    for (int e = threadIdx.x; e < D * D; e += blockDim.x) Ss[e] = S[e];
    __syncthreads();
    const float omw = 1.0f - w;
    const int32_t stride = gridDim.x * nw * NG;
    for (int32_t base = (blockIdx.x * nw + wid) * NG; base < n_rows; base += stride) {   // warp-uniform trip count
        const int32_t slot = base + grp;
        const bool act = slot < n_rows;
        int32_t r = 0;
        int n = 0;
        int64_t o = 0;
        if (act) { r = row_ids[slot]; o = off[r]; n = (int)(off[r + 1] - o); }
        const int nmax = __reduce_max_sync(0xffffffffu, n);
        // this lane's entries t = j + e*G: their row pointers
        const float *yrow[E];
#pragma unroll
        for (int e = 0; e < E; e++) yrow[e] = (j + e * G < n) ? Y + (int64_t)__ldg(idx + o + j + e * G) * D : Y;
        float x[KPL], g[KPL], h[KPL], cw[KPL], inv[KPL], pred[E];
#pragma unroll
        for (int i = 0; i < KPL; i++) {
            x[i] = act ? X[(int64_t)r * D + i * G + j] : 0.f;
            g[i] = 0.f; h[i] = 0.f; cw[i] = 0.f;
        }
        // stage entries [t0, t0 + cnt) of block i: the group's lanes walk the cnt * G/4 float4 pieces; entry t comes from lane t % G
        auto stage = [&](int i, int e0, int e1) {
#pragma unroll
            for (int e = e0; e < e1; e++) {
                if (e * G >= nmax) break;                       // warp-uniform
#pragma unroll
                for (int c = j; c < G * G4; c += G) {
                    const int tt = c / G4, q = c - tt * G4;     // entry e*G + tt, piece q
                    const float *src = (const float *)__shfl_sync(0xffffffffu, (unsigned long long)yrow[e], tt, G);
                    if (e * G + tt < n) {
                        const float4 v = __ldg(reinterpret_cast<const float4 *>(src + i * G) + q);
                        float *dst = ys + (e * G + tt) * GP + 4 * q;
                        dst[0] = v.x; dst[1] = v.y; dst[2] = v.z; dst[3] = v.w;
                    }
                }
            }
        };
        // ---- pass A: pred_t = x . y_t (:661-663), h, c ----
#pragma unroll
        for (int e = 0; e < E; e++) {
            pred[e] = 0.f;
            if (e * G >= nmax) continue;                        // warp-uniform
            float part[G];
#pragma unroll
            for (int tt = 0; tt < G; tt++) part[tt] = 0.f;
#pragma unroll 1
            for (int i = 0; i < KPL; i++) {
                __syncwarp();
                stage(i, e, e + 1);
                __syncwarp();
                float xi = x[0], hi = 0.f, ci = 0.f;
#pragma unroll
                for (int ii = 1; ii < KPL; ii++) if (i == ii) xi = x[ii];
#pragma unroll
                for (int tt = 0; tt < G; tt++) {
                    if (e * G + tt >= nmax) break;              // warp-uniform
                    if (e * G + tt < n) {
                        const float y = ys[(e * G + tt) * GP + j];
                        part[tt] = fmaf(xi, y, part[tt]);
                        hi += y;
                        ci = fmaf(y, y, ci);
                    }
                }
#pragma unroll
                for (int ii = 0; ii < KPL; ii++) if (i == ii) { h[ii] += hi; cw[ii] += ci; }
            }
#pragma unroll
            for (int tt = 0; tt < G; tt++) {
                if (e * G + tt >= nmax) break;
                const float s = group_sum<G>(part[tt]);
                if (tt == j) pred[e] = s;
            }
        }
        // g = S x (S symmetric: row m is column m), cw = (1-w) c + w S_kk, inv = 1 / (cw + reg)
#pragma unroll
        for (int mi = 0; mi < KPL; mi++) {
#pragma unroll 1
            for (int mj = 0; mj < G; mj++) {
                const float xm = __shfl_sync(0xffffffffu, x[mi], mj, G);
                const float *srow = Ss + (mi * G + mj) * D + j;
#pragma unroll
                for (int i = 0; i < KPL; i++) g[i] = fmaf(xm, srow[i * G], g[i]);
            }
        }
#pragma unroll
        for (int i = 0; i < KPL; i++) {
            const int k = i * G + j;
            cw[i] = omw * cw[i] + w * Ss[k * D + k];
            inv[i] = 1.0f / (cw[i] + reg);
        }
        // ---- the sweep, block by block ----
#pragma unroll
        for (int fi = 0; fi < KPL; fi++) {
            __syncwarp();
            stage(fi, 0, E);
            __syncwarp();
#pragma unroll 1
            for (int jo = 0; jo < G; jo++) {
                float ye[E], red = 0.f;
#pragma unroll
                for (int e = 0; e < E; e++) {
                    const int t = j + e * G;
                    ye[e] = t < n ? ys[t * GP + jo] : 0.f;
                    red = fmaf(pred[e], ye[e], red);
                }
                red = group_sum<G>(red);
                const float num = (h[fi] - omw * red) + (x[fi] * cw[fi] - w * g[fi]);
                const float xn = num * inv[fi];
                const float dl = __shfl_sync(0xffffffffu, xn - x[fi], jo, G);
                if (j == jo) x[fi] = xn;
                const float *srow = Ss + (fi * G + jo) * D + j;
#pragma unroll
                for (int i = 0; i < KPL; i++) g[i] = fmaf(dl, srow[i * G], g[i]);
#pragma unroll
                for (int e = 0; e < E; e++) pred[e] = fmaf(dl, ye[e], pred[e]);
            }
        }
        if (act) {
#pragma unroll
            for (int i = 0; i < KPL; i++) X[(int64_t)r * D + i * G + j] = x[i];
        }
        __syncwarp();   // the next row's staging must not overtake this row's column reads
    }
}

template <int G, int E, int KPL>
static int32_t launch_group_blocked(gorse_b200_cf *cf, float *X, const float *Y, const int64_t *off, const int32_t *idx, float reg, float w,
                                    const int32_t *rows, int32_t n_rows)
{
    gorse_b200_ctx *c = cf->ctx;
    constexpr int D = G * KPL, YS = E * G * (G + 1) + (G < 32 ? G : 0);
    const size_t s_bytes = sizeof(float) * D * D, per_warp = sizeof(float) * (32 / G) * YS;
    const int warps = (int)std::max<size_t>(1, std::min<size_t>(G == 16 ? 32 : 16, (220 * 1024 - s_bytes) / per_warp));
    const size_t sm = s_bytes + warps * per_warp;
    const int groups_per_cta = warps * (32 / G);
    const int grid = (int)std::max<int64_t>(1, std::min<int64_t>(((int64_t)n_rows + groups_per_cta - 1) / groups_per_cta, (int64_t)c->sm_count));
    auto *k = als_rows_group_blocked_kernel<G, E, KPL>;
    GB_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
    k<<<grid, 32 * warps, sm, c->stream>>>(X, Y, off, idx, cf->gram.p, reg, w, rows, n_rows);
    GB_LAUNCHED(c);
    return GORSE_B200_OK;
}

template <int G, int E>
static int32_t launch_group_blocked_d(gorse_b200_cf *cf, float *X, const float *Y, const int64_t *off, const int32_t *idx, float reg, float w,
                                      const int32_t *rows, int32_t n_rows)
{
    switch (cf->d / 32) {
        case 1: return launch_group_blocked<G, E, 32 / G>(cf, X, Y, off, idx, reg, w, rows, n_rows);
        case 2: return launch_group_blocked<G, E, 64 / G>(cf, X, Y, off, idx, reg, w, rows, n_rows);
        case 3: return launch_group_blocked<G, E, 96 / G>(cf, X, Y, off, idx, reg, w, rows, n_rows);
        default: return launch_group_blocked<G, E, 128 / G>(cf, X, Y, off, idx, reg, w, rows, n_rows);
    }
}

// ---- chunk Grams, and the Gram form for rows too long to stage (DESIGN.md 5.2) --------------------------------------
// eALS over f for one row is exactly one Gauss-Seidel sweep on  A x = h  with
//     A = (1-w) * G + w * S + reg * I,   G = sum_{t in R} y_t y_t^T,   h = sum_{t in R} y_t
// (a = h_f - (1-w) sum_{k!=f} x_k G[k][f],  b = w sum_{k!=f} x_k S[k][f],  c = (1-w) G[f][f]; model.go:666-680).
// A long row is cut into chunks of <= GB_ALS_CHUNK entries; each CTA turns one chunk into a partial (G, h), the partials
// of a row are summed into its first one, and one CTA per row does the sweep.  S takes the same chunk kernels over the
// list of rows with feedback.
#define GB_ALS_CHUNK 2048

// partial[c] = (G, h) over the rows Y[idx[chunk_begin[c] + t]], t < chunk_len[c]; d <= 128, 16x16 threads with a TxT
// register tile each
template <int T>
__global__ void __launch_bounds__(256) als_chunk_gram_kernel(const float *Y, int d, const int32_t *idx, const int64_t *chunk_begin,
                                                             const int32_t *chunk_len, float *partial)
{
    extern __shared__ float xs[];  // [16][dp]
    const int dp = 16 * T;
    const int ti = threadIdx.x >> 4, tj = threadIdx.x & 15;
    GramTile<T> tile;
    tile.zero();
    float hacc[T];
#pragma unroll
    for (int a = 0; a < T; a++) hacc[a] = 0.f;
    const int64_t b0 = chunk_begin[blockIdx.x];
    const int len = chunk_len[blockIdx.x];
    for (int base = 0; base < len; base += 16) {
        for (int e = threadIdx.x; e < 16 * dp; e += 256) {
            int rr = e / dp, k = e - rr * dp;
            float v = 0.f;
            if (base + rr < len && k < d) v = __ldg(Y + (int64_t)__ldg(idx + b0 + base + rr) * d + k);
            xs[e] = v;
        }
        __syncthreads();
#pragma unroll 4
        for (int rr = 0; rr < 16; rr++) {
            float a[T], b[T];
#pragma unroll
            for (int k = 0; k < T; k++) { a[k] = xs[rr * dp + ti * T + k]; b[k] = xs[rr * dp + tj * T + k]; }
            tile.mac(a, b);
            if (ti == 0) {
#pragma unroll
                for (int y = 0; y < T; y++) hacc[y] += b[y];
            }
        }
        __syncthreads();
    }
    float *out = partial + (int64_t)blockIdx.x * als_partial_stride(d);
#pragma unroll
    for (int x = 0; x < T; x++)
#pragma unroll
        for (int y = 0; y < T; y++) {
            int i = ti * T + x, j = tj * T + y;
            if (i < d && j < d) out[i * d + j] = tile.get(x, y);
        }
    if (ti == 0) {
#pragma unroll
        for (int y = 0; y < T; y++) if (tj * T + y < d) out[d * d + tj * T + y] = hacc[y];
    }
}

// the same partial (G, h) at d > 128: one thread per element (row d of G is h), grid (chunks, element tiles)
__global__ void __launch_bounds__(256) als_chunk_gram_generic_kernel(const float *Y, int d, const int32_t *idx, const int64_t *chunk_begin,
                                                                     const int32_t *chunk_len, float *partial)
{
    const int e = blockIdx.y * 256 + threadIdx.x;
    if (e >= d * d + d) return;
    const int i = e / d, j = e - i * d;
    const int64_t b0 = chunk_begin[blockIdx.x];
    const int len = chunk_len[blockIdx.x];
    float acc = 0.f;
    for (int t = 0; t < len; t++) {
        const float *y = Y + (int64_t)__ldg(idx + b0 + t) * d;
        acc = i < d ? __fmaf_rn(__ldg(y + i), __ldg(y + j), acc) : acc + __ldg(y + j);
    }
    partial[(int64_t)blockIdx.x * als_partial_stride(d) + e] = acc;
}

// partial[first chunk of the row] = sum of the row's chunk partials, in chunk order (deterministic); grid (rows, element tiles).
// Summing inside als_solve_kernel leaves one CTA to walk all chunks of its row alone: the hottest item of C3 has 232 chunks
// = 15 MB, and that single CTA was the tail of the whole kernel.
__global__ void __launch_bounds__(256) als_partial_reduce_kernel(const int32_t *row_chunk0, int stride4, float *partial)
{
    const int c0 = row_chunk0[blockIdx.x], c1 = row_chunk0[blockIdx.x + 1];
    if (c1 - c0 <= 1) return;
    const int e = blockIdx.y * 256 + threadIdx.x;
    if (e >= stride4) return;
    float4 *p = reinterpret_cast<float4 *>(partial);
    float4 acc = p[(int64_t)c0 * stride4 + e];
    for (int c = c0 + 1; c < c1; c++) {
        const float4 v = p[(int64_t)c * stride4 + e];
        acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    p[(int64_t)c0 * stride4 + e] = acc;
}

// one CTA per long row: its (already summed) partial -> A, then one Gauss-Seidel sweep by warp 0 in RESIDUAL form:
//     r = h - A x (all warps);   for f:  delta = r_f / A_ff,  x_f += delta,  r -= delta * A[:, f]
// which is the same sweep (x_f + r_f / A_ff == (h_f - sum_{k != f} A_fk x_k) / A_ff) without a reduction on the sequential
// chain: lane l holds r, x and 1 / A_kk for k = l + 32 j, a step is one multiply, one shuffle and d / 32 FMAs whose A operands
// (column f, conflict-free thanks to the d + 1 row pitch) do not depend on the chain.  A 128-element dot summed across the
// warp per coordinate (5 dependent shuffles + a divide) measured 1.03 ms per half-sweep at C3.
// Any d <= 128: lane-block j covers k = 32 j .. 32 j + 31, and coordinates k >= d are masked.
__global__ void __launch_bounds__(256) als_solve_kernel(float *X, int d, const float *S, float reg, float w, const int32_t *rows,
                                                        const int32_t *row_chunk0, const float *partial)
{
    extern __shared__ float sm[];
    float *A = sm;                 // [d][d+1]
    float *h = A + d * (d + 1);    // [d]   h, then the residual
    float *x = h + d;              // [d]
    const int r = rows[blockIdx.x];
    const int dd = d * d, dp = d + 1;
    const float *g0 = partial + (int64_t)row_chunk0[blockIdx.x] * als_partial_stride(d);
    const float omw = 1.0f - w;
    // the row's summed partial is one 16-byte aligned (G, h) block, and S is allocated to a multiple of 4 floats: float4
    // loads, four in flight per thread.  (A scalar loop with a run-time inner trip count sends its 64 loads per thread one
    // DRAM latency after the other: 0.27 + 1.13 ms per epoch at C3 for what is 0.13 GB of traffic.)
    const float4 *p4 = reinterpret_cast<const float4 *>(g0);
    const float4 *s4 = reinterpret_cast<const float4 *>(S);
#pragma unroll 4
    for (int e4 = threadIdx.x; 4 * e4 < dd; e4 += blockDim.x) {
        const float4 g = p4[e4], sv = __ldg(s4 + e4);
        const float a[4] = {omw * g.x + w * sv.x, omw * g.y + w * sv.y, omw * g.z + w * sv.z, omw * g.w + w * sv.w};
        int i = 4 * e4 / d, j = 4 * e4 - i * d;   // element 4 e4 + q is (i, j) of G, wrapping to the next row at j = d
#pragma unroll
        for (int q = 0; q < 4; q++) {
            if (4 * e4 + q < dd) A[i * dp + j] = i == j ? a[q] + reg : a[q];
            if (++j == d) { i++; j = 0; }
        }
    }
    for (int e = threadIdx.x; e < d; e += blockDim.x) {
        h[e] = g0[dd + e];
        x[e] = X[(int64_t)r * d + e];
    }
    __syncthreads();
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
    // residual rows k = wid, wid + nw, ...: r_k = h_k - A[k, :] x
    float res[16];   // d / nw <= 16 rows per warp
#pragma unroll
    for (int q = 0; q < 16; q++) {
        const int k = wid + q * nw;
        float s = 0.f;
        if (k < d)
            for (int jx = lane; jx < d; jx += 32) s += A[k * dp + jx] * x[jx];
        res[q] = warp_sum(s);
    }
    __syncthreads();   // every warp has read h's neighbours' x; now h becomes the residual
#pragma unroll
    for (int q = 0; q < 16; q++) {
        const int k = wid + q * nw;
        if (k < d && lane == 0) h[k] -= res[q];
    }
    __syncthreads();
    if (wid == 0) {
        const int kpl = (d + 31) >> 5;
        bool ok[4];
        float rr[4], xv[4], inv[4];
#pragma unroll
        for (int jx = 0; jx < 4; jx++) {
            const int k = lane + 32 * jx;
            ok[jx] = k < d;
            rr[jx] = ok[jx] ? h[k] : 0.f;
            xv[jx] = ok[jx] ? x[k] : 0.f;
            inv[jx] = ok[jx] ? 1.0f / A[k * dp + k] : 0.f;
        }
        // the last block stops at f = d - 1 through its trip count.  (A break at f = d inside the unrolled loop keeps the
        // compiler from issuing the A loads of later steps early, which puts their latency on the chain.)
#pragma unroll
        for (int jf = 0; jf < 4; jf++) {
            if (jf < kpl) {
                const int n_o = min(32, d - 32 * jf);
#pragma unroll 4
                for (int o = 0; o < n_o; o++) {
                    const int f = 32 * jf + o;
                    const float delta = __shfl_sync(0xffffffffu, rr[jf] * inv[jf], o);
                    if (lane == o) xv[jf] += delta;
#pragma unroll
                    for (int jx = 0; jx < 4; jx++)
                        if (ok[jx]) rr[jx] = fmaf(-delta, A[(lane + 32 * jx) * dp + f], rr[jx]);
                }
            }
        }
#pragma unroll
        for (int jx = 0; jx < 4; jx++)
            if (ok[jx]) X[(int64_t)r * d + lane + 32 * jx] = xv[jx];
    }
}

// partial[c] = (G, h) of chunk c: the rows Y[idx[begin[c] + t]], t < len[c]
static int32_t chunk_gram(gorse_b200_cf *cf, const float *Y, const int32_t *idx, const int64_t *begin, const int32_t *len, int32_t nc)
{
    gorse_b200_ctx *c = cf->ctx;
    const int d = cf->d;
    float *partial = cf->als_partial.p;
    if (d == 128) return als_chunk_gram_tc(c, Y, idx, begin, len, nc, partial);
    if (d > 128) als_chunk_gram_generic_kernel<<<dim3(nc, div_up(d * d + d, 256)), 256, 0, c->stream>>>(Y, d, idx, begin, len, partial);
    else if (d > 64) als_chunk_gram_kernel<8><<<nc, 256, sizeof(float) * 16 * 16 * 8, c->stream>>>(Y, d, idx, begin, len, partial);
    else if (d > 32) als_chunk_gram_kernel<4><<<nc, 256, sizeof(float) * 16 * 16 * 4, c->stream>>>(Y, d, idx, begin, len, partial);
    else if (d > 16) als_chunk_gram_kernel<2><<<nc, 256, sizeof(float) * 16 * 16 * 2, c->stream>>>(Y, d, idx, begin, len, partial);
    else als_chunk_gram_kernel<1><<<nc, 256, sizeof(float) * 16 * 16 * 1, c->stream>>>(Y, d, idx, begin, len, partial);
    GB_LAUNCHED(c);
    return GORSE_B200_OK;
}

// S = sum of x x^T over this rank's rows with feedback (X is the whole table): the chunk partials are summed in chunk order,
// so S is the same every run; in a distributed context the d x d sums are all-reduced, so every rank ends with the same bits.
static int32_t run_gram(gorse_b200_cf *cf, int side, const float *X)
{
    gorse_b200_ctx *c = cf->ctx;
    const int dd = cf->d * cf->d, nc = cf->als_s_chunks[side];
    if (nc > 0) {
        GB_TRY(chunk_gram(cf, X, cf->als_s_rows[side].p, cf->als_s_begin[side].p, cf->als_s_len[side].p, nc));
        gram_reduce_kernel<<<div_up(dd, 256), 256, 0, c->stream>>>(cf->als_partial.p, nc, dd, als_partial_stride(cf->d), cf->gram.p);
        GB_LAUNCHED(c);
    } else {
        GB_CUDA(cudaMemsetAsync(cf->gram.p, 0, sizeof(float) * dd, c->stream));
    }
    if (c->world > 1) {
        GB_NCCL_API(nc_api);
        GB_NCCL(nc_api, AllReduce(cf->gram.p, cf->gram.p, (size_t)dd, ncclFloat32, ncclSum, c->comm, c->stream));
    }
    return GORSE_B200_OK;
}

// Rows are bucketed by length, one launch per class.  At d % 32 == 0, d <= 128 the short classes are kRowClasses: a row of
// n entries takes the first class with n <= max_n, run by `launch`.  Lane groups with blocked staging beat the thread-per-row
// kernel in every class above 4 entries (<= 8: 0.80 vs 1.16 ms, <= 16: 1.27 vs 1.99 ms per half-sweep at C3); the thread
// kernel keeps the shortest rows, where it is 0.14 ms ahead (also when they are many: the 300 K short user rows of C3 take
// 1.69 ms there and 2.0 ms on the 8-lane kernel).  33..64 entries are a class of their own: 8.4 instead of 12.7 KB of
// staging per warp, so 16 warps per SM instead of 12.
// At other d, als_rows_kernel takes the rows with n (d+1) <= kStageFloats[k] floats (12 / 48 KB per warp) as class k.
// Longer rows form class GB_ALS_LONG: the Gram form at d <= 128, als_rows_kernel without staging above.
using RowLauncher = int32_t (*)(gorse_b200_cf *cf, float *X, const float *Y, const int64_t *off, const int32_t *idx, float reg, float w,
                                const int32_t *rows, int32_t n_rows);
struct RowClass { int max_n; RowLauncher launch; };
#define GB_ALS_CLASSES 7
#define GB_ALS_LONG 6   // index of the long-row class
static const RowClass kRowClasses[GB_ALS_LONG] = {
    {4, als_thread_rows},
    {8, launch_group_blocked_d<8, 1>},
    {16, launch_group_blocked_d<16, 1>},
    {32, launch_group_blocked_d<16, 2>},
    {64, launch_group_blocked_d<32, 2>},
    {96, launch_group_blocked_d<32, 3>},
};
static const int kStageFloats[2] = {3072, 12288};

static bool als_grouped(const gorse_b200_cf *cf) { return cf->d % 32 == 0 && cf->d <= 128; }

// rows of `side` (0 users, 1 items) this rank updates: users as in cf_create (cf->u_lo/u_hi), items by the same rule
static void shard_range(const gorse_b200_cf *cf, int side, int32_t &lo, int32_t &hi)
{
    lo = side == 0 ? cf->u_lo : cf->i_lo;
    hi = side == 0 ? cf->u_hi : cf->i_hi;
}

// [b, e) in chunks of at most GB_ALS_CHUNK
static void cut_chunks(int64_t b, int64_t e, std::vector<int64_t> &begin, std::vector<int32_t> &len)
{
    for (int64_t p = b; p < e; p += GB_ALS_CHUNK) {
        begin.push_back(p);
        len.push_back((int32_t)std::min<int64_t>(GB_ALS_CHUNK, e - p));
    }
}

template <typename T>
static int32_t upload(DevBuf<T> &dst, const std::vector<T> &src)
{
    GB_TRY(dst.alloc(src.size()));
    if (!src.empty()) GB_CUDA(cudaMemcpy(dst.p, src.data(), sizeof(T) * src.size(), cudaMemcpyHostToDevice));
    return GORSE_B200_OK;
}

static int32_t prepare_als(gorse_b200_cf *cf)
{
    if (cf->als_ready) return GORSE_B200_OK;
    const int d = cf->d, dp = d + 1;
    const bool grouped = als_grouped(cf);
    int32_t max_chunks = 0;
    for (int side = 0; side < 2; side++) {
        // multi-rank: this rank updates its own range of users and of items only (SURVEY 8e).  The host offsets hold this
        // rank's rows only, rebased: row r sits at index r - r_lo
        int32_t r_lo = 0, r_hi = 0;
        shard_range(cf, side, r_lo, r_hi);
        const int64_t *off = (side == 0 ? cf->h_user_off : cf->h_item_off).data() - r_lo;
        std::vector<int32_t> cls[GB_ALS_CLASSES], s_rows;
        for (int32_t r = r_lo; r < r_hi; r++) {
            const int64_t n = off[(size_t)r + 1] - off[r];
            if (n > 0) s_rows.push_back(r);   // the rows S sums over (model.go:651,699)
            int k;
            if (grouped) {
                k = GB_ALS_LONG;
                for (int q = 0; q < GB_ALS_LONG; q++) if (n <= kRowClasses[q].max_n) { k = q; break; }
            } else k = n * dp <= kStageFloats[0] ? 0 : n * dp <= kStageFloats[1] ? 1 : GB_ALS_LONG;
            cls[k].push_back(r);
        }
        for (int k = 0; k < GB_ALS_CLASSES; k++) {
            // longest rows first inside a class: better tail behaviour
            std::stable_sort(cls[k].begin(), cls[k].end(), [&](int32_t a, int32_t b) {
                return off[(size_t)a + 1] - off[a] > off[(size_t)b + 1] - off[b];
            });
            cf->als_rows_n[side][k] = (int32_t)cls[k].size();
            GB_TRY(upload(cf->als_rows[side][k], cls[k]));
        }
        // long rows take the Gram form when d <= 128: their entries in chunks, row i's from chunk row_chunk0[i] on
        std::vector<int64_t> chunk_begin, s_begin;
        std::vector<int32_t> chunk_len, row_chunk0, s_len;
        if (d <= 128) {
            for (const int32_t r : cls[GB_ALS_LONG]) {
                row_chunk0.push_back((int32_t)chunk_begin.size());
                cut_chunks(off[r], off[(size_t)r + 1], chunk_begin, chunk_len);
            }
            row_chunk0.push_back((int32_t)chunk_begin.size());
        }
        cut_chunks(0, (int64_t)s_rows.size(), s_begin, s_len);
        cf->als_n_chunks[side] = (int32_t)chunk_begin.size();
        cf->als_s_chunks[side] = (int32_t)s_begin.size();
        max_chunks = std::max({max_chunks, cf->als_n_chunks[side], cf->als_s_chunks[side]});
        GB_TRY(upload(cf->als_chunk_begin[side], chunk_begin));
        GB_TRY(upload(cf->als_chunk_len[side], chunk_len));
        GB_TRY(upload(cf->als_row_chunk0[side], row_chunk0));
        GB_TRY(upload(cf->als_s_rows[side], s_rows));
        GB_TRY(upload(cf->als_s_begin[side], s_begin));
        GB_TRY(upload(cf->als_s_len[side], s_len));
    }
    GB_TRY(cf->als_partial.alloc((size_t)max_chunks * als_partial_stride(d)));
    GB_TRY(cf->gram.alloc(((size_t)d * d + 3) & ~(size_t)3));   // a multiple of 4 floats: als_solve_kernel reads S as float4
    GB_CUDA(cudaFuncSetAttribute(als_solve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
    GB_CUDA(cudaFuncSetAttribute(als_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
    cf->als_ready = true;
    return GORSE_B200_OK;
}

static int32_t run_rows(gorse_b200_cf *cf, int side, float *X, const float *Y, const int64_t *off, const int32_t *idx,
                        float reg, float w, float *pred_scratch)
{
    gorse_b200_ctx *c = cf->ctx;
    const int d = cf->d;
    const bool grouped = als_grouped(cf);
    for (int k = 0; k < GB_ALS_CLASSES; k++) {
        const int32_t n_rows = cf->als_rows_n[side][k];
        if (n_rows == 0) continue;
        const int32_t *rows = cf->als_rows[side][k].p;
        if (grouped && k != GB_ALS_LONG) {
            GB_TRY(kRowClasses[k].launch(cf, X, Y, off, idx, reg, w, rows, n_rows));
        } else if (k == GB_ALS_LONG && d <= 128) {
            // Gram form: chunk partials, summed per row into its first chunk, then one sweep per row
            const int32_t *row_chunk0 = cf->als_row_chunk0[side].p;
            const int stride4 = als_partial_stride(d) / 4;
            GB_TRY(chunk_gram(cf, Y, idx, cf->als_chunk_begin[side].p, cf->als_chunk_len[side].p, cf->als_n_chunks[side]));
            als_partial_reduce_kernel<<<dim3(n_rows, div_up(stride4, 256)), 256, 0, c->stream>>>(row_chunk0, stride4, cf->als_partial.p);
            GB_LAUNCHED(c);
            const size_t sm = sizeof(float) * ((size_t)d * (d + 1) + 2 * d);
            als_solve_kernel<<<n_rows, 256, sm, c->stream>>>(X, d, cf->gram.p, reg, w, rows, row_chunk0, cf->als_partial.p);
            GB_LAUNCHED(c);
        } else {
            // one warp per row; the long class (d > 128) gathers from L2 without staging
            const int stage = k == GB_ALS_LONG ? 0 : kStageFloats[k];
            const size_t sm = sizeof(float) * GB_ALS_WARPS * (size_t)(d + stage);
            const int ctas_per_sm = k == 0 ? 4 : 1;
            const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((n_rows + GB_ALS_WARPS - 1) / GB_ALS_WARPS, (int64_t)c->sm_count * ctas_per_sm * (k == GB_ALS_LONG ? 8 : 1)));
            als_rows_kernel<<<grid, 32 * GB_ALS_WARPS, sm, c->stream>>>(X, Y, d, off, idx, cf->gram.p, reg, w, rows, n_rows, stage, pred_scratch);
            GB_LAUNCHED(c);
        }
    }
    return GORSE_B200_OK;
}

}  // namespace gb

using namespace gb;

// every rank sends its own row range of `table` (rows x d, present in full on every rank) to all the others
static int32_t exchange_shards(gorse_b200_cf *cf, int side, float *table)
{
    gorse_b200_ctx *c = cf->ctx;
    GB_NCCL_API(nc);
    if (!nc->Broadcast || !nc->GroupStart || !nc->GroupEnd) {
        set_error("the loaded libnccl lacks ncclBroadcast/ncclGroupStart/ncclGroupEnd");
        return GORSE_B200_ERR_NCCL;
    }
    const int64_t rows = side == 0 ? cf->n_users : cf->n_items;
    GB_NCCL(nc, GroupStart());
    for (int r = 0; r < c->world; r++) {
        const int64_t lo = rows * r / c->world, hi = rows * (r + 1) / c->world;
        if (hi == lo) continue;
        float *p = table + lo * cf->d;
        GB_NCCL(nc, Broadcast(p, p, (size_t)(hi - lo) * cf->d, ncclFloat32, r, c->comm, c->stream));
    }
    GB_NCCL(nc, GroupEnd());
    return GORSE_B200_OK;
}

int32_t gb::als_epoch_tables(gorse_b200_cf *cf, float *P_own, float *Q, float reg, float alpha)
{
    gorse_b200_ctx *c = cf->ctx;
    const bool multi = c->world > 1;
    GB_TRY(prepare_als(cf));
    // scratch kept in the model: a cudaMalloc/cudaFree pair per epoch costs more than some of the kernels of a C3 epoch
    const size_t n_pred = (size_t)std::max<int64_t>(1, std::max(cf->n_feedback, cf->n_item_feedback));
    GB_TRY(cf->als_pred.grow(n_pred));
    DevBuf<float> &pred = cf->als_pred;
    int32_t st;
    auto done = [&](int32_t s) {
        cudaStreamSynchronize(c->stream);
        return s;
    };
    // Multi-rank (SURVEY 8e): Q is replicated and P is range-sharded as for BPR.  The user half-sweep needs only Q, the item
    // half-sweep needs ALL of P, so the epoch works on a full copy P_all: own rows in, user sweep on the own range, ranges
    // exchanged, S^p and the item sweep (own item range) on P_all, item ranges of Q exchanged, own rows of P_all back.
    // Each Gram is the all-reduced sum of the ranks' partial Grams over their own row ranges, so every rank holds
    // bit-identical S^q, S^p and Q (the sums differ from the single-GPU epoch by reassociation only).
    float *P = P_own;
    const int64_t own = (int64_t)(cf->u_hi - cf->u_lo) * cf->d;
    if (multi) {
        if (cf->P_all.n == 0 && (st = cf->P_all.alloc((size_t)cf->n_users * cf->d))) return done(st);
        P = cf->P_all.p;
        if (own) {
            cudaError_t e = cudaMemcpyAsync(P + (int64_t)cf->u_lo * cf->d, P_own, own * sizeof(float), cudaMemcpyDeviceToDevice, c->stream);
            if (e != cudaSuccess) { set_error("als_epoch: %s", cudaGetErrorString(e)); return done(GORSE_B200_ERR_CUDA); }
        }
    }
    // the row kernels index the offsets with GLOBAL row ids: hand them the rank's arrays shifted by the range start
    const int64_t *uoff = cf->user_off.p - cf->u_lo, *ioff = cf->item_off.p - cf->i_lo;
    if ((st = run_gram(cf, 1, Q))) return done(st);
    if ((st = run_rows(cf, 0, P, Q, uoff, cf->user_items.p, reg, alpha, pred.p))) return done(st);
    if (multi && (st = exchange_shards(cf, 0, P))) return done(st);
    if ((st = run_gram(cf, 0, P))) return done(st);
    if ((st = run_rows(cf, 1, Q, P, ioff, cf->item_users.p, reg, alpha, pred.p))) return done(st);
    if (multi) {
        if ((st = exchange_shards(cf, 1, Q))) return done(st);
        cudaError_t e = cudaSuccess;
        if (own) e = cudaMemcpyAsync(P_own, P + (int64_t)cf->u_lo * cf->d, own * sizeof(float), cudaMemcpyDeviceToDevice, c->stream);
        // the BPR exchange keeps the last synchronised item table in Q0
        if (e == cudaSuccess && cf->Q0.n) e = cudaMemcpyAsync(cf->Q0.p, Q, cf->Q.n * sizeof(float), cudaMemcpyDeviceToDevice, c->stream);
        if (e != cudaSuccess) { set_error("als_epoch: %s", cudaGetErrorString(e)); return done(GORSE_B200_ERR_CUDA); }
    }
    cudaError_t e = cudaStreamSynchronize(c->stream);
    if (e != cudaSuccess) { set_error("als_epoch: %s", cudaGetErrorString(e)); return done(GORSE_B200_ERR_CUDA); }
    return done(GORSE_B200_OK);
}

extern "C" int32_t gorse_b200_als_epoch(gorse_b200_cf *cf, float reg, float alpha)
{
    GB_CHECK_ARG(cf != nullptr, "cf is NULL");
    if (!cf->has_item_csr) { set_error("als_epoch needs the item CSR (item_off/item_users) at cf_create"); return GORSE_B200_ERR_STATE; }
    ScopedDevice sd(cf->ctx->device);
    return als_epoch_tables(cf, cf->P.p, cf->Q.p, reg, alpha);
}
