// embedding_eval.cu -- `gorse-bench embedding` on device: EvaluateEmbedding (cmd/gorse-bench/main.go:403-465) for every test
// user in one call.  Per user, each candidate with an embedding is scored total = 0 - Euclidean(c, s_1) - Euclidean(c, s_2) ...
// over the shots with an embedding, in shot order; then TopKFilter, NDCG, Precision and Recall as cf.Evaluate does them.
//
//   emb_dist_kernel   one CTA per 16 consecutive 4 x 4 micro-tiles of one user.  The rows they touch are staged in shared
//                     memory 64 floats at a time (cp.async, two buffers); a group of 16 threads owns 4 x 4 pairs, thread l of
//                     the group running lane l of floats.Euclidean's 16-lane accumulator (floats_avx512.c:374-441: sub, mul,
//                     add, no fusing) over the elements l, l + 16, ... in chunk order, the partials kept in registers across
//                     the 64-float steps.  The group then forms the reference's reduction tree with shuffles, thread p adds
//                     the d % 16 tail of pair p (8-lane block, then fused steps) and takes __fsqrt_rn.  The distances of a
//                     chunk of users go to a buffer, pair (c, s) of user u at base(u) + s m_u + c.
//   emb_total_kernel  one CTA per user: per candidate, total = 0 and total -= dist in shot order (__fsub_rn), so a user whose
//                     shots span many CTAs still gets the reference's sequential sum.
//   ranking           eval_rank_kernel (evaluate.cu), unchanged, on the candidates with an embedding; a user the reference
//                     skips gets an empty test row.  Device-sampled negatives come from eval_negatives_kernel.
#include <algorithm>
#include <cmath>
#include <cstdlib>

#include "evaluate.cuh"

namespace gb {
namespace {

// A user's pairs are cut into 4 x 4 micro-tiles (a candidate quad x a shot quad), numbered candidate quad major.  A CTA
// takes MT consecutive micro-tiles of one user, one per 16-thread group, so only the user's last CTA has idle groups and a
// micro-tile wastes at most the padding of its quads.  MT consecutive micro-tiles touch at most 18 quads: with q shot quads
// per candidate quad, at most 15 / q + 2 candidate quads and min(16, q) shot quads.
constexpr int MT = 16;            // micro-tiles per CTA
constexpr int DK = 64;            // floats of a row staged per step
constexpr int LD = DK + 4;        // smem row stride: groups of a warp that read rows 4 apart hit banks 16 apart
constexpr int ROWS = 72;          // staged rows: at most 18 quads
constexpr int THREADS = 16 * MT;
constexpr int64_t MAX_USER_PAIRS = int64_t(1) << 28;    // distances of one user held at once (1 GB)
constexpr int64_t CHUNK_PAIRS = int64_t(1) << 26;       // distances per chunk of users (256 MB)

__device__ __forceinline__ void cp_async16(float *smem, const float *gmem)
{
    const unsigned s = (unsigned)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async4(float *smem, const float *gmem)
{
    const unsigned s = (unsigned)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"(s), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory"); }

// any non-finite value in a present row sets *bad: one warp per row
__global__ void emb_finite_kernel(const float *emb, int64_t n_items, int32_t dim, const uint8_t *mask, int32_t *bad)
{
    const int lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < n_items; r += warps) {
        if (mask && !mask[r]) continue;
        const float *row = emb + r * dim;
        bool ok = true;
        for (int32_t i = lane; i < dim; i += 32) ok &= isfinite(row[i]);
        if (!ok) *bad = 1;
    }
}

// candidates of user u with an embedding: test(u) then negatives(u), in order (main.go:417-426); none when the user has no
// test item or no shot with an embedding (main.go:412-414, 423-425, 446-448)
__global__ void emb_cand_kernel(const int64_t *test_off, const int32_t *test_items, const int64_t *neg_off, const int32_t *neg_items,
                                const uint8_t *mask, const int64_t *shot_off, int32_t n_users, bool count_only, int32_t *count,
                                const int64_t *cand_off, int32_t *cand_items)
{
    const int32_t u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= n_users) return;
    int32_t k = 0;
    int32_t *out = count_only ? nullptr : cand_items + cand_off[u];
    if (test_off[u + 1] > test_off[u] && shot_off[u + 1] > shot_off[u]) {
        for (int64_t a = test_off[u]; a < test_off[u + 1]; a++) {
            const int32_t v = test_items[a];
            if (!mask || mask[v]) { if (out) out[k] = v; k++; }
        }
        for (int64_t a = neg_off[u]; a < neg_off[u + 1]; a++) {
            const int32_t v = neg_items[a];
            if (!mask || mask[v]) { if (out) out[k] = v; k++; }
        }
    }
    if (count_only) count[u] = k;
}

// distances of MT micro-tiles; the users of the launch are [u0, u0 + n_users) with tile_off / pair_base pointing at u0
template <bool VEC4>
__global__ void __launch_bounds__(THREADS) emb_dist_kernel(const float *__restrict__ emb, int32_t dim, const int64_t *__restrict__ cand_off,
                                                           const int32_t *__restrict__ cand_items, const int64_t *__restrict__ shot_off,
                                                           const int32_t *__restrict__ shot_items, const int64_t *__restrict__ tile_off,
                                                           const int64_t *__restrict__ pair_base, int32_t n_users, float *__restrict__ dist)
{
    __shared__ __align__(16) float sm[2][ROWS * LD];
    __shared__ int32_t row_item[ROWS];
    const int64_t b = tile_off[0] + blockIdx.x;
    int32_t lo = 0, hi = n_users;   // the last user whose tiles start at or before b
    while (hi - lo > 1) {
        const int32_t mid = (lo + hi) >> 1;
        if (tile_off[mid] <= b) lo = mid; else hi = mid;
    }
    const int32_t u = lo;
    const int64_t c_beg = cand_off[u], m = cand_off[u + 1] - c_beg;
    const int64_t s_beg = shot_off[u], k = shot_off[u + 1] - s_beg;
    const int64_t nq_s = (k + 3) / 4, total = ((m + 3) / 4) * nq_s;
    const int64_t t0 = (b - tile_off[u]) * MT;
    const int nt = (int)min((int64_t)MT, total - t0);
    // staged rows: candidate quads cq_lo .. of the CTA's micro-tiles, then shot quad slots j = 0 .. n_ss - 1 holding shot
    // quads (sq_first + j) mod nq_s; micro-tile i of the CTA reads candidate slot cq - cq_lo and shot slot i mod nq_s
    const int64_t cq_lo = t0 / nq_s, sq_first = t0 % nq_s;
    const int rows_c = 4 * (int)((t0 + nt - 1) / nq_s - cq_lo + 1);
    const int rows = rows_c + 4 * (int)min((int64_t)nt, nq_s);
    const int tid = threadIdx.x, lane = tid & 15, g = tid >> 4;
    const bool active = g < nt;
    const int64_t t = t0 + (active ? g : 0), cq = t / nq_s, sq = t % nq_s;
    const int crow = 4 * (int)(cq - cq_lo), srow = rows_c + 4 * (int)((active ? g : 0) % nq_s);
    for (int r = tid; r < rows; r += THREADS) {   // padding rows repeat the first row of their side; their pairs are not written
        if (r < rows_c) {
            const int64_t c = 4 * cq_lo + r;
            row_item[r] = cand_items[c_beg + (c < m ? c : 0)];
        } else {
            const int64_t s = 4 * ((sq_first + (r - rows_c) / 4) % nq_s) + (r - rows_c) % 4;
            row_item[r] = shot_items[s_beg + (s < k ? s : 0)];
        }
    }
    __syncthreads();

    const int32_t dmain = dim & ~15;
    const int n_steps = (dmain + DK - 1) / DK;
    auto stage = [&](int step, int buf) {
        const int32_t k0 = step * DK, w = min(DK, dmain - k0);
        float *dst = sm[buf];
        if (VEC4) {
            const int per_row = w / 4;
            for (int i = tid; i < rows * (DK / 4); i += THREADS) {
                const int row = i / (DK / 4), c4 = i % (DK / 4);
                if (c4 < per_row) cp_async16(dst + row * LD + 4 * c4, emb + (int64_t)row_item[row] * dim + k0 + 4 * c4);
            }
        } else {
            for (int i = tid; i < rows * DK; i += THREADS) {
                const int row = i / DK, c = i % DK;
                if (c < w) cp_async4(dst + row * LD + c, emb + (int64_t)row_item[row] * dim + k0 + c);
            }
        }
        cp_async_commit();
    };

    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) acc[i][j] = 0.f;
    if (n_steps > 0) stage(0, 0);
    for (int step = 0; step < n_steps; step++) {
        if (step + 1 < n_steps) { stage(step + 1, (step + 1) & 1); cp_async_wait<1>(); }
        else cp_async_wait<0>();
        __syncthreads();
        const float *A = sm[step & 1] + crow * LD + lane;
        const float *B = sm[step & 1] + srow * LD + lane;
        const int chunks = min(DK, dmain - step * DK) / 16;
        for (int ch = 0; ch < chunks; ch++) {
            float a[4], bb[4];
#pragma unroll
            for (int i = 0; i < 4; i++) { a[i] = A[i * LD + 16 * ch]; bb[i] = B[i * LD + 16 * ch]; }
#pragma unroll
            for (int i = 0; i < 4; i++)
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    float v = __fsub_rn(a[i], bb[j]);
                    v = __fmul_rn(v, v);
                    acc[i][j] = __fadd_rn(v, acc[i][j]);   // the first chunk: 0 + v*v == v*v
                }
        }
        __syncthreads();
    }

    // reduction tree of the 16 lanes (floats_avx512.c:327-339): s[l] + s[l+8], then +4, then even/odd, then e + o;
    // thread p of the group keeps the sum of pair p = (p / 4, p % 4)
    float mine = 0.f;
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) {
            float x = acc[i][j];
            x = __fadd_rn(x, __shfl_down_sync(0xffffffffu, x, 8, 16));
            x = __fadd_rn(x, __shfl_down_sync(0xffffffffu, x, 4, 16));
            x = __fadd_rn(x, __shfl_down_sync(0xffffffffu, x, 2, 16));
            x = __fadd_rn(x, __shfl_down_sync(0xffffffffu, x, 1, 16));
            x = __shfl_sync(0xffffffffu, x, 0, 16);
            if (lane == 4 * i + j) mine = x;
        }
    const int64_t c = 4 * cq + (lane >> 2), s = 4 * sq + (lane & 3);
    if (!active || c >= m || s >= k) return;
    float sum = mine;
    const float *pa = emb + (int64_t)row_item[crow + (lane >> 2)] * dim + dmain;
    const float *pb = emb + (int64_t)row_item[srow + (lane & 3)] * dim + dmain;
    int rem = dim - dmain;
    if (rem >= 8) {   // 8-lane block (:349-358)
        float p[8];
#pragma unroll
        for (int l = 0; l < 8; l++) { const float v = __fsub_rn(pa[l], pb[l]); p[l] = __fmul_rn(v, v); }
        float q4[4];
#pragma unroll
        for (int l = 0; l < 4; l++) q4[l] = __fadd_rn(p[l + 4], p[l]);
        sum = __fadd_rn(sum, __fadd_rn(__fadd_rn(q4[0], q4[2]), __fadd_rn(q4[1], q4[3])));
        pa += 8; pb += 8; rem -= 8;
    }
    for (int l = 0; l < rem; l++) { const float v = __fsub_rn(pa[l], pb[l]); sum = __fmaf_rn(v, v, sum); }
    dist[(pair_base[u] - pair_base[0]) + s * m + c] = __fsqrt_rn(sum);
}

// total of each candidate over the user's shots in shot order (main.go:427-442): one CTA per user of the launch
__global__ void emb_total_kernel(const int64_t *cand_off, const int64_t *shot_off, const int64_t *pair_base, const float *dist, float *score)
{
    const int32_t u = blockIdx.x;
    const int64_t m = cand_off[u + 1] - cand_off[u], k = shot_off[u + 1] - shot_off[u];
    const float *d = dist + (pair_base[u] - pair_base[0]);
    for (int64_t c = threadIdx.x; c < m; c += blockDim.x) {
        float t = 0.f;
        int64_t s = 0;
        for (; s + 4 <= k; s += 4) {
            const float d0 = d[s * m + c], d1 = d[(s + 1) * m + c], d2 = d[(s + 2) * m + c], d3 = d[(s + 3) * m + c];
            t = __fsub_rn(t, d0); t = __fsub_rn(t, d1); t = __fsub_rn(t, d2); t = __fsub_rn(t, d3);
        }
        for (; s < k; s++) t = __fsub_rn(t, d[s * m + c]);
        score[cand_off[u] + c] = t;
    }
}

// the call's device buffers, freed on every return
struct EmbWork {
    DevBuf<float> emb, dist, score, inv, metrics;
    DevBuf<uint8_t> mask;
    DevBuf<int64_t> test_off, shot_off, excl_off, neg_off, cand_off, rt_off, tile_off, pair_base;
    DevBuf<int32_t> test_items, shot_items, excl_items, neg_items, cand_items, rt_items, count;
    ~EmbWork()
    {
        emb.free(); dist.free(); score.free(); inv.free(); metrics.free(); mask.free();
        test_off.free(); shot_off.free(); excl_off.free(); neg_off.free(); cand_off.free(); rt_off.free(); tile_off.free(); pair_base.free();
        test_items.free(); shot_items.free(); excl_items.free(); neg_items.free(); cand_items.free(); rt_items.free(); count.free();
    }
};

template <typename T>
int32_t upload(DevBuf<T> &d, const T *h, size_t n, cudaStream_t s)
{
    GB_TRY(d.alloc(std::max<size_t>(n, 1)));
    if (n) GB_CUDA(cudaMemcpyAsync(d.p, h, sizeof(T) * n, cudaMemcpyHostToDevice, s));
    return GORSE_B200_OK;
}

// a CSR argument: offsets non-decreasing, ids in [0, n_items); rebased to start at 0
int32_t check_csr(const char *what, int64_t n_users, const int64_t *off, const int32_t *items, int32_t n_items, std::vector<int64_t> &rebased)
{
    GB_CHECK_ARG(off != nullptr, "%s_off is NULL", what);
    for (int64_t u = 0; u < n_users; u++) GB_CHECK_ARG(off[u + 1] >= off[u], "%s_off not non-decreasing at user %lld", what, (long long)u);
    const int64_t n = off[n_users] - off[0];
    GB_CHECK_ARG(n == 0 || items != nullptr, "%s_items is NULL", what);
    for (int64_t a = 0; a < n; a++)
        GB_CHECK_ARG(items[a] >= 0 && items[a] < n_items, "%s item %d out of range [0, %d)", what, items[a], n_items);
    rebased.resize((size_t)n_users + 1);
    for (int64_t u = 0; u <= n_users; u++) rebased[(size_t)u] = off[u] - off[0];
    return GORSE_B200_OK;
}

}  // namespace
}  // namespace gb

using namespace gb;

extern "C" int32_t gorse_b200_embedding_eval(gorse_b200_ctx *ctx, int32_t n_items, int32_t dim, const float *emb, const uint8_t *emb_mask,
                                             int64_t n_users, const int64_t *shot_off, const int32_t *shot_items, const int64_t *test_off,
                                             const int32_t *test_items, const int64_t *excl_off, const int32_t *excl_items,
                                             const int64_t *neg_off, const int32_t *neg_items, int32_t n_candidates, uint64_t seed,
                                             int32_t topk, float *out, int64_t *users_out)
{
    GB_CHECK_ARG(out != nullptr, "NULL out");
    GB_CHECK_ARG(n_items >= 0, "negative n_items");
    GB_CHECK_ARG(dim >= 1 && dim <= 16384, "dim %d out of range [1, 16384]", dim);
    GB_CHECK_ARG(n_items == 0 || emb != nullptr, "emb is NULL");
    GB_CHECK_ARG(topk >= 1 && topk <= GB_EVAL_MAX_TOPK, "topk %d out of range [1, %d]", topk, GB_EVAL_MAX_TOPK);
    GB_CHECK_ARG(n_users >= 0 && n_users < INT32_MAX, "n_users %lld out of range", (long long)n_users);
    const int32_t U = (int32_t)n_users;
    std::vector<int64_t> soff, toff, xoff, noff;
    GB_TRY(check_csr("shot", U, shot_off, shot_items, n_items, soff));
    GB_TRY(check_csr("test", U, test_off, test_items, n_items, toff));
    const bool sample = neg_off == nullptr;
    if (sample) {
        GB_CHECK_ARG(n_candidates >= 0, "negative n_candidates");
        GB_TRY(check_csr("excl", U, excl_off, excl_items, n_items, xoff));
    } else {
        GB_TRY(check_csr("neg", U, neg_off, neg_items, n_items, noff));
    }
    // the shots with an embedding, in order: a shot without one adds nothing to any total (main.go:431-433)
    std::vector<int64_t> vs_off((size_t)U + 1, 0);
    std::vector<int32_t> vs_items;
    vs_items.reserve((size_t)soff[(size_t)U]);
    for (int32_t u = 0; u < U; u++) {
        for (int64_t a = soff[(size_t)u]; a < soff[(size_t)u + 1]; a++)
            if (!emb_mask || emb_mask[shot_items[a]]) vs_items.push_back(shot_items[a]);
        vs_off[(size_t)u + 1] = (int64_t)vs_items.size();
    }
    // the per-user bound: every distance of one user is held at once
    for (int32_t u = 0; u < U; u++) {
        const int64_t nc = (toff[(size_t)u + 1] - toff[(size_t)u]) + (sample ? n_candidates : noff[(size_t)u + 1] - noff[(size_t)u]);
        const int64_t k = vs_off[(size_t)u + 1] - vs_off[(size_t)u];
        if (nc > 0 && k > MAX_USER_PAIRS / nc) {
            set_error("user %d: %lld candidates x %lld shots exceed %lld distances", u, (long long)nc, (long long)k, (long long)MAX_USER_PAIRS);
            return GORSE_B200_ERR_UNSUPPORTED;
        }
    }
    GB_CHECK_ARG(ctx != nullptr, "NULL ctx");

    // the sampler's membership test searches sorted rows; a row that is not sorted is sorted in a copy
    std::vector<int32_t> xs;
    if (sample) {
        xs.assign(excl_items, excl_items + xoff[(size_t)U]);
        for (int32_t u = 0; u < U; u++) {
            int32_t *a = xs.data() + xoff[(size_t)u], *e = xs.data() + xoff[(size_t)u + 1];
            if (!std::is_sorted(a, e)) std::sort(a, e);
        }
    }

    ScopedDevice sd(ctx->device);
    cudaStream_t s = ctx->stream;
    EmbWork W;
    cudaError_t e = cudaSuccess;
    auto cuda_fail = [&](cudaError_t err) {
        set_error("embedding_eval: %s", cudaGetErrorString(err));
        return err == cudaErrorMemoryAllocation ? GORSE_B200_ERR_OOM : GORSE_B200_ERR_CUDA;
    };
    const int ub = std::max(1, (U + 127) / 128);
    GB_TRY(upload(W.emb, emb, (size_t)n_items * dim, s));
    if (emb_mask) GB_TRY(upload(W.mask, emb_mask, (size_t)n_items, s));
    GB_TRY(upload(W.test_off, toff.data(), (size_t)U + 1, s));
    GB_TRY(upload(W.test_items, test_items, (size_t)toff[(size_t)U], s));
    GB_TRY(upload(W.shot_off, vs_off.data(), (size_t)U + 1, s));
    GB_TRY(upload(W.shot_items, vs_items.data(), vs_items.size(), s));
    GB_TRY(W.count.alloc((size_t)U + 1));
    GB_CUDA(cudaMemsetAsync(W.count.p, 0, sizeof(int32_t) * ((size_t)U + 1), s));
    // one pass over the present rows before anything is scored: the reference would push NaN into its heap
    if ((int64_t)n_items * dim > 0) {
        emb_finite_kernel<<<ctx->sm_count * 8, 256, 0, s>>>(W.emb.p, n_items, dim, emb_mask ? W.mask.p : nullptr, W.count.p + U);
        GB_LAUNCHED(ctx);
    }
    const uint64_t base = eval_negatives_base(seed);
    std::vector<int32_t> hc((size_t)U + 1);
    if (sample) {
        GB_TRY(upload(W.excl_off, xoff.data(), (size_t)U + 1, s));
        GB_TRY(upload(W.excl_items, xs.data(), xs.size(), s));
        launch_eval_negatives(s, W.excl_off.p, W.excl_items.p, W.test_off.p, W.test_items.p, U, 0, n_items, n_candidates, base, true,
                              W.count.p, nullptr, nullptr);
        GB_LAUNCHED(ctx);
    }
    if ((e = cudaMemcpyAsync(hc.data(), W.count.p, sizeof(int32_t) * ((size_t)U + 1), cudaMemcpyDeviceToHost, s)) != cudaSuccess ||
        (e = cudaStreamSynchronize(s)) != cudaSuccess)
        return cuda_fail(e);
    if (hc[(size_t)U]) { set_error("embedding_eval: a present embedding holds a non-finite value"); return GORSE_B200_ERR_ARG; }
    if (sample) {
        noff.assign((size_t)U + 1, 0);
        for (int32_t u = 0; u < U; u++) noff[(size_t)u + 1] = noff[(size_t)u] + hc[(size_t)u];
        GB_TRY(upload(W.neg_off, noff.data(), (size_t)U + 1, s));
        GB_TRY(W.neg_items.alloc(std::max<size_t>((size_t)noff[(size_t)U], 1)));
        launch_eval_negatives(s, W.excl_off.p, W.excl_items.p, W.test_off.p, W.test_items.p, U, 0, n_items, n_candidates, base, false,
                              nullptr, W.neg_off.p, W.neg_items.p);
        GB_LAUNCHED(ctx);
    } else {
        GB_TRY(upload(W.neg_off, noff.data(), (size_t)U + 1, s));
        GB_TRY(upload(W.neg_items, neg_items, (size_t)noff[(size_t)U], s));
    }
    if (U > 0) {
        emb_cand_kernel<<<ub, 128, 0, s>>>(W.test_off.p, W.test_items.p, W.neg_off.p, W.neg_items.p, emb_mask ? W.mask.p : nullptr, W.shot_off.p,
                                           U, true, W.count.p, nullptr, nullptr);
        GB_LAUNCHED(ctx);
    }
    if ((e = cudaMemcpyAsync(hc.data(), W.count.p, sizeof(int32_t) * (size_t)U, cudaMemcpyDeviceToHost, s)) != cudaSuccess ||
        (e = cudaStreamSynchronize(s)) != cudaSuccess)
        return cuda_fail(e);

    // the users the reference scores have a candidate and a shot with an embedding; the others get an empty test row
    std::vector<int64_t> coff((size_t)U + 1, 0), rt_off((size_t)U + 1, 0), tile_off((size_t)U + 1, 0), pair_base((size_t)U + 1, 0);
    std::vector<int32_t> rt_items;
    for (int32_t u = 0; u < U; u++) {
        const int64_t m = hc[(size_t)u], k = vs_off[(size_t)u + 1] - vs_off[(size_t)u];
        coff[(size_t)u + 1] = coff[(size_t)u] + m;
        if (m > 0) rt_items.insert(rt_items.end(), test_items + toff[(size_t)u], test_items + toff[(size_t)u + 1]);
        rt_off[(size_t)u + 1] = (int64_t)rt_items.size();
        tile_off[(size_t)u + 1] = tile_off[(size_t)u] + (m > 0 ? (((m + 3) / 4) * ((k + 3) / 4) + MT - 1) / MT : 0);
        pair_base[(size_t)u + 1] = pair_base[(size_t)u] + (m > 0 ? m * k : 0);
    }
    GB_TRY(upload(W.cand_off, coff.data(), (size_t)U + 1, s));
    GB_TRY(W.cand_items.alloc(std::max<size_t>((size_t)coff[(size_t)U], 1)));
    GB_TRY(W.score.alloc(std::max<size_t>((size_t)coff[(size_t)U], 1)));
    GB_TRY(upload(W.rt_off, rt_off.data(), (size_t)U + 1, s));
    GB_TRY(upload(W.rt_items, rt_items.data(), rt_items.size(), s));
    GB_TRY(upload(W.tile_off, tile_off.data(), (size_t)U + 1, s));
    GB_TRY(upload(W.pair_base, pair_base.data(), (size_t)U + 1, s));
    if (U > 0) {
        emb_cand_kernel<<<ub, 128, 0, s>>>(W.test_off.p, W.test_items.p, W.neg_off.p, W.neg_items.p, emb_mask ? W.mask.p : nullptr, W.shot_off.p,
                                           U, false, nullptr, W.cand_off.p, W.cand_items.p);
        GB_LAUNCHED(ctx);
    }

    // users in chunks of at most CHUNK_PAIRS distances (or one user's); GORSE_B200_EMBEDDING_EVAL_CHUNK_PAIRS lowers the cap
    int64_t cap = CHUNK_PAIRS;
    if (const char *env = getenv("GORSE_B200_EMBEDDING_EVAL_CHUNK_PAIRS")) {
        const long long v = atoll(env);
        if (v > 0 && v < cap) cap = v;
    }
    int64_t biggest = 0;
    for (int32_t u = 0; u < U; u++) biggest = std::max(biggest, pair_base[(size_t)u + 1] - pair_base[(size_t)u]);
    GB_TRY(W.dist.alloc((size_t)std::max<int64_t>(1, std::min(pair_base[(size_t)U], std::max(cap, biggest)))));
    for (int32_t u0 = 0; u0 < U;) {
        int32_t u1 = u0 + 1;
        while (u1 < U && pair_base[(size_t)u1 + 1] - pair_base[(size_t)u0] <= cap) u1++;
        const int64_t tiles = tile_off[(size_t)u1] - tile_off[(size_t)u0];
        if (tiles > 0) {
            if (dim % 4 == 0)
                emb_dist_kernel<true><<<(unsigned)tiles, THREADS, 0, s>>>(W.emb.p, dim, W.cand_off.p + u0, W.cand_items.p, W.shot_off.p + u0,
                                                                          W.shot_items.p, W.tile_off.p + u0, W.pair_base.p + u0, u1 - u0, W.dist.p);
            else
                emb_dist_kernel<false><<<(unsigned)tiles, THREADS, 0, s>>>(W.emb.p, dim, W.cand_off.p + u0, W.cand_items.p, W.shot_off.p + u0,
                                                                           W.shot_items.p, W.tile_off.p + u0, W.pair_base.p + u0, u1 - u0, W.dist.p);
            GB_LAUNCHED(ctx);
            emb_total_kernel<<<u1 - u0, 128, 0, s>>>(W.cand_off.p + u0, W.shot_off.p + u0, W.pair_base.p + u0, W.dist.p, W.score.p);
            GB_LAUNCHED(ctx);
        }
        u0 = u1;
    }

    std::vector<float> inv((size_t)topk);
    eval_inv_log2(topk, inv.data());
    GB_TRY(upload(W.inv, inv.data(), (size_t)topk, s));
    GB_TRY(W.metrics.alloc((size_t)4 * std::max(U, 1)));
    launch_eval_rank(s, W.cand_off.p, W.cand_items.p, W.score.p, W.rt_off.p, W.rt_items.p, U, topk, W.inv.p, W.metrics.p);
    GB_LAUNCHED(ctx);
    std::vector<float> hm((size_t)4 * U);
    if ((U > 0 && (e = cudaMemcpyAsync(hm.data(), W.metrics.p, sizeof(float) * 4 * (size_t)U, cudaMemcpyDeviceToHost, s)) != cudaSuccess) ||
        (e = cudaStreamSynchronize(s)) != cudaSuccess)
        return cuda_fail(e);
    // main.go:452-465 with jobs = 1: fp32 sums in user order, each divided by the count; no scored user gives a zero score
    volatile float sum0 = 0.f, sum1 = 0.f, sum2 = 0.f, count = 0.f;
    int64_t users = 0;
    for (int32_t u = 0; u < U; u++) {
        const float *mu = hm.data() + 4 * (size_t)u;
        if (mu[3] != 0.f) {
            sum0 = sum0 + mu[0]; sum1 = sum1 + mu[1]; sum2 = sum2 + mu[2]; count = count + 1.0f;
            users++;
        }
    }
    out[0] = out[1] = out[2] = 0.f;
    if (count > 0.f) { out[0] = sum0 / count; out[1] = sum1 / count; out[2] = sum2 / count; }
    if (users_out) *users_out = users;
    return GORSE_B200_OK;
}
