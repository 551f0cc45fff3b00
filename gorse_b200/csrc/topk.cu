// topk.cu -- brute-force vector index: ann.Bruteforce (common/ann/bruteforce.go:24-83) behind ann.Index.
//
// Two stages share one result contract (k smallest distances, ascending; ties broken by ascending index --
// the reference's tie order is an artefact of Go's container/heap and is not pinned by any reference test):
//   stage 1  candidate generation.  Small problems: exact scan (this file).  Large d % 16 == 0 problems:
//            bf16 wgmma GEMM with a fused threshold filter (topk_mma.cu), which over-fetches by a rigorous
//            error margin so the true top-k is always among the candidates.
//   stage 2  exact re-rank of the candidates with the reference's fp32 summation order
//            (floats.Euclidean / -floats.Dot, AVX-512 tree), final sort, prune0.
#include <algorithm>
#include <cmath>

#include "cf.cuh"
#include "topk.cuh"

namespace gb {

// (dist, idx) ordering used everywhere: ascending distance, then ascending index
__device__ __forceinline__ bool before(float da, int32_t ia, float db, int32_t ib) { return da < db || (da == db && ia < ib); }

// sorted insertion into a warp-private list kept in shared memory (lane 0 only); list holds <= k entries
__device__ __forceinline__ void list_insert(float *ld, int32_t *li, int &len, int k, float dv, int32_t iv)
{
    if (len == k && !before(dv, iv, ld[k - 1], li[k - 1])) return;
    int pos = len < k ? len : k - 1;
    while (pos > 0 && before(dv, iv, ld[pos - 1], li[pos - 1])) {
        ld[pos] = ld[pos - 1];
        li[pos] = li[pos - 1];
        pos--;
    }
    ld[pos] = dv;
    li[pos] = iv;
    if (len < k) len++;
}

// the same insertion done by the whole warp: every lane owns list slots lane, lane+32, ...; the position is a ballot count
// and the shift is one read + one write per owned slot.  All arguments are warp-uniform; len lives in every lane.
__device__ __forceinline__ void list_insert_warp(float *ld, int32_t *li, int &len, int k, float dv, int32_t iv, int lane)
{
    if (len == k && !before(dv, iv, ld[k - 1], li[k - 1])) return;
    const int n = len;
    float od[4];
    int32_t oi[4];
    int pos = 0;
#pragma unroll
    for (int r = 0; r < 4; r++) {
        const int e = lane + 32 * r;
        const bool has = e < n;
        od[r] = has ? ld[e] : 0.f;
        oi[r] = has ? li[e] : 0;
        pos += __popc(__ballot_sync(0xffffffffu, has && before(od[r], oi[r], dv, iv)));
    }
    __syncwarp();
#pragma unroll
    for (int r = 0; r < 4; r++) {
        const int e = lane + 32 * r;
        if (e < n && e >= pos && e + 1 < k) { ld[e + 1] = od[r]; li[e + 1] = oi[r]; }
    }
    if (lane == 0) { ld[pos] = dv; li[pos] = iv; }
    if (len < k) len++;
    __syncwarp();
}

// Exact scan: one warp per query over vectors [0, N) or over a candidate list.
//   queries:   nq rows of d floats (q_ptr), or rows of X selected by q_idx when q_ptr == nullptr
//   self skip: SearchIndex never returns q itself (bruteforce.go:47)
//   cand:      optional candidate lists [nq][cand_stride] (idx < 0 = empty slot) -> stage-2 re-rank
__global__ void __launch_bounds__(128)
topk_exact_kernel(const float *X, int64_t N, int d, int metric, const float *q_ptr, const int64_t *q_idx, int64_t q0,
                  int64_t nq, int k, const int32_t *cand, const int32_t *cand_count, int cand_stride, const int32_t *row_list,
                  int32_t *out_idx, float *out_dist, int32_t *out_count, int prune0, int *nan_flag, int n_seg, int64_t seg_len,
                  int cand_by_slot, const uint8_t *allow /* optional per-vector filter (vecdb.cu): 0 = never returned */)
{
    extern __shared__ unsigned char sm_raw[];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
    float *ld = reinterpret_cast<float *>(sm_raw) + (size_t)wid * k;
    int32_t *li = reinterpret_cast<int32_t *>(reinterpret_cast<float *>(sm_raw) + (size_t)nw * k) + (size_t)wid * k;
    float *qs = reinterpret_cast<float *>(sm_raw) + (size_t)2 * nw * k + (size_t)wid * d;
    const int lane4 = lane & 3, quad = lane >> 2;
    const unsigned qmask = quad_mask();
    // nq counts work slots: slot = (row_slot, segment).  With n_seg > 1 every slot scans one segment of the vectors and
    // writes its own partial top-k at out[slot]; a second pass merges the partial lists (cand_by_slot) into out[row].
    for (int64_t slot = (int64_t)blockIdx.x * nw + wid; slot < nq; slot += (int64_t)gridDim.x * nw) {
        const int64_t row_slot = slot / n_seg;
        const int seg = (int)(slot % n_seg);
        const int64_t qi = row_list ? (int64_t)row_list[row_slot] : row_slot;
        const int64_t oq = n_seg > 1 ? slot : qi;
        int64_t self = -1;
        const float *qsrc;
        if (q_ptr) qsrc = q_ptr + qi * d;
        else { self = q_idx ? q_idx[qi] : q0 + qi; qsrc = X + self * d; }
        for (int e = lane; e < d; e += 32) qs[e] = qsrc[e];
        __syncwarp();
        const float qq = metric == GORSE_B200_METRIC_COSINE ? dot_any(qs, qs, d) : 0.f;
        int len = 0;
        const int64_t cidx = cand_by_slot ? row_slot : qi;
        const int32_t *cl = cand ? cand + cidx * cand_stride : nullptr;
        const int64_t begin = cand ? 0 : (int64_t)seg * seg_len;
        const int64_t total = cand ? (cand_count ? (int64_t)min(cand_count[cidx], cand_stride) : (int64_t)cand_stride) : min(N, begin + seg_len);
        if (d % 16 == 0 && d <= 256) {
            const int chunks = d / 16;
            float4 qreg[16];
#pragma unroll
            for (int c = 0; c < 16; c++)
                if (c < chunks) qreg[c] = *reinterpret_cast<const float4 *>(qs + 16 * c + 4 * lane4);
            for (int64_t base = begin; base < total; base += 8) {
                int64_t t = base + quad;
                int64_t v = -1;
                if (t < total) v = cl ? (int64_t)cl[t] : t;
                bool valid = v >= 0 && v != self && (allow == nullptr || allow[v] != 0);
                float dv = 0.f;
                if (valid) dv = quad_dist(qreg, X + v * d, chunks, lane4, qmask, metric, qq);
                // lane 0 consumes the 8 quads' results in index order
                for (int s = 0; s < 8; s++) {
                    float dd = __shfl_sync(0xffffffffu, dv, 4 * s);
                    int64_t vv = __shfl_sync(0xffffffffu, v, 4 * s);
                    int ok = __shfl_sync(0xffffffffu, (int)valid, 4 * s);
                    if (ok) {
                        if (dd != dd) { if (lane == 0) *nan_flag = 1; }
                        else if (k <= 128) list_insert_warp(ld, li, len, k, dd, (int32_t)vv, lane);
                        else if (lane == 0) list_insert(ld, li, len, k, dd, (int32_t)vv);
                    }
                }
                __syncwarp();
            }
        } else {
            for (int64_t base = begin; base < total; base += 32) {
                int64_t t = base + lane;
                int64_t v = -1;
                if (t < total) v = cl ? (int64_t)cl[t] : t;
                bool valid = v >= 0 && v != self && (allow == nullptr || allow[v] != 0);
                float dv = 0.f;
                if (valid) dv = dist_any(qs, X + v * d, d, metric, qq);
                for (int s = 0; s < 32; s++) {
                    float dd = __shfl_sync(0xffffffffu, dv, s);
                    int64_t vv = __shfl_sync(0xffffffffu, v, s);
                    int ok = __shfl_sync(0xffffffffu, (int)valid, s);
                    if (ok) {
                        if (dd != dd) { if (lane == 0) *nan_flag = 1; }
                        else if (k <= 128) list_insert_warp(ld, li, len, k, dd, (int32_t)vv, lane);
                        else if (lane == 0) list_insert(ld, li, len, k, dd, (int32_t)vv);
                    }
                }
                __syncwarp();
            }
        }
        len = __shfl_sync(0xffffffffu, len, 0);
        __syncwarp();
        // prune0 keeps score > 0 while popping (bruteforce.go:58,78); the list is ascending so survivors are a suffix
        int first = 0;
        if (prune0) {
            while (first < len && !(ld[first] > 0.f)) first++;
        }
        int cnt = len - first;
        for (int e = lane; e < k; e += 32) {
            bool has = e < cnt;
            out_idx[oq * k + e] = has ? li[first + e] : -1;
            out_dist[oq * k + e] = has ? ld[first + e] : 0.f;
        }
        if (lane == 0) out_count[oq] = cnt;
        __syncwarp();
    }
}

int32_t launch_exact(gorse_b200_index *ix, const float *d_q, const int64_t *d_qidx, int64_t q0, int64_t nq, int k,
                     const int32_t *d_cand, const int32_t *d_cand_count, int cand_stride, const int32_t *row_list,
                     int32_t *d_idx, float *d_dist, int32_t *d_count, int prune0, int *d_nan)
{
    gorse_b200_ctx *c = ix->ctx;
    const int warps = 4;
    size_t sm = (size_t)warps * (2 * (size_t)k * 4 + (size_t)ix->d * 4);
    if (sm > 200 * 1024) { set_error("k = %d with dim = %d needs %zu bytes of shared memory per CTA", k, ix->d, sm); return GORSE_B200_ERR_UNSUPPORTED; }
    GB_CUDA(cudaFuncSetAttribute(topk_exact_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    int grid = (int)std::max<int64_t>(1, std::min<int64_t>((nq + warps - 1) / warps, (int64_t)c->sm_count * 8));
    topk_exact_kernel<<<grid, 32 * warps, sm, c->stream>>>(ix->X.p, ix->n, ix->d, ix->metric, d_q, d_qidx, q0, nq, k, d_cand,
                                                         d_cand_count, cand_stride, row_list, d_idx, d_dist, d_count, prune0, d_nan, 1, ix->n, 0, nullptr);
    GB_LAUNCHED(c);
    return GORSE_B200_OK;
}

// A few rows, each against ALL vectors (the tensor path's certified-fallback): split every row's scan into segments
// handled by different warps (partial top-k per segment, no prune0 yet), then merge the partial lists exactly.
int32_t launch_exact_split(gorse_b200_index *ix, const float *d_q, const int64_t *d_qidx, int64_t q0, int32_t n_rows, int k,
                           const int32_t *row_list, int32_t *d_idx, float *d_dist, int32_t *d_count, int prune0, int *d_nan,
                           const uint8_t *allow)
{
    gorse_b200_ctx *c = ix->ctx;
    const int warps = 4;
    size_t sm = (size_t)warps * (2 * (size_t)k * 4 + (size_t)ix->d * 4);
    // (round 2 tried finer segments to fill the machine with a handful of rows: the scan got faster but the merge, one
    // warp re-scoring n_seg * k candidates per row, took 4x longer than what was saved)
    const int64_t seg_len = 16384;
    const int n_seg = (int)((ix->n + seg_len - 1) / seg_len);
    DevBuf<int32_t> p_idx, p_cnt;
    DevBuf<float> p_dist;
    int32_t st;
    auto done = [&](int32_t s) { cudaStreamSynchronize(c->stream); p_idx.free(); p_cnt.free(); p_dist.free(); return s; };
    const int64_t slots = (int64_t)n_rows * n_seg;
    if ((st = p_idx.alloc((size_t)slots * k)) || (st = p_dist.alloc((size_t)slots * k)) || (st = p_cnt.alloc(slots))) return done(st);
    GB_CUDA(cudaFuncSetAttribute(topk_exact_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    int grid = (int)std::max<int64_t>(1, std::min<int64_t>((slots + warps - 1) / warps, (int64_t)c->sm_count * 16));
    topk_exact_kernel<<<grid, 32 * warps, sm, c->stream>>>(ix->X.p, ix->n, ix->d, ix->metric, d_q, d_qidx, q0, slots, k, nullptr, nullptr, 0,
                                                         row_list, p_idx.p, p_dist.p, p_cnt.p, 0, d_nan, n_seg, seg_len, 0, allow);
    c->launches++;
    grid = (int)std::max<int64_t>(1, std::min<int64_t>((n_rows + warps - 1) / warps, (int64_t)c->sm_count * 8));
    topk_exact_kernel<<<grid, 32 * warps, sm, c->stream>>>(ix->X.p, ix->n, ix->d, ix->metric, d_q, d_qidx, q0, n_rows, k, p_idx.p, nullptr,
                                                         n_seg * k, row_list, d_idx, d_dist, d_count, prune0, d_nan, 1, ix->n, 1, nullptr);
    c->launches++;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("exact fallback: %s", cudaGetErrorString(e)); return done(GORSE_B200_ERR_CUDA); }
    return done(GORSE_B200_OK);
}

// run a search whose queries are already described by (d_q | d_qidx | q0); copies results to the host
static int32_t search_common(gorse_b200_index *ix, const float *h_queries, const int64_t *h_qidx, int64_t q0, int64_t nq,
                             int32_t k, int32_t prune0, int32_t *idx_out, float *dist_out, int32_t *count_out)
{
    GB_CHECK_ARG(k >= 0, "negative k");
    GB_CHECK_ARG(nq >= 0, "negative query count");
    if (nq == 0) return GORSE_B200_OK;
    GB_CHECK_ARG(count_out != nullptr, "count_out is NULL");
    if (k == 0 || ix->n == 0) {
        for (int64_t i = 0; i < nq; i++) count_out[i] = 0;
        return GORSE_B200_OK;
    }
    GB_CHECK_ARG(idx_out != nullptr && dist_out != nullptr, "NULL output");
    ScopedDevice sd(ix->ctx->device);
    gorse_b200_ctx *c = ix->ctx;
    DevBuf<float> d_q;
    DevBuf<int64_t> d_qidx;
    DevBuf<int> d_nan;
    DevBuf<int32_t> &d_idx = ix->r_idx, &d_count = ix->r_count;   // grow-only staging kept in the index
    DevBuf<float> &d_dist = ix->r_dist;
    int32_t st = GORSE_B200_OK;
    auto done = [&](int32_t s) {
        cudaStreamSynchronize(c->stream);
        cudaStreamSynchronize(c->copy_stream);
        d_q.free(); d_qidx.free(); d_nan.free();
        return s;
    };
    if ((d_idx.n < (size_t)nq * k && (st = d_idx.alloc((size_t)nq * k))) || (d_dist.n < (size_t)nq * k && (st = d_dist.alloc((size_t)nq * k))) ||
        (d_count.n < (size_t)nq && (st = d_count.alloc(nq))) || (st = d_nan.alloc(1)))
        return done(st);
    cudaError_t e = cudaMemsetAsync(d_nan.p, 0, sizeof(int), c->stream);
    if (h_queries) {
        if ((st = d_q.alloc((size_t)nq * ix->d))) return done(st);
        if (e == cudaSuccess) e = cudaMemcpyAsync(d_q.p, h_queries, sizeof(float) * nq * ix->d, cudaMemcpyHostToDevice, c->stream);
    } else if (h_qidx) {
        if ((st = d_qidx.alloc(nq))) return done(st);
        if (e == cudaSuccess) e = cudaMemcpyAsync(d_qidx.p, h_qidx, sizeof(int64_t) * nq, cudaMemcpyHostToDevice, c->stream);
    }
    if (e != cudaSuccess) { set_error("search upload: %s", cudaGetErrorString(e)); return done(GORSE_B200_ERR_CUDA); }
    // large all-pairs / batched problems go through the tensor-core candidate generator + exact re-rank
    bool downloaded = false;
    if (mma_path_eligible(ix, nq, k)) {
        st = search_mma(ix, d_q.p, d_qidx.p, q0, nq, k, prune0, d_idx.p, d_dist.p, d_count.p, d_nan.p, idx_out, dist_out, count_out);
        downloaded = true;
    } else {
        st = launch_exact(ix, d_q.p, d_qidx.p, q0, nq, k, nullptr, nullptr, 0, nullptr, d_idx.p, d_dist.p, d_count.p, prune0, d_nan.p);
    }
    if (st) return done(st);
    int h_nan = 0;
    if ((!downloaded && ((e = cudaMemcpyAsync(idx_out, d_idx.p, sizeof(int32_t) * nq * k, cudaMemcpyDeviceToHost, c->stream)) != cudaSuccess ||
                         (e = cudaMemcpyAsync(dist_out, d_dist.p, sizeof(float) * nq * k, cudaMemcpyDeviceToHost, c->stream)) != cudaSuccess ||
                         (e = cudaMemcpyAsync(count_out, d_count.p, sizeof(int32_t) * nq, cudaMemcpyDeviceToHost, c->stream)) != cudaSuccess)) ||
        (e = cudaMemcpyAsync(&h_nan, d_nan.p, sizeof(int), cudaMemcpyDeviceToHost, c->stream)) != cudaSuccess ||
        (e = cudaStreamSynchronize(c->stream)) != cudaSuccess || (e = cudaStreamSynchronize(c->copy_stream)) != cudaSuccess) {
        set_error("search: %s", cudaGetErrorString(e));
        return done(GORSE_B200_ERR_CUDA);
    }
    if (h_nan) { set_error("NaN weight is forbidden");  /* the reference panics, common/heap/pq.go:82-83 */ return done(GORSE_B200_ERR_ARG); }
    return done(GORSE_B200_OK);
}

// make room for `need` vectors (amortised doubling); the caller holds ix->mu
int32_t index_reserve(gorse_b200_index *ix, int64_t need)
{
    if (need <= ix->cap) return GORSE_B200_OK;
    cudaStream_t s = ix->ctx->stream;
    const int64_t ncap = std::max<int64_t>(need, ix->cap * 2);
    DevBuf<float> nb;
    GB_TRY(nb.alloc((size_t)ncap * ix->d));
    if (ix->n) GB_CUDA(cudaMemcpyAsync(nb.p, ix->X.p, sizeof(float) * ix->n * ix->d, cudaMemcpyDeviceToDevice, s));
    GB_CUDA(cudaStreamSynchronize(s));
    ix->X.free();
    ix->X = nb;
    ix->cap = ncap;
    return GORSE_B200_OK;
}

}  // namespace gb

using namespace gb;

extern "C" {

int32_t gorse_b200_index_create(gorse_b200_ctx *ctx, int32_t dim, int32_t metric, gorse_b200_index **out)
{
    GB_CHECK_ARG(ctx != nullptr && out != nullptr, "NULL ctx/out");
    *out = nullptr;
    GB_CHECK_ARG(dim >= 1 && dim <= 16384, "dim %d out of range", dim);
    GB_CHECK_ARG(metric == GORSE_B200_METRIC_EUCLIDEAN || metric == GORSE_B200_METRIC_NEG_DOT || metric == GORSE_B200_METRIC_COSINE,
                 "unknown metric %d", metric);
    gorse_b200_index *ix = new (std::nothrow) gorse_b200_index();
    if (!ix) { set_error("host allocation failed"); return GORSE_B200_ERR_OOM; }
    ix->ctx = ctx;
    ix->d = dim;
    ix->metric = metric;
    *out = ix;
    return GORSE_B200_OK;
}

int32_t gorse_b200_index_destroy(gorse_b200_index *ix)
{
    if (!ix) return GORSE_B200_OK;
    ScopedDevice sd(ix->ctx->device);
    cudaStreamSynchronize(ix->ctx->stream);
    ix->X.free();
    ix->Xb.free();
    ix->norm.free();
    ix->perm.free();
    if (ix->ev0) { cudaEventDestroy(ix->ev0); cudaEventDestroy(ix->ev1); }
    ix->w_qb.free(); ix->w_eps.free(); ix->w_cval.free(); ix->w_theta.free();
    ix->w_ccol.free(); ix->w_ccnt.free(); ix->w_ids.free(); ix->w_idcnt.free(); ix->w_flag.free(); ix->w_flist.free();
    ix->r_idx.free(); ix->r_count.free(); ix->r_dist.free();
    delete ix;
    return GORSE_B200_OK;
}

int32_t gorse_b200_index_add(gorse_b200_index *ix, const float *vectors, int64_t n, int64_t *count_out)
{
    GB_CHECK_ARG(ix != nullptr, "index is NULL");
    GB_CHECK_ARG(n >= 0, "negative n");
    std::lock_guard<std::mutex> lk(ix->mu);
    if (n > 0) {
        GB_CHECK_ARG(vectors != nullptr, "vectors is NULL");
        ScopedDevice sd(ix->ctx->device);
        cudaStream_t s = ix->ctx->stream;
        int64_t need = ix->n + n;
        GB_TRY(index_reserve(ix, need));
        GB_CUDA(cudaMemcpyAsync(ix->X.p + ix->n * ix->d, vectors, sizeof(float) * n * ix->d, cudaMemcpyHostToDevice, s));
        GB_CUDA(cudaStreamSynchronize(s));
        ix->n = need;
        ix->mma_ready = false;  // bf16 mirror and norms are rebuilt lazily
    }
    if (count_out) *count_out = ix->n;
    return GORSE_B200_OK;
}

int32_t gorse_b200_index_len(const gorse_b200_index *ix, int64_t *count_out)
{
    GB_CHECK_ARG(ix != nullptr && count_out != nullptr, "NULL argument");
    *count_out = ix->n;
    return GORSE_B200_OK;
}

int32_t gorse_b200_index_search_vectors(gorse_b200_index *ix, const float *queries, int64_t nq, int32_t k, int32_t prune0,
                                        int32_t *idx_out, float *dist_out, int32_t *count_out)
{
    GB_CHECK_ARG(ix != nullptr, "index is NULL");
    GB_CHECK_ARG(nq == 0 || queries != nullptr, "queries is NULL");
    std::lock_guard<std::mutex> lk(ix->mu);
    return search_common(ix, queries, nullptr, 0, nq, k, prune0, idx_out, dist_out, count_out);
}

int32_t gorse_b200_index_search_indices(gorse_b200_index *ix, const int64_t *q_idx, int64_t nq, int32_t k, int32_t prune0,
                                        int32_t *idx_out, float *dist_out, int32_t *count_out)
{
    GB_CHECK_ARG(ix != nullptr, "index is NULL");
    GB_CHECK_ARG(nq == 0 || q_idx != nullptr, "q_idx is NULL");
    std::lock_guard<std::mutex> lk(ix->mu);
    for (int64_t i = 0; i < nq; i++)
        if (q_idx[i] < 0 || q_idx[i] >= ix->n) {
            set_error("index out of range: %lld", (long long)q_idx[i]);  // bruteforce.go:41-43
            return GORSE_B200_ERR_RANGE;
        }
    return search_common(ix, nullptr, q_idx, 0, nq, k, prune0, idx_out, dist_out, count_out);
}

int32_t gorse_b200_index_search_range(gorse_b200_index *ix, int64_t q0, int64_t q1, int32_t k, int32_t prune0,
                                      int32_t *idx_out, float *dist_out, int32_t *count_out)
{
    GB_CHECK_ARG(ix != nullptr, "index is NULL");
    std::lock_guard<std::mutex> lk(ix->mu);
    if (q0 < 0 || q1 < q0 || q1 > ix->n) {
        set_error("index out of range: [%lld, %lld)", (long long)q0, (long long)q1);
        return GORSE_B200_ERR_RANGE;
    }
    return search_common(ix, nullptr, nullptr, q0, q1 - q0, k, prune0, idx_out, dist_out, count_out);
}

// ---- measurement / test hooks (declared in include/gorse_b200.h) ----------------------------------------
// since the last call: device time and algorithmic flop (2 * nq * N * d) of the stage-1 tensor-core kernel, and the rows
// that fell back to the exact scan
int32_t gorse_b200_index_stats(gorse_b200_index *ix, double *stage1_ms, double *stage1_flop, int64_t *fallback_rows)
{
    GB_CHECK_ARG(ix != nullptr, "ix is NULL");
    std::lock_guard<std::mutex> lk(ix->mu);
    if (stage1_ms) *stage1_ms = ix->stage1_ms;
    if (stage1_flop) *stage1_flop = ix->stage1_flop;
    if (fallback_rows) *fallback_rows = ix->last_fallback_rows;
    ix->stage1_ms = ix->stage1_flop = 0.0;
    ix->last_fallback_rows = 0;
    return GORSE_B200_OK;
}

// dense stage-1 (tensor core) scores of stored vectors [q0, q1) against all vectors, in ORIGINAL column order:
// out[(q - q0) * n + x], and (eps_out != NULL) each row's error margin eps.  Small problems only (one chunk of rows).
int32_t gorse_b200_index_stage1_scores(gorse_b200_index *ix, int64_t q0, int64_t q1, float *out, float *eps_out)
{
    GB_CHECK_ARG(ix != nullptr && out != nullptr, "NULL argument");
    std::lock_guard<std::mutex> lk(ix->mu);
    GB_CHECK_ARG(q0 >= 0 && q1 > q0 && q1 <= ix->n, "bad range");
    ScopedDevice sd(ix->ctx->device);
    gorse_b200_ctx *c = ix->ctx;
    const int64_t nq = q1 - q0, n_cols = (ix->n + 127) / 128 * 128;
    DevBuf<float> dense, d_dist;
    DevBuf<int32_t> d_idx, d_count;
    DevBuf<int> d_nan;
    int32_t st;
    auto done = [&](int32_t s) { cudaStreamSynchronize(c->stream); dense.free(); d_dist.free(); d_idx.free(); d_count.free(); d_nan.free(); ix->dbg_scores = nullptr; return s; };
    if ((st = dense.alloc((size_t)nq * n_cols)) || (st = d_idx.alloc(nq)) || (st = d_dist.alloc(nq)) || (st = d_count.alloc(nq)) || (st = d_nan.alloc(1))) return done(st);
    cudaMemsetAsync(d_nan.p, 0, sizeof(int), c->stream);
    ix->dbg_scores = dense.p;
    if ((st = search_mma(ix, nullptr, nullptr, q0, nq, 1, 0, d_idx.p, d_dist.p, d_count.p, d_nan.p))) return done(st);
    if (ix->w_cq < nq) { set_error("stage1_scores: %lld rows do not fit one sweep", (long long)nq); return done(GORSE_B200_ERR_ARG); }
    std::vector<float> h((size_t)nq * n_cols);
    std::vector<int32_t> perm((size_t)ix->n);
    cudaError_t e = cudaMemcpyAsync(h.data(), dense.p, sizeof(float) * h.size(), cudaMemcpyDeviceToHost, c->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(perm.data(), ix->perm.p, sizeof(int32_t) * perm.size(), cudaMemcpyDeviceToHost, c->stream);
    if (e == cudaSuccess && eps_out) e = cudaMemcpyAsync(eps_out, ix->w_eps.p, sizeof(float) * nq, cudaMemcpyDeviceToHost, c->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
    if (e != cudaSuccess) { set_error("debug scores: %s", cudaGetErrorString(e)); return done(GORSE_B200_ERR_CUDA); }
    for (int64_t r = 0; r < nq; r++)
        for (int64_t p = 0; p < ix->n; p++) out[r * ix->n + perm[p]] = h[r * n_cols + p];
    return done(GORSE_B200_OK);
}

}  // extern "C"
