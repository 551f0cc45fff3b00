// sparse.cu -- brute-force search over SPARSE vectors with the Dot metric: what logics.item_to_item / user_to_user of the
// types "tags", "users" and "auto" ask their vector store for (storage/vectors/xvec.go:244-248 flat sparse index, :405
// query; vectors built by appendSparseVector, logics/vector_writer.go:200-209).  SURVEY 8f-1, the row after the dense index.
//
// First hardware run in round 2 (tests/test_sparse_gpu.py green).  The arithmetic it must reproduce: merge-join dot of two
// sparse vectors summed in ascending index order, fp32, multiply and add unfused (the test suite's CPU restatement).
//
// Layout: the vectors as CSR (row -> ascending feature indices + values) and the same entries as CSC (feature -> ascending
// rows + values, the posting lists).  One warp answers one query row r:
//   1. for every feature f of r in ascending order: acc[c] += v_rf * v_cf over the posting list of f (the lanes take distinct
//      rows c, a __syncwarp orders the features) -- every candidate's dot is summed in ascending feature order, i.e. exactly
//      the merge-join order of the oracle, bit for bit;
//   2. one coalesced pass over the warp's private accumulator row acc[0..N): keep the k largest positive dots with the
//      warp-cooperative sorted list (order: dot descending, then row ascending) and reset the accumulator to zero.
// Only rows that share a feature with the query can have a non-zero dot; rows with dot <= 0 are never returned (the
// reference drops them right after the query, logics/item_to_item.go:73).  Roofline class: HBM/L2 (N floats scanned per query).
#include <algorithm>

#include <cub/cub.cuh>

#include "sparse.cuh"

using namespace gb;

namespace {

// (dist, idx) ordering of topk.cu: ascending distance (= descending dot), then ascending index
__device__ __forceinline__ bool before(float da, int32_t ia, float db, int32_t ib) { return da < db || (da == db && ia < ib); }

// topk.cu list_insert_warp: sorted insertion done by the whole warp; all arguments warp-uniform, k <= 128
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

template <bool ROW_LIST>
__global__ void __launch_bounds__(128)
sparse_search_kernel(const int64_t *off, const uint32_t *ind, const float *val, const int64_t *foff, const int32_t *frow,
                     const float *fval, int64_t N, uint32_t n_features, int64_t q0, int64_t nq, int k, float *acc, int32_t *out_idx,
                     float *out_dot, int32_t *out_count, const int64_t *q_off, const uint32_t *q_ind, const float *q_val,
                     const uint8_t *allow, const int64_t *q_rows)
{
    // queries: stored rows q0 + q, or q_rows[q] with ROW_LIST (a device list, item_to_item.cu) -- never returned themselves --
    // or, q_off != nullptr, rows of an external CSR (vecdb.cu: QueryVectors passes the vector, not its id); allow: optional
    // per-row filter
    extern __shared__ unsigned char sm_raw[];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
    float *ld = reinterpret_cast<float *>(sm_raw) + (size_t)wid * k;
    int32_t *li = reinterpret_cast<int32_t *>(reinterpret_cast<float *>(sm_raw) + (size_t)nw * k) + (size_t)wid * k;
    float *a = acc + ((int64_t)blockIdx.x * nw + wid) * N;   // this warp's accumulator row, all zero between queries
    for (int64_t q = (int64_t)blockIdx.x * nw + wid; q < nq; q += (int64_t)gridDim.x * nw) {
        const int64_t row = q_off ? -1 : ROW_LIST ? q_rows[q] : q0 + q;
        const int64_t tb = q_off ? q_off[q] : off[row], te = q_off ? q_off[q + 1] : off[row + 1];
        const uint32_t *qi = q_off ? q_ind : ind;
        const float *qv = q_off ? q_val : val;
        for (int64_t t = tb; t < te; t++) {
            const uint32_t f = qi[t];
            const float v = qv[t];
            if (f >= n_features) continue;   // a feature no stored vector has (warp-uniform)
            for (int64_t p = foff[f] + lane; p < foff[f + 1]; p += 32) {
                const int32_t c = frow[p];
                a[c] = a[c] + v * fval[p];        // unfused multiply and add, like the oracle (-fmad=false)
            }
            __syncwarp();
        }
        int len = 0;
        for (int64_t base = 0; base < N; base += 32) {
            const int64_t c = base + lane;
            float x = 0.f;
            if (c < N) {
                x = a[c];
                if (x != 0.f) a[c] = 0.f;
            }
            const bool valid = c < N && c != row && x > 0.f && (allow == nullptr || allow[c] != 0);
            // cheap pre-filter against the current k-th best before the warp-wide insertion
            const bool cand = valid && (len < k || before(-x, (int32_t)c, ld[k - 1], li[k - 1]));
            unsigned m = __ballot_sync(0xffffffffu, cand);
            while (m) {
                const int s = __ffs(m) - 1;
                m &= m - 1;
                const float dd = __shfl_sync(0xffffffffu, -x, s);
                const int32_t vv = (int32_t)(base + s);
                list_insert_warp(ld, li, len, k, dd, vv, lane);
            }
        }
        __syncwarp();
        for (int e = lane; e < k; e += 32) {
            const bool has = e < len;
            out_idx[q * k + e] = has ? li[e] : -1;
            out_dot[q * k + e] = has ? -ld[e] : 0.f;
        }
        if (lane == 0) out_count[q] = len;
        __syncwarp();
    }
}

int32_t sync_device(gorse_b200_sparse_index *ix)
{
    if (!ix->dirty) return GORSE_B200_OK;
    gorse_b200_ctx *c = ix->ctx;
    const int64_t n = (int64_t)ix->h_off.size() - 1, nnz = (int64_t)ix->h_ind.size();
    // CSC by counting sort: postings of a feature in ascending row order
    std::vector<int64_t> foff((size_t)ix->n_features + 1, 0);
    for (int64_t t = 0; t < nnz; t++) foff[(size_t)ix->h_ind[(size_t)t] + 1]++;
    for (size_t f = 0; f < ix->n_features; f++) foff[f + 1] += foff[f];
    std::vector<int64_t> cur(foff.begin(), foff.end() - 1);
    std::vector<int32_t> frow((size_t)nnz);
    std::vector<float> fval((size_t)nnz);
    for (int64_t r = 0; r < n; r++)
        for (int64_t t = ix->h_off[(size_t)r]; t < ix->h_off[(size_t)r + 1]; t++) {
            const int64_t p = cur[ix->h_ind[(size_t)t]]++;
            frow[(size_t)p] = (int32_t)r;
            fval[(size_t)p] = ix->h_val[(size_t)t];
        }
    GB_TRY(ix->off.alloc((size_t)n + 1));
    GB_TRY(ix->foff.alloc(foff.size()));
    GB_TRY(ix->ind.alloc((size_t)nnz));
    GB_TRY(ix->val.alloc((size_t)nnz));
    GB_TRY(ix->frow.alloc((size_t)nnz));
    GB_TRY(ix->fval.alloc((size_t)nnz));
    cudaStream_t s = c->stream;
    GB_CUDA(cudaMemcpyAsync(ix->off.p, ix->h_off.data(), sizeof(int64_t) * ((size_t)n + 1), cudaMemcpyHostToDevice, s));
    GB_CUDA(cudaMemcpyAsync(ix->foff.p, foff.data(), sizeof(int64_t) * foff.size(), cudaMemcpyHostToDevice, s));
    if (nnz) {
        GB_CUDA(cudaMemcpyAsync(ix->ind.p, ix->h_ind.data(), sizeof(uint32_t) * (size_t)nnz, cudaMemcpyHostToDevice, s));
        GB_CUDA(cudaMemcpyAsync(ix->val.p, ix->h_val.data(), sizeof(float) * (size_t)nnz, cudaMemcpyHostToDevice, s));
        GB_CUDA(cudaMemcpyAsync(ix->frow.p, frow.data(), sizeof(int32_t) * (size_t)nnz, cudaMemcpyHostToDevice, s));
        GB_CUDA(cudaMemcpyAsync(ix->fval.p, fval.data(), sizeof(float) * (size_t)nnz, cudaMemcpyHostToDevice, s));
    }
    GB_CUDA(cudaStreamSynchronize(s));   // the staging vectors die here
    ix->acc.free();                      // sized for the old N
    ix->acc_slots = 0;
    ix->dirty = false;
    return GORSE_B200_OK;
}

// ---- compaction (sparse_compact): `scan` is the exclusive sum of the rows' live flags, row r is live iff scan[r + 1] != scan[r]
// keep[t] = 1 for the CSR entries of live rows, keep[nnz] = 0; one warp per row
__global__ void sparse_row_keep_kernel(const int64_t *off, int64_t n, const int64_t *scan, int64_t *keep)
{
    const int lane = threadIdx.x & 31;
    const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < n; r += nw) {
        const int64_t k = scan[r + 1] != scan[r];
        for (int64_t t = off[r] + lane; t < off[r + 1]; t += 32) keep[t] = k;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) keep[off[n]] = 0;
}
// keep[p] = 1 for the CSC entries whose row is live, keep[nnz] = 0
__global__ void sparse_col_keep_kernel(const int32_t *frow, int64_t nnz, const int64_t *scan, int64_t *keep)
{
    const int64_t st = (int64_t)gridDim.x * blockDim.x;
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p <= nnz; p += st)
        keep[p] = p < nnz && scan[frow[p] + 1] != scan[frow[p]];
}
// entries are grouped by row (by feature), so a list's new offset is the entry scan read at its old one:
// off'[scan[r]] = e_scan[off[r]] for live r and off'[live] = e_scan[nnz]; rows == nullptr: every list is kept, out[i] = e_scan[in[i]]
__global__ void sparse_compact_off_kernel(const int64_t *in, int64_t m, const int64_t *rows, const int64_t *e_scan, int64_t *out)
{
    const int64_t st = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i <= m; i += st) {
        if (!rows) out[i] = e_scan[in[i]];
        else if (i == m) out[rows[m]] = e_scan[in[m]];
        else if (rows[i + 1] != rows[i]) out[rows[i]] = e_scan[in[i]];
    }
}
// the kept entries to their scanned positions; CSC rows are renamed through the row scan (monotone: lists stay ascending)
__global__ void sparse_compact_csr_kernel(const uint32_t *ind, const float *val, int64_t nnz, const int64_t *e_scan, uint32_t *ind_n, float *val_n)
{
    const int64_t st = (int64_t)gridDim.x * blockDim.x;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < nnz; t += st) {
        const int64_t to = e_scan[t];
        if (e_scan[t + 1] != to) { ind_n[to] = ind[t]; val_n[to] = val[t]; }
    }
}
__global__ void sparse_compact_csc_kernel(const int32_t *frow, const float *fval, int64_t nnz, const int64_t *e_scan, const int64_t *scan,
                                          int32_t *frow_n, float *fval_n)
{
    const int64_t st = (int64_t)gridDim.x * blockDim.x;
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < nnz; p += st) {
        const int64_t to = e_scan[p];
        if (e_scan[p + 1] != to) { frow_n[to] = (int32_t)scan[frow[p]]; fval_n[to] = fval[p]; }
    }
}

}  // namespace

extern "C" {

int32_t gorse_b200_sparse_index_create(gorse_b200_ctx *ctx, gorse_b200_sparse_index **out)
{
    GB_CHECK_ARG(ctx != nullptr && out != nullptr, "NULL argument");
    gorse_b200_sparse_index *ix = new gorse_b200_sparse_index();
    ix->ctx = ctx;
    *out = ix;
    return GORSE_B200_OK;
}

int32_t gorse_b200_sparse_index_destroy(gorse_b200_sparse_index *ix)
{
    if (!ix) return GORSE_B200_OK;
    {
        ScopedDevice sd(ix->ctx->device);
        cudaStreamSynchronize(ix->ctx->stream);
        ix->off.free(); ix->foff.free(); ix->ind.free(); ix->val.free(); ix->frow.free(); ix->fval.free(); ix->acc.free();
    }
    delete ix;
    return GORSE_B200_OK;
}

int32_t gorse_b200_sparse_index_add(gorse_b200_sparse_index *ix, const int64_t *off, const uint32_t *indices, const float *values,
                                    int64_t n, int64_t *count_out)
{
    GB_CHECK_ARG(ix != nullptr, "index is NULL");
    GB_CHECK_ARG(n >= 0, "negative n");
    std::lock_guard<std::mutex> lk(ix->mu);
    if (n > 0) {
        GB_CHECK_ARG(off != nullptr, "off is NULL");
        GB_CHECK_ARG(off[0] == 0, "off[0] must be 0");
        for (int64_t r = 0; r < n; r++) {
            GB_CHECK_ARG(off[r + 1] >= off[r], "offsets must not decrease (row %lld)", (long long)r);
            for (int64_t t = off[r]; t < off[r + 1]; t++) {
                GB_CHECK_ARG(indices != nullptr && values != nullptr, "NULL indices/values");
                GB_CHECK_ARG(t == off[r] || indices[t] > indices[t - 1], "indices of row %lld are not strictly ascending", (long long)r);
                GB_CHECK_ARG(values[t] == values[t], "NaN value in row %lld", (long long)r);
                GB_CHECK_ARG(indices[t] < 0x7fffffffu, "feature index too large");
            }
        }
        if ((int64_t)ix->h_off.size() - 1 + n >= (1ll << 31)) { set_error("more than 2^31 vectors"); return GORSE_B200_ERR_UNSUPPORTED; }
        const int64_t base = ix->h_off.back();
        for (int64_t r = 0; r < n; r++) ix->h_off.push_back(base + off[r + 1]);
        ix->h_ind.insert(ix->h_ind.end(), indices, indices + off[n]);
        ix->h_val.insert(ix->h_val.end(), values, values + off[n]);
        for (int64_t t = 0; t < off[n]; t++) ix->n_features = std::max(ix->n_features, indices[t] + 1);
        ix->dirty = true;
    }
    if (count_out) *count_out = (int64_t)ix->h_off.size() - 1;
    return GORSE_B200_OK;
}

int32_t gorse_b200_sparse_index_len(const gorse_b200_sparse_index *ix, int64_t *count_out)
{
    GB_CHECK_ARG(ix != nullptr && count_out != nullptr, "NULL argument");
    *count_out = (int64_t)ix->h_off.size() - 1;
    return GORSE_B200_OK;
}

int32_t gorse_b200_sparse_index_search_range(gorse_b200_sparse_index *ix, int64_t q0, int64_t q1, int32_t k, int32_t *idx_out,
                                             float *dot_out, int32_t *count_out)
{
    GB_CHECK_ARG(ix != nullptr, "index is NULL");
    GB_CHECK_ARG(k > 0 && k <= 128, "k must be in 1..128 (got %d)", k);
    std::lock_guard<std::mutex> lk(ix->mu);
    const int64_t n = (int64_t)ix->h_off.size() - 1;
    if (q0 < 0 || q1 < q0 || q1 > n) {
        set_error("index out of range: [%lld, %lld)", (long long)q0, (long long)q1);
        return GORSE_B200_ERR_RANGE;
    }
    const int64_t nq = q1 - q0;
    if (nq == 0) return GORSE_B200_OK;
    GB_CHECK_ARG(idx_out != nullptr && dot_out != nullptr && count_out != nullptr, "NULL output");
    return gb::sparse_search_host(ix, q0, nq, nullptr, nullptr, nullptr, nullptr, k, idx_out, dot_out, count_out);
}

}  // extern "C"

namespace gb {

// queries = stored rows [q0, q0 + nq) (q_off == nullptr) or nq rows of a HOST CSR (q_off/q_ind/q_val); allow = optional DEVICE
// per-row filter; results to host buffers.  The caller holds ix->mu.
static constexpr int SEARCH_WARPS = 4;

// one accumulator row per resident warp, at most ~1 GB of them; returns the grid of sparse_search_kernel
static int32_t reserve_acc(gorse_b200_sparse_index *ix, int64_t n, int64_t nq, int *grid)
{
    gorse_b200_ctx *c = ix->ctx;
    const int warps = SEARCH_WARPS;
    int64_t slots = std::min<int64_t>((nq + warps - 1) / warps * warps, (int64_t)c->sm_count * 4 * warps);
    slots = std::max<int64_t>(warps, std::min<int64_t>(slots, ((1ll << 30) / 4 / std::max<int64_t>(1, n)) / warps * warps));
    if (ix->acc_slots < slots) {
        GB_TRY(ix->acc.alloc((size_t)slots * (size_t)n));
        GB_CUDA(cudaMemsetAsync(ix->acc.p, 0, sizeof(float) * (size_t)slots * (size_t)n, c->stream));
        ix->acc_slots = slots;
    }
    *grid = (int)(slots / warps);
    return GORSE_B200_OK;
}

int32_t sparse_search_rows(gorse_b200_sparse_index *ix, const int64_t *d_rows, int64_t nq, const uint8_t *d_allow, int32_t k, int32_t *d_idx,
                           float *d_dot, int32_t *d_cnt)
{
    const int64_t n = (int64_t)ix->h_off.size() - 1;
    gorse_b200_ctx *c = ix->ctx;
    GB_TRY(sync_device(ix));
    int grid = 0;
    GB_TRY(reserve_acc(ix, n, nq, &grid));
    sparse_search_kernel<true><<<grid, 32 * SEARCH_WARPS, (size_t)SEARCH_WARPS * 2 * (size_t)k * 4, c->stream>>>(
        ix->off.p, ix->ind.p, ix->val.p, ix->foff.p, ix->frow.p, ix->fval.p, n, ix->n_features, 0, nq, k, ix->acc.p, d_idx, d_dot, d_cnt,
        nullptr, nullptr, nullptr, d_allow, d_rows);
    GB_LAUNCHED(c);
    return GORSE_B200_OK;
}

int32_t sparse_search_host(gorse_b200_sparse_index *ix, int64_t q0, int64_t nq, const int64_t *q_off, const uint32_t *q_ind,
                           const float *q_val, const uint8_t *d_allow, int32_t k, int32_t *idx_out, float *dot_out, int32_t *count_out)
{
    const int64_t n = (int64_t)ix->h_off.size() - 1;
    gorse_b200_ctx *c = ix->ctx;
    ScopedDevice sd(c->device);
    GB_TRY(sync_device(ix));
    if (n == 0) {
        for (int64_t q = 0; q < nq; q++) count_out[q] = 0;
        return GORSE_B200_OK;
    }
    const int warps = SEARCH_WARPS;
    int grid = 0;
    GB_TRY(reserve_acc(ix, n, nq, &grid));
    DevBuf<int32_t> d_idx, d_cnt;
    DevBuf<float> d_dot, dq_val;
    DevBuf<int64_t> dq_off;
    DevBuf<uint32_t> dq_ind;
    int32_t st = GORSE_B200_OK;
    auto done = [&](int32_t s) { cudaStreamSynchronize(c->stream); d_idx.free(); d_cnt.free(); d_dot.free(); dq_val.free(); dq_off.free(); dq_ind.free(); return s; };
    if ((st = d_idx.alloc((size_t)nq * k)) || (st = d_dot.alloc((size_t)nq * k)) || (st = d_cnt.alloc((size_t)nq))) return done(st);
    cudaError_t e = cudaSuccess;
    if (q_off) {
        const int64_t qn = q_off[nq];
        if ((st = dq_off.alloc((size_t)nq + 1)) || (st = dq_ind.alloc((size_t)qn)) || (st = dq_val.alloc((size_t)qn))) return done(st);
        e = cudaMemcpyAsync(dq_off.p, q_off, sizeof(int64_t) * ((size_t)nq + 1), cudaMemcpyHostToDevice, c->stream);
        if (e == cudaSuccess && qn) e = cudaMemcpyAsync(dq_ind.p, q_ind, sizeof(uint32_t) * (size_t)qn, cudaMemcpyHostToDevice, c->stream);
        if (e == cudaSuccess && qn) e = cudaMemcpyAsync(dq_val.p, q_val, sizeof(float) * (size_t)qn, cudaMemcpyHostToDevice, c->stream);
        if (e != cudaSuccess) { set_error("sparse search upload: %s", cudaGetErrorString(e)); return done(GORSE_B200_ERR_CUDA); }
    }
    const size_t sm = (size_t)warps * 2 * (size_t)k * 4;
    sparse_search_kernel<false><<<grid, 32 * warps, sm, c->stream>>>(ix->off.p, ix->ind.p, ix->val.p, ix->foff.p, ix->frow.p, ix->fval.p, n,
                                                             ix->n_features, q0, nq, k, ix->acc.p, d_idx.p, d_dot.p, d_cnt.p,
                                                             q_off ? dq_off.p : nullptr, dq_ind.p, dq_val.p, d_allow, nullptr);
    c->launches++;
    e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaMemcpyAsync(idx_out, d_idx.p, sizeof(int32_t) * (size_t)nq * k, cudaMemcpyDeviceToHost, c->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(dot_out, d_dot.p, sizeof(float) * (size_t)nq * k, cudaMemcpyDeviceToHost, c->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(count_out, d_cnt.p, sizeof(int32_t) * (size_t)nq, cudaMemcpyDeviceToHost, c->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
    if (e != cudaSuccess) { set_error("sparse search: %s", cudaGetErrorString(e)); return done(GORSE_B200_ERR_CUDA); }
    return done(GORSE_B200_OK);
}

int32_t sparse_compact(gorse_b200_sparse_index *ix, const int64_t *scan, int64_t live)
{
    GB_TRY(sync_device(ix));
    gorse_b200_ctx *c = ix->ctx;
    cudaStream_t s = c->stream;
    const int64_t n = (int64_t)ix->h_off.size() - 1, nnz = (int64_t)ix->h_ind.size(), F = ix->n_features;
    DevBuf<int64_t> rs, cs, off_n, foff_n;   // entry keep flags, scanned in place: CSR (rs) and CSC (cs)
    DevBuf<uint8_t> tmp;
    DevBuf<uint32_t> ind_n;
    DevBuf<float> val_n, fval_n;
    DevBuf<int32_t> frow_n;
    auto done = [&](int32_t st) {
        cudaStreamSynchronize(s);
        rs.free(); cs.free(); tmp.free();
        if (st) { off_n.free(); foff_n.free(); ind_n.free(); val_n.free(); fval_n.free(); frow_n.free(); }
        return st;
    };
    int32_t st;
    if ((st = rs.alloc((size_t)nnz + 1)) || (st = cs.alloc((size_t)nnz + 1))) return done(st);
    const unsigned grid = (unsigned)c->sm_count * 8;
    sparse_row_keep_kernel<<<grid, 256, 0, s>>>(ix->off.p, n, scan, rs.p);
    sparse_col_keep_kernel<<<grid, 256, 0, s>>>(ix->frow.p, nnz, scan, cs.p);
    c->launches += 2;
    size_t tmp_bytes = 0;
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, rs.p, nnz + 1, s);
    if (e != cudaSuccess) { set_error("sparse compact: %s", cudaGetErrorString(e)); return done(GORSE_B200_ERR_CUDA); }
    if ((st = tmp.alloc(tmp_bytes))) return done(st);
    int64_t live_nnz = 0;
    e = cub::DeviceScan::ExclusiveSum(tmp.p, tmp_bytes, rs.p, nnz + 1, s);
    if (e == cudaSuccess) e = cub::DeviceScan::ExclusiveSum(tmp.p, tmp_bytes, cs.p, nnz + 1, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(&live_nnz, rs.p + nnz, sizeof(int64_t), cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) { set_error("sparse compact: %s", cudaGetErrorString(e)); return done(GORSE_B200_ERR_CUDA); }
    // every buffer of the compacted index, then the host CSR, before any state changes
    if ((st = off_n.alloc((size_t)live + 1)) || (st = foff_n.alloc((size_t)F + 1)) || (st = ind_n.alloc((size_t)live_nnz)) ||
        (st = val_n.alloc((size_t)live_nnz)) || (st = frow_n.alloc((size_t)live_nnz)) || (st = fval_n.alloc((size_t)live_nnz)))
        return done(st);
    std::vector<int64_t> h_off((size_t)live + 1);
    std::vector<uint32_t> h_ind((size_t)live_nnz);
    std::vector<float> h_val((size_t)live_nnz);
    sparse_compact_off_kernel<<<div_up(n + 1, 256), 256, 0, s>>>(ix->off.p, n, scan, rs.p, off_n.p);
    sparse_compact_off_kernel<<<div_up((int64_t)F + 1, 256), 256, 0, s>>>(ix->foff.p, F, nullptr, cs.p, foff_n.p);
    sparse_compact_csr_kernel<<<grid, 256, 0, s>>>(ix->ind.p, ix->val.p, nnz, rs.p, ind_n.p, val_n.p);
    sparse_compact_csc_kernel<<<grid, 256, 0, s>>>(ix->frow.p, ix->fval.p, nnz, cs.p, scan, frow_n.p, fval_n.p);
    c->launches += 4;
    e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaMemcpyAsync(h_off.data(), off_n.p, sizeof(int64_t) * h_off.size(), cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess && live_nnz) e = cudaMemcpyAsync(h_ind.data(), ind_n.p, sizeof(uint32_t) * h_ind.size(), cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess && live_nnz) e = cudaMemcpyAsync(h_val.data(), val_n.p, sizeof(float) * h_val.size(), cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) { set_error("sparse compact: %s", cudaGetErrorString(e)); return done(GORSE_B200_ERR_CUDA); }
    ix->off.free(); ix->foff.free(); ix->ind.free(); ix->val.free(); ix->frow.free(); ix->fval.free();
    ix->off = off_n; ix->foff = foff_n; ix->ind = ind_n; ix->val = val_n; ix->frow = frow_n; ix->fval = fval_n;
    ix->h_off.swap(h_off); ix->h_ind.swap(h_ind); ix->h_val.swap(h_val);
    ix->acc.free();   // [slots x N]; reserve_acc allocates and zeroes it again for the new N
    ix->acc_slots = 0;
    return done(GORSE_B200_OK);
}

size_t sparse_bytes(const gorse_b200_sparse_index *ix)
{
    return ix->off.bytes() + ix->foff.bytes() + ix->ind.bytes() + ix->val.bytes() + ix->frow.bytes() + ix->fval.bytes() + ix->acc.bytes();
}

}  // namespace gb
