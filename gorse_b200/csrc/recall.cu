// recall.cu -- batched collaborative-filtering recall: gorse_b200_vecdb_query_excluding.
//
// The worker's CF recall (worker/pipeline.go:403-449) asks, per user, QueryVectors(user embedding, topK = n + |E_u|) and then
// drops the user's feedback items E_u (logics/recommend.go:67-80).  Here one call answers many users: row q's answer is the
// first k_q = n + |E_q| allowed slots by (score desc, slot asc), minus the slots in E_q, with the scores of
// gorse_b200_vecdb_query's exact scan, bit for bit.
//
//   routing   rows with k_q <= 128 / 256 / 512 form classes; each class is swept by the tensor-core stage 1 (topk_mma.cu) with
//             a sample sized for the class bound.  Rows above 512, calls the sweep does not serve (mma_path_eligible: small
//             collections, few rows, Cosine) and rows whose window cannot be certified go to the exact kernel.
//   stage 2   recall_window_kernel, one CTA per row: drops the candidates the filter rejects, certifies the row against its
//             own k_q (k_q-th best approximate score >= theta + 2 eps, as prune_kernel), re-scores the window exactly, sorts it
//             in shared memory and writes the first k_q minus E_q.
//   exact     recall_exact_kernel, one CTA per row: scores every allowed vector into scratch, selects the k_q-th key by radix
//             select, and emits the result in sorted rounds of at most SORT_CAP entries.
// Both paths order by the same key and write the same score bits, so a row's answer does not depend on its path.
#include <algorithm>

#include "cf.cuh"
#include "recall.cuh"
#include "topk.cuh"
#include "vecdb.cuh"

namespace gb {
namespace recall {

constexpr int N_CLASSES = 3;
constexpr int CLASS_K[N_CLASSES] = {128, 256, 512};
constexpr int SORT_CAP = mma::CAP;   // entries one CTA sorts at a time (a window never holds more)
constexpr int WIN_THREADS = 128, EXACT_THREADS = 256;

// order key of a score: larger score = larger key; -0 and +0 are one score (the exact scan compares floats); NaN = 0 = no entry
__device__ __forceinline__ uint32_t rank_key(float s) { return s != s ? 0u : float_key(s == 0.f ? 0.f : s); }
// sort key: ascending order = score descending, then slot ascending
__device__ __forceinline__ uint64_t sort_key(uint32_t key, int64_t slot) { return ((uint64_t)~key << 32) | (uint32_t)slot; }

struct RowInfo {              // per row of a chunk (chunk-local row ids)
    const float *q;           // [rows][d] queries
    const int32_t *k;         // n + |E_q|
    const int64_t *ex_off;    // [rows + 1] into ex
    const int64_t *ex;        // each row's excluded slots, ascending (-1 entries dropped)
    const int64_t *out_off;   // where the row's answer starts in slots / scores
    int32_t *need_exact;      // 1 = the exact kernel answers the row
    int64_t *slots;
    float *scores;
    int32_t *count;           // [rows]
    int *flags;               // [0] NaN score seen, [1] rows the window kernel handed to the exact kernel
};

// the sorted entries [0, m) minus the row's excluded slots, appended at out + written
template <int NT>
__device__ void block_emit(const uint64_t *key, const float *val, int m, const int64_t *ex, int64_t n_ex, int64_t *out_slots,
                           float *out_scores, int &written, int *s_warp)
{
    for (int base = 0; base < m; base += NT) {
        const int i = base + threadIdx.x;
        int64_t slot = 0;
        bool keep = false;
        if (i < m) {
            slot = (int64_t)(uint32_t)key[i];
            keep = !contains(ex, n_ex, slot);
        }
        int total;
        const int r = block_rank<NT>(keep, s_warp, total);
        if (keep) {
            out_slots[written + r] = slot;
            out_scores[written + r] = val[i];
        }
        written += total;
    }
}

// score = -distance of the exact scan (topk_exact_kernel's arithmetic) for count vectors: slot_at(j) < 0 skips entry j.
// put(j, score, valid) is called once per entry.
template <int NT, typename SlotAt, typename Put>
__device__ __forceinline__ void block_score(const float *X, int d, int metric, const float *qs, float qq, int64_t count, SlotAt slot_at, Put put)
{
    if (d % 16 == 0 && d <= 256) {
        const int lane4 = threadIdx.x & 3, chunks = d / 16;
        const unsigned qmask = quad_mask();
        float4 qreg[16];
#pragma unroll
        for (int c = 0; c < 16; c++)
            if (c < chunks) qreg[c] = *reinterpret_cast<const float4 *>(qs + 16 * c + 4 * lane4);
        for (int64_t j = threadIdx.x >> 2; j < count; j += NT / 4) {   // a quad per entry: its 4 lanes share j
            const int64_t v = slot_at(j);
            float s = 0.f;
            if (v >= 0) s = -quad_dist(qreg, X + v * d, chunks, lane4, qmask, metric, qq);
            if (lane4 == 0) put(j, s, v >= 0);
        }
    } else {
        for (int64_t j = threadIdx.x; j < count; j += NT) {
            const int64_t v = slot_at(j);
            put(j, v >= 0 ? -dist_any(qs, X + v * d, d, metric, qq) : 0.f, v >= 0);
        }
    }
}

template <int NT>
__device__ __forceinline__ float load_query(const float *q, int d, int metric, float *qs)
{
    for (int e = threadIdx.x; e < d; e += NT) qs[e] = q[e];
    __syncthreads();
    return metric == GORSE_B200_METRIC_COSINE ? dot_any(qs, qs, d) : 0.f;
}

// ---- stage 2: one CTA per row of a class (rows[i] = chunk-local row; candidate list i belongs to it) ------------------------
__global__ void __launch_bounds__(WIN_THREADS)
recall_window_kernel(const int32_t *cand_col, const float *cand_val, const int32_t *cand_cnt, const float *theta, const float *eps,
                     const int32_t *perm, const uint8_t *allow, const float *X, int d, int metric, const int64_t *rows, int64_t n_rows,
                     RowInfo R)
{
    constexpr int NT = WIN_THREADS;
    extern __shared__ __align__(16) uint8_t sm[];
    uint64_t *s_key = reinterpret_cast<uint64_t *>(sm);                     // [SORT_CAP] window, sort keys
    float *s_val = reinterpret_cast<float *>(s_key + SORT_CAP);            // [SORT_CAP] window, exact scores
    int32_t *g_slot = reinterpret_cast<int32_t *>(s_val + SORT_CAP);       // [CAP] candidates: slot
    uint32_t *g_key = reinterpret_cast<uint32_t *>(g_slot + mma::CAP);     // [CAP] candidates: approximate key (0 = dropped)
    int *hist = reinterpret_cast<int *>(g_key + mma::CAP);                 // [256]
    int *s_warp = hist + 256;                                              // [32]
    int *s_bc = s_warp + 32;                                               // [4]
    float *qs = reinterpret_cast<float *>(s_bc + 4);                       // [d]
    for (int64_t i = blockIdx.x; i < n_rows; i += gridDim.x) {
        const int64_t r = rows[i];
        const int k = R.k[r];
        // every column with approximate score >= max over the parts' thresholds was pushed by one of the parts
        int np[mma::PARTS], n = 0;
        float th = -INFINITY;
        bool bad = !(eps[i] == eps[i]);
#pragma unroll
        for (int p = 0; p < mma::PARTS; p++) {
            const int raw = cand_cnt[mma::PARTS * i + p];
            bad |= raw > mma::PART_CAP;
            np[p] = min(raw, mma::PART_CAP);
            n += np[p];
            th = fmaxf(th, theta[mma::PARTS * i + p]);
        }
        if (!(th == th)) bad = true;
        int have = 0;
        for (int e = threadIdx.x; e < n; e += NT) {
            int p = 0, rr = e;   // entry e of the concatenated part lists
#pragma unroll
            for (int q = 0; q + 1 < mma::PARTS; q++)
                if (p == q && rr >= np[q]) { rr -= np[q]; p++; }
            const int64_t src = i * mma::CAP + p * mma::PART_CAP + rr;
            const int32_t slot = perm[cand_col[src]];
            const uint32_t key = allow[slot] ? rank_key(cand_val[src]) : 0u;
            g_slot[e] = slot;
            g_key[e] = key;
            have += key != 0u;
        }
        have = block_sum<NT>(have, s_warp);   // (synchronises: g_* are complete)
        if (have < k) bad = true;
        float kth = 0.f;
        if (!bad) {
            int ties;
            kth = key_float(block_select<NT>(n, k, [&](int64_t e) { return g_key[e]; }, hist, s_bc, &ties));
            // at least k allowed candidates clear theta + 2 eps: every allowed column outside the list ranks below them
            if (!(kth >= th + 2.f * eps[i])) bad = true;
        }
        if (bad) {
            if (threadIdx.x == 0) { R.need_exact[r] = 1; atomicAdd(&R.flags[1], 1); }
            continue;
        }
        // the window: candidates whose exact score can reach the k-th best (approximate >= kth - 2 eps)
        const uint32_t lim = rank_key(kth - 2.f * eps[i]);
        if (threadIdx.x == 0) s_bc[2] = 0;
        __syncthreads();
        for (int e = threadIdx.x; e < n; e += NT)
            if (g_key[e] != 0u && g_key[e] >= lim) s_key[atomicAdd(&s_bc[2], 1)] = (uint64_t)g_slot[e];
        const float qq = load_query<NT>(R.q + r * d, d, metric, qs);   // (synchronises)
        const int w = s_bc[2];
        block_score<NT>(X, d, metric, qs, qq, w, [&](int64_t j) { return (int64_t)s_key[j]; }, [&](int64_t j, float s, bool) {
            if (s != s) R.flags[0] = 1;
            s_val[j] = s;
        });
        __syncthreads();
        const int p2 = pow2_at_least(w);
        for (int j = threadIdx.x; j < p2; j += NT)
            s_key[j] = j < w ? sort_key(rank_key(s_val[j]), (int64_t)s_key[j]) : ~0ull;
        __syncthreads();
        block_sort<NT>(s_key, s_val, p2);
        int written = 0;
        block_emit<NT>(s_key, s_val, min(k, w), R.ex + R.ex_off[r], R.ex_off[r + 1] - R.ex_off[r], R.slots + R.out_off[r],
                       R.scores + R.out_off[r], written, s_warp);
        if (threadIdx.x == 0) R.count[r] = written;
        __syncthreads();
    }
}

// ---- exact path: one CTA per row with need_exact set; sc = this CTA's [N] score scratch ------------------------------------
__global__ void __launch_bounds__(EXACT_THREADS)
recall_exact_kernel(const float *X, int64_t N, int d, int metric, const uint8_t *allow, int64_t n_rows, RowInfo R, float *scratch)
{
    constexpr int NT = EXACT_THREADS;
    extern __shared__ __align__(16) uint8_t sm[];
    uint64_t *s_key = reinterpret_cast<uint64_t *>(sm);                // [SORT_CAP]
    float *s_val = reinterpret_cast<float *>(s_key + SORT_CAP);       // [SORT_CAP]
    int *hist = reinterpret_cast<int *>(s_val + SORT_CAP);            // [256]
    int *s_warp = hist + 256;                                         // [32]
    int *s_bc = s_warp + 32;                                          // [4]
    float *qs = reinterpret_cast<float *>(s_bc + 4);                  // [d]
    float *sc = scratch + (int64_t)blockIdx.x * N;
    const float none = __int_as_float(0x7fffffff);                    // NaN: rank_key 0
    for (int64_t r = blockIdx.x; r < n_rows; r += gridDim.x) {
        if (!R.need_exact[r]) continue;
        const float qq = load_query<NT>(R.q + r * d, d, metric, qs);
        int have = 0;
        block_score<NT>(X, d, metric, qs, qq, N, [&](int64_t j) { return allow[j] ? j : (int64_t)-1; }, [&](int64_t j, float s, bool valid) {
            if (valid && s != s) R.flags[0] = 1;
            sc[j] = valid ? s : none;
            have += valid && s == s;
        });
        have = block_sum<NT>(have, s_warp);   // (synchronises: sc is complete)
        const int K = min(R.k[r], have);
        int written = 0;
        // rounds of at most SORT_CAP: select the round's last key, gather, sort, emit, then retire the emitted entries
        for (int emitted = 0; emitted < K;) {
            const int m = min(SORT_CAP, K - emitted);
            int ties;
            const uint32_t t = block_select<NT>(N, m, [&](int64_t j) { return rank_key(sc[j]); }, hist, s_bc, &ties);
            if (threadIdx.x == 0) s_bc[2] = 0;
            int eq_taken = 0;   // entries equal to t go in slot order: the lowest slots win the tie
            __syncthreads();
            for (int64_t base = 0; base < N; base += NT) {
                const int64_t j = base + threadIdx.x;
                const uint32_t key = j < N ? rank_key(sc[j]) : 0u;
                int n_eq;
                const int er = block_rank<NT>(key == t, s_warp, n_eq);
                int pos = -1;
                if (key > t) pos = atomicAdd(&s_bc[2], 1);
                else if (key == t && eq_taken + er < ties) pos = m - ties + eq_taken + er;
                if (pos >= 0) { s_key[pos] = sort_key(key, j); s_val[pos] = sc[j]; }
                eq_taken += n_eq;
            }
            const int p2 = pow2_at_least(m);
            for (int j = m + threadIdx.x; j < p2; j += NT) s_key[j] = ~0ull;
            __syncthreads();
            block_sort<NT>(s_key, s_val, p2);
            block_emit<NT>(s_key, s_val, m, R.ex + R.ex_off[r], R.ex_off[r + 1] - R.ex_off[r], R.slots + R.out_off[r], R.scores + R.out_off[r],
                           written, s_warp);
            for (int j = threadIdx.x; j < m; j += NT) sc[(uint32_t)s_key[j]] = none;
            __syncthreads();
            emitted += m;
        }
        if (threadIdx.x == 0) R.count[r] = written;
        __syncthreads();
    }
}

// q[r] = X[slots[r]]: the query rows of stored vectors, one CTA per row
__global__ void recall_gather_kernel(const float *X, int d, const int64_t *slots, int64_t rows, float *q)
{
    for (int64_t r = blockIdx.x; r < rows; r += gridDim.x)
        for (int e = threadIdx.x; e < d; e += blockDim.x) q[r * d + e] = X[slots[r] * d + e];
}

size_t window_smem(int d) { return (size_t)SORT_CAP * 12 + (size_t)mma::CAP * 8 + (256 + 32 + 4) * 4 + (size_t)d * 4; }
size_t exact_smem(int d) { return (size_t)SORT_CAP * 12 + (256 + 32 + 4) * 4 + (size_t)d * 4; }

}  // namespace recall
}  // namespace gb

using namespace gb;

extern "C" int32_t gorse_b200_vecdb_query_excluding(gorse_b200_vecdb *db, int64_t nq, const float *q_values, const int32_t *categories,
                                                    int32_t n_categories, int32_t n, const int64_t *excl_off, const int64_t *excl_slots,
                                                    int64_t *slots_out, float *scores_out, int32_t *count_out, int64_t *exact_rows_out)
{
    using namespace gb::recall;
    GB_CHECK_ARG(db != nullptr, "collection is NULL");
    GB_CHECK_ARG(nq >= 0 && n_categories >= 0, "negative count");
    if (exact_rows_out) *exact_rows_out = 0;
    if (nq == 0) return GORSE_B200_OK;
    GB_CHECK_ARG(count_out != nullptr && excl_off != nullptr, "count_out / excl_off is NULL");
    GB_CHECK_ARG(excl_off[0] == 0, "excl_off[0] must be 0");
    for (int64_t q = 0; q < nq; q++)
        GB_CHECK_ARG(excl_off[q + 1] >= excl_off[q], "excl_off not non-decreasing at %lld", (long long)q);
    GB_CHECK_ARG(excl_off[nq] == 0 || excl_slots != nullptr, "excl_slots is NULL");
    if (db->dim == 0) {
        set_error("query_excluding serves dense collections only");
        return GORSE_B200_ERR_UNSUPPORTED;
    }
    if (n <= 0) {
        for (int64_t q = 0; q < nq; q++) count_out[q] = 0;
        return GORSE_B200_OK;
    }
    GB_CHECK_ARG(q_values != nullptr && slots_out != nullptr && scores_out != nullptr, "NULL query / output");
    GB_CHECK_ARG(n_categories == 0 || categories != nullptr, "categories is NULL");
    std::lock_guard<std::mutex> lk(db->mu);
    const int64_t n_slots = (int64_t)db->ts.size();
    // each row's exclusions once, sorted, -1 entries dropped (they still count in k_q)
    std::vector<int64_t> ex;
    std::vector<int64_t> ex_off((size_t)nq + 1, 0);
    ex.reserve((size_t)excl_off[nq]);
    for (int64_t q = 0; q < nq; q++) {
        GB_CHECK_ARG((int64_t)n + (excl_off[q + 1] - excl_off[q]) <= INT32_MAX, "row %lld: n + |E| overflows", (long long)q);
        const size_t b = ex.size();
        for (int64_t t = excl_off[q]; t < excl_off[q + 1]; t++) {
            const int64_t s = excl_slots[t];
            GB_CHECK_ARG(s >= -1 && s < n_slots, "row %lld: excluded slot %lld is not a slot of the collection", (long long)q, (long long)s);
            if (s >= 0) ex.push_back(s);
        }
        std::sort(ex.begin() + b, ex.end());
        for (size_t t = b + 1; t < ex.size(); t++)
            GB_CHECK_ARG(ex[t] != ex[t - 1], "row %lld: slot %lld is excluded twice", (long long)q, (long long)ex[t]);
        ex_off[(size_t)q + 1] = (int64_t)ex.size();
    }
    if (n_slots == 0) {
        for (int64_t q = 0; q < nq; q++) count_out[q] = 0;
        return GORSE_B200_OK;
    }
    ScopedDevice sd(db->ctx->device);
    GB_TRY(vecdb_allow(db, categories, n_categories));
    return recall_rows(db, nq, q_values, nullptr, n, excl_off, ex, ex_off, slots_out, scores_out, count_out, exact_rows_out);
}

namespace gb {
namespace recall {

int32_t recall_rows(gorse_b200_vecdb *db, int64_t nq, const float *q_host, const int64_t *d_qslots, int32_t n, const int64_t *excl_off,
                    const std::vector<int64_t> &ex, const std::vector<int64_t> &ex_off, int64_t *slots_out, float *scores_out,
                    int32_t *count_out, int64_t *exact_rows_out)
{
    gorse_b200_ctx *c = db->ctx;
    gorse_b200_index *ix = db->dense;
    std::lock_guard<std::mutex> lk2(ix->mu);
    RecallWork &W = db->recall;
    const int d = ix->d;
    const int64_t N = ix->n, total_out = nq * (int64_t)n + excl_off[nq];
    auto out_at = [&](int64_t q) { return q * (int64_t)n + excl_off[q]; };
    // the sweep serves Dot and Euclidean collections of >= 32768 vectors for >= 64 rows; GORSE_B200_TOPK_EXACT=1 turns it off
    const bool tensor = mma_path_eligible(ix, nq, 1);
    const int64_t cq = std::min<int64_t>(nq, (int64_t)c->sm_count * mma::GROUP_ROWS * 8);
    // exact scratch: one [N] score row per CTA, at most 512 MB
    const int exact_grid = (int)std::max<int64_t>(1, std::min<int64_t>({(int64_t)c->sm_count * 2, cq, (512ll << 20) / (4 * N)}));
    int32_t st = GORSE_B200_OK;
    auto done = [&](int32_t s) {
        cudaStreamSynchronize(c->stream);
        cudaStreamSynchronize(c->copy_stream);
        return s;
    };
    if ((st = grow(W.q, (size_t)cq * d)) || (st = grow(W.k, (size_t)cq)) || (st = grow(W.ex_off, (size_t)cq + 1)) || (st = grow(W.out_off, (size_t)cq)) ||
        (st = grow(W.rows, (size_t)cq)) || (st = grow(W.need, (size_t)cq)) || (st = grow(W.count, (size_t)nq)) || (st = grow(W.flags, 2)) ||
        (st = grow(W.slots, (size_t)std::max<int64_t>(total_out, 1))) || (st = grow(W.scores, (size_t)std::max<int64_t>(total_out, 1))) ||
        (st = grow(W.scratch, (size_t)exact_grid * N)) || (st = grow(W.ex, std::max<size_t>(ex.size(), 1))))
        return done(st);
    if (tensor && (st = mma_reserve(ix, cq))) return done(st);
    cudaError_t e = cudaFuncSetAttribute(recall_window_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)window_smem(d));
    if (e == cudaSuccess) e = cudaFuncSetAttribute(recall_exact_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)exact_smem(d));
    if (e == cudaSuccess) e = cudaMemsetAsync(W.flags.p, 0, 2 * sizeof(int), c->stream);
    if (e != cudaSuccess) { set_error("query_excluding: %s", cudaGetErrorString(e)); return done(GORSE_B200_ERR_CUDA); }
    int64_t host_exact = 0;
    std::vector<int32_t> h_k, h_need;
    std::vector<int64_t> h_exoff, h_outoff, h_rows;
    for (int64_t q0 = 0; q0 < nq; q0 += cq) {
        const int64_t rows = std::min(cq, nq - q0);
        // rows grouped by class; class N_CLASSES = the exact kernel
        h_k.resize(rows); h_need.assign(rows, 0); h_exoff.resize(rows + 1); h_outoff.resize(rows); h_rows.resize(rows);
        int64_t cls_begin[N_CLASSES + 2] = {0};
        std::vector<int8_t> cls(rows);
        for (int64_t r = 0; r < rows; r++) {
            const int64_t q = q0 + r;
            h_k[r] = n + (int32_t)(excl_off[q + 1] - excl_off[q]);
            h_exoff[r] = ex_off[q] - ex_off[q0];
            h_outoff[r] = out_at(q);
            int8_t k_cls = N_CLASSES;
            if (tensor)
                for (int8_t t = N_CLASSES - 1; t >= 0; t--)
                    if (h_k[r] <= CLASS_K[t]) k_cls = t;
            cls[r] = k_cls;
            cls_begin[k_cls + 1]++;
        }
        h_exoff[rows] = ex_off[q0 + rows] - ex_off[q0];
        for (int t = 0; t <= N_CLASSES; t++) cls_begin[t + 1] += cls_begin[t];
        {
            int64_t fill[N_CLASSES + 1];
            std::copy(cls_begin, cls_begin + N_CLASSES + 1, fill);
            for (int64_t r = 0; r < rows; r++) {
                h_rows[fill[cls[r]]++] = r;
                if (cls[r] == N_CLASSES) h_need[r] = 1;
            }
        }
        host_exact += cls_begin[N_CLASSES + 1] - cls_begin[N_CLASSES];
        const int64_t n_ex = h_exoff[rows];
        if (!q_host) {   // stored vectors: gathered from the collection in place of the upload
            recall_gather_kernel<<<(unsigned)std::min<int64_t>(rows, (int64_t)c->sm_count * 16), 128, 0, c->stream>>>(ix->X.p, d, d_qslots + q0, rows, W.q.p);
            c->launches++;
        }
        if ((q_host && (e = cudaMemcpyAsync(W.q.p, q_host + q0 * d, sizeof(float) * rows * d, cudaMemcpyHostToDevice, c->stream)) != cudaSuccess) ||
            (e = cudaMemcpyAsync(W.k.p, h_k.data(), sizeof(int32_t) * rows, cudaMemcpyHostToDevice, c->stream)) != cudaSuccess ||
            (e = cudaMemcpyAsync(W.need.p, h_need.data(), sizeof(int32_t) * rows, cudaMemcpyHostToDevice, c->stream)) != cudaSuccess ||
            (e = cudaMemcpyAsync(W.ex_off.p, h_exoff.data(), sizeof(int64_t) * (rows + 1), cudaMemcpyHostToDevice, c->stream)) != cudaSuccess ||
            (e = cudaMemcpyAsync(W.out_off.p, h_outoff.data(), sizeof(int64_t) * rows, cudaMemcpyHostToDevice, c->stream)) != cudaSuccess ||
            (e = cudaMemcpyAsync(W.rows.p, h_rows.data(), sizeof(int64_t) * rows, cudaMemcpyHostToDevice, c->stream)) != cudaSuccess ||
            (n_ex && (e = cudaMemcpyAsync(W.ex.p, ex.data() + ex_off[q0], sizeof(int64_t) * n_ex, cudaMemcpyHostToDevice, c->stream)) != cudaSuccess)) {
            set_error("query_excluding upload: %s", cudaGetErrorString(e));
            return done(GORSE_B200_ERR_CUDA);
        }
        RowInfo R;
        R.q = W.q.p; R.k = W.k.p; R.ex_off = W.ex_off.p; R.ex = W.ex.p; R.out_off = W.out_off.p; R.need_exact = W.need.p;
        R.slots = W.slots.p; R.scores = W.scores.p; R.count = W.count.p + q0; R.flags = W.flags.p;
        for (int t = 0; t < N_CLASSES; t++) {
            const int64_t nr = cls_begin[t + 1] - cls_begin[t];
            if (nr == 0) continue;
            // the sample aims at 4 k columns per row, at most CAP / 2 so that a row's lists rarely overflow (Gamma(R_TOP) spread)
            const int m_tiles = mma_sample_tiles(ix, std::min(4.0 * CLASS_K[t], mma::CAP / 2.0));
            if ((st = mma_sweep(ix, W.q.p, nullptr, W.rows.p + cls_begin[t], 0, nr, m_tiles, nullptr, nullptr))) return done(st);
            recall_window_kernel<<<(unsigned)std::min<int64_t>(nr, (int64_t)c->sm_count * 16), WIN_THREADS, window_smem(d), c->stream>>>(
                ix->w_ccol.p, ix->w_cval.p, ix->w_ccnt.p, ix->w_theta.p, ix->w_eps.p, ix->perm.p, db->d_allow.p, ix->X.p, d, ix->metric,
                W.rows.p + cls_begin[t], nr, R);
            c->launches++;
        }
        recall_exact_kernel<<<(unsigned)std::min<int64_t>(rows, exact_grid), EXACT_THREADS, exact_smem(d), c->stream>>>(
            ix->X.p, N, d, ix->metric, db->d_allow.p, rows, R, W.scratch.p);
        c->launches++;
        if ((e = cudaGetLastError()) != cudaSuccess) { set_error("query_excluding: %s", cudaGetErrorString(e)); return done(GORSE_B200_ERR_CUDA); }
        if (!slots_out) continue;   // the caller reads the answers on the device
        // this chunk is final: download it on the copy stream while the next chunk computes
        const int64_t o0 = out_at(q0), o1 = out_at(q0 + rows);
        if ((e = cudaEventRecord(c->copy_ev, c->stream)) != cudaSuccess || (e = cudaStreamWaitEvent(c->copy_stream, c->copy_ev, 0)) != cudaSuccess ||
            (e = cudaMemcpyAsync(count_out + q0, W.count.p + q0, sizeof(int32_t) * rows, cudaMemcpyDeviceToHost, c->copy_stream)) != cudaSuccess ||
            (o1 > o0 && ((e = cudaMemcpyAsync(slots_out + o0, W.slots.p + o0, sizeof(int64_t) * (o1 - o0), cudaMemcpyDeviceToHost, c->copy_stream)) != cudaSuccess ||
                         (e = cudaMemcpyAsync(scores_out + o0, W.scores.p + o0, sizeof(float) * (o1 - o0), cudaMemcpyDeviceToHost, c->copy_stream)) != cudaSuccess))) {
            set_error("query_excluding download: %s", cudaGetErrorString(e));
            return done(GORSE_B200_ERR_CUDA);
        }
    }
    int flags[2] = {0, 0};
    if ((e = cudaMemcpyAsync(flags, W.flags.p, sizeof(flags), cudaMemcpyDeviceToHost, c->stream)) != cudaSuccess ||
        (e = cudaStreamSynchronize(c->stream)) != cudaSuccess || (e = cudaStreamSynchronize(c->copy_stream)) != cudaSuccess) {
        set_error("query_excluding: %s", cudaGetErrorString(e));
        return done(GORSE_B200_ERR_CUDA);
    }
    if (flags[0]) { set_error("NaN distance"); return done(GORSE_B200_ERR_ARG); }
    if (exact_rows_out) *exact_rows_out = host_exact + flags[1];
    return done(GORSE_B200_OK);
}

}  // namespace recall
}  // namespace gb
