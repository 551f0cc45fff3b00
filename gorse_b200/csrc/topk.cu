// topk.cu -- the dense top-k pipeline, and the brute-force vector index on it: ann.Bruteforce (common/ann/bruteforce.go:24-83)
// behind ann.Index.
//
// One result contract for every caller (the index's searches, the collection query, the batched recall and item-to-item):
// the first k allowed vectors by (distance ascending = score descending, slot ascending), scored with the reference's fp32
// summation order (floats.Euclidean / -floats.Dot, AVX-512 tree).  The reference's tie order is an artefact of Go's
// container/heap and is not pinned by any reference test.  A row whose query is a stored vector never returns that vector
// (bruteforce.go:47).
//
//   routing   rows with k_q <= 128 / 256 / 512 form classes; each class is swept by the tensor-core stage 1 (topk_mma.cu) with
//             a sample aimed at min(4 x the class's largest k_q, CAP / 2) columns per row.  Rows above 512, calls the sweep does
//             not serve (mma_path_eligible: small indexes, few rows, Cosine, d > 4096), calls whose mirror or work buffers
//             cannot be allocated and rows whose window cannot be certified go to the exact kernel.
//   stage 2   recall_window_kernel, one CTA per row: drops the candidates the filter rejects and the row's own vector,
//             certifies the row against its own k_q (k_q-th best approximate score >= theta + 2 eps), re-scores the window
//             exactly, sorts it in shared memory and writes the first k_q minus the row's exclusions.
//   exact     recall_exact_kernel, one CTA per row: scores every allowed vector into scratch, selects the k_q-th key by radix
//             select, and emits the result in sorted rounds of at most SORT_CAP entries.
//   table     table_kernel: the answers as a fixed-stride table (the index's int32 ids and distances, prune0; item-to-item's
//             neighbour table).
// Both paths order by the same key and write the same score bits, so a row's answer does not depend on its path.
#include <algorithm>
#include <cmath>

#include "cf.cuh"
#include "recall.cuh"
#include "topk.cuh"

namespace gb {
namespace recall {

constexpr int N_CLASSES = 3;
constexpr int CLASS_K[N_CLASSES] = {128, 256, 512};
constexpr int WIN_THREADS = 256, EXACT_THREADS = 256;

struct RowInfo {              // per row of a chunk (chunk-local row ids)
    const float *q;           // [rows][d] queries
    const int32_t *k;         // n + |E_q|
    const int64_t *ex_off;    // [rows + 1] into ex
    const int64_t *ex;        // each row's excluded slots, ascending (-1 entries dropped)
    const int64_t *out_off;   // where the row's answer starts in slots / scores
    const int64_t *self;      // [rows] the slot of a stored query (never returned), or nullptr
    int64_t *exact;           // rows the exact kernel answers: n_routed routed by the host, then the window kernel's hand-offs
    int64_t n_routed;
    int64_t *slots;
    float *scores;
    int32_t *count;           // [rows]
    int *flags;               // [0] NaN score seen, [1] rows the window kernel handed to the exact kernel, [2] of them in this chunk
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

// score = -distance in the reference's arithmetic for count vectors: slot_at(j) < 0 skips entry j.
// put(j, score, valid) is called once per entry.  T: the element type of the stored rows (float, or uint16_t for bf16).
template <int NT, typename T, typename SlotAt, typename Put>
__device__ __forceinline__ void block_score(const T *X, int d, int metric, const float *qs, float qq, int64_t count, SlotAt slot_at, Put put)
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
template <typename T>
__global__ void __launch_bounds__(WIN_THREADS)
recall_window_kernel(const int32_t *cand_col, const float *cand_val, const int32_t *cand_cnt, const float *theta, const float *eps,
                     const int32_t *perm, const uint8_t *allow, const T *X, int d, int metric, const int64_t *rows, int64_t n_rows,
                     RowInfo R)
{
    constexpr int NT = WIN_THREADS;
    extern __shared__ __align__(16) uint8_t sm[];
    uint64_t *s_key = reinterpret_cast<uint64_t *>(sm);                     // [SORT_CAP] window, sort keys
    int32_t *g_slot = reinterpret_cast<int32_t *>(s_key + SORT_CAP);       // [CAP] candidates: slot
    uint32_t *g_key = reinterpret_cast<uint32_t *>(g_slot + mma::CAP);     // [CAP] candidates: approximate key (0 = dropped)
    float *s_val = reinterpret_cast<float *>(g_key);                       // [SORT_CAP] window, exact scores (g_key is read by then)
    int *hist = reinterpret_cast<int *>(g_key + mma::CAP);                 // [256]
    int *s_warp = hist + 256;                                              // [32]
    int *s_bc = s_warp + 32;                                               // [4]
    float *qs = reinterpret_cast<float *>(s_bc + 4);                       // [d]
    for (int64_t i = blockIdx.x; i < n_rows; i += gridDim.x) {
        const int64_t r = rows[i];
        const int k = R.k[r];
        const int64_t self = R.self ? R.self[r] : -1;
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
            const uint32_t key = slot != self && (!allow || allow[slot]) ? rank_key(cand_val[src]) : 0u;
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
            if (threadIdx.x == 0) { R.exact[R.n_routed + atomicAdd(&R.flags[2], 1)] = r; atomicAdd(&R.flags[1], 1); }
            continue;
        }
        // the window: candidates whose exact score can reach the k-th best (approximate >= kth - 2 eps)
        const uint32_t lim = rank_key(kth - 2.f * eps[i]);
        if (threadIdx.x == 0) s_bc[2] = 0;
        __syncthreads();
        for (int e0 = 0; e0 < n; e0 += NT) {   // a warp takes its places in the window with one atomic
            const int e = e0 + threadIdx.x, lane = threadIdx.x & 31;
            const bool in = e < n && g_key[e] != 0u && g_key[e] >= lim;
            const unsigned b = __ballot_sync(0xffffffffu, in);
            int at = 0;
            if (lane == 0 && b) at = atomicAdd(&s_bc[2], __popc(b));
            at = __shfl_sync(0xffffffffu, at, 0);
            if (in) s_key[at + __popc(b & ((1u << lane) - 1))] = (uint64_t)g_slot[e];
        }
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

// ---- exact path: one CTA per row of R.exact; sc = this CTA's [N] score scratch ---------------------------------------------
template <typename T>
__global__ void __launch_bounds__(EXACT_THREADS)
recall_exact_kernel(const T *X, int64_t N, int d, int metric, const uint8_t *allow, RowInfo R, float *scratch)
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
    const int64_t n_rows = R.n_routed + R.flags[2];
    for (int64_t i = blockIdx.x; i < n_rows; i += gridDim.x) {
        const int64_t r = R.exact[i];
        const int64_t self = R.self ? R.self[r] : -1;
        const float qq = load_query<NT>(R.q + r * d, d, metric, qs);
        int have = 0;
        block_score<NT>(X, d, metric, qs, qq, N, [&](int64_t j) { return j != self && (!allow || allow[j]) ? j : (int64_t)-1; }, [&](int64_t j, float s, bool valid) {
            if (valid && s != s) R.flags[0] = 1;
            sc[j] = valid ? s : none;
            have += valid && s == s;
        });
        have = block_sum<NT>(have, s_warp);   // (synchronises: sc is complete)
        const int K = min(R.k[r], have);
        int written = 0;
        emit_in_rounds<NT>(sc, N, K, s_key, s_val, hist, s_warp, s_bc, [&](int m) {
            block_emit<NT>(s_key, s_val, m, R.ex + R.ex_off[r], R.ex_off[r + 1] - R.ex_off[r], R.slots + R.out_off[r], R.scores + R.out_off[r],
                           written, s_warp);
        });
        if (threadIdx.x == 0) R.count[r] = written;
        __syncthreads();
    }
}

// the Table rows of one chunk's rows [0, rows), at t_slot / t_val + r * n and t_cnt[r]
template <int NT>
__global__ void __launch_bounds__(NT)
table_kernel(const int64_t *slots, const float *scores, const int32_t *count, const int64_t *out_off, int64_t rows, int n, bool negate,
             bool positive, int32_t *t_slot, float *t_val, int32_t *t_cnt)
{
    __shared__ int s_warp[32];
    for (int64_t r = blockIdx.x; r < rows; r += gridDim.x) {
        const int c = count[r];
        const int64_t src = out_off[r], dst = r * n;
        int kept = 0;
        for (int base = 0; base < c; base += NT) {
            const int j = base + threadIdx.x;
            const float v = j < c ? (negate ? -scores[src + j] : scores[src + j]) : 0.f;
            const bool keep = j < c && (!positive || v > 0.f);
            int total;
            const int at = kept + block_rank<NT>(keep, s_warp, total);
            if (keep) { t_slot[dst + at] = (int32_t)slots[src + j]; t_val[dst + at] = v; }
            kept += total;
        }
        for (int j = kept + threadIdx.x; j < n; j += NT) { t_slot[dst + j] = -1; t_val[dst + j] = 0.f; }
        if (threadIdx.x == 0) t_cnt[r] = kept;
    }
}

// slots[r] = q0 + r: the stored rows of a range
__global__ void range_slots_kernel(int64_t *slots, int64_t rows, int64_t q0)
{
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r < rows) slots[r] = q0 + r;
}

// q[r] = X[slots[r]]: the query rows of stored vectors (fp32 values), one CTA per row
template <typename T>
__global__ void recall_gather_kernel(const T *X, int d, const int64_t *slots, int64_t rows, float *q)
{
    for (int64_t r = blockIdx.x; r < rows; r += gridDim.x)
        for (int e = threadIdx.x; e < d; e += blockDim.x) q[r * d + e] = row_val(X, slots[r] * d + e);
}

// the row tables of a chunk without exclusions: k = n, answers at q * n, one class in row order
__global__ void uniform_rows_kernel(int64_t rows, int64_t q0, int n, int32_t *k, int64_t *ex_off, int64_t *out_off, int64_t *order)
{
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r <= rows) ex_off[r] = 0;
    if (r < rows) { k[r] = n; out_off[r] = (q0 + r) * n; order[r] = r; }
}

size_t window_smem(int d) { return (size_t)SORT_CAP * 8 + (size_t)mma::CAP * 8 + (256 + 32 + 4) * 4 + (size_t)d * 4; }
size_t exact_smem(int d) { return (size_t)SORT_CAP * 12 + (256 + 32 + 4) * 4 + (size_t)d * 4; }


int32_t recall_rows(gorse_b200_index *ix, const uint8_t *allow, int64_t nq, const float *q_host, const int64_t *d_qslots, int32_t n,
                    const int64_t *excl_off, const int64_t *ex, const int64_t *ex_off, const Table *table, int64_t *slots_out,
                    float *scores_out, int32_t *count_out, int64_t *exact_rows_out)
{
    gorse_b200_ctx *c = ix->ctx;
    RecallWork &W = ix->recall;
    const int d = ix->d;
    auto out_at = [&](int64_t q) { return q * (int64_t)n + (excl_off ? excl_off[q] : 0); };
    const int64_t N = ix->n, total_out = out_at(nq);
    bool tensor = mma_path_eligible(ix, nq);
    const int64_t cq = std::min<int64_t>(nq, (int64_t)c->sm_count * mma::GROUP_ROWS * 8);
    // exact scratch: one [N] score row per CTA, at most 512 MB
    const int exact_grid = (int)std::max<int64_t>(1, std::min<int64_t>({(int64_t)c->sm_count * 2, cq, (512ll << 20) / (4 * N)}));
    int32_t st = GORSE_B200_OK;
    auto done = [&](int32_t s) {
        cudaStreamSynchronize(c->stream);
        cudaStreamSynchronize(c->copy_stream);
        return s;
    };
    if ((st = W.q.grow((size_t)cq * d)) || (st = W.k.grow((size_t)cq)) || (st = W.ex_off.grow((size_t)cq + 1)) || (st = W.out_off.grow((size_t)cq)) ||
        (st = W.rows.grow(2 * (size_t)cq)) || (st = W.count.grow((size_t)nq)) || (st = W.flags.grow(3)) ||
        (st = W.slots.grow((size_t)std::max<int64_t>(total_out, 1))) || (st = W.scores.grow((size_t)std::max<int64_t>(total_out, 1))) ||
        (st = W.scratch.grow((size_t)exact_grid * N)) || (st = W.ex.grow((size_t)std::max<int64_t>(excl_off ? ex_off[nq] : 0, 1))))
        return done(st);
    if (tensor && (st = mma_reserve(ix, cq))) {
        if (st != GORSE_B200_ERR_OOM) return done(st);
        tensor = false;   // no room for the mirror or the sweep's buffers: every row takes the exact kernel, with the same answers
    }
    const RowView X = ix->rows();
    cudaError_t e = with_rows(X, [&](auto x) {
        using T = row_elem_t<decltype(x)>;
        cudaError_t r = cudaFuncSetAttribute(recall_window_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)window_smem(d));
        if (r == cudaSuccess) r = cudaFuncSetAttribute(recall_exact_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)exact_smem(d));
        return r;
    });
    if (e == cudaSuccess) e = cudaMemsetAsync(W.flags.p, 0, 2 * sizeof(int), c->stream);
    if (e != cudaSuccess) { set_error("top-k: %s", cudaGetErrorString(e)); return done(GORSE_B200_ERR_CUDA); }
    int64_t host_exact = 0;
    size_t sweeps = 0;   // event pairs ix->ev[2 s], [2 s + 1] around sweep s
    std::vector<int32_t> &h_k = W.h_k;
    std::vector<int64_t> &h_exoff = W.h_exoff, &h_outoff = W.h_outoff, &h_rows = W.h_rows;
    std::vector<int8_t> &cls = W.h_cls;
    auto class_of = [&](int32_t k) {   // class N_CLASSES = the exact kernel
        int8_t cl = N_CLASSES;
        if (tensor)
            for (int8_t t = N_CLASSES - 1; t >= 0; t--)
                if (k <= CLASS_K[t]) cl = t;
        return cl;
    };
    for (int64_t q0 = 0; q0 < nq; q0 += cq) {
        const int64_t rows = std::min(cq, nq - q0);
        if (!q_host) {   // stored vectors: gathered from the collection in place of the upload
            with_rows(X, [&](auto x) {
                recall_gather_kernel<<<(unsigned)std::min<int64_t>(rows, (int64_t)c->sm_count * 16), 128, 0, c->stream>>>(x, d, d_qslots + q0, rows, W.q.p);
            });
            c->launches++;
        }
        if ((q_host && (e = cudaMemcpyAsync(W.q.p, q_host + q0 * d, sizeof(float) * rows * d, cudaMemcpyHostToDevice, c->stream)) != cudaSuccess) ||
            (e = cudaMemsetAsync(W.flags.p + 2, 0, sizeof(int), c->stream)) != cudaSuccess) {
            set_error("top-k upload: %s", cudaGetErrorString(e));
            return done(GORSE_B200_ERR_CUDA);
        }
        // rows grouped by class: class t holds rows W.rows[cls_begin[t] .. cls_begin[t + 1])
        int64_t cls_begin[N_CLASSES + 2] = {0};
        int cls_k[N_CLASSES] = {0};   // the largest k_q of each class
        if (!excl_off) {   // every row in one class, in row order; the tables are written on the device
            const int8_t t = class_of(n);
            for (int u = t + 1; u <= N_CLASSES + 1; u++) cls_begin[u] = rows;
            if (t < N_CLASSES) cls_k[t] = n;
            uniform_rows_kernel<<<div_up(rows + 1, 256), 256, 0, c->stream>>>(rows, q0, n, W.k.p, W.ex_off.p, W.out_off.p, W.rows.p);
            c->launches++;
        } else {
            h_k.resize(rows); h_exoff.resize(rows + 1); h_outoff.resize(rows); h_rows.resize(rows); cls.resize(rows);
            for (int64_t r = 0; r < rows; r++) {
                const int64_t q = q0 + r;
                h_k[r] = n + (int32_t)(excl_off[q + 1] - excl_off[q]);
                h_exoff[r] = ex_off[q] - ex_off[q0];
                h_outoff[r] = out_at(q);
                cls[r] = class_of(h_k[r]);
                cls_begin[cls[r] + 1]++;
                if (cls[r] < N_CLASSES) cls_k[cls[r]] = std::max(cls_k[cls[r]], h_k[r]);
            }
            h_exoff[rows] = ex_off[q0 + rows] - ex_off[q0];
            for (int t = 0; t <= N_CLASSES; t++) cls_begin[t + 1] += cls_begin[t];
            int64_t fill[N_CLASSES + 1];
            std::copy(cls_begin, cls_begin + N_CLASSES + 1, fill);
            for (int64_t r = 0; r < rows; r++) h_rows[fill[cls[r]]++] = r;
            const int64_t n_ex = h_exoff[rows];
            if ((e = cudaMemcpyAsync(W.k.p, h_k.data(), sizeof(int32_t) * rows, cudaMemcpyHostToDevice, c->stream)) != cudaSuccess ||
                (e = cudaMemcpyAsync(W.ex_off.p, h_exoff.data(), sizeof(int64_t) * (rows + 1), cudaMemcpyHostToDevice, c->stream)) != cudaSuccess ||
                (e = cudaMemcpyAsync(W.out_off.p, h_outoff.data(), sizeof(int64_t) * rows, cudaMemcpyHostToDevice, c->stream)) != cudaSuccess ||
                (e = cudaMemcpyAsync(W.rows.p, h_rows.data(), sizeof(int64_t) * rows, cudaMemcpyHostToDevice, c->stream)) != cudaSuccess ||
                (n_ex && (e = cudaMemcpyAsync(W.ex.p, ex + ex_off[q0], sizeof(int64_t) * n_ex, cudaMemcpyHostToDevice, c->stream)) != cudaSuccess)) {
                set_error("top-k upload: %s", cudaGetErrorString(e));
                return done(GORSE_B200_ERR_CUDA);
            }
        }
        host_exact += cls_begin[N_CLASSES + 1] - cls_begin[N_CLASSES];
        RowInfo R;
        R.q = W.q.p; R.k = W.k.p; R.ex_off = W.ex_off.p; R.ex = W.ex.p; R.out_off = W.out_off.p;
        R.exact = W.rows.p + cls_begin[N_CLASSES]; R.n_routed = cls_begin[N_CLASSES + 1] - cls_begin[N_CLASSES];
        R.self = q_host ? nullptr : d_qslots + q0;
        R.slots = W.slots.p; R.scores = W.scores.p; R.count = W.count.p + q0; R.flags = W.flags.p;
        for (int t = 0; t < N_CLASSES; t++) {
            const int64_t nr = cls_begin[t + 1] - cls_begin[t];
            if (nr == 0) continue;
            // the sample aims at 4 k columns per row, at most CAP / 2 so that a row's lists rarely overflow (Gamma(R_TOP) spread)
            const int m_tiles = mma_sample_tiles(ix, std::min(4.0 * cls_k[t], mma::CAP / 2.0));
            if (ix->ev.size() < 2 * sweeps + 2) {
                ix->ev.resize(2 * sweeps + 2, nullptr);
                if ((e = cudaEventCreate(&ix->ev[2 * sweeps])) != cudaSuccess || (e = cudaEventCreate(&ix->ev[2 * sweeps + 1])) != cudaSuccess) {
                    set_error("top-k events: %s", cudaGetErrorString(e));
                    return done(GORSE_B200_ERR_CUDA);
                }
            }
            if ((st = mma_sweep(ix, RowView{W.q.p, false}, nullptr, W.rows.p + cls_begin[t], 0, nr, m_tiles, ix->ev[2 * sweeps], ix->ev[2 * sweeps + 1])))
                return done(st);
            sweeps++;
            ix->stage1_flop += 2.0 * (double)nr * (double)N * (double)d;
            with_rows(X, [&](auto x) {
                recall_window_kernel<<<(unsigned)std::min<int64_t>(nr, (int64_t)c->sm_count * 16), WIN_THREADS, window_smem(d), c->stream>>>(
                    ix->w_ccol.p, ix->w_cval.p, ix->w_ccnt.p, ix->w_theta.p, ix->w_eps.p, ix->perm.p, allow, x, d, ix->metric,
                    W.rows.p + cls_begin[t], nr, R);
            });
            c->launches++;
        }
        with_rows(X, [&](auto x) {
            recall_exact_kernel<<<(unsigned)std::min<int64_t>(rows, exact_grid), EXACT_THREADS, exact_smem(d), c->stream>>>(
                x, N, d, ix->metric, allow, R, W.scratch.p);
        });
        c->launches++;
        const int64_t t0 = q0 * n;
        if (table) {
            table_kernel<128><<<(unsigned)std::min<int64_t>(rows, (int64_t)c->sm_count * 16), 128, 0, c->stream>>>(
                W.slots.p, W.scores.p, R.count, W.out_off.p, rows, n, table->negate, table->positive, table->slot + t0, table->val + t0,
                table->cnt + q0);
            c->launches++;
        }
        if ((e = cudaGetLastError()) != cudaSuccess) { set_error("top-k: %s", cudaGetErrorString(e)); return done(GORSE_B200_ERR_CUDA); }
        const bool h_table = table && table->h_slot;
        if (!slots_out && !h_table) continue;   // the caller reads the answers on the device
        // this chunk is final: download it on the copy stream while the next chunk computes
        const int64_t o0 = out_at(q0), o1 = out_at(q0 + rows);
        if ((e = cudaEventRecord(c->copy_ev, c->stream)) != cudaSuccess || (e = cudaStreamWaitEvent(c->copy_stream, c->copy_ev, 0)) != cudaSuccess ||
            (slots_out &&
             ((e = cudaMemcpyAsync(count_out + q0, W.count.p + q0, sizeof(int32_t) * rows, cudaMemcpyDeviceToHost, c->copy_stream)) != cudaSuccess ||
              (o1 > o0 && ((e = cudaMemcpyAsync(slots_out + o0, W.slots.p + o0, sizeof(int64_t) * (o1 - o0), cudaMemcpyDeviceToHost, c->copy_stream)) != cudaSuccess ||
                           (e = cudaMemcpyAsync(scores_out + o0, W.scores.p + o0, sizeof(float) * (o1 - o0), cudaMemcpyDeviceToHost, c->copy_stream)) != cudaSuccess)))) ||
            (h_table &&
             ((e = cudaMemcpyAsync(table->h_slot + t0, table->slot + t0, sizeof(int32_t) * rows * n, cudaMemcpyDeviceToHost, c->copy_stream)) != cudaSuccess ||
              (e = cudaMemcpyAsync(table->h_val + t0, table->val + t0, sizeof(float) * rows * n, cudaMemcpyDeviceToHost, c->copy_stream)) != cudaSuccess ||
              (e = cudaMemcpyAsync(table->h_cnt + q0, table->cnt + q0, sizeof(int32_t) * rows, cudaMemcpyDeviceToHost, c->copy_stream)) != cudaSuccess))) {
            set_error("top-k download: %s", cudaGetErrorString(e));
            return done(GORSE_B200_ERR_CUDA);
        }
    }
    int flags[2] = {0, 0};
    if ((e = cudaMemcpyAsync(flags, W.flags.p, sizeof(flags), cudaMemcpyDeviceToHost, c->stream)) != cudaSuccess ||
        (e = cudaStreamSynchronize(c->stream)) != cudaSuccess || (e = cudaStreamSynchronize(c->copy_stream)) != cudaSuccess) {
        set_error("top-k: %s", cudaGetErrorString(e));
        return done(GORSE_B200_ERR_CUDA);
    }
    for (size_t s = 0; s < sweeps; s++) {
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, ix->ev[2 * s], ix->ev[2 * s + 1]) == cudaSuccess) ix->stage1_ms += ms;
    }
    ix->last_fallback_rows += flags[1];
    if (flags[0]) { set_error("NaN distance"); return done(GORSE_B200_ERR_ARG); }
    if (exact_rows_out) *exact_rows_out = host_exact + flags[1];
    return done(GORSE_B200_OK);
}

}  // namespace recall

// the index's searches: rows from host vectors, a host list of stored rows, or the stored rows [q0, q0 + nq); the distances and
// int32 ids go through the pipeline's table (prune0 keeps distance > 0, bruteforce.go:58,78) into the host buffers
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
    DevBuf<int64_t> d_qidx;
    StreamSync sync{c->stream};
    GB_TRY(ix->r_idx.grow((size_t)nq * k));
    GB_TRY(ix->r_dist.grow((size_t)nq * k));
    GB_TRY(ix->r_count.grow((size_t)nq));
    if (!h_queries) {   // stored rows: a device slot list
        GB_TRY(d_qidx.alloc(nq));
        cudaError_t e = cudaSuccess;
        if (h_qidx) e = cudaMemcpyAsync(d_qidx.p, h_qidx, sizeof(int64_t) * nq, cudaMemcpyHostToDevice, c->stream);
        else {
            recall::range_slots_kernel<<<div_up(nq, 256), 256, 0, c->stream>>>(d_qidx.p, nq, q0);
            c->launches++;
        }
        if (e == cudaSuccess) e = cudaGetLastError();
        if (e != cudaSuccess) { set_error("search upload: %s", cudaGetErrorString(e)); return GORSE_B200_ERR_CUDA; }
    }
    const recall::Table table{ix->r_idx.p, ix->r_dist.p, ix->r_count.p, true, prune0 != 0, idx_out, dist_out, count_out};
    return recall::recall_rows(ix, nullptr, nq, h_queries, d_qidx.p, k, nullptr, nullptr, nullptr, &table, nullptr, nullptr, nullptr, nullptr);
}

// make room for `need` vectors (amortised doubling); the caller holds ix->mu
int32_t index_reserve(gorse_b200_index *ix, int64_t need)
{
    if (need <= ix->cap) return GORSE_B200_OK;
    cudaStream_t s = ix->ctx->stream;
    const int64_t ncap = std::max<int64_t>(need, ix->cap * 2);
    if (ix->value_bytes == 2) {
        DevBuf<uint16_t> nb;
        GB_TRY(nb.alloc((size_t)ncap * ix->d));
        if (ix->n) GB_CUDA(cudaMemcpyAsync(nb.p, ix->Xh.p, sizeof(uint16_t) * ix->n * ix->d, cudaMemcpyDeviceToDevice, s));
        GB_CUDA(cudaStreamSynchronize(s));
        ix->Xh = std::move(nb);
        ix->cap = ncap;
        return GORSE_B200_OK;
    }
    DevBuf<float> nb;
    GB_TRY(nb.alloc((size_t)ncap * ix->d));
    if (ix->n) GB_CUDA(cudaMemcpyAsync(nb.p, ix->X.p, sizeof(float) * ix->n * ix->d, cudaMemcpyDeviceToDevice, s));
    GB_CUDA(cudaStreamSynchronize(s));
    ix->X = std::move(nb);
    ix->cap = ncap;
    return GORSE_B200_OK;
}

// X[s] = src[map[s]] for m rows of d4 float4 (device to device)
__global__ void index_gather_rows_kernel(const float *Q, int d4, const int32_t *items, int64_t n, float *X)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t total = n * d4, st = (int64_t)gridDim.x * blockDim.x;
    for (; i < total; i += st) {
        const int64_t s = i / d4, c = i - s * d4;
        reinterpret_cast<float4 *>(X)[s * d4 + c] = reinterpret_cast<const float4 *>(Q)[(int64_t)items[s] * d4 + c];
    }
}

// ---- bf16 rows: narrowing on upload, widening on promotion -------------------------------------------------------------------
// narrowing keeps the high 16 bits; the value was bf16-exact iff the low 16 are zero
__device__ __forceinline__ bool narrow(float v, uint16_t &h)
{
    const uint32_t u = __float_as_uint(v);
    h = (uint16_t)(u >> 16);
    return (u & 0xffffu) != 0u;
}
__device__ __forceinline__ bool narrow(float4 v, uint2 &h)
{
    const uint32_t a = __float_as_uint(v.x), b = __float_as_uint(v.y), c = __float_as_uint(v.z), e = __float_as_uint(v.w);
    h.x = (a >> 16) | (b & 0xffff0000u);
    h.y = (c >> 16) | (e & 0xffff0000u);
    return ((a | b | c | e) & 0xffffu) != 0u;
}

// dst[s * dv + c] = narrow(src[(map ? map[s] : s) * dv + c]) for m rows; inexact[0] = 1 when a value is not bf16-exact.
// V / H = float4 / uint2 when d % 4 == 0 (dv = d / 4), else float / uint16_t (dv = d).
template <typename V, typename H>
__global__ void narrow_rows_kernel(const V *src, const int32_t *map, int64_t m, int dv, H *dst, int32_t *inexact)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t total = m * dv, st = (int64_t)gridDim.x * blockDim.x;
    bool bad = false;
    for (; i < total; i += st) {
        const int64_t s = i / dv, c = i - s * dv;
        bad |= narrow(src[(map ? (int64_t)map[s] : s) * dv + c], dst[i]);
    }
    if (bad) *inexact = 1;
}

// dst[i] = widen(src[i]) for count elements: promotion's one pass over the bf16 rows
template <typename H, typename V>
__global__ void widen_rows_kernel(const H *src, int64_t count, V *dst)
{
    const int64_t st = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += st) dst[i] = widen(src[i]);
}

cudaError_t index_narrow(int d, gorse_b200_ctx *c, cudaStream_t s, const float *src, const int32_t *map, int64_t m, uint16_t *dst,
                         int32_t *inexact)
{
    if (m == 0) return cudaSuccess;
    const unsigned grid = (unsigned)std::min<int64_t>(div_up(m * d, 256), (int64_t)c->sm_count * 8);
    if (d % 4 == 0)
        narrow_rows_kernel<<<grid, 256, 0, s>>>(reinterpret_cast<const float4 *>(src), map, m, d / 4, reinterpret_cast<uint2 *>(dst), inexact);
    else
        narrow_rows_kernel<<<grid, 256, 0, s>>>(src, map, m, d, dst, inexact);
    c->launches++;
    return cudaGetLastError();
}

// dst[0, rows * d) = the widened bf16 rows src, on the context's stream
static cudaError_t widen_rows(gorse_b200_ctx *c, int d, const uint16_t *src, int64_t rows, float *dst)
{
    if (rows == 0) return cudaSuccess;
    const unsigned grid = (unsigned)c->sm_count * 8;
    if (d % 4 == 0)
        widen_rows_kernel<<<grid, 256, 0, c->stream>>>(reinterpret_cast<const uint2 *>(src), rows * d / 4, reinterpret_cast<float4 *>(dst));
    else
        widen_rows_kernel<<<grid, 256, 0, c->stream>>>(src, rows * d, dst);
    c->launches++;
    return cudaGetLastError();
}

int32_t index_promote(gorse_b200_index *ix, int64_t rows)
{
    if (ix->value_bytes == 4) return GORSE_B200_OK;
    gorse_b200_ctx *c = ix->ctx;
    DevBuf<float> nx;
    if (nx.alloc((size_t)ix->cap * ix->d)) {   // the documented code of a promotion that cannot allocate
        set_error("promotion to fp32: cannot allocate %lld bytes", (long long)(4 * ix->cap * ix->d));
        return GORSE_B200_ERR_CUDA;
    }
    cudaError_t e = widen_rows(c, ix->d, ix->Xh.p, rows, nx.p);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
    if (e != cudaSuccess) { set_error("promote: %s", cudaGetErrorString(e)); return GORSE_B200_ERR_CUDA; }
    ix->X = std::move(nx);
    ix->Xh.free();
    ix->stage.free();
    ix->value_bytes = 4;
    return GORSE_B200_OK;
}

// copies m fp32 rows (row s = src[(map ? map[s] : s) * d ..], host or device) into the fp32 rows dst on the context's stream
static cudaError_t copy_rows_f32(gorse_b200_index *ix, const float *src, const int32_t *map, const int32_t *h_map, int64_t m, bool host, float *dst)
{
    gorse_b200_ctx *c = ix->ctx;
    const int d = ix->d;
    if (!map) return cudaMemcpyAsync(dst, src, sizeof(float) * m * d, host ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice, c->stream);
    cudaError_t e = cudaSuccess;
    if (d % 4 == 0) {
        index_gather_rows_kernel<<<c->sm_count * 8, 256, 0, c->stream>>>(src, d / 4, map, m, dst);
        c->launches++;
        e = cudaGetLastError();
    } else
        for (int64_t s = 0; s < m && e == cudaSuccess; s++)
            e = cudaMemcpyAsync(dst + s * d, src + (int64_t)h_map[s] * d, sizeof(float) * d, cudaMemcpyDeviceToDevice, c->stream);
    return e;
}

int32_t index_append(gorse_b200_index *ix, const float *src, const int32_t *map, int64_t m, bool host)
{
    if (m == 0) return GORSE_B200_OK;
    gorse_b200_ctx *c = ix->ctx;
    const int d = ix->d;
    const int64_t n = ix->n, need = n + m;
    std::vector<int32_t> h_map;
    if (map && d % 4 != 0) {   // the row-by-row copy of an fp32 target reads the map on the host
        h_map.resize((size_t)m);
        GB_CUDA(cudaMemcpyAsync(h_map.data(), map, sizeof(int32_t) * m, cudaMemcpyDeviceToHost, c->stream));
        GB_CUDA(cudaStreamSynchronize(c->stream));
    }
    if (ix->value_bytes == 4) {
        GB_TRY(index_reserve(ix, need));
        GB_CUDA(copy_rows_f32(ix, src, map, h_map.data(), m, host, ix->X.p + n * d));
        GB_CUDA(cudaStreamSynchronize(c->stream));
        ix->n = need;
        ix->mma_ready = false;  // bf16 mirror and norms are rebuilt lazily
        return GORSE_B200_OK;
    }
    // bf16: every chunk is narrowed into the free rows past n (or into a grown copy) on the stream, with no wait in between;
    // one flag covers the call and is read at the end.  If a value was not exact, the narrowed rows are dropped: the stored
    // rows are widened into new fp32 rows and the call's rows are copied in again from the caller's source.  The index takes
    // the new buffers only at the end, so every error leaves it as it was.
    const int64_t ncap = need > ix->cap ? std::max<int64_t>(need, ix->cap * 2) : ix->cap;
    const int64_t R = host ? std::max<int64_t>(1, APPEND_STAGE_BYTES / 4 / d) : m;   // rows per chunk
    DevBuf<uint16_t> nh;
    StreamSync sync{c->stream};
    GB_TRY(ix->inexact.grow(1));
    if (host) GB_TRY(ix->stage.grow((size_t)std::min(R, m) * d));
    uint16_t *th = ix->Xh.p;
    if (ncap > ix->cap) {
        GB_TRY(nh.alloc((size_t)ncap * d));
        if (n) GB_CUDA(cudaMemcpyAsync(nh.p, ix->Xh.p, sizeof(uint16_t) * n * d, cudaMemcpyDeviceToDevice, c->stream));
        th = nh.p;
    }
    GB_CUDA(cudaMemsetAsync(ix->inexact.p, 0, sizeof(int32_t), c->stream));
    for (int64_t j0 = 0; j0 < m; j0 += R) {   // stream order keeps chunk k + 1's upload behind chunk k's narrowing
        const int64_t rows = std::min(R, m - j0);
        if (host) GB_CUDA(cudaMemcpyAsync(ix->stage.p, src + j0 * d, sizeof(float) * rows * d, cudaMemcpyHostToDevice, c->stream));
        GB_CUDA(index_narrow(d, c, c->stream, host ? ix->stage.p : src, map ? map + j0 : nullptr, rows, th + (n + j0) * d, ix->inexact.p));
    }
    int32_t inexact = 0;
    GB_CUDA(cudaMemcpyAsync(&inexact, ix->inexact.p, sizeof(int32_t), cudaMemcpyDeviceToHost, c->stream));
    GB_CUDA(cudaStreamSynchronize(c->stream));
    if (inexact) {   // promote: the stored rows [0, n) are exact (Xh holds them), the call's rows come from the source
        nh.free();   // before the fp32 rows exist: an empty collection never holds both
        DevBuf<float> nf;
        if (nf.alloc((size_t)ncap * d)) {
            set_error("promotion to fp32: cannot allocate %lld bytes", (long long)(4 * ncap * d));
            return GORSE_B200_ERR_CUDA;
        }
        GB_CUDA(widen_rows(c, d, ix->Xh.p, n, nf.p));
        GB_CUDA(copy_rows_f32(ix, src, map, h_map.data(), m, host, nf.p + n * d));
        GB_CUDA(cudaStreamSynchronize(c->stream));
        ix->X = std::move(nf);
        ix->Xh.free();
        ix->stage.free();   // an fp32 index adds without staging
        ix->value_bytes = 4;
    } else if (nh.p)
        ix->Xh = std::move(nh);
    ix->cap = ncap;
    ix->n = need;
    ix->mma_ready = false;
    return GORSE_B200_OK;
}

int32_t index_download_rows(gorse_b200_index *ix, const int64_t *rows, int64_t n, float *out)
{
    gorse_b200_ctx *c = ix->ctx;
    const int64_t d = ix->d;
    if (ix->value_bytes == 4) {   // one copy per row, straight into the caller's buffer
        for (int64_t i = 0; i < n; i++)
            if (rows[i] >= 0)
                GB_CUDA(cudaMemcpyAsync(out + i * d, ix->X.p + rows[i] * d, sizeof(float) * d, cudaMemcpyDeviceToHost, c->stream));
        GB_CUDA(cudaStreamSynchronize(c->stream));
        return GORSE_B200_OK;
    }
    // bf16: the rows' bits into a host buffer, one copy per row, then widened on the host (bits << 16, exact)
    std::vector<uint16_t> h;
    std::vector<int64_t> at;
    for (int64_t i = 0; i < n; i++)
        if (rows[i] >= 0) at.push_back(i);
    h.resize(at.size() * (size_t)d);
    for (size_t j = 0; j < at.size(); j++)
        GB_CUDA(cudaMemcpyAsync(h.data() + j * d, ix->Xh.p + rows[at[j]] * d, sizeof(uint16_t) * d, cudaMemcpyDeviceToHost, c->stream));
    GB_CUDA(cudaStreamSynchronize(c->stream));
    for (size_t j = 0; j < at.size(); j++) {
        uint32_t *o = reinterpret_cast<uint32_t *>(out + at[j] * d);
        for (int64_t e = 0; e < d; e++) o[e] = (uint32_t)h[j * d + e] << 16;
    }
    return GORSE_B200_OK;
}

// Xn[scan[s]] = X[s] for every live slot s (scan[s + 1] != scan[s]); V = float4 when d % 4 == 0, one V per thread (bf16 rows:
// uint2, 4 values, or uint16_t)
template <typename V>
__global__ void index_compact_rows_kernel(const V *X, int64_t n, int dv, const int64_t *scan, V *Xn)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t total = n * dv, st = (int64_t)gridDim.x * blockDim.x;
    for (; i < total; i += st) {
        const int64_t s = i / dv, c = i - s * dv, to = scan[s];
        if (scan[s + 1] != to) Xn[to * dv + c] = X[i];
    }
}

// the live rows of one element type into a new buffer nx: T = float (V4 = float4) or uint16_t (V4 = uint2)
template <typename T, typename V4>
static int32_t compact_rows(gorse_b200_index *ix, const T *X, const int64_t *scan, int64_t live, DevBuf<T> &nx)
{
    gorse_b200_ctx *c = ix->ctx;
    GB_TRY(nx.alloc((size_t)live * ix->d));
    cudaError_t e = cudaSuccess;
    if (live > 0) {
        const unsigned grid = (unsigned)c->sm_count * 8;
        if (ix->d % 4 == 0)
            index_compact_rows_kernel<<<grid, 256, 0, c->stream>>>(reinterpret_cast<const V4 *>(X), ix->n, ix->d / 4, scan,
                                                                   reinterpret_cast<V4 *>(nx.p));
        else
            index_compact_rows_kernel<<<grid, 256, 0, c->stream>>>(X, ix->n, ix->d, scan, nx.p);
        c->launches++;
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
    if (e != cudaSuccess) {
        set_error("compact: %s", cudaGetErrorString(e));
        return GORSE_B200_ERR_CUDA;
    }
    return GORSE_B200_OK;
}

int32_t index_compact(gorse_b200_index *ix, const int64_t *scan, int64_t live)
{
    if (ix->value_bytes == 2) {   // bf16 rows stay bf16
        DevBuf<uint16_t> nx;
        GB_TRY((compact_rows<uint16_t, uint2>(ix, ix->Xh.p, scan, live, nx)));
        ix->Xh = std::move(nx);
    } else {
        DevBuf<float> nx;
        GB_TRY((compact_rows<float, float4>(ix, ix->X.p, scan, live, nx)));
        ix->X = std::move(nx);
    }
    ix->n = ix->cap = live;
    ix->mma_ready = false;   // the next sweep rebuilds the mirror, norms and permutation for the new n
    ix->Xb.free(); ix->norm.free(); ix->perm.free();
    ix->recall.scratch.free();   // [N] per exact CTA
    ix->stage.free();            // the next bf16 add allocates its upload staging again
    ix->last_fallback_rows = 0;
    ix->stage1_ms = ix->stage1_flop = 0.0;
    return GORSE_B200_OK;
}

size_t index_bytes(const gorse_b200_index *ix)
{
    return ix->X.bytes() + ix->Xh.bytes() + ix->stage.bytes() + ix->inexact.bytes() + ix->Xb.bytes() + ix->norm.bytes() + ix->perm.bytes() +
           ix->w_qb.bytes() + ix->w_eps.bytes() + ix->w_cval.bytes() + ix->w_theta.bytes() + ix->w_ccol.bytes() + ix->w_ccnt.bytes() +
           ix->recall.bytes() + ix->r_idx.bytes() + ix->r_count.bytes() + ix->r_dist.bytes();
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
    for (cudaEvent_t e : ix->ev)
        if (e) cudaEventDestroy(e);
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
        GB_TRY(index_append(ix, vectors, nullptr, n, true));
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
// since the last call: device time and algorithmic flop (2 * nq * N * d) of the stage-1 tensor-core kernels, and the rows
// whose candidate set failed certification (the window kernel handed them to the exact kernel)
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
// out[(q - q0) * n + x], and (eps_out != NULL) each row's error margin eps.  Small problems only (one sweep of all rows).
int32_t gorse_b200_index_stage1_scores(gorse_b200_index *ix, int64_t q0, int64_t q1, float *out, float *eps_out)
{
    GB_CHECK_ARG(ix != nullptr && out != nullptr, "NULL argument");
    std::lock_guard<std::mutex> lk(ix->mu);
    GB_CHECK_ARG(q0 >= 0 && q1 > q0 && q1 <= ix->n, "bad range");
    ScopedDevice sd(ix->ctx->device);
    gorse_b200_ctx *c = ix->ctx;
    const int64_t nq = q1 - q0, n_cols = (ix->n + 127) / 128 * 128;
    DevBuf<float> dense;
    int32_t st;
    auto done = [&](int32_t s) { cudaStreamSynchronize(c->stream); ix->dbg_scores = nullptr; return s; };
    if ((st = dense.alloc((size_t)nq * n_cols)) || (st = mma_reserve(ix, nq))) return done(st);
    ix->dbg_scores = dense.p;
    if ((st = mma_sweep(ix, ix->rows(), nullptr, nullptr, q0, nq, mma_sample_tiles(ix, 4.0), nullptr, nullptr))) return done(st);
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
