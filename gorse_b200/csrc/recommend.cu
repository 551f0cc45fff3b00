// recommend.cu -- batched offline recommendation: gorse_b200_recommend.
//
// The worker's offline loop (Pipeline.Recommend, worker/pipeline.go:124-319) runs, per user, the CF recall, the recommenders
// in the configured order with one growing exclude set (Recommender.RecommendSequential, logics/recommend.go:135-156), the
// candidate list, the replacement items, the FM ranking and the replacement decay.  Here one call does that for many users,
// and the exclude sets and candidate lists never leave the device between stages:
//
//   once per call    the CF recall rows (recall::recall_rows with E0 mapped to CF slots), and the neighbour table of every
//                    item-to-item / user-to-user stage (neighbour_table, stages.cuh), each on the distinct rows of the batch.
//   per chunk        users in chunks of at most sm_count * 1024, every buffer laid out by host-known bounds, so no chunk waits
//                    for a device count:
//     rec_grow_kernel     E_u (sorted item indices, padded with PAD to the host-known capacity) and, per item-to-item stage,
//                         the same set in that collection's slots: E0 expanded, and after every stage the union with the
//                         items the stage appended (sorted and deduplicated in shared memory, merged by binary search).
//     rec_list_kernel     a list stage: the entries not in E_u, appended in order (ordered compaction with block_rank).
//     rec_cf_kernel       the collaborative stage: the CF row mapped to items, live items only, cut at n, then minus E_u.
//     i2i / u2u aggregate the existing stage-B kernels (i2i_aggregate_kernel, u2u_route_kernel, u2u_aggregate_kernel) with
//                         the device exclude sets; rec_append_kernel maps their rows to items and appends them.
//     rec_assemble_kernel the candidates minus non-live items, in order, then the replacement items that are live and not
//                         yet candidates.
//     FM                  rec_scan_kernel (candidate offsets), rec_pack_kernel (contiguous candidates, D_u, attention chunk
//                         table), then fm::rank_pass: the existing fm_pair_kernel, fm_attn_kernel and fm_sort_kernel.
//     rec_emit_kernel     the replacement decay in float64 and, when it touched a score, the re-sort on (float64 score desc,
//                         position asc) with 128-bit keys; else the FM order.
//   A finished chunk is downloaded on the copy stream while the next one computes (two output buffers, alternating).
#include <algorithm>

#include "fm.cuh"
#include "stages.cuh"
#include "topk.cuh"

namespace gb {
namespace rec {

using u128 = unsigned __int128;
constexpr int NT = 256;
constexpr int MAX_LIST = 4096;                    // a stage's appended items are sorted in shared memory
constexpr int64_t PAD = INT64_MAX;                // the padding of an exclude set: above every item and slot
constexpr int64_t CHUNK_ENTRIES = int64_t(1) << 26;   // candidate / exclude-set entries of one chunk (bounds its buffers)

// ascending bitonic sort of key[0, p), p a power of two, by the whole CTA
template <typename K>
__device__ void bitonic(K *key, int p)
{
    for (int size = 2; size <= p; size <<= 1)
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            for (int i = threadIdx.x; i < p / 2; i += NT) {
                const int lo = 2 * i - (i & (stride - 1)), hi = lo + stride;
                const bool up = (lo & size) == 0;
                const K a = key[lo], b = key[hi];
                if ((a > b) == up) { key[lo] = b; key[hi] = a; }
            }
            __syncthreads();
        }
}

// first index of a[0, n) that is >= v (a ascending)
__device__ __forceinline__ int64_t lower(const int64_t *a, int64_t n, int64_t v)
{
    int64_t lo = 0, hi = n;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (a[mid] < v) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

// out row u = in row u (ascending, padded with PAD or packed) united with the candidates [start[u], cnt[u]) of row u (through
// map when given, -1 dropped), padded with PAD to out's capacity.  cand == nullptr: a copy.  The new items are not in row u.
__global__ void __launch_bounds__(NT) rec_grow_kernel(const int64_t *in, const int64_t *in_off, int64_t *out, const int64_t *out_off,
                                                      const int32_t *cand, const int64_t *cand_off, const int32_t *start, const int32_t *cnt,
                                                      const int64_t *map, int64_t rows)
{
    __shared__ int64_t s_new[MAX_LIST];
    __shared__ int s_warp[32];
    for (int64_t u = blockIdx.x; u < rows; u += gridDim.x) {
        const int64_t *a = in + in_off[u];
        const int64_t a_cap = in_off[u + 1] - in_off[u];
        int64_t *o = out + out_off[u];
        const int64_t o_cap = out_off[u + 1] - out_off[u];
        const int m = cand ? cnt[u] - start[u] : 0;
        const int p = recall::pow2_at_least(max(m, 1));
        for (int j = threadIdx.x; j < p; j += NT) {
            int64_t v = PAD;
            if (j < m) {
                v = cand[cand_off[u] + start[u] + j];
                if (map) v = map[v] < 0 ? PAD : map[v];
            }
            s_new[j] = v;
        }
        __syncthreads();
        bitonic<int64_t>(s_new, p);
        // duplicates become PAD, a second sort moves them behind the distinct items
        int dup = 0;
        for (int j = threadIdx.x; j < p; j += NT) dup |= j > 0 && s_new[j] != PAD && s_new[j] == s_new[j - 1];
        if (__syncthreads_or(dup)) {
            int64_t mine[MAX_LIST / NT];
            for (int j = threadIdx.x, t = 0; j < p; j += NT, t++) mine[t] = j > 0 && s_new[j] == s_new[j - 1] ? PAD : s_new[j];
            __syncthreads();
            for (int j = threadIdx.x, t = 0; j < p; j += NT, t++) s_new[j] = mine[t];
            __syncthreads();
            bitonic<int64_t>(s_new, p);
        }
        int distinct = 0;
        for (int j = threadIdx.x; j < p; j += NT) distinct += s_new[j] != PAD;
        distinct = recall::block_sum<NT>(distinct, s_warp);
        const int64_t na = lower(a, a_cap, PAD);
        for (int64_t i = threadIdx.x; i < na; i += NT) o[i + lower(s_new, distinct, a[i])] = a[i];
        for (int j = threadIdx.x; j < distinct; j += NT) o[j + lower(a, na, s_new[j])] = s_new[j];
        for (int64_t i = na + distinct + threadIdx.x; i < o_cap; i += NT) o[i] = PAD;
        __syncthreads();
    }
}

// a list stage: entries of the shared list (off == nullptr) or of row u0 + u of the per-user lists, not in E_u, appended
__global__ void __launch_bounds__(NT) rec_list_kernel(const int32_t *items, const double *scores, const int64_t *off, int64_t len, int64_t u0,
                                                      const int64_t *E, const int64_t *E_off, int32_t *cand, double *cscore,
                                                      const int64_t *cand_off, int32_t *cnt, int64_t rows)
{
    __shared__ int s_warp[32];
    for (int64_t u = blockIdx.x; u < rows; u += gridDim.x) {
        const int64_t b = off ? off[u0 + u] : 0, n = off ? off[u0 + u + 1] - b : len;
        const int64_t *e = E + E_off[u], ne = E_off[u + 1] - E_off[u];
        int kept = cnt[u];
        for (int64_t base = 0; base < n; base += NT) {
            const int64_t j = base + threadIdx.x;
            const int32_t it = j < n ? items[b + j] : 0;
            const bool f = j < n && !recall::contains(e, ne, (int64_t)it);
            int total;
            const int pos = kept + recall::block_rank<NT>(f, s_warp, total);
            if (f) {
                cand[cand_off[u] + pos] = it;
                cscore[cand_off[u] + pos] = scores[b + j];
            }
            kept += total;
        }
        __syncthreads();
        if (threadIdx.x == 0) cnt[u] = kept;
    }
}

// the collaborative stage: CF row u0 + u (slots, float scores, at row_at(u0 + u)) through item_of_slot, live items only, the
// first n of them, then the ones not in E_u, appended
__global__ void __launch_bounds__(NT) rec_cf_kernel(const int64_t *slots, const float *scores, const int32_t *rcount, const int64_t *excl_off,
                                                    int n, int64_t u0, const int32_t *item_of_slot, const uint8_t *live, const int64_t *E,
                                                    const int64_t *E_off, int32_t *cand, double *cscore, const int64_t *cand_off, int32_t *cnt,
                                                    int64_t rows)
{
    __shared__ int s_warp[32];
    for (int64_t u = blockIdx.x; u < rows; u += gridDim.x) {
        const int64_t g = u0 + u, r0 = g * n + excl_off[g];
        const int c = rcount[g];
        const int64_t *e = E + E_off[u], ne = E_off[u + 1] - E_off[u];
        int seen = 0, kept = cnt[u];
        for (int base = 0; base < c && seen < n; base += NT) {
            const int j = base + threadIdx.x;
            const int32_t it = j < c ? item_of_slot[slots[r0 + j]] : -1;
            const bool ok = it >= 0 && live[it];
            int t1, t2;
            const int r1 = recall::block_rank<NT>(ok, s_warp, t1);
            const bool f = ok && seen + r1 < n && !recall::contains(e, ne, (int64_t)it);
            const int pos = kept + recall::block_rank<NT>(f, s_warp, t2);
            if (f) {
                cand[cand_off[u] + pos] = it;
                cscore[cand_off[u] + pos] = (double)scores[r0 + j];
            }
            seen += t1;
            kept += t2;
        }
        __syncthreads();
        if (threadIdx.x == 0) cnt[u] = kept;
    }
}

// an item-to-item / user-to-user row (u * n, rcount[u] entries; slots through item_of_slot when given), appended whole
__global__ void rec_append_kernel(const int64_t *ids, const double *scores, const int32_t *rcount, int n, const int32_t *item_of_slot,
                                  int32_t *cand, double *cscore, const int64_t *cand_off, int32_t *cnt, int64_t rows)
{
    for (int64_t u = blockIdx.x; u < rows; u += gridDim.x) {
        const int c = rcount[u], k = cnt[u];
        for (int j = threadIdx.x; j < c; j += blockDim.x) {
            const int64_t id = ids[u * n + j];
            cand[cand_off[u] + k + j] = item_of_slot ? item_of_slot[id] : (int32_t)id;
            cscore[cand_off[u] + k + j] = scores[u * n + j];
        }
        __syncthreads();
        if (threadIdx.x == 0) cnt[u] = k + c;
    }
}

// the candidates minus the non-live items, in order; then (repl_off != nullptr) the live replacement items of row u0 + u
// that are not candidates, in order, with score 0
__global__ void __launch_bounds__(NT) rec_assemble_kernel(const uint8_t *live, const int64_t *repl_off, const int32_t *repl_items, int64_t u0,
                                                          int32_t *cand, double *cscore, const int64_t *cand_off, int32_t *cnt, int64_t rows)
{
    __shared__ int s_warp[32];
    for (int64_t u = blockIdx.x; u < rows; u += gridDim.x) {
        int32_t *ci = cand + cand_off[u];
        double *cs = cscore + cand_off[u];
        const int c = cnt[u];
        int kept = 0;
        for (int base = 0; base < c; base += NT) {
            const int j = base + threadIdx.x;
            const int32_t it = j < c ? ci[j] : 0;
            const double s = j < c ? cs[j] : 0.0;
            const bool f = j < c && live[it];
            int total;
            const int pos = kept + recall::block_rank<NT>(f, s_warp, total);   // reads before writes: block_rank syncs
            if (f) { ci[pos] = it; cs[pos] = s; }
            kept += total;
        }
        __syncthreads();
        if (repl_off) {
            const int64_t rb = repl_off[u0 + u], rn = repl_off[u0 + u + 1] - rb;
            const int base_cands = kept;
            for (int64_t base = 0; base < rn; base += NT) {
                const int64_t j = base + threadIdx.x;
                const int32_t it = j < rn ? repl_items[rb + j] : 0;
                bool f = j < rn && live[it];
                for (int t = 0; f && t < base_cands; t++) f = ci[t] != it;
                int total;
                const int pos = kept + recall::block_rank<NT>(f, s_warp, total);
                if (f) { ci[pos] = it; cs[pos] = 0.0; }
                kept += total;
            }
            __syncthreads();
        }
        if (threadIdx.x == 0) cnt[u] = kept;
    }
}

// exclusive prefix sums of cnt[0, rows) into off[0, rows] (one CTA of 1024 threads)
__global__ void __launch_bounds__(1024) rec_scan_kernel(const int32_t *cnt, int64_t rows, int64_t *off)
{
    __shared__ int64_t s[1024];
    const int64_t per = (rows + 1023) / 1024, b = threadIdx.x * per, e = min(rows, b + per);
    int64_t sum = 0;
    for (int64_t i = b; i < e; i++) sum += cnt[i];
    s[threadIdx.x] = sum;
    __syncthreads();
    for (int o = 1; o < 1024; o <<= 1) {
        const int64_t t = threadIdx.x >= o ? s[threadIdx.x - o] : 0;
        __syncthreads();
        s[threadIdx.x] += t;
        __syncthreads();
    }
    int64_t run = s[threadIdx.x] - sum;
    for (int64_t i = b; i < e; i++) {
        off[i] = run;
        run += cnt[i];
    }
    if (threadIdx.x == 1023) off[rows] = s[1023];
}

// one warp per user: the candidates made contiguous at off[u], D_u = max(num_dim, the user's row + the longest item row),
// and the user's attention chunks at ch_off[u] .. ch_off[u + 1] (host-known count; chunks past the candidates have 0 rows)
__global__ void rec_pack_kernel(const int32_t *cand, const int64_t *cand_off, const int32_t *cnt, const int64_t *off, const int32_t *u_len,
                                const int32_t *i_len, int num_dim, int32_t *packed, int32_t *dims, const int64_t *ch_off, int batch,
                                int64_t *ch_start, int32_t *ch_rows, int64_t rows)
{
    const int lane = threadIdx.x & 31;
    const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t u = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); u < rows; u += warps) {
        const int c = cnt[u];
        int longest = 0;
        for (int j = lane; j < c; j += 32) {
            const int32_t it = cand[cand_off[u] + j];
            packed[off[u] + j] = it;
            longest = max(longest, i_len[it]);
        }
        for (int o = 16; o; o >>= 1) longest = max(longest, __shfl_xor_sync(0xffffffffu, longest, o));
        if (lane == 0) dims[u] = max(num_dim, u_len[u] + longest);
        if (ch_off)
            for (int64_t j = lane; j < ch_off[u + 1] - ch_off[u]; j += 32) {
                ch_start[ch_off[u] + j] = off[u] + j * batch;
                ch_rows[ch_off[u] + j] = (int32_t)max((int64_t)0, min((int64_t)batch, (int64_t)c - j * batch));
            }
    }
}

// order-preserving key of a float64 score, -0 == +0, NaN lowest
__device__ __forceinline__ uint64_t score_key(double v)
{
    if (v != v) return 0;
    if (v == 0.0) v = 0.0;
    const uint64_t b = (uint64_t)__double_as_longlong(v);
    return (b >> 63) ? ~b : (b | (1ull << 63));
}

// the ranked row of user u: FM scores through float64 with the replacement decay; the FM order, or a re-sort by (score desc,
// position asc) when a decay was applied.  sort: per-CTA global scratch of sort_stride 128-bit keys.
__global__ void __launch_bounds__(NT) rec_emit_kernel(const int32_t *packed, const int64_t *off, const float *score, const int32_t *order,
                                                      const int64_t *repl_off, const int32_t *repl_items, const uint8_t *repl_pos, int64_t u0,
                                                      double pos_decay, double read_decay, double *dscore, u128 *sort, int64_t sort_stride,
                                                      const int64_t *out_off, int32_t *out_items, double *out_scores, int32_t *out_cnt,
                                                      int64_t rows)
{
    u128 *key = sort + (int64_t)blockIdx.x * sort_stride;
    for (int64_t u = blockIdx.x; u < rows; u += gridDim.x) {
        const int64_t c0 = off[u];
        const int n = (int)(off[u + 1] - c0);
        const int64_t rb = repl_off ? repl_off[u0 + u] : 0, rn = repl_off ? repl_off[u0 + u + 1] - rb : 0;
        int touched = 0;
        for (int p = threadIdx.x; p < n; p += NT) {
            const int32_t it = packed[c0 + p];
            double s = (double)score[c0 + p];
            for (int64_t t = 0; t < rn; t++)
                if (repl_items[rb + t] == it) {   // every candidate is live: applyReplacementDecay's sets hold live items only
                    s = __dmul_rn(s, repl_pos[rb + t] ? pos_decay : read_decay);
                    touched = 1;
                    break;
                }
            dscore[c0 + p] = s;
        }
        int32_t *oi = out_items + out_off[u];
        double *os = out_scores + out_off[u];
        if (__syncthreads_or(touched)) {
            const int p2 = recall::pow2_at_least(max(n, 1));
            for (int p = threadIdx.x; p < p2; p += NT) key[p] = p < n ? ((u128)~score_key(dscore[c0 + p]) << 64) | (uint32_t)p : ~(u128)0;
            __syncthreads();
            bitonic<u128>(key, p2);
            for (int i = threadIdx.x; i < n; i += NT) {
                const int p = (int)(uint32_t)key[i];
                oi[i] = packed[c0 + p];
                os[i] = dscore[c0 + p];
            }
        } else {
            for (int i = threadIdx.x; i < n; i += NT) {
                const int p = order[c0 + i];
                oi[i] = packed[c0 + p];
                os[i] = dscore[c0 + p];
            }
        }
        if (threadIdx.x == 0) out_cnt[u] = n;
        __syncthreads();
    }
}

template <typename T>
using Buf = DevBuf<T>;   // grow-only, kept with the context between calls

// the device buffers of gorse_b200_recommend, grow-only and kept with the context (the global accumulator rows are zero
// between calls: the aggregation kernels clear what they touch), so a worker's batches do not allocate
struct Work {
    std::mutex mu;                           // one call at a time per context
    Buf<uint8_t> d_live, d_repl_pos;
    Buf<int32_t> d_repl_items, d_cf_item_of_slot, d_u_len, d_i_len;
    Buf<int64_t> d_repl_off, d_cf_excl_off;
    struct List { Buf<int32_t> items; Buf<double> scores; Buf<int64_t> off; };
    std::vector<List> lists;                 // per list stage
    std::vector<NeighbourStage> sd;          // per item-to-item / user-to-user stage
    Buf<int64_t> d_cand_off, d_E_off, d_e0_off, d_e0, d_E[2], d_fm_off, d_ch_off, d_rids;
    Buf<int32_t> d_cand, d_cnt, d_start, d_rcount, d_out_items[2], d_out_cnt[2], d_dims;
    Buf<double> d_cscore, d_rscore, d_dscore, d_out_scores[2];
    Buf<u128> d_sort;
};

std::mutex work_mu;   // guards the creation of a context's Work

Work *work(gorse_b200_ctx *ctx)
{
    std::lock_guard<std::mutex> lk(work_mu);
    if (!ctx->rec_work) ctx->rec_work = new (std::nothrow) Work();
    return ctx->rec_work;
}

}  // namespace rec

void recommend_work_free(gorse_b200_ctx *ctx)
{
    delete ctx->rec_work;
    ctx->rec_work = nullptr;
}

}  // namespace gb

namespace gb {
namespace rec {

// one call: its arguments, what its phases hand on to each other, and the phases
struct Call {
    gorse_b200_ctx *ctx;
    int64_t n_users;
    const int64_t *excl_off;
    const int32_t *excl_items;
    int32_t n_items;
    const uint8_t *item_live;
    int32_t n_stages;
    const gorse_b200_recommend_stage *stages;
    const gorse_b200_recommend_cf *cf;
    const gorse_b200_recommend_ranker *ranker;
    const int64_t *repl_off;
    const int32_t *repl_items;
    const uint8_t *repl_positive;
    double positive_decay, read_decay;
    int32_t *items_out;
    double *scores_out;
    int32_t *count_out;
    // checks
    bool with_repl = false;
    gorse_b200_fm *m = nullptr;
    std::vector<int64_t> e0, e0_off;         // E0: each user's items once, sorted, -1 dropped
    std::vector<int64_t> bound, cap;         // per user: the most candidates, and the most exclude-set entries a stage reads
    std::vector<int32_t> u_len, i_len;       // the ranker's row lengths, for D_u
    std::vector<std::unique_lock<std::mutex>> locks;   // the collections, each locked once, in address order
    std::unique_lock<std::mutex> fm_lock;
    // tables, CF recall and FM tables
    int64_t total_rows = 0, exact_total = 0;
    const int64_t *cf_slots = nullptr;       // the CF recall rows, in the CF index's recall buffers
    const float *cf_scores = nullptr;
    const int32_t *cf_count = nullptr;
    fm::Feats FI{};
    fm::Slot FS[fm::MAX_SLOTS];
    // the chunk plan
    std::vector<int64_t> chunk_at{0}, out_at;
    int64_t n_chunks = 0, sort_stride = 0;
    int grid = 0, emit_grid = 0;
    std::vector<int64_t> h_cand_off, h_E_off, h_e0_off, h_ch_off;

    // slot_of_item / item_of_slot of a stage's collection: one slot per item and back
    int32_t check_map(const char *what, gorse_b200_vecdb *db, const int64_t *slot_of_item, const int32_t *item_of_slot) const
    {
        GB_CHECK_ARG(slot_of_item != nullptr && (item_of_slot != nullptr || db->ts.empty()), "%s: slot_of_item / item_of_slot is NULL", what);
        const int64_t S = (int64_t)db->ts.size();
        for (int32_t i = 0; i < n_items; i++)
            GB_CHECK_ARG(slot_of_item[i] >= -1 && slot_of_item[i] < S, "%s: slot_of_item[%d] = %lld is not a slot", what, i, (long long)slot_of_item[i]);
        // one slot per item and back: two items naming one slot would break the slot-space exclude sets
        for (int32_t i = 0; i < n_items; i++)
            GB_CHECK_ARG(slot_of_item[i] < 0 || item_of_slot[slot_of_item[i]] == i, "%s: slot_of_item[%d] = %lld holds item %d", what, i,
                         (long long)slot_of_item[i], item_of_slot[slot_of_item[i]]);
        for (int64_t s = 0; s < S; s++) {
            const int32_t it = item_of_slot[s];
            GB_CHECK_ARG(it >= -1 && it < n_items, "%s: item_of_slot[%lld] = %d is not an item", what, (long long)s, it);
            if (db->dead[(size_t)s]) continue;
            GB_CHECK_ARG(it >= 0, "%s: live slot %lld has no item", what, (long long)s);
            GB_CHECK_ARG(slot_of_item[it] == s, "%s: live slot %lld holds item %d whose slot is %lld", what, (long long)s, it, (long long)slot_of_item[it]);
        }
        return GORSE_B200_OK;
    }

    // stage s's arguments, and the most candidates it gives each user, in b
    int32_t check_stage(int32_t s, std::vector<int64_t> &b) const
    {
        const auto &g = stages[s];
        char who[32];
        snprintf(who, sizeof who, "stage %d", s);
        if (g.kind == GORSE_B200_STAGE_LIST) {
            if (g.list_off) {
                GB_TRY(check_offsets(g.list_off, n_users, who, "list_off"));
                for (int64_t u = 0; u < n_users; u++) b[(size_t)u] = g.list_off[u + 1] - g.list_off[u];
            } else {
                GB_CHECK_ARG(g.list_len >= 0, "stage %d: negative list_len", s);
                std::fill(b.begin(), b.end(), g.list_len);
            }
            const int64_t total = g.list_off ? g.list_off[n_users] : g.list_len;
            GB_CHECK_ARG(total == 0 || (g.list_items != nullptr && g.list_scores != nullptr), "stage %d: list_items / list_scores is NULL", s);
            for (int64_t t = 0; t < total; t++) {
                GB_CHECK_ARG(g.list_items[t] >= 0 && g.list_items[t] < n_items, "stage %d: list entry %lld: item %d is not in [0, %d)", s, (long long)t,
                             g.list_items[t], n_items);
                GB_CHECK_ARG(g.list_scores[t] == g.list_scores[t], "stage %d: list entry %lld: score is NaN", s, (long long)t);
            }
            for (int64_t u = 0; u < n_users; u++)
                if (b[(size_t)u] > MAX_LIST) {
                    set_error("stage %d: a list of %lld entries, at most %d", s, (long long)b[(size_t)u], MAX_LIST);
                    return GORSE_B200_ERR_UNSUPPORTED;
                }
            return GORSE_B200_OK;
        }
        if (g.kind == GORSE_B200_STAGE_COLLABORATIVE) {
            std::fill(b.begin(), b.end(), std::max(cf->n, 0));
            return GORSE_B200_OK;
        }
        gorse_b200_vecdb *db = g.db;
        GB_CHECK_ARG(g.score_scale == g.score_scale, "stage %d: score_scale is NaN", s);
        GB_TRY(check_stage_db(db, g.n, who));
        std::fill(b.begin(), b.end(), std::max(g.n, 0));
        if (g.kind == GORSE_B200_STAGE_ITEM_TO_ITEM) {
            GB_TRY(check_map("item-to-item stage", db, g.slot_of_item, g.item_of_slot));
            GB_CHECK_ARG(g.ctx_off != nullptr, "stage %d: ctx_off is NULL", s);
            GB_TRY(check_offsets(g.ctx_off, n_users, who, "ctx_off"));
            GB_CHECK_ARG(g.n_categories >= 0 && (g.n_categories == 0 || g.categories != nullptr), "stage %d: categories", s);
            GB_CHECK_ARG(g.ctx_off[n_users] == 0 || g.ctx_items != nullptr, "stage %d: ctx_items is NULL", s);
            for (int64_t t = 0; t < g.ctx_off[n_users]; t++)
                GB_CHECK_ARG(g.ctx_items[t] >= -1 && g.ctx_items[t] < n_items, "stage %d: context entry %lld: item %d is not in [-1, %d)", s,
                             (long long)t, g.ctx_items[t], n_items);
            return GORSE_B200_OK;
        }
        GB_CHECK_ARG(g.user_slots != nullptr, "stage %d: user_slots is NULL", s);
        for (int64_t u = 0; u < n_users; u++)
            GB_CHECK_ARG(g.user_slots[u] >= -1 && g.user_slots[u] < (int64_t)db->ts.size(), "stage %d: user %lld: slot %lld is not a slot", s,
                         (long long)u, (long long)g.user_slots[u]);
        return check_feedback(who, g.n_fb_rows, g.fb_off, g.fb_items, n_items);
    }

    // the ranker: features checked as gorse_b200_fm_rank checks them; the row lengths for D_u
    int32_t check_ranker()
    {
        const auto &R = *ranker;
        GB_TRY(fm::check_feats("user", n_users, R.user_feat, R.user_lab_off, R.user_lab_idx, R.user_lab_val, m->n_features));
        GB_TRY(fm::check_feats("item", n_items, R.item_feat, R.item_lab_off, R.item_lab_idx, R.item_lab_val, m->n_features));
        if (m->n_emb > 0 && n_items > 0) {
            GB_CHECK_ARG(R.item_emb != nullptr, "item_emb is NULL");
            for (int s = 0; s < m->n_emb; s++) GB_CHECK_ARG(R.item_emb[s] != nullptr, "item_emb[%d] is NULL", s);
        }
        u_len.resize((size_t)n_users);
        i_len.resize((size_t)n_items);
        int64_t longest_item = 0;
        for (int32_t i = 0; i < n_items; i++) {
            const int64_t l = (R.item_feat[i] >= 0) + R.item_lab_off[i + 1] - R.item_lab_off[i];
            GB_CHECK_ARG(l <= INT32_MAX / 2, "item %d: a row of 2^30 or more features", i);
            i_len[(size_t)i] = (int32_t)l;
            longest_item = std::max(longest_item, l);
        }
        for (int64_t u = 0; u < n_users; u++) {
            const int64_t l = (R.user_feat[u] >= 0) + R.user_lab_off[u + 1] - R.user_lab_off[u];
            GB_CHECK_ARG(l + longest_item <= INT32_MAX, "user %lld: rows of 2^31 or more features", (long long)u);
            u_len[(size_t)u] = (int32_t)l;
        }
        return GORSE_B200_OK;
    }

    // every argument but the context, on the host; locks the collections and the ranker
    int32_t check()
    {
        GB_CHECK_ARG(count_out != nullptr && excl_off != nullptr, "count_out / excl_off is NULL");
        GB_CHECK_ARG(n_stages == 0 || stages != nullptr, "stages is NULL");
        GB_CHECK_ARG(n_items == 0 || item_live != nullptr, "item_live is NULL");
        GB_TRY(check_offsets(excl_off, n_users, "recommend", "excl_off"));
        GB_CHECK_ARG(excl_off[n_users] == 0 || excl_items != nullptr, "excl_items is NULL");
        GB_TRY(exclusion_rows(n_users, excl_off, excl_items, n_items, "user", "item", e0, e0_off));
        std::vector<gorse_b200_vecdb *> dbs;
        for (int32_t s = 0; s < n_stages; s++) {
            const auto &g = stages[s];
            GB_CHECK_ARG(g.kind >= GORSE_B200_STAGE_LIST && g.kind <= GORSE_B200_STAGE_USER_TO_USER, "stage %d: unknown kind %d", s, g.kind);
            if (g.kind == GORSE_B200_STAGE_ITEM_TO_ITEM || g.kind == GORSE_B200_STAGE_USER_TO_USER) {
                GB_CHECK_ARG(g.db != nullptr && g.db->ctx == ctx, "stage %d: collection is NULL or of another context", s);
                dbs.push_back(g.db);
            }
            if (g.kind == GORSE_B200_STAGE_COLLABORATIVE) GB_CHECK_ARG(cf != nullptr, "stage %d: a collaborative stage needs the CF inputs", s);
        }
        if (cf) {
            GB_CHECK_ARG(cf->db != nullptr && cf->db->ctx == ctx, "CF collection is NULL or of another context");
            dbs.push_back(cf->db);
        }
        std::sort(dbs.begin(), dbs.end());
        dbs.erase(std::unique(dbs.begin(), dbs.end()), dbs.end());
        for (auto *db : dbs) locks.emplace_back(db->mu);
        if (ranker) {
            GB_CHECK_ARG(ranker->fm != nullptr && ranker->fm->ctx == ctx, "ranker: fm handle is NULL or of another context");
            fm_lock = std::unique_lock<std::mutex>(ranker->fm->mu);
        }

        // per stage: checks and the per-user bound
        bound.assign((size_t)n_users, 0);
        cap.resize((size_t)n_users);
        for (int64_t u = 0; u < n_users; u++) cap[(size_t)u] = e0_off[(size_t)u + 1] - e0_off[(size_t)u];
        std::vector<int64_t> b((size_t)n_users);
        for (int32_t s = 0; s < n_stages; s++) {
            std::fill(b.begin(), b.end(), 0);
            GB_TRY(check_stage(s, b));
            for (int64_t u = 0; u < n_users; u++) {
                bound[(size_t)u] += b[(size_t)u];
                if (s + 1 < n_stages) cap[(size_t)u] += b[(size_t)u];
            }
        }
        if (cf) {
            if (cf->db->dim == 0) { set_error("the CF collection must be dense"); return GORSE_B200_ERR_UNSUPPORTED; }
            GB_CHECK_ARG(cf->n >= 0 && cf->n <= MAX_N_DENSE, "CF n = %d is not in [0, %d]", cf->n, MAX_N_DENSE);
            GB_CHECK_ARG(cf->user_vectors != nullptr, "CF user_vectors is NULL");
            GB_TRY(check_map("CF", cf->db, cf->slot_of_item, cf->item_of_slot));
            for (int64_t u = 0; u < n_users; u++)
                GB_CHECK_ARG((int64_t)cf->n + (excl_off[u + 1] - excl_off[u]) <= INT32_MAX, "user %lld: n + |E0| overflows", (long long)u);
        }
        with_repl = ranker && repl_off;
        if (with_repl) {
            GB_TRY(check_offsets(repl_off, n_users, "recommend", "repl_off"));
            GB_CHECK_ARG(positive_decay == positive_decay && read_decay == read_decay, "a decay is NaN");
            GB_CHECK_ARG(repl_off[n_users] == 0 || (repl_items != nullptr && repl_positive != nullptr), "repl_items / repl_positive is NULL");
            std::vector<int32_t> row;
            for (int64_t u = 0; u < n_users; u++) {
                row.assign(repl_items + repl_off[u], repl_items + repl_off[u + 1]);
                for (int32_t it : row) GB_CHECK_ARG(it >= 0 && it < n_items, "user %lld: replacement item %d is not in [0, %d)", (long long)u, it, n_items);
                std::sort(row.begin(), row.end());
                GB_CHECK_ARG(std::adjacent_find(row.begin(), row.end()) == row.end(), "user %lld: a replacement item twice", (long long)u);
                bound[(size_t)u] += repl_off[u + 1] - repl_off[u];
            }
        }
        m = ranker ? ranker->fm : nullptr;
        if (m) GB_TRY(check_ranker());
        for (int64_t u = 0; u < n_users; u++)
            GB_CHECK_ARG(bound[(size_t)u] <= INT32_MAX / 2, "user %lld: %lld candidates at most, above 2^30", (long long)u, (long long)bound[(size_t)u]);
        GB_CHECK_ARG(items_out != nullptr && scores_out != nullptr, "NULL output");
        return GORSE_B200_OK;
    }

    // E0 of every user through slot_of_item, -1 dropped, sorted: the exclude sets in a collection's slots
    void slot_rows(const int64_t *slot_of_item, std::vector<int64_t> &ex, std::vector<int64_t> &ex_off) const
    {
        ex.reserve(e0.size());
        ex_off.assign((size_t)n_users + 1, 0);
        for (int64_t u = 0; u < n_users; u++) {
            const size_t b = ex.size();
            for (int64_t t = e0_off[(size_t)u]; t < e0_off[(size_t)u + 1]; t++)
                if (slot_of_item[e0[(size_t)t]] >= 0) ex.push_back(slot_of_item[e0[(size_t)t]]);
            std::sort(ex.begin() + b, ex.end());
            ex_off[(size_t)u + 1] = (int64_t)ex.size();
        }
    }

    // once per call: the live and replacement items, the list stages' rows, and every item-to-item / user-to-user stage's table
    // rows and neighbour table
    int32_t tables(Work &W)
    {
        const cudaStream_t st = ctx->stream;
        GB_TRY(W.d_live.upload(item_live, (size_t)n_items, st));
        if (with_repl) {
            GB_TRY(W.d_repl_off.upload(repl_off, (size_t)n_users + 1, st));
            GB_TRY(W.d_repl_items.upload(repl_items, (size_t)repl_off[n_users], st));
            GB_TRY(W.d_repl_pos.upload(repl_positive, (size_t)repl_off[n_users], st));
        }
        if (W.lists.size() < (size_t)n_stages) W.lists.resize((size_t)n_stages);
        if (W.sd.size() < (size_t)n_stages) W.sd.resize((size_t)n_stages);
        for (int32_t s = 0; s < n_stages; s++) {
            const auto &g = stages[s];
            if (g.kind == GORSE_B200_STAGE_LIST) {
                const int64_t total = g.list_off ? g.list_off[n_users] : g.list_len;
                Work::List &L = W.lists[(size_t)s];
                GB_TRY(L.items.upload(g.list_items, (size_t)total, st));
                GB_TRY(L.scores.upload(g.list_scores, (size_t)total, st));
                if (g.list_off) GB_TRY(L.off.upload(g.list_off, (size_t)n_users + 1, st));
                continue;
            }
            if (g.kind == GORSE_B200_STAGE_COLLABORATIVE) continue;
            NeighbourStage &D = W.sd[(size_t)s];
            const bool i2i = g.kind == GORSE_B200_STAGE_ITEM_TO_ITEM;
            if (i2i) {
                D.prepare_items(g.db, n_users, g.ctx_off, g.ctx_items, g.slot_of_item, g.n, 0, g.n, g.score_scale, nullptr);
                slot_rows(g.slot_of_item, D.es0, D.es0_off);
            } else {
                D.prepare_users(g.db, n_users, g.user_slots, g.n_fb_rows, g.fb_off, g.fb_items, n_items, g.n, g.score_scale, g.item_ok);
            }
            total_rows += (int64_t)D.nb.size();
            if (g.n <= 0) continue;
            if (i2i) {
                GB_TRY(D.map.upload(g.slot_of_item, (size_t)n_items, st));
                GB_TRY(D.item_of_slot.upload(g.item_of_slot, g.db->ts.size(), st));
            }
            int64_t exact = 0;
            GB_TRY(D.table(i2i ? g.categories : nullptr, i2i ? g.n_categories : 0, &exact));
            exact_total += exact;
        }
        return GORSE_B200_OK;
    }

    // once per call, after every neighbour table (which may use the CF index): the CF recall rows, left in the CF index's recall
    // buffers; the ranker's user rows and the dictionary's item table
    int32_t recall_and_ranker(Work &W)
    {
        const cudaStream_t st = ctx->stream;
        bool need_cf = false;
        for (int32_t s = 0; s < n_stages; s++) need_cf |= stages[s].kind == GORSE_B200_STAGE_COLLABORATIVE;
        if (need_cf) {
            std::vector<int64_t> cf_ex, cf_ex_off;
            slot_rows(cf->slot_of_item, cf_ex, cf_ex_off);
            GB_TRY(W.d_cf_excl_off.upload(excl_off, (size_t)n_users + 1, st));
            GB_TRY(W.d_cf_item_of_slot.upload(cf->item_of_slot, cf->db->ts.size(), st));
            if (cf->n > 0 && !cf->db->ts.empty()) {
                GB_TRY(vecdb_allow(cf->db, nullptr, 0));
                std::lock_guard<std::mutex> lk2(cf->db->dense->mu);
                int64_t exact = 0;
                GB_TRY(recall::recall_rows(cf->db->dense, cf->db->d_allow.p, n_users, cf->user_vectors, nullptr, cf->n, excl_off, cf_ex.data(),
                                           cf_ex_off.data(), nullptr, nullptr, nullptr, nullptr, &exact));
                exact_total += exact;
                cf_slots = cf->db->dense->recall.slots.p;
                cf_scores = cf->db->dense->recall.scores.p;
                cf_count = cf->db->dense->recall.count.p;
            }
        }
        if (!m) return GORSE_B200_OK;
        const auto &R = *ranker;
        GB_TRY(fm::upload_feats(m, n_users, R.user_feat, R.user_lab_off, R.user_lab_idx, R.user_lab_val, n_items, R.item_feat, R.item_lab_off,
                                R.item_lab_idx, R.item_lab_val, R.item_emb, R.item_emb_mask, FS));
        GB_TRY(W.d_u_len.upload(u_len.data(), u_len.size(), st));
        GB_TRY(W.d_i_len.upload(i_len.data(), i_len.size(), st));
        FI = fm::Feats{m->i_feat.p, m->i_off.p, m->i_idx.p, m->i_val.p};
        return GORSE_B200_OK;
    }

    // the chunks: at most sm_count * 1024 users and CHUNK_ENTRIES candidate / exclude-set entries (or one user; with embedding
    // slots a sixteenth: the attention's vx rows take n_factors floats per candidate), and every buffer sized for the largest
    int32_t plan(Work &W)
    {
        const cudaStream_t st = ctx->stream;
        const int64_t lim = m && m->n_emb > 0 ? CHUNK_ENTRIES / 16 : CHUNK_ENTRIES;
        // one pass: the cuts, each chunk's rows and entries, and the output rows of the whole call at the bound prefix
        int64_t max_rows = 0, max_b = 0, max_c = 0, max_e0 = 0, max_bound = 0, b = 0, c = 0;
        out_at.assign((size_t)n_users + 1, 0);
        for (int64_t u = 0; u <= n_users; u++) {
            const int64_t a = chunk_at.back();
            if (u == n_users ||
                (u > a && (u - a == (int64_t)ctx->sm_count * 1024 || b + bound[(size_t)u] > lim || c + cap[(size_t)u] > lim))) {
                max_rows = std::max(max_rows, u - a);
                max_b = std::max(max_b, b);
                max_c = std::max(max_c, c);
                max_e0 = std::max(max_e0, e0_off[(size_t)u] - e0_off[(size_t)a]);
                chunk_at.push_back(u);
                b = c = 0;
            }
            if (u == n_users) break;
            b += bound[(size_t)u];
            c += cap[(size_t)u];
            max_bound = std::max(max_bound, bound[(size_t)u]);
            out_at[(size_t)u + 1] = out_at[(size_t)u] + bound[(size_t)u];
        }
        n_chunks = (int64_t)chunk_at.size() - 1;
        int max_n = 0;
        for (int32_t s = 0; s < n_stages; s++)
            if (stages[s].kind >= GORSE_B200_STAGE_ITEM_TO_ITEM) max_n = std::max(max_n, stages[s].n);
        grid = (int)std::min<int64_t>(max_rows, (int64_t)ctx->sm_count * 8);
        sort_stride = recall::pow2_at_least((int)std::max<int64_t>(max_bound, 1));
        // the re-sort's per-CTA key buffers, at most 256 MB of them (as fm_sort_kernel's)
        emit_grid = (int)std::max<int64_t>(1, std::min<int64_t>(grid, (int64_t(256) << 20) / (sort_stride * (int64_t)sizeof(u128))));
        const size_t rows = (size_t)max_rows, B = (size_t)std::max<int64_t>(max_b, 1), Cn = (size_t)std::max<int64_t>(max_c, 1);
        for (auto *b : {&W.d_cand_off, &W.d_E_off, &W.d_e0_off}) GB_TRY(b->grow(rows + 1));
        for (auto *b : {&W.d_cnt, &W.d_start, &W.d_rcount, &W.d_out_cnt[0], &W.d_out_cnt[1]}) GB_TRY(b->grow(rows));
        for (auto *b : {&W.d_cand, &W.d_out_items[0], &W.d_out_items[1]}) GB_TRY(b->grow(B));
        for (auto *b : {&W.d_cscore, &W.d_out_scores[0], &W.d_out_scores[1]}) GB_TRY(b->grow(B));
        GB_TRY(W.d_e0.grow((size_t)std::max<int64_t>(max_e0, 1)));
        GB_TRY(W.d_E[0].grow(Cn));
        GB_TRY(W.d_E[1].grow(Cn));
        GB_TRY(W.d_rids.grow((size_t)std::max<int64_t>(max_rows * max_n, 1)));
        GB_TRY(W.d_rscore.grow((size_t)std::max<int64_t>(max_rows * max_n, 1)));
        for (int32_t s = 0; s < n_stages; s++) {
            const auto &g = stages[s];
            NeighbourStage &D = W.sd[(size_t)s];
            if (g.kind == GORSE_B200_STAGE_ITEM_TO_ITEM) {
                GB_TRY(D.d_es0.upload(D.es0.data(), D.es0.size(), st));
                GB_TRY(D.d_es0_off.upload(D.es0_off.data(), D.es0_off.size(), st));
                GB_TRY(D.es[0].grow(Cn));
                GB_TRY(D.es[1].grow(Cn));
            }
            if (g.kind >= GORSE_B200_STAGE_ITEM_TO_ITEM && g.n > 0) GB_TRY(D.reserve(max_rows, n_chunks));
        }
        if (!m) return GORSE_B200_OK;
        GB_TRY(W.d_fm_off.grow(rows + 1));
        GB_TRY(W.d_dims.grow(rows));
        GB_TRY(W.d_dscore.grow(B));
        for (auto *b : {&m->cand, &m->order}) GB_TRY(b->grow(B));
        GB_TRY(m->score.grow(B));
        GB_TRY(W.d_sort.grow((size_t)emit_grid * sort_stride));
        if (m->n_emb > 0) {
            GB_TRY(m->vx.grow(B * m->k));
            GB_TRY(m->rowsum.grow(B));
        }
        return GORSE_B200_OK;
    }

    // chunk k: E_u, every stage in order, the assembly, the ranking, and the download of its answer on the copy stream into the
    // output buffers of parity k & 1, free once the download of chunk k - 2 has finished (reuse[k & 1])
    int32_t run_chunk(Work &W, int64_t k, Event *reuse)
    {
        const cudaStream_t st = ctx->stream;
        const int64_t u0 = chunk_at[(size_t)k], rows = chunk_at[(size_t)k + 1] - u0;
        const int p = (int)(k & 1);
        h_cand_off.resize((size_t)rows + 1);
        h_E_off.assign((size_t)rows + 1, 0);
        h_e0_off.resize((size_t)rows + 1);
        for (int64_t r = 0; r <= rows; r++) {
            h_cand_off[(size_t)r] = out_at[(size_t)(u0 + r)] - out_at[(size_t)u0];
            h_e0_off[(size_t)r] = e0_off[(size_t)(u0 + r)] - e0_off[(size_t)u0];
            if (r < rows) h_E_off[(size_t)r + 1] = h_E_off[(size_t)r] + cap[(size_t)(u0 + r)];
        }
        GB_CUDA(cudaMemcpyAsync(W.d_cand_off.p, h_cand_off.data(), sizeof(int64_t) * (rows + 1), cudaMemcpyHostToDevice, st));
        GB_CUDA(cudaMemcpyAsync(W.d_E_off.p, h_E_off.data(), sizeof(int64_t) * (rows + 1), cudaMemcpyHostToDevice, st));
        GB_CUDA(cudaMemcpyAsync(W.d_e0_off.p, h_e0_off.data(), sizeof(int64_t) * (rows + 1), cudaMemcpyHostToDevice, st));
        if (h_e0_off[(size_t)rows])
            GB_CUDA(cudaMemcpyAsync(W.d_e0.p, e0.data() + e0_off[(size_t)u0], sizeof(int64_t) * h_e0_off[(size_t)rows], cudaMemcpyHostToDevice, st));
        GB_CUDA(cudaMemsetAsync(W.d_cnt.p, 0, sizeof(int32_t) * rows, st));
        // E_u from E0, and the item-to-item stages' sets in slots
        int e_cur = 0;
        rec_grow_kernel<<<grid, NT, 0, st>>>(W.d_e0.p, W.d_e0_off.p, W.d_E[0].p, W.d_E_off.p, nullptr, nullptr, nullptr, nullptr, nullptr, rows);
        ctx->launches++;
        for (int32_t s = 0; s < n_stages; s++) {
            NeighbourStage &D = W.sd[(size_t)s];
            if (stages[s].kind != GORSE_B200_STAGE_ITEM_TO_ITEM) continue;
            rec_grow_kernel<<<grid, NT, 0, st>>>(D.d_es0.p, D.d_es0_off.p + u0, D.es[0].p, W.d_E_off.p, nullptr, nullptr, nullptr, nullptr, nullptr,
                                                 rows);
            ctx->launches++;
        }
        GB_CUDA(cudaGetLastError());
        for (int32_t s = 0; s < n_stages; s++) {
            const auto &g = stages[s];
            NeighbourStage &D = W.sd[(size_t)s];
            GB_CUDA(cudaMemcpyAsync(W.d_start.p, W.d_cnt.p, sizeof(int32_t) * rows, cudaMemcpyDeviceToDevice, st));
            const int64_t *E = W.d_E[e_cur].p;
            if (g.kind == GORSE_B200_STAGE_LIST) {
                const Work::List &L = W.lists[(size_t)s];
                rec_list_kernel<<<grid, NT, 0, st>>>(L.items.p, L.scores.p, g.list_off ? L.off.p : nullptr, g.list_len, u0, E, W.d_E_off.p, W.d_cand.p,
                                                     W.d_cscore.p, W.d_cand_off.p, W.d_cnt.p, rows);
                ctx->launches++;
            } else if (g.kind == GORSE_B200_STAGE_COLLABORATIVE) {
                if (cf_slots) {
                    rec_cf_kernel<<<grid, NT, 0, st>>>(cf_slots, cf_scores, cf_count, W.d_cf_excl_off.p, cf->n, u0, W.d_cf_item_of_slot.p,
                                                       W.d_live.p, E, W.d_E_off.p, W.d_cand.p, W.d_cscore.p, W.d_cand_off.p, W.d_cnt.p, rows);
                    ctx->launches++;
                }
            } else if (g.n > 0 && !D.nb.empty()) {
                // the item-to-item stage excludes in its collection's slots and maps its row back to items
                const bool i2i = g.kind == GORSE_B200_STAGE_ITEM_TO_ITEM;
                GB_TRY(D.run_chunk(k, u0, rows, W.d_E_off.p, i2i ? D.es[e_cur].p : E, W.d_rids.p, W.d_rscore.p, W.d_rcount.p));
                rec_append_kernel<<<grid, NT, 0, st>>>(W.d_rids.p, W.d_rscore.p, W.d_rcount.p, g.n, i2i ? D.item_of_slot.p : nullptr, W.d_cand.p,
                                                       W.d_cscore.p, W.d_cand_off.p, W.d_cnt.p, rows);
                ctx->launches++;
            }
            GB_CUDA(cudaGetLastError());
            if (s + 1 == n_stages) break;
            // E_u grows by what the stage appended, after the whole stage
            rec_grow_kernel<<<grid, NT, 0, st>>>(W.d_E[e_cur].p, W.d_E_off.p, W.d_E[e_cur ^ 1].p, W.d_E_off.p, W.d_cand.p, W.d_cand_off.p, W.d_start.p,
                                                 W.d_cnt.p, nullptr, rows);
            ctx->launches++;
            for (int32_t t = s + 1; t < n_stages; t++) {
                NeighbourStage &Dt = W.sd[(size_t)t];
                if (stages[t].kind != GORSE_B200_STAGE_ITEM_TO_ITEM) continue;
                rec_grow_kernel<<<grid, NT, 0, st>>>(Dt.es[e_cur].p, W.d_E_off.p, Dt.es[e_cur ^ 1].p, W.d_E_off.p, W.d_cand.p, W.d_cand_off.p,
                                                     W.d_start.p, W.d_cnt.p, Dt.map.p, rows);
                ctx->launches++;
            }
            GB_CUDA(cudaGetLastError());
            e_cur ^= 1;
        }
        const int64_t *repl_off = with_repl ? W.d_repl_off.p : nullptr;
        rec_assemble_kernel<<<grid, NT, 0, st>>>(W.d_live.p, repl_off, W.d_repl_items.p, u0, W.d_cand.p, W.d_cscore.p, W.d_cand_off.p, W.d_cnt.p, rows);
        ctx->launches++;
        GB_CUDA(cudaGetLastError());
        if (k >= 2) GB_CUDA(cudaStreamWaitEvent(st, reuse[p].e, 0));
        if (m) {
            rec_scan_kernel<<<1, 1024, 0, st>>>(W.d_cnt.p, rows, W.d_fm_off.p);
            ctx->launches++;
            const int64_t *ch_off = nullptr;
            int64_t n_ch = 0;
            if (m->n_emb > 0) {
                h_ch_off.assign((size_t)rows + 1, 0);
                for (int64_t r = 0; r < rows; r++)
                    h_ch_off[(size_t)r + 1] = h_ch_off[(size_t)r] + (bound[(size_t)(u0 + r)] + m->batch_size - 1) / m->batch_size;
                n_ch = h_ch_off[(size_t)rows];
                GB_TRY(W.d_ch_off.upload(h_ch_off.data(), h_ch_off.size(), st));
                GB_TRY(m->ch_start.grow((size_t)std::max<int64_t>(n_ch, 1)));
                GB_TRY(m->ch_rows.grow((size_t)std::max<int64_t>(n_ch, 1)));
                ch_off = W.d_ch_off.p;
            }
            rec_pack_kernel<<<(unsigned)std::min<int64_t>((rows + 7) / 8, (int64_t)ctx->sm_count * 16), 256, 0, st>>>(
                W.d_cand.p, W.d_cand_off.p, W.d_cnt.p, W.d_fm_off.p, W.d_u_len.p + u0, W.d_i_len.p, m->num_dimension, m->cand.p, W.d_dims.p, ch_off,
                m->batch_size, m->ch_start.p, m->ch_rows.p, rows);
            ctx->launches++;
            GB_CUDA(cudaGetLastError());
            const fm::Feats U{m->u_feat.p + u0, m->u_off.p + u0, m->u_idx.p, m->u_val.p};
            int64_t mb = 0;
            for (int64_t r = 0; r < rows; r++) mb = std::max(mb, bound[(size_t)(u0 + r)]);
            bool gs = false;
            GB_TRY(fm::rank_pass(m, U, FI, W.d_fm_off.p, m->cand.p, W.d_dims.p, 0, rows, 0, FS, m->ch_start.p, m->ch_rows.p, 0, n_ch, mb, m->score.p,
                                 m->order.p, &gs));
            rec_emit_kernel<<<emit_grid, NT, 0, st>>>(m->cand.p, W.d_fm_off.p, m->score.p, m->order.p, repl_off, W.d_repl_items.p, W.d_repl_pos.p, u0,
                                                        positive_decay, read_decay, W.d_dscore.p, W.d_sort.p, sort_stride, W.d_cand_off.p,
                                                        W.d_out_items[p].p, W.d_out_scores[p].p, W.d_out_cnt[p].p, rows);
            ctx->launches++;
            GB_CUDA(cudaGetLastError());
        } else {   // the merged candidates are the answer; copied so that the next chunk may reuse the work buffers
            GB_CUDA(cudaMemcpyAsync(W.d_out_items[p].p, W.d_cand.p, sizeof(int32_t) * h_cand_off[(size_t)rows], cudaMemcpyDeviceToDevice, st));
            GB_CUDA(cudaMemcpyAsync(W.d_out_scores[p].p, W.d_cscore.p, sizeof(double) * h_cand_off[(size_t)rows], cudaMemcpyDeviceToDevice, st));
            GB_CUDA(cudaMemcpyAsync(W.d_out_cnt[p].p, W.d_cnt.p, sizeof(int32_t) * rows, cudaMemcpyDeviceToDevice, st));
        }
        const int64_t ob = out_at[(size_t)u0], on = h_cand_off[(size_t)rows];
        GB_CUDA(cudaEventRecord(ctx->copy_ev, st));
        GB_CUDA(cudaStreamWaitEvent(ctx->copy_stream, ctx->copy_ev, 0));
        GB_CUDA(cudaMemcpyAsync(count_out + u0, W.d_out_cnt[p].p, sizeof(int32_t) * rows, cudaMemcpyDeviceToHost, ctx->copy_stream));
        if (on) {
            GB_CUDA(cudaMemcpyAsync(items_out + ob, W.d_out_items[p].p, sizeof(int32_t) * on, cudaMemcpyDeviceToHost, ctx->copy_stream));
            GB_CUDA(cudaMemcpyAsync(scores_out + ob, W.d_out_scores[p].p, sizeof(double) * on, cudaMemcpyDeviceToHost, ctx->copy_stream));
        }
        GB_CUDA(cudaEventRecord(reuse[p].e, ctx->copy_stream));
        return GORSE_B200_OK;
    }
};

}  // namespace rec
}  // namespace gb

using namespace gb;

extern "C" int32_t gorse_b200_recommend(gorse_b200_ctx *ctx, int64_t n_users, const int64_t *excl_off, const int32_t *excl_items, int32_t n_items,
                                        const uint8_t *item_live, int32_t n_stages, const gorse_b200_recommend_stage *stages,
                                        const gorse_b200_recommend_cf *cf, const gorse_b200_recommend_ranker *ranker, const int64_t *repl_off,
                                        const int32_t *repl_items, const uint8_t *repl_positive, double positive_decay, double read_decay,
                                        int32_t *items_out, double *scores_out, int32_t *count_out, int64_t *stats_out)
{
    using namespace gb::rec;
    GB_CHECK_ARG(n_users >= 0 && n_items >= 0 && n_stages >= 0, "negative count");
    if (stats_out) std::fill(stats_out, stats_out + 4, 0);
    if (n_users == 0) return GORSE_B200_OK;
    Call C{ctx, n_users, excl_off, excl_items, n_items, item_live, n_stages, stages, cf, ranker, repl_off, repl_items, repl_positive,
           positive_decay, read_decay, items_out, scores_out, count_out};
    GB_TRY(C.check());
    // the context last: every other argument is checked without it
    GB_CHECK_ARG(ctx != nullptr, "ctx is NULL");
    Work *Wp = work(ctx);
    if (!Wp) { set_error("host allocation failed"); return GORSE_B200_ERR_OOM; }
    Work &W = *Wp;
    std::lock_guard<std::mutex> wlk(W.mu);
    ScopedDevice sdev(ctx->device);
    Event reuse[2];
    StreamSync sync{ctx->stream, ctx->copy_stream};
    GB_TRY(C.tables(W));
    GB_TRY(C.recall_and_ranker(W));
    GB_TRY(C.plan(W));
    GB_TRY(reuse[0].create());
    GB_TRY(reuse[1].create());
    for (int64_t k = 0; k < C.n_chunks; k++) GB_TRY(C.run_chunk(W, k, reuse));
    GB_CUDA(cudaStreamSynchronize(ctx->stream));
    GB_CUDA(cudaStreamSynchronize(ctx->copy_stream));
    int64_t ranked = 0;
    for (int64_t u = 0; u < n_users; u++) ranked += count_out[u];
    if (stats_out) {
        stats_out[0] = C.n_chunks;
        stats_out[1] = ranked;
        stats_out[2] = C.total_rows;
        stats_out[3] = C.exact_total;
    }
    return GORSE_B200_OK;
}
