// item_to_item.cu -- batched item-to-item and session recommendation: gorse_b200_vecdb_item_to_item and
// gorse_b200_vecdb_session_recommend.
//
// The worker's item-to-item recommender (logics/recommend.go:244-283) asks, per user, QueryItemToItem(c, categories, n) for
// every positive feedback item c, newest first (logics/item_to_item.go:50-86: top n + 1, drop c itself, drop Dot scores <= 0,
// stop at n), sums the neighbour scores per item id in float64, skipping the user's exclude set, and keeps the best n.  The
// REST server's session recommendation (sessionRecommend, server/rest.go:1069-1173) does the same with no category filter,
// keeps the neighbours that FilterVisibleItemsByCategories passes (rest.go:815-832), stops once ContextSize items have given
// a non-empty filtered list, and answers TopKFilter(n + offset).  Here one call answers many users or sessions:
//
//   stage A   the neighbour table, once per call: the distinct live context items of the whole batch are queried once each.
//             Dense collections run the index's top-k pipeline (recall_rows, topk.cu) with k = n on the stored vectors (a
//             row never returns its own vector), and its table keeps Dot scores > 0 only.  Sparse collections run
//             the tiled sparse search (sparse.cu) on the list of stored rows (a row never finds itself; it keeps positive dots only).
//             The table holds n (int32 slot, float32 score) entries per item, scores bit-identical to gorse_b200_vecdb_query.
//             A session's walk cannot stop at its cut here: whether an entry counts depends on its filtered list.  With the
//             collection's neighbour cache on, only the rows it does not hold are computed (neighbour_table, below).
//   stage B   i2i_aggregate_kernel, one CTA per user: for a session, first the cut (context_cut); then walks C_u (the
//             session's prefix) in order and adds s = (double)score * scale (Euclidean: 1 / (1 - s)) per neighbour slot that
//             item_ok passes and that is not in E_u, with a barrier between context entries so that every sum is formed in
//             the reference's order; then selects the first n (session: top) by (score desc, slot asc) with a 64-bit radix
//             select and sorts them (agg::select_first_n, aggregate.cuh).  The accumulator is an open-addressing table in
//             shared memory when |C_u| * n <= TABLE_KEYS, else this CTA's float64 row of length N in global memory, with a
//             touched flag per slot and the list of touched slots.
#include <algorithm>

#include "sparse.cuh"
#include "stages.cuh"

namespace gb {
namespace i2i {

using agg::TABLE_CAP;
constexpr int AGG_THREADS = agg::THREADS;

// One past the context entry e of [cb, ce) at which the count of entries with a non-empty filtered neighbour list reaches
// need, or ce when it never does.  Each window of NT entries: warp w tests entries w*32 .. w*32+31, its lanes splitting each
// list (__any_sync, stopping at the first passing neighbour), and records them as one bit mask; warp 0 scans the window's
// masks and picks the entry.  Every thread of the CTA calls it.
template <int NT>
__device__ int64_t context_cut(int64_t cb, int64_t ce, const int32_t *c_row, const NeighbourTable &T, int n, const uint8_t *item_ok, int need,
                               unsigned *s_mask, int64_t *s_cut)
{
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    for (int64_t base = cb; base < ce; base += NT) {
        unsigned mask = 0;
        for (int i = 0; i < 32; i++) {
            const int64_t e = base + w * 32 + i;
            if (e >= ce) break;
            const int64_t r = c_row[e];
            const int cnt = T.cnt[r];
            bool any = item_ok == nullptr && cnt > 0;
            for (int j0 = 0; item_ok != nullptr && !any && j0 < cnt; j0 += 32) {
                const int j = j0 + lane;
                any = __any_sync(0xffffffffu, j < cnt && item_ok[T.slot[r * n + j]]);
            }
            mask |= (unsigned)any << i;
        }
        if (lane == 0) s_mask[w] = mask;
        __syncthreads();
        if (w == 0) {
            const unsigned m = lane < NT / 32 ? s_mask[lane] : 0u;
            const int c = __popc(m);
            int incl = c;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int t = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += t;
            }
            const unsigned hit = __ballot_sync(0xffffffffu, incl >= need);
            if (hit == 0u) {
                if (lane == 0) *s_cut = -1;
            } else if (lane == __ffs(hit) - 1) {
                unsigned b = m;   // the (need - before)-th set bit of this lane's mask
                for (int k = need - (incl - c); k > 1; k--) b &= b - 1;
                *s_cut = base + lane * 32 + __ffs(b);
            }
        }
        __syncthreads();
        const int64_t cut = *s_cut;
        if (cut >= 0) return cut;
#pragma unroll
        for (int i = 0; i < NT / 32; i++) need -= __popc(s_mask[i]);
        __syncthreads();   // s_mask and s_cut are rewritten by the next window
    }
    return ce;
}

// one CTA per user of `users`.  SHARED: the accumulator is a table in shared memory; else acc_rows / seen_rows /
// touched_rows hold one [N] float64 row, one [N] flag row (all zero between users) and one [N] slot list per CTA.  CUT
// (session): the walk stops at context_cut's entry for need and skips the neighbours that item_ok (a slot mask or NULL) does
// not pass; else it takes the whole context, and item_ok and need are not read.  Row u of the answer is U.slots / U.scores
// [u * top, u * top + U.count[u]); the table's rows hold n entries.
template <bool SHARED, bool CUT>
__global__ void __launch_bounds__(AGG_THREADS)
i2i_aggregate_kernel(const int32_t *users, int64_t n_users, Users U, NeighbourTable T, const uint8_t *item_ok, int n, int need, int top,
                     double scale, int euclid, int64_t N, double *acc_rows, uint8_t *seen_rows, int32_t *touched_rows)
{
    using namespace gb::recall;
    using namespace gb::agg;
    constexpr int NT = AGG_THREADS;
    extern __shared__ __align__(16) uint8_t sm[];
    __shared__ unsigned s_mask[NT / 32];
    __shared__ int64_t s_cut;
    const int p2 = pow2_at_least(top);
    const Smem S = carve(sm, p2);
    int *s_bc = S.s_bc;                                            // [3]: distinct slots
    int32_t *t_key = S.t_key;                                      // SHARED: slot, -1 = empty
    double *t_val = S.t_val;                                       // SHARED: sum
    double *acc = SHARED ? nullptr : acc_rows + (int64_t)blockIdx.x * N;
    uint8_t *seen = SHARED ? nullptr : seen_rows + (int64_t)blockIdx.x * N;
    int32_t *touched = SHARED ? nullptr : touched_rows + (int64_t)blockIdx.x * N;
    for (int64_t i = blockIdx.x; i < n_users; i += gridDim.x) {
        const int64_t u = users[i];
        const int64_t cb = U.c_off[u];
        const int64_t ce = CUT ? context_cut<NT>(cb, U.c_off[u + 1], U.c_row, T, n, item_ok, need, s_mask, &s_cut) : U.c_off[u + 1];
        const int64_t *ex = U.ex + U.ex_off[u], n_ex = U.ex_off[u + 1] - U.ex_off[u];
        int cap = 0, lg = 0;
        if (SHARED) {   // a power of two >= 2 * (the walk's adds), at most TABLE_CAP: the load stays <= 3/4
            cap = min(TABLE_CAP, pow2_at_least(max(64, (int)(2 * (ce - cb) * n))));
            lg = __ffs(cap) - 1;
            for (int j = threadIdx.x; j < cap; j += NT) t_key[j] = -1;
        }
        if (threadIdx.x == 0) s_bc[3] = 0;
        __syncthreads();
        // C_u in order.  The neighbours of one entry are distinct slots, so its adds touch distinct sums; the barrier after
        // each entry makes every sum the reference's left-to-right sum over the context.
        for (int64_t e = cb; e < ce; e++) {
            const int64_t r = U.c_row[e];
            const int cnt = T.cnt[r];
            for (int j = threadIdx.x; j < cnt; j += NT) {
                const int32_t slot = T.slot[r * n + j];
                if ((CUT && item_ok != nullptr && !item_ok[slot]) || contains(ex, n_ex, (int64_t)slot)) continue;
                add_sum<SHARED>(slot, neighbour_score(T.score[r * n + j], scale, euclid), t_key, t_val, cap, lg, acc, seen, touched, &s_bc[3]);
            }
            __syncthreads();
        }
        const int distinct = s_bc[3];
        auto slot_at = [&](int64_t j) -> int32_t { return SHARED ? t_key[j] : touched[j]; };
        auto val_at = [&](int64_t j) -> double { return SHARED ? t_val[j] : acc[touched[j]]; };
        const int m = select_first_n<NT>(SHARED ? cap : distinct, distinct, top, p2, slot_at, val_at, S);
        for (int j = threadIdx.x; j < m; j += NT) {
            U.slots[u * top + j] = (int64_t)(uint32_t)S.s_key[j];
            U.scores[u * top + j] = S.s_val[j];
        }
        if (threadIdx.x == 0) U.count[u] = m;
        if (!SHARED)
            for (int j = threadIdx.x; j < distinct; j += NT) seen[touched[j]] = 0;
        __syncthreads();
    }
}

int32_t aggregate(gorse_b200_ctx *c, const int32_t *d_users, int64_t fill, int64_t heavy, const Users &U, const NeighbourTable &T,
                  const uint8_t *item_ok, int n, int need, int top, double scale, bool euclid, int64_t N, double *acc, uint8_t *seen,
                  int32_t *touched)
{
    // item-to-item (need <= 0) runs the instances without the cut and the item_ok test
    auto *k_shared = need > 0 ? i2i_aggregate_kernel<true, true> : i2i_aggregate_kernel<true, false>;
    auto *k_global = need > 0 ? i2i_aggregate_kernel<false, true> : i2i_aggregate_kernel<false, false>;
    const size_t sm_shared = agg::smem_bytes(top, true), sm_global = agg::smem_bytes(top, false);
    GB_CUDA(cudaFuncSetAttribute(k_shared, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm_shared));
    GB_CUDA(cudaFuncSetAttribute(k_global, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm_global));
    if (fill > 0) {
        k_shared<<<(unsigned)std::min<int64_t>(fill, (int64_t)c->sm_count * 8), AGG_THREADS, sm_shared, c->stream>>>(
            d_users, fill, U, T, item_ok, n, need, top, scale, euclid, N, nullptr, nullptr, nullptr);
        c->launches++;
    }
    if (heavy > 0) {
        k_global<<<(unsigned)std::min<int64_t>(heavy, heavy_grid(c, N, ROW_BYTES)), AGG_THREADS, sm_global, c->stream>>>(
            d_users + fill, heavy, U, T, item_ok, n, need, top, scale, euclid, N, acc, seen, touched);
        c->launches++;
    }
    GB_CUDA(cudaGetLastError());
    return GORSE_B200_OK;
}

}  // namespace i2i

int32_t NeighbourStage::table(const int32_t *categories, int32_t n_categories, int64_t *exact_rows)
{
    cudaStream_t s = db->ctx->stream;
    if (users) {
        GB_TRY(row.upload(q_row.data(), q_row.size(), s));
        GB_TRY(fb_off.upload(h_fb_off, fb_rows ? (size_t)fb_rows + 1 : 0, s));
        GB_TRY(fb_items.upload(h_fb_items, fb_rows ? (size_t)h_fb_off[fb_rows] : 0, s));
    } else {
        GB_TRY(row.upload(c_row.data(), c_row.size(), s));
        GB_TRY(d_c_off.upload(c_off.data(), c_off.size(), s));
    }
    if (h_item_ok) GB_TRY(item_ok.upload(h_item_ok, (size_t)item_ok_len, s));
    const int64_t R = (int64_t)nb.size();
    if (R == 0) return GORSE_B200_OK;
    GB_TRY(d_nb.grow((size_t)R));
    GB_TRY(t_slot.grow((size_t)R * n));
    GB_TRY(t_score.grow((size_t)R * n));
    GB_TRY(t_cnt.grow((size_t)R));
    return neighbour_table(db, nb, d_nb.p, n, categories, n_categories, t_slot.p, t_score.p, t_cnt.p, exact_rows);
}

int32_t NeighbourStage::reserve(int64_t max_rows, int64_t n_chunks)
{
    gorse_b200_ctx *c = db->ctx;
    GB_TRY(list.grow((size_t)max_rows));
    if (users) {
        GB_TRY(work.grow((size_t)max_rows));
        GB_TRY(route.grow((size_t)n_chunks * 2));
        GB_CUDA(cudaMemsetAsync(route.p, 0, sizeof(int32_t) * n_chunks * 2, c->stream));
    }
    if (!heavy) return GORSE_B200_OK;
    const size_t rows = (size_t)heavy_grid(c, N, users ? u2u::ROW_BYTES : i2i::ROW_BYTES) * N;
    if (users) {
        GB_TRY(uacc.grow_zeroed(rows, c->stream));
        GB_TRY(flag.grow_zeroed(rows, c->stream));
    } else {
        GB_TRY(acc.grow(rows));
        GB_TRY(seen.grow_zeroed(rows, c->stream));
    }
    return touched.grow(rows);
}

int32_t NeighbourStage::run_chunk(int64_t k, int64_t u0, int64_t rows, const int64_t *ex_off_, const int64_t *ex_, int64_t *ids_, double *scores_,
                                  int32_t *count_)
{
    gorse_b200_ctx *c = db->ctx;
    const NeighbourTable T{t_slot.p, t_score.p, t_cnt.p};
    const bool euclid = db->distance == GORSE_B200_DISTANCE_EUCLIDEAN;
    const uint8_t *ok = h_item_ok ? item_ok.p : nullptr;
    if (users) {
        const u2u::Users U{row.p + u0, ex_off_, ex_, ok, ids_, scores_, count_};
        const u2u::Route Rt{list.p, route.p + 2 * k, work.p, rows};
        return u2u::aggregate(c, Rt, U, T, u2u::Feedback{fb_off.p, fb_items.p, fb_rows}, n, scale, euclid, N, heavy, uacc.p, flag.p, touched.p);
    }
    // the chunk's users routed by |C_u| n
    const int64_t fill = i2i::route(c_off.data() + u0, rows, n, h_users);
    n_shared += fill;
    GB_CUDA(cudaMemcpyAsync(list.p, h_users.data(), sizeof(int32_t) * rows, cudaMemcpyHostToDevice, c->stream));
    const i2i::Users U{d_c_off.p + u0, row.p, ex_off_, ex_, ids_, scores_, count_};
    return i2i::aggregate(c, list.p, fill, rows - fill, U, T, ok, n, need, top, scale, euclid, N, acc.p, seen.p, touched.p);
}

int32_t neighbour_call(NeighbourStage &S, int64_t n_users, const int32_t *categories, int32_t n_categories, const std::vector<int64_t> &ex,
                       const std::vector<int64_t> &ex_off, int64_t *ids_out, double *scores_out, int32_t *count_out, int64_t *stats_out)
{
    const int64_t R = (int64_t)S.nb.size();
    if (R == 0) {
        std::fill(count_out, count_out + n_users, 0);
        return GORSE_B200_OK;
    }
    gorse_b200_ctx *c = S.db->ctx;
    ScopedDevice sd(c->device);
    StreamSync sync{c->stream, c->copy_stream};
    int64_t exact_rows = 0;
    GB_TRY(S.table(categories, n_categories, &exact_rows));
    GB_CUDA(cudaGetLastError());
    const int64_t cu = std::min<int64_t>(n_users, (int64_t)c->sm_count * 1024), n_chunks = div_up(n_users, cu), top = S.top;
    GB_TRY(S.reserve(cu, n_chunks));
    GB_TRY(S.ex_off.upload(ex_off.data(), ex_off.size(), c->stream));
    GB_TRY(S.ex.upload(ex.data(), ex.size(), c->stream));
    GB_TRY(S.ids.grow((size_t)n_users * top));
    GB_TRY(S.scores.grow((size_t)n_users * top));
    GB_TRY(S.count.grow((size_t)n_users));
    for (int64_t k = 0, u0 = 0; u0 < n_users; k++, u0 += cu) {
        const int64_t rows = std::min(cu, n_users - u0);
        GB_TRY(S.run_chunk(k, u0, rows, S.ex_off.p + u0, S.ex.p, S.ids.p + u0 * top, S.scores.p + u0 * top, S.count.p + u0));
        // a finished chunk is downloaded on the copy stream while the next one computes
        GB_CUDA(cudaEventRecord(c->copy_ev, c->stream));
        GB_CUDA(cudaStreamWaitEvent(c->copy_stream, c->copy_ev, 0));
        GB_CUDA(cudaMemcpyAsync(count_out + u0, S.count.p + u0, sizeof(int32_t) * rows, cudaMemcpyDeviceToHost, c->copy_stream));
        GB_CUDA(cudaMemcpyAsync(ids_out + u0 * top, S.ids.p + u0 * top, sizeof(int64_t) * rows * top, cudaMemcpyDeviceToHost, c->copy_stream));
        GB_CUDA(cudaMemcpyAsync(scores_out + u0 * top, S.scores.p + u0 * top, sizeof(double) * rows * top, cudaMemcpyDeviceToHost, c->copy_stream));
    }
    // the users per accumulator: item-to-item routes on the host (run_chunk counts), user-to-user on the device
    std::vector<int32_t> routed(S.users ? (size_t)n_chunks * 2 : 0);
    if (S.users)
        GB_CUDA(cudaMemcpyAsync(routed.data(), S.route.p, sizeof(int32_t) * n_chunks * 2, cudaMemcpyDeviceToHost, c->stream));
    GB_CUDA(cudaStreamSynchronize(c->stream));
    GB_CUDA(cudaStreamSynchronize(c->copy_stream));
    int64_t st[4] = {R, exact_rows, S.n_shared, S.users ? 0 : n_users - S.n_shared};
    for (size_t k = 0; k < routed.size(); k += 2) {
        st[2] += routed[k];
        st[3] += routed[k + 1];
    }
    if (stats_out) std::copy(st, st + 4, stats_out);
    return GORSE_B200_OK;
}

// stage A proper: the table rows of the R stored vectors d_nb (device) under db->d_allow
static int32_t compute_rows(gorse_b200_vecdb *db, int64_t R, const int64_t *d_nb, int n, int32_t *t_slot, float *t_score, int32_t *t_cnt,
                            int64_t *exact_rows)
{
    if (db->dim > 0) {
        std::lock_guard<std::mutex> lk2(db->dense->mu);
        const recall::Table table{t_slot, t_score, t_cnt, false, db->distance == GORSE_B200_DISTANCE_DOT, nullptr, nullptr, nullptr};
        return recall::recall_rows(db->dense, db->d_allow.p, R, nullptr, d_nb, n, nullptr, nullptr, nullptr, &table, nullptr, nullptr, nullptr,
                                   exact_rows);
    }
    std::lock_guard<std::mutex> lk2(db->sparse->mu);
    return sparse_search_rows(db->sparse, d_nb, R, db->d_allow.p, n, t_slot, t_score, t_cnt);
}

constexpr int ASSEMBLE_THREADS = 256;

// The call's table from the neighbour cache and the rows stage A computed, one warp per table row r: src[r] >= 0 is the
// pool row that holds r, else r is computed row m = -1 - src[r], and ins[m] >= 0 is the pool row it is also stored in.
// Only the first cnt entries of a row are read by stage B, so only they are copied.
__global__ void __launch_bounds__(ASSEMBLE_THREADS)
ncache_assemble_kernel(const int32_t *src, const int32_t *ins, int64_t R, int n, const int32_t *m_slot, const float *m_score, const int32_t *m_cnt,
                       uint2 *pool, int32_t *pool_cnt, int32_t *t_slot, float *t_score, int32_t *t_cnt)
{
    const int64_t r = ((int64_t)blockIdx.x * ASSEMBLE_THREADS + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (r >= R) return;
    const int32_t s = src[r];
    int32_t *ts = t_slot + r * n;
    float *tv = t_score + r * n;
    if (s >= 0) {
        const uint2 *e = pool + (int64_t)s * n;
        const int c = pool_cnt[s];
        for (int j = lane; j < c; j += 32) {
            const uint2 x = e[j];
            ts[j] = (int32_t)x.x;
            tv[j] = __uint_as_float(x.y);
        }
        if (lane == 0) t_cnt[r] = c;
        return;
    }
    const int64_t m = -1 - (int64_t)s;
    const int32_t p = ins[m];
    const int c = m_cnt[m];
    const int32_t *ms = m_slot + m * n;
    const float *mv = m_score + m * n;
    uint2 *e = pool + (int64_t)max(p, 0) * n;
    for (int j = lane; j < c; j += 32) {
        const int32_t slot = ms[j];
        const float score = mv[j];
        ts[j] = slot;
        tv[j] = score;
        if (p >= 0) e[j] = make_uint2((uint32_t)slot, __float_as_uint(score));
    }
    if (lane == 0) {
        t_cnt[r] = c;
        if (p >= 0) pool_cnt[p] = c;
    }
}

void ncache_reset(gorse_b200_vecdb *db)
{
    NeighbourCache &K = db->ncache;
    K.used = 0;
    K.row_of_slot.assign(db->ts.size(), -1);
    K.gen = db->gen;
}

int32_t neighbour_table(gorse_b200_vecdb *db, const std::vector<int64_t> &nb, int64_t *d_nb, int n, const int32_t *categories,
                        int32_t n_categories, int32_t *t_slot, float *t_score, int32_t *t_cnt, int64_t *exact_rows)
{
    gorse_b200_ctx *c = db->ctx;
    const int64_t R = (int64_t)nb.size();
    GB_TRY(vecdb_allow(db, categories, n_categories));
    NeighbourCache &K = db->ncache;
    if (K.cap == 0 || n != K.n || n_categories > 0) {
        GB_CUDA(cudaMemcpyAsync(d_nb, nb.data(), sizeof(int64_t) * R, cudaMemcpyHostToDevice, c->stream));
        return compute_rows(db, R, d_nb, n, t_slot, t_score, t_cnt, exact_rows);
    }
    if (K.gen != db->gen) {
        if (K.used > 0) K.emptied++;
        ncache_reset(db);
    }
    // hits and misses; a miss takes the next free pool row while there is one
    std::vector<int32_t> src((size_t)R);
    std::vector<int64_t> miss;
    std::vector<int32_t> ins;
    for (int64_t r = 0; r < R; r++) {
        int32_t &p = K.row_of_slot[(size_t)nb[(size_t)r]];
        if (p >= 0) {
            src[(size_t)r] = p;
            continue;
        }
        src[(size_t)r] = -1 - (int32_t)miss.size();
        miss.push_back(nb[(size_t)r]);
        ins.push_back(K.used < K.cap ? (int32_t)K.used++ : -1);
        p = ins.back();
    }
    const int64_t M = (int64_t)miss.size();
    src.insert(src.end(), ins.begin(), ins.end());
    auto fail = [&](int32_t st) {   // the rows claimed above may not have been written
        ncache_reset(db);
        return st;
    };
    int32_t st = GORSE_B200_OK;
    if (exact_rows) *exact_rows = 0;
    if (M > 0) {
        if ((st = K.m_slot.grow((size_t)M * n)) || (st = K.m_score.grow((size_t)M * n)) || (st = K.m_cnt.grow((size_t)M))) return fail(st);
        cudaError_t e = cudaMemcpyAsync(d_nb, miss.data(), sizeof(int64_t) * M, cudaMemcpyHostToDevice, c->stream);
        if (e != cudaSuccess) { set_error("neighbour cache upload: %s", cudaGetErrorString(e)); return fail(GORSE_B200_ERR_CUDA); }
        if ((st = compute_rows(db, M, d_nb, n, K.m_slot.p, K.m_score.p, K.m_cnt.p, exact_rows))) return fail(st);
    }
    if ((st = K.src.upload(src.data(), src.size(), c->stream))) return fail(st);
    ncache_assemble_kernel<<<div_up(R * 32, ASSEMBLE_THREADS), ASSEMBLE_THREADS, 0, c->stream>>>(
        K.src.p, K.src.p + R, R, n, K.m_slot.p, K.m_score.p, K.m_cnt.p, K.entry.p, K.cnt.p, t_slot, t_score, t_cnt);
    c->launches++;
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("neighbour cache: %s", cudaGetErrorString(e)); return fail(GORSE_B200_ERR_CUDA); }
    K.served += R - M;
    K.computed += M;
    return GORSE_B200_OK;
}

// the bytes per row of one fill chunk: the stage's table and slot list (8 n + 12), the cache's computed rows and sources
// (8 n + 12); their sum over a chunk stays within FILL_CHUNK_BYTES.  Stage A's own work buffers (recall_rows,
// sparse_search_rows) are sized by the chunk's rows as for any call of that many rows, and are not part of the bound.
constexpr int64_t FILL_CHUNK_BYTES = 64ll << 20;

// gorse_b200_vecdb_neighbour_cache_fill: the rows of every live slot the cache does not hold, in slot order, while the pool
// has room, through neighbour_table in chunks (every row a miss), so that each row is exactly what stage A stores for it.
// The chunk's table lands in the collection stage's grow-only buffers, which stage A of the entries uses as well.
static int32_t ncache_fill(gorse_b200_vecdb *db, int64_t *stats_out)
{
    gorse_b200_ctx *c = db->ctx;
    NeighbourCache &K = db->ncache;
    if (K.gen != db->gen) {
        if (K.used > 0) K.emptied++;
        ncache_reset(db);
    }
    const int n = K.n;
    std::vector<int64_t> todo;
    int64_t left = 0;
    for (size_t s = 0; s < db->dead.size(); s++) {
        if (db->dead[s] || K.row_of_slot[s] >= 0) continue;
        if (K.used + (int64_t)todo.size() < K.cap) todo.push_back((int64_t)s);
        else left++;
    }
    const int64_t chunk = std::max<int64_t>(1, FILL_CHUNK_BYTES / (16ll * n + 24));
    NeighbourStage &S = db->stage;
    Event ev[2];   // timed: the device time of the fill
    GB_TRY(ev[0].create(cudaEventDefault));
    if (ev[1].create(cudaEventDefault) != GORSE_B200_OK || cudaEventRecord(ev[0].e, c->stream) != cudaSuccess) {
        set_error("neighbour cache fill: events");
        return GORSE_B200_ERR_CUDA;
    }
    const int64_t computed = K.computed;
    std::vector<int64_t> nb;
    for (size_t i = 0; i < todo.size(); i += (size_t)chunk) {
        nb.assign(todo.begin() + (ptrdiff_t)i, todo.begin() + (ptrdiff_t)std::min(todo.size(), i + (size_t)chunk));
        const size_t R = nb.size();
        int32_t st = S.d_nb.grow(R);
        if (!st) st = S.t_slot.grow(R * n);
        if (!st) st = S.t_score.grow(R * n);
        if (!st) st = S.t_cnt.grow(R);
        if (!st) st = neighbour_table(db, nb, S.d_nb.p, n, nullptr, 0, S.t_slot.p, S.t_score.p, S.t_cnt.p, nullptr);
        if (st) {
            cudaStreamSynchronize(c->stream);
            return st;
        }
    }
    float ms = 0.f;
    cudaError_t e = cudaEventRecord(ev[1].e, c->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
    if (e == cudaSuccess) e = cudaEventElapsedTime(&ms, ev[0].e, ev[1].e);
    if (e != cudaSuccess) {
        set_error("neighbour cache fill: %s", cudaGetErrorString(e));
        return GORSE_B200_ERR_CUDA;
    }
    const int64_t st[4] = {K.computed - computed, K.used, left, (int64_t)(ms * 1000.0 + 0.5)};
    if (stats_out) std::copy(st, st + 4, stats_out);
    return GORSE_B200_OK;
}

}  // namespace gb

using namespace gb;

extern "C" int32_t gorse_b200_vecdb_neighbour_cache(gorse_b200_vecdb *db, int32_t n, int64_t rows)
{
    GB_CHECK_ARG(rows >= 0, "negative rows");
    GB_CHECK_ARG(n >= 1 && n <= MAX_N_DENSE, "n = %d outside [1, %d]", n, MAX_N_DENSE);
    GB_CHECK_ARG(db != nullptr, "collection is NULL");
    std::lock_guard<std::mutex> lk(db->mu);
    GB_TRY(check_stage_db(db, n, "neighbour cache"));
    NeighbourCache &K = db->ncache;
    if (rows == K.cap && (rows == 0 || n == K.n)) return GORSE_B200_OK;
    GB_CHECK_ARG(rows <= INT32_MAX, "rows = %lld above 2^31 - 1", (long long)rows);
    ScopedDevice sd(db->ctx->device);   // the old pool is freed on the collection's device too
    if (rows == 0) {
        K = NeighbourCache();
        return GORSE_B200_OK;
    }
    NeighbourCache fresh;   // allocated before the old pool goes, so a failure leaves the cache as it was
    GB_TRY(fresh.entry.alloc((size_t)rows * n));
    GB_TRY(fresh.cnt.alloc((size_t)rows));
    fresh.n = n;
    fresh.cap = rows;
    K = std::move(fresh);
    ncache_reset(db);
    return GORSE_B200_OK;
}

extern "C" int32_t gorse_b200_vecdb_neighbour_cache_stats(gorse_b200_vecdb *db, int64_t *stats_out)
{
    GB_CHECK_ARG(db != nullptr && stats_out != nullptr, "NULL collection or stats_out");
    std::lock_guard<std::mutex> lk(db->mu);
    const NeighbourCache &K = db->ncache;
    const int64_t s[7] = {K.cap ? K.n : 0, K.cap, K.used, (int64_t)K.bytes(), K.served, K.computed, K.emptied};
    std::copy(s, s + 7, stats_out);
    return GORSE_B200_OK;
}

extern "C" int32_t gorse_b200_vecdb_neighbour_cache_fill(gorse_b200_vecdb *db, int64_t *stats_out)
{
    GB_CHECK_ARG(db != nullptr, "collection is NULL");
    std::lock_guard<std::mutex> lk(db->mu);
    NeighbourCache &K = db->ncache;
    GB_TRY(check_stage_db(db, K.n, "neighbour cache fill"));
    if (K.cap == 0) {
        set_error("neighbour cache fill: the collection's neighbour cache is off");
        return GORSE_B200_ERR_STATE;
    }
    ScopedDevice sd(db->ctx->device);
    try {
        return ncache_fill(db, stats_out);
    } catch (const std::bad_alloc &) {
        set_error("neighbour cache fill: host allocation failed");
        return GORSE_B200_ERR_OOM;
    }
}

// the context and exclusion rows of both entries
static int32_t check_rows(const char *who, int64_t rows, const int32_t *count_out, const int64_t *ctx_off, const int64_t *ctx_slots,
                          const int64_t *excl_off, const int64_t *excl_slots)
{
    GB_CHECK_ARG(count_out != nullptr && ctx_off != nullptr && excl_off != nullptr, "count_out / ctx_off / excl_off is NULL");
    GB_TRY(check_offsets(ctx_off, rows, who, "ctx_off"));
    GB_TRY(check_offsets(excl_off, rows, who, "excl_off"));
    GB_CHECK_ARG(ctx_off[rows] == 0 || ctx_slots != nullptr, "ctx_slots is NULL");
    GB_CHECK_ARG(excl_off[rows] == 0 || excl_slots != nullptr, "excl_slots is NULL");
    return GORSE_B200_OK;
}

extern "C" int32_t gorse_b200_vecdb_item_to_item(gorse_b200_vecdb *db, int64_t n_users, const int64_t *ctx_off, const int64_t *ctx_slots,
                                                 const int64_t *excl_off, const int64_t *excl_slots, const int32_t *categories,
                                                 int32_t n_categories, int32_t n, double score_scale, int64_t *slots_out, double *scores_out,
                                                 int32_t *count_out, int64_t *stats_out)
{
    GB_CHECK_ARG(db != nullptr, "collection is NULL");
    GB_CHECK_ARG(n_users >= 0 && n_categories >= 0, "negative count");
    if (stats_out) std::fill(stats_out, stats_out + 4, 0);
    if (n_users == 0) return GORSE_B200_OK;
    GB_TRY(check_rows("item_to_item", n_users, count_out, ctx_off, ctx_slots, excl_off, excl_slots));
    GB_CHECK_ARG(score_scale == score_scale, "score_scale is NaN");
    std::lock_guard<std::mutex> lk(db->mu);
    GB_TRY(check_stage_db(db, n, "item_to_item"));
    if (n <= 0) {
        std::fill(count_out, count_out + n_users, 0);
        return GORSE_B200_OK;
    }
    GB_CHECK_ARG(slots_out != nullptr && scores_out != nullptr, "NULL output");
    GB_CHECK_ARG(n_categories == 0 || categories != nullptr, "categories is NULL");
    const int64_t n_slots = (int64_t)db->ts.size();
    for (int64_t u = 0; u < n_users; u++)
        for (int64_t t = ctx_off[u]; t < ctx_off[u + 1]; t++)
            GB_CHECK_ARG(ctx_slots[t] >= -1 && ctx_slots[t] < n_slots, "user %lld: context slot %lld is not a slot of the collection",
                         (long long)u, (long long)ctx_slots[t]);
    std::vector<int64_t> ex, ex_off;
    GB_TRY(exclusion_rows(n_users, excl_off, excl_slots, n_slots, "user", "slot", ex, ex_off));
    db->stage.prepare_items(db, n_users, ctx_off, ctx_slots, nullptr, n, 0, n, score_scale, nullptr);
    return neighbour_call(db->stage, n_users, categories, n_categories, ex, ex_off, slots_out, scores_out, count_out, stats_out);
}

extern "C" int32_t gorse_b200_vecdb_session_recommend(gorse_b200_vecdb *db, int64_t n_sessions, const int64_t *ctx_off, const int64_t *ctx_slots,
                                                      const int64_t *excl_off, const int64_t *excl_slots, const uint8_t *item_ok, int32_t n,
                                                      int32_t context_size, int32_t top, double score_scale, int64_t *slots_out,
                                                      double *scores_out, int32_t *count_out, int64_t *stats_out)
{
    // every check that needs no collection comes first, so that a bad argument is reported whatever db is
    GB_CHECK_ARG(n_sessions >= 0, "negative n_sessions");
    if (stats_out) std::fill(stats_out, stats_out + 4, 0);
    std::vector<int64_t> ex, ex_off;
    if (n_sessions > 0) {
        GB_TRY(check_rows("session_recommend", n_sessions, count_out, ctx_off, ctx_slots, excl_off, excl_slots));
        GB_CHECK_ARG(top <= 0 || (slots_out != nullptr && scores_out != nullptr), "slots_out / scores_out is NULL");
        for (int64_t t = 0; t < ctx_off[n_sessions]; t++)
            GB_CHECK_ARG(ctx_slots[t] >= -1, "context slot %lld is not a slot of the collection", (long long)ctx_slots[t]);
        // the upper bound of a slot needs the collection: checked below
        GB_TRY(exclusion_rows(n_sessions, excl_off, excl_slots, INT64_MAX, "session", "slot", ex, ex_off));
    }
    GB_CHECK_ARG(score_scale == score_scale, "score_scale is NaN");
    if (top > MAX_N_DENSE) {
        set_error("session_recommend: top = %d above %d", top, MAX_N_DENSE);
        return GORSE_B200_ERR_UNSUPPORTED;
    }
    GB_CHECK_ARG(db != nullptr, "collection is NULL");
    std::lock_guard<std::mutex> lk(db->mu);
    GB_TRY(check_stage_db(db, n, "session_recommend"));
    if (n <= 0) {   // n = 0 asks the store for one neighbour (n + 1) and keeps it: not served here
        set_error("session_recommend: n = %d is not at least 1", n);
        return GORSE_B200_ERR_UNSUPPORTED;
    }
    if (n_sessions == 0) return GORSE_B200_OK;
    const int64_t n_slots = (int64_t)db->ts.size();
    for (int64_t t = 0; t < ctx_off[n_sessions]; t++)
        GB_CHECK_ARG(ctx_slots[t] < n_slots, "context slot %lld is not a slot of the collection", (long long)ctx_slots[t]);
    for (int64_t t = 0; t < (int64_t)ex.size(); t++)
        GB_CHECK_ARG(ex[t] < n_slots, "excluded slot %lld is not a slot of the collection", (long long)ex[t]);
    if (top <= 0) {
        std::fill(count_out, count_out + n_sessions, 0);
        return GORSE_B200_OK;
    }
    const int need = std::max(context_size, 1);   // the handler stops once used >= ContextSize, after at least one list
    db->stage.prepare_items(db, n_sessions, ctx_off, ctx_slots, nullptr, n, need, top, score_scale, item_ok);
    return neighbour_call(db->stage, n_sessions, nullptr, 0, ex, ex_off, slots_out, scores_out, count_out, stats_out);
}
