// session.cu -- batched session recommendation: gorse_b200_vecdb_session_recommend.
//
// The REST server's session recommendation (sessionRecommend, server/rest.go:1069-1173) visits the posted session's positive
// feedback items, newest first; for each it asks QueryItemToItem(c, nil, CacheSize) (logics/item_to_item.go:50-86, no
// category filter), keeps the neighbours that FilterVisibleItemsByCategories passes (rest.go:815-832), adds their scores
// per id in float64 unless the id is in the session, and stops once ContextSize items have given a non-empty filtered list;
// the answer is TopKFilter(n + offset) of the sums.  Here one call answers many sessions:
//
//   stage A   the neighbour table of item_to_item.cu (neighbour_table, stages.cuh) for the distinct live context items of the
//             whole call, with the collection's own allow mask (live, not hidden) and k = n.  It cannot stop at the cut: whether
//             an entry counts depends on its filtered list.
//   stage B   session_aggregate_kernel, one CTA per session: finds the cut (the entry where the count of non-empty
//             item_ok-filtered lists reaches context_size) in one pass over the context with a warp scan of per-entry
//             ballots; adds s = (double)score * scale (Euclidean: 1 / (1 - s)) per filtered neighbour not in E_s over the
//             prefix, in order, with a barrier between entries (agg::add_sum: a shared-memory table when |C_s| * n <=
//             TABLE_KEYS, else this CTA's float64 row in global memory); then selects the first `top` by (score desc, slot
//             asc) with agg::select_first_n.
#include <algorithm>

#include "sparse.cuh"
#include "stages.cuh"

namespace gb {
namespace session {

constexpr int THREADS = agg::THREADS;
constexpr int MAX_TOP = 1024;                    // the sort buffer holds top entries

// One past the context entry e of [cb, ce) at which the count of entries with a non-empty filtered neighbour list reaches
// need, or ce when it never does.  Each window of NT entries: warp w tests entries w*32 .. w*32+31, its lanes splitting each
// list (__any_sync, stopping at the first passing neighbour), and records them as one bit mask; warp 0 scans the window's
// masks and picks the entry.  Every thread of the CTA calls it.
template <int NT>
__device__ int64_t context_cut(int64_t cb, int64_t ce, const int32_t *c_row, const i2i::Table &T, int n, const uint8_t *item_ok, int need,
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

// one CTA per session of `sessions`.  SHARED: the accumulator is a table in shared memory; else acc_rows / seen_rows /
// touched_rows hold one [N] float64 row, one [N] flag row (all zero between sessions) and one [N] slot list per CTA.  Row u
// of the answer is U.slots / U.scores [u * top, u * top + U.count[u]).
template <bool SHARED>
__global__ void __launch_bounds__(THREADS)
session_aggregate_kernel(const int32_t *sessions, int64_t n_sessions, i2i::Users U, i2i::Table T, const uint8_t *item_ok, int n, int need,
                         int top, double scale, int euclid, int64_t N, double *acc_rows, uint8_t *seen_rows, int32_t *touched_rows)
{
    using namespace gb::recall;
    using namespace gb::agg;
    constexpr int NT = THREADS;
    extern __shared__ __align__(16) uint8_t sm[];
    __shared__ unsigned s_mask[NT / 32];
    __shared__ int64_t s_cut;
    const int p2 = pow2_at_least(top);
    const Smem S = carve(sm, p2);
    int *s_bc = S.s_bc;
    int32_t *t_key = S.t_key;
    double *t_val = S.t_val;
    double *acc = SHARED ? nullptr : acc_rows + (int64_t)blockIdx.x * N;
    uint8_t *seen = SHARED ? nullptr : seen_rows + (int64_t)blockIdx.x * N;
    int32_t *touched = SHARED ? nullptr : touched_rows + (int64_t)blockIdx.x * N;
    for (int64_t i = blockIdx.x; i < n_sessions; i += gridDim.x) {
        const int64_t u = sessions[i];
        const int64_t cb = U.c_off[u];
        const int64_t ce = context_cut<NT>(cb, U.c_off[u + 1], U.c_row, T, n, item_ok, need, s_mask, &s_cut);
        const int64_t *ex = U.ex + U.ex_off[u], n_ex = U.ex_off[u + 1] - U.ex_off[u];
        int cap = 0, lg = 0;
        if (SHARED) {   // a power of two >= 2 * (the prefix's adds), at most TABLE_CAP: the load stays <= 3/4
            cap = min(TABLE_CAP, pow2_at_least(max(64, (int)(2 * (ce - cb) * n))));
            lg = __ffs(cap) - 1;
            for (int j = threadIdx.x; j < cap; j += NT) t_key[j] = -1;
        }
        if (threadIdx.x == 0) s_bc[3] = 0;
        __syncthreads();
        // the prefix in order; a barrier after each entry makes every sum the handler's left-to-right sum
        for (int64_t e = cb; e < ce; e++) {
            const int64_t r = U.c_row[e];
            const int cnt = T.cnt[r];
            for (int j = threadIdx.x; j < cnt; j += NT) {
                const int32_t slot = T.slot[r * n + j];
                if ((item_ok != nullptr && !item_ok[slot]) || contains(ex, n_ex, (int64_t)slot)) continue;
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

}  // namespace session
}  // namespace gb

using namespace gb;

extern "C" int32_t gorse_b200_vecdb_session_recommend(gorse_b200_vecdb *db, int64_t n_sessions, const int64_t *ctx_off, const int64_t *ctx_slots,
                                                      const int64_t *excl_off, const int64_t *excl_slots, const uint8_t *item_ok, int32_t n,
                                                      int32_t context_size, int32_t top, double score_scale, int64_t *slots_out,
                                                      double *scores_out, int32_t *count_out, int64_t *stats_out)
{
    using namespace gb::session;
    using gb::agg::grow_zeroed;
    using gb::agg::TABLE_KEYS;
    using gb::recall::grow;
    // every check that needs no collection comes first, so that a bad argument is reported whatever db is
    GB_CHECK_ARG(n_sessions >= 0, "negative n_sessions");
    if (stats_out) std::fill(stats_out, stats_out + 4, 0);
    std::vector<int64_t> ex, ex_off((size_t)n_sessions + 1, 0);
    if (n_sessions > 0) {
        GB_CHECK_ARG(count_out != nullptr && ctx_off != nullptr && excl_off != nullptr, "count_out / ctx_off / excl_off is NULL");
        GB_CHECK_ARG(ctx_off[0] == 0 && excl_off[0] == 0, "ctx_off[0] and excl_off[0] must be 0");
        for (int64_t u = 0; u < n_sessions; u++) {
            GB_CHECK_ARG(ctx_off[u + 1] >= ctx_off[u], "ctx_off decreases at %lld", (long long)u);
            GB_CHECK_ARG(excl_off[u + 1] >= excl_off[u], "excl_off decreases at %lld", (long long)u);
        }
        GB_CHECK_ARG(ctx_off[n_sessions] == 0 || ctx_slots != nullptr, "ctx_slots is NULL");
        GB_CHECK_ARG(excl_off[n_sessions] == 0 || excl_slots != nullptr, "excl_slots is NULL");
        GB_CHECK_ARG(top <= 0 || (slots_out != nullptr && scores_out != nullptr), "slots_out / scores_out is NULL");
        for (int64_t t = 0; t < ctx_off[n_sessions]; t++)
            GB_CHECK_ARG(ctx_slots[t] >= -1, "context slot %lld is not a slot of the collection", (long long)ctx_slots[t]);
        // each session's exclusions once, sorted, -1 entries dropped (as gorse_b200_vecdb_query_excluding)
        ex.reserve((size_t)excl_off[n_sessions]);
        for (int64_t u = 0; u < n_sessions; u++) {
            const size_t b = ex.size();
            for (int64_t t = excl_off[u]; t < excl_off[u + 1]; t++) {
                GB_CHECK_ARG(excl_slots[t] >= -1, "session %lld: excluded slot %lld is not a slot of the collection", (long long)u,
                             (long long)excl_slots[t]);
                if (excl_slots[t] >= 0) ex.push_back(excl_slots[t]);
            }
            std::sort(ex.begin() + b, ex.end());
            for (size_t t = b + 1; t < ex.size(); t++)
                GB_CHECK_ARG(ex[t] != ex[t - 1], "session %lld: slot %lld is excluded twice", (long long)u, (long long)ex[t]);
            ex_off[(size_t)u + 1] = (int64_t)ex.size();
        }
    }
    GB_CHECK_ARG(score_scale == score_scale, "score_scale is NaN");
    if (top > MAX_TOP) {
        set_error("session_recommend: top = %d above %d", top, MAX_TOP);
        return GORSE_B200_ERR_UNSUPPORTED;
    }
    GB_CHECK_ARG(db != nullptr, "collection is NULL");
    if (db->distance == GORSE_B200_DISTANCE_COSINE) {
        set_error("session collections are Dot or Euclidean");
        return GORSE_B200_ERR_UNSUPPORTED;
    }
    const bool sparse = db->dim == 0;
    const int max_n = sparse ? i2i::MAX_N_SPARSE : i2i::MAX_N_DENSE;
    if (n <= 0 || n > max_n) {   // n = 0 asks the store for one neighbour (n + 1) and keeps it: not served here
        set_error("session_recommend: n = %d outside [1, %d] for a %s collection", n, max_n, sparse ? "sparse" : "dense");
        return GORSE_B200_ERR_UNSUPPORTED;
    }
    if (n_sessions == 0) return GORSE_B200_OK;
    std::lock_guard<std::mutex> lk(db->mu);
    const int64_t n_slots = (int64_t)db->ts.size();
    if (n_slots > INT32_MAX) { set_error("session_recommend: more than 2^31 slots"); return GORSE_B200_ERR_UNSUPPORTED; }
    for (int64_t t = 0; t < ctx_off[n_sessions]; t++)
        GB_CHECK_ARG(ctx_slots[t] < n_slots, "context slot %lld is not a slot of the collection", (long long)ctx_slots[t]);
    for (int64_t t = 0; t < (int64_t)ex.size(); t++)
        GB_CHECK_ARG(ex[t] < n_slots, "excluded slot %lld is not a slot of the collection", (long long)ex[t]);
    if (top <= 0) {
        std::fill(count_out, count_out + n_sessions, 0);
        return GORSE_B200_OK;
    }
    // the live context entries as rows of the neighbour table: one row per distinct item, in first-visit order.  -1 and
    // deleted slots give an empty list (QueryItemToItem returns nil, logics/item_to_item.go:56-58) and never count; hidden
    // ones are queried.
    std::vector<int32_t> row_of((size_t)n_slots, -1), c_row;
    std::vector<int64_t> nb, c_off((size_t)n_sessions + 1, 0);
    c_row.reserve((size_t)ctx_off[n_sessions]);
    for (int64_t u = 0; u < n_sessions; u++) {
        for (int64_t t = ctx_off[u]; t < ctx_off[u + 1]; t++) {
            const int64_t s = ctx_slots[t];
            if (s < 0 || db->dead[(size_t)s]) continue;
            if (row_of[(size_t)s] < 0) {
                row_of[(size_t)s] = (int32_t)nb.size();
                nb.push_back(s);
            }
            c_row.push_back(row_of[(size_t)s]);
        }
        c_off[(size_t)u + 1] = (int64_t)c_row.size();
    }
    const int64_t R = (int64_t)nb.size();
    if (R == 0) {
        std::fill(count_out, count_out + n_sessions, 0);
        return GORSE_B200_OK;
    }
    gorse_b200_ctx *c = db->ctx;
    ScopedDevice sd(c->device);
    GB_TRY(vecdb_allow(db, nullptr, 0));
    ItemToItemWork &V = db->i2i;
    int32_t st = GORSE_B200_OK;
    auto done = [&](int32_t s) {
        cudaStreamSynchronize(c->stream);
        cudaStreamSynchronize(c->copy_stream);
        return s;
    };
    if ((st = grow(V.nb, (size_t)R)) || (st = grow(V.t_slot, (size_t)R * n)) || (st = grow(V.t_score, (size_t)R * n)) || (st = grow(V.t_cnt, (size_t)R)) ||
        (item_ok && (st = grow(V.item_ok, (size_t)n_slots))))
        return done(st);
    cudaError_t e = cudaMemcpyAsync(V.nb.p, nb.data(), sizeof(int64_t) * R, cudaMemcpyHostToDevice, c->stream);
    if (e == cudaSuccess && item_ok) e = cudaMemcpyAsync(V.item_ok.p, item_ok, (size_t)n_slots, cudaMemcpyHostToDevice, c->stream);
    if (e != cudaSuccess) { set_error("session_recommend upload: %s", cudaGetErrorString(e)); return done(GORSE_B200_ERR_CUDA); }

    // ---- stage A: the neighbour table
    int64_t exact_rows = 0;
    if ((st = neighbour_table(db, R, V.nb.p, n, V.t_slot.p, V.t_score.p, V.t_cnt.p, &exact_rows))) return done(st);
    if ((e = cudaGetLastError()) != cudaSuccess) { set_error("session_recommend: %s", cudaGetErrorString(e)); return done(GORSE_B200_ERR_CUDA); }

    // ---- stage B: sessions in chunks; a finished chunk is downloaded on the copy stream while the next one computes
    const int64_t cu = std::min<int64_t>(n_sessions, (int64_t)c->sm_count * 1024);
    const int64_t N = n_slots;
    const int hg = i2i::heavy_grid(c, N);
    const int64_t total_ctx = c_off[(size_t)n_sessions];
    if ((st = grow(V.c_off, (size_t)cu + 1)) || (st = grow(V.ex_off, (size_t)cu + 1)) || (st = grow(V.users, (size_t)cu)) ||
        (st = grow(V.c_row, (size_t)std::max<int64_t>(total_ctx, 1))) || (st = grow(V.ex, std::max<size_t>(ex.size(), 1))) ||
        (st = grow(V.slots, (size_t)n_sessions * top)) || (st = grow(V.scores, (size_t)n_sessions * top)) || (st = grow(V.count, (size_t)n_sessions)))
        return done(st);
    const size_t sm_shared = agg::smem_bytes(top, true), sm_global = agg::smem_bytes(top, false);
    if ((e = cudaFuncSetAttribute(session_aggregate_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm_shared)) != cudaSuccess ||
        (e = cudaFuncSetAttribute(session_aggregate_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm_global)) != cudaSuccess) {
        set_error("session_recommend: %s", cudaGetErrorString(e));
        return done(GORSE_B200_ERR_CUDA);
    }
    i2i::Table T;
    T.slot = V.t_slot.p; T.score = V.t_score.p; T.cnt = V.t_cnt.p;
    const bool euclid = db->distance == GORSE_B200_DISTANCE_EUCLIDEAN;
    const int need = std::max(context_size, 1);   // the handler stops once used >= ContextSize, after at least one list
    const uint8_t *d_ok = item_ok ? V.item_ok.p : nullptr;
    int64_t n_shared = 0, n_heavy = 0;
    std::vector<int64_t> h_coff, h_exoff;
    std::vector<int32_t> h_users;
    for (int64_t u0 = 0; u0 < n_sessions; u0 += cu) {
        const int64_t rows = std::min(cu, n_sessions - u0);
        h_coff.resize(rows + 1); h_exoff.resize(rows + 1); h_users.resize(rows);
        int64_t fill = 0, back = rows;   // table sessions from the front, heavy sessions from the back
        for (int64_t r = 0; r <= rows; r++) {
            h_coff[r] = c_off[u0 + r] - c_off[u0];
            h_exoff[r] = ex_off[u0 + r] - ex_off[u0];
        }
        for (int64_t r = 0; r < rows; r++) {
            if ((h_coff[r + 1] - h_coff[r]) * n <= TABLE_KEYS) h_users[fill++] = (int32_t)r;
            else h_users[--back] = (int32_t)r;
        }
        const int64_t heavy = rows - fill;
        n_shared += fill;
        n_heavy += heavy;
        if (heavy > 0 && ((st = grow(V.acc, (size_t)hg * N)) || (st = grow_zeroed(V.seen, (size_t)hg * N, c->stream)) ||
                          (st = grow(V.touched, (size_t)hg * N))))
            return done(st);
        const int64_t n_c = h_coff[rows], n_e = h_exoff[rows];
        if ((e = cudaMemcpyAsync(V.c_off.p, h_coff.data(), sizeof(int64_t) * (rows + 1), cudaMemcpyHostToDevice, c->stream)) != cudaSuccess ||
            (e = cudaMemcpyAsync(V.ex_off.p, h_exoff.data(), sizeof(int64_t) * (rows + 1), cudaMemcpyHostToDevice, c->stream)) != cudaSuccess ||
            (e = cudaMemcpyAsync(V.users.p, h_users.data(), sizeof(int32_t) * rows, cudaMemcpyHostToDevice, c->stream)) != cudaSuccess ||
            (n_c && (e = cudaMemcpyAsync(V.c_row.p + c_off[u0], c_row.data() + c_off[u0], sizeof(int32_t) * n_c, cudaMemcpyHostToDevice, c->stream)) != cudaSuccess) ||
            (n_e && (e = cudaMemcpyAsync(V.ex.p + ex_off[u0], ex.data() + ex_off[u0], sizeof(int64_t) * n_e, cudaMemcpyHostToDevice, c->stream)) != cudaSuccess)) {
            set_error("session_recommend upload: %s", cudaGetErrorString(e));
            return done(GORSE_B200_ERR_CUDA);
        }
        i2i::Users U;
        U.c_off = V.c_off.p; U.c_row = V.c_row.p + c_off[u0]; U.ex_off = V.ex_off.p; U.ex = V.ex.p + ex_off[u0];
        U.slots = V.slots.p + u0 * top; U.scores = V.scores.p + u0 * top; U.count = V.count.p + u0;
        if (fill > 0) {
            session_aggregate_kernel<true><<<(unsigned)std::min<int64_t>(fill, (int64_t)c->sm_count * 8), THREADS, sm_shared, c->stream>>>(
                V.users.p, fill, U, T, d_ok, n, need, top, score_scale, euclid, N, nullptr, nullptr, nullptr);
            c->launches++;
        }
        if (heavy > 0) {
            session_aggregate_kernel<false><<<(unsigned)std::min<int64_t>(heavy, hg), THREADS, sm_global, c->stream>>>(
                V.users.p + fill, heavy, U, T, d_ok, n, need, top, score_scale, euclid, N, V.acc.p, V.seen.p, V.touched.p);
            c->launches++;
        }
        if ((e = cudaGetLastError()) != cudaSuccess || (e = cudaEventRecord(c->copy_ev, c->stream)) != cudaSuccess ||
            (e = cudaStreamWaitEvent(c->copy_stream, c->copy_ev, 0)) != cudaSuccess ||
            (e = cudaMemcpyAsync(count_out + u0, V.count.p + u0, sizeof(int32_t) * rows, cudaMemcpyDeviceToHost, c->copy_stream)) != cudaSuccess ||
            (e = cudaMemcpyAsync(slots_out + u0 * top, V.slots.p + u0 * top, sizeof(int64_t) * rows * top, cudaMemcpyDeviceToHost, c->copy_stream)) != cudaSuccess ||
            (e = cudaMemcpyAsync(scores_out + u0 * top, V.scores.p + u0 * top, sizeof(double) * rows * top, cudaMemcpyDeviceToHost, c->copy_stream)) != cudaSuccess) {
            set_error("session_recommend: %s", cudaGetErrorString(e));
            return done(GORSE_B200_ERR_CUDA);
        }
    }
    if ((e = cudaStreamSynchronize(c->stream)) != cudaSuccess || (e = cudaStreamSynchronize(c->copy_stream)) != cudaSuccess) {
        set_error("session_recommend: %s", cudaGetErrorString(e));
        return done(GORSE_B200_ERR_CUDA);
    }
    if (stats_out) {
        stats_out[0] = R;
        stats_out[1] = exact_rows;
        stats_out[2] = n_shared;
        stats_out[3] = n_heavy;
    }
    return done(GORSE_B200_OK);
}
