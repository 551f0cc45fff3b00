// user_to_user.cu -- batched user-to-user recommendation: gorse_b200_vecdb_user_to_user.
//
// The worker's user-to-user recommender (logics/recommend.go:285-348) asks, per user, QueryUserToUser(u, n)
// (logics/user_to_user.go:50-86: top n + 1, drop u itself, drop Dot scores <= 0, stop at n), then for each similar user v
// in that order adds v's score to every item of v's positive feedback that is not in the exclude set, in float64, keeps
// the best n with TopKFilter and only then drops the items that are missing, hidden, too old or outside the categories.
// Here one call answers many users:
//
//   stage A   the neighbour table, once per call: the distinct live query slots of the batch are searched once each, with
//             the same stage A as item-to-item (item_to_item.cu): recall_rows with k = n and self-skip on dense
//             collections, sparse_search_rows on sparse ones, and no category filter.
//   routing   u2u_route_kernel, one thread per user: W_u = the feedback entries of u's neighbours; empty users are answered
//             here, the rest go to the shared-memory list (W_u <= TABLE_KEYS) or the global-row list.
//   stage B   u2u_aggregate_kernel, one CTA per user: walks the neighbours in table order with a barrier after each one;
//             the threads split the neighbour's feedback row and add s_v with float64 atomics; then the first n by
//             (sum desc, item asc) (agg::select_first_n), then the item filter as an ordered compaction.
#include <algorithm>

#include "sparse.cuh"
#include "stages.cuh"

namespace gb {
namespace u2u {

using agg::TABLE_CAP;
using agg::TABLE_KEYS;                           // a user takes the table when W_u <= this
constexpr int AGG_THREADS = agg::THREADS;

// W_u for each user of the chunk.  Users without a vector, neighbours or feedback get an empty row here.
__global__ void u2u_route_kernel(Users U, NeighbourTable T, Feedback F, int n, Route R)
{
    const int64_t u = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= R.users) return;
    const int32_t r = U.q_row[u];
    int64_t w = 0;
    if (r >= 0)
        for (int j = 0, cnt = T.cnt[r]; j < cnt; j++) {
            const int32_t v = T.slot[(int64_t)r * n + j];
            if (v < F.rows) w += F.off[v + 1] - F.off[v];
        }
    if (w == 0) {
        U.count[u] = 0;
        return;
    }
    if (w <= TABLE_KEYS) {
        R.work[u] = (int32_t)w;
        R.list[atomicAdd(&R.cnt[0], 1)] = (int32_t)u;
    } else {
        R.list[R.users - 1 - atomicAdd(&R.cnt[1], 1)] = (int32_t)u;
    }
}

// one CTA per user of the routed list, a fixed grid looping over the device's count.  SHARED: the accumulator is a table in
// shared memory; else acc_rows / flag_rows / touched_rows hold one [n_items] float64 row, one [n_items] flag row (all zero
// between users) and one [n_items] item list per CTA.
template <bool SHARED>
__global__ void __launch_bounds__(AGG_THREADS)
u2u_aggregate_kernel(Route R, Users U, NeighbourTable T, Feedback F, int n, double scale, int euclid, int64_t n_items, double *acc_rows,
                     int32_t *flag_rows, int32_t *touched_rows)
{
    using namespace gb::recall;
    using namespace gb::agg;
    constexpr int NT = AGG_THREADS;
    extern __shared__ __align__(16) uint8_t sm[];
    const int p2 = pow2_at_least(n);
    const Smem S = carve(sm, p2);
    double *acc = SHARED ? nullptr : acc_rows + (int64_t)blockIdx.x * n_items;
    int32_t *flag = SHARED ? nullptr : flag_rows + (int64_t)blockIdx.x * n_items;
    int32_t *touched = SHARED ? nullptr : touched_rows + (int64_t)blockIdx.x * n_items;
    const int n_list = R.cnt[SHARED ? 0 : 1];
    for (int64_t i = blockIdx.x; i < n_list; i += gridDim.x) {
        const int64_t u = SHARED ? R.list[i] : R.list[R.users - 1 - i];
        const int64_t r = U.q_row[u];
        const int64_t *ex = U.ex + U.ex_off[u], n_ex = U.ex_off[u + 1] - U.ex_off[u];
        int cap = 0, lg = 0;
        if (SHARED) {   // a power of two >= 2 W_u, at most TABLE_CAP: the load stays <= 3/4
            cap = min(TABLE_CAP, pow2_at_least(max(64, 2 * R.work[u])));
            lg = __ffs(cap) - 1;
            for (int j = threadIdx.x; j < cap; j += NT) {
                S.t_key[j] = -1;
                S.t_val[j] = 0.0;
            }
        }
        if (threadIdx.x == 0) S.s_bc[3] = 0;
        __syncthreads();
        // The neighbours in order, one step each.  Every sum starts at +0.0, the Go map's zero value, and each add is an
        // atomic float64 add, which rounds once like __dadd_rn.  Inside one step every add to an item adds the same s_v
        // (one neighbour's row may hold an item twice), so the sequence of values an item's sum takes does not depend on
        // the order of the atomics: the sum after the step is exactly the reference's sequential one.  The barrier after
        // each step orders the steps, so every sum is formed in neighbour order, as the reference forms it.
        for (int j = 0, cnt = T.cnt[r]; j < cnt; j++) {
            const int32_t v = T.slot[r * n + j];
            if (v >= F.rows) continue;   // no feedback: nothing to add, for every thread
            const double s = neighbour_score(T.score[r * n + j], scale, euclid);
            for (int64_t t = F.off[v] + threadIdx.x, e = F.off[v + 1]; t < e; t += NT) {
                const int32_t item = F.items[t];
                if (contains(ex, n_ex, (int64_t)item)) continue;
                if (SHARED) {
                    uint32_t h = ((uint32_t)item * 0x9E3779B1u) >> (32 - lg);
                    for (;;) {
                        const int32_t k = ((volatile int32_t *)S.t_key)[h];
                        if (k == item) break;
                        if (k < 0) {
                            // a failed claim returns what the bucket now holds: another thread's claim for the same item
                            // is this item's bucket; only another item's sends the probe on
                            const int32_t old = atomicCAS(&S.t_key[h], -1, item);
                            if (old == -1) atomicAdd(&S.s_bc[3], 1);
                            if (old == -1 || old == item) break;
                        }
                        h = (h + 1) & (uint32_t)(cap - 1);
                    }
                    atomicAdd(&S.t_val[h], s);
                } else {
                    // the first thread to flip the flag lists the item; a plain flag store could list it twice
                    if (atomicExch(&flag[item], 1) == 0) touched[atomicAdd(&S.s_bc[3], 1)] = item;
                    atomicAdd(&acc[item], s);
                }
            }
            __syncthreads();
        }
        const int distinct = S.s_bc[3];
        auto item_at = [&](int64_t j) -> int32_t { return SHARED ? S.t_key[j] : touched[j]; };
        auto val_at = [&](int64_t j) -> double { return SHARED ? S.t_val[j] : acc[touched[j]]; };
        const int m = select_first_n<NT>(SHARED ? cap : distinct, distinct, n, p2, item_at, val_at, S);
        // the item filter after the cut (the reference's BatchGetItems + categories check), keeping the order
        int kept = 0;
        for (int base = 0; base < m; base += NT) {
            const int j = base + threadIdx.x;
            const int32_t item = j < m ? (int32_t)(uint32_t)S.s_key[j] : 0;
            const bool ok = j < m && (U.item_ok == nullptr || U.item_ok[item]);
            int total;
            const int pos = kept + block_rank<NT>(ok, S.s_warp, total);
            if (ok) {
                U.items[u * n + pos] = item;
                U.scores[u * n + pos] = S.s_val[j];
            }
            kept += total;
        }
        if (threadIdx.x == 0) U.count[u] = kept;
        if (!SHARED)
            for (int j = threadIdx.x; j < distinct; j += NT) {
                const int32_t item = touched[j];
                flag[item] = 0;
                acc[item] = 0.0;
            }
        __syncthreads();
    }
}

int32_t aggregate(gorse_b200_ctx *c, const Route &R, const Users &U, const NeighbourTable &T, const Feedback &F, int n, double scale,
                  bool euclid, int64_t NI, bool heavy, double *acc, int32_t *flag, int32_t *touched)
{
    const size_t sm_shared = agg::smem_bytes(n, true), sm_global = agg::smem_bytes(n, false);
    GB_CUDA(cudaFuncSetAttribute(u2u_aggregate_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm_shared));
    GB_CUDA(cudaFuncSetAttribute(u2u_aggregate_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm_global));
    const int64_t rows = R.users;
    u2u_route_kernel<<<(unsigned)((rows + 255) / 256), 256, 0, c->stream>>>(U, T, F, n, R);
    u2u_aggregate_kernel<true><<<(unsigned)std::min<int64_t>(rows, (int64_t)c->sm_count * 8), AGG_THREADS, sm_shared, c->stream>>>(
        R, U, T, F, n, scale, euclid, NI, nullptr, nullptr, nullptr);
    c->launches += 2;
    if (heavy) {
        u2u_aggregate_kernel<false><<<(unsigned)std::min<int64_t>(rows, heavy_grid(c, NI, ROW_BYTES)), AGG_THREADS, sm_global, c->stream>>>(
            R, U, T, F, n, scale, euclid, NI, acc, flag, touched);
        c->launches++;
    }
    GB_CUDA(cudaGetLastError());
    return GORSE_B200_OK;
}

}  // namespace u2u
}  // namespace gb

using namespace gb;

extern "C" int32_t gorse_b200_vecdb_user_to_user(gorse_b200_vecdb *db, int64_t n_users, const int64_t *user_slots, int64_t n_fb_rows,
                                                 const int64_t *fb_off, const int32_t *fb_items, int32_t n_items, const uint8_t *item_ok,
                                                 const int64_t *excl_off, const int64_t *excl_items, int32_t n, double score_scale,
                                                 int64_t *items_out, double *scores_out, int32_t *count_out, int64_t *stats_out)
{
    GB_CHECK_ARG(db != nullptr, "collection is NULL");
    GB_CHECK_ARG(n_users >= 0 && n_fb_rows >= 0 && n_items >= 0, "negative count");
    if (stats_out) std::fill(stats_out, stats_out + 4, 0);
    if (n_users == 0) return GORSE_B200_OK;
    GB_CHECK_ARG(count_out != nullptr && user_slots != nullptr && excl_off != nullptr, "count_out / user_slots / excl_off is NULL");
    GB_TRY(check_offsets(excl_off, n_users, "user_to_user", "excl_off"));
    GB_CHECK_ARG(excl_off[n_users] == 0 || excl_items != nullptr, "excl_items is NULL");
    GB_TRY(check_feedback("user_to_user", n_fb_rows, fb_off, fb_items, n_items));
    GB_CHECK_ARG(score_scale == score_scale, "score_scale is NaN");
    std::lock_guard<std::mutex> lk(db->mu);
    GB_TRY(check_stage_db(db, n, "user_to_user"));
    if (n <= 0) {
        std::fill(count_out, count_out + n_users, 0);
        return GORSE_B200_OK;
    }
    GB_CHECK_ARG(items_out != nullptr && scores_out != nullptr, "NULL output");
    const int64_t n_slots = (int64_t)db->ts.size();
    for (int64_t u = 0; u < n_users; u++)
        GB_CHECK_ARG(user_slots[u] >= -1 && user_slots[u] < n_slots, "user %lld: slot %lld is not a slot of the collection", (long long)u,
                     (long long)user_slots[u]);
    std::vector<int64_t> ex, ex_off;
    GB_TRY(exclusion_rows(n_users, excl_off, excl_items, n_items, "user", "item", ex, ex_off));
    db->stage.prepare_users(db, n_users, user_slots, n_fb_rows, fb_off, fb_items, n_items, n, score_scale, item_ok);
    return neighbour_call(db->stage, n_users, nullptr, 0, ex, ex_off, items_out, scores_out, count_out, stats_out);
}
