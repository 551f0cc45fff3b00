// vecdb.cuh -- state of one vector collection (vecdb.cu), shared with the batched recall (recall.cu), item-to-item and
// session (item_to_item.cu) and user-to-user (user_to_user.cu).
#pragma once
#include "topk.cuh"

namespace gb {
// grow-only work buffers of gorse_b200_vecdb_item_to_item and gorse_b200_vecdb_session_recommend (item_to_item.cu),
// which both hold the collection's lock: the neighbour table of stage A, the user or session batches, answers
// and accumulator scratch of stage B, and the session call's item mask
struct ItemToItemWork {
    DevBuf<int64_t> nb, c_off, ex_off, ex, slots;
    DevBuf<int32_t> t_slot, t_cnt, c_row, users, count;
    DevBuf<float> t_score;
    DevBuf<double> scores, acc;
    DevBuf<uint8_t> seen, item_ok;
    DevBuf<int32_t> touched;
    size_t bytes() const
    {
        return nb.bytes() + c_off.bytes() + ex_off.bytes() + ex.bytes() + slots.bytes() + t_slot.bytes() + t_cnt.bytes() + c_row.bytes() +
               users.bytes() + count.bytes() + t_score.bytes() + scores.bytes() + acc.bytes() + seen.bytes() + item_ok.bytes() + touched.bytes();
    }
};

// grow-only work buffers of gorse_b200_vecdb_user_to_user (user_to_user.cu): the neighbour table of stage A, the caller's
// feedback rows and item filter, the user chunks, their routing and answers, and the global-row accumulators of stage B
struct UserToUserWork {
    DevBuf<int64_t> nb, fb_off, ex_off, ex, items;
    DevBuf<int32_t> t_slot, t_cnt, fb_items, q_row, list, work, route_cnt, count, flag, touched;
    DevBuf<uint8_t> item_ok;
    DevBuf<float> t_score;
    DevBuf<double> scores, acc;
    size_t bytes() const
    {
        return nb.bytes() + fb_off.bytes() + ex_off.bytes() + ex.bytes() + items.bytes() + t_slot.bytes() + t_cnt.bytes() + fb_items.bytes() +
               q_row.bytes() + list.bytes() + work.bytes() + route_cnt.bytes() + count.bytes() + flag.bytes() + touched.bytes() +
               item_ok.bytes() + t_score.bytes() + scores.bytes() + acc.bytes();
    }
};

// gorse_b200_vecdb_neighbour_cache: the first n neighbours of up to `cap` stored vectors, as stage A (neighbour_table,
// item_to_item.cu) computes them without a category filter.  Pool row p holds cnt[p] entries (int32 slot, float32 score
// bits) of 8 bytes each at entry[p * n].  Rows are taken in the order they are computed and never evicted; the cache empties
// when the collection's generation moves past `gen`.
struct NeighbourCache {
    int32_t n = 0;
    int64_t cap = 0, used = 0;             // cap = 0: off
    DevBuf<uint2> entry;                   // [cap x n]
    DevBuf<int32_t> cnt;                   // [cap]
    std::vector<int32_t> row_of_slot;      // [slots]: the pool row of a slot, -1 = not held
    uint64_t gen = 0;                      // the collection's generation the held rows belong to
    int64_t served = 0, computed = 0, emptied = 0;
    // one call's work: the rows stage A computes, their table and each table row's source (see ncache_assemble_kernel)
    DevBuf<int32_t> m_slot, m_cnt, src;
    DevBuf<float> m_score;
    size_t bytes() const { return entry.bytes() + cnt.bytes() + m_slot.bytes() + m_cnt.bytes() + src.bytes() + m_score.bytes(); }
};
}  // namespace gb

struct gorse_b200_vecdb {
    gorse_b200_ctx *ctx = nullptr;
    int32_t dim = 0, distance = 0;
    gorse_b200_index *dense = nullptr;           // dim > 0
    gorse_b200_sparse_index *sparse = nullptr;   // dim == 0
    std::mutex mu;
    // host metadata (authoritative) + lazily refreshed device copies for the filter kernel
    std::vector<uint8_t> hidden, dead;
    std::vector<int64_t> ts;
    std::vector<int64_t> cat_off{0};
    std::vector<int32_t> cats;
    int64_t live = 0;
    bool meta_dirty = true;
    uint64_t gen = 0;   // moves with every change of the collection (wherever meta_dirty is set): empties the neighbour cache
    gb::DevBuf<uint8_t> d_blocked, d_allow;   // blocked = hidden | dead
    gb::DevBuf<int64_t> d_cat_off;
    gb::DevBuf<int32_t> d_cats, d_want;
    gb::ItemToItemWork i2i;  // batched item-to-item and session recommendation (item_to_item.cu)
    gb::UserToUserWork u2u;  // batched user-to-user recommendation (user_to_user.cu)
    gb::NeighbourCache ncache;   // stage A's rows kept between calls (gorse_b200_vecdb_neighbour_cache, item_to_item.cu)
};

namespace gb {
// allow mask d_allow[slot] of one query filter (live, not hidden, every wanted category); the caller holds db->mu
int32_t vecdb_allow(gorse_b200_vecdb *db, const int32_t *categories, int32_t n_categories);
// the renumbering of compaction and snapshots: scan[slots + 1] (device, allocated here) = the exclusive sum of the live flags,
// so slot s is live iff scan[s + 1] != scan[s] and then moves to scan[s]; new_slot[slots + 1] (host, may be nullptr) receives
// a copy.  Ends with the stream synchronised.  The caller holds db->mu and the device.
int32_t vecdb_live_scan(gorse_b200_vecdb *db, DevBuf<int64_t> &scan, int64_t *new_slot);
}  // namespace gb
