// vecdb.cuh -- state of one vector collection (vecdb.cu), shared with the batched recall (recall.cu), item-to-item and
// session (item_to_item.cu) and user-to-user (user_to_user.cu).
#pragma once
#include "topk.cuh"

namespace gb {
// One item-to-item or user-to-user stage over a collection: a batch's table rows on the host, and the grow-only device
// buffers of stage A and stage B.  The collection keeps one for its entries (db->stage, under db->mu), gorse_b200_recommend
// one per stage (rec::Work).  A call runs prepare_items or prepare_users, table, reserve, then run_chunk per chunk of users.
struct NeighbourStage {
    gorse_b200_vecdb *db = nullptr;
    bool users = false;                      // user-to-user; else item-to-item (session: need > 0)
    int n = 0, need = 0, top = 0;            // top: the answer row length (user-to-user: n)
    double scale = 1.0;
    int64_t N = 0;                           // the length of a global accumulator row: slots, or items (at least 1)
    bool heavy = false;                      // some user may need a global accumulator row
    int64_t n_shared = 0;                    // item-to-item: the users run_chunk routed to the shared-memory table
    std::vector<int64_t> nb;                 // the distinct query slots, as the table's rows
    std::vector<int64_t> c_off;              // item-to-item: [users + 1] into c_row
    std::vector<int32_t> c_row;              // item-to-item: the table row of each live context entry, in order
    std::vector<int32_t> q_row;              // user-to-user: [users] the table row of each user, -1 = no vector
    const uint8_t *h_item_ok = nullptr;      // the caller's item mask (session: slots; user-to-user: items) or NULL
    int64_t item_ok_len = 0;
    const int64_t *h_fb_off = nullptr;       // user-to-user: the caller's feedback CSR
    const int32_t *h_fb_items = nullptr;
    int64_t fb_rows = 0;
    std::vector<int32_t> h_users;            // item-to-item: one chunk's routing

    DevBuf<int64_t> d_nb, fb_off, d_c_off, ex_off, ex, ids;
    DevBuf<int32_t> t_slot, t_cnt, row, fb_items, list, work, route, count, flag, touched;
    DevBuf<float> t_score;
    DevBuf<uint8_t> item_ok, seen;
    // the global rows: item-to-item leaves acc dirty (seen is zero between users), user-to-user's uacc must be zero
    // between users (its kernel adds into it), so the two are kept apart
    DevBuf<double> scores, acc, uacc;
    // gorse_b200_recommend's item-to-item stage, whose exclude sets hold items: slot_of_item and item_of_slot on the
    // device, and the exclude set in slots (E0 on the host and the device, and two copies that take turns)
    std::vector<int64_t> es0, es0_off;
    DevBuf<int64_t> map, d_es0, d_es0_off, es[2];
    DevBuf<int32_t> item_of_slot;

    size_t bytes() const
    {
        size_t b = 0;
        for (const auto *x : {&d_nb, &fb_off, &d_c_off, &ex_off, &ex, &ids, &map, &d_es0, &d_es0_off, &es[0], &es[1]}) b += x->bytes();
        for (const auto *x : {&t_slot, &t_cnt, &row, &fb_items, &list, &work, &route, &count, &flag, &touched, &item_of_slot}) b += x->bytes();
        for (const auto *x : {&scores, &acc, &uacc}) b += x->bytes();
        return b + t_score.bytes() + item_ok.bytes() + seen.bytes();
    }

    // item-to-item: the live context entries ctx[ctx_off[u], ctx_off[u + 1]) of each user as table rows, the entries being
    // slots, or items through slot_of_item when it is given.  item_ok: a slot mask or NULL; need > 0: session
    // (i2i::aggregate).  stages.cuh.
    template <typename Id>
    void prepare_items(gorse_b200_vecdb *d, int64_t n_users, const int64_t *ctx_off, const Id *ctx, const int64_t *slot_of_item, int n_,
                       int need_, int top_, double scale_, const uint8_t *item_ok_);
    // user-to-user: the live query slot of each user as a table row, and the caller's feedback rows (slots at or beyond
    // fb_rows have none).  item_ok: an item mask or NULL.  stages.cuh.
    void prepare_users(gorse_b200_vecdb *d, int64_t n_users, const int64_t *user_slots, int64_t fb_rows_, const int64_t *fb_off_,
                       const int32_t *fb_items_, int32_t n_items, int n_, double scale_, const uint8_t *item_ok_);
    // the inputs of stage B (table rows, feedback, item mask), then stage A (neighbour_table) when the batch has rows.
    // categories: the neighbour query's filter (item-to-item only).  The caller holds db->mu.
    int32_t table(const int32_t *categories, int32_t n_categories, int64_t *exact_rows);
    // the chunk buffers for chunks of at most max_rows users, n_chunks of them, and the global rows when heavy
    int32_t reserve(int64_t max_rows, int64_t n_chunks);
    // stage B of chunk k, the users [u0, u0 + rows), against their exclusion rows ex_off [rows + 1] / ex on the device
    // (ascending per user; slots for item-to-item, items for user-to-user); answer row u of the chunk at ids / scores +
    // u * top, its length in count[u]
    int32_t run_chunk(int64_t k, int64_t u0, int64_t rows, const int64_t *ex_off, const int64_t *ex, int64_t *ids, double *scores,
                      int32_t *count);

private:
    void start(gorse_b200_vecdb *d, bool users_, int n_, double scale_, const uint8_t *item_ok_, int64_t item_ok_len_)
    {
        db = d;
        users = users_;
        n = n_;
        scale = scale_;
        h_item_ok = item_ok_;
        item_ok_len = item_ok_len_;
        heavy = false;
        n_shared = 0;
        h_fb_off = nullptr;
        h_fb_items = nullptr;
        fb_rows = 0;
        nb.clear(); c_off.clear(); c_row.clear(); q_row.clear(); es0.clear(); es0_off.clear();
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
    gb::NeighbourStage stage;   // item-to-item, session and user-to-user recommendation (item_to_item.cu, user_to_user.cu)
    gb::NeighbourCache ncache;   // stage A's rows kept between calls (gorse_b200_vecdb_neighbour_cache, item_to_item.cu)
};

namespace gb {
// allow mask d_allow[slot] of one query filter (live, not hidden, every wanted category); the caller holds db->mu
int32_t vecdb_allow(gorse_b200_vecdb *db, const int32_t *categories, int32_t n_categories);
// the renumbering of compaction and snapshots: scan[slots + 1] (device, allocated here) = the exclusive sum of the live flags,
// so slot s is live iff scan[s + 1] != scan[s] and then moves to scan[s]; new_slot[slots + 1] (host, may be nullptr) receives
// a copy.  Ends with the stream synchronised.  The caller holds db->mu and the device.
int32_t vecdb_live_scan(gorse_b200_vecdb *db, DevBuf<int64_t> &scan, int64_t *new_slot);
// the neighbour cache as it was turned on: nothing held, every slot of the collection's current generation unknown
// (item_to_item.cu).  The caller holds db->mu.
void ncache_reset(gorse_b200_vecdb *db);
}  // namespace gb
