// stages.cuh -- the device bodies of the batched neighbour recommenders and their host preparation: item-to-item and
// session (item_to_item.cu), user-to-user (user_to_user.cu), taking device pointers, so that the vecdb entries and the
// batched offline recommendation (recommend.cu) launch the same kernels and prepare their inputs the same way.
#pragma once
#include <algorithm>
#include <vector>

#include "aggregate.cuh"
#include "vecdb.cuh"

namespace gb {

constexpr int MAX_N_DENSE = 1024;                // the sort buffer of agg::select_first_n holds n (session: top) entries
constexpr int MAX_N_SPARSE = 128;                // the sparse search's k

// stage A of every neighbour recommender: the first n neighbours of each of the distinct stored vectors nb (host slots) of db
// among the vectors that pass categories[n_categories] (vecdb_allow runs here), as a table of n (int32 slot, float32 score)
// entries per row, Dot collections keeping scores > 0 only (dense: the index's top-k pipeline; sparse: sparse_search_rows).
// A call with the neighbour cache's n and no category filter takes the rows the cache holds and computes only the others
// (gorse_b200_vecdb_neighbour_cache); every row is the same either way.  d_nb: device scratch of nb.size() entries.  The
// caller holds db->mu.  *exact_rows: computed rows the exact scan answered.
int32_t neighbour_table(gorse_b200_vecdb *db, const std::vector<int64_t> &nb, int64_t *d_nb, int n, const int32_t *categories,
                        int32_t n_categories, int32_t *t_slot, float *t_score, int32_t *t_cnt, int64_t *exact_rows);

struct NeighbourTable {       // stage A: the first n neighbours of each distinct query
    const int32_t *slot;      // [rows x n]
    const float *score;       // [rows x n] the vector store's score (dot, or the negated distance)
    const int32_t *cnt;       // [rows]
};

// global accumulator rows (one [N] entry of row_bytes per CTA, at most 512 MB): how many CTAs
inline int heavy_grid(const gorse_b200_ctx *c, int64_t N, int64_t row_bytes)
{
    return (int)std::max<int64_t>(1, std::min<int64_t>((int64_t)c->sm_count * 2, (512ll << 20) / (row_bytes * N)));
}

// Each row's ids once, ascending, -1 entries dropped: the ids [off[r], off[r + 1]) of row r into ex, with ex_off [rows + 1].
// An id outside [-1, bound) or twice in one row is an argument error; `row` and `id` name them in its message ("user",
// "slot").
template <typename Id>
int32_t exclusion_rows(int64_t rows, const int64_t *off, const Id *ids, int64_t bound, const char *row, const char *id, std::vector<int64_t> &ex,
                       std::vector<int64_t> &ex_off)
{
    ex.clear();
    ex.reserve((size_t)off[rows]);
    ex_off.assign((size_t)rows + 1, 0);
    for (int64_t r = 0; r < rows; r++) {
        const size_t b = ex.size();
        for (int64_t t = off[r]; t < off[r + 1]; t++) {
            const int64_t s = ids[t];
            GB_CHECK_ARG(s >= -1 && s < bound, "%s %lld: excluded %s %lld is not a%s %s", row, (long long)r, id, (long long)s,
                         id[0] == 'i' ? "n" : "", id);
            if (s >= 0) ex.push_back(s);
        }
        std::sort(ex.begin() + b, ex.end());
        for (size_t t = b + 1; t < ex.size(); t++)
            GB_CHECK_ARG(ex[t] != ex[t - 1], "%s %lld: %s %lld is excluded twice", row, (long long)r, id, (long long)ex[t]);
        ex_off[(size_t)r + 1] = (int64_t)ex.size();
    }
    return GORSE_B200_OK;
}

// The neighbour-table row of slot s of db: -1 for -1 and for a deleted slot (GetVectors returns nothing); else the rows
// follow the first visit of each slot, a new slot appended to nb.  row_of: [slots], all -1 before the first call.
inline int32_t table_row(const gorse_b200_vecdb *db, int64_t s, std::vector<int32_t> &row_of, std::vector<int64_t> &nb)
{
    if (s < 0 || db->dead[(size_t)s]) return -1;
    if (row_of[(size_t)s] < 0) {
        row_of[(size_t)s] = (int32_t)nb.size();
        nb.push_back(s);
    }
    return row_of[(size_t)s];
}

namespace i2i {
constexpr int64_t ROW_BYTES = 8 + 1 + 4;         // a global row entry: float64 sum, seen flag, touched slot

struct Users {                // one chunk of users (chunk-local ids)
    const int64_t *c_off;     // [users + 1] into c_row
    const int32_t *c_row;     // the neighbour-table row of each live context entry, in the caller's order
    const int64_t *ex_off;    // [users + 1] into ex
    const int64_t *ex;        // each user's excluded slots, ascending (-1 entries dropped; may be padded with INT64_MAX)
    int64_t *slots;           // [users x top]
    double *scores;           // [users x top]
    int32_t *count;           // [users]
};

// The users rows [0, rows) of a context CSR c_off in routing order: users[0, fill) take the shared-memory table
// (|C_u| * n <= TABLE_KEYS), in order, users[fill, rows) a global row, in reverse order.  Returns fill.
inline int64_t route(const int64_t *c_off, int64_t rows, int n, std::vector<int32_t> &users)
{
    users.resize((size_t)rows);
    int64_t fill = 0, back = rows;
    for (int64_t r = 0; r < rows; r++) {
        if ((c_off[r + 1] - c_off[r]) * n <= agg::TABLE_KEYS) users[(size_t)fill++] = (int32_t)r;
        else users[(size_t)--back] = (int32_t)r;
    }
    return fill;
}

// stage B for one chunk: d_users[0, fill) aggregate in shared memory, d_users[fill, fill + heavy) in the global rows acc /
// seen (zeroed) / touched of heavy_grid(c, N, ROW_BYTES) CTAs.  item_ok: a slot mask or NULL; need > 0: walk each context
// only up to the need-th entry whose item_ok-filtered list is not empty (session); the answer rows hold top entries.
int32_t aggregate(gorse_b200_ctx *c, const int32_t *d_users, int64_t fill, int64_t heavy, const Users &U, const NeighbourTable &T,
                  const uint8_t *item_ok, int n, int need, int top, double scale, bool euclid, int64_t N, double *acc, uint8_t *seen,
                  int32_t *touched);
}  // namespace i2i

namespace u2u {
constexpr int64_t ROW_BYTES = 8 + 4 + 4;         // a global row entry: float64 sum, flag, touched item

struct Feedback {             // the caller's positive feedback per slot, as item indices
    const int64_t *off;       // [rows + 1]
    const int32_t *items;
    int64_t rows;             // slots at or beyond have none
};

struct Users {                // one chunk of users (chunk-local ids)
    const int32_t *q_row;     // [users] the neighbour-table row of each user, -1 = no vector
    const int64_t *ex_off;    // [users + 1] into ex
    const int64_t *ex;        // each user's excluded items, ascending (-1 entries dropped; may be padded with INT64_MAX)
    const uint8_t *item_ok;   // [n_items] or NULL
    int64_t *items;           // [users x n]
    double *scores;           // [users x n]
    int32_t *count;           // [users]
};

struct Route {                // the device's routing of one chunk
    int32_t *list;            // [users]: shared-memory users from the front, global-row users from the back
    int32_t *cnt;             // [2]: how many of each (zeroed by the caller)
    int32_t *work;            // [users] W_u
    int64_t users;
};

// routing and stage B for one chunk of R.users users; heavy: some user may need a global row (acc / flag zeroed, touched,
// heavy_grid(c, NI, ROW_BYTES) CTAs)
int32_t aggregate(gorse_b200_ctx *c, const Route &R, const Users &U, const NeighbourTable &T, const Feedback &F, int n, double scale,
                  bool euclid, int64_t NI, bool heavy, double *acc, int32_t *flag, int32_t *touched);
}  // namespace u2u

// -1 and deleted slots are skipped (GetVectors returns nothing, logics/item_to_item.go:56-58) and never count for a session;
// hidden ones are queried
template <typename Id>
void NeighbourStage::prepare_items(gorse_b200_vecdb *d, int64_t n_users, const int64_t *ctx_off, const Id *ctx, const int64_t *slot_of_item,
                                   int n_, int need_, int top_, double scale_, const uint8_t *item_ok_)
{
    start(d, false, n_, scale_, item_ok_, (int64_t)d->ts.size());
    need = need_;
    top = top_;
    N = std::max<int64_t>((int64_t)d->ts.size(), 1);
    std::vector<int32_t> row_of(d->ts.size(), -1);
    c_off.assign((size_t)n_users + 1, 0);
    c_row.reserve((size_t)ctx_off[n_users]);
    for (int64_t u = 0; u < n_users; u++) {
        for (int64_t t = ctx_off[u]; t < ctx_off[u + 1]; t++) {
            const int64_t id = ctx[t];
            const int32_t r = table_row(d, id < 0 || !slot_of_item ? id : slot_of_item[id], row_of, nb);
            if (r >= 0) c_row.push_back(r);
        }
        c_off[(size_t)u + 1] = (int64_t)c_row.size();
    }
    heavy = i2i::route(c_off.data(), n_users, n, h_users) < n_users;
}

// -1 and deleted slots have no row (GetVectors returns nothing, logics/user_to_user.go:55-58); hidden ones are searched
inline void NeighbourStage::prepare_users(gorse_b200_vecdb *d, int64_t n_users, const int64_t *user_slots, int64_t fb_rows_, const int64_t *fb_off_,
                                          const int32_t *fb_items_, int32_t n_items, int n_, double scale_, const uint8_t *item_ok_)
{
    start(d, true, n_, scale_, item_ok_, n_items);
    top = n_;
    N = std::max<int64_t>(n_items, 1);
    h_fb_off = fb_off_;
    h_fb_items = fb_items_;
    fb_rows = fb_rows_;
    std::vector<int32_t> row_of(d->ts.size(), -1);
    q_row.resize((size_t)n_users);
    for (int64_t u = 0; u < n_users; u++) q_row[(size_t)u] = table_row(d, user_slots[u], row_of, nb);
    // the most any user can add: n neighbours with the longest feedback row.  Below the table's limit no user needs a
    // global row, so none is allocated.
    int64_t longest = 0;
    for (int64_t v = 0; v < fb_rows; v++) longest = std::max(longest, fb_off_[v + 1] - fb_off_[v]);
    heavy = longest * std::max(n, 0) > agg::TABLE_KEYS;
}

// The collection entries after their checks and prepare: stage A, then the users in chunks of sm_count * 1024 against the
// checked exclusion rows ex / ex_off, each finished chunk downloaded on the copy stream while the next one computes.
// stats_out: the table's rows, those the exact scan answered, the users per accumulator.  The caller holds db->mu.
int32_t neighbour_call(NeighbourStage &S, int64_t n_users, const int32_t *categories, int32_t n_categories, const std::vector<int64_t> &ex,
                       const std::vector<int64_t> &ex_off, int64_t *ids_out, double *scores_out, int32_t *count_out, int64_t *stats_out);

// The checks every neighbour stage makes of its collection at n: Cosine, n above the dense or sparse limit and 2^31 slots
// or more are GORSE_B200_ERR_UNSUPPORTED.  In this and the checks below, `who` names the caller or stage in the message.
inline int32_t check_stage_db(const gorse_b200_vecdb *db, int n, const char *who)
{
    if (db->distance == GORSE_B200_DISTANCE_COSINE) {
        set_error("%s: item-to-item, session and user-to-user collections are Dot or Euclidean", who);
        return GORSE_B200_ERR_UNSUPPORTED;
    }
    const bool sparse = db->dim == 0;
    if (n > (sparse ? MAX_N_SPARSE : MAX_N_DENSE)) {
        set_error("%s: n = %d above %d for a %s collection", who, n, sparse ? MAX_N_SPARSE : MAX_N_DENSE, sparse ? "sparse" : "dense");
        return GORSE_B200_ERR_UNSUPPORTED;
    }
    if ((int64_t)db->ts.size() > INT32_MAX) {
        set_error("%s: more than 2^31 slots", who);
        return GORSE_B200_ERR_UNSUPPORTED;
    }
    return GORSE_B200_OK;
}

// off[0, rows] of a CSR named `what`: off[0] == 0 and non-decreasing
inline int32_t check_offsets(const int64_t *off, int64_t rows, const char *who, const char *what)
{
    GB_CHECK_ARG(off[0] == 0, "%s: %s[0] must be 0", who, what);
    for (int64_t r = 0; r < rows; r++) GB_CHECK_ARG(off[r + 1] >= off[r], "%s: %s decreases at %lld", who, what, (long long)r);
    return GORSE_B200_OK;
}

// a feedback CSR of rows rows whose entries are items of [0, n_items)
inline int32_t check_feedback(const char *who, int64_t rows, const int64_t *fb_off, const int32_t *fb_items, int32_t n_items)
{
    GB_CHECK_ARG(rows >= 0 && (rows == 0 || fb_off != nullptr), "%s: fb_off is NULL or n_fb_rows < 0", who);
    if (rows == 0) return GORSE_B200_OK;
    GB_TRY(check_offsets(fb_off, rows, who, "fb_off"));
    GB_CHECK_ARG(fb_off[rows] == 0 || fb_items != nullptr, "%s: fb_items is NULL", who);
    for (int64_t t = 0; t < fb_off[rows]; t++)
        GB_CHECK_ARG(fb_items[t] >= 0 && fb_items[t] < n_items, "%s: feedback entry %lld: item %d is not in [0, %d)", who, (long long)t, fb_items[t],
                     n_items);
    return GORSE_B200_OK;
}

}  // namespace gb
