// stages.cuh -- the device bodies of the batched item-to-item and user-to-user recommenders (item_to_item.cu,
// user_to_user.cu), taking device pointers, so that gorse_b200_vecdb_item_to_item / _user_to_user and the batched offline
// recommendation (recommend.cu) launch the same kernels.
#pragma once
#include <algorithm>

#include "aggregate.cuh"
#include "vecdb.cuh"

namespace gb {

// stage A of both recommenders: the first n neighbours of each of the R stored vectors d_nb[R] (device) of db, as a table of
// n (int32 slot, float32 score) entries per row, Dot collections keeping scores > 0 only (dense: the index's top-k pipeline;
// sparse: sparse_search_rows).  The caller holds db->mu and has filled db->d_allow.  *exact_rows: rows of the exact scan.
int32_t neighbour_table(gorse_b200_vecdb *db, int64_t R, const int64_t *d_nb, int n, int32_t *t_slot, float *t_score, int32_t *t_cnt,
                        int64_t *exact_rows);

namespace i2i {
constexpr int MAX_N_DENSE = 1024;                // the sort buffer holds n entries
constexpr int MAX_N_SPARSE = 128;                // sparse_search_kernel's k

struct Users {                // one chunk of users (chunk-local ids)
    const int64_t *c_off;     // [users + 1] into c_row
    const int32_t *c_row;     // the neighbour-table row of each live context entry, in the caller's order
    const int64_t *ex_off;    // [users + 1] into ex
    const int64_t *ex;        // each user's excluded slots, ascending (-1 entries dropped; may be padded with INT64_MAX)
    int64_t *slots;           // [users x n]
    double *scores;           // [users x n]
    int32_t *count;           // [users]
};

struct Table {                // stage A: the first n neighbours of each distinct context item
    const int32_t *slot;      // [rows x n]
    const float *score;       // [rows x n] the vector store's score (dot, or the negated distance)
    const int32_t *cnt;       // [rows]
};

// global accumulator rows (one [N] float64 row, flag row and slot list per CTA, at most 512 MB): how many CTAs
inline int heavy_grid(const gorse_b200_ctx *c, int64_t N)
{
    return (int)std::max<int64_t>(1, std::min<int64_t>((int64_t)c->sm_count * 2, (512ll << 20) / (13 * N)));
}
// stage B for one chunk: d_users[0, fill) aggregate in shared memory, d_users[fill, fill + heavy) in the global rows acc /
// seen (zeroed) / touched of heavy_grid(c, N) CTAs
int32_t aggregate(gorse_b200_ctx *c, const int32_t *d_users, int64_t fill, int64_t heavy, const Users &U, const Table &T, int n, double scale,
                  bool euclid, int64_t N, double *acc, uint8_t *seen, int32_t *touched);
}  // namespace i2i

namespace u2u {
constexpr int MAX_N_DENSE = 1024;
constexpr int MAX_N_SPARSE = 128;

struct Table {                // stage A: the first n neighbours of each distinct query user
    const int32_t *slot;      // [rows x n]
    const float *score;       // [rows x n] the vector store's score (dot, or the negated distance)
    const int32_t *cnt;       // [rows]
};

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

inline int heavy_grid(const gorse_b200_ctx *c, int64_t NI)
{
    return (int)std::max<int64_t>(1, std::min<int64_t>((int64_t)c->sm_count * 2, (512ll << 20) / (16 * NI)));
}
// routing and stage B for one chunk of R.users users; heavy: some user may need a global row (acc / flag zeroed, touched,
// heavy_grid(c, NI) CTAs)
int32_t aggregate(gorse_b200_ctx *c, const Route &R, const Users &U, const Table &T, const Feedback &F, int n, double scale, bool euclid,
                  int64_t NI, bool heavy, double *acc, int32_t *flag, int32_t *touched);
}  // namespace u2u

}  // namespace gb
