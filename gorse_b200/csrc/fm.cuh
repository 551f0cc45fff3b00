// fm.cuh -- the FM ranker's model handle and the device body of gorse_b200_fm_rank (fm.cu), taking device pointers, so that
// the batched FM ranking and the batched offline recommendation (recommend.cu) launch the same kernels.
#pragma once
#include <algorithm>

#include "recall.cuh"

namespace gb {
namespace fm {

constexpr int MAX_FACTORS = 32;     // one factor per lane of a warp
constexpr int MAX_EMB_DIM = 1024;   // fm_attn_kernel keeps one row of Mul(softmax, e) per warp in shared memory
constexpr int MAX_SLOTS = 8;
constexpr int ATTN_WARPS = 8;
constexpr int SORT_THREADS = 256;
constexpr int SORT_SMEM = 2048;     // users with more candidates sort in a global-memory buffer
constexpr int64_t GROUP_PAIRS = int64_t(1) << 22;   // pairs per device pass (bounds the vx / row-sum buffers)

struct Model {
    const float *V, *W;
    float bias;
    int k;
};

struct Feats {                // id feature + labels CSR, per user or per item-table row
    const int32_t *feat;      // [rows] or -1
    const int64_t *off;       // [rows + 1]
    const int32_t *idx;
    const float *val;
};

struct Slot {
    const float *H, *AW, *Ab, *EW, *Eb;
    const uint16_t *emb;      // [n_items x dim] bf16 bits
    const uint8_t *mask;      // [n_items x n_emb] or NULL (every embedding present)
    int n_emb, s, dim;
    float *z, *zmax;          // [n_items x dim], [n_items]
};

}  // namespace fm
}  // namespace gb

struct gorse_b200_fm {
    gorse_b200_ctx *ctx = nullptr;
    int64_t n_features = 0;
    int32_t k = 0, num_dimension = 0, batch_size = 0, n_emb = 0;
    std::vector<int32_t> dim;
    std::vector<size_t> slot_off;        // per slot: offset of H in params (AW, Ab, EW, Eb follow)
    float bias = 0.0f;
    gb::DevBuf<float> params;
    std::mutex mu;
    // per-call buffers, grow-only
    gb::DevBuf<int32_t> u_feat, u_idx, i_feat, i_idx, cand, dims, ch_rows, order, sort_val;
    gb::DevBuf<int64_t> u_off, i_off, c_off, ch_start;
    gb::DevBuf<float> u_val, i_val, score, vx, rowsum;
    gb::DevBuf<uint16_t> emb[gb::fm::MAX_SLOTS];
    gb::DevBuf<float> z[gb::fm::MAX_SLOTS], zmax[gb::fm::MAX_SLOTS];
    gb::DevBuf<uint8_t> mask;
    gb::DevBuf<uint64_t> sort_key;
};

namespace gb {
namespace fm {

// the row of V / W an index selects once it has travelled as float32; false when it leaves the table (Go panics there)
inline bool feature_ok(int64_t idx, int64_t n_features)
{
    if (idx < 0 || idx >= n_features) return false;
    return (int64_t)(float)idx < n_features;
}

// a features CSR (id feature + labels) of `rows` rows, checked on the host; `what` ("user", "item") names it
inline int32_t check_feats(const char *what, int64_t rows, const int32_t *feat, const int64_t *off, const int32_t *idx, const float *val,
                           int64_t n_features)
{
    GB_CHECK_ARG(rows == 0 || (feat != nullptr && off != nullptr), "%s: NULL id features or label offsets", what);
    if (rows == 0) return GORSE_B200_OK;
    GB_CHECK_ARG(off[0] == 0, "%s: label offsets must start at 0", what);
    for (int64_t r = 0; r < rows; r++) {
        GB_CHECK_ARG(off[r + 1] >= off[r], "%s %lld: label offsets decrease", what, (long long)r);
        GB_CHECK_ARG(feat[r] == -1 || feature_ok(feat[r], n_features), "%s %lld: id feature %d is not -1 or a feature of [0, %lld)", what,
                     (long long)r, feat[r], (long long)n_features);
    }
    GB_CHECK_ARG(off[rows] == 0 || (idx != nullptr && val != nullptr), "%s: NULL label indices / values", what);
    for (int64_t j = 0; j < off[rows]; j++)
        GB_CHECK_ARG(feature_ok(idx[j], n_features), "%s label entry %lld: feature %d is not in [0, %lld) once rounded to float32", what,
                     (long long)j, idx[j], (long long)n_features);
    return GORSE_B200_OK;
}

// the model's parameters as the kernels read them
Model model(const gorse_b200_fm *m);

// per slot: the slot's parameters and the item table m->emb[s] / m->mask (uploaded by the caller; mask used when `masked`)
// in S[s], and fm_item_kernel over the n_items rows into m->z[s] / m->zmax[s] (grown here).  The caller holds m->mu.
int32_t item_tables(gorse_b200_fm *m, int64_t n_items, bool masked, Slot *S);

// the users' and the item table's feature CSRs into m->u_* / m->i_*, and with slots the item embeddings (and the mask, when
// given) and their tables in S (item_tables).  The caller holds m->mu.
int32_t upload_feats(gorse_b200_fm *m, int64_t n_users, const int32_t *user_feat, const int64_t *user_lab_off, const int32_t *user_lab_idx,
                     const float *user_lab_val, int64_t n_items, const int32_t *item_feat, const int64_t *item_lab_off, const int32_t *item_lab_idx,
                     const float *item_lab_val, const uint16_t *const *item_emb, const uint8_t *item_emb_mask, Slot *S);

// one device pass over users [u0, u1) of the device candidate CSR c_off / cand (dims[u] = D_u): fm_pair_kernel, fm_attn_kernel
// per slot over the attention chunks [ch0, ch1) of ch_start / ch_rows, and fm_sort_kernel.  Pair p's vx / row sum sit at
// p - pair_base in m->vx / m->rowsum (grown by the caller to the pass's pairs when there are slots); scores / order in
// score / order at the pair's position.  max_n: the most candidates of one user of the pass.  *global_sort: whether the pass
// sorted in global memory.  The caller holds m->mu.
int32_t rank_pass(gorse_b200_fm *m, const Feats &U, const Feats &I, const int64_t *c_off, const int32_t *cand, const int32_t *dims, int64_t u0,
                  int64_t u1, int64_t pair_base, const Slot *S, const int64_t *ch_start, const int32_t *ch_rows, int64_t ch0, int64_t ch1,
                  int64_t max_n, float *score, int32_t *order, bool *global_sort);

}  // namespace fm
}  // namespace gb
