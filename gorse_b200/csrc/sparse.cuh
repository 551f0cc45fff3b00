// sparse.cuh -- state of the sparse Dot index (sparse.cu), shared with the vector-collection layer (vecdb.cu).
#pragma once
#include <mutex>
#include <vector>

#include "common.cuh"

struct gorse_b200_sparse_index {
    gorse_b200_ctx *ctx = nullptr;
    std::mutex mu;
    // host copy (append-friendly); device mirrors are rebuilt lazily after an add
    std::vector<int64_t> h_off{0};
    std::vector<uint32_t> h_ind;
    std::vector<float> h_val;
    uint32_t n_features = 0;
    bool dirty = true;
    gb::DevBuf<int64_t> off, foff;
    gb::DevBuf<uint32_t> ind;
    gb::DevBuf<float> val, fval;
    gb::DevBuf<int32_t> frow;
    // grow-only work buffers of the tiled search: each (query, tile) work item's best k (tl_*; for k > 128, tl_dot holds the
    // chunk's score rows instead), the chunks' work-item counters (next) and the push / pull work-item counts since the last
    // gorse_b200_sparse_index_stats (paths)
    gb::DevBuf<float> tl_dot;
    gb::DevBuf<int32_t> tl_idx, tl_cnt;
    gb::DevBuf<unsigned long long> next, paths;
    // measurement: events around the last search (folded into search_ms by the next search or the stats call)
    cudaEvent_t ev[2] = {nullptr, nullptr};
    bool ev_pending = false;
    double search_ms = 0.0;
    int64_t tiles = 0;
};


namespace gb {
int32_t sparse_search_host(gorse_b200_sparse_index *ix, int64_t q0, int64_t nq, const int64_t *q_off, const uint32_t *q_ind,
                           const float *q_val, const uint8_t *d_allow, int32_t k, int32_t *idx_out, float *dot_out, int32_t *count_out);
// queries = the stored rows of the DEVICE list d_rows[nq] (each never returned itself), results left on the device in the
// layout of sparse_search_host (d_idx / d_dot [nq x k] padded with -1 / 0, d_cnt[nq]); enqueued on the context's stream.  The
// index holds at least one vector; the caller holds ix->mu and the device.
int32_t sparse_search_rows(gorse_b200_sparse_index *ix, const int64_t *d_rows, int64_t nq, const uint8_t *d_allow, int32_t k, int32_t *d_idx,
                           float *d_dot, int32_t *d_cnt);
// compaction (gorse_b200_vecdb_compact): scan[n + 1] (device) is the exclusive sum of the live flags (row r is live iff
// scan[r + 1] != scan[r] and then becomes row scan[r]), live = scan[n].  Both layouts are compacted on the device, the host
// CSR is replaced by the compacted one and the index ends clean; the search's work buffers are released.  On an error the rows are
// unchanged (the device mirrors may have been brought up to date).  The caller holds ix->mu and the device.
int32_t sparse_compact(gorse_b200_sparse_index *ix, const int64_t *scan, int64_t live);
// device bytes held by the index
size_t sparse_bytes(const gorse_b200_sparse_index *ix);
// the device layouts from the host CSR, as the next search would build them: the CSR is uploaded and the CSC built on the
// device, and the index ends clean (gorse_b200_vecdb_load).  The caller holds ix->mu and the device.
int32_t sparse_sync_device(gorse_b200_sparse_index *ix);

// vectors built on the device by sparse_idf_rows and not yet part of any index: the CSR of the non-empty rows (off on the host,
// m + 1 entries from 0; ind / val on the device), row_off[n + 1] = each input row's first entry (an empty row's equals the next
// row's), n_features = the largest index + 1 (0 without entries)
struct SparseRows {
    std::vector<int64_t> off, row_off;
    DevBuf<uint32_t> ind;
    DevBuf<float> val;
    uint32_t n_features = 0;
};
// appendSparseVector of n rows on the device (gorse_b200_vecdb_add_idf_vectors): part A rows a_off[n + 1] / a_ids over
// a_idf[a_n_idf] at a_offset, then optionally part B (b_off == nullptr: none).  The arguments are checked by the caller except
// what needs the ids: a used NaN idf, an index >= 0x7fffffff or a row whose B indices do not follow its A indices is
// GORSE_B200_ERR_ARG.  Nothing but `out` changes; on an error the caller discards `out`.  The caller holds the device.
int32_t sparse_idf_rows(gorse_b200_ctx *c, int64_t n, const int64_t *a_off, const int32_t *a_ids, const float *a_idf, int32_t a_n_idf,
                        uint32_t a_offset, const int64_t *b_off, const int32_t *b_ids, const float *b_idf, int32_t b_n_idf, uint32_t b_offset,
                        SparseRows &out);
// appends the rows of `rows` to the index as rows n .. n + m - 1: the device CSR grows, the new postings are merged into the CSC
// on the device, the host CSR is brought up to date from the device, and the index ends clean.  On an error the index's rows
// are unchanged (its device layouts may have been brought up to date).  The caller holds ix->mu and the device.
int32_t sparse_append(gorse_b200_sparse_index *ix, const SparseRows &rows);
}
