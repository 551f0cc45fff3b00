// topk.cuh -- brute-force index state shared by topk.cu (exact scan / re-rank) and topk_mma.cu (tensor-core stage 1).
#pragma once
#include <cuda_bf16.h>

#include "common.cuh"

struct gorse_b200_index {
    gorse_b200_ctx *ctx = nullptr;
    int32_t d = 0, metric = 0;
    int64_t n = 0, cap = 0;
    gb::DevBuf<float> X;            // [cap x d] fp32, row-major: the vectors as added (exact re-rank reads these)
    gb::DevBuf<__nv_bfloat16> Xb;   // [n_pad x d] bf16 mirror feeding the tensor cores (built lazily)
    gb::DevBuf<float> norm;         // per-vector fp32 norms (+ max at [n]), built lazily
    gb::DevBuf<int32_t> perm;       // mirror row p holds vector perm[p] (random: the first columns are a uniform sample)
    float max_norm = 0.f;
    bool mma_ready = false;
    float *dbg_scores = nullptr;    // tests only: dense stage-1 scores
    int64_t last_fallback_rows = 0; // rows of the last searches that needed the exact scan
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;  // CUDA events around the stage-1 kernel (bench.py roofline)
    double stage1_ms = 0.0, stage1_flop = 0.0; // accumulated since the last debug read
    // reusable work buffers of the tensor path (sized for w_cq query rows at mirror width w_kp)
    int64_t w_cq = 0;
    int w_kp = 0;
    gb::DevBuf<__nv_bfloat16> w_qb;
    gb::DevBuf<float> w_eps, w_cval, w_theta;
    gb::DevBuf<int32_t> w_ccol, w_ccnt, w_ids, w_idcnt, w_flag, w_flist;
    // result staging of search_common (grow-only: a 120 MB cudaMalloc + cudaFree per all-pairs call otherwise)
    gb::DevBuf<int32_t> r_idx, r_count;
    gb::DevBuf<float> r_dist;
    std::mutex mu;
};

namespace gb {

// exact scan / re-rank.  row_list != nullptr: only those query rows (nq = length of the list) are processed
int32_t launch_exact(gorse_b200_index *ix, const float *d_q, const int64_t *d_qidx, int64_t q0, int64_t nq, int k,
                     const int32_t *d_cand, const int32_t *d_cand_count, int cand_stride, const int32_t *row_list,
                     int32_t *d_idx, float *d_dist, int32_t *d_count, int prune0, int *d_nan);

int32_t launch_exact_split(gorse_b200_index *ix, const float *d_q, const int64_t *d_qidx, int64_t q0, int32_t n_rows, int k,
                           const int32_t *row_list, int32_t *d_idx, float *d_dist, int32_t *d_count, int prune0, int *d_nan,
                           const uint8_t *allow = nullptr);

int32_t index_reserve(gorse_b200_index *ix, int64_t need);
bool mma_path_eligible(const gorse_b200_index *ix, int64_t nq, int k);
// h_*: optional host result buffers; when given, every finished chunk of queries is downloaded on the context's copy stream
// while the next chunk's kernels run
int32_t search_mma(gorse_b200_index *ix, const float *d_q, const int64_t *d_qidx, int64_t q0, int64_t nq, int k, int prune0,
                   int32_t *d_idx, float *d_dist, int32_t *d_count, int *d_nan, int32_t *h_idx = nullptr, float *h_dist = nullptr,
                   int32_t *h_count = nullptr);

}  // namespace gb
