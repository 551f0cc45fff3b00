// evaluate.cuh -- the ranking, metric and negative-sampling kernels of cf.Evaluate (evaluate.cu), launched for other
// callers through these host functions: gorse_b200_embedding_eval (embedding_eval.cu) ranks and samples with them.
#pragma once
#include "cf.cuh"

#define GB_EVAL_MAX_TOPK 128

namespace gb {

// 1 / math32.Log2(i + 2) for i < topk: the discounts of NDCG (evaluator.go:75-89), what eval_rank_kernel reads
void eval_inv_log2(int32_t topk, float *out);
// eval_rank_kernel on the stream: per user the TopKFilter of its candidates (cand_off / cand_item / score, absolute offsets)
// and NDCG, Precision, Recall against test(u); metrics[4 u + 3] = 1 for a user with a test row, else the row is zeros
void launch_eval_rank(cudaStream_t s, const int64_t *cand_off, const int32_t *cand_item, const float *score, const int64_t *test_off,
                      const int32_t *test_items, int32_t n_users, int32_t topk, const float *inv_log2, float *metrics);
// eval_negatives_kernel on the stream: count_only fills n_neg[u], else neg_items at neg_off[u]; excl rows sorted ascending;
// the draws of user u come from stream base + (u_lo + u)
void launch_eval_negatives(cudaStream_t s, const int64_t *excl_off, const int32_t *excl_items, const int64_t *test_off,
                           const int32_t *test_items, int32_t n_users, int32_t u_lo, int32_t n_items, int32_t n_cand, uint64_t base,
                           bool count_only, int32_t *n_neg, const int64_t *neg_off, int32_t *neg_items);
// the stream base of gorse_b200_eval_create's sampler for `seed`
inline uint64_t eval_negatives_base(uint64_t seed) { return mix64(seed ^ 0xbb67ae8584caa73bull); }

}  // namespace gb
