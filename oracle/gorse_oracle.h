/*
 * gorse_oracle.h -- CPU ORACLE for the gorse CF hot path.  TEST INFRASTRUCTURE ONLY.
 *
 * This is a plain-C restatement of the reference's algorithms (gorse-io/gorse @ 5404aefa)
 * used as the checker for the CUDA path.  Only tests/, __graft_entry__.smoke() and
 * bench.py's cpu_baseline / --impl reference legs may link or call it.  The product
 * (libgorse_b200.so) never does, and has no CPU fallback.
 *
 * Every function cites the reference file:line it follows.  Parity status:
 *   - floats kernels: PINNED (floats_test.go known answers + bit-equality against the reference's
 *     own C kernels compiled into oracle/_ref, golden vectors in tests/golden/floats_golden.json)
 *   - go heap / TopKFilter / PriorityQueue: PINNED by common/heap/*_test.go known answers
 *     (tie order: parity unpinned -- the reference has no tie tests; we restate container/heap)
 *   - metrics: PINNED by model/cf/evaluator_test.go known answers
 *   - BPR step / ALS epoch / Bruteforce: restated from model/cf/model.go and common/ann/bruteforce.go;
 *     the Go code cannot run here (no Go toolchain) -> anchored on the pinned primitives above and on
 *     the reference's call sites.  math32.Exp (chewxy/math32 v1.11.1, absent from the reference) is
 *     restated from its published algorithm: PARITY UNPINNED for Exp (<= 1-2 ulp expected).
 *   - RNG streams (Go math/rand): PARITY UNPINNED and unreproducible (SURVEY F9); samplers here are
 *     our own counter-based design shared bit-for-bit with the CUDA path.
 */
#ifndef GORSE_ORACLE_H
#define GORSE_ORACLE_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- common/floats (AVX-512 dispatch order, common/floats/src/floats_avx512.c) ---- */
float gbo_dot(const float *a, const float *b, int64_t n);             /* :306-367 */
float gbo_euclidean(const float *a, const float *b, int64_t n);       /* :374-441 */
void gbo_mul_const_to(const float *a, float c, float *dst, int64_t n);  /* :82-109 */
void gbo_mul_const_add(const float *a, float c, float *dst, int64_t n); /* :51-80 */
void gbo_mul_const_add_to(const float *a, float b, const float *c, float *dst, int64_t n); /* :18-49 */
void gbo_mul_const(float *a, float c, int64_t n);                       /* :111-136 */
void gbo_sub_to(const float *a, const float *b, float *c, int64_t n);   /* :165-194 */
/* scalar Go definitions, common/floats/floats.go:21-33 */
float gbo_dot_scalar(const float *a, const float *b, int64_t n);
float gbo_euclidean_scalar(const float *a, const float *b, int64_t n);

/* ---- chewxy/math32 restatements ---- */
float gbo_exp(float x);
float gbo_log2(float x);

/* ---- common/heap ---- */
typedef struct { int32_t value; float weight; } gbo_elem;
/* TopKFilter (filter.go:23-59): push all (value, weight) in order, return values in decreasing
 * weight order.  Returns number written (<= k). */
int32_t gbo_topk_filter(const int32_t *values, const float *weights, int64_t n, int32_t k,
                        int32_t *out_values, float *out_weights);
/* PriorityQueue known-answer helper (pq.go): push all, then pop all. desc as in NewPriorityQueue. */
int32_t gbo_pq_push_pop_all(const int32_t *values, const float *weights, int64_t n, int32_t desc,
                            int32_t reverse_first, int32_t *out_values, float *out_weights);

/* ---- model/cf BPR (model.go:408-540) ---- */
/* one SGD step, model.go:469-488.  P is U x d row-major, Q is I x d row-major. */
void gbo_bpr_step(float *P, float *Q, int32_t d, int32_t u, int32_t i, int32_t j, float lr, float reg);
/* sequential application of n triples (= the reference with Jobs=1 given this triple stream) */
void gbo_bpr_apply_triples(float *P, float *Q, int32_t d, const int32_t *uij, int64_t n, float lr, float reg);
/* our counter-based sampler (distributionally identical to model.go:449-468; see DESIGN.md).
 * user rows must be sorted ascending.  active_users = users with >=1 feedback, ascending. */
void gbo_bpr_sample_triples(int32_t n_items, const int64_t *user_off, const int32_t *user_items,
                            const int32_t *active_users, int32_t n_active,
                            uint64_t seed, int64_t first_step, int64_t n, int32_t *uij_out);
/* multi-threaded Hogwild epoch used as the CPU baseline (not a parity target): returns seconds */
/* dataset.SampleUserNegatives, dataset/dataset.go:242-253 + common/util/random.go:108-132 (our counter RNG) */
void gbo_sample_user_negatives(int32_t n_items, int32_t n_users, int32_t u_base, const int64_t *train_off, const int32_t *train_items,
                               const int64_t *test_off, const int32_t *test_items, int32_t n_cand, uint64_t seed,
                               int64_t *neg_off_out, int32_t *neg_items_out);
/* CPU-arm hygiene: N(0, std) fill, first-touched page-interleaved by pinned workers */
void gbo_fill_normal_interleaved(float *buf, int64_t n, float std, uint64_t seed, int32_t n_threads);
double gbo_bpr_epoch_threads(float *P, float *Q, int32_t n_items, int32_t d,
                             const int64_t *user_off, const int32_t *user_items,
                             const int32_t *active_users, int32_t n_active,
                             uint64_t seed, int64_t n_steps, float lr, float reg, int32_t n_threads,
                             int32_t use_ref_kernels);

/* ---- model/cf ALS (eALS, "CCD") model.go:609-775, one epoch, Jobs-independent ---- */
void gbo_als_epoch(float *P, float *Q, int32_t n_users, int32_t n_items, int32_t d,
                   const int64_t *user_off, const int32_t *user_items,
                   const int64_t *item_off, const int32_t *item_users, float reg, float alpha);
double gbo_als_epoch_threads(float *P, float *Q, int32_t n_users, int32_t n_items, int32_t d,
                   const int64_t *user_off, const int32_t *user_items,
                   const int64_t *item_off, const int32_t *item_users, float reg, float alpha,
                   int32_t n_threads);

/* ---- common/ann Bruteforce (bruteforce.go:39-83) ---- */
enum { GBO_METRIC_EUCLIDEAN = 0, GBO_METRIC_NEG_DOT = 1 };
/* returns count written (<= k).  self = -1 for SearchVector, else SearchIndex(q=self). */
int32_t gbo_bruteforce_search(const float *X, int64_t N, int32_t d, const float *q, int64_t self,
                              int32_t k, int32_t prune0, int32_t metric,
                              int32_t *out_idx, float *out_score);
/* all-pairs SearchIndex over queries [q0, q1) with n_threads; out rows padded with idx=-1 */
double gbo_bruteforce_all(const float *X, int64_t N, int32_t d, int64_t q0, int64_t q1, int32_t k,
                          int32_t prune0, int32_t metric, int32_t n_threads,
                          int32_t *out_idx, float *out_score, int32_t *out_count);

/* ---- model/cf/evaluator.go ---- */
/* test helper: data part of the eALS objective (see tests/als_checks.py) */
double gbo_als_observed_loss(const float *P, const float *Q, int32_t n_users, int32_t d, const int64_t *user_off,
                             const int32_t *user_items, double w, int32_t n_threads);
/* logics: similarity vectors and scores (item_to_item.go, user_to_user.go, vector_writer.go) */
void gbo_bf16_truncate(const float *in, int64_t n, float *out);                                    /* bfloats.go:23-37 */
int32_t gbo_sparse_vector(const int32_t *ids, int32_t n_ids, const float *idf, int32_t n_idf, uint32_t offset,
                          uint32_t *indices_out, float *values_out);                               /* vector_writer.go:200-209 */
int32_t gbo_similar_scores(int32_t euclidean, double score_scale, int32_t self_id, int32_t n,
                           const int32_t *nbr_ids, const float *nbr_score, int32_t n_nbr,
                           int32_t *ids_out, double *scores_out);                                  /* item_to_item.go:63-85 */

/* sparse Dot search (xvec flat sparse index, storage/vectors/xvec.go:244-248): parity unpinned beyond id orders */
float gbo_sparse_dot(const uint32_t *ia, const float *va, int32_t na, const uint32_t *ib, const float *vb, int32_t nb);
int32_t gbo_sparse_bruteforce_search(const int64_t *off, const uint32_t *indices, const float *values, int64_t N,
                                     const uint32_t *q_ind, const float *q_val, int32_t q_n, int64_t self, int32_t k,
                                     int32_t *out_idx, float *out_dot);

float gbo_ndcg(const int32_t *target, int32_t n_target, const int32_t *rank, int32_t n_rank);      /* :75-89 */
float gbo_precision(const int32_t *target, int32_t n_target, const int32_t *rank, int32_t n_rank); /* :94-102 */
float gbo_recall(const int32_t *target, int32_t n_target, const int32_t *rank, int32_t n_rank);    /* :108-116 */
float gbo_hr(const int32_t *target, int32_t n_target, const int32_t *rank, int32_t n_rank);        /* :119-126 */
float gbo_map(const int32_t *target, int32_t n_target, const int32_t *rank, int32_t n_rank);       /* :130-140 */
float gbo_mrr(const int32_t *target, int32_t n_target, const int32_t *rank, int32_t n_rank);       /* :154-161 */
/* Evaluate (evaluator.go:35-72) with Jobs=1: out = {NDCG, Precision, Recall} @topk.
 * negatives are passed in (the reference samples them with Go math/rand, unpinned). */
void gbo_evaluate(const float *P, const float *Q, int32_t n_users, int32_t d,
                  const int64_t *test_off, const int32_t *test_items,
                  const int64_t *neg_off, const int32_t *neg_items, int32_t topk, float out[3]);

/* optional: bind the reference's own compiled kernels (oracle/_ref/libfloats_ref.so) */
int32_t gbo_ref_bind(const char *path);

#ifdef __cplusplus
}
#endif
#endif
