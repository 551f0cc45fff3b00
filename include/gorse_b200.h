/*
 * gorse_b200.h -- C ABI of libgorse_b200.so: the H100 (sm_90a) implementation of Gorse's
 * collaborative-filtering training and brute-force top-k hot path.
 *
 * This is exactly what the reference-side cgo shim binds (go/ in this repo, INTEGRATION.md):
 * plain pointers and sizes, no C++/torch types.  Every entry point names the reference
 * interface it replaces (paths into gorse-io/gorse @ 5404aefa).
 *
 * Conventions
 *   - all pointers are HOST pointers owned by the caller; the library copies during the call and
 *     never retains them (cgo rule; reference precedent common/blas/blas_openblas.go:24-25)
 *   - matrices are row-major contiguous fp32; ids are int32; CSR offsets are int64 (len rows+1)
 *   - every function returns 0 on success, a negative gorse_b200_status otherwise;
 *     gorse_b200_last_error() gives the message for the calling thread.  Nothing throws or aborts
 *     across the boundary.
 *   - there is no CPU fallback: without a CUDA device every call except
 *     gorse_b200_version/_last_error fails with GORSE_B200_ERR_CUDA.
 *   - one context = one GPU (+ optionally one rank of an NCCL communicator).  Objects created from
 *     a context run on its stream; calls on the same object are serialised by the caller
 *     (cf.Fit runs on one goroutine, master/master.go:457-484) except gorse_b200_index_search*,
 *     which is thread-safe (ann.Index may be searched concurrently, common/ann/ann_test.go:200-213).
 */
#ifndef GORSE_B200_H
#define GORSE_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GORSE_B200_ABI_VERSION 1

typedef enum {
    GORSE_B200_OK = 0,
    GORSE_B200_ERR_ARG = -1,      /* bad argument (null, negative size, out-of-range id ...) */
    GORSE_B200_ERR_CUDA = -2,     /* CUDA runtime/driver error, or no device */
    GORSE_B200_ERR_NCCL = -3,     /* NCCL error */
    GORSE_B200_ERR_OOM = -4,      /* device or host allocation failed */
    GORSE_B200_ERR_RANGE = -5,    /* index out of range (ann.Bruteforce.SearchIndex error, bruteforce.go:41-43) */
    GORSE_B200_ERR_STATE = -6,    /* call not valid in the object's current state */
    GORSE_B200_ERR_UNSUPPORTED = -7
} gorse_b200_status;

typedef struct gorse_b200_ctx gorse_b200_ctx;     /* one GPU, one stream, optional NCCL rank */
typedef struct gorse_b200_cf gorse_b200_cf;       /* factor tables + feedback CSR resident in HBM */
typedef struct gorse_b200_index gorse_b200_index; /* brute-force vector index resident in HBM */

int32_t gorse_b200_version(void);
const char *gorse_b200_last_error(void); /* thread-local, never NULL */

/* ------------------------------------------------------------------------------------------
 * Context.  Replaces: common/parallel.Parallel (common/parallel/parallel.go:33-94), the
 * reference's data-parallel scheduler for Fit -- a kernel launch on the context's stream.
 * ---------------------------------------------------------------------------------------- */
int32_t gorse_b200_device_count(int32_t *count);
int32_t gorse_b200_ctx_create(int32_t device, gorse_b200_ctx **out);
/* multi-GPU: one context per GPU, rank in [0, world).  nccl_id = GORSE_B200_NCCL_ID_BYTES bytes
 * produced by gorse_b200_nccl_unique_id() on rank 0 and carried to the other ranks by the host
 * (gRPC between Gorse nodes, torch.distributed in bench.py).  Collective: all ranks must call. */
#define GORSE_B200_NCCL_ID_BYTES 128
int32_t gorse_b200_nccl_unique_id(void *id_out);
int32_t gorse_b200_ctx_create_dist(int32_t device, int32_t rank, int32_t world, const void *nccl_id,
                                   gorse_b200_ctx **out);
int32_t gorse_b200_ctx_destroy(gorse_b200_ctx *ctx);
int32_t gorse_b200_ctx_sync(gorse_b200_ctx *ctx);
int32_t gorse_b200_ctx_rank(const gorse_b200_ctx *ctx, int32_t *rank, int32_t *world);
/* measurement hooks (bench.py): CUDA events on the context's own stream, and the number of this
 * library's kernels launched on it so far */
int32_t gorse_b200_ctx_timer_begin(gorse_b200_ctx *ctx);
int32_t gorse_b200_ctx_timer_end(gorse_b200_ctx *ctx, float *ms_out); /* records, syncs, returns elapsed */
int32_t gorse_b200_ctx_launch_count(const gorse_b200_ctx *ctx, int64_t *count);
int32_t gorse_b200_ctx_flush_l2(gorse_b200_ctx *ctx); /* writes a buffer larger than L2 */
int32_t gorse_b200_ctx_barrier(gorse_b200_ctx *ctx);  /* NCCL barrier across ranks (no-op for world 1) */
/* page-locked host memory for the shim's flat factor mirror (SURVEY 8b "ownership"): factor uploads and
 * downloads from it run at full PCIe rate.  Plain host pointers work everywhere too, just slower. */
int32_t gorse_b200_host_alloc(size_t bytes, void **out);
int32_t gorse_b200_host_free(void *p);

/* ------------------------------------------------------------------------------------------
 * CF model state.  Replaces cf.BaseMatrixFactorization's UserFactor/ItemFactor ([][]float32,
 * model/cf/model.go:118-127) and the dataset.CFSplit accessors GetUserFeedback/GetItemFeedback
 * (dataset/dataset.go:40-60) flattened to CSR by the shim.
 *
 * user_off[rows+1], user_items : R_u  (any order inside a row, duplicates allowed; the device copy is sorted
 *     per row for the negative-sampling membership test)
 * item_off[rows+1], item_users : R_i  (may be NULL when ALS is not used)
 * Offsets need not start at 0: user_items / item_users point at the entry user_off[0] / item_off[0] refers to, so a
 * slice of a larger CSR can be passed without rebasing.
 *
 * One GPU (world = 1): rows = all n_users / n_items.
 * Distributed context (SURVEY 8e): n_users / n_items stay GLOBAL, but every rank passes ONLY ITS OWN ROWS --
 * users [n_users*r/W, n_users*(r+1)/W) and items [n_items*r/W, n_items*(r+1)/W) -- so host work, upload and HBM
 * per rank are 1/W of the job (BASELINE configs[4]: 10 M users x 200 M feedback over 8 GPUs).  Rank r owns those rows
 * of P; Q is replicated.  Collective: all ranks must call (the global feedback count is all-reduced, and a rank whose
 * arguments fail validation makes every rank fail instead of hanging the others).
 * ---------------------------------------------------------------------------------------- */
int32_t gorse_b200_cf_create(gorse_b200_ctx *ctx, int32_t n_users, int32_t n_items, int32_t n_factors,
                             const int64_t *user_off, const int32_t *user_items,
                             const int64_t *item_off, const int32_t *item_users,
                             gorse_b200_cf **out);
int32_t gorse_b200_cf_destroy(gorse_b200_cf *cf);
/* warm start / parity mode: upload full tables (P: n_users x d, Q: n_items x d) */
int32_t gorse_b200_cf_set_factors(gorse_b200_cf *cf, const float *P, const float *Q);
/* BPR.Init / ALS.Init (model/cf/model.go:532-540, 598-606 -> util.NormalMatrix,
 * common/util/random.go:54-60): i.i.d. N(mean, std) rows, users then items.  The Go math/rand
 * stream is not reproducible (SURVEY F9); the distribution is. */
int32_t gorse_b200_cf_init_normal(gorse_b200_cf *cf, float mean, float stddev, uint64_t seed);
/* host mirror fill: GetUserFactor/GetItemFactor reads (master/tasks.go:946,969) are served from it */
int32_t gorse_b200_cf_get_factors(gorse_b200_cf *cf, float *P, float *Q);
/* Predict / internalPredict (model/cf/model.go:182-203) for a batch of (user, item) index pairs;
 * floats.Dot summation order (AVX-512 tree), bit-equal to the host mirror */
int32_t gorse_b200_cf_predict(gorse_b200_cf *cf, const int32_t *users, const int32_t *items, int64_t n,
                              float *out);

/* ------------------------------------------------------------------------------------------
 * BPR.  Replaces the body of BPR.Fit's epoch loop, model/cf/model.go:448-490.
 * ---------------------------------------------------------------------------------------- */
typedef enum {
    /* racy read-modify-write exactly like the reference's lock-free goroutines: new row =
     * fma(t, lr, row as read by this step).  Bit-exact vs the oracle when the triples of one launch
     * touch disjoint rows. */
    GORSE_B200_SCATTER_STORE = 0,
    /* vectorised atomics (red.global.add.v4.f32): no update is ever lost; gorse_b200_bpr_epoch runs in rounds whose
       triples read the rows as the previous round left them, so an epoch gives the same factors every run up to rounding */
    GORSE_B200_SCATTER_ATOMIC = 1
} gorse_b200_scatter;

typedef enum {
    GORSE_B200_ORDER_HOGWILD = 0,   /* all triples in one launch, like Jobs = many */
    /* the host splits the list into conflict-free waves and launches them in order: identical to the
     * reference with Jobs = 1 on this triple stream (bit-exact with SCATTER_STORE) */
    GORSE_B200_ORDER_SEQUENTIAL = 1
} gorse_b200_order;

/* apply an explicit list of n (u, i, j) triples (uij[3n]); a triple with j < 0 is skipped */
int32_t gorse_b200_bpr_apply_triples(gorse_b200_cf *cf, const int32_t *uij, int64_t n, float lr, float reg,
                                     int32_t scatter, int32_t order);
/* the triples gorse_b200_bpr_epoch(seed) samples for steps [first_step, first_step + n):
 * u uniform over users with feedback, i uniform in R_u, j uniform over items rejected while in R_u
 * (model/cf/model.go:449-468).  A user whose row covers every item yields j = -1. */
int32_t gorse_b200_bpr_sample_triples(gorse_b200_cf *cf, uint64_t seed, int64_t first_step, int64_t n,
                                      int32_t *uij_out);
/* one epoch = n_steps fused sample-gather-dot-sigmoid-scatter steps (n_steps = trainSet.CountFeedback(),
 * model/cf/model.go:448).  SCATTER_STORE: one free-running kernel launch.  SCATTER_ATOMIC: rounds of 8192 steps at
 * every d, in one cooperative launch at d = 16, 32, 64, 128 and two launches per round (deltas, then additions) at
 * any other d; the first ATOMIC epoch at such a d allocates a 3 * 8192 * d float buffer that lives as long as cf.
 * In a distributed context each rank runs n_steps/world steps on its user shard, then item-factor deltas are
 * all-reduced. */
int32_t gorse_b200_bpr_epoch(gorse_b200_cf *cf, float lr, float reg, int64_t n_steps, uint64_t seed,
                             int32_t scatter);

/* ------------------------------------------------------------------------------------------
 * ALS / eALS ("CCD").  Replaces one iteration of ALS.Fit's epoch loop, model/cf/model.go:641-738
 * (Gram S^q, user rows, Gram S^p, item rows).  Needs item_off/item_users at create time.
 * ---------------------------------------------------------------------------------------- */
int32_t gorse_b200_als_epoch(gorse_b200_cf *cf, float reg, float alpha);

/* ------------------------------------------------------------------------------------------
 * Evaluate.  Replaces cf.Evaluate (model/cf/evaluator.go:35-72) with scorers NDCG, Precision,
 * Recall at topk.  test CSR: test positives per user; neg CSR: sampled negatives per user
 * (dataset.SampleUserNegatives, dataset/dataset.go:242-256 -- sampled by the caller).
 * out[3] = {NDCG, Precision, Recall}.
 * Distributed context: every rank passes the rows of ITS users (as in gorse_b200_cf_create); the per-user metrics are
 * summed per rank and all-reduced, so every rank returns the global score (the reference with Jobs = W workers).
 * Collective.
 * ---------------------------------------------------------------------------------------- */
int32_t gorse_b200_cf_evaluate(gorse_b200_cf *cf, const int64_t *test_off, const int32_t *test_items,
                               const int64_t *neg_off, const int32_t *neg_items, int32_t topk,
                               float *out);
/* The same in three steps, so that Fit's repeated evaluations (every Verbose epochs, model/cf/model.go:496-507) upload
 * their inputs once: gorse_b200_eval_create puts the test rows and the negatives in HBM, gorse_b200_eval_run scores
 * the model's CURRENT factors.  With neg_off == NULL the negatives are sampled on the device the way
 * testSet.SampleUserNegatives(trainSet, n_candidates) does (dataset/dataset.go:242-253 -> util.SampleInt32,
 * common/util/random.go:108-132: n_candidates distinct items outside train(u) and test(u); all remaining items, ascending,
 * when fewer are left) -- the reference caches them per dataset (:243), the plan per Fit.  The Go math/rand stream is not
 * reproducible (SURVEY F9): draws come from the library's counter RNG under `seed`.  gorse_b200_eval_negatives returns
 * what was sampled: neg_off_out[rows+1]; neg_items_out may be NULL to learn the size (neg_off_out[rows]) first. */
typedef struct gorse_b200_eval gorse_b200_eval;
int32_t gorse_b200_eval_create(gorse_b200_cf *cf, const int64_t *test_off, const int32_t *test_items,
                               const int64_t *neg_off, const int32_t *neg_items, int32_t n_candidates, uint64_t seed,
                               int32_t topk, gorse_b200_eval **out);
int32_t gorse_b200_eval_run(gorse_b200_eval *ev, float *out);
int32_t gorse_b200_eval_negatives(gorse_b200_eval *ev, int64_t *neg_off_out, int32_t *neg_items_out);
int32_t gorse_b200_eval_destroy(gorse_b200_eval *ev);

/* ------------------------------------------------------------------------------------------
 * Whole Fit.  Replaces cf.BPR.Fit / cf.ALS.Fit (model/cf/model.go:408-530, 609-775): Init, Evaluate at
 * epoch 0, the epoch loop, Evaluate every `verbose` epochs and after the last one, early stopping when the
 * best NDCG is older than `patience` epochs (:508-517).  The shim may call this once per Fit, or keep the
 * loop in Go and call the per-epoch entry points.  Hyper-parameters are model.Params
 * (model/params.go) + cf.FitConfig (model/cf/model.go:50-65); FitConfig.Jobs has no equivalent.
 * The factor tables of `cf` are created with n_factors = params->n_factors by the caller.
 * neg_off / neg_items may be NULL: the negatives are then sampled on the device (gorse_b200_eval_create), which is what
 * the reference's Fit does itself.  In a distributed context the test rows are the rank's own users'.
 * ---------------------------------------------------------------------------------------- */
typedef struct {
    int32_t n_factors;   /* NFactors, default 16 */
    int32_t n_epochs;    /* NEpochs, default 100 (BPR) / 50 (ALS) */
    float lr;            /* Lr, BPR only, default 0.05 */
    float reg;           /* Reg, default 0.01 (BPR) / 0.06 (ALS) */
    float init_mean;     /* InitMean, default 0 */
    float init_stddev;   /* InitStdDev, default 0.001 (BPR) / 0.1 (ALS) */
    float alpha;         /* Alpha (eALS weight), ALS only, default 0.001 */
    uint64_t seed;       /* RandomState */
    int32_t verbose;     /* FitConfig.Verbose, default 10 */
    int32_t candidates;  /* FitConfig.Candidates, default 100: negatives per user when neg_off == NULL (sampled on the device) */
    int32_t topk;        /* FitConfig.TopK, default 10 */
    int32_t patience;    /* FitConfig.Patience, default 0 = no early stopping */
} gorse_b200_fit_params;

typedef struct {
    float ndcg, precision, recall; /* cf.Score of the LAST evaluation; all zero when cancelled (:491-493) */
    int32_t epochs_run;
    int32_t early_stopped, best_epoch;
    int32_t cancelled;
} gorse_b200_fit_result;

/* called after every epoch (monitor span.Add(1), model.go:519); ndcg < 0 when the epoch was not evaluated.
 * Return non-zero to cancel (ctx.Err() != nil): Fit then returns a zero Score like the reference. */
typedef int32_t (*gorse_b200_progress_fn)(void *user, int32_t epoch, int32_t n_epochs, float ndcg);

int32_t gorse_b200_fit_params_default(int32_t als, gorse_b200_fit_params *params);
int32_t gorse_b200_bpr_fit(gorse_b200_cf *cf, const gorse_b200_fit_params *params, const int64_t *test_off,
                           const int32_t *test_items, const int64_t *neg_off, const int32_t *neg_items,
                           gorse_b200_progress_fn progress, void *user, gorse_b200_fit_result *result);
int32_t gorse_b200_als_fit(gorse_b200_cf *cf, const gorse_b200_fit_params *params, const int64_t *test_off,
                           const int32_t *test_items, const int64_t *neg_off, const int32_t *neg_items,
                           gorse_b200_progress_fn progress, void *user, gorse_b200_fit_result *result);

/* ------------------------------------------------------------------------------------------
 * Model search.  The trials of ModelSearch.Objective (model/cf/optimize.go:61-81), which
 * optimizeCollaborativeFiltering (master/tasks.go:1268-1316) runs on every dataset load when
 * recommend.collaborative.optimize_period > 0, fitted in one call.  Trial k (als[k] != 0: eALS, else BPR) is what
 * gorse_b200_als_fit / gorse_b200_bpr_fit does with trials[k] on tables of its own: Init, Evaluate at epoch 0, n_epochs
 * epochs, Evaluate every `verbose` epochs and on the last one, Patience with the first-maximum rule; results[k] equals
 * that fit's result.  The trials share the search's FitConfig and RandomState: n_factors (== cf's d), seed, verbose,
 * candidates, topk and patience must be equal in every trial (else GORSE_B200_ERR_ARG); n_epochs and the model's
 * hyper-parameters may differ.  At one seed every BPR trial samples the same triples, so each epoch samples every triple
 * once for all the BPR trials and runs their arithmetic in the same cooperative launch (16 models per launch at d = 16,
 * 9 at 32, 4 at 64, 2 at 128; more run as successive launches); ALS trials run gorse_b200_als_epoch's kernels on their
 * own tables.  One evaluation plan serves every trial (negatives drawn at seed 0 when neg_off is NULL, as each solo fit
 * draws them).  A trial that stops or finishes leaves the batch with its tables as they are.
 * progress (may be NULL) is called once per epoch of the batch with the state of every trial; a non-zero return
 * cancels: a trial not reported finished in that call returns cancelled = 1 and a zero score, the others keep theirs.
 * P_out / Q_out (each may be NULL, as may any entry): trial k's final factors are copied to P_out[k] (n_users x d) and
 * Q_out[k] (n_items x d).  The trial tables are allocated in the call and freed before it returns; cf's own factors are
 * not touched.  Every argument is checked on the host before the device is touched (cf last): BPR trials need d in
 * {16, 32, 64, 128} and ALS trials the item CSR (GORSE_B200_ERR_UNSUPPORTED / GORSE_B200_ERR_STATE); a distributed
 * context is GORSE_B200_ERR_UNSUPPORTED.
 * ---------------------------------------------------------------------------------------- */
typedef struct {
    int32_t epochs_run;  /* epochs the trial has run so far */
    float ndcg;          /* NDCG of this epoch's evaluation, < 0 when the trial was not evaluated in this epoch */
    int32_t finished;    /* 1 once the trial has run its n_epochs or stopped early */
} gorse_b200_trial_state;
typedef int32_t (*gorse_b200_trials_progress_fn)(void *user, int32_t epoch, int32_t n_trials, const gorse_b200_trial_state *states);

int32_t gorse_b200_cf_fit_trials(gorse_b200_cf *cf, int32_t n_trials, const int32_t *als, const gorse_b200_fit_params *trials,
                                 const int64_t *test_off, const int32_t *test_items, const int64_t *neg_off,
                                 const int32_t *neg_items, gorse_b200_trials_progress_fn progress, void *user,
                                 gorse_b200_fit_result *results, float *const *P_out, float *const *Q_out);

/* ------------------------------------------------------------------------------------------
 * Brute-force index.  Replaces ann.Bruteforce[[]float32] (common/ann/bruteforce.go:24-83)
 * behind ann.Index (common/ann/ann.go:21-25).
 * ---------------------------------------------------------------------------------------- */
typedef enum {
    GORSE_B200_METRIC_EUCLIDEAN = 0, /* floats.Euclidean (common/ann/ann_test.go:126) */
    GORSE_B200_METRIC_NEG_DOT = 1,   /* -floats.Dot (logics/cf.go:32-34) */
    GORSE_B200_METRIC_COSINE = 2     /* 1 - cos (vector collections only, storage/vectors/database.go:30; always the exact scan) */
} gorse_b200_metric;

int32_t gorse_b200_index_create(gorse_b200_ctx *ctx, int32_t dim, int32_t metric, gorse_b200_index **out);
int32_t gorse_b200_index_destroy(gorse_b200_index *ix);
/* Bruteforce.Add (bruteforce.go:33-37) for n vectors at once; *count_out = len after append
 * (the reference returns the 1-based length) */
int32_t gorse_b200_index_add(gorse_b200_index *ix, const float *vectors, int64_t n, int64_t *count_out);
int32_t gorse_b200_index_len(const gorse_b200_index *ix, int64_t *count_out);
/* SearchVector (bruteforce.go:65-83) for nq query vectors; results ascending by distance.
 * idx_out/dist_out: nq x k, rows padded with idx = -1; count_out[nq] = results per query
 * (fewer than k when the index is small or prune0 dropped score <= 0). */
int32_t gorse_b200_index_search_vectors(gorse_b200_index *ix, const float *queries, int64_t nq, int32_t k,
                                        int32_t prune0, int32_t *idx_out, float *dist_out, int32_t *count_out);
/* SearchIndex (bruteforce.go:39-63) for nq stored vectors q_idx[nq]; never returns the query itself;
 * GORSE_B200_ERR_RANGE if any index is out of range */
int32_t gorse_b200_index_search_indices(gorse_b200_index *ix, const int64_t *q_idx, int64_t nq, int32_t k,
                                        int32_t prune0, int32_t *idx_out, float *dist_out, int32_t *count_out);
/* all-pairs SearchIndex for stored vectors [q0, q1): item-to-item / user-to-user neighbours
 * (what logics.item_to_item asks its vector store for, logics/item_to_item.go:50-62) */
int32_t gorse_b200_index_search_range(gorse_b200_index *ix, int64_t q0, int64_t q1, int32_t k, int32_t prune0,
                                      int32_t *idx_out, float *dist_out, int32_t *count_out);
/* measurement hook (bench.py), like gorse_b200_ctx_timer_*: since the previous call, the device time (ms) and algorithmic
 * flop (2 nq N d) of the tensor-core candidate sweep, and the number of query rows that were redone by the exact scan because
 * their candidate set could not be certified.  Any pointer may be NULL. */
int32_t gorse_b200_index_stats(gorse_b200_index *ix, double *stage1_ms, double *stage1_flop, int64_t *fallback_rows);
/* test hook: the dense tensor-core scores of stored vectors [q0, q1) against all N vectors, original column order,
 * out[(q - q0) * N + x] (what the candidate sweep thresholds; small problems only), and when eps_out is not NULL each row's
 * error margin, eps_out[q - q0]: the sweep relies on |score - exact score| <= eps for every column */
int32_t gorse_b200_index_stage1_scores(gorse_b200_index *ix, int64_t q0, int64_t q1, float *out, float *eps_out);


/* ------------------------------------------------------------------------------------------
 * Similarity vectors and scores: the host logic of logics.item_to_item / logics.user_to_user
 * around the neighbour search (SURVEY 8a row J).  Pure host functions except _index_query_similar.
 * ---------------------------------------------------------------------------------------- */
/* dense embedding as the reference stores it: bfloats.FromFloat32 + ToFloat32
 * (common/bfloats/bfloats.go:23-37; logics/item_to_item.go:151-164).  in == out is allowed. */
int32_t gorse_b200_bf16_truncate(const float *in, int64_t n, float *out);
/* appendSparseVector (logics/vector_writer.go:200-209): ids outside [0, n_idf) or with idf <= 0 are
 * skipped; value = (float)sqrt((double)idf[id]); index = offset + id ("auto" appends users after tags
 * with offset = len(tagsIDF), logics/item_to_item.go:238-239).  Outputs hold up to n_ids entries. */
int32_t gorse_b200_sparse_vector(const int32_t *ids, int32_t n_ids, const float *idf, int32_t n_idf, uint32_t offset,
                                 uint32_t *indices_out, float *values_out, int32_t *count_out);
/* QueryItemToItem / QueryUserToUser score post-processing (logics/item_to_item.go:63-85,
 * logics/user_to_user.go:63-85) applied to one result row of this library (ascending distance,
 * id -1 padding): drop self_id; NEG_DOT: drop dot <= 0, score = dot * scale; EUCLIDEAN:
 * score = 1 / (1 + dist * scale); stop at n.  score_scale is 0.5 for type "auto", else 1. */
int32_t gorse_b200_similar_scores(int32_t metric, double score_scale, int32_t self_id, int32_t n, const int32_t *nbr_ids,
                                  const float *nbr_dist, int32_t n_nbr, int32_t *ids_out, double *scores_out, int32_t *count_out);
/* QueryItemToItem for the stored vectors [q0, q1): ids_out / scores_out are (q1-q0) x n (id -1 padding),
 * count_out[q1-q0] */
int32_t gorse_b200_index_query_similar(gorse_b200_index *ix, int64_t q0, int64_t q1, int32_t n, double score_scale,
                                       int32_t *ids_out, double *scores_out, int32_t *count_out);
/* Model hand-off (SURVEY 8f-4): the factor block of cf.BaseMatrixFactorization.Marshal (model/cf/model.go:212-245) for one
 * table straight from the flat host mirror: int64 LE count of predictable rows, then one varint-delimited
 * protocol.LatentFactor{id = 1, data = 2 packed} per predictable row (protocol/encoding.proto:27-30), byte for byte what
 * pbutil.WriteDelimited emits.  predictable == NULL: every row.  Host function.  *len_out = bytes needed; with out == NULL
 * only the size is computed; a too small buffer gives GORSE_B200_ERR_RANGE. */
int32_t gorse_b200_marshal_latent_factors(const float *factors, int32_t rows, int32_t d, const uint8_t *predictable, const char *const *ids,
                                          uint8_t *out, size_t cap, size_t *len_out);

/* ------------------------------------------------------------------------------------------
 * Sparse index (SURVEY 8f-1): brute-force search over sparse
 * vectors with the Dot metric -- what the "tags" / "users" / "auto" similarity types ask their vector
 * store for (storage/vectors/xvec.go:244-248 flat sparse index, :405 query).
 * ---------------------------------------------------------------------------------------- */
typedef struct gorse_b200_sparse_index gorse_b200_sparse_index;
int32_t gorse_b200_sparse_index_create(gorse_b200_ctx *ctx, gorse_b200_sparse_index **out);
int32_t gorse_b200_sparse_index_destroy(gorse_b200_sparse_index *ix);
/* append n vectors given as CSR (off[n+1] with off[0] = 0; indices strictly ascending inside a vector,
 * as appendSparseVector produces them from sorted ids); *count_out = number of vectors afterwards */
int32_t gorse_b200_sparse_index_add(gorse_b200_sparse_index *ix, const int64_t *off, const uint32_t *indices, const float *values,
                                    int64_t n, int64_t *count_out);
int32_t gorse_b200_sparse_index_len(const gorse_b200_sparse_index *ix, int64_t *count_out);
/* the k (<= 128) stored vectors with the largest POSITIVE dot with each stored vector in [q0, q1), the vector
 * itself excluded; best first (ties: lower index first); idx_out/dot_out are (q1-q0) x k padded with -1 / 0.
 * Feed a row to gorse_b200_similar_scores with GORSE_B200_METRIC_NEG_DOT after negating the dots. */
int32_t gorse_b200_sparse_index_search_range(gorse_b200_sparse_index *ix, int64_t q0, int64_t q1, int32_t k, int32_t *idx_out,
                                             float *dot_out, int32_t *count_out);

/* ------------------------------------------------------------------------------------------
 * Vector collection: the GPU backend of vectors.Database (storage/vectors/database.go:107-120; semantics of the
 * reference's default backend storage/vectors/xvec.go:288-449), registered from Go with
 * vectors.Register([]string{"b200://"}, ...) (database.go:161-165; go/storage/vectors/b200.go).  One handle = one
 * collection.  Vectors live in SLOTS (int64, insertion order); the shim owns the id string <-> slot map and the category
 * string <-> int32 map.  dim = 0: sparse vectors, Dot only (xvec.go:243-248).  Thread-safe per collection.
 * ---------------------------------------------------------------------------------------- */
typedef enum {   /* vectors.Distance, storage/vectors/database.go:27-33 */
    GORSE_B200_DISTANCE_COSINE = 0,
    GORSE_B200_DISTANCE_EUCLIDEAN = 1,
    GORSE_B200_DISTANCE_DOT = 2
} gorse_b200_distance;
typedef struct gorse_b200_vecdb gorse_b200_vecdb;
int32_t gorse_b200_vecdb_create(gorse_b200_ctx *ctx, int32_t dim, int32_t distance, gorse_b200_vecdb **out); /* AddCollection */
int32_t gorse_b200_vecdb_destroy(gorse_b200_vecdb *db);                                                     /* DeleteCollection */
/* CountVectors (xvec.go:274-286): live vectors; *slots_out = slots ever assigned */
int32_t gorse_b200_vecdb_count(gorse_b200_vecdb *db, int64_t *live_out, int64_t *slots_out);
/* AddVectors (xvec.go:288-318; an UPSERT by id): n vectors go to slots *first_slot_out .. +n-1.
 * dense: values[n*dim]; sparse: sp_off[n+1] (from 0), sp_indices strictly ascending per vector, values[sp_off[n]].
 * hidden[n], timestamp_ms[n] (Vector.Timestamp.UnixMilli()), categories as CSR cat_off[n+1] / cats (any may be NULL = none).
 * replace[n]: the slot currently holding the same id (it is tombstoned), or -1; NULL = all new. */
int32_t gorse_b200_vecdb_add(gorse_b200_vecdb *db, int64_t n, const float *values, const int64_t *sp_off, const uint32_t *sp_indices,
                             const uint8_t *hidden, const int64_t *timestamp_ms, const int64_t *cat_off, const int32_t *cats,
                             const int64_t *replace, int64_t *first_slot_out);
/* GetVectors (xvec.go:320-363) by slot; live_out[i] = 0 for unknown or deleted slots.  Dense values_out[n*dim]. */
int32_t gorse_b200_vecdb_get(gorse_b200_vecdb *db, const int64_t *slots, int64_t n, float *values_out, uint8_t *hidden_out,
                             int64_t *timestamp_out, uint8_t *live_out);
int32_t gorse_b200_vecdb_get_sparse(gorse_b200_vecdb *db, int64_t slot, uint32_t *indices_out, float *values_out, int32_t cap,
                                    int32_t *nnz_out);
/* DeleteVectors(timestamp) (xvec.go:365-371): tombstones live vectors with timestamp < timestamp_ms; the first `cap` deleted
 * slots are written to slots_out (the shim drops their ids), *count_out = how many were deleted */
int32_t gorse_b200_vecdb_delete_before(gorse_b200_vecdb *db, int64_t timestamp_ms, int64_t *slots_out, int64_t cap, int64_t *count_out);
/* QueryVectors (xvec.go:373-449) for nq query vectors sharing one category filter: candidates are live, not hidden and
 * carry ALL of categories[n_categories] (CONTAIN_ALL, :381-389).  Results per query: slots_out / scores_out [nq x topk],
 * best first, count_out[nq]; entries past count_out[q] in a row are not part of the answer and are left unspecified; score = dot (Dot) or the NEGATED distance (Euclidean, Cosine) -- higher is more similar
 * (database.go:101, xvec.go:425-427).  Sparse: only positive dots are returned (the reference drops score 0, :421-423, and
 * its callers drop score <= 0, logics/item_to_item.go:73); topk <= 128.  topk <= 0 -> no results (:374-376). */
/* Model hand-off (master/tasks.go:925-961): the item factors of every item with >= 1 training feedback (IsItemPredictable)
 * become vectors of a Dot collection, device to device -- no GetItemFactor round trip.  hidden[n_items], categories CSR over
 * items (may be NULL), one timestamp (the model id, :925).  slot_of_item_out[n_items]: slot per item, -1 = not predictable. */
int32_t gorse_b200_vecdb_add_item_factors(gorse_b200_vecdb *db, gorse_b200_cf *cf, const uint8_t *hidden, int64_t timestamp_ms,
                                          const int64_t *cat_off, const int32_t *cats, int64_t *slot_of_item_out);
int32_t gorse_b200_vecdb_query(gorse_b200_vecdb *db, int64_t nq, const float *q_values, const int64_t *q_sp_off, const uint32_t *q_sp_indices,
                               const int32_t *categories, int32_t n_categories, int32_t topk, int64_t *slots_out, float *scores_out,
                               int32_t *count_out);
/* Batched CF recall: for nq users at once, what the worker's collaborative-filtering recall does per user
 * (worker/pipeline.go:403-449): QueryVectors(user embedding, categories, topK = n + |E_q|) followed by dropping every id of the
 * user's exclude set E_q (the feedback items, logics/recommend.go:67-80).
 *   E_q = excl_slots[excl_off[q] .. excl_off[q+1]) (excl_off[0] = 0), any order; an entry is a slot of this collection or -1
 *   for an excluded id the collection does not hold (it still counts in |E_q|).  A slot twice in one row is GORSE_B200_ERR_ARG.
 *   Row q: the candidates of gorse_b200_vecdb_query (live, not hidden, CONTAIN_ALL categories) by score descending, exact ties
 *   by lower slot; the first k_q = n + |E_q| of them; minus the slots in E_q -- so a row may hold more than n results, as in
 *   the reference.  Scores are bit-identical to gorse_b200_vecdb_query's (dot, or the negated distance).
 *   Output: row q starts at q*n + excl_off[q] in slots_out / scores_out and has room for n + |E_q| entries (buffers of
 *   nq*n + excl_off[nq]); count_out[q] = entries written.  n <= 0: every count is 0.  A NaN score: GORSE_B200_ERR_ARG.
 *   Sparse collections: GORSE_B200_ERR_UNSUPPORTED.  exact_rows_out (may be NULL): rows answered by the exact scan rather than
 *   the tensor-core sweep; the answer does not depend on it.  Thread-safe per collection. */
int32_t gorse_b200_vecdb_query_excluding(gorse_b200_vecdb *db, int64_t nq, const float *q_values, const int32_t *categories,
                                         int32_t n_categories, int32_t n, const int64_t *excl_off, const int64_t *excl_slots,
                                         int64_t *slots_out, float *scores_out, int32_t *count_out, int64_t *exact_rows_out);
/* Batched item-to-item recommendation: for n_users users at once, what the worker's item-to-item recommender does per user
 * (Recommender.recommendItemToItem, logics/recommend.go:244-283) on one item-to-item collection: Euclidean for type
 * "embedding", sparse Dot for "tags" / "users" / "auto".
 *   C_u = ctx_slots[ctx_off[u] .. ctx_off[u+1]) (ctx_off[0] = 0): the user's positive feedback items, visited in the given
 *   order (the reference's is newest first); a slot may repeat (its neighbours are then added again).  Entries -1 (an id
 *   without a vector) and deleted slots are skipped; a hidden item is still a context item.  A slot outside [-1, slots) is
 *   GORSE_B200_ERR_ARG.
 *   E_u = excl_slots[excl_off[u] .. excl_off[u+1]): the user's exclude set, with the rules of
 *   gorse_b200_vecdb_query_excluding (-1 allowed, a slot twice in one row is GORSE_B200_ERR_ARG).
 *   Neighbours of a context item c: the candidates of gorse_b200_vecdb_query (live, not hidden, ALL of
 *   categories[n_categories]) other than c, by score descending, exact ties by lower slot; Dot collections drop scores <= 0;
 *   the first n.  Their scores are bit-identical to gorse_b200_vecdb_query's.
 *   Neighbour score s = (double)score * score_scale (0.5 for type "auto", else 1); Euclidean: s = 1 / (1 - s).
 *   Row u: for every context entry in order and every neighbour j not in E_u, acc[j] += s in float64; the first n of acc by
 *   score descending, exact ties by lower slot.  Each sum is formed in context order, as the reference's, so the scores match
 *   it bit for bit.  The reference ranks exact ties in Go map order, so which of them it keeps at the cut is unpinned.
 *   Output: row u at u*n in slots_out / scores_out (buffers of n_users*n), count_out[u] <= n entries.  n <= 0: every count
 *   is 0.  n above 128 (sparse) or 1024 (dense): GORSE_B200_ERR_UNSUPPORTED; Cosine collections: GORSE_B200_ERR_UNSUPPORTED.
 *   A NaN score (or score_scale): GORSE_B200_ERR_ARG.  Every argument is checked before the device is touched.
 *   stats_out[4] (may be NULL): distinct context items queried, of them answered by the exact scan rather than the tensor-core
 *   sweep (dense), users aggregated in shared memory, users aggregated in a global-memory row; the answer does not depend
 *   on them.  Thread-safe per collection. */
int32_t gorse_b200_vecdb_item_to_item(gorse_b200_vecdb *db, int64_t n_users, const int64_t *ctx_off, const int64_t *ctx_slots,
                                      const int64_t *excl_off, const int64_t *excl_slots, const int32_t *categories, int32_t n_categories,
                                      int32_t n, double score_scale, int64_t *slots_out, double *scores_out, int32_t *count_out,
                                      int64_t *stats_out);
/* Batched user-to-user recommendation: for n_users users at once, what the worker's user-to-user recommender does per user
 * (Recommender.recommendUserToUser, logics/recommend.go:285-348) on one user-to-user collection: Euclidean for type
 * "embedding", sparse Dot for "tags" / "items" / "auto" (a dense Dot collection follows the Dot rules).
 *   user_slots[u]: the user's slot, or -1 for a user without a vector; -1 and deleted slots give an empty row, a hidden user
 *   is still queried, a slot may repeat.  A slot outside [-1, slots) is GORSE_B200_ERR_ARG.
 *   Neighbours of u: the live, not hidden vectors other than u (no category filter) by score descending, exact ties by lower
 *   slot; Dot collections drop scores <= 0; the first n (QueryUserToUser, logics/user_to_user.go:50-86).  Their scores are
 *   bit-identical to gorse_b200_vecdb_query's.  Neighbour score s = (double)score * score_scale (0.5 for type "auto",
 *   else 1); Euclidean: s = 1 / (1 - s).
 *   Feedback: fb_off[n_fb_rows + 1] (fb_off[0] = 0; may be NULL when n_fb_rows = 0) / fb_items: each slot's positive
 *   feedback as item indices in [0, n_items) of the caller's item dictionary; slots at or beyond n_fb_rows have none.  A row
 *   may repeat an item (it is then added again); the order within a row does not matter.
 *   E_u = excl_items[excl_off[u] .. excl_off[u+1]) (excl_off[0] = 0): the user's exclude set as item indices, -1 for an id
 *   outside the dictionary; an item twice in one row is GORSE_B200_ERR_ARG.
 *   item_ok[n_items] (may be NULL = every item passes): 1 for the items that exist, are not hidden, are within the TTL and
 *   hold all of the requested categories; the same filter for every user of the call.
 *   Row u: for every neighbour in order and every feedback entry of it not in E_u, acc[item] += s in float64 (each sum
 *   starting at 0 + s); the first n by (sum descending, item ascending); then the entries with item_ok = 0 are dropped,
 *   keeping the order, so a row may hold fewer than n.  Each sum is formed in neighbour order, as the reference's, so the
 *   scores match it bit for bit.  The reference ranks exact ties in Go map order, so which of them it keeps at the cut is
 *   unpinned.
 *   Output: row u at u*n in items_out / scores_out (buffers of n_users*n), count_out[u] <= n entries.  n <= 0: every count
 *   is 0.  n above 128 (sparse) or 1024 (dense): GORSE_B200_ERR_UNSUPPORTED; Cosine collections: GORSE_B200_ERR_UNSUPPORTED.
 *   A NaN score (or score_scale): GORSE_B200_ERR_ARG.  Every argument, each fb_items entry included, is checked before the
 *   device is touched.  stats_out[4] (may be NULL): distinct query users searched, of them answered by the exact scan
 *   rather than the tensor-core sweep (dense), users aggregated in shared memory, users aggregated in a global-memory row
 *   (users with nothing to add are in neither); the answer does not depend on them.  Thread-safe per collection. */
int32_t gorse_b200_vecdb_user_to_user(gorse_b200_vecdb *db, int64_t n_users, const int64_t *user_slots, int64_t n_fb_rows,
                                      const int64_t *fb_off, const int32_t *fb_items, int32_t n_items, const uint8_t *item_ok,
                                      const int64_t *excl_off, const int64_t *excl_items, int32_t n, double score_scale,
                                      int64_t *items_out, double *scores_out, int32_t *count_out, int64_t *stats_out);

/* ------------------------------------------------------------------------------------------
 * Batched FM ranking: the worker's "fm" ranker (rankByClickTroughRate, worker/pipeline.go:450-499) for many users in one
 * call -- AFM.BatchPredict (model/ctr/fm.go:180-229) on every (user, candidate) pair of each user, then the candidates by
 * score.  Training is gorse_b200_fm_fit below for models without embedding slots, and gorse_b200_fm_fit_emb for models
 * with them.
 * gorse_b200_fm_create uploads one trained model once; the handle is read-only afterwards and thread-safe.
 *   n_features = fm.numFeatures (the unified index's Len), n_factors = nFactors, num_dimension = fm.numDimension,
 *   batch_size = the BatchSize param (default 1024), emb_dim[n_emb] = fm.embeddingDim.
 *   params[n_params]: fm.Parameters() (fm.go:136-146) concatenated in order: B[1], V[n_features x n_factors],
 *   W[n_features], then per slot H[n_factors x dim], AW[dim x n_factors], Ab[n_factors], EW[dim x n_factors],
 *   Eb[n_factors].  A wrong n_params is GORSE_B200_ERR_ARG.  n_factors above 32, an embedding dim above 1024 or more than 8
 *   slots: GORSE_B200_ERR_UNSUPPORTED.
 * gorse_b200_fm_rank takes the pairs factored, as the reference builds them once per user and once per item:
 *   users: user_feat[n_users] (fm.Index.EncodeUser, -1 = unknown) and the known labels as a CSR user_lab_off[n_users + 1]
 *   (from 0) / user_lab_idx / user_lab_val, in label order, values already through fm.Scalers (applyScalers, fm.go:232-245).
 *   item table of the call: item_feat[n_items], item_lab_off / item_lab_idx / item_lab_val the same way; item_emb[s]
 *   [n_items x emb_dim[s]] bf16 bits per slot, item_emb_mask[n_items x n_emb] 1 where the item's embedding of slot s is
 *   present with the right length (NULL: all present); an absent one is zeros (convertToTensors, fm.go:555-561).
 *   candidates: cand_off[n_users + 1] (from 0) / cand_items, rows of the item table, repeats allowed.
 *   Row of pair (u, i): user id (value 1), item id (value 1), user labels, item labels; padded to
 *   D_u = max(num_dimension, the user's longest row) with index 0, value 0; indices travel as float32; chunks of
 *   batch_size pairs in candidate order; the softmax of a chunk couples its rows as the reference's does (DESIGN §8.4).
 *   Output: scores_out[cand_off[n_users]] float32 in candidate order, bit-identical to the reference's restatement;
 *   order_out[cand_off[n_users]]: per user, the candidate positions (0-based within the user) by score descending, exact
 *   ties (-0 == +0) by position, NaN last.  The reference's sort (cache.SortDocuments) is not stable, so its order on ties is
 *   unpinned.  stats_out[4] (may be NULL): pairs, attention chunks, device passes, users sorted in global memory.
 *   Every index is checked on the host before the device is touched (GORSE_B200_ERR_ARG): a feature outside
 *   [0, n_features) -- also after rounding to float32 -- an item row outside the table, decreasing offsets. */
typedef struct gorse_b200_fm gorse_b200_fm;
int32_t gorse_b200_fm_create(gorse_b200_ctx *ctx, int64_t n_features, int32_t n_factors, int32_t num_dimension, int32_t batch_size,
                             int32_t n_emb, const int32_t *emb_dim, const float *params, int64_t n_params, gorse_b200_fm **out);
int32_t gorse_b200_fm_destroy(gorse_b200_fm *fm);
int32_t gorse_b200_fm_rank(gorse_b200_fm *fm, int64_t n_users, const int32_t *user_feat, const int64_t *user_lab_off,
                           const int32_t *user_lab_idx, const float *user_lab_val, int64_t n_items, const int32_t *item_feat,
                           const int64_t *item_lab_off, const int32_t *item_lab_idx, const float *item_lab_val,
                           const uint16_t *const *item_emb, const uint8_t *item_emb_mask, const int64_t *cand_off,
                           const int32_t *cand_items, float *scores_out, int32_t *order_out, int64_t *stats_out);

/* ------------------------------------------------------------------------------------------
 * Batched offline recommendation: for n_users users at once, what the worker's offline loop does per user after
 * NewRecommender (worker/pipeline.go:124-319): the CF recall (updateCollaborativeRecommend, :403-449), the recommenders in the
 * configured order (Recommender.RecommendSequential with limit 0, logics/recommend.go:135-156), the candidate list
 * (pipeline.go:228-243), the replacement items (addReplacementCandidates, :573-611) and the FM ranking
 * (rankByClickTroughRate, :451-499) followed by the replacement decay (applyReplacementDecay, :613-643).  The exclude set
 * and the candidates of every user stay on the device from the first stage to the ranked list.  Everything runs in the item
 * index space [0, n_items) of the call's item DICTIONARY, which must hold every id a stage can return.
 *   E0_u = excl_items[excl_off[u] .. excl_off[u+1]) (excl_off[0] = 0): the user's feedback items (NewRecommender,
 *   logics/recommend.go:61-93, offline: every feedback item), an item index or -1 for an id outside the dictionary; every
 *   entry counts in |E0_u| (excludeSet.Cardinality()); an item twice is GORSE_B200_ERR_ARG.
 *   item_live[n_items]: 1 for the items that exist and are not hidden (ItemCache).
 *   CF recall (cf, needed by a COLLABORATIVE stage): the first cf->n + |E0_u| results of gorse_b200_vecdb_query_excluding on
 *   the CF collection for the user's vector, minus E0_u; scores float64(float32).
 *   Stages, in order.  Each produces a list; entries in the running exclude set E_u are dropped as the reference's
 *   recommender drops them; the list is appended to the candidates, and only then is every produced id added to E_u (so a
 *   duplicate inside one stage survives).  Kinds (gorse_b200_recommend_stage.kind):
 *     LIST            non-personalized / latest (list_off == NULL: one list list_items / list_scores[list_len] for every
 *                     user) or external (list_off[n_users + 1] from 0: one list per user); entries in E_u are dropped
 *                     (recommend.go:180-225, :350-384).  Bound: the list's length.
 *     COLLABORATIVE   the CF recall row, minus the items with item_live = 0, cut at cf->n, then minus E_u
 *                     (recommend.go:227-242: SearchScores(0, CacheSize) on the cached row, then the filter).  Bound: cf->n.
 *     ITEM_TO_ITEM    gorse_b200_vecdb_item_to_item's row on db (n, score_scale, categories) with E_u as its exclude set;
 *                     context ctx_items[ctx_off[u] ..) as item indices, newest first, -1 skipped; slot_of_item[n_items] /
 *                     item_of_slot[slots of db] map between the dictionary and the collection (-1 = none).  Bound: n.
 *     USER_TO_USER    gorse_b200_vecdb_user_to_user's row on db (user_slots, feedback rows, item_ok, n, score_scale) with
 *                     E_u as its exclude set.  Bound: n.
 *   Candidates: the stage lists concatenated in order, minus the items with item_live = 0, in order (a dropped item still
 *   excludes).  With a ranker and a replacement CSR repl_off[n_users + 1] (from 0) / repl_items / repl_positive (distinct
 *   feedback items per user, 1 = positive, 0 = read): the live replacement items that are not candidates yet are appended in
 *   the given order.  The reference's order here is mapset order, so it is unpinned.
 *   Ranking (ranker != NULL): gorse_b200_fm_rank's semantics on the final candidates -- D_u, the attention chunks in
 *   candidate order, float32 scores; then the scores of the live positive / read replacement items are multiplied in
 *   float64 by positive_decay / read_decay, and the row is sorted by score descending, exact ties (-0 == +0) by candidate
 *   position, NaN last.  The reference's sort is not stable, so its order on ties is unpinned.  ranker == NULL
 *   (Ranker.Type = "none"): the candidates in merged order with their stage scores, no replacement.
 *   Output: B_u = the sum of the stage bounds + |repl_u| (the replacement count only with a ranker).  Row u starts at
 *   B_0 + ... + B_{u-1} in items_out (int32 item indices) / scores_out (float64); count_out[u] <= B_u entries.
 *   Limits are those of the entries reused: n <= 1024 (dense) / 128 (sparse), Cosine collections and sparse CF collections
 *   are GORSE_B200_ERR_UNSUPPORTED, gorse_b200_fm_create's limits; a list may hold at most 4096 entries.  Every argument is
 *   checked on the host before the device is touched (GORSE_B200_ERR_ARG): offsets, items, slots, a live slot whose
 *   item_of_slot is -1 or whose slot_of_item does not point back, NaN scores or decays, features as gorse_b200_fm_rank
 *   checks them, collections or a ranker of another context.  The library keeps no host pointer after the call.
 *   stats_out[4] (may be NULL): chunks, candidates ranked or returned, neighbour-table rows of all stages, rows answered
 *   by the exact scan rather than the tensor-core sweep; the answer does not depend on them. */
typedef enum {
    GORSE_B200_STAGE_LIST = 0,
    GORSE_B200_STAGE_COLLABORATIVE = 1,
    GORSE_B200_STAGE_ITEM_TO_ITEM = 2,
    GORSE_B200_STAGE_USER_TO_USER = 3
} gorse_b200_stage_kind;

typedef struct {
    int32_t kind;                  /* gorse_b200_stage_kind */
    /* LIST */
    int64_t list_len;              /* shared list: its length; per-user lists: ignored */
    const int64_t *list_off;       /* NULL = one shared list; else [n_users + 1] from 0 */
    const int32_t *list_items;     /* item indices */
    const double *list_scores;     /* not NaN */
    /* ITEM_TO_ITEM, USER_TO_USER */
    gorse_b200_vecdb *db;
    int32_t n;                     /* CacheSize */
    double score_scale;            /* 0.5 for type "auto", else 1 */
    /* ITEM_TO_ITEM */
    const int64_t *ctx_off;        /* [n_users + 1] from 0 */
    const int32_t *ctx_items;      /* item indices, -1 = an id outside the dictionary */
    const int64_t *slot_of_item;   /* [n_items] */
    const int32_t *item_of_slot;   /* [slots of db] */
    const int32_t *categories;
    int32_t n_categories;
    /* USER_TO_USER */
    const int64_t *user_slots;     /* [n_users], -1 = no vector */
    int64_t n_fb_rows;
    const int64_t *fb_off;         /* [n_fb_rows + 1] from 0 */
    const int32_t *fb_items;       /* item indices */
    const uint8_t *item_ok;        /* [n_items] or NULL */
} gorse_b200_recommend_stage;

typedef struct {
    gorse_b200_vecdb *db;          /* the dense CF collection (collaborative_filtering_<id>) */
    const float *user_vectors;     /* [n_users x dim] */
    const int64_t *slot_of_item;   /* [n_items] */
    const int32_t *item_of_slot;   /* [slots of db] */
    int32_t n;                     /* CacheSize */
} gorse_b200_recommend_cf;

typedef struct {
    gorse_b200_fm *fm;
    const int32_t *user_feat;      /* users as gorse_b200_fm_rank takes them, [n_users] */
    const int64_t *user_lab_off;
    const int32_t *user_lab_idx;
    const float *user_lab_val;
    const int32_t *item_feat;      /* the dictionary's item table, [n_items] rows */
    const int64_t *item_lab_off;
    const int32_t *item_lab_idx;
    const float *item_lab_val;
    const uint16_t *const *item_emb;
    const uint8_t *item_emb_mask;
} gorse_b200_recommend_ranker;

int32_t gorse_b200_recommend(gorse_b200_ctx *ctx, int64_t n_users, const int64_t *excl_off, const int32_t *excl_items, int32_t n_items,
                             const uint8_t *item_live, int32_t n_stages, const gorse_b200_recommend_stage *stages,
                             const gorse_b200_recommend_cf *cf, const gorse_b200_recommend_ranker *ranker, const int64_t *repl_off,
                             const int32_t *repl_items, const uint8_t *repl_positive, double positive_decay, double read_decay,
                             int32_t *items_out, double *scores_out, int32_t *count_out, int64_t *stats_out);

/* ------------------------------------------------------------------------------------------
 * FM training: AFM.Fit (model/ctr/fm.go:307-417) for a model without item-embedding slots (plain FM: bias, linear and
 * pairwise terms), step for step.  The master runs it every ranker.fit_period (master/tasks.go:1047-1155) and
 * optimize_trials more times (:1318-1363).  Init and the scalers stay with the caller: it passes fm.Parameters() after
 * Init as params_in, and rows already through fm.Scalers.
 *   n_features = the unified index's Len, num_dimension = fm.numDimension (the longest training row), n_emb = the number
 *   of embedding slots: any slot, or n_factors above 32, is GORSE_B200_ERR_UNSUPPORTED (train those with the reference).
 *   train rows: CSR train_off[n_train + 1] (from 0) / train_idx / train_val, one row per trainSet.Get(i) in dataset order,
 *   train_target[n_train]; test rows the same way (targets > 0 are the positives of EvaluateClassification).
 *   params_in / params_out[n_params], n_params = 1 + n_features n_factors + n_features (another length is
 *   GORSE_B200_ERR_ARG): B, V, W in gorse_b200_fm_create's layout, so a fitted model goes straight into the ranker.  moments_out[2 n_params] (may be NULL): Adam's m then v (zeros for SGD).
 * What runs: evaluation at epoch 0; per epoch, the rows in dataset order in batches of batch_size (the last may be
 * partial), each padded to D = max(num_dimension, the longest training row) with index 0, value 0, indices through
 * float32; BCEWithLogits, its backward in the reference's order, then Adam (default) or SGD with weight decay `reg` over
 * every parameter; evaluation every `verbose` epochs and on the last one, then the NaN break (cost or Precision, which is
 * score.GetValue()) and early stopping on AUC with `patience` (0: none), best = the first maximum.  Every parameter and
 * moment is bit-identical to the project's CPU restatement (DESIGN §8.5); Log and Adam's Pow are restated algorithms whose
 * agreement with Go's math32 is not pinned.
 * progress (may be NULL) is called after the epoch-0 evaluation and after every epoch with the epoch and its AUC (-1 when
 * the epoch was not evaluated); a non-zero return cancels where the reference would see ctx.Err() -- at the next batch --
 * and Fit returns a zero score with `cancelled` set.  An epoch runs as one CUDA graph, so the callback and with it a
 * cancel come at most one epoch late; params_out then holds that epoch's updates.  max_steps > 0 stops after that many optimiser steps (tests and
 * benchmarks); the scores are then those of the last evaluation.
 * Every index is checked on the host before the device is touched (GORSE_B200_ERR_ARG), also after rounding to float32. */
typedef struct {
    int32_t n_factors;   /* NFactors, default 16 */
    int32_t n_epochs;    /* NEpochs, default 50 */
    float lr;            /* Lr, default 0.001 */
    float reg;           /* Reg (weight decay), default 0.0002 */
    int32_t optimizer;   /* GORSE_B200_FM_ADAM (default) or GORSE_B200_FM_SGD */
    int32_t batch_size;  /* BatchSize, default 1024 */
    int32_t verbose;     /* FitConfig.Verbose, default 10; must be >= 1 */
    int32_t patience;    /* FitConfig.Patience, default 10; 0 = no early stopping */
    int64_t max_steps;   /* 0 = no limit */
} gorse_b200_fm_fit_params;

enum { GORSE_B200_FM_ADAM = 0, GORSE_B200_FM_SGD = 1 };

typedef struct {
    float auc, precision, recall, accuracy; /* Score of the LAST evaluation; all zero when cancelled */
    float cost;                             /* sum of the batch losses of the last epoch run */
    int32_t epochs_run, best_epoch;         /* best_epoch: the first epoch with the highest AUC among the evaluations */
    int32_t early_stopped, diverged, cancelled;
    int64_t steps;                          /* optimiser steps run */
} gorse_b200_fm_fit_result;

int32_t gorse_b200_fm_fit_params_default(gorse_b200_fm_fit_params *params);
int32_t gorse_b200_fm_fit(gorse_b200_ctx *ctx, int64_t n_features, int32_t num_dimension, int32_t n_emb,
                          const gorse_b200_fm_fit_params *params, int64_t n_train, const int64_t *train_off, const int32_t *train_idx,
                          const float *train_val, const float *train_target, int64_t n_test, const int64_t *test_off,
                          const int32_t *test_idx, const float *test_val, const float *test_target, const float *params_in,
                          int64_t n_params, float *params_out, float *moments_out, gorse_b200_progress_fn progress, void *user,
                          gorse_b200_fm_fit_result *result);

/* FM training of a model with item-embedding slots: the same fit, with the attention and encoder layers of every slot
 * (common/nn/layers.go:160-185, fm.go:128-132) trained too.  gorse_b200_fm_fit's arguments, its params / result structs
 * and its progress / cancel / max_steps contract, plus
 *   n_emb, emb_dim[n_emb] = fm.embeddingDim; n_emb = 0 is gorse_b200_fm_fit, bit for bit.  n_factors above 32, a dim above
 *   1024 or more than 8 slots: GORSE_B200_ERR_UNSUPPORTED.
 *   the item-embedding table as gorse_b200_fm_rank takes it: item_emb[s] [n_emb_rows x emb_dim[s]] bf16 bits per slot,
 *   item_emb_mask[n_emb_rows x n_emb] 1 where the row's embedding of slot s is present (NULL: all present); an absent one
 *   is a row of zeros (convertToTensors, fm.go:555-561).  A mask that marks the wrong rows cannot be detected.
 *   train_emb_row[n_train] / test_emb_row[n_test]: the table row of each sample (dataset.Items[i]), -1 = no embeddings
 *   (zeros in every slot).  The kernels gather from the table.
 *   params_in / params_out[n_params] in gorse_b200_fm_create's layout: B, V, W, then per slot H, AW, Ab, EW, Eb; a fitted
 *   model goes straight into gorse_b200_fm_create.  moments_out[2 n_params] as above.
 * The softmax of a batch, and of every chunk of batch_size rows of the two evaluation lists, couples its rows as the
 * reference's does, in the forward and in the backward.  Every parameter and moment is bit-identical to the project's CPU
 * restatement (DESIGN §8.5).  A table row outside [-1, n_emb_rows), a NULL table with n_emb > 0 and a wrong n_params are
 * GORSE_B200_ERR_ARG, checked on the host before the device is touched. */
int32_t gorse_b200_fm_fit_emb(gorse_b200_ctx *ctx, int64_t n_features, int32_t num_dimension, const gorse_b200_fm_fit_params *params,
                              int64_t n_train, const int64_t *train_off, const int32_t *train_idx, const float *train_val,
                              const float *train_target, const int32_t *train_emb_row, int64_t n_test, const int64_t *test_off,
                              const int32_t *test_idx, const float *test_val, const float *test_target, const int32_t *test_emb_row,
                              int32_t n_emb, const int32_t *emb_dim, int64_t n_emb_rows, const uint16_t *const *item_emb,
                              const uint8_t *item_emb_mask, const float *params_in, int64_t n_params, float *params_out,
                              float *moments_out, gorse_b200_progress_fn progress, void *user, gorse_b200_fm_fit_result *result);

/* FM model search: the trials of AFM's ModelSearch (model/ctr/fm.go SuggestParams), which
 * optimizeClickThroughRatePrediction (master/tasks.go:1318-1363) runs on every dataset load when the ranker's
 * optimize_period > 0, fitted in one call.  gorse_b200_fm_fit_emb's arguments (n_emb = 0: the model without slots), with
 * per trial k: trials[k], params_in[k] (fm.Parameters() after the trial's own Init), params_out[k] and moments_out[k]
 * (each array and each entry may be NULL) and results[k].
 *   What each result equals: results[k], params_out[k] and moments_out[k] are bit-identical to what
 *   gorse_b200_fm_fit_emb returns for trials[k] and params_in[k] alone (with n_emb = 0 that is also gorse_b200_fm_fit),
 *   NaN payloads aside as there: every score, cost, epochs_run, best_epoch, the flags and steps.
 *   What the trials share: n_factors, batch_size, verbose, patience and max_steps must be equal in every trial (else
 *   GORSE_B200_ERR_ARG); lr, reg, optimizer and n_epochs may differ.  n_params is one value for all trials.
 *   Leaving the batch: a trial leaves when it has run its n_epochs, stops early or diverges; its tables are not touched
 *   after that.
 *   progress (may be NULL) gets every trial's state after the epoch-0 evaluation and after every epoch of the batch (not
 *   after an epoch cut short by max_steps, as the solo fit); auc is -1 for a trial not evaluated in that epoch.  A non-zero
 *   return cancels: each unfinished trial then gets exactly what a solo fit cancelled at that epoch gets (cancelled = 1, a
 *   zero score, params_out holding that epoch's updates); finished trials keep their results.  The callback is not
 *   called again.
 *   Groups: the trials run in groups of at most 16, one CUDA graph per epoch of a group, fewer when their tables do not
 *   fit the free device memory (DESIGN §8.8 has the bytes per trial); the groups run one after another, a later group's
 *   trials reporting {0, -1, 0} until it starts.  A cancel also cancels the trials of the later groups at their epoch 0.
 *   The trial tables are allocated in the call and freed before it returns.
 * Every argument is checked on the host before the device is touched, ctx last; n_factors above 32, more than 8 slots or a
 * dim above 1024 are GORSE_B200_ERR_UNSUPPORTED. */
typedef struct {
    int32_t epochs_run;  /* epochs the trial has run so far */
    float auc;           /* AUC of this epoch's evaluation, -1 when the trial was not evaluated in this epoch */
    int32_t finished;    /* 1 once the trial has run its n_epochs, stopped early or diverged */
} gorse_b200_fm_trial_state;
typedef int32_t (*gorse_b200_fm_trials_progress_fn)(void *user, int32_t epoch, int32_t n_trials, const gorse_b200_fm_trial_state *states);

int32_t gorse_b200_fm_fit_trials(gorse_b200_ctx *ctx, int64_t n_features, int32_t num_dimension, int32_t n_trials,
                                 const gorse_b200_fm_fit_params *trials, int64_t n_train, const int64_t *train_off,
                                 const int32_t *train_idx, const float *train_val, const float *train_target,
                                 const int32_t *train_emb_row, int64_t n_test, const int64_t *test_off, const int32_t *test_idx,
                                 const float *test_val, const float *test_target, const int32_t *test_emb_row, int32_t n_emb,
                                 const int32_t *emb_dim, int64_t n_emb_rows, const uint16_t *const *item_emb,
                                 const uint8_t *item_emb_mask, const float *const *params_in, int64_t n_params,
                                 float *const *params_out, float *const *moments_out, gorse_b200_fm_trials_progress_fn progress,
                                 void *user, gorse_b200_fm_fit_result *results);

/* Ranker GAUC: the AFM half of `gorse-bench reranker` after the fit (EvaluateAFM, cmd/gorse-bench/main.go:125-207) -- how
 * an operator weighs the factorization-machine ranker against an LLM reranker.
 *   The model as gorse_b200_fm_create takes it (n_features .. n_params, the same limits); the test rows as
 *   gorse_b200_fm_fit_emb takes them: CSR test_off[n_test + 1] (from 0) / test_idx / test_val (values already through
 *   fm.Scalers), test_target[n_test], test_emb_row[n_test] (may be NULL without slots) and the bf16 item-embedding table
 *   item_emb / item_emb_mask over n_emb_rows rows.
 *   Per user: feedback_count[n_users] = the training rows with target > 0 whose first index is the user (main.go:133-140),
 *   context_size = the config's recommend.context_size (default 100).  The user of test row r is test_idx[test_off[r]];
 *   a row without features, or a user outside [0, n_users), is GORSE_B200_ERR_ARG.
 * What runs: BatchInternalPredict (fm.go:156-178) on every test row as one list in test order, padded to
 *   D = max(num_dimension, the longest test row), in chunks of batch_size rows whose softmax couples the chunk's rows
 *   (DESIGN §8.4); these are not the predictions of the positive / negative lists of the fit's evaluation.  Then per user
 *   with P > 0 positive (target > 0) and N > 0 negative rows and 0 < feedback_count <= context_size: AUC(pos, neg)
 *   (model/ctr/evaluator.go:136-153) -- the negatives strictly below each positive (-0 == +0), summed as a float32 chain
 *   over the positives in ascending order, divided by float32(P N).  GAUC = float64(sum / count) with sum += AUC
 *   float32(P + N) and count += float32(P + N) in float32, unfused; 0 when no user is scored.  The reference visits the
 *   users in Go map order, which varies from run to run: here they are visited in ascending user index.  A user with a
 *   NaN prediction gets AUC = NaN (the reference's sort order with NaN is unpinned), which makes GAUC NaN.
 *   Outputs: pred_out[n_test] (may be NULL) the predictions in test order, bit-identical to the project's CPU restatement;
 *   per scored user in ascending user order, each array sized for n_users and each may be NULL: user_out, feedback_out
 *   (feedback_count), cand_out (P + N), auc_out; *n_scored_out and *gauc_out (not NULL); stats_out[5] (may be NULL):
 *   rows, users with rows, scored users, users summed by the sequential chain (P N > 2^24), scored users with a NaN
 *   prediction.
 * Every argument is checked on the host before the device is touched, ctx last, with gorse_b200_fm_fit's index and float32
 * rounding checks.  n_test >= 2^31 is GORSE_B200_ERR_UNSUPPORTED.  The call keeps no state. */
int32_t gorse_b200_fm_gauc(gorse_b200_ctx *ctx, int64_t n_features, int32_t n_factors, int32_t num_dimension, int32_t batch_size,
                           int32_t n_emb, const int32_t *emb_dim, const float *params, int64_t n_params, int64_t n_test,
                           const int64_t *test_off, const int32_t *test_idx, const float *test_val, const float *test_target,
                           const int32_t *test_emb_row, int64_t n_emb_rows, const uint16_t *const *item_emb,
                           const uint8_t *item_emb_mask, int64_t n_users, const int64_t *feedback_count, int64_t context_size,
                           float *pred_out, int32_t *user_out, int64_t *feedback_out, int64_t *cand_out, float *auc_out,
                           int64_t *n_scored_out, double *gauc_out, int64_t *stats_out);

/* ------------------------------------------------------------------------------------------
 * Embedding evaluation: `gorse-bench embedding`'s scoring (EvaluateEmbedding, cmd/gorse-bench/main.go:322-467) for every test
 * user in one call -- how an operator picks the embedding behind an "embedding" item-to-item recommender.
 *   emb[n_items x dim] fp32 as the column expression returns it (no bf16 truncation); emb_mask[n_items] 1 where the item has
 *   an embedding (NULL: every item has one).  dim outside [1, 16384]: GORSE_B200_ERR_ARG.  A non-finite value in a present
 *   row is GORSE_B200_ERR_ARG (the reference would push NaN into its heap); it is found on the device before anything is scored.
 *   Per user u, as CSRs over [n_users] (offsets non-decreasing, need not start at 0; the items pointer points at the entry
 *   off[0] refers to; every id in [0, n_items)):
 *     shot_off / shot_items   the train side of dataset.SplitLatest(shots): newest first, the order the totals are formed in;
 *     test_off / test_items   the test side (the newest item);
 *     excl_off / excl_items   the user's whole dataset feedback, what the cached negatives exclude (SampleUserNegatives called
 *                             on the full dataset, main.go:517-518); read only when neg_off is NULL;
 *     neg_off / neg_items     the negatives; NULL: n_candidates distinct items outside test(u) and excl(u) are sampled on the
 *                             device under `seed`, or all remaining items ascending when fewer are left, exactly as
 *                             gorse_b200_eval_create samples them (the Go math/rand stream is not reproducible, SURVEY F9).
 *   Per user (main.go:410-456): skipped without a test item or a shot; candidates = test(u) then negatives(u), a candidate
 *   without an embedding skipped; total = 0, then total -= floats.Euclidean(candidate, shot) in fp32 for every shot with an
 *   embedding, in shot order; a candidate enters TopKFilter(topk) only when some shot had an embedding; a user whose filter
 *   stays empty is skipped; else NDCG, Precision and Recall of the ranked list against the set of test items.  Every distance
 *   is bit for bit the reference's AVX-512 Euclidean and every total its sequential sum.
 *   out[3] = {NDCG, Precision, Recall}: the per-user values summed in fp32 in user order (the reference with jobs = 1; with
 *   more jobs its summation order is unpinned), each divided by the number of scored users; all zero when no user is scored.
 *   *users_out (may be NULL) = that number.
 *   Bounds: topk in [1, 128] (GORSE_B200_ERR_ARG).  A user's distances are held at once: (|test(u)| + its negatives, or
 *   n_candidates when sampling) x (its shots with an embedding) above 2^28 is GORSE_B200_ERR_UNSUPPORTED.  Users run in
 *   chunks of at most 2^26 distances (or one user's); the answer does not depend on the chunking.
 *   Every argument is checked on the host before the device is touched, ctx last.  Thread-safe per context: the call keeps
 *   no state and frees its device buffers before it returns. */
int32_t gorse_b200_embedding_eval(gorse_b200_ctx *ctx, int32_t n_items, int32_t dim, const float *emb, const uint8_t *emb_mask,
                                  int64_t n_users, const int64_t *shot_off, const int32_t *shot_items, const int64_t *test_off,
                                  const int32_t *test_items, const int64_t *excl_off, const int32_t *excl_items,
                                  const int64_t *neg_off, const int32_t *neg_items, int32_t n_candidates, uint64_t seed,
                                  int32_t topk, float *out, int64_t *users_out);

/* ------------------------------------------------------------------------------------------
 * NCF-format datasets: dataset.LoadDataFromBuiltIn (dataset/dataset.go:398-490), the loader `gorse-bench cf`
 * (gorse_b200/csrc/gorse_bench_cf.cpp; BASELINE configs[0]) feeds the model with.  Host code.
 *   train file  "user<TAB>item[<TAB>...]" per line (loadTrain :420-453)
 *   test file   "(user,item)<TAB>neg<TAB>neg..." per line (loadTest :455-490), may be NULL
 * gorse_b200_ncf_get fills CSR arrays sized from gorse_b200_ncf_shape (offsets n_users + 1); any pointer may be NULL.
 * ---------------------------------------------------------------------------------------- */
typedef struct gorse_b200_ncf gorse_b200_ncf;
int32_t gorse_b200_ncf_load(const char *train_path, const char *test_path, gorse_b200_ncf **out);
int32_t gorse_b200_ncf_shape(const gorse_b200_ncf *d, int32_t *n_users, int32_t *n_items, int64_t *n_train, int64_t *n_test, int64_t *n_neg);
int32_t gorse_b200_ncf_get(const gorse_b200_ncf *d, int64_t *train_off, int32_t *train_items, int64_t *test_off, int32_t *test_items,
                           int64_t *neg_off, int32_t *neg_items);
int32_t gorse_b200_ncf_free(gorse_b200_ncf *d);

#ifdef __cplusplus
}
#endif
#endif /* GORSE_B200_H */
