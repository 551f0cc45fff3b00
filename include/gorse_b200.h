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
/* one epoch = n_steps fused sample-gather-dot-sigmoid-scatter steps in ONE kernel launch
 * (n_steps = trainSet.CountFeedback(), model/cf/model.go:448).  In a distributed context each
 * rank runs n_steps/world steps on its user shard, then item-factor deltas are all-reduced. */
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
 * out[(q - q0) * N + x] (what the candidate sweep thresholds; small problems only) */
int32_t gorse_b200_index_stage1_scores(gorse_b200_index *ix, int64_t q0, int64_t q1, float *out);


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
 * best first, count_out[nq]; score = dot (Dot) or the NEGATED distance (Euclidean, Cosine) -- higher is more similar
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
