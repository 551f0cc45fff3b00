/*
 * embedding_oracle.c -- CPU restatement of `gorse-bench embedding`'s scoring.  TEST INFRASTRUCTURE ONLY.
 *
 * EvaluateEmbedding (cmd/gorse-bench/main.go:403-465) with jobs = 1, built only from the general oracle's pinned
 * primitives (oracle/gorse_oracle.h): gbo_euclidean (floats.Euclidean, the AVX-512 order), gbo_topk_filter (TopKFilter)
 * and gbo_ndcg / gbo_precision / gbo_recall (cf.NDCG / Precision / Recall).  It checks gorse_b200_embedding_eval.
 * Compiled with -ffp-contract=off: every subtraction and addition rounds to fp32 on its own, as Go's do.
 */
#include <stdint.h>
#include <stdlib.h>

#include "../oracle/gorse_oracle.h"

/* the shot lists are shot_off / shot_items (newest first), the test lists test_off / test_items and the negatives
 * neg_off / neg_items, each a CSR over n_users from 0; mask[n_items] (NULL: every item has an embedding).  out[3] = NDCG,
 * Precision, Recall; returns the number of users scored. */
int64_t gbo_evaluate_embedding(int32_t n_items, int32_t dim, const float *emb, const uint8_t *mask, int32_t n_users,
                               const int64_t *shot_off, const int32_t *shot_items, const int64_t *test_off, const int32_t *test_items,
                               const int64_t *neg_off, const int32_t *neg_items, int32_t topk, float out[3])
{
    (void)n_items;
    float ndcg = 0, precision = 0, recall = 0, count = 0;
    int64_t users = 0, maxc = 1;
    for (int32_t u = 0; u < n_users; u++) {
        int64_t c = (test_off[u + 1] - test_off[u]) + (neg_off[u + 1] - neg_off[u]);
        if (c > maxc) maxc = c;
    }
    int32_t *values = (int32_t *)malloc(sizeof(int32_t) * (size_t)maxc);
    float *weights = (float *)malloc(sizeof(float) * (size_t)maxc);
    int32_t *rank = (int32_t *)malloc(sizeof(int32_t) * (size_t)topk);
    for (int32_t u = 0; u < n_users; u++) {
        const int32_t *target = test_items + test_off[u];
        const int32_t nt = (int32_t)(test_off[u + 1] - test_off[u]);
        if (nt == 0) continue;                                       /* :412-414 */
        const int64_t nshot = shot_off[u + 1] - shot_off[u];
        if (nshot == 0) continue;                                    /* :423-425 */
        int64_t n = 0;
        const int64_t nc = nt + (neg_off[u + 1] - neg_off[u]);
        for (int64_t a = 0; a < nc; a++) {                           /* candidates = test ++ negatives, :416-418 */
            const int32_t c = a < nt ? target[a] : neg_items[neg_off[u] + (a - nt)];
            if (mask && !mask[c]) continue;                          /* :430-432 */
            float total = 0;
            int valid = 0;
            for (int64_t b = 0; b < nshot; b++) {                    /* :433-441 */
                const int32_t s = shot_items[shot_off[u] + b];
                if (mask && !mask[s]) continue;
                total = total - gbo_euclidean(emb + (int64_t)c * dim, emb + (int64_t)s * dim, dim);
                valid++;
            }
            if (valid > 0) { values[n] = c; weights[n] = total; n++; }
        }
        const int32_t nr = gbo_topk_filter(values, weights, n, topk, rank, NULL);
        if (nr == 0) continue;                                       /* :446-448 */
        ndcg = ndcg + gbo_ndcg(target, nt, rank, nr);                /* :450-454 */
        precision = precision + gbo_precision(target, nt, rank, nr);
        recall = recall + gbo_recall(target, nt, rank, nr);
        count = count + 1;
        users++;
    }
    out[0] = out[1] = out[2] = 0;
    if (count > 0) { out[0] = ndcg / count; out[1] = precision / count; out[2] = recall / count; }   /* :457-464 */
    free(values); free(weights); free(rank);
    return users;
}
