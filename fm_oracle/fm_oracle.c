/* fm_oracle.c -- CPU restatement of the reference's factorization-machine inference (model/ctr/fm.go), the checker of
 * the batched FM ranker (gorse_b200_fm_rank).  TEST INFRASTRUCTURE ONLY: the product never links it.
 *
 * It follows the reference tensor op by tensor op, in the reference's order:
 *   AFM.BatchPredict (fm.go:180-229)        features of a (user, item) pair: user id, item id, user labels, item labels
 *   BatchInternalPredict / convertToTensors  every row of one call padded to D = max(numDimension, longest row) with
 *     (fm.go:156-178, 527-577)             index 0, value 0; indices stored as float32; chunks of batchSize rows
 *   AFM.Forward (fm.go:111-134)             vx = V^T x, ((linear + 0.5 sum(vx^2 - (V^2)^T x^2)) + B) + <vx, enc_s> per slot
 *   Attention (common/nn/layers.go:180-185) Mul(Softmax(MatMul(ReLU(e AW + Ab), H), 1), e), then E: . EW + Eb
 *   Softmax (common/nn/op.go:760-767)       subtracts x.max(1, true) and divides by y.sum(1, true) through Tensor.sub /
 *                                            Tensor.div, which index the [B, 1] tensor with i % B (tensor.go:328-379): element
 *                                            (r, c) of a chunk uses row (r dim + c) % B's max and sum.  fmo_softmax with
 *                                            coupled = 0 is the textbook row-wise softmax, kept only to show the difference.
 * Arithmetic: floats.MM (_mm512_mm, common/floats/src/floats_avx512.c:443-480; the committed Go assembly fuses every
 * update, vfmadd231ss / vfmadd231ps) is a fused chain over the contracted index from +0 -- fmaf here -- except x y^T, which
 * assigns floats.Dot (lane accumulators and a reduce tree, fmo_dot) to every element; Tensor.square is
 * _mm512_mul_to; Tensor.add with a scalar is _mm512_add_const, otherwise floats.Add (a Go loop); everything else is a
 * plain float32 operation.  Go's max(a, b) propagates NaN and orders -0 below +0.  Build: -ffp-contract=off. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../gorse_b200/csrc/fm_exp.h"

/* ---- the floats kernels the forward uses ------------------------------------------------------------------------- */
/* the dot of two contiguous vectors (floats_avx512.c:306-367): 16 lane accumulators (a product, then fused updates), a
 * fixed reduce tree, one 8-lane block of unfused products through its own tree, then a fused scalar tail */
float fmo_dot(const float *a, const float *b, int64_t n)
{
    const int64_t epoch = n / 16;
    int64_t remain = n % 16;
    float s[16], r8[8], r4[4];
    for (int l = 0; l < 16; l++) s[l] = epoch > 0 ? a[l] * b[l] : 0.0f;
    for (int64_t c = 1; c < epoch; c++)
        for (int l = 0; l < 16; l++) s[l] = fmaf(a[16 * c + l], b[16 * c + l], s[l]);
    for (int l = 0; l < 8; l++) r8[l] = s[l + 8] + s[l];
    for (int l = 0; l < 4; l++) r4[l] = r8[l + 4] + r8[l];
    float sum = (r4[0] + r4[2]) + (r4[1] + r4[3]);
    a += 16 * epoch;
    b += 16 * epoch;
    if (remain >= 8) {
        for (int l = 0; l < 4; l++) r4[l] = a[l + 4] * b[l + 4] + a[l] * b[l];
        sum = sum + ((r4[0] + r4[2]) + (r4[1] + r4[3]));
        a += 8;
        b += 8;
        remain -= 8;
    }
    for (int64_t i = 0; i < remain; i++) sum = fmaf(a[i], b[i], sum);
    return sum;
}

void fmo_mm(int transA, int transB, int64_t m, int64_t n, int64_t k, const float *a, int64_t lda, const float *b, int64_t ldb,
            float *c, int64_t ldc)
{
    if (!transA && transB) { /* c = dot(row of a, row of b): assigned, not accumulated (floats_avx512.c:454-460) */
        for (int64_t i = 0; i < m; i++)
            for (int64_t j = 0; j < n; j++) c[i * ldc + j] = fmo_dot(a + i * lda, b + j * ldb, k);
        return;
    }
    for (int64_t i = 0; i < m; i++)
        for (int64_t l = 0; l < k; l++)
            for (int64_t j = 0; j < n; j++) {
                const float av = transA ? a[l * lda + i] : a[i * lda + l];
                const float bv = transB ? b[j * ldb + l] : b[l * ldb + j];
                c[i * ldc + j] = fmaf(av, bv, c[i * ldc + j]);
            }
}

void fmo_mul_to(const float *a, const float *b, float *c, int64_t n)
{
    for (int64_t i = 0; i < n; i++) c[i] = a[i] * b[i];
}

void fmo_add_const(float *a, float c, int64_t n)
{
    for (int64_t i = 0; i < n; i++) a[i] += c;
}

static float go_max(float a, float b)
{
    if (a != a) return a;
    if (b != b) return b;
    if (a == b) { /* equal values; for zeros the result is +0 unless both are -0 */
        uint32_t x, y;
        memcpy(&x, &a, 4);
        memcpy(&y, &b, 4);
        x &= y;
        memcpy(&a, &x, 4);
        return a;
    }
    return a > b ? a : b;
}

float fmo_exp(float x) { return fmx_expf(x); }

/* Softmax(x, 1) of a [B, dim] tensor in place; coupled = 1 is the reference's, 0 the row-wise one */
void fmo_softmax(float *y, int64_t B, int64_t dim, int coupled)
{
    float *mx = malloc(sizeof(float) * (size_t)B), *sm = malloc(sizeof(float) * (size_t)B);
    for (int64_t r = 0; r < B; r++) {
        float m = y[r * dim];
        for (int64_t c = 1; c < dim; c++) m = go_max(m, y[r * dim + c]);
        mx[r] = m;
    }
    for (int64_t i = 0; i < B * dim; i++) y[i] -= mx[coupled ? i % B : i / dim];
    for (int64_t i = 0; i < B * dim; i++) y[i] = fmx_expf(y[i]);
    for (int64_t r = 0; r < B; r++) {
        float s = y[r * dim];
        for (int64_t c = 1; c < dim; c++) s += y[r * dim + c];
        sm[r] = s;
    }
    for (int64_t i = 0; i < B * dim; i++) y[i] /= sm[coupled ? i % B : i / dim];
    free(mx);
    free(sm);
}

/* ---- the model --------------------------------------------------------------------------------------------------- */
typedef struct {
    int64_t n_features;
    int32_t k, n_emb;
    const int32_t *dim;
    const float *Bias, *V, *W;
    const float *H[8], *AW[8], *Ab[8], *EW[8], *Eb[8];
} fm_t;

static int fm_bind(fm_t *m, int64_t n_features, int32_t k, int32_t n_emb, const int32_t *dim, const float *params)
{
    if (n_emb > 8) return -1;
    m->n_features = n_features;
    m->k = k;
    m->n_emb = n_emb;
    m->dim = dim;
    const float *p = params;
    m->Bias = p; p += 1;
    m->V = p; p += n_features * k;
    m->W = p; p += n_features;
    for (int s = 0; s < n_emb; s++) {
        const int64_t d = dim[s];
        m->H[s] = p; p += k * d;
        m->AW[s] = p; p += d * k;
        m->Ab[s] = p; p += k;
        m->EW[s] = p; p += d * k;
        m->Eb[s] = p; p += k;
    }
    return 0;
}

/* Attention then E on a chunk: enc[B x k] */
static void encode(const fm_t *m, int s, const float *e, int64_t B, int coupled, float *enc)
{
    const int64_t k = m->k, d = m->dim[s];
    float *h = calloc((size_t)(B * k), sizeof(float)), *z = calloc((size_t)(B * d), sizeof(float));
    fmo_mm(0, 0, B, k, d, e, d, m->AW[s], k, h, k);
    for (int64_t i = 0; i < B * k; i++) h[i] += m->Ab[s][i % k];   /* Tensor.add: floats.Add per row */
    for (int64_t i = 0; i < B * k; i++) h[i] = go_max(h[i], 0.0f); /* ReLU: Tensor.maximum(0) */
    fmo_mm(0, 0, B, d, k, h, k, m->H[s], d, z, d);
    fmo_softmax(z, B, d, coupled);
    for (int64_t i = 0; i < B * d; i++) z[i] *= e[i];              /* Mul(softmax, x) */
    memset(enc, 0, sizeof(float) * (size_t)(B * k));
    fmo_mm(0, 0, B, k, d, z, d, m->EW[s], k, enc, k);
    for (int64_t i = 0; i < B * k; i++) enc[i] += m->Eb[s][i % k];
    free(h);
    free(z);
}

/* AFM.Forward on one chunk of B rows of D features: idx / val [B x D] (indices as float32), emb[s] [B x dim_s] */
static void forward(const fm_t *m, const float *idx, const float *val, float *const *emb, int64_t B, int64_t D, int coupled,
                    float *out)
{
    const int64_t k = m->k;
    float *v = malloc(sizeof(float) * (size_t)(B * D * k)), *e2 = malloc(sizeof(float) * (size_t)(B * D * k));
    float *x2 = malloc(sizeof(float) * (size_t)(B * D)), *w = malloc(sizeof(float) * (size_t)(B * D));
    float *vx = calloc((size_t)(B * k), sizeof(float)), *ss = calloc((size_t)(B * k), sizeof(float));
    float *sq = malloc(sizeof(float) * (size_t)(B * k)), *sum = calloc((size_t)B, sizeof(float));
    float *lin = calloc((size_t)B, sizeof(float)), *enc = malloc(sizeof(float) * (size_t)(B * k));
    float *dot = malloc(sizeof(float) * (size_t)B);
    for (int64_t i = 0; i < B * D; i++) { /* Embedding: row (int)index */
        const int64_t r = (int64_t)idx[i];
        memcpy(v + i * k, m->V + r * k, sizeof(float) * (size_t)k);
        w[i] = m->W[r];
    }
    for (int64_t b = 0; b < B; b++) fmo_mm(1, 0, k, 1, D, v + b * D * k, k, val + b * D, 1, vx + b * k, 1);
    fmo_mul_to(vx, vx, sq, B * k);
    fmo_mul_to(v, v, e2, B * D * k);
    fmo_mul_to(val, val, x2, B * D);
    for (int64_t b = 0; b < B; b++) fmo_mm(1, 0, k, 1, D, e2 + b * D * k, k, x2 + b * D, 1, ss + b * k, 1);
    for (int64_t i = 0; i < B * k; i++) sq[i] -= ss[i];
    for (int64_t b = 0; b < B; b++)
        for (int64_t f = 0; f < k; f++) sum[b] += sq[b * k + f];
    for (int64_t b = 0; b < B; b++) sum[b] *= 0.5f;
    for (int64_t b = 0; b < B; b++) fmo_mm(1, 0, 1, 1, D, w + b * D, 1, val + b * D, 1, lin + b, 1);
    for (int64_t b = 0; b < B; b++) lin[b] += sum[b];
    fmo_add_const(lin, m->Bias[0], B);
    for (int s = 0; s < m->n_emb; s++) {
        encode(m, s, emb[s], B, coupled, enc);
        memset(dot, 0, sizeof(float) * (size_t)B);
        for (int64_t b = 0; b < B; b++) fmo_mm(1, 0, 1, 1, k, vx + b * k, 1, enc + b * k, 1, dot + b, 1);
        for (int64_t b = 0; b < B; b++) lin[b] += dot[b];
    }
    memcpy(out, lin, sizeof(float) * (size_t)B);
    free(v); free(e2); free(x2); free(w); free(vx); free(ss); free(sq); free(sum); free(lin); free(enc); free(dot);
}

/* BatchInternalPredict on already-built rows: row i has len[i] features idx / val at off[i]; emb[s] [n x dim_s] float */
int32_t fmo_batch_predict(int64_t n_features, int32_t k, int32_t num_dimension, int32_t batch_size, int32_t n_emb, const int32_t *dim,
                          const float *params, int64_t n, const int64_t *off, const int32_t *idx, const float *val,
                          float *const *emb, int32_t coupled, float *out)
{
    fm_t m;
    if (fm_bind(&m, n_features, k, n_emb, dim, params) != 0 || batch_size <= 0) return -1;
    int64_t D = num_dimension;
    for (int64_t i = 0; i < n; i++)
        if (off[i + 1] - off[i] > D) D = off[i + 1] - off[i];
    float *fi = calloc((size_t)(n * D) + 1, sizeof(float)), *fv = calloc((size_t)(n * D) + 1, sizeof(float));
    for (int64_t i = 0; i < n; i++)
        for (int64_t j = off[i]; j < off[i + 1]; j++) {
            fi[i * D + j - off[i]] = (float)idx[j];
            fv[i * D + j - off[i]] = val[j];
        }
    float *es[8];
    for (int64_t a = 0; a < n; a += batch_size) {
        const int64_t b = a + batch_size < n ? a + batch_size : n;
        for (int s = 0; s < n_emb; s++) es[s] = emb[s] + a * dim[s];
        forward(&m, fi + a * D, fv + a * D, es, b - a, D, coupled, out + a);
    }
    free(fi);
    free(fv);
    return 0;
}

/* the ranked order of a user's scores: descending, exact ties (-0 == +0) by position, NaN last -- what the library
 * documents (the reference's sort.Slice is not stable, so its order on ties is unpinned) */
static uint64_t rank_key(float s, uint32_t pos)
{
    uint32_t b;
    memcpy(&b, &s, 4);
    uint32_t hi;
    if (s != s) hi = 0xffffffffu;
    else {
        if (s == 0.0f) b = 0;
        const uint32_t ord = (b & 0x80000000u) ? ~b : (b | 0x80000000u);
        hi = ~ord;
    }
    return ((uint64_t)hi << 32) | pos;
}

static int cmp_u64(const void *a, const void *b)
{
    const uint64_t x = *(const uint64_t *)a, y = *(const uint64_t *)b;
    return x < y ? -1 : x > y;
}

/* gorse_b200_fm_rank's factored input, restated one user at a time as the worker calls BatchPredict (the arguments are
 * those of include/gorse_b200.h; they are assumed valid).  item_emb[s]: [n_items x dim_s] bf16 bits. */
int32_t fmo_rank(int64_t n_features, int32_t k, int32_t num_dimension, int32_t batch_size, int32_t n_emb, const int32_t *dim,
                 const float *params, int64_t n_users, const int32_t *user_feat, const int64_t *user_lab_off, const int32_t *user_lab_idx,
                 const float *user_lab_val, int64_t n_items, const int32_t *item_feat, const int64_t *item_lab_off,
                 const int32_t *item_lab_idx, const float *item_lab_val, const uint16_t *const *item_emb, const uint8_t *item_emb_mask,
                 const int64_t *cand_off, const int32_t *cand_items, int32_t coupled, float *scores_out, int32_t *order_out)
{
    (void)n_items;
    for (int64_t u = 0; u < n_users; u++) {
        const int64_t c0 = cand_off[u], n = cand_off[u + 1] - c0;
        if (n == 0) continue;
        const int64_t nul = user_lab_off[u + 1] - user_lab_off[u];
        int64_t cap = 0;
        for (int64_t t = 0; t < n; t++) {
            const int32_t it = cand_items[c0 + t];
            cap += 2 + nul + item_lab_off[it + 1] - item_lab_off[it];
        }
        int64_t *off = malloc(sizeof(int64_t) * (size_t)(n + 1));
        int32_t *ix = malloc(sizeof(int32_t) * (size_t)cap + 4);
        float *vl = malloc(sizeof(float) * (size_t)cap + 4);
        float *emb[8];
        off[0] = 0;
        int64_t p = 0;
        for (int64_t t = 0; t < n; t++) {
            const int32_t it = cand_items[c0 + t];
            if (user_feat[u] >= 0) { ix[p] = user_feat[u]; vl[p++] = 1.0f; }
            if (item_feat[it] >= 0) { ix[p] = item_feat[it]; vl[p++] = 1.0f; }
            for (int64_t j = user_lab_off[u]; j < user_lab_off[u + 1]; j++) { ix[p] = user_lab_idx[j]; vl[p++] = user_lab_val[j]; }
            for (int64_t j = item_lab_off[it]; j < item_lab_off[it + 1]; j++) { ix[p] = item_lab_idx[j]; vl[p++] = item_lab_val[j]; }
            off[t + 1] = p;
        }
        for (int s = 0; s < n_emb; s++) {
            const int64_t d = dim[s];
            emb[s] = calloc((size_t)(n * d), sizeof(float));
            for (int64_t t = 0; t < n; t++) {
                const int32_t it = cand_items[c0 + t];
                if (!item_emb_mask[(int64_t)it * n_emb + s]) continue;
                for (int64_t c = 0; c < d; c++) {
                    const uint32_t bits = (uint32_t)item_emb[s][(int64_t)it * d + c] << 16;
                    memcpy(&emb[s][t * d + c], &bits, 4);
                }
            }
        }
        if (fmo_batch_predict(n_features, k, num_dimension, batch_size, n_emb, dim, params, n, off, ix, vl, emb, coupled,
                              scores_out + c0) != 0)
            return -1;
        uint64_t *key = malloc(sizeof(uint64_t) * (size_t)n);
        for (int64_t t = 0; t < n; t++) key[t] = rank_key(scores_out[c0 + t], (uint32_t)t);
        qsort(key, (size_t)n, sizeof(uint64_t), cmp_u64);
        for (int64_t t = 0; t < n; t++) order_out[c0 + t] = (int32_t)(key[t] & 0xffffffffu);
        for (int s = 0; s < n_emb; s++) free(emb[s]);
        free(key); free(off); free(ix); free(vl);
    }
    return 0;
}
