/* fm_fit_oracle.c -- CPU restatement of the reference's FM training (AFM.Fit, model/ctr/fm.go:307-417) for models without
 * item-embedding slots (fmf_fit, the checker of gorse_b200_fm_fit) and with them (fmf_fit_emb, the checker of
 * gorse_b200_fm_fit_emb).  TEST INFRASTRUCTURE ONLY: the product never links it.
 *
 * It restates this one model's graph, not a general autograd:
 *   forward   (fm.go:111-134)  the floats.MM chains of fm_oracle.c's forward, per row of a batch of padded rows
 *   loss      BCEWithLogits (common/nn/functions.go:218-243): Mean(ReLU(p) - p (t + 1) / 2 + Log(1 + Exp(-|p|)))
 *   backward  Tensor.Backward (tensor.go:267-291) pops the ops from a container/heap ordered by generation; a tensor with
 *             several consumers is assigned the first gradient and adds the later ones.  The logit p has three consumers
 *             (ReLU, Mul, Abs); fmf_p_order replays that heap over this graph's ops to find the order of their
 *             gradients.  v = V[idx] has two (BMM, Square), whose two terms add the same in either order.
 *   Embedding dw = Zeros, then dw[idx] += dy over the batch's positions in row-major order (op.go:687-701)
 *   optimiser Adam (optimizers.go:118-156) or SGD (:70-84) over every element of B, V and W, each a sequence of floats
 *             kernels whose fusing depends on the element's place in its tensor (mul_const_add[_to]: the 16-lane body
 *             and the scalar tail fuse, the 8-lane block rounds twice; floats_avx512.c:18-80)
 *   Evaluate  EvaluateClassification (evaluator.go:46-153): BatchInternalPredict on the positive and the negative test
 *             rows as two lists, float32 counters, AUC as a sequential float32 chain over the sorted positives
 *   Fit       the epoch loop, Verbose / Patience / NaN break, cancellation
 * The scalar Log and Pow are gorse_b200/csrc/fm_fit_math.h, the Exp is fm_exp.h, shared with the kernel.
 * Build: -ffp-contract=off (only the explicit fmaf() calls fuse). */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../gorse_b200/csrc/fm_exp.h"
#include "../gorse_b200/csrc/fm_fit_math.h"

int32_t fmo_batch_predict(int64_t n_features, int32_t k, int32_t num_dimension, int32_t batch_size, int32_t n_emb, const int32_t *dim,
                          const float *params, int64_t n, const int64_t *off, const int32_t *idx, const float *val,
                          float *const *emb, int32_t coupled, float *out);

float fmf_logf(float x) { return fmx_logf(x); }
float fmf_pow_steps(float beta, int64_t t) { return fmx_pow_steps(beta, t); }

/* ---- the backward heap --------------------------------------------------------------------------------------------- */
/* The ops of one training step in creation order (Forward, then BCEWithLogits), each with its generation (1 + the
 * largest generation of its inputs, leaves 0) and the ops producing its inputs (-1: a leaf). */
enum { OP_RELU = 17, OP_MUL = 20, OP_ABS = 21, N_OPS = 29, N_FWD = 16, OP_VX = 2, OP_SQUARE_VX = 3, SLOT_OPS = 12, MAX_SLOTS = 8,
       MAX_OPS = N_OPS + SLOT_OPS * MAX_SLOTS };
static const int op_in[N_OPS][2] = {
    {-1, -1}, /*  0 Embedding(V, idx)          */ {-1, -1}, /*  1 Reshape(values) = x       */
    {0, 1},   /*  2 BMM(v, x) = vx             */ {2, -1},  /*  3 Square(vx)                */
    {0, -1},  /*  4 Square(v)                  */ {1, -1},  /*  5 Square(x)                 */
    {4, 5},   /*  6 BMM(e2, x2)                */ {3, 6},   /*  7 Sub                       */
    {7, -1},  /*  8 Sum(., 1)                  */ {8, -1},  /*  9 Mul(., 0.5)               */
    {-1, -1}, /* 10 Embedding(W, idx)          */ {10, 1},  /* 11 BMM(w, x) = linear        */
    {11, -1}, /* 12 Reshape(linear)            */ {9, -1},  /* 13 Reshape(sum)              */
    {12, 13}, /* 14 Add(linear, sum)           */ {14, -1}, /* 15 Add(., B)                 */
    {15, -1}, /* 16 Flatten = p                */ {16, -1}, /* 17 ReLU(p)                   */
    {-1, -1}, /* 18 Add(target, 1)             */ {18, -1}, /* 19 Div(., 2) = y             */
    {16, 19}, /* 20 Mul(p, y)                  */ {16, -1}, /* 21 Abs(p)                    */
    {21, -1}, /* 22 Neg                        */ {22, -1}, /* 23 Exp                       */
    {23, -1}, /* 24 Add(exp, 1)                */ {24, -1}, /* 25 Log                       */
    {17, 20}, /* 26 Sub(relu, mul)             */ {26, 25}, /* 27 Add(sub, log)             */
    {27, -1}, /* 28 Mean                       */
};

static int g_order_override = 0, g_order[3];
static int g_vx_override = 0, g_vx_order[1 + MAX_SLOTS];

/* container/heap over ops, Less(i, j) = gen[i] > gen[j] (op.go:823-845) */
static int heap_less(const int *h, const int *gen, int i, int j) { return gen[h[i]] > gen[h[j]]; }
static void heap_swap(int *h, int i, int j) { int t = h[i]; h[i] = h[j]; h[j] = t; }
static void heap_up(int *h, const int *gen, int j)
{
    for (;;) {
        int i = (j - 1) / 2; /* Go's division truncates: j = 0 gives i = 0 */
        if (i == j || !heap_less(h, gen, j, i)) break;
        heap_swap(h, i, j);
        j = i;
    }
}
static void heap_down(int *h, const int *gen, int i, int n)
{
    for (;;) {
        int j1 = 2 * i + 1;
        if (j1 >= n || j1 < 0) break;
        int j = j1;
        if (j1 + 1 < n && heap_less(h, gen, j1 + 1, j1)) j = j1 + 1;
        if (!heap_less(h, gen, j, i)) break;
        heap_swap(h, i, j);
        i = j;
    }
}

/* Tensor.Backward's pop order on any graph of up to MAX_OPS ops in creation order (inputs: the producing ops, -1 a leaf),
 * seeded with the last op */
int32_t fmf_heap_order(int32_t n, const int32_t *in, int32_t *out)
{
    if (n < 1 || n > MAX_OPS) return -1;
    int gen[MAX_OPS], h[MAX_OPS], seen[MAX_OPS] = {0}, hn = 0, m = 0;
    for (int o = 0; o < n; o++) {
        int g = 0;
        for (int q = 0; q < 2; q++)
            if (in[2 * o + q] >= 0 && gen[in[2 * o + q]] > g) g = gen[in[2 * o + q]];
        gen[o] = g + 1;
    }
    h[hn++] = n - 1;
    seen[n - 1] = 1;
    while (hn > 0) {
        heap_swap(h, 0, hn - 1); /* heap.Pop: swap the root to the end, fix the rest, take the end */
        heap_down(h, gen, 0, hn - 1);
        const int o = h[--hn];
        out[m++] = o;
        for (int q = 0; q < 2; q++) {
            const int x = in[2 * o + q];
            if (x >= 0 && !seen[x]) {
                h[hn++] = x;
                heap_up(h, gen, hn - 1);
                seen[x] = 1;
            }
        }
    }
    return m;
}

/* The graph with n_emb item-embedding slots (fm.go:128-132): after op 15, per slot in creation order
 *   MatMul(e, AW), Add(., Ab), ReLU, MatMul(., H), Softmax, Mul(., e), MatMul(., EW), Add(., Eb), Reshape, BMM(vx, .), Reshape,
 *   Add(fmOutput, .)
 * then Flatten and the loss.  Tensor.Backward replayed on it gives the order in which ReLU (0), Mul (1) and Abs (2) hand
 * their gradients to p, and the order in which Square (0) and slot s's BMM (1 + s) hand theirs to vx. */
int32_t fmf_backward_order(int32_t n_emb, int32_t *p_out, int32_t *vx_out)
{
    if (n_emb < 0 || n_emb > MAX_SLOTS) return -1;
    int32_t in[MAX_OPS][2];
    int bmm[MAX_SLOTS], n = N_FWD, out = N_FWD - 1, mp = 0, mv = 0;
    for (int o = 0; o < N_FWD; o++) { in[o][0] = op_in[o][0]; in[o][1] = op_in[o][1]; }
    for (int s = 0; s < n_emb; s++) {
        const int b = n;
        in[n][0] = -1; in[n++][1] = -1;
        for (int q = 0; q < 8; q++) { in[n][0] = b + q; in[n++][1] = -1; }
        bmm[s] = n;
        in[n][0] = OP_VX; in[n++][1] = b + 8;
        in[n][0] = b + 9; in[n++][1] = -1;
        in[n][0] = out; in[n++][1] = b + 10;
        out = n - 1;
    }
    const int shift = n - N_FWD;
    for (int o = N_FWD; o < N_OPS; o++, n++)
        for (int q = 0; q < 2; q++) {
            const int x = op_in[o][q];
            in[n][q] = x < 0 ? -1 : x == N_FWD - 1 ? out : x + shift;
        }
    int32_t order[MAX_OPS];
    const int32_t popped = fmf_heap_order(n, &in[0][0], order);
    for (int i = 0; i < popped; i++) {
        const int o = order[i];
        if (o == OP_RELU + shift || o == OP_MUL + shift || o == OP_ABS + shift) p_out[mp++] = o == OP_RELU + shift ? 0 : o == OP_MUL + shift ? 1 : 2;
        if (o == OP_SQUARE_VX) vx_out[mv++] = 0;
        for (int s = 0; s < n_emb; s++) if (o == bmm[s]) vx_out[mv++] = 1 + s;
    }
    return mp == 3 && mv == 1 + n_emb ? 0 : -1;
}

/* the order in which ReLU (0), Mul (1) and Abs (2) hand their gradients to p in the graph without slots */
int32_t fmf_p_order(int32_t *out)
{
    int32_t vx[1];
    return fmf_backward_order(0, out, vx);
}

/* tests only: add p's three gradients, or vx's 1 + n_emb, in another order (NULL: the replayed one) */
void fmf_set_p_order(const int32_t *ord)
{
    g_order_override = ord != NULL;
    if (ord) memcpy(g_order, ord, sizeof g_order);
}
/* tests only: what the alternatives to three pinned rules would give.  1: the softmax backward takes each row's own sum
 * instead of row i % B's; 2: the x0^T dy products walk the batch rows last to first; 4: so do the biases' sums */
enum { ALT_SOFTMAX_ROWWISE = 1, ALT_CONTRACT_REVERSED = 2, ALT_BIAS_REVERSED = 4 };
static int g_alt = 0;
void fmf_set_alternative(int32_t bits) { g_alt = bits; }

void fmf_set_vx_order(const int32_t *ord, int32_t n)
{
    g_vx_override = ord != NULL;
    if (ord) memcpy(g_vx_order, ord, sizeof(int32_t) * (size_t)n);
}

/* ---- floats pieces with the per-index fusing rule -------------------------------------------------------------------- */
static int in_block8(int64_t i, int64_t n)
{
    const int64_t body = (n / 16) * 16;
    return i >= body && n - body >= 8 && i < body + 8;
}
/* MulConstAddTo(a, c, b, dst): dst = a c + b */
static float mca_to(float a, float c, float b, int64_t i, int64_t n)
{
    if (in_block8(i, n)) { float m = a * c; return m + b; }
    return fmaf(a, c, b);
}
/* MulConstAdd(a, c, dst): dst += a c */
static float mca(float a, float c, float dst, int64_t i, int64_t n)
{
    if (in_block8(i, n)) { float m = a * c; return m + dst; }
    return fmaf(a, c, dst);
}

void fmf_mul_const_add_to(const float *a, float c, const float *b, float *dst, int64_t n)
{
    for (int64_t i = 0; i < n; i++) dst[i] = mca_to(a[i], c, b[i], i, n);
}
void fmf_mul_const_add(const float *a, float c, float *dst, int64_t n)
{
    for (int64_t i = 0; i < n; i++) dst[i] = mca(a[i], c, dst[i], i, n);
}

/* one parameter tensor through Adam (optimizers.go:138-151) or SGD (:78-79) */
static void adam_tensor(float *p, float *m, float *v, const float *g, int64_t n, float wd, float c1, float c2, float eps, float lr)
{
    for (int64_t i = 0; i < n; i++) {
        float b1 = mca_to(p[i], wd, g[i], i, n);
        float b2 = b1 - m[i];
        m[i] = mca(b2, c1, m[i], i, n);
        b2 = b1 * b1;
        b2 = b2 - v[i];
        v[i] = mca(b2, c2, v[i], i, n);
        b2 = sqrtf(v[i]);
        b2 = b2 + eps;
        b1 = m[i] / b2;
        p[i] = mca(b1, -lr, p[i], i, n);
    }
}
static void sgd_tensor(float *p, const float *g, int64_t n, float wd, float lr)
{
    for (int64_t i = 0; i < n; i++) {
        const float b = mca_to(p[i], wd, g[i], i, n);
        p[i] = mca(b, -lr, p[i], i, n);
    }
}

static float go_max(float a, float b)
{
    if (a != a) return a;
    if (b != b) return b;
    if (a == b) {
        uint32_t x, y;
        memcpy(&x, &a, 4);
        memcpy(&y, &b, 4);
        x &= y;
        memcpy(&a, &x, 4);
        return a;
    }
    return a > b ? a : b;
}

/* ---- the ops of the graph, as common/nn/op.go forms them ----------------------------------------------------------- */
/* The per-element rules of each op's forward and backward.  train_step below uses exactly these, and fmf_op_* apply them
 * to whole tensors with the reference's broadcasting (the second input's shape a suffix of the first's: element i uses
 * x1[i % n1]), so tests/test_oracle_fm_fit.py can pin them on the known answers of common/nn/op_test.go. */
static float r_add_g1(float acc, float dy) { return acc + dy; }          /* Add: gx1 = Zeros, then += dy (:112-123) */
static float r_sub_g1(float acc, float dy) { return acc - dy; }          /* Sub: gx1 = Zeros, then -= dy (:139-150) */
static float r_mul_g0(float dy, float x1) { return dy * x1; }            /* Mul: gx0 = dy x1 (:166-178) */
static float r_mul_g1(float acc, float dy, float x0) { return acc + dy * x0; }
static float r_div_g0(float dy, float x1) { return dy / x1; }            /* Div (:194-208) */
static float r_div_g1(float acc, float dy, float x0, float x1) { return acc - dy * x0 / x1 / x1; }
static float r_square(float x) { return x * x; }                         /* floats.MulTo(x, x) */
static float r_square_g(float x, float dy) { return (x * dy) * 2.0f; }   /* MulTo(x, dy), MulConst(2) (:267-272) */
static float r_exp(float x) { return fmx_expf(x); }                      /* float32(math.Exp(float64)) */
static float r_exp_g(float x, float dy) { return fmx_expf(x) * dy; }     /* (:319-324) */
static float r_log(float x) { return fmx_logf(x); }                      /* math32.Log */
static float r_log_g(float x, float dy) { return dy / x; }               /* (:340-344) */
static float r_abs(float x) { return x < 0.0f ? -x : x; }                /* (:354-372) */
static float r_abs_g(float x, float dy) { return x < 0.0f ? -dy : dy; }
static float r_neg(float x) { return -x; }
static float r_relu(float x);                                            /* max(x, 0), Go's max */
static float r_relu_g(float x, float dy) { return (x > 0.0f ? 1.0f : 0.0f) * dy; } /* gt(x, 0).mul(dy) (:745-749) */
static float r_mean_g(float dy, int64_t n) { return dy / (float)n; }     /* (:484-490) */
static float r_dot1(float a, float b) { return fmaf(a, b, 0.0f); }       /* floats.MM's transB path: dot of length 1 */

/* ---- one training step --------------------------------------------------------------------------------------------- */
typedef struct {
    int64_t nf;
    int32_t k, D;
    float *P, *M, *Vm;   /* parameters B, V, W and the two Adam moments, one layout */
    float *gV, *gW;      /* [nf x k], [nf] */
    float *vx, *dvx, *g, *dss, *loss;
    /* item-embedding slots: the table as gorse_b200_fm_rank takes it, and per slot the batch's tensors */
    int32_t n_emb, dim[MAX_SLOTS];
    const uint16_t *const *table;
    const uint8_t *mask;
    int64_t slot_off[MAX_SLOTS]; /* of H in P; AW, Ab, EW, Eb follow */
    float *gS;                   /* the slot tensors' gradients, laid out as P from slot_off[0] */
    float *p, *e[MAX_SLOTS], *h[MAX_SLOTS], *hr[MAX_SLOTS], *y[MAX_SLOTS], *att[MAX_SLOTS], *enc[MAX_SLOTS];
    float *denc, *dh, *dbig, *gx, *sumdx; /* scratch: [bs x k], [bs x k], [bs x maxdim], [bs x maxdim], [bs] */
} state_t;

void fmo_mm(int transA, int transB, int64_t m, int64_t n, int64_t k, const float *a, int64_t lda, const float *b, int64_t ldb,
            float *c, int64_t ldc);
void fmo_softmax(float *y, int64_t B, int64_t dim, int coupled);

/* convertToTensors' embedding rows (fm.go:555-561): table row `row` of slot s widened from bf16, zeros when the sample
 * has no item (row < 0) or the item lacks the slot */
static void gather_emb(int32_t n_emb, const int32_t *dim, const uint16_t *const *table, const uint8_t *mask, int s, const int32_t *rows,
                       int64_t n, float *out)
{
    const int64_t d = dim[s];
    for (int64_t i = 0; i < n; i++)
        for (int64_t c = 0; c < d; c++) {
            uint32_t bits = 0;
            if (rows[i] >= 0 && (!mask || mask[(int64_t)rows[i] * n_emb + s])) bits = (uint32_t)table[s][(int64_t)rows[i] * d + c] << 16;
            memcpy(&out[i * d + c], &bits, 4);
        }
}

/* slot s on the batch (layers.go:50-52, 180-185; fm.go:129-131): leaves e, h = e AW + Ab, ReLU(h), the softmax y,
 * att = y e and enc = att EW + Eb, and adds <vx, enc> to every row's logit */
static void slot_forward(state_t *S, int s, const int32_t *rows, int64_t B)
{
    const int64_t k = S->k, d = S->dim[s];
    const float *H = S->P + S->slot_off[s], *AW = H + k * d, *Ab = AW + d * k, *EW = Ab + k, *Eb = EW + d * k;
    float *e = S->e[s], *h = S->h[s], *hr = S->hr[s], *y = S->y[s], *att = S->att[s], *enc = S->enc[s];
    gather_emb(S->n_emb, S->dim, S->table, S->mask, s, rows, B, e);
    memset(h, 0, sizeof(float) * (size_t)(B * k));
    fmo_mm(0, 0, B, k, d, e, d, AW, k, h, k);
    for (int64_t i = 0; i < B * k; i++) { h[i] += Ab[i % k]; hr[i] = r_relu(h[i]); }
    memset(y, 0, sizeof(float) * (size_t)(B * d));
    fmo_mm(0, 0, B, d, k, hr, k, H, d, y, d);
    fmo_softmax(y, B, d, 1);
    for (int64_t i = 0; i < B * d; i++) att[i] = y[i] * e[i];
    memset(enc, 0, sizeof(float) * (size_t)(B * k));
    fmo_mm(0, 0, B, k, d, att, d, EW, k, enc, k);
    for (int64_t i = 0; i < B * k; i++) enc[i] += Eb[i % k];
    for (int64_t b = 0; b < B; b++) {
        float dot = 0.0f;
        fmo_mm(1, 0, 1, 1, k, S->vx + b * k, 1, enc + b * k, 1, &dot, 1);
        S->p[b] += dot;
    }
}

/* Softmax(x, 1)'s backward on the output y [B, dim] for dy (op.go:769-777): gx = y dy, sumdx = gx.sum(1, true) (the first
 * element, then the rest in order), then y.mul(sumdx) and gx.sub(y) through Tensor.mul / Tensor.sub, which index the
 * [B, 1] sums with i % B: two roundings per element.  (y is the live output there and is overwritten; here it is kept.) */
static void softmax_backward(const float *y, const float *dy, int64_t B, int64_t d, int coupled, float *sumdx, float *gx)
{
    for (int64_t i = 0; i < B * d; i++) gx[i] = y[i] * dy[i];
    for (int64_t r = 0; r < B; r++) {
        float sm = gx[r * d];
        for (int64_t c = 1; c < d; c++) sm += gx[r * d + c];
        sumdx[r] = sm;
    }
    for (int64_t i = 0; i < B * d; i++) gx[i] = gx[i] - y[i] * sumdx[coupled ? i % B : i / d];
}

/* forward and backward of Softmax(x, 1) as an op, for the known answers */
void fmf_op_softmax(const float *x, int64_t B, int64_t d, const float *dy, int32_t coupled, float *y, float *gx)
{
    float *sumdx = malloc(sizeof(float) * (size_t)B);
    memcpy(y, x, sizeof(float) * (size_t)(B * d));
    fmo_softmax(y, B, d, coupled);
    softmax_backward(y, dy, B, d, coupled, sumdx, gx);
    free(sumdx);
}

/* dx1 = x0^T dy (op.go:513): c [m x n] = a^T b over the B batch rows, a fused chain in row order (fmo_mm's transA case) */
static void contract_batch(int64_t m, int64_t n, int64_t B, const float *a, const float *b, float *c)
{
    if (!(g_alt & ALT_CONTRACT_REVERSED)) { fmo_mm(1, 0, m, n, B, a, m, b, n, c, n); return; }
    for (int64_t i = 0; i < m; i++)
        for (int64_t l = B - 1; l >= 0; l--)
            for (int64_t j = 0; j < n; j++) c[i * n + j] = fmaf(a[l * m + i], b[l * n + j], c[i * n + j]);
}

/* Add(., bias)'s gx1[i % k] += dy[i] from zeros (op.go:112-123) */
static void bias_backward(const float *dy, int64_t B, int64_t k, float *g)
{
    for (int64_t i = 0; i < B * k; i++) {
        const int64_t j = g_alt & ALT_BIAS_REVERSED ? B * k - 1 - i : i;
        g[j % k] = r_add_g1(g[j % k], dy[j]);
    }
}

/* slot s's backward from the rows' dp = S->g: the gradients of H, AW, Ab, EW, Eb into S->gS.  The gradients towards the
 * input embedding e (Mul's gx1, the attention Linear's dx0) reach no parameter and are not formed. */
static void slot_backward(state_t *S, int s, int64_t B)
{
    const int64_t k = S->k, d = S->dim[s];
    const float *H = S->P + S->slot_off[s], *EW = H + 2 * k * d + k;
    float *gH = S->gS + (S->slot_off[s] - S->slot_off[0]), *gAW = gH + k * d, *gAb = gAW + d * k, *gEW = gAb + k, *gEb = gEW + d * k;
    const float *e = S->e[s], *h = S->h[s], *hr = S->hr[s], *y = S->y[s], *att = S->att[s];
    float *denc = S->denc, *dh = S->dh, *dz = S->dbig, *gx = S->gx;
    memset(gH, 0, sizeof(float) * (size_t)(3 * k * d + 2 * k));
    /* Add(fmOutput, .): 0 + dp; Reshape; BMM(vx, enc): denc = vx dp (op.go:555-559); Reshape; Add(., Eb): a clone, and Eb's
     * gx1[i % k] += dy[i] from zeros (op.go:112-123) */
    for (int64_t b = 0; b < B; b++)
        for (int64_t f = 0; f < k; f++) denc[b * k + f] = fmaf(S->vx[b * k + f], r_add_g1(0.0f, S->g[b]), 0.0f);
    bias_backward(denc, B, k, gEb);
    /* MatMul(att, EW) (op.go:509-513): datt = denc EW^T, dEW = att^T denc */
    fmo_mm(0, 1, B, d, k, denc, k, EW, k, dz, d);
    contract_batch(d, k, B, att, denc, gEW);
    /* Mul(y, e): gx0 = datt e, then the softmax's backward.  Mul's backward, the only other reader of the softmax's live
     * output, has the higher generation and has already run when the softmax overwrites it. */
    for (int64_t i = 0; i < B * d; i++) gx[i] = r_mul_g0(dz[i], e[i]);
    softmax_backward(y, gx, B, d, !(g_alt & ALT_SOFTMAX_ROWWISE), S->sumdx, dz);
    /* MatMul(ReLU(h), H): dReLU = dz H^T, dH = ReLU(h)^T dz; ReLU: gt(h, 0) dy; Add(., Ab); MatMul(e, AW): dAW = e^T dh */
    fmo_mm(0, 1, B, k, d, dz, d, H, d, dh, k);
    contract_batch(k, d, B, hr, dz, gH);
    for (int64_t i = 0; i < B * k; i++) dh[i] = r_relu_g(h[i], dh[i]);
    bias_backward(dh, B, k, gAb);
    contract_batch(d, k, B, e, dh, gAW);
}

static float r_relu(float x) { return go_max(x, 0.0f); }

/* forward of one padded row: p and vx */
static float forward_row(const state_t *S, const float *fi, const float *fv, float *vx)
{
    const int k = S->k, D = S->D;
    const float *V = S->P + 1, *W = S->P + 1 + S->nf * k;
    float ss[32], lin = 0.0f, sum = 0.0f;
    for (int f = 0; f < k; f++) vx[f] = ss[f] = 0.0f;
    for (int l = 0; l < D; l++) {
        const int64_t r = (int64_t)fi[l];
        const float x = fv[l], x2 = r_square(x);
        for (int f = 0; f < k; f++) {
            const float v = V[r * k + f];
            vx[f] = fmaf(v, x, vx[f]);
            ss[f] = fmaf(r_square(v), x2, ss[f]);
        }
        lin = fmaf(W[r], x, lin);
    }
    for (int f = 0; f < k; f++) sum += r_square(vx[f]) - ss[f];
    sum *= 0.5f;
    return (lin + sum) + S->P[0];
}

/* rows [r0, r0 + B) of the padded training set; returns the batch's loss (Mean) */
static float train_step(state_t *S, const float *fi, const float *fv, const float *tgt, const int32_t *emb_row, int64_t r0, int64_t B,
                        int adam, float lr_t, float wd, float sgd_lr)
{
    const int k = S->k, D = S->D, n_emb = S->n_emb;
    const int64_t nf = S->nf;
    int32_t ord[3], vord[1 + MAX_SLOTS];
    fmf_backward_order(n_emb, ord, vord);
    if (g_order_override) memcpy(ord, g_order, sizeof ord);
    if (g_vx_override) memcpy(vord, g_vx_order, sizeof(int32_t) * (size_t)(1 + n_emb));
    for (int64_t b = 0; b < B; b++) S->p[b] = forward_row(S, fi + (r0 + b) * D, fv + (r0 + b) * D, S->vx + b * k);
    for (int s = 0; s < n_emb; s++) slot_forward(S, s, emb_row + r0, B);
    const float mgrad = r_mean_g(1.0f, B); /* Mean's backward of dy = 1 */
    float mean = 0.0f;
    for (int64_t b = 0; b < B; b++) {
        const int64_t row = r0 + b;
        const float *vx = S->vx + b * k;
        const float p = S->p[b];
        const float t = tgt[row];
        const float term1 = r_relu(p);
        const float y = (t + 1.0f) / 2.0f;
        const float term2 = p * y;
        const float na = r_neg(r_abs(p));
        const float E = r_exp(na);
        const float lin_ = E + 1.0f;
        const float loss = (term1 - term2) + r_log(lin_);
        S->loss[b] = loss;
        mean += loss;
        /* backward of the loss: Add -> (Sub: m, Log: 0 + m); Log: dy / x; Exp: exp(x) dy; Neg; Sub -> (ReLU: m, Mul: 0 - m) */
        const float dlog = r_log_g(lin_, r_add_g1(0.0f, mgrad));
        const float dexp = r_exp_g(na, dlog);
        const float dneg = r_neg(dexp);          /* Neg's backward: -dy */
        float c[3];
        c[0] = r_relu_g(p, mgrad);                    /* ReLU */
        c[1] = r_mul_g0(r_sub_g1(0.0f, mgrad), y);   /* Mul(p, y), dy from Sub's second input */
        c[2] = r_abs_g(p, dneg);                      /* Abs */
        const float g = (c[ord[0]] + c[ord[1]]) + c[ord[2]];
        S->g[b] = g;
        /* Add(linear, sum) -> sum: 0 + g; Mul(., 0.5); Sum(., 1); Sub -> (Square(vx): d, BMM(e2, x2): 0 - d); Square: x dy 2 */
        const float dsub = r_mul_g0(r_add_g1(0.0f, g), 0.5f);
        S->dss[b] = r_sub_g1(0.0f, dsub);
        /* vx's gradients in pop order: Square's, and per slot BMM(vx, enc)'s dvx = enc dp^T, a dot of length 1 */
        for (int f = 0; f < k; f++) {
            float acc = 0.0f;
            for (int q = 0; q <= n_emb; q++) {
                const float term = vord[q] == 0 ? r_square_g(vx[f], dsub) : r_dot1(S->enc[vord[q] - 1][b * k + f], r_add_g1(0.0f, g));
                acc = q == 0 ? term : acc + term;
            }
            S->dvx[b * k + f] = acc;
        }
    }
    for (int s = 0; s < n_emb; s++) slot_backward(S, s, B);
    mean /= (float)B;
    /* Embedding backward: zeros, then += in position order */
    memset(S->gV, 0, sizeof(float) * (size_t)(nf * k));
    memset(S->gW, 0, sizeof(float) * (size_t)nf);
    const float *V = S->P + 1;
    for (int64_t b = 0; b < B; b++)
        for (int l = 0; l < D; l++) {
            const int64_t pos = (r0 + b) * D + l, r = (int64_t)fi[pos];
            const float x = fv[pos], x2 = r_square(x);
            for (int f = 0; f < k; f++) {
                const float dv_bmm = r_dot1(x, S->dvx[b * k + f]);                       /* BMM(v, x)'s dv = x dvx^T */
                const float dv_sq = r_square_g(V[r * k + f], r_dot1(x2, S->dss[b]));    /* Square(v) of BMM(e2, x2)'s de2 */
                S->gV[r * k + f] = r_add_g1(S->gV[r * k + f], dv_bmm + dv_sq);          /* Embedding: dw[idx] += dy */
            }
            S->gW[r] = r_add_g1(S->gW[r], r_dot1(x, S->g[b]));                          /* BMM(w, x)'s dw = x dlinear */
        }
    float gB = 0.0f; /* Add(., B)'s backward: the batch sum */
    for (int64_t b = 0; b < B; b++) gB = r_add_g1(gB, S->g[b]);
    const int64_t nV = nf * k;
    float *P = S->P;
    if (adam) {
        const float c1 = 1.0f - 0.9f, c2 = 1.0f - 0.999f, eps = 1e-8f;
        adam_tensor(P, S->M, S->Vm, &gB, 1, wd, c1, c2, eps, lr_t);
        adam_tensor(P + 1, S->M + 1, S->Vm + 1, S->gV, nV, wd, c1, c2, eps, lr_t);
        adam_tensor(P + 1 + nV, S->M + 1 + nV, S->Vm + 1 + nV, S->gW, nf, wd, c1, c2, eps, lr_t);
    } else {
        sgd_tensor(P, &gB, 1, wd, sgd_lr);
        sgd_tensor(P + 1, S->gV, nV, wd, sgd_lr);
        sgd_tensor(P + 1 + nV, S->gW, nf, wd, sgd_lr);
    }
    /* the five tensors of each slot, each with its own length in the fusing rule (AFM.Parameters, fm.go:136-146) */
    for (int s = 0; s < n_emb; s++) {
        const int64_t kd = (int64_t)k * S->dim[s], len[5] = {kd, kd, k, kd, k};
        int64_t o = S->slot_off[s];
        for (int q = 0; q < 5; o += len[q++]) {
            if (adam) adam_tensor(P + o, S->M + o, S->Vm + o, S->gS + (o - S->slot_off[0]), len[q], wd, 1.0f - 0.9f, 1.0f - 0.999f, 1e-8f, lr_t);
            else sgd_tensor(P + o, S->gS + (o - S->slot_off[0]), len[q], wd, sgd_lr);
        }
    }
    return mean;
}

/* ---- whole-tensor ops for the known answers ------------------------------------------------------------------------- */
enum { OPB_ADD, OPB_SUB, OPB_MUL, OPB_DIV };
/* y = x0 op x1 (x1 broadcast over x0 by i % n1), and both gradients for the output gradient dy */
void fmf_op_binary(int32_t op, const float *x0, int64_t n0, const float *x1, int64_t n1, const float *dy, float *y, float *g0, float *g1)
{
    for (int64_t i = 0; i < n1; i++) g1[i] = 0.0f;
    for (int64_t i = 0; i < n0; i++) {
        const float a = x0[i], b = x1[i % n1];
        switch (op) {
        case OPB_ADD: y[i] = a + b; g0[i] = dy[i]; g1[i % n1] = r_add_g1(g1[i % n1], dy[i]); break;
        case OPB_SUB: y[i] = a - b; g0[i] = dy[i]; g1[i % n1] = r_sub_g1(g1[i % n1], dy[i]); break;
        case OPB_MUL: y[i] = a * b; g0[i] = r_mul_g0(dy[i], b); g1[i % n1] = r_mul_g1(g1[i % n1], dy[i], a); break;
        default: y[i] = a / b; g0[i] = r_div_g0(dy[i], b); g1[i % n1] = r_div_g1(g1[i % n1], dy[i], a, b); break;
        }
    }
}

enum { OPU_SQUARE, OPU_EXP, OPU_LOG, OPU_ABS, OPU_RELU, OPU_NEG };
void fmf_op_unary(int32_t op, const float *x, int64_t n, const float *dy, float *y, float *g)
{
    for (int64_t i = 0; i < n; i++) switch (op) {
        case OPU_SQUARE: y[i] = r_square(x[i]); g[i] = r_square_g(x[i], dy[i]); break;
        case OPU_EXP: y[i] = r_exp(x[i]); g[i] = r_exp_g(x[i], dy[i]); break;
        case OPU_LOG: y[i] = r_log(x[i]); g[i] = r_log_g(x[i], dy[i]); break;
        case OPU_ABS: y[i] = r_abs(x[i]); g[i] = r_abs_g(x[i], dy[i]); break;
        case OPU_RELU: y[i] = r_relu(x[i]); g[i] = r_relu_g(x[i], dy[i]); break;
        default: y[i] = r_neg(x[i]); g[i] = r_neg(dy[i]); break;
        }
}

/* Sum (all, :382-397) or Mean (:474-490): y[0] and the gradient for dy[0] */
void fmf_op_sum(int32_t mean, const float *x, int64_t n, float dy, float *y, float *g)
{
    float s = 0.0f;
    for (int64_t i = 0; i < n; i++) s += x[i];
    y[0] = mean ? s / (float)n : s;
    for (int64_t i = 0; i < n; i++) g[i] = mean ? r_mean_g(dy, n) : dy;
}

/* Sum(x, axis) of x squashed to [s1, s2, s3] along s2 (:408-464) */
void fmf_op_sum_axis(const float *x, int64_t s1, int64_t s2, int64_t s3, const float *dy, float *y, float *g)
{
    for (int64_t i = 0; i < s1 * s3; i++) y[i] = 0.0f;
    for (int64_t i = 0; i < s1; i++)
        for (int64_t j = 0; j < s2; j++)
            for (int64_t k = 0; k < s3; k++) {
                y[i * s3 + k] += x[i * s2 * s3 + j * s3 + k];
                g[i * s2 * s3 + j * s3 + k] = dy[i * s3 + k];
            }
}

void fmo_mm(int transA, int transB, int64_t m, int64_t n, int64_t k, const float *a, int64_t lda, const float *b, int64_t ldb,
            float *c, int64_t ldc);

/* Tensor.batchMatMul (tensor.go:550-597) of t [bt, tr, tc] and o [bt, or, oc] into out (zeroed here); returns m, n */
static void tbmm(const float *t, int64_t bt, int64_t tr, int64_t tc, const float *o, int64_t or_, int64_t oc, int t1, int t2, float *out,
                 int64_t *mo, int64_t *no)
{
    const int64_t m = t1 ? tc : tr, n = t2 ? or_ : oc, k = t1 ? tr : tc;
    const int64_t lda = t1 ? m : k, ldb = t2 ? k : n;
    memset(out, 0, sizeof(float) * (size_t)(bt * m * n));
    for (int64_t i = 0; i < bt; i++) fmo_mm(t1, t2, m, n, k, t + i * tr * tc, lda, o + i * or_ * oc, ldb, out + i * m * n, n);
    *mo = m;
    *no = n;
}

/* BMM(x, y, t1, t2) forward and backward (op.go:544-572) */
void fmf_op_bmm(int32_t t1, int32_t t2, int64_t bt, int64_t xr, int64_t xc, int64_t yr, int64_t yc, const float *x, const float *y,
                const float *dz, float *z, float *gx, float *gy)
{
    int64_t m, n, a, b;
    tbmm(x, bt, xr, xc, y, yr, yc, t1, t2, z, &m, &n);
    if (!t1 && !t2) { tbmm(dz, bt, m, n, y, yr, yc, 0, 1, gx, &a, &b); tbmm(x, bt, xr, xc, dz, m, n, 1, 0, gy, &a, &b); }
    else if (t1 && !t2) { tbmm(y, bt, yr, yc, dz, m, n, 0, 1, gx, &a, &b); tbmm(x, bt, xr, xc, dz, m, n, 0, 0, gy, &a, &b); }
    else if (!t1 && t2) { tbmm(dz, bt, m, n, y, yr, yc, 0, 0, gx, &a, &b); tbmm(dz, bt, m, n, x, xr, xc, 1, 0, gy, &a, &b); }
    else { tbmm(y, bt, yr, yc, dz, m, n, 1, 1, gx, &a, &b); tbmm(dz, bt, m, n, x, xr, xc, 1, 1, gy, &a, &b); }
}

/* Embedding(w [rows x dim], idx [n] as float32): y [n x dim], gw = Zeros then += per position (op.go:662-701) */
void fmf_op_embedding(const float *w, int64_t rows, int64_t dim, const float *idx, int64_t n, const float *dy, float *y, float *gw)
{
    for (int64_t i = 0; i < rows * dim; i++) gw[i] = 0.0f;
    for (int64_t i = 0; i < n; i++) {
        const int64_t r = (int64_t)idx[i];
        for (int64_t j = 0; j < dim; j++) {
            y[i * dim + j] = w[r * dim + j];
            gw[r * dim + j] = r_add_g1(gw[r * dim + j], dy[i * dim + j]);
        }
    }
}

/* Broadcast(x [n], w): y [n x w], gx[i] = 0 + the sum of row i of dy (op.go:583-619) */
void fmf_op_broadcast(const float *x, int64_t n, int64_t w, const float *dy, float *y, float *g)
{
    for (int64_t i = 0; i < n; i++) {
        g[i] = 0.0f;
        for (int64_t j = i * w; j < (i + 1) * w; j++) {
            y[j] = x[i];
            g[i] = r_add_g1(g[i], dy[j]);
        }
    }
}

/* ---- Evaluate ------------------------------------------------------------------------------------------------------ */
static int cmp_f32(const void *a, const void *b)
{
    const float x = *(const float *)a, y = *(const float *)b;
    return x < y ? -1 : x > y;
}

/* Precision, Recall, Accuracy, AUC of two prediction lists (evaluator.go:85-153), literally; the lists are sorted in place */
void fmf_metrics(int64_t n_pos, float *pos, int64_t n_neg, float *neg, float *out)
{
    float tp = 0, fp = 0, fn = 0, correct = 0;
    for (int64_t i = 0; i < n_pos; i++) if (pos[i] > 0) tp++;
    for (int64_t i = 0; i < n_neg; i++) if (neg[i] > 0) fp++;
    out[0] = tp + fp == 0 ? 0.0f : tp / (tp + fp);
    tp = 0;
    for (int64_t i = 0; i < n_pos; i++) { if (pos[i] > 0) tp++; else fn++; }
    out[1] = tp + fn == 0 ? 0.0f : tp / (tp + fn);
    for (int64_t i = 0; i < n_pos; i++) if (pos[i] > 0) correct++;
    for (int64_t i = 0; i < n_neg; i++) if (neg[i] < 0) correct++;
    out[2] = n_pos + n_neg == 0 ? 0.0f : correct / (float)(n_pos + n_neg);
    qsort(pos, (size_t)n_pos, sizeof(float), cmp_f32);
    qsort(neg, (size_t)n_neg, sizeof(float), cmp_f32);
    float sum = 0;
    int64_t j = 0;
    for (int64_t i = 0; i < n_pos; i++) {
        while (j < n_neg && neg[j] < pos[i]) j++;
        sum += (float)j;
    }
    out[3] = n_pos * n_neg == 0 ? 0.0f : sum / (float)(n_pos * n_neg);
}

/* the item-embedding side of a fit: dims, the table, and the table row of every training and test sample */
typedef struct {
    int32_t n_emb;
    const int32_t *dim;
    const uint16_t *const *table;
    const uint8_t *mask;
    const int32_t *tr_row, *te_row;
} emb_t;

/* EvaluateClassification on test rows (CSR off / idx / val, targets): out = Precision, Recall, Accuracy, AUC.  With slots
 * each list runs in chunks of batch_size rows with the chunk-coupled softmax (BatchInternalPredict, fm.go:156-178). */
static void evaluate(int64_t nf, int32_t k, int32_t num_dim, int32_t bs, const emb_t *E, const float *P, int64_t n, const int64_t *off,
                     const int32_t *idx, const float *val, const float *tgt, float *out)
{
    memset(out, 0, 4 * sizeof(float));
    if (n == 0) return;
    const int32_t n_emb = E ? E->n_emb : 0;
    float *pred[2];
    int64_t cnt[2] = {0, 0};
    for (int s = 0; s < 2; s++) {
        int64_t rows = 0, ent = 0;
        for (int64_t i = 0; i < n; i++)
            if ((tgt[i] > 0) == (s == 0)) { rows++; ent += off[i + 1] - off[i]; }
        int64_t *o = malloc(sizeof(int64_t) * (size_t)(rows + 1));
        int32_t *ix = malloc(sizeof(int32_t) * (size_t)(ent + 1)), *er = malloc(sizeof(int32_t) * (size_t)(rows + 1));
        float *vl = malloc(sizeof(float) * (size_t)(ent + 1)), *emb[MAX_SLOTS];
        o[0] = 0;
        int64_t r = 0, e = 0;
        for (int64_t i = 0; i < n; i++) {
            if ((tgt[i] > 0) != (s == 0)) continue;
            for (int64_t j = off[i]; j < off[i + 1]; j++, e++) { ix[e] = idx[j]; vl[e] = val[j]; }
            if (n_emb) er[r] = E->te_row[i];
            o[++r] = e;
        }
        for (int q = 0; q < n_emb; q++) {
            emb[q] = malloc(sizeof(float) * (size_t)(rows * E->dim[q] + 1));
            gather_emb(n_emb, E->dim, E->table, E->mask, q, er, rows, emb[q]);
        }
        pred[s] = malloc(sizeof(float) * (size_t)(rows + 1));
        fmo_batch_predict(nf, k, num_dim, n_emb ? bs : 1 << 30, n_emb, n_emb ? E->dim : NULL, P, rows, o, ix, vl, n_emb ? emb : NULL, 1, pred[s]);
        cnt[s] = rows;
        for (int q = 0; q < n_emb; q++) free(emb[q]);
        free(o); free(ix); free(vl); free(er);
    }
    fmf_metrics(cnt[0], pred[0], cnt[1], pred[1], out);
    free(pred[0]);
    free(pred[1]);
}

void fmf_evaluate(int64_t nf, int32_t k, int32_t num_dim, const float *P, int64_t n, const int64_t *off, const int32_t *idx,
                  const float *val, const float *tgt, float *out)
{
    evaluate(nf, k, num_dim, 0, NULL, P, n, off, idx, val, tgt, out);
}

/* ---- Fit ----------------------------------------------------------------------------------------------------------- */
/* ip: n_factors, n_epochs, optimizer (0 Adam, 1 SGD), batch_size, verbose, patience, cancel_epoch (-1: never; the progress
 * callback cancels after that epoch, 0 = after the first evaluation);  fp: lr, reg;  max_steps (0: no limit).
 * res_f: AUC, Precision, Recall, Accuracy, cost;  res_i: epochs_run, best_epoch, early_stopped, diverged, cancelled, steps.
 * moments_out [2 x n_params] may be NULL. */
static int32_t fit(int64_t nf, int32_t num_dim, const int32_t *ip, const float *fp, int64_t max_steps, int64_t n_train, const int64_t *tr_off,
                   const int32_t *tr_idx, const float *tr_val, const float *tr_tgt, int64_t n_test, const int64_t *te_off, const int32_t *te_idx,
                   const float *te_val, const float *te_tgt, const emb_t *E, const float *params_in, float *params_out, float *moments_out,
                   float *res_f, int64_t *res_i)
{
    const int32_t k = ip[0], n_epochs = ip[1], adam = ip[2] == 0, bs = ip[3], verbose = ip[4], patience = ip[5], cancel_epoch = ip[6];
    const float lr = fp[0], reg = fp[1];
    if (k < 1 || k > 32 || bs < 1 || verbose < 1) return -1;
    int64_t n_params = 1 + nf * k + nf, maxdim = 1;
    state_t S;
    memset(&S, 0, sizeof S);
    S.nf = nf;
    S.k = k;
    S.n_emb = E->n_emb;
    S.table = E->table;
    S.mask = E->mask;
    if (S.n_emb < 0 || S.n_emb > MAX_SLOTS) return -1;
    for (int s = 0; s < S.n_emb; s++) {
        S.dim[s] = E->dim[s];
        S.slot_off[s] = n_params;
        n_params += 3 * (int64_t)k * S.dim[s] + 2 * k;
        if (S.dim[s] > maxdim) maxdim = S.dim[s];
    }
    int64_t D = num_dim;
    for (int64_t i = 0; i < n_train; i++) if (tr_off[i + 1] - tr_off[i] > D) D = tr_off[i + 1] - tr_off[i];
    S.D = (int32_t)D;
    S.P = params_out;
    memcpy(S.P, params_in, sizeof(float) * (size_t)n_params);
    S.M = calloc((size_t)n_params, sizeof(float));
    S.Vm = calloc((size_t)n_params, sizeof(float));
    S.gV = malloc(sizeof(float) * (size_t)(nf * k));
    S.gW = malloc(sizeof(float) * (size_t)nf);
    S.vx = malloc(sizeof(float) * (size_t)bs * k);
    S.dvx = malloc(sizeof(float) * (size_t)bs * k);
    S.g = malloc(sizeof(float) * (size_t)bs);
    S.dss = malloc(sizeof(float) * (size_t)bs);
    S.loss = malloc(sizeof(float) * (size_t)bs);
    S.p = malloc(sizeof(float) * (size_t)bs);
    S.sumdx = malloc(sizeof(float) * (size_t)bs);
    S.denc = malloc(sizeof(float) * (size_t)bs * k);
    S.dh = malloc(sizeof(float) * (size_t)bs * k);
    S.dbig = malloc(sizeof(float) * (size_t)bs * (size_t)maxdim);
    S.gx = malloc(sizeof(float) * (size_t)bs * (size_t)maxdim);
    S.gS = malloc(sizeof(float) * (size_t)(n_params - (1 + nf * k + nf)) + 4);
    for (int s = 0; s < S.n_emb; s++) {
        const size_t bd = (size_t)bs * (size_t)S.dim[s], bk = (size_t)bs * k;
        S.e[s] = malloc(sizeof(float) * bd); S.y[s] = malloc(sizeof(float) * bd); S.att[s] = malloc(sizeof(float) * bd);
        S.h[s] = malloc(sizeof(float) * bk); S.hr[s] = malloc(sizeof(float) * bk); S.enc[s] = malloc(sizeof(float) * bk);
    }
    float *fi = calloc((size_t)(n_train * D) + 1, sizeof(float)), *fv = calloc((size_t)(n_train * D) + 1, sizeof(float));
    for (int64_t i = 0; i < n_train; i++)
        for (int64_t j = tr_off[i]; j < tr_off[i + 1]; j++) {
            fi[i * D + j - tr_off[i]] = (float)tr_idx[j]; /* convertToTensors: indices stored as float32 */
            fv[i * D + j - tr_off[i]] = tr_val[j];
        }
    float score[4];
    evaluate(nf, k, num_dim, bs, E, S.P, n_test, te_off, te_idx, te_val, te_tgt, score);
    int32_t *ep = malloc(sizeof(int32_t) * (size_t)(n_epochs + 1));
    float *auc = malloc(sizeof(float) * (size_t)(n_epochs + 1));
    int64_t n_scores = 0, steps = 0;
    ep[n_scores] = 0;
    auc[n_scores++] = score[3];
    int32_t epochs_run = 0, early = 0, diverged = 0, cancelled = 0, limited = 0;
    float cost = 0.0f, t_adam = 0.0f;
    if (cancel_epoch == 0 && n_epochs >= 1 && n_train > 0) cancelled = 1;
    for (int32_t epoch = 1; epoch <= n_epochs && !cancelled; epoch++) {
        cost = 0.0f;
        for (int64_t i = 0; i < n_train; i += bs) {
            if (max_steps > 0 && steps == max_steps) { limited = 1; break; }
            const int64_t j = i + bs < n_train ? i + bs : n_train;
            float lr_t = 0.0f;
            if (adam) {
                t_adam += 1.0f;
                const float fix1 = 1.0f - fmx_pow_steps(0.9f, (int64_t)t_adam), fix2 = 1.0f - fmx_pow_steps(0.999f, (int64_t)t_adam);
                lr_t = lr * sqrtf(fix2) / fix1;
            }
            cost += train_step(&S, fi, fv, tr_tgt, E->tr_row, i, j - i, adam, lr_t, reg, lr);
            steps++;
        }
        epochs_run = epoch;
        if (limited) break;
        int stop = 0;
        if (epoch % verbose == 0 || epoch == n_epochs) {
            evaluate(nf, k, num_dim, bs, E, S.P, n_test, te_off, te_idx, te_val, te_tgt, score);
            ep[n_scores] = epoch;
            auc[n_scores++] = score[3];
            if (cost != cost || score[0] != score[0]) { diverged = 1; stop = 1; } /* score.GetValue() is Precision */
            else if (patience > 0 && epoch > patience) {
                int64_t best = 0; /* lo.MaxBy(a.B > b.B) keeps the first maximum */
                for (int64_t q = 1; q < n_scores; q++) if (auc[q] > auc[best]) best = q;
                if (ep[best] <= epoch - patience) { early = 1; stop = 1; }
            }
        }
        if (stop) break;
        if (cancel_epoch == epoch && epoch < n_epochs && n_train > 0) cancelled = 1;
    }
    int64_t best = 0;
    for (int64_t q = 1; q < n_scores; q++) if (auc[q] > auc[best]) best = q;
    res_f[0] = score[3]; res_f[1] = score[0]; res_f[2] = score[1]; res_f[3] = score[2]; res_f[4] = cost;
    if (cancelled) memset(res_f, 0, 5 * sizeof(float));
    res_i[0] = epochs_run; res_i[1] = ep[best]; res_i[2] = early; res_i[3] = diverged; res_i[4] = cancelled; res_i[5] = steps;
    if (moments_out) {
        memcpy(moments_out, S.M, sizeof(float) * (size_t)n_params);
        memcpy(moments_out + n_params, S.Vm, sizeof(float) * (size_t)n_params);
    }
    free(S.M); free(S.Vm); free(S.gV); free(S.gW); free(S.vx); free(S.dvx); free(S.g); free(S.dss); free(S.loss);
    free(S.p); free(S.sumdx); free(S.denc); free(S.dh); free(S.dbig); free(S.gx); free(S.gS);
    for (int s = 0; s < S.n_emb; s++) { free(S.e[s]); free(S.y[s]); free(S.att[s]); free(S.h[s]); free(S.hr[s]); free(S.enc[s]); }
    free(fi); free(fv); free(ep); free(auc);
    return 0;
}

int32_t fmf_fit(int64_t nf, int32_t num_dim, const int32_t *ip, const float *fp, int64_t max_steps, int64_t n_train, const int64_t *tr_off,
                const int32_t *tr_idx, const float *tr_val, const float *tr_tgt, int64_t n_test, const int64_t *te_off, const int32_t *te_idx,
                const float *te_val, const float *te_tgt, const float *params_in, float *params_out, float *moments_out, float *res_f,
                int64_t *res_i)
{
    const emb_t none = {0, NULL, NULL, NULL, NULL, NULL};
    return fit(nf, num_dim, ip, fp, max_steps, n_train, tr_off, tr_idx, tr_val, tr_tgt, n_test, te_off, te_idx, te_val, te_tgt, &none, params_in,
               params_out, moments_out, res_f, res_i);
}

/* the fit of a model with item-embedding slots: dim [n_emb], table[s] [n_emb_rows x dim_s] bf16 bits, mask [n_emb_rows x n_emb]
 * or NULL, and the table row (-1: none) of every training and test sample; parameters in gorse_b200_fm_create's layout */
int32_t fmf_fit_emb(int64_t nf, int32_t num_dim, const int32_t *ip, const float *fp, int64_t max_steps, int64_t n_train, const int64_t *tr_off,
                    const int32_t *tr_idx, const float *tr_val, const float *tr_tgt, int64_t n_test, const int64_t *te_off,
                    const int32_t *te_idx, const float *te_val, const float *te_tgt, int32_t n_emb, const int32_t *dim,
                    const uint16_t *const *table, const uint8_t *mask, const int32_t *tr_row, const int32_t *te_row, const float *params_in,
                    float *params_out, float *moments_out, float *res_f, int64_t *res_i)
{
    const emb_t E = {n_emb, dim, table, mask, tr_row, te_row};
    return fit(nf, num_dim, ip, fp, max_steps, n_train, tr_off, tr_idx, tr_val, tr_tgt, n_test, te_off, te_idx, te_val, te_tgt, &E, params_in,
               params_out, moments_out, res_f, res_i);
}

/* ---- GAUC ---------------------------------------------------------------------------------------------------------- */
/* EvaluateAFM's scoring after the fit (cmd/gorse-bench/main.go:133-206), literally, on the predictions of the whole test
 * list in test order (fmo_batch_predict): user[i] = indices[0] of test row i, tgt[i] its target, feedback[u] the user's
 * positive training rows.  The users are visited in ascending order (the reference's map order is unpinned); a user with a
 * NaN prediction gets AUC = NaN (Go's sort order on NaN is unpinned).  Per scored user j: user_out[j], cand_out[j] = P + N,
 * auc_out[j] (each sized n_users); returns the number of users scored, *gauc the GAUC. */
int64_t fmo_gauc(int64_t n, const float *pred, const int32_t *user, const float *tgt, int64_t n_users, const int64_t *feedback,
                 int64_t context_size, int32_t *user_out, int64_t *cand_out, float *auc_out, double *gauc)
{
    int64_t *po = calloc((size_t)n_users + 1, sizeof(int64_t)), *no = calloc((size_t)n_users + 1, sizeof(int64_t));
    for (int64_t i = 0; i < n; i++) (tgt[i] > 0 ? po : no)[user[i] + 1]++;
    for (int64_t u = 0; u < n_users; u++) { po[u + 1] += po[u]; no[u + 1] += no[u]; }
    float *pos = malloc(sizeof(float) * (size_t)(po[n_users] + 1)), *neg = malloc(sizeof(float) * (size_t)(no[n_users] + 1));
    int64_t *pf = calloc((size_t)n_users + 1, sizeof(int64_t)), *nf = calloc((size_t)n_users + 1, sizeof(int64_t));
    for (int64_t i = 0; i < n; i++) {   /* positives[u] and negatives[u] in test order */
        const int32_t u = user[i];
        if (tgt[i] > 0) pos[po[u] + pf[u]++] = pred[i];
        else neg[no[u] + nf[u]++] = pred[i];
    }
    float sum = 0, count = 0;
    int64_t ns = 0;
    for (int64_t u = 0; u < n_users; u++) {
        const int64_t P = po[u + 1] - po[u], N = no[u + 1] - no[u];
        if (P == 0 || N == 0 || feedback[u] == 0 || feedback[u] > context_size) continue;
        float *pp = pos + po[u], *nn = neg + no[u];
        int nan = 0;
        for (int64_t i = 0; i < P; i++) nan |= isnan(pp[i]);
        for (int64_t i = 0; i < N; i++) nan |= isnan(nn[i]);
        float auc = NAN;
        if (!nan) {   /* ctr.AUC (evaluator.go:136-153) */
            qsort(pp, (size_t)P, sizeof(float), cmp_f32);
            qsort(nn, (size_t)N, sizeof(float), cmp_f32);
            float s = 0;
            int64_t j = 0;
            for (int64_t i = 0; i < P; i++) {
                while (j < N && nn[j] < pp[i]) j++;
                s += (float)j;
            }
            auc = s / (float)(P * N);
        }
        user_out[ns] = (int32_t)u;
        cand_out[ns] = P + N;
        auc_out[ns] = auc;
        ns++;
        const float cnt = (float)(P + N);
        sum += auc * cnt;
        count += cnt;
    }
    *gauc = count > 0 ? (double)(sum / count) : 0.0;
    free(po); free(no); free(pos); free(neg); free(pf); free(nf);
    return ns;
}
