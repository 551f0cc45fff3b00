// fm_fit.cu -- FM training: gorse_b200_fm_fit, AFM.Fit (model/ctr/fm.go:307-417) for models without embedding slots, and
// gorse_b200_fm_fit_emb for models with them (the slots' kernels and what they add to a step: fm_fit_emb.cuh).
//
// The reference's fit is deterministic: each epoch walks the training rows in dataset order in batches, with no
// shuffling, and only the initial parameters come from Go's RNG (the caller hands them over).  So every step here forms
// each value with the reference's operations in the reference's order, and the parameters and Adam moments are the
// CPU restatement's bit for bit (the test suite's fm_fit_oracle.c, DESIGN §8.5):
//
//   once per Fit   the padded training rows go to the device (indices already through float32); for every batch the
//                  positions of each distinct feature, in row-major order, come from one stable radix sort of
//                  (batch, feature) keys, because the batches never change.
//   per step       fm_fit_forward_kernel  one warp per row, one factor per lane: the forward of fm_pair_kernel, the loss
//                                         and its backward down to the row's dvx (kept), g = dL/dp and dL/d(squareSum).
//                  fm_fit_grad_kernel     one warp per distinct feature of the batch: the Embedding backward of V and W,
//                                         summing the feature's real positions in position order from +0 (the padding
//                                         adds +0 or NaN, so it is flagged per step instead); one warp also
//                                         forms B's gradient and the batch loss as sequential chains.
//                  fm_fit_opt_kernel      Adam or SGD over every element of B, V and W.  A row absent from the batch
//                                         has gradient +0 (its stamp is not this step's), and still decays.
//                  An epoch is one CUDA graph of these launches (GORSE_B200_FM_FIT_NO_GRAPH=1: plain launches).
//   Evaluate       fm_fit_predict_kernel on the positive and the negative test rows, a radix sort of both lists, the
//                  count of negatives below each positive, and the sequential float32 AUC chain on one thread.
// The arithmetic is fp32 with explicit __fmaf_rn / __fmul_rn / __fadd_rn / __fsub_rn / __fdiv_rn / __fsqrt_rn.
// gorse_b200_fm_fit_trials fits several trials in lockstep through the same kernels: each kernel takes a Group and block b
// runs trial b % n on that trial's tables (DESIGN §8.8); a solo fit is one trial.
// gorse_b200_fm_gauc predicts every test row as one list through Fit::predict, the evaluation's forward, and scores each
// user's rows with the kernels of fm_gauc.cuh (DESIGN §8.10).
#include <cub/cub.cuh>

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <vector>

#include "common.cuh"
#include "fm_exp.h"
#include "fm_fit_math.h"

namespace gb {
namespace fmfit {

constexpr int MAX_FACTORS = 32;
constexpr int WARPS = 8;
constexpr unsigned FULL = 0xffffffffu;

struct Rows {            // padded rows on the device: [n x D] feature rows (float32-rounded) and values
    const int32_t *idx;
    const float *val;
    int32_t D;
};

// The trials of one launch (gorse_b200_fm_fit_trials; a solo fit is one trial).  Every per-trial table lies in one arena
// per trial, all arenas alike: a kernel gets trial 0's pointers and block b runs trial b % n on trial 0's tables plus
// (b % n) stride bytes, so the blocks of one row block run next to each other and read the shared rows from L2.
constexpr int MAX_TRIALS = 16;

struct Group {
    int n;
    int64_t stride;       // bytes from one trial's arena to the next
    const int32_t *on;    // [n]: 0 once the trial has left the batch; its tables are then not touched
};

struct Blk {              // this block's trial, its byte offset, and its place among the trial's blocks
    int tr, x, nx;
    int64_t off;
};

__device__ __forceinline__ bool trial_block(const Group &G, Blk &b)
{
    b.tr = (int)(blockIdx.x % (unsigned)G.n);
    b.x = (int)(blockIdx.x / (unsigned)G.n);
    b.nx = (int)(gridDim.x / (unsigned)G.n);
    b.off = b.tr * G.stride;
    return G.on[b.tr] != 0;
}

template <typename T>
__host__ __device__ __forceinline__ T *at(T *p, int64_t off) { return (T *)((char *)p + off); }
template <typename T>
__host__ __device__ __forceinline__ const T *at(const T *p, int64_t off) { return (const T *)((const char *)p + off); }

// Go's max(a, b) on float32: NaN propagates, max(-0, +0) = +0
__device__ __forceinline__ float go_max(float a, float b)
{
    if (a != a) return a;
    if (b != b) return b;
    if (a == b) return __int_as_float(__float_as_int(a) & __float_as_int(b));
    return a > b ? a : b;
}

// AFM.Forward of one row by one warp, lane = factor: returns p, leaves the lane's vx
__device__ __forceinline__ float row_forward(const float *P, int64_t nf, int k, const Rows &R, int64_t row, int lane, float &vx)
{
    const float *V = P + 1, *W = P + 1 + nf * k;
    const int32_t *ix = R.idx + row * R.D;
    const float *xv = R.val + row * R.D;
    float ss = 0.0f, lin = 0.0f;
    vx = 0.0f;
    for (int l = 0; l < R.D; l++) {
        const int64_t r = ix[l];
        const float x = xv[l], x2 = __fmul_rn(x, x);
        if (lane < k) {
            const float v = V[r * k + lane];
            vx = __fmaf_rn(v, x, vx);                       // BMM(v, x)
            ss = __fmaf_rn(__fmul_rn(v, v), x2, ss);        // BMM(Square(v), Square(x))
        }
        lin = __fmaf_rn(W[r], x, lin);                      // BMM(w, x)
    }
    const float d = __fsub_rn(__fmul_rn(vx, vx), ss);
    float s = 0.0f;
    for (int q = 0; q < k; q++) s = __fadd_rn(s, __shfl_sync(FULL, d, q));   // Sum(., 1) from 0 in factor order
    s = __fmul_rn(s, 0.5f);
    return __fadd_rn(__fadd_rn(lin, s), P[0]);                                // Add(linear, sum, B)
}

__global__ void fm_fit_predict_kernel(Group G, const float *P, int64_t nf, int k, Rows R, int64_t n, float *pred)
{
    Blk tb;
    if (!trial_block(G, tb)) return;
    P = at(P, tb.off);
    pred = at(pred, tb.off);
    const int lane = threadIdx.x & 31;
    const int64_t warps = (int64_t)tb.nx * WARPS;
    for (int64_t row = (int64_t)tb.x * WARPS + (threadIdx.x >> 5); row < n; row += warps) {
        float vx;
        const float p = row_forward(P, nf, k, R, row, lane, vx);
        if (lane == 0) pred[row] = p;
    }
}

// dL/d(squareSum) of a row from its dL/dsum: Sub's second input gets 0 - dy
__device__ __forceinline__ float dss_b(float dsub) { return __fsub_rn(0.0f, dsub); }

constexpr int MAX_SLOTS = 8;
constexpr int MAX_EMB_DIM = 1024;

// The order in which Tensor.Backward hands vx its gradients in the graph with n slots: 0 is Square(vx)'s, 1 + s is slot s's
// BMM(vx, enc).  The ops of equal generation leave the container/heap in this order (the restatement replays the heap:
// fmf_backward_order); the terms are added in it, and fp32 addition does not associate.
constexpr int8_t VX_ORDER[MAX_SLOTS + 1][MAX_SLOTS + 1] = {
    {0}, {1, 0}, {2, 1, 0}, {1, 3, 2, 0}, {3, 4, 2, 1, 0}, {4, 5, 1, 2, 3, 0}, {3, 6, 4, 2, 5, 1, 0}, {7, 4, 2, 5, 3, 1, 6, 0},
    {8, 5, 6, 2, 1, 4, 3, 7, 0}};

struct SlotLogits {              // what the slots leave for the loss: the rows' logits and vx, and every slot's enc
    const float *p, *vx;
    const float *enc[MAX_SLOTS];
    int n;
    int8_t ord[MAX_SLOTS + 1];
};

// forward, BCEWithLogits and its backward for rows [r0, r0 + B).  EMB: the forward (with the slots' terms) has already run
// and left p and vx in L; vx's gradient then collects Square's term and every slot's enc dp in L.ord's order.
template <bool EMB>
__global__ void __launch_bounds__(WARPS * 32) fm_fit_forward_kernel(Group G, const float *P, int64_t nf, int k, Rows R, const float *tgt,
                                                                   int64_t bs, int64_t n, int s, float *g, float *dss, float *dvx,
                                                                   float *loss, const int32_t *row_len, int32_t *padnan, const int64_t *t_base,
                                                                   const __grid_constant__ SlotLogits L)
{
    Blk tb;
    if (!trial_block(G, tb)) return;
    P = at(P, tb.off);
    g = at(g, tb.off);
    dss = at(dss, tb.off);
    dvx = at(dvx, tb.off);
    loss = at(loss, tb.off);
    padnan = at(padnan, tb.off);
    const int lane = threadIdx.x & 31;
    const int64_t r0 = (int64_t)s * bs;
    const int B = (int)(n - r0 < bs ? n - r0 : bs);
    const float m = __fdiv_rn(1.0f, (float)B);                  // Mean's backward: dy / len
    for (int b = tb.x * WARPS + (threadIdx.x >> 5); b < B; b += tb.nx * WARPS) {
        float vx, p;
        if (EMB) {
            p = at(L.p, tb.off)[b];
            vx = lane < k ? at(L.vx, tb.off)[(int64_t)b * k + lane] : 0.0f;
        } else {
            p = row_forward(P, nf, k, R, r0 + b, lane, vx);
        }
        const float t = tgt[r0 + b];
        const float y = __fdiv_rn(__fadd_rn(t, 1.0f), 2.0f);    // Div(Add(1, target), 2)
        const float a = p < 0.0f ? -p : p;                       // Abs
        const float E = fmx_expf(-a);                            // Exp(Neg(.)): float32(math.Exp(float64))
        const float lin1 = __fadd_rn(E, 1.0f);                   // Add(1, exp)
        if (lane == 0) loss[b] = __fadd_rn(__fsub_rn(go_max(p, 0.0f), __fmul_rn(p, y)), fmx_logf(lin1));
        // backward: Mean -> Add -> (Sub: m; Log: 0 + m) -> Log: dy / x -> Exp: exp(x) dy -> Neg; Sub -> (ReLU: m; Mul: 0 - m)
        const float dexp = __fmul_rn(E, __fdiv_rn(__fadd_rn(0.0f, m), lin1));
        const float g_relu = __fmul_rn(p > 0.0f ? 1.0f : 0.0f, m);
        const float g_mul = __fmul_rn(__fsub_rn(0.0f, m), y);
        const float g_abs = p < 0.0f ? dexp : -dexp;             // Abs of Neg's -dexp
        // p's three gradients in Tensor.Backward's heap order: Mul, Abs, then ReLU (fmf_p_order)
        const float gp = __fadd_rn(__fadd_rn(g_mul, g_abs), g_relu);
        // Add(linear, sum): sum gets 0 + g; Mul(., 0.5); Sum(., 1); Sub -> (Square(vx): d, BMM(e2, x2): 0 - d); Square: vx dy 2
        const float dsub = __fmul_rn(__fadd_rn(0.0f, gp), 0.5f);
        if (lane == 0) {
            g[b] = gp;
            dss[b] = dss_b(dsub);
        }
        float dvx_f = __fmul_rn(__fmul_rn(vx, dsub), 2.0f);
        if (EMB && lane < k) {
            const float sq = dvx_f, dp = __fadd_rn(0.0f, gp);   // Add(fmOutput, .): the slot's dot gets 0 + dp
            for (int q = 0; q <= L.n; q++) {
                const int o = L.ord[q];
                const float term = o == 0 ? sq : __fmaf_rn(at(L.enc[o - 1], tb.off)[(int64_t)b * k + lane], dp, 0.0f);   // enc dp^T, a dot of length 1
                dvx_f = q == 0 ? term : __fadd_rn(dvx_f, term);
            }
        }
        if (lane < k) dvx[(int64_t)b * k + lane] = dvx_f;
        // A padded position (index 0, value 0) adds fma(0, dvx, 0) + (V[0] fma(0, dss, 0)) 2 to V's row 0 and fma(0, g, 0)
        // to W's: +0, a no-op on a sum that starts at +0, or NaN when dvx, dss, g or V[0] is not finite.  So the padding
        // is not walked position by position: a NaN marks the factor for this step and fm_fit_grad_kernel applies it.
        if (row_len[r0 + b] < R.D) {
            const int32_t t_step = (int32_t)(*t_base + s + 1);
            if (lane < k) {
                const float c = __fadd_rn(__fmaf_rn(0.0f, dvx_f, 0.0f), __fmul_rn(__fmul_rn(P[1 + lane], __fmaf_rn(0.0f, dss_b(dsub), 0.0f)), 2.0f));
                if (c != c) padnan[lane] = t_step;
            }
            if (lane == 0 && __fmaf_rn(0.0f, gp, 0.0f) != __fmaf_rn(0.0f, gp, 0.0f)) padnan[k] = t_step;
        }
    }
}

// Embedding backward of V and W over the batch's distinct features; q = 0 is B's gradient and the batch loss
// The stamp is shared by the trials of a group (they walk the same batches); so row 0 is stamped by every trial whenever
// feature 0 has no real position in the batch, its gradient then +0 or the padding's NaN.
__global__ void __launch_bounds__(WARPS * 32) fm_fit_grad_kernel(Group G, const float *P, int64_t nf, int k, Rows R, int64_t bs, int64_t n,
                                                                int s, const int64_t *batch_seg, const int32_t *seg_start,
                                                                const int32_t *seg_feat, const int32_t *seg_pos, const float *g,
                                                                const float *dss, const float *dvx, const float *loss, float *gV, float *gW,
                                                                float *gB, int32_t *stamp, float *batch_loss, const int64_t *t_base,
                                                                const int32_t *padnan)
{
    Blk tb;
    if (!trial_block(G, tb)) return;
    P = at(P, tb.off);
    g = at(g, tb.off);
    dss = at(dss, tb.off);
    dvx = at(dvx, tb.off);
    loss = at(loss, tb.off);
    gV = at(gV, tb.off);
    gW = at(gW, tb.off);
    gB = at(gB, tb.off);
    batch_loss = at(batch_loss, tb.off);
    padnan = at(padnan, tb.off);
    const int lane = threadIdx.x & 31;
    const int64_t r0 = (int64_t)s * bs;
    const int B = (int)(n - r0 < bs ? n - r0 : bs);
    const int32_t t = (int32_t)(*t_base + s + 1);
    const int64_t j0 = batch_seg[s], nseg = batch_seg[s + 1] - j0;
    const float *V = P + 1;
    const int64_t warps = (int64_t)tb.nx * WARPS;
    const float qnan = __int_as_float(0x7fffffff);
    for (int64_t q = (int64_t)tb.x * WARPS + (threadIdx.x >> 5); q <= nseg; q += warps) {
        if (q == 0) {
            // the padding's NaNs (fm_fit_forward_kernel) when feature 0 has no real position in the batch: they alone make
            // row 0's gradient; without any, it is +0, the same as an absent row
            if (nseg == 0 || seg_feat[j0] != 0) {
                const bool nan_v = lane < k && padnan[lane] == t, nan_w = padnan[k] == t;
                if (lane < k) gV[lane] = nan_v ? qnan : 0.0f;
                if (lane == 0) {
                    gW[0] = nan_w ? qnan : 0.0f;
                    stamp[0] = t;
                }
            }
            if (lane == 0) {            // Add(., B)'s backward: +0 plus every row's g in order
                float acc = 0.0f;
#pragma unroll 16
                for (int b = 0; b < B; b++) acc = __fadd_rn(acc, g[b]);
                *gB = acc;
            } else if (lane == 1) {     // Mean: 0 plus every row's loss in order, over len
                float acc = 0.0f;
#pragma unroll 16
                for (int b = 0; b < B; b++) acc = __fadd_rn(acc, loss[b]);
                batch_loss[s] = __fdiv_rn(acc, (float)B);
            }
            continue;
        }
        const int64_t j = j0 + q - 1;
        const int32_t r = seg_feat[j];
        float accV = 0.0f, accW = 0.0f;
        for (int32_t i = seg_start[j]; i < seg_start[j + 1]; i++) {
            const int32_t pos = seg_pos[i];
            const int b = (int)(pos / R.D - r0);
            const float x = R.val[pos];
            if (lane < k) {
                const float dv_bmm = __fmaf_rn(x, dvx[(int64_t)b * k + lane], 0.0f);                          // BMM(v, x): x dvx^T
                const float de2 = __fmaf_rn(__fmul_rn(x, x), dss[b], 0.0f);                                    // BMM(e2, x2): x2 dss^T
                const float dv_sq = __fmul_rn(__fmul_rn(V[(int64_t)r * k + lane], de2), 2.0f);                 // Square(v)
                accV = __fadd_rn(accV, __fadd_rn(dv_bmm, dv_sq));
            }
            if (lane == 0) accW = __fadd_rn(accW, __fmaf_rn(x, g[b], 0.0f));                                   // BMM(w, x): x dlinear
        }
        if (r == 0) {   // the padding's NaNs of this step
            if (lane < k && padnan[lane] == t) accV = qnan;
            if (lane == 0 && padnan[k] == t) accW = qnan;
        }
        if (lane < k) gV[(int64_t)r * k + lane] = accV;
        if (lane == 0) {
            gW[r] = accW;
            stamp[r] = t;
        }
    }
}

// the reference's per-index fusing of mul_const_add[_to] (floats_avx512.c:18-80): the 8-lane block rounds twice
__device__ __forceinline__ float mca(float a, float c, float b, int64_t i, int64_t n)
{
    const int64_t body = (n / 16) * 16;
    const bool blk8 = i >= body && n - body >= 8 && i < body + 8;
    return blk8 ? __fadd_rn(__fmul_rn(a, c), b) : __fmaf_rn(a, c, b);
}

struct Opt {
    int adam;
    float wd, c1, c2, eps, sgd_lr;
    const float *lr_tab;   // Adam's step size per global step
};

// element e of the parameters, the i-th of a tensor of n, through Adam or SGD
__device__ __forceinline__ void opt_element(float *P, float *M, float *Vm, int64_t e, float grad, int64_t i, int64_t n, float lr, const Opt &o)
{
    const float p = P[e];
    float b1 = mca(p, o.wd, grad, i, n);             // MulConstAddTo: grad + wd p
    if (!o.adam) {
        P[e] = mca(b1, -lr, p, i, n);
        return;
    }
    float m = M[e], v = Vm[e];
    float b2 = __fsub_rn(b1, m);                     // SubTo
    m = mca(b2, o.c1, m, i, n);                      // m += (1 - beta1) (grad - m)
    b2 = __fmul_rn(b1, b1);                          // MulTo
    b2 = __fsub_rn(b2, v);                           // Sub
    v = mca(b2, o.c2, v, i, n);                      // v += (1 - beta2) (grad^2 - v)
    b2 = __fadd_rn(__fsqrt_rn(v), o.eps);            // SqrtTo, AddConst
    b1 = __fdiv_rn(m, b2);                           // DivTo
    P[e] = mca(b1, -lr, p, i, n);                    // MulConstAdd(., -lr, param)
    M[e] = m;
    Vm[e] = v;
}

struct Opts {                    // every trial's optimiser (lr_tab: in the trial's own arena)
    Opt o[MAX_TRIALS];
};

// one optimiser step over B, V and W: the elementwise sequences of optimizers.go:138-151 (Adam) and :78-79 (SGD)
__global__ void fm_fit_opt_kernel(Group G, float *P, float *M, float *Vm, int64_t nf, int k, const float *gV, const float *gW, const float *gB,
                                  const int32_t *stamp, const int64_t *t_base, int s, const __grid_constant__ Opts O)
{
    Blk tb;
    if (!trial_block(G, tb)) return;
    P = at(P, tb.off);
    M = at(M, tb.off);
    Vm = at(Vm, tb.off);
    gV = at(gV, tb.off);
    gW = at(gW, tb.off);
    gB = at(gB, tb.off);
    const Opt &o = O.o[tb.tr];
    const int64_t nV = nf * k, n_params = 1 + nV + nf;
    const int64_t t = *t_base + s + 1;
    const float lr = o.adam ? o.lr_tab[t - 1] : o.sgd_lr;
    for (int64_t e = (int64_t)tb.x * blockDim.x + threadIdx.x; e < n_params; e += (int64_t)tb.nx * blockDim.x) {
        int64_t i, n;
        float grad;
        if (e == 0) { i = 0; n = 1; grad = *gB; }
        else if (e <= nV) { i = e - 1; n = nV; grad = stamp[i / k] == (int32_t)t ? gV[i] : 0.0f; }
        else { i = e - 1 - nV; n = nf; grad = stamp[i] == (int32_t)t ? gW[i] : 0.0f; }
        opt_element(P, M, Vm, e, grad, i, n, lr, o);
    }
}

struct SlotTensors {             // the 5 tensors of every slot in parameter order: where each ends, counted from the first
    int32_t end[5 * MAX_SLOTS];
    int n;
};

// the same step over the slots' tensors (dense gradients gS, laid out as the parameters from `base`); the fusing rule
// takes each element's index in its own tensor
__global__ void fm_fit_emb_opt_kernel(Group G, float *P, float *M, float *Vm, int64_t base, const float *gS, SlotTensors T, const int64_t *t_base,
                                      int s, const __grid_constant__ Opts O)
{
    Blk tb;
    if (!trial_block(G, tb)) return;
    P = at(P, tb.off);
    M = at(M, tb.off);
    Vm = at(Vm, tb.off);
    gS = at(gS, tb.off);
    const Opt &o = O.o[tb.tr];
    const int64_t t = *t_base + s + 1;
    const float lr = o.adam ? o.lr_tab[t - 1] : o.sgd_lr;
    const int32_t total = T.end[T.n - 1];
    for (int32_t e = tb.x * blockDim.x + threadIdx.x; e < total; e += tb.nx * blockDim.x) {
        int q = 0;
        while (e >= T.end[q]) q++;
        const int32_t start = q ? T.end[q - 1] : 0;
        opt_element(P, M, Vm, base + e, gS[e], e - start, T.end[q] - start, lr, o);
    }
}

#include "fm_fit_emb.cuh"
#include "fm_gauc.cuh"

__global__ void fm_fit_set_kernel(int64_t *dst, int64_t v) { *dst = v; }

// segment keys: (batch << 32) | feature of every real training position; padded positions get all ones, which sort
// after every real key within the sorted bits, so the real positions come first
__global__ void fm_fit_keys_kernel(const int32_t *idx, const int32_t *row_len, int32_t D, int64_t np, int64_t per_batch, uint64_t *key,
                                   int32_t *pos)
{
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < np; i += (int64_t)gridDim.x * blockDim.x) {
        const bool real = i % D < row_len[i / D];
        key[i] = real ? ((uint64_t)(i / per_batch) << 32) | (uint32_t)idx[i] : ~0ull;
        pos[i] = (int32_t)i;
    }
}

__global__ void fm_fit_heads_kernel(const uint64_t *key, int64_t np, int32_t *head)
{
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < np; i += (int64_t)gridDim.x * blockDim.x)
        head[i] = i == 0 || key[i] != key[i - 1];
}

__global__ void fm_fit_segments_kernel(const uint64_t *key, const int32_t *head, const int32_t *seg_id, int64_t np, int32_t *seg_start,
                                       int32_t *seg_feat, int32_t *seg_batch)
{
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < np; i += (int64_t)gridDim.x * blockDim.x)
        if (head[i]) {
            const int32_t j = seg_id[i];
            seg_start[j] = (int32_t)i;
            seg_feat[j] = (int32_t)(key[i] & 0xffffffffu);
            seg_batch[j] = (int32_t)(key[i] >> 32);
        }
}

// batch_seg[b] = the first segment of batch b (b in [0, n_batches])
__global__ void fm_fit_batch_seg_kernel(const int32_t *seg_batch, int64_t n_segs, int64_t n_batches, int64_t *batch_seg)
{
    for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b <= n_batches; b += (int64_t)gridDim.x * blockDim.x) {
        int64_t lo = 0, hi = n_segs;
        while (lo < hi) {
            const int64_t mid = (lo + hi) >> 1;
            if (seg_batch[mid] < b) lo = mid + 1;
            else hi = mid;
        }
        batch_seg[b] = lo;
    }
}

// per sorted positive: the negatives strictly below it; and the counts Precision / Recall / Accuracy need
// (counts: 3 per trial)
__global__ void fm_fit_auc_counts_kernel(Group G, const float *pos, int64_t n_pos, const float *neg, int64_t n_neg, int32_t *below,
                                         unsigned long long *counts)
{
    Blk tb;
    if (!trial_block(G, tb)) return;
    pos = at(pos, tb.off);
    neg = at(neg, tb.off);
    below = at(below, tb.off);
    counts += 3 * tb.tr;
    const int lane = threadIdx.x & 31;
    const int64_t n = n_pos > n_neg ? n_pos : n_neg;
    for (int64_t i0 = (int64_t)tb.x * blockDim.x; i0 < n; i0 += (int64_t)tb.nx * blockDim.x) {
        const int64_t i = i0 + threadIdx.x;
        bool tp = false, fp = false, tn = false;
        if (i < n_pos) {
            const float p = pos[i];
            int64_t lo = 0, hi = n_neg;
            while (lo < hi) {
                const int64_t mid = (lo + hi) >> 1;
                if (neg[mid] < p) lo = mid + 1;
                else hi = mid;
            }
            below[i] = (int32_t)lo;
            tp = p > 0.0f;
        }
        if (i < n_neg) {
            fp = neg[i] > 0.0f;
            tn = neg[i] < 0.0f;
        }
        const unsigned a = __ballot_sync(FULL, tp), b = __ballot_sync(FULL, fp), c = __ballot_sync(FULL, tn);
        if (lane == 0) {
            if (a) atomicAdd(&counts[0], (unsigned long long)__popc(a));
            if (b) atomicAdd(&counts[1], (unsigned long long)__popc(b));
            if (c) atomicAdd(&counts[2], (unsigned long long)__popc(c));
        }
    }
}

// AUC's sum: float32(count) added in sequence over the positives in ascending order (evaluator.go:139-148); one thread
// per trial (sum: one per trial)
__global__ void fm_fit_auc_chain_kernel(Group G, const int32_t *below, int64_t n_pos, float *sum)
{
    const int tr = threadIdx.x;
    if (tr >= G.n || !G.on[tr]) return;
    below = at(below, tr * G.stride);
    float acc = 0.0f;
#pragma unroll 16
    for (int64_t i = 0; i < n_pos; i++) acc = __fadd_rn(acc, __int2float_rn(below[i]));
    sum[tr] = acc;
}

// the float32 counter of evaluator.go after n increments: exact up to 2^24, where adding 1 no longer changes it
inline float go_count(uint64_t n) { return n <= (1u << 24) ? (float)n : 16777216.0f; }

inline bool feature_ok(int64_t idx, int64_t n_features)
{
    if (idx < 0 || idx >= n_features) return false;
    return (int64_t)(float)idx < n_features;
}

struct TestSet {                  // one list of EvaluateClassification: padded rows, their table rows and (per trial) their predictions
    DevBuf<int32_t> idx, emb_row;
    DevBuf<float> val;
    float *pred = nullptr, *sorted = nullptr;
    int64_t n = 0;
    int32_t D = 0;
};

int32_t check_rows(const char *what, int64_t n, const int64_t *off, const int32_t *idx, const float *val, const float *tgt, int64_t nf)
{
    GB_CHECK_ARG(n >= 0, "%s: negative row count", what);
    if (n == 0) return GORSE_B200_OK;
    GB_CHECK_ARG(off != nullptr && tgt != nullptr, "%s: NULL offsets or targets", what);
    GB_CHECK_ARG(off[0] == 0, "%s: offsets must start at 0", what);
    for (int64_t r = 0; r < n; r++)
        GB_CHECK_ARG(off[r + 1] >= off[r] && off[r + 1] - off[r] <= INT32_MAX, "%s row %lld: offsets decrease", what, (long long)r);
    GB_CHECK_ARG(off[n] == 0 || (idx != nullptr && val != nullptr), "%s: NULL indices or values", what);
    for (int64_t j = 0; j < off[n]; j++)
        GB_CHECK_ARG(feature_ok(idx[j], nf), "%s entry %lld: feature %d is not in [0, %lld) once rounded to float32", what, (long long)j,
                     idx[j], (long long)nf);
    return GORSE_B200_OK;
}

// rows [rows] of a CSR padded to D: features through float32, values, zeros beyond each row
void pad_rows(const int64_t *off, const int32_t *idx, const float *val, const std::vector<int64_t> &rows, int32_t D, std::vector<int32_t> &pi,
              std::vector<float> &pv)
{
    pi.assign(rows.size() * (size_t)D, 0);
    pv.assign(rows.size() * (size_t)D, 0.0f);
    for (size_t i = 0; i < rows.size(); i++) {
        const int64_t r = rows[i];
        for (int64_t j = off[r]; j < off[r + 1]; j++) {
            pi[i * D + (size_t)(j - off[r])] = (int32_t)(int64_t)(float)idx[j];
            pv[i * D + (size_t)(j - off[r])] = val[j];
        }
    }
}

int32_t longest(const int64_t *off, const std::vector<int64_t> &rows, int32_t num_dimension, int32_t *D)
{
    int64_t d = num_dimension;
    for (int64_t r : rows) d = std::max<int64_t>(d, off[r + 1] - off[r]);
    GB_CHECK_ARG(d <= INT32_MAX, "rows of 2^31 or more features");
    *D = (int32_t)d;
    return GORSE_B200_OK;
}

}  // namespace fmfit
}  // namespace gb

using namespace gb;
using namespace gb::fmfit;

namespace {

struct EmbArgs {                  // the item-embedding side of gorse_b200_fm_fit_emb
    int32_t n_emb;
    const int32_t *dim;
    int64_t n_rows;
    const uint16_t *const *table;
    const uint8_t *mask;
    const int32_t *train_row, *test_row;
};

struct Data {                     // what every trial of a call shares: the rows, the table and the model's shape
    int64_t n_features;
    int32_t num_dimension, n_emb;
    const EmbArgs *E;             // NULL: gorse_b200_fm_fit, which takes no embeddings and so no model with slots
    int64_t n_train;
    const int64_t *train_off;
    const int32_t *train_idx;
    const float *train_val, *train_target;
    int64_t n_test;
    const int64_t *test_off;
    const int32_t *test_idx;
    const float *test_val, *test_target;
    int64_t n_params;
};

struct Carver {                   // lays out a trial's arena from `base`: every table aligned to 256 bytes
    uintptr_t base;
    size_t bytes = 0;
    template <typename T>
    void take(T *&p, int64_t count)
    {
        p = reinterpret_cast<T *>(base + bytes);
        bytes += (std::max<size_t>((size_t)count, 1) * sizeof(T) + 255) / 256 * 256;
    }
};

struct Fit {
    gorse_b200_ctx *ctx;
    cudaStream_t st;
    int64_t nf;
    int k;
    int32_t num_dimension;
    const gorse_b200_fm_fit_params *prm;   // trial 0's: its shared fields are every trial's
    bool train = true;                     // false: predictions only (gorse_b200_fm_gauc), no optimiser tables
    int64_t n_params = 0, max_total = 0;   // max_total: the most optimiser steps of any trial
    // training set, shared by the trials (so is the stamp: they step in lockstep)
    DevBuf<int32_t> tr_idx, tr_len, seg_start, seg_feat, seg_pos, stamp;
    DevBuf<float> tr_val, tr_tgt;
    DevBuf<int64_t> batch_seg, t_base;
    int64_t n_train = 0, n_batches = 0;
    int32_t D = 0;
    unsigned grad_grid = 1;
    // evaluation lists, shared; the counts and sums: one set per trial of a group
    TestSet te[2];
    DevBuf<unsigned long long> counts;
    DevBuf<float> auc_sum;
    DevBuf<unsigned char> cub_tmp;
    // item-embedding slots: the table and the row maps, shared
    int n_emb = 0, maxdim = 1;
    int64_t base = 0;             // parameters before the first slot
    const EmbArgs *E = nullptr;
    DevBuf<uint16_t> table[MAX_SLOTS];
    DevBuf<uint8_t> mask;
    DevBuf<int32_t> tr_row;
    SlotTensors tens{};
    int64_t rows = 1, slot_rows = 1;   // a batch's rows; the slots' (the largest batch or evaluation chunk)
    unsigned row_grid = 1;
    // the group: G trials with an arena of `stride` bytes each; the pointers below are trial 0's
    int G = 0;
    int64_t stride = 0;
    DevBuf<unsigned char> arena;
    DevBuf<int32_t> on, ev_on;       // [MAX_TRIALS]: the trials stepping, the trials evaluated
    float *P, *M, *Vm, *gV, *gW, *gB, *g, *dss, *dvx, *loss, *batch_loss, *lr_tab;
    int32_t *padnan, *below;
    float *gS, *zmax, *rowsum, *gx, *denc, *dh, *sumdx, *p, *vx;
    float *s_e[MAX_SLOTS], *s_y[MAX_SLOTS], *s_att[MAX_SLOTS], *s_h[MAX_SLOTS], *s_enc[MAX_SLOTS];
    Slot slot[MAX_SLOTS];
    SlotLogits logits{};
    Opts opts{};

    int32_t upload_train(const int64_t *off, const int32_t *idx, const float *val, const float *tgt);
    int32_t upload_list(TestSet &T, const int64_t *off, const int32_t *idx, const float *val, const std::vector<int64_t> &rows_,
                        const int32_t *emb_row);
    int32_t upload_test(const int64_t *off, const int32_t *idx, const float *val, const float *tgt, int64_t n, const int32_t *emb_row);
    int32_t upload_slots();
    size_t carve(uintptr_t b);
    int32_t alloc_group(int g);
    unsigned grid(int64_t blocks) const { return (unsigned)(std::min<int64_t>(blocks, INT32_MAX / G) * G); }
    int32_t slots_forward(Group Gr, const int32_t *emb_row, Batch T, float *logit);
    int32_t run_steps(int s0, int s1);
    int32_t predict(Group Ev, TestSet &T);
    int32_t evaluate(const bool *which, float (*score)[4]);
};

int32_t Fit::upload_train(const int64_t *off, const int32_t *idx, const float *val, const float *tgt)
{
    std::vector<int64_t> rows_((size_t)n_train);
    for (int64_t r = 0; r < n_train; r++) rows_[(size_t)r] = r;
    GB_TRY(longest(off, rows_, num_dimension, &D));
    const int64_t bs = prm->batch_size, np = n_train * D;
    if (np >= INT32_MAX) {
        set_error("fm_fit: %lld training positions, at most 2^31 - 1", (long long)np);
        return GORSE_B200_ERR_UNSUPPORTED;
    }
    n_batches = (n_train + bs - 1) / bs;
    std::vector<int32_t> pi;
    std::vector<float> pv;
    pad_rows(off, idx, val, rows_, D, pi, pv);
    GB_TRY(tr_idx.upload(pi.data(), pi.size(), st));
    GB_TRY(tr_val.upload(pv.data(), pv.size(), st));
    GB_TRY(tr_tgt.upload(tgt, (size_t)n_train, st));
    std::vector<int32_t> len((size_t)n_train);
    for (int64_t r = 0; r < n_train; r++) len[(size_t)r] = (int32_t)(off[r + 1] - off[r]);
    GB_TRY(tr_len.upload(len.data(), len.size(), st));
    const int64_t n_real = n_train > 0 ? off[n_train] : 0;   // positions that are not padding
    GB_TRY(batch_seg.alloc((size_t)n_batches + 1));
    GB_CUDA(cudaMemsetAsync(batch_seg.p, 0, ((size_t)n_batches + 1) * sizeof(int64_t), st));
    GB_TRY(seg_pos.alloc((size_t)std::max<int64_t>(np, 1)));
    GB_TRY(seg_start.alloc((size_t)np + 1));
    GB_TRY(seg_feat.alloc((size_t)std::max<int64_t>(np, 1)));
    int64_t max_segs = 0;
    if (n_real > 0) {
        // the feature lists of every batch: a stable sort of (batch, feature) keys keeps each feature's positions in order;
        // the padding is left out (fm_fit_forward_kernel)
        DevBuf<uint64_t> key, key2;
        DevBuf<int32_t> pos, head, seg_id, seg_batch;
        GB_TRY(key.alloc((size_t)np));
        GB_TRY(key2.alloc((size_t)np));
        GB_TRY(pos.alloc((size_t)np));
        GB_TRY(head.alloc((size_t)np));
        GB_TRY(seg_id.alloc((size_t)np));
        GB_TRY(seg_batch.alloc((size_t)np));
        const unsigned grid_ = (unsigned)std::min<int64_t>(div_up(np, 256), (int64_t)ctx->sm_count * 16);
        fm_fit_keys_kernel<<<grid_, 256, 0, st>>>(tr_idx.p, tr_len.p, D, np, bs * D, key.p, pos.p);
        GB_LAUNCHED(ctx);
        int end_bit = 32;
        while (end_bit < 64 && (uint64_t)n_batches > (1ull << (end_bit - 32))) end_bit++;
        size_t b1 = 0, b2 = 0;
        GB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, b1, key.p, key2.p, pos.p, seg_pos.p, (int)np, 0, end_bit, st));
        GB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, b2, head.p, seg_id.p, (int)n_real, st));
        GB_TRY(cub_tmp.alloc(std::max(b1, b2)));
        b1 = b2 = cub_tmp.n;
        GB_CUDA(cub::DeviceRadixSort::SortPairs(cub_tmp.p, b1, key.p, key2.p, pos.p, seg_pos.p, (int)np, 0, end_bit, st));
        fm_fit_heads_kernel<<<grid_, 256, 0, st>>>(key2.p, n_real, head.p);
        GB_LAUNCHED(ctx);
        GB_CUDA(cub::DeviceScan::ExclusiveSum(cub_tmp.p, b2, head.p, seg_id.p, (int)n_real, st));
        fm_fit_segments_kernel<<<grid_, 256, 0, st>>>(key2.p, head.p, seg_id.p, n_real, seg_start.p, seg_feat.p, seg_batch.p);
        GB_LAUNCHED(ctx);
        int32_t last[2];
        GB_CUDA(cudaMemcpyAsync(&last[0], seg_id.p + n_real - 1, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
        GB_CUDA(cudaMemcpyAsync(&last[1], head.p + n_real - 1, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
        GB_CUDA(cudaStreamSynchronize(st));
        const int64_t n_segs = (int64_t)last[0] + last[1];
        const int32_t end = (int32_t)n_real;
        GB_CUDA(cudaMemcpyAsync(seg_start.p + n_segs, &end, sizeof(int32_t), cudaMemcpyHostToDevice, st));
        fm_fit_batch_seg_kernel<<<(unsigned)div_up(n_batches + 1, 256), 256, 0, st>>>(seg_batch.p, n_segs, n_batches, batch_seg.p);
        GB_LAUNCHED(ctx);
        std::vector<int64_t> h((size_t)n_batches + 1);
        GB_CUDA(cudaMemcpyAsync(h.data(), batch_seg.p, h.size() * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
        GB_CUDA(cudaStreamSynchronize(st));   // the temporaries above are freed on return
        for (int64_t b = 0; b < n_batches; b++) max_segs = std::max(max_segs, h[(size_t)b + 1] - h[(size_t)b]);
    }
    grad_grid = (unsigned)std::max<int64_t>(1, std::min<int64_t>(div_up(max_segs + 1, WARPS), (int64_t)ctx->sm_count * 16));
    return GORSE_B200_OK;
}

// rows [rows] of a CSR as one prediction list, padded to its own longest row
int32_t Fit::upload_list(TestSet &T, const int64_t *off, const int32_t *idx, const float *val, const std::vector<int64_t> &rows_,
                         const int32_t *emb_row)
{
    T.n = (int64_t)rows_.size();
    GB_TRY(longest(off, rows_, num_dimension, &T.D));
    std::vector<int32_t> pi;
    std::vector<float> pv;
    pad_rows(off, idx, val, rows_, T.D, pi, pv);
    GB_TRY(T.idx.upload(pi.data(), pi.size(), st));
    GB_TRY(T.val.upload(pv.data(), pv.size(), st));
    if (emb_row) {
        std::vector<int32_t> er(rows_.size());
        for (size_t i = 0; i < er.size(); i++) er[i] = emb_row[rows_[i]];
        GB_TRY(T.emb_row.upload(er.data(), er.size(), st));
    }
    return GORSE_B200_OK;
}

int32_t Fit::upload_test(const int64_t *off, const int32_t *idx, const float *val, const float *tgt, int64_t n, const int32_t *emb_row)
{
    std::vector<int64_t> rows_[2];
    for (int64_t r = 0; r < n; r++) rows_[tgt[r] > 0 ? 0 : 1].push_back(r);
    int64_t most = 0;
    for (int s = 0; s < 2; s++) {
        GB_TRY(upload_list(te[s], off, idx, val, rows_[s], emb_row));
        most = std::max(most, te[s].n);
    }
    GB_TRY(counts.alloc(3 * MAX_TRIALS));
    GB_TRY(auc_sum.alloc(MAX_TRIALS));
    size_t need = 0;
    if (most > 0)
        GB_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, need, (const float *)nullptr, (float *)nullptr, (int)most, 0, 32, st));
    if (need > cub_tmp.n) GB_TRY(cub_tmp.alloc(need));
    return GORSE_B200_OK;
}

// the table and the row maps, and the slots' tensors in parameter order
int32_t Fit::upload_slots()
{
    base = 1 + nf * k + nf;
    if (n_emb == 0) return GORSE_B200_OK;
    row_grid = (unsigned)div_up(slot_rows, WARPS);
    int64_t total = 0;
    for (int s = 0; s < n_emb; s++) {
        maxdim = std::max(maxdim, E->dim[s]);
        const int64_t kd = (int64_t)k * E->dim[s], len[5] = {kd, kd, k, kd, k};
        for (int q = 0; q < 5; q++) tens.end[tens.n++] = (int32_t)(total += len[q]);
    }
    if (E->mask) GB_TRY(mask.upload(E->mask, (size_t)(E->n_rows * n_emb), st));
    GB_TRY(tr_row.upload(E->train_row, (size_t)n_train, st));
    for (int s = 0; s < n_emb; s++) GB_TRY(table[s].upload(E->table[s], (size_t)(E->n_rows * E->dim[s]), st));
    return GORSE_B200_OK;
}

// one trial's tables in its arena; returns the arena's bytes (DESIGN §8.8 writes them out)
size_t Fit::carve(uintptr_t b)
{
    Carver c{b};
    const int64_t opt = train ? n_params : 0;   // predictions only: no moments and no gradients
    c.take(P, n_params);
    c.take(M, opt);
    c.take(Vm, opt);
    c.take(gV, train ? nf * k : 0);
    c.take(gW, train ? nf : 0);
    c.take(gB, 1);
    c.take(g, rows);
    c.take(dss, rows);
    c.take(loss, rows);
    c.take(dvx, rows * k);
    c.take(batch_loss, n_batches);
    c.take(lr_tab, max_total);
    c.take(padnan, k + 1);
    for (TestSet &T : te) {
        c.take(T.pred, T.n);
        c.take(T.sorted, T.n);
    }
    c.take(below, te[0].n);
    if (n_emb > 0) {
        c.take(gS, train ? tens.end[tens.n - 1] : 0);
        for (float **q : {&zmax, &rowsum, &sumdx, &p}) c.take(*q, slot_rows);
        for (float **q : {&denc, &dh, &vx}) c.take(*q, slot_rows * k);
        c.take(gx, slot_rows * maxdim);
        for (int s = 0; s < n_emb; s++) {
            for (float **q : {&s_e[s], &s_y[s], &s_att[s]}) c.take(*q, slot_rows * E->dim[s]);
            for (float **q : {&s_h[s], &s_enc[s]}) c.take(*q, slot_rows * k);
        }
    }
    return c.bytes;
}

// the arenas of g trials, zeroed (M, Vm and the padding flags start at 0), and the slots' pointers into trial 0's
int32_t Fit::alloc_group(int g)
{
    G = g;
    stride = (int64_t)carve(0);
    GB_TRY(arena.alloc((size_t)stride * g));
    carve((uintptr_t)arena.p);
    GB_CUDA(cudaMemsetAsync(arena.p, 0, arena.n, st));
    if (train) GB_CUDA(cudaMemsetAsync(stamp.p, 0, (size_t)nf * sizeof(int32_t), st));   // steps count from 1
    if (n_emb == 0) return GORSE_B200_OK;
    int64_t o = base;
    logits = SlotLogits{p, vx, {}, n_emb, {}};
    for (int q = 0; q <= n_emb; q++) logits.ord[q] = VX_ORDER[n_emb][q];
    for (int s = 0; s < n_emb; s++) {
        const int d = E->dim[s];
        const int64_t kd = (int64_t)k * d;
        float *w = P + o, *gw = gS + (o - base);
        slot[s] = Slot{w, w + kd, w + 2 * kd, w + 2 * kd + k, w + 3 * kd + k, gw, gw + kd, gw + 2 * kd, gw + 2 * kd + k, gw + 3 * kd + k,
                       table[s].p, E->mask ? mask.p : nullptr, n_emb, s, d, s_e[s], s_y[s], s_att[s], s_h[s], s_enc[s],
                       zmax, rowsum, gx, denc, dh, sumdx};
        logits.enc[s] = s_enc[s];
        o += 3 * kd + 2 * k;
    }
    return GORSE_B200_OK;
}

// BatchInternalPredict (fm.go:156-178) of the list T into T.pred for the trials of Ev
int32_t Fit::predict(Group Ev, TestSet &T)
{
    if (T.n == 0) return GORSE_B200_OK;
    if (n_emb == 0) {
        fm_fit_predict_kernel<<<grid(std::min<int64_t>(div_up(T.n, WARPS), (int64_t)ctx->sm_count * 16)), WARPS * 32, 0, st>>>(
            Ev, P, nf, k, Rows{T.idx.p, T.val.p, T.D}, T.n, T.pred);
        GB_LAUNCHED(ctx);
        return GORSE_B200_OK;
    }
    // chunks of batch_size rows, each with its own softmax coupling
    const int64_t bs = prm->batch_size;
    for (int64_t ch = 0; ch * bs < T.n; ch++) {
        const Batch C{bs, T.n, (int)ch};
        fm_fit_emb_base_kernel<<<grid(row_grid), WARPS * 32, 0, st>>>(Ev, P, nf, k, Rows{T.idx.p, T.val.p, T.D}, C, T.pred + ch * bs, vx);
        GB_LAUNCHED(ctx);
        GB_TRY(slots_forward(Ev, T.emb_row.p, C, T.pred + ch * bs));
    }
    return GORSE_B200_OK;
}

// the evaluation of the trials marked in `which` (EvaluateClassification, evaluator.go:85-153 with float32 counters):
// score[i] = Precision, Recall, Accuracy, AUC of trial i
int32_t Fit::evaluate(const bool *which, float (*score)[4])
{
    int32_t flags[MAX_TRIALS] = {};
    for (int i = 0; i < G; i++)
        if (which[i]) {
            flags[i] = 1;
            std::fill(score[i], score[i] + 4, 0.0f);
        }
    const int64_t np = te[0].n, nn = te[1].n;
    if (np + nn == 0) return GORSE_B200_OK;
    GB_CUDA(cudaMemcpyAsync(ev_on.p, flags, (size_t)G * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    const Group Ev{G, stride, ev_on.p};
    for (int s = 0; s < 2; s++) {
        TestSet &T = te[s];
        if (T.n == 0) continue;
        GB_TRY(predict(Ev, T));
        for (int i = 0; i < G; i++) {
            if (!which[i]) continue;
            size_t bytes = cub_tmp.n;
            GB_CUDA(cub::DeviceRadixSort::SortKeys(cub_tmp.p, bytes, at(T.pred, i * stride), at(T.sorted, i * stride), (int)T.n, 0, 32, st));
        }
    }
    GB_CUDA(cudaMemsetAsync(counts.p, 0, 3 * (size_t)G * sizeof(unsigned long long), st));
    fm_fit_auc_counts_kernel<<<grid(std::min<int64_t>(div_up(std::max(np, nn), 256), (int64_t)ctx->sm_count * 16)), 256, 0, st>>>(
        Ev, te[0].sorted, np, te[1].sorted, nn, below, counts.p);
    GB_LAUNCHED(ctx);
    fm_fit_auc_chain_kernel<<<1, 32, 0, st>>>(Ev, below, np, auc_sum.p);
    GB_LAUNCHED(ctx);
    unsigned long long c[3 * MAX_TRIALS];
    float sum[MAX_TRIALS];
    GB_CUDA(cudaMemcpyAsync(c, counts.p, 3 * (size_t)G * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    GB_CUDA(cudaMemcpyAsync(sum, auc_sum.p, (size_t)G * sizeof(float), cudaMemcpyDeviceToHost, st));
    GB_CUDA(cudaStreamSynchronize(st));
    for (int i = 0; i < G; i++) {
        if (!which[i]) continue;
        const unsigned long long *ci = c + 3 * i;
        const float tp = go_count(ci[0]), fp = go_count(ci[1]), fn = go_count((uint64_t)np - ci[0]), correct = go_count(ci[0] + ci[2]);
        score[i][0] = tp + fp == 0.0f ? 0.0f : tp / (tp + fp);
        score[i][1] = tp + fn == 0.0f ? 0.0f : tp / (tp + fn);
        score[i][2] = correct / (float)(np + nn);
        score[i][3] = np * nn == 0 ? 0.0f : sum[i] / (float)(np * nn);
    }
    return GORSE_B200_OK;
}

int32_t Fit::run_steps(int s0, int s1)
{
    const Group Gr{G, stride, on.p};
    const Rows R{tr_idx.p, tr_val.p, D};
    const int64_t n_base = 1 + nf * k + nf, bs = prm->batch_size;
    const unsigned fwd_grid = grid(div_up(std::min<int64_t>(bs, n_train), WARPS));
    const unsigned opt_grid = grid(std::min<int64_t>(div_up(n_base, 256), (int64_t)ctx->sm_count * 8));
    for (int s = s0; s < s1; s++) {
        const Batch T{bs, n_train, s};
        if (n_emb == 0) {
            fm_fit_forward_kernel<false><<<fwd_grid, WARPS * 32, 0, st>>>(Gr, P, nf, k, R, tr_tgt.p, bs, n_train, s, g, dss, dvx, loss, tr_len.p,
                                                                           padnan, t_base.p, logits);
            GB_LAUNCHED(ctx);
        } else {
            fm_fit_emb_base_kernel<<<grid(row_grid), WARPS * 32, 0, st>>>(Gr, P, nf, k, R, T, p, vx);
            GB_LAUNCHED(ctx);
            GB_TRY(slots_forward(Gr, tr_row.p, T, p));
            fm_fit_forward_kernel<true><<<fwd_grid, WARPS * 32, 0, st>>>(Gr, P, nf, k, R, tr_tgt.p, bs, n_train, s, g, dss, dvx, loss, tr_len.p,
                                                                          padnan, t_base.p, logits);
            GB_LAUNCHED(ctx);
        }
        fm_fit_grad_kernel<<<grid(grad_grid), WARPS * 32, 0, st>>>(Gr, P, nf, k, R, bs, n_train, s, batch_seg.p, seg_start.p, seg_feat.p,
                                                                   seg_pos.p, g, dss, dvx, loss, gV, gW, gB, stamp.p, batch_loss, t_base.p,
                                                                   padnan);
        GB_LAUNCHED(ctx);
        for (int q = 0; q < n_emb; q++) {
            fm_fit_emb_datt_kernel<<<grid(row_grid), WARPS * 32, 0, st>>>(Gr, slot[q], k, T, vx, g);
            GB_LAUNCHED(ctx);
            fm_fit_emb_dh_kernel<<<grid(row_grid), WARPS * 32, 0, st>>>(Gr, slot[q], k, T);
            GB_LAUNCHED(ctx);
            fm_fit_emb_wgrad_kernel<<<grid(div_up(2 * (int64_t)slot[q].dim * k + 2 * k, 128)), 128, 0, st>>>(Gr, slot[q], k, T);
            GB_LAUNCHED(ctx);
        }
        fm_fit_opt_kernel<<<opt_grid, 256, 0, st>>>(Gr, P, M, Vm, nf, k, gV, gW, gB, stamp.p, t_base.p, s, opts);
        GB_LAUNCHED(ctx);
        if (n_emb > 0) {
            fm_fit_emb_opt_kernel<<<grid(div_up((int64_t)tens.end[tens.n - 1], 256)), 256, 0, st>>>(Gr, P, M, Vm, base, gS, tens, t_base.p, s,
                                                                                                   opts);
            GB_LAUNCHED(ctx);
        }
    }
    return GORSE_B200_OK;
}

// every slot's attention and encoder on the batch, in slot order: `logit` gets + <vx, enc> per slot
int32_t Fit::slots_forward(Group Gr, const int32_t *emb_row, Batch T, float *logit)
{
    for (int q = 0; q < n_emb; q++) {
        fm_fit_emb_hz_kernel<<<grid(row_grid), WARPS * 32, 0, st>>>(Gr, slot[q], k, emb_row, T);
        GB_LAUNCHED(ctx);
        fm_fit_emb_exp_kernel<<<grid(row_grid), WARPS * 32, 0, st>>>(Gr, slot[q], T);
        GB_LAUNCHED(ctx);
        fm_fit_emb_enc_kernel<<<grid(row_grid), WARPS * 32, 0, st>>>(Gr, slot[q], k, T, vx, logit);
        GB_LAUNCHED(ctx);
    }
    return GORSE_B200_OK;
}

int32_t check_params(const gorse_b200_fm_fit_params *p)
{
    GB_CHECK_ARG(p->n_factors >= 1 && p->n_epochs >= 0 && p->batch_size >= 1, "n_factors, batch_size >= 1 and n_epochs >= 0");
    GB_CHECK_ARG(p->verbose >= 1, "verbose must be >= 1 (the reference divides by it)");
    GB_CHECK_ARG(p->patience >= 0 && p->max_steps >= 0, "negative patience or max_steps");
    GB_CHECK_ARG(p->optimizer == GORSE_B200_FM_ADAM || p->optimizer == GORSE_B200_FM_SGD, "optimizer %d is not Adam (0) or SGD (1)",
                 p->optimizer);
    return GORSE_B200_OK;
}

// every check of the shared arguments, against params' n_factors; nothing touches the device
int32_t check_data(const Data &d, const gorse_b200_fm_fit_params *params)
{
    const int32_t n_emb = d.n_emb;
    const EmbArgs *E = d.E;
    GB_CHECK_ARG(d.n_features >= 1 && d.n_features <= INT32_MAX, "n_features = %lld is not in [1, 2^31)", (long long)d.n_features);
    GB_CHECK_ARG(d.num_dimension >= 0 && n_emb >= 0, "negative num_dimension or n_emb");
    GB_TRY(check_params(params));
    if ((n_emb > 0 && !E) || params->n_factors > MAX_FACTORS) {
        set_error("fm_fit: %d embedding slots (none supported) or n_factors %d (at most %d)", n_emb, params->n_factors, MAX_FACTORS);
        return GORSE_B200_ERR_UNSUPPORTED;
    }
    int64_t want = 1 + d.n_features * (int64_t)params->n_factors + d.n_features;
    if (n_emb > 0) {
        GB_CHECK_ARG(E->dim != nullptr && E->table != nullptr && E->n_rows >= 0, "NULL emb_dim or item_emb, or a negative n_emb_rows");
        if (n_emb > MAX_SLOTS) {
            set_error("fm_fit_emb: %d embedding slots, at most %d", n_emb, MAX_SLOTS);
            return GORSE_B200_ERR_UNSUPPORTED;
        }
        for (int s = 0; s < n_emb; s++) {
            GB_CHECK_ARG(E->dim[s] >= 1, "embedding slot %d: dim %d", s, E->dim[s]);
            if (E->dim[s] > MAX_EMB_DIM) {
                set_error("fm_fit_emb: embedding slot %d has dim %d, at most %d", s, E->dim[s], MAX_EMB_DIM);
                return GORSE_B200_ERR_UNSUPPORTED;
            }
            GB_CHECK_ARG(E->n_rows == 0 || E->table[s] != nullptr, "item_emb[%d] is NULL", s);
            want += 3 * (int64_t)params->n_factors * E->dim[s] + 2 * (int64_t)params->n_factors;
        }
        GB_CHECK_ARG((d.n_train == 0 || E->train_row != nullptr) && (d.n_test == 0 || E->test_row != nullptr),
                     "NULL train_emb_row or test_emb_row");
        for (int64_t i = 0; i < d.n_train; i++)
            GB_CHECK_ARG(E->train_row[i] >= -1 && E->train_row[i] < E->n_rows, "train row %lld: table row %d is not -1 or in [0, %lld)",
                         (long long)i, E->train_row[i], (long long)E->n_rows);
        for (int64_t i = 0; i < d.n_test; i++)
            GB_CHECK_ARG(E->test_row[i] >= -1 && E->test_row[i] < E->n_rows, "test row %lld: table row %d is not -1 or in [0, %lld)",
                         (long long)i, E->test_row[i], (long long)E->n_rows);
    }
    GB_TRY(check_rows("train", d.n_train, d.train_off, d.train_idx, d.train_val, d.train_target, d.n_features));
    GB_TRY(check_rows("test", d.n_test, d.test_off, d.test_idx, d.test_val, d.test_target, d.n_features));
    GB_CHECK_ARG(d.n_params == want, "n_params = %lld, the model has %lld", (long long)d.n_params, (long long)want);
    return GORSE_B200_OK;
}

// the optimiser steps a fit with `params` runs at most
int32_t total_steps(const Data &d, const gorse_b200_fm_fit_params *params, int64_t *out)
{
    const int64_t bs = params->batch_size, n_batches = (d.n_train + bs - 1) / bs;
    int64_t total = (int64_t)params->n_epochs * n_batches;
    if (params->max_steps > 0) total = std::min<int64_t>(total, params->max_steps);
    if (total >= INT32_MAX) {
        set_error("fm_fit: %lld optimiser steps, at most 2^31 - 1", (long long)total);
        return GORSE_B200_ERR_UNSUPPORTED;
    }
    *out = total;
    return GORSE_B200_OK;
}

struct Trial {                    // one trial's side of AFM.Fit's loop (fm.go:307-417)
    const gorse_b200_fm_fit_params *prm;
    const float *pin;
    float *pout, *mout;
    gorse_b200_fm_fit_result *res;
    int64_t total_steps = 0, steps = 0;
    std::vector<std::pair<int32_t, float>> scores;
    float score[4] = {};          // the last evaluation's Precision, Recall, Accuracy, AUC
    float cost = 0.0f;
    int32_t epochs_run = 0;
    bool done = false, cancelled = false, early_stopped = false, diverged = false;
    std::pair<int32_t, float> best() const   // lo.MaxBy(a.B > b.B) keeps the first maximum
    {
        std::pair<int32_t, float> b = scores[0];
        for (auto &s : scores) if (s.second > b.second) b = s;
        return b;
    }
};

struct Progress {                 // the callback, and every trial's state as it last saw it
    gorse_b200_fm_trials_progress_fn fn;
    void *user;
    bool sticky;                  // a cancel holds for every later call (without asking again); not with no training rows
    std::vector<gorse_b200_fm_trial_state> states;
    bool cancel = false;
    bool ask(int32_t epoch)
    {
        if (cancel) return true;
        const bool c = fn && fn(user, epoch, (int32_t)states.size(), states.data()) != 0;
        if (c && sticky) cancel = true;
        return c;
    }
};

// trials T[0, g) (states from `first`) as one group, from Init's parameters to their results
int32_t run_group(Fit &F, Trial *T, int g, int first, Progress &pg)
{
    cudaStream_t st = F.st;
    gorse_b200_ctx *ctx = F.ctx;
    const gorse_b200_fm_fit_params *sh = F.prm;
    GB_TRY(F.alloc_group(g));
    std::vector<std::vector<float>> lr_tabs((size_t)g);
    for (int i = 0; i < g; i++) {
        Trial &t = T[i];
        GB_CUDA(cudaMemcpyAsync(at(F.P, i * F.stride), t.pin, (size_t)F.n_params * sizeof(float), cudaMemcpyHostToDevice, st));
        // Adam's step size per step (optimizers.go:119-123): t counts in float32, which stops growing at 2^24
        std::vector<float> &lr = lr_tabs[(size_t)i];
        lr.assign((size_t)std::max<int64_t>(t.total_steps, 1), 0.0f);
        if (t.prm->optimizer == GORSE_B200_FM_ADAM)
            for (int64_t s = 1; s <= t.total_steps; s++) {
                const int64_t tf = std::min<int64_t>(s, int64_t(1) << 24);
                const float fix1 = 1.0f - fmx_pow_steps(0.9f, tf), fix2 = 1.0f - fmx_pow_steps(0.999f, tf);
                lr[(size_t)s - 1] = t.prm->lr * std::sqrt(fix2) / fix1;
            }
        float *lr_dev = at(F.lr_tab, i * F.stride);
        GB_CUDA(cudaMemcpyAsync(lr_dev, lr.data(), lr.size() * sizeof(float), cudaMemcpyHostToDevice, st));
        F.opts.o[i] = Opt{t.prm->optimizer == GORSE_B200_FM_ADAM, t.prm->reg, 1.0f - 0.9f, 1.0f - 0.999f, 1e-8f, t.prm->lr, lr_dev};
    }
    int32_t flags[MAX_TRIALS];
    auto set_on = [&]() -> int32_t {
        for (int i = 0; i < g; i++) flags[i] = !T[i].done;
        GB_CUDA(cudaMemcpyAsync(F.on.p, flags, (size_t)g * sizeof(int32_t), cudaMemcpyHostToDevice, st));
        return GORSE_B200_OK;
    };
    bool which[MAX_TRIALS];
    float score[MAX_TRIALS][4];
    std::fill(which, which + g, true);
    GB_TRY(F.evaluate(which, score));
    for (auto &s : pg.states) s.auc = -1.0f;
    for (int i = 0; i < g; i++) {
        Trial &t = T[i];
        std::copy(score[i], score[i] + 4, t.score);
        t.scores.assign(1, {0, score[i][3]});
        t.done = t.prm->n_epochs == 0;
        pg.states[(size_t)(first + i)] = gorse_b200_fm_trial_state{0, score[i][3], t.done};
    }
    if (pg.ask(0) && F.n_train > 0)
        for (int i = 0; i < g; i++)
            if (!T[i].done) T[i].cancelled = T[i].done = true;

    const char *ng = std::getenv("GORSE_B200_FM_FIT_NO_GRAPH");
    const bool use_graph = !(ng && ng[0] == '1') && F.n_batches > 0;
    cudaGraphExec_t exec = nullptr;
    struct GraphGuard { cudaGraphExec_t *e; ~GraphGuard() { if (*e) cudaGraphExecDestroy(*e); } } gguard{&exec};
    const int64_t nb = std::max<int64_t>(F.n_batches, 1);
    std::vector<float> bl((size_t)(g * nb));
    int64_t steps = 0;
    for (int32_t epoch = 1; std::any_of(T, T + g, [](const Trial &t) { return !t.done; }); epoch++) {
        GB_TRY(set_on());
        int64_t run = F.n_batches;
        bool limited = false;
        if (sh->max_steps > 0 && steps + run > sh->max_steps) {
            run = sh->max_steps - steps;
            limited = true;
        }
        fm_fit_set_kernel<<<1, 1, 0, st>>>(F.t_base.p, steps);
        GB_LAUNCHED(ctx);
        if (use_graph && run == F.n_batches) {
            if (!exec) {   // one capture per group: a trial that leaves is skipped through its flag in F.on
                cudaGraph_t graph = nullptr;
                GB_CUDA(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
                const int32_t rs = F.run_steps(0, (int)F.n_batches);
                const cudaError_t ce = cudaStreamEndCapture(st, &graph);
                if (rs != GORSE_B200_OK) { if (graph) cudaGraphDestroy(graph); return rs; }
                GB_CUDA(ce);
                const cudaError_t ie = cudaGraphInstantiate(&exec, graph, 0);
                cudaGraphDestroy(graph);
                GB_CUDA(ie);
            }
            GB_CUDA(cudaGraphLaunch(exec, st));
        } else {
            GB_TRY(F.run_steps(0, (int)run));
        }
        steps += run;
        for (int i = 0; i < g; i++) {
            if (T[i].done) continue;
            T[i].epochs_run = epoch;
            T[i].steps = steps;
            if (run > 0)
                GB_CUDA(cudaMemcpyAsync(bl.data() + i * nb, at(F.batch_loss, i * F.stride), (size_t)run * sizeof(float), cudaMemcpyDeviceToHost, st));
        }
        GB_CUDA(cudaStreamSynchronize(st));
        for (int i = 0; i < g; i++) {
            if (T[i].done) continue;
            float cost = 0.0f;   // the fp32 sum of the batch means in batch order
            for (int64_t b = 0; b < run; b++) cost += bl[(size_t)(i * nb + b)];
            T[i].cost = cost;
            which[i] = epoch % sh->verbose == 0 || epoch == T[i].prm->n_epochs;
        }
        if (limited) {   // max_steps: the scores stay those of the last evaluation, and no callback
            for (int i = 0; i < g; i++) T[i].done = true;
            break;
        }
        bool any = false;
        for (int i = 0; i < g; i++) any |= (which[i] = which[i] && !T[i].done);
        if (any) GB_TRY(F.evaluate(which, score));
        bool stop[MAX_TRIALS] = {};
        for (auto &s : pg.states) s.auc = -1.0f;
        for (int i = 0; i < g; i++) {
            Trial &t = T[i];
            if (t.done) continue;
            gorse_b200_fm_trial_state &s = pg.states[(size_t)(first + i)];
            if (which[i]) {
                std::copy(score[i], score[i] + 4, t.score);
                t.scores.emplace_back(epoch, score[i][3]);
                s.auc = score[i][3];
                if (std::isnan(t.cost) || std::isnan(t.score[0])) {   // score.GetValue() is Precision
                    t.diverged = stop[i] = true;
                } else if (sh->patience > 0 && epoch > sh->patience && t.best().first <= epoch - sh->patience) {
                    t.early_stopped = stop[i] = true;
                }
            }
            s.epochs_run = epoch;
            s.finished = stop[i] || epoch == t.prm->n_epochs;
        }
        const bool cancel_now = pg.ask(epoch);
        for (int i = 0; i < g; i++) {
            Trial &t = T[i];
            if (t.done) continue;
            if (stop[i] || epoch == t.prm->n_epochs) t.done = true;
            else if (cancel_now && F.n_train > 0) t.done = t.cancelled = true;
        }
    }
    for (int i = 0; i < g; i++) {
        const Trial &t = T[i];
        const size_t bytes = (size_t)F.n_params * sizeof(float);
        if (t.pout) GB_CUDA(cudaMemcpyAsync(t.pout, at(F.P, i * F.stride), bytes, cudaMemcpyDeviceToHost, st));
        if (t.mout) {
            GB_CUDA(cudaMemcpyAsync(t.mout, at(F.M, i * F.stride), bytes, cudaMemcpyDeviceToHost, st));
            GB_CUDA(cudaMemcpyAsync(t.mout + F.n_params, at(F.Vm, i * F.stride), bytes, cudaMemcpyDeviceToHost, st));
        }
    }
    GB_CUDA(cudaStreamSynchronize(st));
    for (int i = 0; i < g; i++) {
        const Trial &t = T[i];
        gorse_b200_fm_fit_result &r = *t.res;
        r = gorse_b200_fm_fit_result{};
        r.epochs_run = t.epochs_run;
        r.best_epoch = t.best().first;
        r.steps = t.steps;
        pg.states[(size_t)(first + i)].finished = 1;
        if (t.cancelled) {
            r.cancelled = 1;
            continue;
        }
        r.auc = t.score[3];
        r.precision = t.score[0];
        r.recall = t.score[1];
        r.accuracy = t.score[2];
        r.cost = t.cost;
        r.early_stopped = t.early_stopped;
        r.diverged = t.diverged;
    }
    return GORSE_B200_OK;
}

// n checked trials in groups of at most MAX_TRIALS, smaller when the arenas would not fit the free device memory
int32_t fit_groups(gorse_b200_ctx *ctx, const Data &d, int32_t n, const gorse_b200_fm_fit_params *tp, const float *const *pin,
                   float *const *pout, float *const *mout, Progress &pg, gorse_b200_fm_fit_result *results)
{
    ScopedDevice sd(ctx->device);
    Fit F;
    F.ctx = ctx;
    F.st = ctx->stream;
    F.nf = d.n_features;
    F.k = tp[0].n_factors;
    F.num_dimension = d.num_dimension;
    F.prm = &tp[0];
    F.n_train = d.n_train;
    F.n_params = d.n_params;
    F.n_emb = d.n_emb;
    F.E = d.E;
    std::vector<Trial> T((size_t)n);
    for (int32_t i = 0; i < n; i++) {
        Trial &t = T[(size_t)i];
        t.prm = &tp[i];
        t.pin = pin[i];
        t.pout = pout ? pout[i] : nullptr;
        t.mout = mout ? mout[i] : nullptr;
        t.res = &results[i];
        GB_TRY(total_steps(d, t.prm, &t.total_steps));
        F.max_total = std::max(F.max_total, t.total_steps);
    }
    GB_TRY(F.upload_train(d.train_off, d.train_idx, d.train_val, d.train_target));
    GB_TRY(F.upload_test(d.test_off, d.test_idx, d.test_val, d.test_target, d.n_test, d.n_emb > 0 ? d.E->test_row : nullptr));
    const int64_t bs = F.prm->batch_size;
    F.rows = std::max<int64_t>(1, std::min<int64_t>(bs, d.n_train));
    F.slot_rows = std::max<int64_t>(1, std::min<int64_t>(bs, std::max({d.n_train, F.te[0].n, F.te[1].n})));
    GB_TRY(F.upload_slots());
    GB_TRY(F.stamp.alloc((size_t)d.n_features));
    GB_TRY(F.t_base.alloc(1));
    GB_TRY(F.on.alloc(MAX_TRIALS));
    GB_TRY(F.ev_on.alloc(MAX_TRIALS));
    const int64_t per_trial = (int64_t)F.carve(0);
    size_t free_b = 0, total_b = 0;
    GB_CUDA(cudaMemGetInfo(&free_b, &total_b));
    const size_t reserve = size_t(256) << 20;   // the graph, cub's temporaries and the other users of the device
    const int64_t fits = free_b > reserve ? (int64_t)((free_b - reserve) / (size_t)per_trial) : 0;
    const int per = (int)std::max<int64_t>(1, std::min<int64_t>(MAX_TRIALS, fits));
    pg.states.assign((size_t)n, gorse_b200_fm_trial_state{0, -1.0f, 0});
    for (int32_t first = 0; first < n; first += per) GB_TRY(run_group(F, T.data() + first, std::min<int32_t>(per, n - first), first, pg));
    return GORSE_B200_OK;
}

struct SoloProgress {             // a solo fit's callback behind the trials' one
    gorse_b200_progress_fn fn;
    void *user;
    int32_t n_epochs;
};

int32_t solo_progress(void *user, int32_t epoch, int32_t, const gorse_b200_fm_trial_state *states)
{
    const SoloProgress *s = (const SoloProgress *)user;
    return s->fn(s->user, epoch, s->n_epochs, states[0].auc);
}

// gorse_b200_fm_fit / _fit_emb: one trial
int32_t fit_run(gorse_b200_ctx *ctx, const Data &d, const gorse_b200_fm_fit_params *params, const float *params_in, float *params_out,
                float *moments_out, gorse_b200_progress_fn progress, void *user, gorse_b200_fm_fit_result *result)
{
    GB_CHECK_ARG(ctx != nullptr && params != nullptr && result != nullptr, "NULL ctx/params/result");
    *result = gorse_b200_fm_fit_result{};
    GB_CHECK_ARG(params_in != nullptr && params_out != nullptr, "NULL params_in/params_out");
    GB_TRY(check_data(d, params));
    int64_t steps = 0;
    GB_TRY(total_steps(d, params, &steps));
    SoloProgress sp{progress, user, params->n_epochs};
    Progress pg{progress ? solo_progress : nullptr, &sp, d.n_train > 0, {}};
    return fit_groups(ctx, d, 1, params, &params_in, &params_out, &moments_out, pg, result);
}

struct GaucOut {                  // gorse_b200_fm_gauc's outputs; any may be NULL but n_scored and gauc
    float *pred;
    int32_t *user;
    int64_t *feedback, *cand;
    float *auc;
    int64_t *n_scored;
    double *gauc;
    int64_t *stats;
};

// EvaluateAFM's scoring after the fit (cmd/gorse-bench/main.go:133-206) on checked arguments: the predictions of every test
// row as one list in test order, then per user the AUC of its positives against its negatives, and GAUC
int32_t gauc_run(gorse_b200_ctx *ctx, const Data &d, const gorse_b200_fm_fit_params *prm, const float *params, int64_t n_users,
                 const int64_t *feedback, int64_t context_size, const GaucOut &o)
{
    const int64_t n = d.n_test;
    // per user: P and N, its first key in the sorted list, and whether main.go:184 scores it
    std::vector<int32_t> P((size_t)n_users, 0), N((size_t)n_users, 0);
    std::vector<uint32_t> row_hi((size_t)n);
    for (int64_t r = 0; r < n; r++) {
        const int32_t u = d.test_idx[d.test_off[r]];
        const bool neg = !(d.test_target[r] > 0);
        (neg ? N : P)[(size_t)u]++;
        row_hi[(size_t)r] = (uint32_t)u << 1 | (uint32_t)neg;
    }
    std::vector<GaucUser> scored;
    std::vector<int32_t> who;
    int64_t with_rows = 0, chained = 0;
    for (int64_t u = 0, start = 0; u < n_users; u++) {
        const int32_t p = P[(size_t)u], q = N[(size_t)u];
        with_rows += p + q > 0;
        if (p > 0 && q > 0 && feedback[u] != 0 && feedback[u] <= context_size) {
            scored.push_back(GaucUser{(int32_t)start, p, q});
            who.push_back((int32_t)u);
            chained += (int64_t)p * q > (1 << 24);
        }
        start += p + q;
    }
    const int64_t ns = (int64_t)scored.size();
    std::vector<float> auc((size_t)ns);
    if (n > 0) {
        ScopedDevice sd(ctx->device);
        Fit F;
        F.ctx = ctx;
        F.st = ctx->stream;
        F.nf = d.n_features;
        F.k = prm->n_factors;
        F.num_dimension = d.num_dimension;
        F.prm = prm;
        F.train = false;
        F.n_params = d.n_params;
        F.n_emb = d.n_emb;
        F.E = d.E;
        cudaStream_t st = F.st;
        std::vector<int64_t> all((size_t)n);
        for (int64_t r = 0; r < n; r++) all[(size_t)r] = r;
        GB_TRY(F.upload_list(F.te[0], d.test_off, d.test_idx, d.test_val, all, d.n_emb > 0 ? d.E->test_row : nullptr));
        F.slot_rows = std::min<int64_t>(prm->batch_size, n);
        GB_TRY(F.upload_slots());
        GB_TRY(F.ev_on.alloc(1));
        GB_TRY(F.alloc_group(1));
        const int32_t one = 1;
        GB_CUDA(cudaMemcpyAsync(F.ev_on.p, &one, sizeof(int32_t), cudaMemcpyHostToDevice, st));
        GB_CUDA(cudaMemcpyAsync(F.P, params, (size_t)d.n_params * sizeof(float), cudaMemcpyHostToDevice, st));
        TestSet &T = F.te[0];
        GB_TRY(F.predict(Group{1, F.stride, F.ev_on.p}, T));
        if (o.pred) GB_CUDA(cudaMemcpyAsync(o.pred, T.pred, (size_t)n * sizeof(float), cudaMemcpyDeviceToHost, st));
        if (ns > 0) {
            DevBuf<uint32_t> hi;
            DevBuf<uint64_t> key, sorted;
            DevBuf<GaucUser> us;
            DevBuf<float> auc_d;
            DevBuf<unsigned char> tmp;
            GB_TRY(hi.upload(row_hi.data(), row_hi.size(), st));
            GB_TRY(us.upload(scored.data(), scored.size(), st));
            GB_TRY(key.alloc((size_t)n));
            GB_TRY(sorted.alloc((size_t)n));
            GB_TRY(auc_d.alloc((size_t)ns));
            fm_gauc_keys_kernel<<<(unsigned)std::min<int64_t>(div_up(n, 256), (int64_t)ctx->sm_count * 16), 256, 0, st>>>(T.pred, hi.p, n, key.p);
            GB_LAUNCHED(ctx);
            int end_bit = 33;   // the bits of the largest user index above the prediction and the list bit
            while ((n_users - 1) >> (end_bit - 33)) end_bit++;
            size_t bytes = 0;
            GB_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, bytes, key.p, sorted.p, (int)n, 0, end_bit, st));
            GB_TRY(tmp.alloc(std::max<size_t>(bytes, 1)));
            GB_CUDA(cub::DeviceRadixSort::SortKeys(tmp.p, bytes, key.p, sorted.p, (int)n, 0, end_bit, st));
            fm_gauc_user_kernel<<<(unsigned)std::min<int64_t>(div_up(ns, WARPS), (int64_t)ctx->sm_count * 32), WARPS * 32, 0, st>>>(
                sorted.p, us.p, ns, auc_d.p);
            GB_LAUNCHED(ctx);
            GB_CUDA(cudaMemcpyAsync(auc.data(), auc_d.p, (size_t)ns * sizeof(float), cudaMemcpyDeviceToHost, st));
            GB_CUDA(cudaStreamSynchronize(st));   // the temporaries above are freed on return
        }
        GB_CUDA(cudaStreamSynchronize(st));
    }
    // main.go:199-206: sum += userAUC userCount and count += userCount in float32, in ascending user order, unfused
    float sum = 0.0f, count = 0.0f;
    int64_t with_nan = 0;
    for (int64_t j = 0; j < ns; j++) {
        const GaucUser &u = scored[(size_t)j];
        const float cnt = (float)((int64_t)u.P + u.N), term = auc[(size_t)j] * cnt;
        sum = sum + term;
        count = count + cnt;
        with_nan += std::isnan(auc[(size_t)j]);
        const int32_t w = who[(size_t)j];
        if (o.user) o.user[j] = w;
        if (o.feedback) o.feedback[j] = feedback[w];
        if (o.cand) o.cand[j] = (int64_t)u.P + u.N;
        if (o.auc) o.auc[j] = auc[(size_t)j];
    }
    *o.n_scored = ns;
    *o.gauc = count > 0.0f ? (double)(sum / count) : 0.0;
    if (o.stats) {
        const int64_t s[5] = {n, with_rows, ns, chained, with_nan};
        std::copy(s, s + 5, o.stats);
    }
    return GORSE_B200_OK;
}
}  // namespace

extern "C" int32_t gorse_b200_fm_fit_params_default(gorse_b200_fm_fit_params *p)
{
    GB_CHECK_ARG(p != nullptr, "params is NULL");
    // AFM.SetParams (fm.go:89-100) and NewFitConfig (model/ctr/model.go:62-68)
    *p = gorse_b200_fm_fit_params{16, 50, 0.001f, 0.0002f, GORSE_B200_FM_ADAM, 1024, 10, 10, 0};
    return GORSE_B200_OK;
}

extern "C" int32_t gorse_b200_fm_fit(gorse_b200_ctx *ctx, int64_t n_features, int32_t num_dimension, int32_t n_emb,
                                     const gorse_b200_fm_fit_params *params, int64_t n_train, const int64_t *train_off, const int32_t *train_idx,
                                     const float *train_val, const float *train_target, int64_t n_test, const int64_t *test_off,
                                     const int32_t *test_idx, const float *test_val, const float *test_target, const float *params_in,
                                     int64_t n_params, float *params_out, float *moments_out, gorse_b200_progress_fn progress, void *user,
                                     gorse_b200_fm_fit_result *result)
{
    const Data d{n_features, num_dimension, n_emb, nullptr, n_train, train_off, train_idx, train_val, train_target,
                 n_test, test_off, test_idx, test_val, test_target, n_params};
    return fit_run(ctx, d, params, params_in, params_out, moments_out, progress, user, result);
}

extern "C" int32_t gorse_b200_fm_fit_emb(gorse_b200_ctx *ctx, int64_t n_features, int32_t num_dimension, const gorse_b200_fm_fit_params *params,
                                         int64_t n_train, const int64_t *train_off, const int32_t *train_idx, const float *train_val,
                                         const float *train_target, const int32_t *train_emb_row, int64_t n_test, const int64_t *test_off,
                                         const int32_t *test_idx, const float *test_val, const float *test_target, const int32_t *test_emb_row,
                                         int32_t n_emb, const int32_t *emb_dim, int64_t n_emb_rows, const uint16_t *const *item_emb,
                                         const uint8_t *item_emb_mask, const float *params_in, int64_t n_params, float *params_out,
                                         float *moments_out, gorse_b200_progress_fn progress, void *user, gorse_b200_fm_fit_result *result)
{
    const EmbArgs E{n_emb, emb_dim, n_emb_rows, item_emb, item_emb_mask, train_emb_row, test_emb_row};
    const Data d{n_features, num_dimension, n_emb, &E, n_train, train_off, train_idx, train_val, train_target,
                 n_test, test_off, test_idx, test_val, test_target, n_params};
    return fit_run(ctx, d, params, params_in, params_out, moments_out, progress, user, result);
}

extern "C" int32_t gorse_b200_fm_fit_trials(gorse_b200_ctx *ctx, int64_t n_features, int32_t num_dimension, int32_t n_trials,
                                            const gorse_b200_fm_fit_params *trials, int64_t n_train, const int64_t *train_off,
                                            const int32_t *train_idx, const float *train_val, const float *train_target,
                                            const int32_t *train_emb_row, int64_t n_test, const int64_t *test_off, const int32_t *test_idx,
                                            const float *test_val, const float *test_target, const int32_t *test_emb_row, int32_t n_emb,
                                            const int32_t *emb_dim, int64_t n_emb_rows, const uint16_t *const *item_emb,
                                            const uint8_t *item_emb_mask, const float *const *params_in, int64_t n_params,
                                            float *const *params_out, float *const *moments_out, gorse_b200_fm_trials_progress_fn progress,
                                            void *user, gorse_b200_fm_fit_result *results)
{
    // AFM's ModelSearch trials (optimizeClickThroughRatePrediction, master/tasks.go:1318-1363): one FitConfig, one batch size
    // and one NFactors for every trial; Lr, Reg and the initial parameters differ
    GB_CHECK_ARG(n_trials >= 1, "n_trials must be >= 1, not %d", n_trials);
    GB_CHECK_ARG(trials != nullptr && params_in != nullptr && results != nullptr, "NULL trials/params_in/results");
    for (int32_t i = 0; i < n_trials; i++) results[i] = gorse_b200_fm_fit_result{};
    for (int32_t i = 0; i < n_trials; i++) GB_TRY(check_params(&trials[i]));
    const gorse_b200_fm_fit_params &a = trials[0];
    for (int32_t i = 1; i < n_trials; i++) {
        const gorse_b200_fm_fit_params &t = trials[i];
        GB_CHECK_ARG(t.n_factors == a.n_factors && t.batch_size == a.batch_size && t.verbose == a.verbose && t.patience == a.patience &&
                         t.max_steps == a.max_steps,
                     "trial %d: n_factors, batch_size, verbose, patience and max_steps must equal trial 0's", i);
    }
    for (int32_t i = 0; i < n_trials; i++) GB_CHECK_ARG(params_in[i] != nullptr, "params_in[%d] is NULL", i);
    const EmbArgs E{n_emb, emb_dim, n_emb_rows, item_emb, item_emb_mask, train_emb_row, test_emb_row};
    const Data d{n_features, num_dimension, n_emb, &E, n_train, train_off, train_idx, train_val, train_target,
                 n_test, test_off, test_idx, test_val, test_target, n_params};
    GB_TRY(check_data(d, &a));
    int64_t steps = 0;
    for (int32_t i = 0; i < n_trials; i++) GB_TRY(total_steps(d, &trials[i], &steps));
    GB_CHECK_ARG(ctx != nullptr, "ctx is NULL");
    Progress pg{progress, user, n_train > 0, {}};
    return fit_groups(ctx, d, n_trials, trials, params_in, params_out, moments_out, pg, results);
}

extern "C" int32_t gorse_b200_fm_gauc(gorse_b200_ctx *ctx, int64_t n_features, int32_t n_factors, int32_t num_dimension, int32_t batch_size,
                                      int32_t n_emb, const int32_t *emb_dim, const float *params, int64_t n_params, int64_t n_test,
                                      const int64_t *test_off, const int32_t *test_idx, const float *test_val, const float *test_target,
                                      const int32_t *test_emb_row, int64_t n_emb_rows, const uint16_t *const *item_emb,
                                      const uint8_t *item_emb_mask, int64_t n_users, const int64_t *feedback_count, int64_t context_size,
                                      float *pred_out, int32_t *user_out, int64_t *feedback_out, int64_t *cand_out, float *auc_out,
                                      int64_t *n_scored_out, double *gauc_out, int64_t *stats_out)
{
    GB_CHECK_ARG(n_scored_out != nullptr && gauc_out != nullptr, "NULL n_scored_out/gauc_out");
    *n_scored_out = 0;
    *gauc_out = 0.0;
    GB_CHECK_ARG(batch_size >= 1, "batch_size must be >= 1, not %d", batch_size);
    GB_CHECK_ARG(n_params == 0 || params != nullptr, "params is NULL");
    GB_CHECK_ARG(n_users >= 0 && n_users <= INT32_MAX, "n_users = %lld is not in [0, 2^31)", (long long)n_users);
    GB_CHECK_ARG(n_users == 0 || feedback_count != nullptr, "feedback_count is NULL");
    if (n_test > INT32_MAX) {
        set_error("fm_gauc: %lld test rows, at most 2^31 - 1 (the radix sort counts in int)", (long long)n_test);
        return GORSE_B200_ERR_UNSUPPORTED;
    }
    // the model as gorse_b200_fm_create takes it, the rows as gorse_b200_fm_fit_emb takes its test rows; no training rows
    gorse_b200_fm_fit_params prm{};
    GB_TRY(gorse_b200_fm_fit_params_default(&prm));
    prm.n_factors = n_factors;
    prm.batch_size = batch_size;
    const EmbArgs E{n_emb, emb_dim, n_emb_rows, item_emb, item_emb_mask, nullptr, test_emb_row};
    const Data d{n_features, num_dimension, n_emb, &E, 0, nullptr, nullptr, nullptr, nullptr,
                 n_test, test_off, test_idx, test_val, test_target, n_params};
    GB_TRY(check_data(d, &prm));
    for (int64_t r = 0; r < n_test; r++) {
        GB_CHECK_ARG(test_off[r + 1] > test_off[r], "test row %lld has no features, so no user", (long long)r);
        const int32_t u = test_idx[test_off[r]];
        GB_CHECK_ARG(u >= 0 && u < n_users, "test row %lld: user %d is not in [0, %lld)", (long long)r, u, (long long)n_users);
    }
    for (int64_t u = 0; u < n_users; u++)
        GB_CHECK_ARG(feedback_count[u] >= 0, "user %lld: negative feedback count", (long long)u);
    GB_CHECK_ARG(ctx != nullptr, "ctx is NULL");
    return gauc_run(ctx, d, &prm, params, n_users, feedback_count, context_size,
                    GaucOut{pred_out, user_out, feedback_out, cand_out, auc_out, n_scored_out, gauc_out, stats_out});
}
