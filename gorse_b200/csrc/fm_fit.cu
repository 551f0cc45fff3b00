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

__global__ void fm_fit_predict_kernel(const float *P, int64_t nf, int k, Rows R, int64_t n, float *pred)
{
    const int lane = threadIdx.x & 31;
    const int64_t warps = (int64_t)gridDim.x * WARPS;
    for (int64_t row = (int64_t)blockIdx.x * WARPS + (threadIdx.x >> 5); row < n; row += warps) {
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
__global__ void __launch_bounds__(WARPS * 32) fm_fit_forward_kernel(const float *P, int64_t nf, int k, Rows R, const float *tgt,
                                                                   int64_t bs, int64_t n, int s, float *g, float *dss, float *dvx,
                                                                   float *loss, const int32_t *row_len, int32_t *padnan, const int64_t *t_base,
                                                                   const __grid_constant__ SlotLogits L)
{
    const int lane = threadIdx.x & 31;
    const int64_t r0 = (int64_t)s * bs;
    const int B = (int)(n - r0 < bs ? n - r0 : bs);
    const float m = __fdiv_rn(1.0f, (float)B);                  // Mean's backward: dy / len
    for (int b = blockIdx.x * WARPS + (threadIdx.x >> 5); b < B; b += gridDim.x * WARPS) {
        float vx, p;
        if (EMB) {
            p = L.p[b];
            vx = lane < k ? L.vx[(int64_t)b * k + lane] : 0.0f;
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
                const float term = o == 0 ? sq : __fmaf_rn(L.enc[o - 1][(int64_t)b * k + lane], dp, 0.0f);   // enc dp^T, a dot of length 1
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
__global__ void __launch_bounds__(WARPS * 32) fm_fit_grad_kernel(const float *P, int64_t nf, int k, Rows R, int64_t bs, int64_t n, int s,
                                                                const int64_t *batch_seg, const int32_t *seg_start, const int32_t *seg_feat,
                                                                const int32_t *seg_pos, const float *g, const float *dss, const float *dvx,
                                                                const float *loss, float *gV, float *gW, float *gB, int32_t *stamp,
                                                                float *batch_loss, const int64_t *t_base, const int32_t *padnan)
{
    const int lane = threadIdx.x & 31;
    const int64_t r0 = (int64_t)s * bs;
    const int B = (int)(n - r0 < bs ? n - r0 : bs);
    const int32_t t = (int32_t)(*t_base + s + 1);
    const int64_t j0 = batch_seg[s], nseg = batch_seg[s + 1] - j0;
    const float *V = P + 1;
    const int64_t warps = (int64_t)gridDim.x * WARPS;
    const float qnan = __int_as_float(0x7fffffff);
    for (int64_t q = (int64_t)blockIdx.x * WARPS + (threadIdx.x >> 5); q <= nseg; q += warps) {
        if (q == 0) {
            // the padding's NaNs (fm_fit_forward_kernel) when feature 0 has no real position in the batch: they alone make
            // row 0's gradient; without any, it is +0, the same as an absent row
            if (nseg == 0 || seg_feat[j0] != 0) {
                const bool nan_v = lane < k && padnan[lane] == t, nan_w = padnan[k] == t;
                if (__any_sync(FULL, nan_v) || nan_w) {
                    if (lane < k) gV[lane] = nan_v ? qnan : 0.0f;
                    if (lane == 0) {
                        gW[0] = nan_w ? qnan : 0.0f;
                        stamp[0] = t;
                    }
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

// one optimiser step over B, V and W: the elementwise sequences of optimizers.go:138-151 (Adam) and :78-79 (SGD)
__global__ void fm_fit_opt_kernel(float *P, float *M, float *Vm, int64_t nf, int k, const float *gV, const float *gW, const float *gB,
                                  const int32_t *stamp, const int64_t *t_base, int s, Opt o)
{
    const int64_t nV = nf * k, n_params = 1 + nV + nf;
    const int64_t t = *t_base + s + 1;
    const float lr = o.adam ? o.lr_tab[t - 1] : o.sgd_lr;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n_params; e += (int64_t)gridDim.x * blockDim.x) {
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
__global__ void fm_fit_emb_opt_kernel(float *P, float *M, float *Vm, int64_t base, const float *gS, SlotTensors T, const int64_t *t_base, int s,
                                      Opt o)
{
    const int64_t t = *t_base + s + 1;
    const float lr = o.adam ? o.lr_tab[t - 1] : o.sgd_lr;
    const int32_t total = T.end[T.n - 1];
    for (int32_t e = blockIdx.x * blockDim.x + threadIdx.x; e < total; e += gridDim.x * blockDim.x) {
        int q = 0;
        while (e >= T.end[q]) q++;
        const int32_t start = q ? T.end[q - 1] : 0;
        opt_element(P, M, Vm, base + e, gS[e], e - start, T.end[q] - start, lr, o);
    }
}

#include "fm_fit_emb.cuh"

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
__global__ void fm_fit_auc_counts_kernel(const float *pos, int64_t n_pos, const float *neg, int64_t n_neg, int32_t *below,
                                         unsigned long long *counts)
{
    const int lane = threadIdx.x & 31;
    const int64_t n = n_pos > n_neg ? n_pos : n_neg;
    for (int64_t i0 = (int64_t)blockIdx.x * blockDim.x; i0 < n; i0 += (int64_t)gridDim.x * blockDim.x) {
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

// AUC's sum: float32(count) added in sequence over the positives in ascending order (evaluator.go:139-148)
__global__ void fm_fit_auc_chain_kernel(const int32_t *below, int64_t n_pos, float *sum)
{
    float acc = 0.0f;
#pragma unroll 16
    for (int64_t i = 0; i < n_pos; i++) acc = __fadd_rn(acc, __int2float_rn(below[i]));
    *sum = acc;
}

// the float32 counter of evaluator.go after n increments: exact up to 2^24, where adding 1 no longer changes it
inline float go_count(uint64_t n) { return n <= (1u << 24) ? (float)n : 16777216.0f; }

inline bool feature_ok(int64_t idx, int64_t n_features)
{
    if (idx < 0 || idx >= n_features) return false;
    return (int64_t)(float)idx < n_features;
}

template <typename T>
struct Buf : DevBuf<T> {
    ~Buf() { this->free(); }
    int32_t put(const std::vector<T> &h, cudaStream_t st)
    {
        GB_TRY(this->alloc(std::max<size_t>(h.size(), 1)));
        if (!h.empty()) GB_CUDA(cudaMemcpyAsync(this->p, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice, st));
        return GORSE_B200_OK;
    }
};

struct TestSet {                  // one list of EvaluateClassification: padded rows, their table rows and their predictions
    Buf<int32_t> idx, emb_row;
    Buf<float> val, pred, sorted;
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

struct Fit {
    gorse_b200_ctx *ctx;
    cudaStream_t st;
    int64_t nf;
    int k;
    int32_t num_dimension;
    const gorse_b200_fm_fit_params *prm;
    // training set
    Buf<int32_t> tr_idx, tr_len, seg_start, seg_feat, seg_pos, stamp, padnan;
    Buf<float> tr_val, tr_tgt;
    Buf<int64_t> batch_seg, t_base;
    int64_t n_train = 0, n_batches = 0;
    int32_t D = 0;
    unsigned grad_grid = 1;
    // model and per-step buffers
    Buf<float> P, M, Vm, gV, gW, gB, g, dss, dvx, loss, batch_loss, lr_tab;
    // evaluation
    TestSet te[2];
    Buf<int32_t> below;
    Buf<unsigned long long> counts;
    Buf<float> auc_sum;
    Buf<unsigned char> cub_tmp;

    // item-embedding slots
    int n_emb = 0;
    int64_t base = 0;             // parameters before the first slot
    Buf<uint16_t> table[MAX_SLOTS];
    Buf<uint8_t> mask;
    Buf<int32_t> tr_row;
    Buf<float> s_e[MAX_SLOTS], s_y[MAX_SLOTS], s_att[MAX_SLOTS], s_h[MAX_SLOTS], s_enc[MAX_SLOTS];
    Buf<float> zmax, rowsum, gx, denc, dh, sumdx, p, vx, gS;
    Slot slot[MAX_SLOTS];
    SlotTensors tens{};
    SlotLogits logits{};
    unsigned row_grid = 1;

    int32_t upload_train(const int64_t *off, const int32_t *idx, const float *val, const float *tgt);
    int32_t upload_test(const int64_t *off, const int32_t *idx, const float *val, const float *tgt, int64_t n, const int32_t *emb_row);
    int32_t setup_slots(const EmbArgs &E, size_t rows);
    int32_t slots_forward(const int32_t *emb_row, Batch T, float *logit);
    int32_t run_steps(int s0, int s1);
    int32_t evaluate(float *score);
};

int32_t Fit::upload_train(const int64_t *off, const int32_t *idx, const float *val, const float *tgt)
{
    std::vector<int64_t> rows((size_t)n_train);
    for (int64_t r = 0; r < n_train; r++) rows[(size_t)r] = r;
    GB_TRY(longest(off, rows, num_dimension, &D));
    const int64_t bs = prm->batch_size, np = n_train * D;
    if (np >= INT32_MAX) {
        set_error("fm_fit: %lld training positions, at most 2^31 - 1", (long long)np);
        return GORSE_B200_ERR_UNSUPPORTED;
    }
    n_batches = (n_train + bs - 1) / bs;
    std::vector<int32_t> pi;
    std::vector<float> pv;
    pad_rows(off, idx, val, rows, D, pi, pv);
    GB_TRY(tr_idx.put(pi, st));
    GB_TRY(tr_val.put(pv, st));
    GB_TRY(tr_tgt.put(std::vector<float>(tgt, tgt + n_train), st));
    std::vector<int32_t> len((size_t)n_train);
    for (int64_t r = 0; r < n_train; r++) len[(size_t)r] = (int32_t)(off[r + 1] - off[r]);
    GB_TRY(tr_len.put(len, st));
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
        Buf<uint64_t> key, key2;
        Buf<int32_t> pos, head, seg_id, seg_batch;
        GB_TRY(key.alloc((size_t)np));
        GB_TRY(key2.alloc((size_t)np));
        GB_TRY(pos.alloc((size_t)np));
        GB_TRY(head.alloc((size_t)np));
        GB_TRY(seg_id.alloc((size_t)np));
        GB_TRY(seg_batch.alloc((size_t)np));
        const unsigned grid = (unsigned)std::min<int64_t>(div_up(np, 256), (int64_t)ctx->sm_count * 16);
        fm_fit_keys_kernel<<<grid, 256, 0, st>>>(tr_idx.p, tr_len.p, D, np, bs * D, key.p, pos.p);
        GB_LAUNCHED(ctx);
        int end_bit = 32;
        while (end_bit < 64 && (uint64_t)n_batches > (1ull << (end_bit - 32))) end_bit++;
        size_t b1 = 0, b2 = 0;
        GB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, b1, key.p, key2.p, pos.p, seg_pos.p, (int)np, 0, end_bit, st));
        GB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, b2, head.p, seg_id.p, (int)n_real, st));
        GB_TRY(cub_tmp.alloc(std::max(b1, b2)));
        b1 = b2 = cub_tmp.n;
        GB_CUDA(cub::DeviceRadixSort::SortPairs(cub_tmp.p, b1, key.p, key2.p, pos.p, seg_pos.p, (int)np, 0, end_bit, st));
        fm_fit_heads_kernel<<<grid, 256, 0, st>>>(key2.p, n_real, head.p);
        GB_LAUNCHED(ctx);
        GB_CUDA(cub::DeviceScan::ExclusiveSum(cub_tmp.p, b2, head.p, seg_id.p, (int)n_real, st));
        fm_fit_segments_kernel<<<grid, 256, 0, st>>>(key2.p, head.p, seg_id.p, n_real, seg_start.p, seg_feat.p, seg_batch.p);
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

int32_t Fit::upload_test(const int64_t *off, const int32_t *idx, const float *val, const float *tgt, int64_t n, const int32_t *emb_row)
{
    std::vector<int64_t> rows[2];
    for (int64_t r = 0; r < n; r++) rows[tgt[r] > 0 ? 0 : 1].push_back(r);
    int64_t most = 0;
    for (int s = 0; s < 2; s++) {
        TestSet &T = te[s];
        T.n = (int64_t)rows[s].size();
        GB_TRY(longest(off, rows[s], num_dimension, &T.D));   // each list is padded to its own longest row
        std::vector<int32_t> pi;
        std::vector<float> pv;
        pad_rows(off, idx, val, rows[s], T.D, pi, pv);
        GB_TRY(T.idx.put(pi, st));
        GB_TRY(T.val.put(pv, st));
        if (emb_row) {
            std::vector<int32_t> er(rows[s].size());
            for (size_t i = 0; i < er.size(); i++) er[i] = emb_row[rows[s][i]];
            GB_TRY(T.emb_row.put(er, st));
        }
        GB_TRY(T.pred.alloc((size_t)std::max<int64_t>(T.n, 1)));
        GB_TRY(T.sorted.alloc((size_t)std::max<int64_t>(T.n, 1)));
        most = std::max(most, T.n);
    }
    GB_TRY(below.alloc((size_t)std::max<int64_t>(te[0].n, 1)));
    GB_TRY(counts.alloc(3));
    GB_TRY(auc_sum.alloc(1));
    size_t need = 0;
    if (most > 0) GB_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, need, te[0].pred.p, te[0].sorted.p, (int)most, 0, 32, st));
    if (need > cub_tmp.n) GB_TRY(cub_tmp.alloc(need));
    return GORSE_B200_OK;
}

int32_t Fit::evaluate(float *score)
{
    std::fill(score, score + 4, 0.0f);   // Precision, Recall, Accuracy, AUC
    const int64_t np = te[0].n, nn = te[1].n;
    if (np + nn == 0) return GORSE_B200_OK;
    const float *Pp = P.p;
    for (int s = 0; s < 2; s++) {
        TestSet &T = te[s];
        if (T.n == 0) continue;
        const unsigned grid = (unsigned)std::min<int64_t>(div_up(T.n, WARPS), (int64_t)ctx->sm_count * 16);
        if (n_emb == 0) {
            fm_fit_predict_kernel<<<grid, WARPS * 32, 0, st>>>(Pp, nf, k, Rows{T.idx.p, T.val.p, T.D}, T.n, T.pred.p);
            GB_LAUNCHED(ctx);
        } else {   // BatchInternalPredict's chunks of batch_size rows, each with its own softmax coupling
            const int64_t bs = prm->batch_size;
            for (int64_t ch = 0; ch * bs < T.n; ch++) {
                const Batch C{bs, T.n, (int)ch};
                fm_fit_emb_base_kernel<<<row_grid, WARPS * 32, 0, st>>>(Pp, nf, k, Rows{T.idx.p, T.val.p, T.D}, C, T.pred.p + ch * bs, vx.p);
                GB_LAUNCHED(ctx);
                GB_TRY(slots_forward(T.emb_row.p, C, T.pred.p + ch * bs));
            }
        }
        size_t bytes = cub_tmp.n;
        GB_CUDA(cub::DeviceRadixSort::SortKeys(cub_tmp.p, bytes, T.pred.p, T.sorted.p, (int)T.n, 0, 32, st));
    }
    GB_CUDA(cudaMemsetAsync(counts.p, 0, 3 * sizeof(unsigned long long), st));
    const unsigned grid = (unsigned)std::min<int64_t>(div_up(std::max(np, nn), 256), (int64_t)ctx->sm_count * 16);
    fm_fit_auc_counts_kernel<<<grid, 256, 0, st>>>(te[0].sorted.p, np, te[1].sorted.p, nn, below.p, counts.p);
    GB_LAUNCHED(ctx);
    fm_fit_auc_chain_kernel<<<1, 1, 0, st>>>(below.p, np, auc_sum.p);
    GB_LAUNCHED(ctx);
    unsigned long long c[3];
    float sum;
    GB_CUDA(cudaMemcpyAsync(c, counts.p, sizeof c, cudaMemcpyDeviceToHost, st));
    GB_CUDA(cudaMemcpyAsync(&sum, auc_sum.p, sizeof sum, cudaMemcpyDeviceToHost, st));
    GB_CUDA(cudaStreamSynchronize(st));
    // evaluator.go:85-153 with float32 counters
    const float tp = go_count(c[0]), fp = go_count(c[1]), fn = go_count((uint64_t)np - c[0]), correct = go_count(c[0] + c[2]);
    score[0] = tp + fp == 0.0f ? 0.0f : tp / (tp + fp);
    score[1] = tp + fn == 0.0f ? 0.0f : tp / (tp + fn);
    score[2] = correct / (float)(np + nn);
    score[3] = np * nn == 0 ? 0.0f : sum / (float)(np * nn);
    return GORSE_B200_OK;
}

int32_t Fit::run_steps(int s0, int s1)
{
    const Rows R{tr_idx.p, tr_val.p, D};
    const float wd = prm->reg;
    Opt o{prm->optimizer == GORSE_B200_FM_ADAM, wd, 1.0f - 0.9f, 1.0f - 0.999f, 1e-8f, prm->lr, lr_tab.p};
    const int64_t n_params = 1 + nf * k + nf, bs = prm->batch_size;
    const unsigned fwd_grid = (unsigned)div_up(std::min<int64_t>(bs, n_train), WARPS);
    const unsigned opt_grid = (unsigned)std::min<int64_t>(div_up(n_params, 256), (int64_t)ctx->sm_count * 8);
    for (int s = s0; s < s1; s++) {
        const Batch T{bs, n_train, s};
        if (n_emb == 0) {
            fm_fit_forward_kernel<false><<<fwd_grid, WARPS * 32, 0, st>>>(P.p, nf, k, R, tr_tgt.p, bs, n_train, s, g.p, dss.p, dvx.p, loss.p,
                                                                           tr_len.p, padnan.p, t_base.p, logits);
            GB_LAUNCHED(ctx);
        } else {
            fm_fit_emb_base_kernel<<<row_grid, WARPS * 32, 0, st>>>(P.p, nf, k, R, T, p.p, vx.p);
            GB_LAUNCHED(ctx);
            GB_TRY(slots_forward(tr_row.p, T, p.p));
            fm_fit_forward_kernel<true><<<fwd_grid, WARPS * 32, 0, st>>>(P.p, nf, k, R, tr_tgt.p, bs, n_train, s, g.p, dss.p, dvx.p, loss.p,
                                                                          tr_len.p, padnan.p, t_base.p, logits);
            GB_LAUNCHED(ctx);
        }
        fm_fit_grad_kernel<<<grad_grid, WARPS * 32, 0, st>>>(P.p, nf, k, R, bs, n_train, s, batch_seg.p, seg_start.p, seg_feat.p, seg_pos.p,
                                                             g.p, dss.p, dvx.p, loss.p, gV.p, gW.p, gB.p, stamp.p, batch_loss.p, t_base.p,
                                                             padnan.p);
        GB_LAUNCHED(ctx);
        for (int q = 0; q < n_emb; q++) {
            fm_fit_emb_datt_kernel<<<row_grid, WARPS * 32, 0, st>>>(slot[q], k, T, vx.p, g.p);
            GB_LAUNCHED(ctx);
            fm_fit_emb_dh_kernel<<<row_grid, WARPS * 32, 0, st>>>(slot[q], k, T);
            GB_LAUNCHED(ctx);
            fm_fit_emb_wgrad_kernel<<<(unsigned)div_up(2 * (int64_t)slot[q].dim * k + 2 * k, 128), 128, 0, st>>>(slot[q], k, T);
            GB_LAUNCHED(ctx);
        }
        fm_fit_opt_kernel<<<opt_grid, 256, 0, st>>>(P.p, M.p, Vm.p, nf, k, gV.p, gW.p, gB.p, stamp.p, t_base.p, s, o);
        GB_LAUNCHED(ctx);
        if (n_emb > 0) {
            fm_fit_emb_opt_kernel<<<(unsigned)div_up((int64_t)tens.end[tens.n - 1], 256), 256, 0, st>>>(P.p, M.p, Vm.p, base, gS.p, tens, t_base.p,
                                                                                                      s, o);
            GB_LAUNCHED(ctx);
        }
    }
    return GORSE_B200_OK;
}

// the table, and per slot the batch's tensors (rows: the largest batch or evaluation chunk) and the parameter pointers
int32_t Fit::setup_slots(const EmbArgs &E, size_t rows)
{
    n_emb = E.n_emb;
    base = 1 + nf * k + nf;
    if (n_emb == 0) return GORSE_B200_OK;
    row_grid = (unsigned)div_up((int64_t)rows, WARPS);
    int maxdim = 1;
    int64_t total = 0;
    for (int s = 0; s < n_emb; s++) {
        maxdim = std::max(maxdim, E.dim[s]);
        const int64_t kd = (int64_t)k * E.dim[s], len[5] = {kd, kd, k, kd, k};
        for (int q = 0; q < 5; q++) tens.end[tens.n++] = (int32_t)(total += len[q]);
    }
    if (E.mask) GB_TRY(mask.put(std::vector<uint8_t>(E.mask, E.mask + E.n_rows * n_emb), st));
    GB_TRY(tr_row.put(std::vector<int32_t>(E.train_row, E.train_row + n_train), st));
    GB_TRY(gS.alloc((size_t)total));
    for (auto *b : {&zmax, &rowsum, &sumdx, &p}) GB_TRY(b->alloc(rows));
    for (auto *b : {&denc, &dh, &vx}) GB_TRY(b->alloc(rows * k));
    GB_TRY(gx.alloc(rows * maxdim));
    int64_t o = base;
    logits = SlotLogits{p.p, vx.p, {}, n_emb, {}};
    for (int q = 0; q <= n_emb; q++) logits.ord[q] = VX_ORDER[n_emb][q];
    for (int s = 0; s < n_emb; s++) {
        const int d = E.dim[s];
        const int64_t kd = (int64_t)k * d;
        GB_TRY(table[s].put(std::vector<uint16_t>(E.table[s], E.table[s] + E.n_rows * d), st));
        for (auto *b : {&s_e[s], &s_y[s], &s_att[s]}) GB_TRY(b->alloc(rows * d));
        for (auto *b : {&s_h[s], &s_enc[s]}) GB_TRY(b->alloc(rows * k));
        float *w = P.p + o, *gw = gS.p + (o - base);
        slot[s] = Slot{w, w + kd, w + 2 * kd, w + 2 * kd + k, w + 3 * kd + k, gw, gw + kd, gw + 2 * kd, gw + 2 * kd + k, gw + 3 * kd + k,
                       table[s].p, E.mask ? mask.p : nullptr, n_emb, s, d, s_e[s].p, s_y[s].p, s_att[s].p, s_h[s].p, s_enc[s].p,
                       zmax.p, rowsum.p, gx.p, denc.p, dh.p, sumdx.p};
        logits.enc[s] = s_enc[s].p;
        o += 3 * kd + 2 * k;
    }
    return GORSE_B200_OK;
}

// every slot's attention and encoder on the batch, in slot order: `logit` gets + <vx, enc> per slot
int32_t Fit::slots_forward(const int32_t *emb_row, Batch T, float *logit)
{
    for (int q = 0; q < n_emb; q++) {
        fm_fit_emb_hz_kernel<<<row_grid, WARPS * 32, 0, st>>>(slot[q], k, emb_row, T);
        GB_LAUNCHED(ctx);
        fm_fit_emb_exp_kernel<<<row_grid, WARPS * 32, 0, st>>>(slot[q], T);
        GB_LAUNCHED(ctx);
        fm_fit_emb_enc_kernel<<<row_grid, WARPS * 32, 0, st>>>(slot[q], k, T, vx.p, logit);
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

}  // namespace

extern "C" int32_t gorse_b200_fm_fit_params_default(gorse_b200_fm_fit_params *p)
{
    GB_CHECK_ARG(p != nullptr, "params is NULL");
    // AFM.SetParams (fm.go:89-100) and NewFitConfig (model/ctr/model.go:62-68)
    *p = gorse_b200_fm_fit_params{16, 50, 0.001f, 0.0002f, GORSE_B200_FM_ADAM, 1024, 10, 10, 0};
    return GORSE_B200_OK;
}

namespace {
// E == nullptr: gorse_b200_fm_fit, which takes no embeddings and so no model with slots
int32_t fit_run(gorse_b200_ctx *ctx, int64_t n_features, int32_t num_dimension, int32_t n_emb, const EmbArgs *E,
                const gorse_b200_fm_fit_params *params, int64_t n_train, const int64_t *train_off, const int32_t *train_idx,
                const float *train_val, const float *train_target, int64_t n_test, const int64_t *test_off, const int32_t *test_idx,
                const float *test_val, const float *test_target, const float *params_in, int64_t n_params, float *params_out,
                float *moments_out, gorse_b200_progress_fn progress, void *user, gorse_b200_fm_fit_result *result)
{
    GB_CHECK_ARG(ctx != nullptr && params != nullptr && result != nullptr, "NULL ctx/params/result");
    *result = gorse_b200_fm_fit_result{};
    GB_CHECK_ARG(n_features >= 1 && n_features <= INT32_MAX, "n_features = %lld is not in [1, 2^31)", (long long)n_features);
    GB_CHECK_ARG(num_dimension >= 0 && n_emb >= 0, "negative num_dimension or n_emb");
    GB_TRY(check_params(params));
    GB_CHECK_ARG(params_in != nullptr && params_out != nullptr, "NULL params_in/params_out");
    if ((n_emb > 0 && !E) || params->n_factors > MAX_FACTORS) {
        set_error("fm_fit: %d embedding slots (none supported) or n_factors %d (at most %d)", n_emb, params->n_factors, MAX_FACTORS);
        return GORSE_B200_ERR_UNSUPPORTED;
    }
    int64_t want = 1 + n_features * (int64_t)params->n_factors + n_features;
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
        GB_CHECK_ARG((n_train == 0 || E->train_row != nullptr) && (n_test == 0 || E->test_row != nullptr), "NULL train_emb_row or test_emb_row");
        for (int64_t i = 0; i < n_train; i++)
            GB_CHECK_ARG(E->train_row[i] >= -1 && E->train_row[i] < E->n_rows, "train row %lld: table row %d is not -1 or in [0, %lld)",
                         (long long)i, E->train_row[i], (long long)E->n_rows);
        for (int64_t i = 0; i < n_test; i++)
            GB_CHECK_ARG(E->test_row[i] >= -1 && E->test_row[i] < E->n_rows, "test row %lld: table row %d is not -1 or in [0, %lld)",
                         (long long)i, E->test_row[i], (long long)E->n_rows);
    }
    GB_TRY(check_rows("train", n_train, train_off, train_idx, train_val, train_target, n_features));
    GB_TRY(check_rows("test", n_test, test_off, test_idx, test_val, test_target, n_features));
    const int k = params->n_factors;
    GB_CHECK_ARG(n_params == want, "n_params = %lld, the model has %lld", (long long)n_params, (long long)want);
    const int64_t bs = params->batch_size, n_batches = (n_train + bs - 1) / bs;
    int64_t total_steps = (int64_t)params->n_epochs * n_batches;
    if (params->max_steps > 0) total_steps = std::min<int64_t>(total_steps, params->max_steps);
    if (total_steps >= INT32_MAX) {
        set_error("fm_fit: %lld optimiser steps, at most 2^31 - 1", (long long)total_steps);
        return GORSE_B200_ERR_UNSUPPORTED;
    }

    ScopedDevice sd(ctx->device);
    Fit F;
    F.ctx = ctx;
    F.st = ctx->stream;
    F.nf = n_features;
    F.k = k;
    F.num_dimension = num_dimension;
    F.prm = params;
    F.n_train = n_train;
    cudaStream_t st = F.st;
    GB_TRY(F.upload_train(train_off, train_idx, train_val, train_target));
    GB_TRY(F.upload_test(test_off, test_idx, test_val, test_target, n_test, n_emb > 0 ? E->test_row : nullptr));
    GB_TRY(F.P.put(std::vector<float>(params_in, params_in + n_params), st));
    GB_TRY(F.M.alloc((size_t)n_params));
    GB_TRY(F.Vm.alloc((size_t)n_params));
    GB_CUDA(cudaMemsetAsync(F.M.p, 0, (size_t)n_params * sizeof(float), st));
    GB_CUDA(cudaMemsetAsync(F.Vm.p, 0, (size_t)n_params * sizeof(float), st));
    GB_TRY(F.gV.alloc((size_t)(n_features * k)));
    GB_TRY(F.gW.alloc((size_t)n_features));
    GB_TRY(F.stamp.alloc((size_t)n_features));
    GB_CUDA(cudaMemsetAsync(F.stamp.p, 0, (size_t)n_features * sizeof(int32_t), st));   // steps count from 1
    GB_TRY(F.gB.alloc(1));
    GB_TRY(F.padnan.alloc((size_t)k + 1));
    GB_CUDA(cudaMemsetAsync(F.padnan.p, 0, ((size_t)k + 1) * sizeof(int32_t), st));
    const size_t rows = (size_t)std::max<int64_t>(1, std::min<int64_t>(bs, n_train));
    if (n_emb > 0)   // the slots also run on the evaluation lists' chunks
        GB_TRY(F.setup_slots(*E, (size_t)std::max<int64_t>(1, std::min<int64_t>(bs, std::max({n_train, F.te[0].n, F.te[1].n})))));
    GB_TRY(F.g.alloc(rows));
    GB_TRY(F.dss.alloc(rows));
    GB_TRY(F.loss.alloc(rows));
    GB_TRY(F.dvx.alloc(rows * k));
    GB_TRY(F.batch_loss.alloc((size_t)std::max<int64_t>(n_batches, 1)));
    GB_TRY(F.t_base.alloc(1));
    // Adam's step size per step (optimizers.go:119-123): t counts in float32, which stops growing at 2^24
    std::vector<float> lr_tab((size_t)std::max<int64_t>(total_steps, 1), 0.0f);
    if (params->optimizer == GORSE_B200_FM_ADAM)
        for (int64_t t = 1; t <= total_steps; t++) {
            const int64_t tf = std::min<int64_t>(t, int64_t(1) << 24);
            const float fix1 = 1.0f - fmx_pow_steps(0.9f, tf), fix2 = 1.0f - fmx_pow_steps(0.999f, tf);
            lr_tab[(size_t)t - 1] = params->lr * std::sqrt(fix2) / fix1;
        }
    GB_TRY(F.lr_tab.put(lr_tab, st));

    const char *ng = std::getenv("GORSE_B200_FM_FIT_NO_GRAPH");
    const bool use_graph = !(ng && ng[0] == '1') && n_batches > 0;
    cudaGraphExec_t exec = nullptr;
    struct GraphGuard { cudaGraphExec_t *e; ~GraphGuard() { if (*e) cudaGraphExecDestroy(*e); } } gguard{&exec};

    float score[4];   // Precision, Recall, Accuracy, AUC
    GB_TRY(F.evaluate(score));
    std::vector<std::pair<int32_t, float>> scores{{0, score[3]}};
    auto best = [&]() {   // lo.MaxBy(a.B > b.B) keeps the first maximum
        std::pair<int32_t, float> b = scores[0];
        for (auto &s : scores) if (s.second > b.second) b = s;
        return b;
    };
    int64_t steps = 0;
    int32_t epochs_run = 0;
    float cost = 0.0f;
    bool cancelled = false, limited = false;
    auto cancel = [&](int32_t epoch, float auc) { return progress && progress(user, epoch, params->n_epochs, auc) != 0; };
    if (cancel(0, score[3]) && params->n_epochs >= 1 && n_train > 0) cancelled = true;
    std::vector<float> bl((size_t)std::max<int64_t>(n_batches, 1));
    for (int32_t epoch = 1; epoch <= params->n_epochs && !cancelled; epoch++) {
        int64_t run = n_batches;
        if (params->max_steps > 0 && steps + run > params->max_steps) {
            run = params->max_steps - steps;
            limited = true;
        }
        fm_fit_set_kernel<<<1, 1, 0, st>>>(F.t_base.p, steps);
        GB_LAUNCHED(ctx);
        if (use_graph && run == n_batches) {
            if (!exec) {
                cudaGraph_t graph = nullptr;
                GB_CUDA(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
                const int32_t rs = F.run_steps(0, (int)n_batches);
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
        epochs_run = epoch;
        if (run > 0) GB_CUDA(cudaMemcpyAsync(bl.data(), F.batch_loss.p, (size_t)run * sizeof(float), cudaMemcpyDeviceToHost, st));
        GB_CUDA(cudaStreamSynchronize(st));
        if (limited) {
            cost = 0.0f;
            for (int64_t b = 0; b < run; b++) cost += bl[(size_t)b];
            break;
        }
        cost = 0.0f;   // the fp32 sum of the batch means in batch order
        for (int64_t b = 0; b < run; b++) cost += bl[(size_t)b];
        bool evaluated = false, stop = false;
        if (epoch % params->verbose == 0 || epoch == params->n_epochs) {
            GB_TRY(F.evaluate(score));
            scores.emplace_back(epoch, score[3]);
            evaluated = true;
            if (std::isnan(cost) || std::isnan(score[0])) {   // score.GetValue() is Precision
                result->diverged = 1;
                stop = true;
            } else if (params->patience > 0 && epoch > params->patience && best().first <= epoch - params->patience) {
                result->early_stopped = 1;
                stop = true;
            }
        }
        const bool cancel_now = cancel(epoch, evaluated ? score[3] : -1.0f);
        if (stop) break;
        if (cancel_now && epoch < params->n_epochs && n_train > 0) cancelled = true;
    }
    GB_CUDA(cudaMemcpyAsync(params_out, F.P.p, (size_t)n_params * sizeof(float), cudaMemcpyDeviceToHost, st));
    if (moments_out) {
        GB_CUDA(cudaMemcpyAsync(moments_out, F.M.p, (size_t)n_params * sizeof(float), cudaMemcpyDeviceToHost, st));
        GB_CUDA(cudaMemcpyAsync(moments_out + n_params, F.Vm.p, (size_t)n_params * sizeof(float), cudaMemcpyDeviceToHost, st));
    }
    GB_CUDA(cudaStreamSynchronize(st));
    result->epochs_run = epochs_run;
    result->best_epoch = best().first;
    result->steps = steps;
    if (cancelled) {
        result->cancelled = 1;
        return GORSE_B200_OK;
    }
    result->auc = score[3];
    result->precision = score[0];
    result->recall = score[1];
    result->accuracy = score[2];
    result->cost = cost;
    return GORSE_B200_OK;
}
}  // namespace

extern "C" int32_t gorse_b200_fm_fit(gorse_b200_ctx *ctx, int64_t n_features, int32_t num_dimension, int32_t n_emb,
                                     const gorse_b200_fm_fit_params *params, int64_t n_train, const int64_t *train_off, const int32_t *train_idx,
                                     const float *train_val, const float *train_target, int64_t n_test, const int64_t *test_off,
                                     const int32_t *test_idx, const float *test_val, const float *test_target, const float *params_in,
                                     int64_t n_params, float *params_out, float *moments_out, gorse_b200_progress_fn progress, void *user,
                                     gorse_b200_fm_fit_result *result)
{
    return fit_run(ctx, n_features, num_dimension, n_emb, nullptr, params, n_train, train_off, train_idx, train_val, train_target, n_test,
                   test_off, test_idx, test_val, test_target, params_in, n_params, params_out, moments_out, progress, user, result);
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
    return fit_run(ctx, n_features, num_dimension, n_emb, &E, params, n_train, train_off, train_idx, train_val, train_target, n_test, test_off,
                   test_idx, test_val, test_target, params_in, n_params, params_out, moments_out, progress, user, result);
}
