// bpr.cu -- BPR pairwise SGD: the fused sample-gather-dot-sigmoid-scatter kernel.
// Replaces the body of BPR.Fit's epoch loop, model/cf/model.go:448-490 (arithmetic: SURVEY Appendix A).
//
// Roofline class: HBM/L2 bandwidth.  Algorithmic bytes per triple = 6*d*4 + 12 (3 rows read, 3 rows
// written, 3 ids).  One quad (4 lanes) owns one triple; see cf.cuh for the row->lane mapping that keeps
// the reference's AVX-512 summation order with 128-bit coalesced loads.
#include <cooperative_groups.h>

#include <algorithm>
#include <cstdlib>

#include "cf.cuh"

namespace gb {

struct BprView {
    float *P, *Q;
    const UserMeta *meta;       // per user: row offset, length, 64-bit Bloom signature of the row (one 16-byte load)
    const int32_t *user_items;
    const int32_t *active;      // nullptr when every user of the shard has feedback (active[k] == u_lo + k)
    int32_t n_active, n_items, d, u_lo;
};

// factor rows are read and written by every SM concurrently: keep them out of the (non-coherent) L1
__device__ __forceinline__ float4 ld_row(const float *p) { return __ldcg(reinterpret_cast<const float4 *>(p)); }
__device__ __forceinline__ void st_row(float *p, float4 v) { __stcg(reinterpret_cast<float4 *>(p), v); }
__device__ __forceinline__ void red_row(float *p, float4 v)
{
    asm volatile("red.relaxed.gpu.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z),
                 "f"(v.w)
                 : "memory");
}


#define GB_BPR_ROUND 8192   // triples per round of the atomic-scatter epoch (bpr_round_kernel)

#define GB_F4_OP(dst, expr)                            \
    do {                                               \
        { const int k_ = 0; (dst).x = (expr); }        \
        { const int k_ = 1; (dst).y = (expr); }        \
        { const int k_ = 2; (dst).z = (expr); }        \
        { const int k_ = 3; (dst).w = (expr); }        \
    } while (0)
__device__ __forceinline__ float f4get(const float4 &v, int k) { return k == 0 ? v.x : k == 1 ? v.y : k == 2 ? v.z : v.w; }

// gradient of -log sigmoid: model.go:471  grad = exp(-diff) / (1 + exp(-diff))   (NaN when exp overflows, SURVEY F11)
__device__ __forceinline__ float bpr_grad(float diff)
{
    float e = exp_math32(-diff);
    return __fdiv_rn(e, __fadd_rn(1.0f, e));
}

// the three rows of one triple, register resident (C = d / 16 chunks per lane)
template <int C>
struct Rows {
    float4 p[C], qi[C], qj[C];
};

// Row references are lane-local: `base` already points at this lane's first float4 and chunk c sits at
// base + c * stride floats.  A row of the factor tables has stride 16 (cf.cuh quad layout); a hot item row lives
// in the striped side table (see HotView) where consecutive pieces are whole planes apart.
template <int C>
__device__ __forceinline__ void load_rows(Rows<C> &r, const float *Pu, const float *Qi, int si, const float *Qj, int sj)
{
#pragma unroll
    for (int c = 0; c < C; c++) r.p[c] = ld_row(Pu + 16 * c);
#pragma unroll
    for (int c = 0; c < C; c++) r.qi[c] = ld_row(Qi + si * c);
#pragma unroll
    for (int c = 0; c < C; c++) r.qj[c] = ld_row(Qj + sj * c);
}

// the gradient factor of one triple whose rows are in registers (:469-471)
template <int C>
__device__ __forceinline__ float bpr_grad_rows(const Rows<C> &r, unsigned mask)
{
    float4 ai = make_float4(0.f, 0.f, 0.f, 0.f), aj = ai;
#pragma unroll
    for (int c = 0; c < C; c++) {
        dot_chunk(ai, r.p[c], r.qi[c], c == 0);
        dot_chunk(aj, r.p[c], r.qj[c], c == 0);
    }
    return bpr_grad(__fsub_rn(quad_tree(ai, mask), quad_tree(aj, mask)));
}

// the three row updates of one triple (:477-488), from the rows in registers and the gradient factor g
template <int C, bool ATOMIC>
__device__ __forceinline__ void bpr_scatter_rows(const Rows<C> &r, float g, float *Pu, float *Qi, int si, float *Qj, int sj,
                                                 float lr, float reg)
{
    const float4 *p = r.p, *qi = r.qi, *qj = r.qj;
    const float ng = -g, nreg = -reg;
#pragma unroll
    for (int c = 0; c < C; c++) {
        float4 t, o;
        // :477-479  q_i += lr * (g*p - reg*q_i)
        GB_F4_OP(t, __fmaf_rn(f4get(qi[c], k_), nreg, __fmul_rn(g, f4get(p[c], k_))));
        if (ATOMIC) { GB_F4_OP(o, __fmul_rn(f4get(t, k_), lr)); red_row(Qi + si * c, o); }
        else { GB_F4_OP(o, __fmaf_rn(f4get(t, k_), lr, f4get(qi[c], k_))); st_row(Qi + si * c, o); }
        // :481-483  q_j += lr * (-g*p - reg*q_j)
        GB_F4_OP(t, __fmaf_rn(f4get(qj[c], k_), nreg, __fmul_rn(ng, f4get(p[c], k_))));
        if (ATOMIC) { GB_F4_OP(o, __fmul_rn(f4get(t, k_), lr)); red_row(Qj + sj * c, o); }
        else { GB_F4_OP(o, __fmaf_rn(f4get(t, k_), lr, f4get(qj[c], k_))); st_row(Qj + sj * c, o); }
        // :485-488  p_u += lr * (g*(q_i - q_j) - reg*p_u)
        GB_F4_OP(t, __fmaf_rn(f4get(p[c], k_), nreg, __fmul_rn(__fsub_rn(f4get(qi[c], k_), f4get(qj[c], k_)), g)));
        if (ATOMIC) { GB_F4_OP(o, __fmul_rn(f4get(t, k_), lr)); red_row(Pu + 16 * c, o); }
        else { GB_F4_OP(o, __fmaf_rn(f4get(t, k_), lr, f4get(p[c], k_))); st_row(Pu + 16 * c, o); }
    }
}

// one SGD step by a quad on rows already in registers
template <int C, bool ATOMIC>
__device__ __forceinline__ void bpr_step_rows(const Rows<C> &r, float *Pu, float *Qi, int si, float *Qj, int sj, unsigned mask,
                                              float lr, float reg)
{
    bpr_scatter_rows<C, ATOMIC>(r, bpr_grad_rows<C>(r, mask), Pu, Qi, si, Qj, sj, lr, reg);
}

template <int C, bool ATOMIC>
__device__ __forceinline__ void bpr_step_quad(float *Pu, float *Qi, float *Qj, int lane4, unsigned mask, float lr, float reg)
{
    Rows<C> r;
    Pu += 4 * lane4; Qi += 4 * lane4; Qj += 4 * lane4;
    load_rows<C>(r, Pu, Qi, 16, Qj, 16);
    bpr_step_rows<C, ATOMIC>(r, Pu, Qi, 16, Qj, 16, mask, lr, reg);
}

// same step for any d % 16 == 0 without register-resident rows (two passes over L2-hot rows)
template <bool ATOMIC>
__device__ __forceinline__ void bpr_step_quad_dyn(float *Pu, float *Qi, float *Qj, int chunks, int lane4, unsigned mask,
                                                  float lr, float reg)
{
    Pu += 4 * lane4; Qi += 4 * lane4; Qj += 4 * lane4;
    float4 ai = make_float4(0.f, 0.f, 0.f, 0.f), aj = ai;
    for (int c = 0; c < chunks; c++) {
        float4 p = ld_row(Pu + 16 * c);
        dot_chunk(ai, p, ld_row(Qi + 16 * c), c == 0);
        dot_chunk(aj, p, ld_row(Qj + 16 * c), c == 0);
    }
    float diff = __fsub_rn(quad_tree(ai, mask), quad_tree(aj, mask));
    float g = bpr_grad(diff), ng = -g, nreg = -reg;
    for (int c = 0; c < chunks; c++) {
        float4 p = ld_row(Pu + 16 * c), qi = ld_row(Qi + 16 * c), qj = ld_row(Qj + 16 * c), t, o;
        GB_F4_OP(t, __fmaf_rn(f4get(qi, k_), nreg, __fmul_rn(g, f4get(p, k_))));
        if (ATOMIC) { GB_F4_OP(o, __fmul_rn(f4get(t, k_), lr)); red_row(Qi + 16 * c, o); }
        else { GB_F4_OP(o, __fmaf_rn(f4get(t, k_), lr, f4get(qi, k_))); st_row(Qi + 16 * c, o); }
        GB_F4_OP(t, __fmaf_rn(f4get(qj, k_), nreg, __fmul_rn(ng, f4get(p, k_))));
        if (ATOMIC) { GB_F4_OP(o, __fmul_rn(f4get(t, k_), lr)); red_row(Qj + 16 * c, o); }
        else { GB_F4_OP(o, __fmaf_rn(f4get(t, k_), lr, f4get(qj, k_))); st_row(Qj + 16 * c, o); }
        GB_F4_OP(t, __fmaf_rn(f4get(p, k_), nreg, __fmul_rn(__fsub_rn(f4get(qi, k_), f4get(qj, k_)), g)));
        if (ATOMIC) { GB_F4_OP(o, __fmul_rn(f4get(t, k_), lr)); red_row(Pu + 16 * c, o); }
        else { GB_F4_OP(o, __fmaf_rn(f4get(t, k_), lr, f4get(p, k_))); st_row(Pu + 16 * c, o); }
    }
}

template <int C, bool ATOMIC>
__device__ __forceinline__ void bpr_step_dispatch(float *Pu, float *Qi, float *Qj, int d, int lane4, unsigned mask,
                                                  float lr, float reg)
{
    if (C > 0) bpr_step_quad<(C > 0 ? C : 1), ATOMIC>(Pu, Qi, Qj, lane4, mask, lr, reg);
    else bpr_step_quad_dyn<ATOMIC>(Pu, Qi, Qj, d / 16, lane4, mask, lr, reg);
}

// any d (d % 16 != 0: 8-lane block and fused scalar tails as in the reference), one thread per triple
template <bool ATOMIC>
__device__ inline void bpr_step_any(float *Pu, float *Qi, float *Qj, int d, float lr, float reg)
{
    float diff = __fsub_rn(dot_any(Pu, Qi, d), dot_any(Pu, Qj, d));
    float g = bpr_grad(diff), ng = -g, nreg = -reg;
    for (int k = 0; k < d; k++) {
        float p = __ldcg(Pu + k), qi = __ldcg(Qi + k), qj = __ldcg(Qj + k);
        float t = axpy_elem(qi, nreg, __fmul_rn(p, g), k, d);
        if (ATOMIC) atomicAdd(Qi + k, __fmul_rn(t, lr)); else Qi[k] = axpy_elem(t, lr, qi, k, d);
        t = axpy_elem(qj, nreg, __fmul_rn(p, ng), k, d);
        if (ATOMIC) atomicAdd(Qj + k, __fmul_rn(t, lr)); else Qj[k] = axpy_elem(t, lr, qj, k, d);
        t = axpy_elem(p, nreg, __fmul_rn(__fsub_rn(qi, qj), g), k, d);
        if (ATOMIC) atomicAdd(Pu + k, __fmul_rn(t, lr)); else Pu[k] = axpy_elem(t, lr, p, k, d);
    }
}

// sampling, model.go:449-468 (distribution) on the counter RNG
__device__ __forceinline__ void sample_triple(const BprView &v, uint64_t base, int64_t step, int32_t &u, int32_t &i,
                                              int32_t &j)
{
    SStream s;
    s.x = mix64(base + (uint64_t)step);
    uint32_t ua = s.bounded((uint32_t)v.n_active);
    u = v.active ? __ldg(v.active + ua) : v.u_lo + (int32_t)ua;
    const UserMeta m = ld_meta(v.meta + (u - v.u_lo));
    const int64_t o = m.off();
    const int64_t len = m.len();
    i = __ldg(v.user_items + o + s.bounded((uint32_t)len));
    j = -1;
    if (len < v.n_items) {
        for (;;) {
            int32_t c = (int32_t)s.bounded((uint32_t)v.n_items);
            // the Bloom signature answers "certainly not in R_u" for most candidates without touching the row
            if (!m.maybe_contains(c) || !row_contains(v.user_items + o, len, c)) { j = c; break; }
        }
    }
}

// ---- kernels -----------------------------------------------------------------------------------
template <int C, bool ATOMIC>
__global__ void __launch_bounds__(256) bpr_epoch_kernel(BprView v, int64_t step0, int64_t n_steps, uint64_t base, float lr, float reg)
{
    const int lane4 = threadIdx.x & 3;
    const unsigned mask = quad_mask();
    int64_t q = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 2;
    const int64_t nq = ((int64_t)gridDim.x * blockDim.x) >> 2;
    if (C > 0) {
        // software pipeline: the row gathers of step k are in flight while step k+1 is being sampled
        // (its own chain of 2-3 dependent index loads), so one iteration costs one memory round trip
        constexpr int CC = C > 0 ? C : 1;
        int32_t u = 0, i = 0, j = -1;
        if (q < n_steps) sample_triple(v, base, step0 + q, u, i, j);
        while (q < n_steps) {
            Rows<CC> r;
            const bool live = j >= 0;
            float *Pu = v.P + (int64_t)(u - v.u_lo) * v.d + 4 * lane4, *Qi = v.Q + (int64_t)i * v.d + 4 * lane4,
                  *Qj = v.Q + (int64_t)(live ? j : 0) * v.d + 4 * lane4;
            if (live) load_rows<CC>(r, Pu, Qi, 16, Qj, 16);
            const int64_t qn = q + nq;
            int32_t un = 0, in = 0, jn = -1;
            if (qn < n_steps) sample_triple(v, base, step0 + qn, un, in, jn);
            if (live) bpr_step_rows<CC, ATOMIC>(r, Pu, Qi, 16, Qj, 16, mask, lr, reg);
            q = qn; u = un; i = in; j = jn;
        }
    } else {
        for (; q < n_steps; q += nq) {
            int32_t u, i, j;
            sample_triple(v, base, step0 + q, u, i, j);
            if (j < 0) continue;
            bpr_step_dispatch<C, ATOMIC>(v.P + (int64_t)(u - v.u_lo) * v.d, v.Q + (int64_t)i * v.d, v.Q + (int64_t)j * v.d,
                                         v.d, lane4, mask, lr, reg);
        }
    }
}

// The epoch with atomic scatter, in rounds of one triple per quad of the (co-resident) grid: every triple of a round reads
// its rows as the previous round left them, a grid-wide barrier separates those reads from the round's additions, and a
// second one ends the round.  What a triple reads therefore depends only on the step stream and the round size, not on
// timing; the order of the float additions into a row that several triples of one round update is the only freedom left
// (rounding).  The round size bounds the staleness of a popular row: at GB_BPR_ROUND triples the most popular item of a
// Zipf(1) catalogue of 10^5 items takes ~700 updates from one copy per round, lr * reg * 700 << 2.
template <int C>
__global__ void __launch_bounds__(256) bpr_round_kernel(BprView v, int64_t step0, int64_t n_steps, uint64_t base, float lr, float reg)
{
    namespace cg = cooperative_groups;
    cg::grid_group grid = cg::this_grid();
    const int lane4 = threadIdx.x & 3;
    const unsigned mask = quad_mask();
    const int64_t q = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 2;
    const int64_t nq = ((int64_t)gridDim.x * blockDim.x) >> 2;
    int32_t u = 0, i = 0, j = -1;
    if (q < n_steps) sample_triple(v, base, step0 + q, u, i, j);
    for (int64_t r0 = 0; r0 < n_steps; r0 += nq) {
        const bool live = j >= 0;
        float *Pu = v.P + (int64_t)(u - v.u_lo) * v.d + 4 * lane4, *Qi = v.Q + (int64_t)i * v.d + 4 * lane4,
              *Qj = v.Q + (int64_t)(live ? j : 0) * v.d + 4 * lane4;
        Rows<C> r;
        float g = 0.f;
        if (live) {
            load_rows<C>(r, Pu, Qi, 16, Qj, 16);
            g = bpr_grad_rows<C>(r, mask);   // consumes every loaded value before the barrier
        }
        grid.sync();
        if (live) bpr_scatter_rows<C, true>(r, g, Pu, Qi, 16, Qj, 16, lr, reg);
        // the next round's triple (the sampler reads only the immutable CSR) while the additions drain
        j = -1;
        if (r0 + nq + q < n_steps) sample_triple(v, base, step0 + r0 + nq + q, u, i, j);
        grid.sync();
    }
}

template <int C, bool ATOMIC>
__global__ void __launch_bounds__(256) bpr_apply_kernel(BprView v, const int32_t *uij, int64_t n, float lr, float reg)
{
    const int lane4 = threadIdx.x & 3;
    const unsigned mask = quad_mask();
    int64_t q = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 2;
    const int64_t nq = ((int64_t)gridDim.x * blockDim.x) >> 2;
    for (; q < n; q += nq) {
        int32_t u = __ldg(uij + 3 * q), i = __ldg(uij + 3 * q + 1), j = __ldg(uij + 3 * q + 2);
        if (j < 0) continue;
        bpr_step_dispatch<C, ATOMIC>(v.P + (int64_t)(u - v.u_lo) * v.d, v.Q + (int64_t)i * v.d, v.Q + (int64_t)j * v.d,
                                     v.d, lane4, mask, lr, reg);
    }
}

template <bool ATOMIC>
__global__ void __launch_bounds__(128) bpr_epoch_any_kernel(BprView v, int64_t step0, int64_t n_steps, uint64_t base, float lr, float reg)
{
    int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t nq = (int64_t)gridDim.x * blockDim.x;
    for (; q < n_steps; q += nq) {
        int32_t u, i, j;
        sample_triple(v, base, step0 + q, u, i, j);
        if (j < 0) continue;
        bpr_step_any<ATOMIC>(v.P + (int64_t)(u - v.u_lo) * v.d, v.Q + (int64_t)i * v.d, v.Q + (int64_t)j * v.d, v.d, lr, reg);
    }
}

template <bool ATOMIC>
__global__ void __launch_bounds__(128) bpr_apply_any_kernel(BprView v, const int32_t *uij, int64_t n, float lr, float reg)
{
    int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t nq = (int64_t)gridDim.x * blockDim.x;
    for (; q < n; q += nq) {
        int32_t u = uij[3 * q], i = uij[3 * q + 1], j = uij[3 * q + 2];
        if (j < 0) continue;
        bpr_step_any<ATOMIC>(v.P + (int64_t)(u - v.u_lo) * v.d, v.Q + (int64_t)i * v.d, v.Q + (int64_t)j * v.d, v.d, lr, reg);
    }
}

__global__ void bpr_sample_kernel(BprView v, uint64_t base, int64_t first, int64_t n, int32_t *out)
{
    int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t nq = (int64_t)gridDim.x * blockDim.x;
    for (; q < n; q += nq) {
        int32_t u, i, j;
        sample_triple(v, base, first + q, u, i, j);
        out[3 * q] = u; out[3 * q + 1] = i; out[3 * q + 2] = j;
    }
}

// ---- distributed item-factor exchange ------------------------------------------------------------
// Each rank runs its share of the epoch against its replica Q_r of the item table (started from the common Q0);
// then  Q <- Q0 + s_i * sum_r (Q_r - Q0)  row by row.  Plainly summing the deltas (s = 1) is what one replica
// would have done only while every row moves a small fraction of the way to its local fixed point per epoch.  A
// row that is updated n times moves the fraction a = 1 - (1 - lr*kappa)^n of that way (kappa = reg + curvature of
// the logistic loss), so W ranks summed overshoot by the factor W*a: for the head of the popularity distribution
// a ~ 1 and the sum diverges within a few epochs once W > 2 (tools/dist_rule_sim.py reproduces it with the CPU
// oracle).  Composing the W relaxations one after the other, as the single replica does, gives the total fraction
// 1 - prod_r (1 - a_r); scaling the summed delta by  s_i = (1 - prod_r (1 - a_ir)) / sum_r a_ir  keeps the plain sum
// for rarely-updated rows (s -> 1) and turns into the average of the replicas for saturated ones (s -> 1/W).
// n_ir is the EXPECTED update count (item_rate * local steps), kappa = reg + 2*E|p|^2/d (isotropic estimate of
// 0.25*lambda_max(E[p p^T]) with a safety factor of 8 for anisotropy), E|p|^2 sampled from the local user shard.
__global__ void q_delta_kernel(float4 *q, const float4 *q0, int64_t n4)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, st = (int64_t)gridDim.x * blockDim.x;
    for (; i < n4; i += st) {
        float4 a = q[i], b = q0[i];
        q[i] = make_float4(a.x - b.x, a.y - b.y, a.z - b.z, a.w - b.w);
    }
}
__global__ void q_delta_scalar_kernel(float *q, const float *q0, int64_t n)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, st = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += st) q[i] = q[i] - q0[i];
}
// one warp per sampled row: psq[0] += |p|^2, psq[1] += 1
__global__ void p_norm_sample_kernel(const float *P, int64_t n_rows, int d, int64_t stride, int64_t n_sample, float *psq)
{
    const int lane = threadIdx.x & 31;
    int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    float acc = 0.f, cnt = 0.f;
    for (; w < n_sample; w += nw) {
        const int64_t r = w * stride;
        if (r >= n_rows) break;
        const float *row = P + r * d;
        for (int f = lane; f < d; f += 32) { float x = row[f]; acc += x * x; }
        cnt += 1.f;
    }
    for (int o = 16; o; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0 && cnt > 0.f) { atomicAdd(&psq[0], acc); atomicAdd(&psq[1], cnt); }
}
// xchg = [ a (n_items) | L (n_items) | psq (2) ]: a_i = 1 - (1 - lr*kappa)^{n_i}, L_i = n_i * log(1 - lr*kappa)
__global__ void xchg_prepare_kernel(const float *rate, int32_t n_items, float n_local_steps, float lr, float reg, int d, float *xchg)
{
    const float *psq = xchg + 2 * (int64_t)n_items;
    const float p2 = psq[1] > 0.f ? psq[0] / psq[1] : 0.f;
    const float kappa = reg + 2.0f * p2 / (float)d;
    const float l1 = log1pf(-fminf(fmaxf(lr * kappa, 0.f), 0.5f));
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    for (; i < n_items; i += gridDim.x * blockDim.x) {
        const float L = n_local_steps * rate[i] * l1;
        xchg[i] = -expm1f(L);
        xchg[n_items + i] = L;
    }
}
__device__ __forceinline__ float xchg_scale(const float *xchg, int32_t n_items, int32_t i)
{
    const float a = xchg[i], L = xchg[n_items + i];
    return a > 1e-12f ? fminf(1.0f, -expm1f(L) / a) : 1.0f;
}
__global__ void q_apply_kernel(float4 *q, float4 *q0, int64_t n4, int d4, const float *xchg, int32_t n_items)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, st = (int64_t)gridDim.x * blockDim.x;
    for (; i < n4; i += st) {
        const float s = xchg_scale(xchg, n_items, (int32_t)(i / d4));
        float4 a = q[i], b = q0[i];
        float4 r = make_float4(b.x + s * a.x, b.y + s * a.y, b.z + s * a.z, b.w + s * a.w);
        q[i] = r;
        q0[i] = r;
    }
}
__global__ void q_apply_scalar_kernel(float *q, float *q0, int64_t n, int d, const float *xchg, int32_t n_items)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, st = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += st) { float r = q0[i] + xchg_scale(xchg, n_items, (int32_t)(i / d)) * q[i]; q[i] = r; q0[i] = r; }
}

static BprView make_view(gorse_b200_cf *cf)
{
    BprView v;
    v.P = cf->P.p; v.Q = cf->Q.p;
    v.meta = cf->user_meta.p; v.user_items = cf->user_items.p;
    v.active = cf->all_active ? nullptr : cf->active.p;
    v.n_active = cf->n_active; v.n_items = cf->n_items; v.d = cf->d; v.u_lo = cf->u_lo;
    return v;
}

// grid: persistent, a multiple of the SM count (H100: 132 SMs); 256 threads = 64 quads per CTA
static int quad_grid(const gorse_b200_ctx *c, int64_t n_quads, int ctas_per_sm)
{
    int64_t want = (n_quads + 63) / 64;
    if (const char *e = getenv("GORSE_B200_BPR_CTAS")) { int v = atoi(e); if (v > 0) return (int)std::min<int64_t>(want, v); }  // experiments only
    int64_t cap = (int64_t)c->sm_count * ctas_per_sm;
    return (int)std::max<int64_t>(1, std::min(want, cap));
}

template <int C>
static int32_t launch_round_epoch(gorse_b200_cf *cf, BprView v, int64_t step0, int64_t n, uint64_t base, float lr, float reg)
{
    gorse_b200_ctx *c = cf->ctx;
    auto *k = bpr_round_kernel<C>;
    int per_sm = 0;
    GB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k, 256, 0));
    // the round size is fixed (GB_BPR_ROUND triples) unless the device cannot hold that many quads at once
    const int g = (int)std::min<int64_t>(GB_BPR_ROUND / 64, (int64_t)per_sm * c->sm_count);
    if (g < 1) { set_error("bpr_round_kernel does not fit on the device"); return GORSE_B200_ERR_UNSUPPORTED; }
    void *args[] = {&v, &step0, &n, &base, &lr, &reg};
    GB_CUDA(cudaLaunchCooperativeKernel((const void *)k, dim3(g), dim3(256), args, 0, c->stream));
    return GORSE_B200_OK;
}

template <bool ATOMIC>
static void launch_epoch(gorse_b200_cf *cf, const BprView &v, int64_t step0, int64_t n, uint64_t base, float lr, float reg)
{
    gorse_b200_ctx *c = cf->ctx;
    cudaStream_t s = c->stream;
    if (cf->d % 16 == 0) {
        int C = cf->d / 16;
        int g = quad_grid(c, n, C <= 4 ? 8 : 4);
        switch (C) {
            case 1: bpr_epoch_kernel<1, ATOMIC><<<g, 256, 0, s>>>(v, step0, n, base, lr, reg); break;
            case 2: bpr_epoch_kernel<2, ATOMIC><<<g, 256, 0, s>>>(v, step0, n, base, lr, reg); break;
            case 4: bpr_epoch_kernel<4, ATOMIC><<<g, 256, 0, s>>>(v, step0, n, base, lr, reg); break;
            case 8: bpr_epoch_kernel<8, ATOMIC><<<g, 256, 0, s>>>(v, step0, n, base, lr, reg); break;
            default: bpr_epoch_kernel<0, ATOMIC><<<g, 256, 0, s>>>(v, step0, n, base, lr, reg); break;
        }
    } else {
        int g = (int)std::max<int64_t>(1, std::min<int64_t>((n + 127) / 128, (int64_t)c->sm_count * 8));
        bpr_epoch_any_kernel<ATOMIC><<<g, 128, 0, s>>>(v, step0, n, base, lr, reg);
    }
}

template <bool ATOMIC>
static void launch_apply(gorse_b200_cf *cf, const BprView &v, const int32_t *d_uij, int64_t n, float lr, float reg)
{
    gorse_b200_ctx *c = cf->ctx;
    cudaStream_t s = c->stream;
    if (cf->d % 16 == 0) {
        int C = cf->d / 16;
        int g = quad_grid(c, n, C <= 4 ? 8 : 4);
        switch (C) {
            case 1: bpr_apply_kernel<1, ATOMIC><<<g, 256, 0, s>>>(v, d_uij, n, lr, reg); break;
            case 2: bpr_apply_kernel<2, ATOMIC><<<g, 256, 0, s>>>(v, d_uij, n, lr, reg); break;
            case 4: bpr_apply_kernel<4, ATOMIC><<<g, 256, 0, s>>>(v, d_uij, n, lr, reg); break;
            case 8: bpr_apply_kernel<8, ATOMIC><<<g, 256, 0, s>>>(v, d_uij, n, lr, reg); break;
            default: bpr_apply_kernel<0, ATOMIC><<<g, 256, 0, s>>>(v, d_uij, n, lr, reg); break;
        }
    } else {
        int g = (int)std::max<int64_t>(1, std::min<int64_t>((n + 127) / 128, (int64_t)c->sm_count * 8));
        bpr_apply_any_kernel<ATOMIC><<<g, 128, 0, s>>>(v, d_uij, n, lr, reg);
    }
}

}  // namespace gb

using namespace gb;

extern "C" {

int32_t gorse_b200_bpr_apply_triples(gorse_b200_cf *cf, const int32_t *uij, int64_t n, float lr, float reg,
                                     int32_t scatter, int32_t order)
{
    GB_CHECK_ARG(cf != nullptr, "cf is NULL");
    GB_CHECK_ARG(n >= 0, "negative n");
    GB_CHECK_ARG(scatter == GORSE_B200_SCATTER_STORE || scatter == GORSE_B200_SCATTER_ATOMIC, "bad scatter mode %d", scatter);
    GB_CHECK_ARG(order == GORSE_B200_ORDER_HOGWILD || order == GORSE_B200_ORDER_SEQUENTIAL, "bad order %d", order);
    if (n == 0) return GORSE_B200_OK;
    GB_CHECK_ARG(uij != nullptr, "uij is NULL");
    for (int64_t t = 0; t < n; t++) {
        int32_t u = uij[3 * t], i = uij[3 * t + 1], j = uij[3 * t + 2];
        if (j < 0) continue;
        GB_CHECK_ARG(u >= cf->u_lo && u < cf->u_hi, "triple %lld: user %d outside shard [%d, %d)", (long long)t, u, cf->u_lo, cf->u_hi);
        GB_CHECK_ARG(i >= 0 && i < cf->n_items && j < cf->n_items, "triple %lld: item out of range", (long long)t);
    }
    ScopedDevice sd(cf->ctx->device);
    gorse_b200_ctx *c = cf->ctx;
    BprView v = make_view(cf);
    DevBuf<int32_t> d_uij;
    GB_TRY(d_uij.alloc((size_t)3 * n));
    auto done = [&](int32_t s) {
        cudaStreamSynchronize(c->stream);
        d_uij.free();
        return s;
    };
    auto check = [&]() -> int32_t {
        c->launches++;
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) {
            set_error("bpr_apply launch: %s", cudaGetErrorString(e));
            return GORSE_B200_ERR_CUDA;
        }
        return GORSE_B200_OK;
    };
    if (order == GORSE_B200_ORDER_HOGWILD) {
        cudaError_t e = cudaMemcpyAsync(d_uij.p, uij, sizeof(int32_t) * 3 * n, cudaMemcpyHostToDevice, c->stream);
        if (e != cudaSuccess) { set_error("upload: %s", cudaGetErrorString(e)); return done(GORSE_B200_ERR_CUDA); }
        if (scatter == GORSE_B200_SCATTER_ATOMIC) launch_apply<true>(cf, v, d_uij.p, n, lr, reg);
        else launch_apply<false>(cf, v, d_uij.p, n, lr, reg);
        int32_t st = check();
        if (st) return done(st);
    } else {
        // conflict-free waves: wave(t) = 1 + max(last wave that touched u, i or j).  Launching the waves in
        // order is exactly the reference with Jobs = 1 on this triple stream.
        std::vector<int32_t> last_u((size_t)(cf->u_hi - cf->u_lo), 0), last_i((size_t)cf->n_items, 0), wave((size_t)n, 0);
        int32_t n_waves = 0;
        for (int64_t t = 0; t < n; t++) {
            int32_t u = uij[3 * t] - cf->u_lo, i = uij[3 * t + 1], j = uij[3 * t + 2];
            if (j < 0) { wave[t] = 0; continue; }
            int32_t w = 1 + std::max(last_u[u], std::max(last_i[i], last_i[j]));
            wave[t] = w;
            last_u[u] = last_i[i] = last_i[j] = w;
            n_waves = std::max(n_waves, w);
        }
        std::vector<int64_t> start((size_t)n_waves + 2, 0);
        for (int64_t t = 0; t < n; t++) start[(size_t)wave[t] + 1]++;
        for (int32_t w = 0; w <= n_waves; w++) start[(size_t)w + 1] += start[w];
        std::vector<int32_t> sorted((size_t)3 * n);
        std::vector<int64_t> pos(start.begin(), start.end() - 1);
        for (int64_t t = 0; t < n; t++) {
            int64_t p = pos[wave[t]]++;
            sorted[3 * p] = uij[3 * t]; sorted[3 * p + 1] = uij[3 * t + 1]; sorted[3 * p + 2] = uij[3 * t + 2];
        }
        cudaError_t e = cudaMemcpyAsync(d_uij.p, sorted.data(), sizeof(int32_t) * 3 * n, cudaMemcpyHostToDevice, c->stream);
        if (e != cudaSuccess) { set_error("upload: %s", cudaGetErrorString(e)); return done(GORSE_B200_ERR_CUDA); }
        for (int32_t w = 1; w <= n_waves; w++) {
            int64_t cnt = start[(size_t)w + 1] - start[w];
            if (cnt == 0) continue;
            if (scatter == GORSE_B200_SCATTER_ATOMIC) launch_apply<true>(cf, v, d_uij.p + 3 * start[w], cnt, lr, reg);
            else launch_apply<false>(cf, v, d_uij.p + 3 * start[w], cnt, lr, reg);
            int32_t st = check();
            if (st) return done(st);
        }
        cudaError_t e2 = cudaStreamSynchronize(c->stream);  // `sorted` dies here
        if (e2 != cudaSuccess) { set_error("bpr_apply: %s", cudaGetErrorString(e2)); return done(GORSE_B200_ERR_CUDA); }
    }
    cudaError_t e = cudaStreamSynchronize(c->stream);
    if (e != cudaSuccess) { set_error("bpr_apply: %s", cudaGetErrorString(e)); return done(GORSE_B200_ERR_CUDA); }
    return done(GORSE_B200_OK);
}

int32_t gorse_b200_bpr_sample_triples(gorse_b200_cf *cf, uint64_t seed, int64_t first_step, int64_t n, int32_t *uij_out)
{
    GB_CHECK_ARG(cf != nullptr, "cf is NULL");
    GB_CHECK_ARG(n >= 0 && first_step >= 0, "negative n/first_step");
    if (n == 0) return GORSE_B200_OK;
    GB_CHECK_ARG(uij_out != nullptr, "uij_out is NULL");
    if (cf->n_active == 0) { set_error("no user with feedback in this shard"); return GORSE_B200_ERR_STATE; }
    ScopedDevice sd(cf->ctx->device);
    gorse_b200_ctx *c = cf->ctx;
    DevBuf<int32_t> d;
    GB_TRY(d.alloc((size_t)3 * n));
    int g = (int)std::max<int64_t>(1, std::min<int64_t>((n + 127) / 128, (int64_t)c->sm_count * 8));
    bpr_sample_kernel<<<g, 128, 0, c->stream>>>(make_view(cf), mix64(seed), first_step, n, d.p);
    c->launches++;
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaMemcpyAsync(uij_out, d.p, sizeof(int32_t) * 3 * n, cudaMemcpyDeviceToHost, c->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
    d.free();
    if (e != cudaSuccess) { set_error("bpr_sample: %s", cudaGetErrorString(e)); return GORSE_B200_ERR_CUDA; }
    return GORSE_B200_OK;
}

int32_t gorse_b200_bpr_epoch(gorse_b200_cf *cf, float lr, float reg, int64_t n_steps, uint64_t seed, int32_t scatter)
{
    GB_CHECK_ARG(cf != nullptr, "cf is NULL");
    GB_CHECK_ARG(n_steps >= 0, "negative n_steps");
    GB_CHECK_ARG(scatter == GORSE_B200_SCATTER_STORE || scatter == GORSE_B200_SCATTER_ATOMIC, "bad scatter mode %d", scatter);
    ScopedDevice sd(cf->ctx->device);
    gorse_b200_ctx *c = cf->ctx;
    // rank r runs steps [n*r/W, n*(r+1)/W) of the global step stream on its own user shard
    int64_t s0 = n_steps * c->rank / c->world, s1 = n_steps * (c->rank + 1) / c->world;
    if (s1 > s0 && cf->n_active == 0 && c->world == 1) { set_error("no user with feedback"); return GORSE_B200_ERR_STATE; }
    // a rank whose shard has no feedback runs zero local steps and still joins the exchange below
    if (s1 > s0 && cf->n_active > 0) {
        BprView v = make_view(cf);
        const int C = cf->d / 16;
        const int64_t n_local = s1 - s0;
        if (scatter == GORSE_B200_SCATTER_ATOMIC && cf->d % 16 == 0 && (C == 1 || C == 2 || C == 4 || C == 8)) {
            int32_t st = C == 1 ? launch_round_epoch<1>(cf, v, s0, n_local, mix64(seed), lr, reg)
                       : C == 2 ? launch_round_epoch<2>(cf, v, s0, n_local, mix64(seed), lr, reg)
                       : C == 4 ? launch_round_epoch<4>(cf, v, s0, n_local, mix64(seed), lr, reg)
                                : launch_round_epoch<8>(cf, v, s0, n_local, mix64(seed), lr, reg);
            if (st) return st;
        } else if (scatter == GORSE_B200_SCATTER_ATOMIC) {
            launch_epoch<true>(cf, v, s0, n_local, mix64(seed), lr, reg);
        } else {
            launch_epoch<false>(cf, v, s0, n_local, mix64(seed), lr, reg);
        }
        GB_LAUNCHED(c);
    }
    if (c->world > 1) {
        int64_t n = (int64_t)cf->Q.n;
        int g = c->sm_count * 8;
        if (cf->d % 4 == 0) q_delta_kernel<<<g, 256, 0, c->stream>>>((float4 *)cf->Q.p, (const float4 *)cf->Q0.p, n / 4);
        else q_delta_scalar_kernel<<<g, 256, 0, c->stream>>>(cf->Q.p, cf->Q0.p, n);
        GB_LAUNCHED(c);
        // per-row damping inputs (see the comment above q_delta_kernel)
        float *psq = cf->xchg.p + 2 * (int64_t)cf->n_items;
        GB_CUDA(cudaMemsetAsync(psq, 0, 4 * sizeof(float), c->stream));
        const int64_t n_rows = cf->u_hi - cf->u_lo;
        if (n_rows > 0 && s1 > s0 && cf->n_active > 0) {
            const int64_t n_sample = std::min<int64_t>(n_rows, 65536), stride = std::max<int64_t>(1, n_rows / n_sample);
            p_norm_sample_kernel<<<(int)std::min<int64_t>(div_up(n_sample * 32, 256), c->sm_count * 8), 256, 0, c->stream>>>(cf->P.p, n_rows, cf->d, stride, n_sample, psq);
            GB_LAUNCHED(c);
        }
        xchg_prepare_kernel<<<(int)std::min<int64_t>(div_up(cf->n_items, 256), c->sm_count * 8), 256, 0, c->stream>>>(cf->item_rate.p, cf->n_items, (float)(cf->n_active > 0 ? s1 - s0 : 0), lr, reg, cf->d, cf->xchg.p);
        GB_LAUNCHED(c);
        GB_NCCL_API(nc);
        GB_NCCL(nc, AllReduce(cf->Q.p, cf->Q.p, (size_t)n, ncclFloat32, ncclSum, c->comm, c->stream));
        GB_NCCL(nc, AllReduce(cf->xchg.p, cf->xchg.p, (size_t)2 * cf->n_items, ncclFloat32, ncclSum, c->comm, c->stream));
        if (cf->d % 4 == 0) q_apply_kernel<<<g, 256, 0, c->stream>>>((float4 *)cf->Q.p, (float4 *)cf->Q0.p, n / 4, cf->d / 4, cf->xchg.p, cf->n_items);
        else q_apply_scalar_kernel<<<g, 256, 0, c->stream>>>(cf->Q.p, cf->Q0.p, n, cf->d, cf->xchg.p, cf->n_items);
        GB_LAUNCHED(c);
    }
    return GORSE_B200_OK;
}

}  // extern "C"
