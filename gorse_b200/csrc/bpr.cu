// bpr.cu -- BPR pairwise SGD: the fused sample-gather-dot-sigmoid-scatter kernel.
// Replaces the body of BPR.Fit's epoch loop, model/cf/model.go:448-490 (arithmetic: SURVEY Appendix A).
//
// Roofline class: HBM/L2 bandwidth.  Algorithmic bytes per triple = 6*d*4 + 12 (3 rows read, 3 rows
// written, 3 ids).  One quad (4 lanes) owns one triple; see cf.cuh for the row->lane mapping that keeps
// the reference's AVX-512 summation order with 128-bit coalesced loads.
#include <algorithm>
#include <cstdlib>

#include "cf.cuh"
#include "tables.cuh"
#include "wgmma.cuh"

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


#define GB_BPR_ROUND 8192   // triples per round of the atomic-scatter epoch (bpr_round_kernel, bpr_round_delta_*_kernel)

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

// chunk c of the three update directions of one triple: row += lr * t for q_i, q_j, p_u
template <int C>
__device__ __forceinline__ void bpr_dirs(const Rows<C> &r, int c, float g, float nreg, float4 &ti, float4 &tj, float4 &tp)
{
    const float4 *p = r.p, *qi = r.qi, *qj = r.qj;
    const float ng = -g;
    // :477-479  q_i += lr * (g*p - reg*q_i)
    GB_F4_OP(ti, __fmaf_rn(f4get(qi[c], k_), nreg, __fmul_rn(g, f4get(p[c], k_))));
    // :481-483  q_j += lr * (-g*p - reg*q_j)
    GB_F4_OP(tj, __fmaf_rn(f4get(qj[c], k_), nreg, __fmul_rn(ng, f4get(p[c], k_))));
    // :485-488  p_u += lr * (g*(q_i - q_j) - reg*p_u)
    GB_F4_OP(tp, __fmaf_rn(f4get(p[c], k_), nreg, __fmul_rn(__fsub_rn(f4get(qi[c], k_), f4get(qj[c], k_)), g)));
}

// the three row updates of one triple (:477-488), from the rows in registers and the gradient factor g
template <int C, bool ATOMIC>
__device__ __forceinline__ void bpr_scatter_rows(const Rows<C> &r, float g, float *Pu, float *Qi, int si, float *Qj, int sj,
                                                 float lr, float reg)
{
    const float4 *p = r.p, *qi = r.qi, *qj = r.qj;
    const float nreg = -reg;
#pragma unroll
    for (int c = 0; c < C; c++) {
        float4 ti, tj, tp, o;
        bpr_dirs<C>(r, c, g, nreg, ti, tj, tp);
        if (ATOMIC) { GB_F4_OP(o, __fmul_rn(f4get(ti, k_), lr)); red_row(Qi + si * c, o); }
        else { GB_F4_OP(o, __fmaf_rn(f4get(ti, k_), lr, f4get(qi[c], k_))); st_row(Qi + si * c, o); }
        if (ATOMIC) { GB_F4_OP(o, __fmul_rn(f4get(tj, k_), lr)); red_row(Qj + sj * c, o); }
        else { GB_F4_OP(o, __fmaf_rn(f4get(tj, k_), lr, f4get(qj[c], k_))); st_row(Qj + sj * c, o); }
        if (ATOMIC) { GB_F4_OP(o, __fmul_rn(f4get(tp, k_), lr)); red_row(Pu + 16 * c, o); }
        else { GB_F4_OP(o, __fmaf_rn(f4get(tp, k_), lr, f4get(p[c], k_))); st_row(Pu + 16 * c, o); }
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
// The store-scatter epoch, free-running: every triple reads its rows whenever it runs and stores what it computed.
template <int C>
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
            if (live) bpr_step_rows<CC, false>(r, Pu, Qi, 16, Qj, 16, mask, lr, reg);
            q = qn; u = un; i = in; j = jn;
        }
    } else {
        for (; q < n_steps; q += nq) {
            int32_t u, i, j;
            sample_triple(v, base, step0 + q, u, i, j);
            if (j < 0) continue;
            bpr_step_dispatch<C, false>(v.P + (int64_t)(u - v.u_lo) * v.d, v.Q + (int64_t)i * v.d, v.Q + (int64_t)j * v.d,
                                        v.d, lane4, mask, lr, reg);
        }
    }
}

// ---- the round epoch ------------------------------------------------------------------------------
// A CTA of bpr_round_kernel is 8 consumer warps (64 quads: one triple each per round) and sampler warps (one thread per
// quad and round).  The samplers draw the CTA's triples up to kRing rounds ahead into a shared-memory ring, prefetch the rows those
// triples will gather into L2, and link the entries of a round that update the same item row, so that the consumers sum
// those deltas in shared memory and send one reduction per distinct item row and CTA.
constexpr int kRoundQuads = 64, kConsumers = 4 * kRoundQuads, kSamplers = kRoundQuads;
// one sampler thread draws one triple per round, a chain of 3-4 dependent loads that takes about as long as a round:
// two groups of samplers take alternate rounds
constexpr int kSamplerGroups = 2, kRoundThreads = kConsumers + kSamplerGroups * kSamplers;
constexpr int kRing = 2 * kSamplerGroups;
constexpr int kConsumerBar = 1, kSamplerBar0 = 2;   // named barriers (0 is __syncthreads; kSamplerBar0 + g for sampler group g)

// one round of one CTA, as the samplers hand it to the consumers.  Entry e of the item arrays is the Q row that triple e
// (e < 64: its positive i) or triple e - 64 (its negative j) updates; -1 when the triple has no update (no valid
// negative, or past the last step).
struct __align__(16) RoundSlot {
    int32_t u[kRoundQuads];
    int32_t item[2 * kRoundQuads];
    int32_t next[2 * kRoundQuads];    // the next entry with the same item, -1 at the end of the chain
    uint8_t first[2 * kRoundQuads];   // 1 when no earlier entry has the same item: this entry sends the row's sum
};

__device__ __forceinline__ void consumer_bar() { asm volatile("bar.sync %0, %1;" ::"n"(kConsumerBar), "n"(kConsumers) : "memory"); }
// the same named barrier, entered only once `dep` is in a register (see consumer_grid_sync)
__device__ __forceinline__ void consumer_bar(float dep)
{
    asm volatile("bar.sync %0, %1;" ::"n"(kConsumerBar), "n"(kConsumers), "f"(dep) : "memory");
}
__device__ __forceinline__ void sampler_bar(int group) { asm volatile("bar.sync %0, %1;" ::"r"(kSamplerBar0 + group), "n"(kSamplers) : "memory"); }

// Grid barrier over the consumer threads only (the samplers run ahead and never join it): `count` starts at 0 and
// `target` is the number of the barrier within the launch times the grid size.  Thread 0 of each CTA adds 1 to `count`
// and polls it; the CTA's other consumers wait at the named barriers.  The two barriers of a round order different
// things (PTX ISA, "Memory Consistency Model"):
//  - The barrier that ends a round (RELEASE) orders the round's additions before the next round's loads.  The fence
//    after the named barrier makes fence + relaxed add a release pattern, and bar.sync and the fence's cumulativity put
//    every consumer's reductions in it; it is also what waits for those reductions to complete.  The adds are
//    read-modify-writes of one location, so the one ld.acquire after the count is reached observes every CTA's add and
//    synchronizes with every CTA's release.  That is one MEMBAR.GPU per barrier; a red.release would fence a second time,
//    and an ld.acquire in the poll loop would invalidate L1 on every poll.
//  - The barrier between a round's loads and its additions orders those loads before other CTAs' later reductions to
//    the same rows.  It needs no fence and no acquire: every load of the CTA has returned its value before thread 0
//    arrives, because each consumer enters the named barrier with `dep`, a value computed from all its loads (the
//    triple's gradient factor; the trials kernel stores its deltas to shared memory before the barrier instead).  A load
//    that read a reduction issued after the barrier would close a cycle of dependencies and observations, which the
//    model's No Thin Air axiom rules out.  The CTA's own writes were released by the previous round's barrier.
//    Measured in DESIGN 5.1.
template <bool RELEASE>
__device__ __forceinline__ void consumer_grid_sync(uint32_t *count, uint32_t target, float dep)
{
    consumer_bar(dep);
    if (threadIdx.x == 0) {
        if (RELEASE) asm volatile("fence.acq_rel.gpu;" ::: "memory");
        asm volatile("red.relaxed.gpu.global.add.u32 [%0], 1;" ::"l"(count) : "memory");
        uint32_t seen;
        do {
            asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(seen) : "l"(count) : "memory");
        } while ((int32_t)(seen - target) < 0);
        if (RELEASE) asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(seen) : "l"(count) : "memory");
    }
    consumer_bar();
}

__device__ __forceinline__ void prefetch_l2(const float *p, uint32_t bytes)
{
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(p), "r"(bytes) : "memory");
}

// The epoch with atomic scatter, in rounds of one triple per quad of the (co-resident) grid: every triple of a round reads
// its rows as the previous round left them, a grid-wide barrier separates those reads from the round's additions, and a
// second one ends the round.  What a triple reads therefore depends only on the step stream and the round size, not on
// timing; the order of the float additions into a row that several triples of one round update is the only freedom left
// (rounding).  The round size bounds the staleness of a popular row: at GB_BPR_ROUND triples the most popular item of a
// Zipf(1) catalogue of 10^5 items takes ~700 updates from one copy per round, lr * reg * 700 << 2.
// Dynamic shared memory: the round's item-row deltas, 2 * kRoundQuads rows of d floats.
template <int C>
__global__ void __launch_bounds__(kRoundThreads, 1)
    bpr_round_kernel(BprView v, int64_t step0, int64_t n_steps, uint64_t base, float lr, float reg, uint32_t *barrier_count)
{
    __shared__ RoundSlot ring[kRing];
    __shared__ uint64_t full[kRing], empty[kRing];
    extern __shared__ float4 delta_smem[];
    const int64_t nq = (int64_t)gridDim.x * kRoundQuads;
    const int64_t n_rounds = (n_steps + nq - 1) / nq;
    if (threadIdx.x == 0) {
        for (int s = 0; s < kRing; s++) {
            mma::mbar_init(&full[s], kSamplers);
            mma::mbar_init(&empty[s], kConsumers / 32);
        }
    }
    __syncthreads();

    if (threadIdx.x >= kConsumers) {
        // sampler: triple t of this CTA in every kSamplerGroups-th round; the ring slot of round r is free once round
        // r - kRing is done
        const int t = (threadIdx.x - kConsumers) % kSamplers, group = (threadIdx.x - kConsumers) / kSamplers;
        for (int64_t r = group; r < n_rounds; r += kSamplerGroups) {
            const int s = (int)(r % kRing);
            if (r >= kRing) mma::mbar_wait_backoff(&empty[s], (uint32_t)((r / kRing - 1) & 1));
            RoundSlot &S = ring[s];
            const int64_t q = r * nq + (int64_t)blockIdx.x * kRoundQuads + t;
            int32_t u = v.u_lo, i = -1, j = -1;
            if (q < n_steps) sample_triple(v, base, step0 + q, u, i, j);
            if (j < 0) i = -1;
            else {
                // the rows leave L2 only by eviction: the round's additions are performed there, so these lines are never stale
                prefetch_l2(v.P + (int64_t)(u - v.u_lo) * v.d, 64 * C);
                prefetch_l2(v.Q + (int64_t)j * v.d, 64 * C);
            }
            S.u[t] = u; S.item[t] = i; S.item[kRoundQuads + t] = j;
            sampler_bar(group);
            // link this triple's two entries to the other entries of the round with the same item
            const int e0 = t, e1 = kRoundQuads + t;
            int nxt0 = -1, nxt1 = -1;
            bool first0 = i >= 0, first1 = j >= 0;
            auto see = [&](int32_t id, int k) {
                if (id == i) { if (k < e0) first0 = false; else if (k > e0) nxt0 = k; }
                if (id == j) { if (k < e1) first1 = false; else if (k > e1) nxt1 = k; }
            };
            const int4 *items4 = reinterpret_cast<const int4 *>(S.item);
            for (int k = 2 * kRoundQuads - 4; k >= 0; k -= 4) {   // descending: the last match after e is the next one
                const int4 x = items4[k / 4];
                see(x.w, k + 3); see(x.z, k + 2); see(x.y, k + 1); see(x.x, k);
            }
            S.next[e0] = nxt0; S.first[e0] = first0;
            S.next[e1] = nxt1; S.first[e1] = first1;
            mma::mbar_arrive(&full[s]);
        }
        return;
    }

    // consumer: quad t of this CTA
    const int t = threadIdx.x >> 2, lane4 = threadIdx.x & 3;
    const unsigned mask = quad_mask();
    const float nreg = -reg;
    constexpr int d = 16 * C;
    float *const D = reinterpret_cast<float *>(delta_smem) + 4 * lane4;   // entry e, chunk c at D + e * d + 16 * c
    uint32_t n_sync = 0;
    for (int64_t r = 0; r < n_rounds; r++) {
        const int s = (int)(r % kRing);
        mma::mbar_wait(&full[s], (uint32_t)((r / kRing) & 1));
        const RoundSlot &S = ring[s];
        const int32_t u = S.u[t], i = S.item[t], j = S.item[kRoundQuads + t];
        const bool live = j >= 0;
        float *Pu = v.P + (int64_t)(u - v.u_lo) * v.d + 4 * lane4;
        Rows<C> rw;
        float g = 0.f;
        if (live) {
            load_rows<C>(rw, Pu, v.Q + (int64_t)i * v.d + 4 * lane4, 16, v.Q + (int64_t)j * v.d + 4 * lane4, 16);
            g = bpr_grad_rows<C>(rw, mask);   // consumes every loaded value before the barrier
        }
        consumer_grid_sync<false>(barrier_count, ++n_sync * gridDim.x, g);
        if (live) {
            float *Di = D + t * d, *Dj = D + (kRoundQuads + t) * d;
#pragma unroll
            for (int c = 0; c < C; c++) {
                float4 ti, tj, tp, o;
                bpr_dirs<C>(rw, c, g, nreg, ti, tj, tp);
                GB_F4_OP(o, __fmul_rn(f4get(tp, k_), lr)); red_row(Pu + 16 * c, o);
                GB_F4_OP(o, __fmul_rn(f4get(ti, k_), lr)); *reinterpret_cast<float4 *>(Di + 16 * c) = o;
                GB_F4_OP(o, __fmul_rn(f4get(tj, k_), lr)); *reinterpret_cast<float4 *>(Dj + 16 * c) = o;
            }
        }
        consumer_bar();
        // the first entry of each item chain adds the chain's deltas in entry order and sends one reduction
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int e = t + h * kRoundQuads;
            if (!S.first[e]) continue;
            float4 acc[C];
#pragma unroll
            for (int c = 0; c < C; c++) acc[c] = *reinterpret_cast<const float4 *>(D + e * d + 16 * c);
            for (int k = S.next[e]; k >= 0; k = S.next[k]) {
#pragma unroll
                for (int c = 0; c < C; c++) {
                    const float4 x = *reinterpret_cast<const float4 *>(D + k * d + 16 * c);
                    GB_F4_OP(acc[c], __fadd_rn(f4get(acc[c], k_), f4get(x, k_)));
                }
            }
            float *Qe = v.Q + (int64_t)S.item[e] * v.d + 4 * lane4;
#pragma unroll
            for (int c = 0; c < C; c++) red_row(Qe + 16 * c, acc[c]);
        }
        __syncwarp();
        if ((threadIdx.x & 31) == 0) mma::mbar_arrive(&empty[s]);
        consumer_grid_sync<true>(barrier_count, ++n_sync * gridDim.x, 0.f);
    }
}

// ---- the round epoch of several models on one triple stream (gorse_b200_cf_fit_trials) -------------------------------
// The trials of a model search share the CSR, the seed and the factor count, so their epochs sample the same triples.
// bpr_trials_round_kernel runs one round epoch for up to kMaxTrialModels models: the samplers draw and link each triple once,
// and the consumers do each model's arithmetic on that model's rows.  The rounds, the triple-to-(CTA, quad) placement and
// the chain order are bpr_round_kernel's, so every model reads what its solo epoch reads and computes the same deltas.
constexpr int kMaxTrialModels = 16;
struct TrialModels {
    float *P[kMaxTrialModels], *Q[kMaxTrialModels];
    float lr[kMaxTrialModels], reg[kMaxTrialModels];
    int32_t n;
};

// Dynamic shared memory: per model, the round's deltas of 64 user rows and 2 * 64 item rows of d floats (3 * 64 * d floats).
// A consumer writes its triple's three deltas for every model before the first grid barrier, so no model's rows need to
// stay in registers across it; after the barrier it sends the user row and sums the item chains of every model.
template <int C>
__global__ void __launch_bounds__(kRoundThreads, 1)
    bpr_trials_round_kernel(BprView v, TrialModels M, int64_t step0, int64_t n_steps, uint64_t base, uint32_t *barrier_count)
{
    __shared__ RoundSlot ring[kRing];
    __shared__ uint64_t full[kRing], empty[kRing];
    extern __shared__ float4 delta_smem[];
    constexpr int d = 16 * C;
    constexpr int kModelFloats = 3 * kRoundQuads * d;
    const int64_t nq = (int64_t)gridDim.x * kRoundQuads;
    const int64_t n_rounds = (n_steps + nq - 1) / nq;
    if (threadIdx.x == 0) {
        for (int s = 0; s < kRing; s++) {
            mma::mbar_init(&full[s], kSamplers);
            mma::mbar_init(&empty[s], kConsumers / 32);
        }
    }
    __syncthreads();

    if (threadIdx.x >= kConsumers) {
        // sampler: as in bpr_round_kernel, with the rows of every model prefetched
        const int t = (threadIdx.x - kConsumers) % kSamplers, group = (threadIdx.x - kConsumers) / kSamplers;
        for (int64_t r = group; r < n_rounds; r += kSamplerGroups) {
            const int s = (int)(r % kRing);
            if (r >= kRing) mma::mbar_wait_backoff(&empty[s], (uint32_t)((r / kRing - 1) & 1));
            RoundSlot &S = ring[s];
            const int64_t q = r * nq + (int64_t)blockIdx.x * kRoundQuads + t;
            int32_t u = v.u_lo, i = -1, j = -1;
            if (q < n_steps) sample_triple(v, base, step0 + q, u, i, j);
            if (j < 0) i = -1;
            else {
                for (int m = 0; m < M.n; m++) {
                    prefetch_l2(M.P[m] + (int64_t)(u - v.u_lo) * d, 64 * C);
                    prefetch_l2(M.Q[m] + (int64_t)j * d, 64 * C);
                }
            }
            S.u[t] = u; S.item[t] = i; S.item[kRoundQuads + t] = j;
            sampler_bar(group);
            const int e0 = t, e1 = kRoundQuads + t;
            int nxt0 = -1, nxt1 = -1;
            bool first0 = i >= 0, first1 = j >= 0;
            auto see = [&](int32_t id, int k) {
                if (id == i) { if (k < e0) first0 = false; else if (k > e0) nxt0 = k; }
                if (id == j) { if (k < e1) first1 = false; else if (k > e1) nxt1 = k; }
            };
            const int4 *items4 = reinterpret_cast<const int4 *>(S.item);
            for (int k = 2 * kRoundQuads - 4; k >= 0; k -= 4) {
                const int4 x = items4[k / 4];
                see(x.w, k + 3); see(x.z, k + 2); see(x.y, k + 1); see(x.x, k);
            }
            S.next[e0] = nxt0; S.first[e0] = first0;
            S.next[e1] = nxt1; S.first[e1] = first1;
            mma::mbar_arrive(&full[s]);
        }
        return;
    }

    // consumer: quad t of this CTA; entry e of model m, chunk c at D + m * kModelFloats + e * d + 16 * c, where entries
    // 0..63 are the user rows and 64..191 the item entries of the ring slot (item entry k at 64 + k)
    const int t = threadIdx.x >> 2, lane4 = threadIdx.x & 3;
    const unsigned mask = quad_mask();
    float *const D = reinterpret_cast<float *>(delta_smem) + 4 * lane4;
    uint32_t n_sync = 0;
    for (int64_t r = 0; r < n_rounds; r++) {
        const int s = (int)(r % kRing);
        mma::mbar_wait(&full[s], (uint32_t)((r / kRing) & 1));
        const RoundSlot &S = ring[s];
        const int32_t u = S.u[t], i = S.item[t], j = S.item[kRoundQuads + t];
        if (j >= 0) {
#pragma unroll 1
            for (int m = 0; m < M.n; m++) {
                const float lr = M.lr[m], nreg = -M.reg[m];
                Rows<C> rw;
                load_rows<C>(rw, M.P[m] + (int64_t)(u - v.u_lo) * d + 4 * lane4, M.Q[m] + (int64_t)i * d + 4 * lane4, 16,
                             M.Q[m] + (int64_t)j * d + 4 * lane4, 16);
                const float g = bpr_grad_rows<C>(rw, mask);
                float *Dm = D + m * kModelFloats, *Dp = Dm + t * d, *Di = Dm + (kRoundQuads + t) * d, *Dj = Dm + (2 * kRoundQuads + t) * d;
#pragma unroll
                for (int c = 0; c < C; c++) {
                    float4 ti, tj, tp, o;
                    bpr_dirs<C>(rw, c, g, nreg, ti, tj, tp);
                    GB_F4_OP(o, __fmul_rn(f4get(tp, k_), lr)); *reinterpret_cast<float4 *>(Dp + 16 * c) = o;
                    GB_F4_OP(o, __fmul_rn(f4get(ti, k_), lr)); *reinterpret_cast<float4 *>(Di + 16 * c) = o;
                    GB_F4_OP(o, __fmul_rn(f4get(tj, k_), lr)); *reinterpret_cast<float4 *>(Dj + 16 * c) = o;
                }
            }
        }
        consumer_grid_sync<false>(barrier_count, ++n_sync * gridDim.x, 0.f);   // the loads are consumed into shared memory
#pragma unroll 1
        for (int m = 0; m < M.n; m++) {
            const float *Dm = D + m * kModelFloats;
            if (j >= 0) {
                float *Pu = M.P[m] + (int64_t)(u - v.u_lo) * d + 4 * lane4;
#pragma unroll
                for (int c = 0; c < C; c++) red_row(Pu + 16 * c, *reinterpret_cast<const float4 *>(Dm + t * d + 16 * c));
            }
            // the first entry of each item chain adds the chain's deltas in entry order and sends one reduction
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const int e = t + h * kRoundQuads;
                if (!S.first[e]) continue;
                const float *De = Dm + kRoundQuads * d;
                float4 acc[C];
#pragma unroll
                for (int c = 0; c < C; c++) acc[c] = *reinterpret_cast<const float4 *>(De + e * d + 16 * c);
                for (int k = S.next[e]; k >= 0; k = S.next[k]) {
#pragma unroll
                    for (int c = 0; c < C; c++) {
                        const float4 x = *reinterpret_cast<const float4 *>(De + k * d + 16 * c);
                        GB_F4_OP(acc[c], __fadd_rn(f4get(acc[c], k_), f4get(x, k_)));
                    }
                }
                float *Qe = M.Q[m] + (int64_t)S.item[e] * d + 4 * lane4;
#pragma unroll
                for (int c = 0; c < C; c++) red_row(Qe + 16 * c, acc[c]);
            }
        }
        __syncwarp();
        if ((threadIdx.x & 31) == 0) mma::mbar_arrive(&empty[s]);
        consumer_grid_sync<true>(barrier_count, ++n_sync * gridDim.x, 0.f);
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

// the store-scatter epoch for d % 16 != 0, free-running like bpr_epoch_kernel
__global__ void __launch_bounds__(128) bpr_epoch_any_kernel(BprView v, int64_t step0, int64_t n_steps, uint64_t base, float lr, float reg)
{
    int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t nq = (int64_t)gridDim.x * blockDim.x;
    for (; q < n_steps; q += nq) {
        int32_t u, i, j;
        sample_triple(v, base, step0 + q, u, i, j);
        if (j < 0) continue;
        bpr_step_any<false>(v.P + (int64_t)(u - v.u_lo) * v.d, v.Q + (int64_t)i * v.d, v.Q + (int64_t)j * v.d, v.d, lr, reg);
    }
}

// ---- the round epoch at the other d: two stream-ordered launches per round ---------------------------------------------
// bpr_round_kernel keeps a CTA's rows in registers and its item deltas in shared memory, which bounds it to d = 16...128.
// At any other d a round is a delta launch, in which each triple of the round reads its rows and writes lr * t for its three
// rows into a buffer, then an add launch, which adds the buffer into the rows.  Stream order puts every read of round r
// after every addition of round r - 1 and before any addition of round r: the same semantics as bpr_round_kernel.
// Buffer layout: entry e = role * GB_BPR_ROUND + t of triple t (role 0: its user row, 1: q_i, 2: q_j) is the d floats at
// delta + e * d, added to P or Q row rows[e] (a row of the shard's P for role 0); rows[e] = -1 for no addition.

// one quad per triple, d % 16 == 0: the arithmetic of bpr_step_quad_dyn
__global__ void __launch_bounds__(256) bpr_round_delta_quad_kernel(BprView v, int64_t step0, int64_t n_steps, uint64_t base,
                                                                   float lr, float reg, float *delta, int32_t *rows)
{
    const int lane4 = threadIdx.x & 3;
    const unsigned mask = quad_mask();
    const int t = (int)(((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 2);
    int32_t u = v.u_lo, i = -1, j = -1;
    if (t < n_steps) sample_triple(v, base, step0 + t, u, i, j);
    const bool live = j >= 0;
    if (lane4 == 0) {
        rows[t] = live ? u - v.u_lo : -1;
        rows[GB_BPR_ROUND + t] = live ? i : -1;
        rows[2 * GB_BPR_ROUND + t] = live ? j : -1;
    }
    if (!live) return;   // the whole quad leaves together
    const int d = v.d, chunks = d / 16;
    const float4 *Pu = reinterpret_cast<const float4 *>(v.P + (int64_t)(u - v.u_lo) * d) + lane4;
    const float4 *Qi = reinterpret_cast<const float4 *>(v.Q + (int64_t)i * d) + lane4;
    const float4 *Qj = reinterpret_cast<const float4 *>(v.Q + (int64_t)j * d) + lane4;
    // nothing writes the tables during this launch, so the rows may come through L1 (the second pass re-reads them)
    float4 ai = make_float4(0.f, 0.f, 0.f, 0.f), aj = ai;
    for (int c = 0; c < chunks; c++) {
        const float4 p = __ldg(Pu + 4 * c);
        dot_chunk(ai, p, __ldg(Qi + 4 * c), c == 0);
        dot_chunk(aj, p, __ldg(Qj + 4 * c), c == 0);
    }
    const float g = bpr_grad(__fsub_rn(quad_tree(ai, mask), quad_tree(aj, mask))), ng = -g, nreg = -reg;
    float4 *Dp = reinterpret_cast<float4 *>(delta + (int64_t)t * d) + lane4;
    float4 *Di = reinterpret_cast<float4 *>(delta + (int64_t)(GB_BPR_ROUND + t) * d) + lane4;
    float4 *Dj = reinterpret_cast<float4 *>(delta + (int64_t)(2 * GB_BPR_ROUND + t) * d) + lane4;
    for (int c = 0; c < chunks; c++) {
        const float4 p = __ldg(Pu + 4 * c), qi = __ldg(Qi + 4 * c), qj = __ldg(Qj + 4 * c);
        float4 tt, o;
        GB_F4_OP(tt, __fmaf_rn(f4get(qi, k_), nreg, __fmul_rn(g, f4get(p, k_))));
        GB_F4_OP(o, __fmul_rn(f4get(tt, k_), lr)); Di[4 * c] = o;
        GB_F4_OP(tt, __fmaf_rn(f4get(qj, k_), nreg, __fmul_rn(ng, f4get(p, k_))));
        GB_F4_OP(o, __fmul_rn(f4get(tt, k_), lr)); Dj[4 * c] = o;
        GB_F4_OP(tt, __fmaf_rn(f4get(p, k_), nreg, __fmul_rn(__fsub_rn(f4get(qi, k_), f4get(qj, k_)), g)));
        GB_F4_OP(o, __fmul_rn(f4get(tt, k_), lr)); Dp[4 * c] = o;
    }
}

// one thread per triple, any d: the arithmetic of bpr_step_any
__global__ void __launch_bounds__(64) bpr_round_delta_any_kernel(BprView v, int64_t step0, int64_t n_steps, uint64_t base,
                                                                 float lr, float reg, float *delta, int32_t *rows)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    int32_t u = v.u_lo, i = -1, j = -1;
    if (t < n_steps) sample_triple(v, base, step0 + t, u, i, j);
    const bool live = j >= 0;
    rows[t] = live ? u - v.u_lo : -1;
    rows[GB_BPR_ROUND + t] = live ? i : -1;
    rows[2 * GB_BPR_ROUND + t] = live ? j : -1;
    if (!live) return;
    const int d = v.d;
    const float *Pu = v.P + (int64_t)(u - v.u_lo) * d, *Qi = v.Q + (int64_t)i * d, *Qj = v.Q + (int64_t)j * d;
    float *Dp = delta + (int64_t)t * d, *Di = delta + (int64_t)(GB_BPR_ROUND + t) * d,
          *Dj = delta + (int64_t)(2 * GB_BPR_ROUND + t) * d;
    const float g = bpr_grad(__fsub_rn(dot_any(Pu, Qi, d), dot_any(Pu, Qj, d))), ng = -g, nreg = -reg;
    for (int k = 0; k < d; k++) {
        const float p = Pu[k], qi = Qi[k], qj = Qj[k];
        Di[k] = __fmul_rn(axpy_elem(qi, nreg, __fmul_rn(p, g), k, d), lr);
        Dj[k] = __fmul_rn(axpy_elem(qj, nreg, __fmul_rn(p, ng), k, d), lr);
        Dp[k] = __fmul_rn(axpy_elem(p, nreg, __fmul_rn(__fsub_rn(qi, qj), g), k, d), lr);
    }
}

// adds the round's deltas into the rows: one thread per float4 of an entry when d % 4 == 0, per float otherwise
template <bool V4>
__global__ void __launch_bounds__(256) bpr_round_add_kernel(float *P, float *Q, int d, const float *delta, const int32_t *rows)
{
    const int per = V4 ? d / 4 : d;
    const int64_t x = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= (int64_t)3 * GB_BPR_ROUND * per) return;
    const int e = (int)(x / per), k = (int)(x % per);
    const int32_t r = __ldg(rows + e);
    if (r < 0) return;
    float *row = (e < GB_BPR_ROUND ? P : Q) + (int64_t)r * d;
    if (V4) red_row(row + 4 * k, __ldg(reinterpret_cast<const float4 *>(delta + (int64_t)e * d) + k));
    else atomicAdd(row + k, __ldg(delta + (int64_t)e * d + k));
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
    const size_t smem = (size_t)2 * kRoundQuads * 16 * C * sizeof(float);
    GB_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 0;
    GB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k, kRoundThreads, smem));
    // the round size is fixed (GB_BPR_ROUND triples) unless the device cannot hold that many quads at once
    const int g = (int)std::min<int64_t>(GB_BPR_ROUND / kRoundQuads, (int64_t)per_sm * c->sm_count);
    if (g < 1) { set_error("bpr_round_kernel does not fit on the device"); return GORSE_B200_ERR_UNSUPPORTED; }
    uint32_t *count = cf->bpr_barrier.p;
    GB_CUDA(cudaMemsetAsync(count, 0, sizeof(uint32_t), c->stream));
    void *args[] = {&v, &step0, &n, &base, &lr, &reg, &count};
    GB_CUDA(cudaLaunchCooperativeKernel((const void *)k, dim3(g), dim3(kRoundThreads), args, smem, c->stream));
    return GORSE_B200_OK;
}

// One atomic round epoch for each of n models on cf's triple stream, in launches of as many models as the kernel's shared
// memory holds.  The grid is launch_round_epoch's, so the rounds and the placement are the solo epoch's.
template <int C>
static int32_t launch_trials_epoch(gorse_b200_cf *cf, int n, float *const *P, float *const *Q, const float *lr, const float *reg,
                                   uint64_t base)
{
    gorse_b200_ctx *c = cf->ctx;
    auto *k = bpr_trials_round_kernel<C>;
    const size_t per_model = (size_t)3 * kRoundQuads * 16 * C * sizeof(float);
    int optin = 0;
    GB_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, c->device));
    cudaFuncAttributes fa;
    GB_CUDA(cudaFuncGetAttributes(&fa, k));
    const int cap = (int)std::min<size_t>(kMaxTrialModels, ((size_t)optin - fa.sharedSizeBytes) / per_model);
    if (cap < 1) { set_error("bpr_trials_round_kernel does not fit on the device"); return GORSE_B200_ERR_UNSUPPORTED; }
    const int group = std::min(cap, n);
    const size_t smem_max = (size_t)group * per_model;
    GB_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_max));
    int per_sm = 0;
    GB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k, kRoundThreads, smem_max));
    const int g = (int)std::min<int64_t>(GB_BPR_ROUND / kRoundQuads, (int64_t)per_sm * c->sm_count);
    if (g < 1) { set_error("bpr_trials_round_kernel does not fit on the device"); return GORSE_B200_ERR_UNSUPPORTED; }
    BprView v = make_view(cf);
    int64_t step0 = 0, n_steps = cf->n_feedback_global;
    uint32_t *count = cf->bpr_barrier.p;
    for (int m0 = 0; m0 < n; m0 += group) {
        TrialModels M{};
        M.n = std::min(group, n - m0);
        for (int m = 0; m < M.n; m++) { M.P[m] = P[m0 + m]; M.Q[m] = Q[m0 + m]; M.lr[m] = lr[m0 + m]; M.reg[m] = reg[m0 + m]; }
        const size_t smem = (size_t)M.n * per_model;
        GB_CUDA(cudaMemsetAsync(count, 0, sizeof(uint32_t), c->stream));
        void *args[] = {&v, &M, &step0, &n_steps, &base, &count};
        GB_CUDA(cudaLaunchCooperativeKernel((const void *)k, dim3(g), dim3(kRoundThreads), args, smem, c->stream));
        GB_LAUNCHED(c);
    }
    return GORSE_B200_OK;
}

// the atomic-scatter epoch at d outside 16/32/64/128: rounds of GB_BPR_ROUND steps, a delta and an add launch each
static int32_t launch_round_epoch_any(gorse_b200_cf *cf, BprView v, int64_t step0, int64_t n, uint64_t base, float lr, float reg)
{
    gorse_b200_ctx *c = cf->ctx;
    cudaStream_t s = c->stream;
    const int d = cf->d;
    if (cf->bpr_delta.n == 0) GB_TRY(cf->bpr_delta.alloc((size_t)3 * GB_BPR_ROUND * d));
    if (cf->bpr_rows.n == 0) GB_TRY(cf->bpr_rows.alloc((size_t)3 * GB_BPR_ROUND));
    float *delta = cf->bpr_delta.p;
    int32_t *rows = cf->bpr_rows.p;
    const bool quad = d % 16 == 0, v4 = d % 4 == 0;
    const int per = v4 ? d / 4 : d;
    const int add_grid = (int)div_up((int64_t)3 * GB_BPR_ROUND * per, 256);
    for (int64_t r0 = 0; r0 < n; r0 += GB_BPR_ROUND) {
        const int64_t nr = std::min<int64_t>(GB_BPR_ROUND, n - r0);
        if (quad) bpr_round_delta_quad_kernel<<<GB_BPR_ROUND / 64, 256, 0, s>>>(v, step0 + r0, nr, base, lr, reg, delta, rows);
        else bpr_round_delta_any_kernel<<<GB_BPR_ROUND / 64, 64, 0, s>>>(v, step0 + r0, nr, base, lr, reg, delta, rows);
        GB_LAUNCHED(c);
        if (v4) bpr_round_add_kernel<true><<<add_grid, 256, 0, s>>>(v.P, v.Q, d, delta, rows);
        else bpr_round_add_kernel<false><<<add_grid, 256, 0, s>>>(v.P, v.Q, d, delta, rows);
        GB_LAUNCHED(c);
    }
    return GORSE_B200_OK;
}

static void launch_store_epoch(gorse_b200_cf *cf, const BprView &v, int64_t step0, int64_t n, uint64_t base, float lr, float reg)
{
    gorse_b200_ctx *c = cf->ctx;
    cudaStream_t s = c->stream;
    if (cf->d % 16 == 0) {
        int C = cf->d / 16;
        int g = quad_grid(c, n, C <= 4 ? 8 : 4);
        switch (C) {
            case 1: bpr_epoch_kernel<1><<<g, 256, 0, s>>>(v, step0, n, base, lr, reg); break;
            case 2: bpr_epoch_kernel<2><<<g, 256, 0, s>>>(v, step0, n, base, lr, reg); break;
            case 4: bpr_epoch_kernel<4><<<g, 256, 0, s>>>(v, step0, n, base, lr, reg); break;
            case 8: bpr_epoch_kernel<8><<<g, 256, 0, s>>>(v, step0, n, base, lr, reg); break;
            default: bpr_epoch_kernel<0><<<g, 256, 0, s>>>(v, step0, n, base, lr, reg); break;
        }
    } else {
        int g = (int)std::max<int64_t>(1, std::min<int64_t>((n + 127) / 128, (int64_t)c->sm_count * 8));
        bpr_epoch_any_kernel<<<g, 128, 0, s>>>(v, step0, n, base, lr, reg);
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

int32_t bpr_trials_epoch(gorse_b200_cf *cf, int n, float *const *P, float *const *Q, const float *lr, const float *reg, uint64_t seed)
{
    if (n == 0 || cf->n_feedback_global == 0) return GORSE_B200_OK;
    const uint64_t base = mix64(seed);
    switch (cf->d) {
        case 16: return launch_trials_epoch<1>(cf, n, P, Q, lr, reg, base);
        case 32: return launch_trials_epoch<2>(cf, n, P, Q, lr, reg, base);
        case 64: return launch_trials_epoch<4>(cf, n, P, Q, lr, reg, base);
        case 128: return launch_trials_epoch<8>(cf, n, P, Q, lr, reg, base);
        default: set_error("batched BPR trials need d in {16, 32, 64, 128}, not %d", cf->d); return GORSE_B200_ERR_UNSUPPORTED;
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
            GB_LAUNCHED(c);
        } else if (scatter == GORSE_B200_SCATTER_ATOMIC) {
            GB_TRY(launch_round_epoch_any(cf, v, s0, n_local, mix64(seed), lr, reg));
        } else {
            launch_store_epoch(cf, v, s0, n_local, mix64(seed), lr, reg);
            GB_LAUNCHED(c);
        }
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
