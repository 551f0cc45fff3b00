// fm_fit_emb.cuh -- the item-embedding slots of FM training (gorse_b200_fm_fit_emb): per slot the attention and encoder
// layers' forward on a batch (also the chunks of the evaluation lists) and their backward (DESIGN §8.5).  Included by
// fm_fit.cu inside gb::fmfit, after go_max.
//
//   forward   fm_fit_emb_hz_kernel    a warp per row: e (the bf16 table row widened, zeros when absent) is kept as fp32;
//                                     h = e AW + Ab (kept), z = ReLU(h) H and its row max
//             fm_fit_emb_exp_kernel   a warp per row: exp(z - the partner row's max), kept, and the row's sum in order
//             fm_fit_emb_enc_kernel   a warp per row: y = . / the partner row's sum (kept), att = y e (kept),
//                                     enc = att EW + Eb (kept), and <vx, enc> added to the row's logit
//   backward  fm_fit_emb_datt_kernel  a warp per row: denc = vx dp, datt = denc EW^T, gx = y (datt e) and its row sum
//             fm_fit_emb_dh_kernel    a warp per row: dz = gx - y (the partner row's sum), dReLU = dz H^T, dh
//             fm_fit_emb_wgrad_kernel a thread per element of dEW, dAW, dH, dEb, dAb: the chain over the batch rows in order
// The partner of element (r, c) in a batch of B rows is row (r dim + c) % B, in the forward and in the backward.
// floats.MM's x y^T path assigns floats.Dot to every element: 16 lane accumulators, a reduce tree, an 8-lane block and a
// fused tail, not one chain; avx_dot and avx_dot16 are that.  Every other product is a fused chain from +0.
#pragma once

struct Slot {
    const float *H, *AW, *Ab, *EW, *Eb;      // in the parameters
    float *gH, *gAW, *gAb, *gEW, *gEb;       // their gradients
    const uint16_t *table;                   // [n_emb_rows x dim] bf16 bits
    const uint8_t *mask;                     // [n_emb_rows x n_emb] or NULL
    int n_emb, s, dim;
    float *e, *y, *att;                      // [bs x dim]
    float *h, *enc;                          // [bs x k]
    float *zmax, *rowsum;                    // [bs]
    float *gx, *denc, *dh, *sumdx;           // backward scratch shared by the slots: [bs x dim], [bs x k], [bs x k], [bs]
};

struct Batch {                               // rows [s bs, s bs + B) of a list of n rows
    int64_t bs, n;
    int s;
    __device__ int64_t r0() const { return (int64_t)s * bs; }
    __device__ int rows() const { return (int)(n - r0() < bs ? n - r0() : bs); }
};

// trial `off`'s view of a slot: its parameters, gradients and batch tensors; the table and the mask are shared
__device__ __forceinline__ Slot slot_at(const Slot &S, int64_t off)
{
    return Slot{at(S.H, off), at(S.AW, off), at(S.Ab, off), at(S.EW, off), at(S.Eb, off), at(S.gH, off), at(S.gAW, off), at(S.gAb, off),
                at(S.gEW, off), at(S.gEb, off), S.table, S.mask, S.n_emb, S.s, S.dim, at(S.e, off), at(S.y, off), at(S.att, off),
                at(S.h, off), at(S.enc, off), at(S.zmax, off), at(S.rowsum, off), at(S.gx, off), at(S.denc, off), at(S.dh, off),
                at(S.sumdx, off)};
}

// floats.Dot (floats_avx512.c:306-367) by one thread
__device__ __forceinline__ float avx_dot(const float *a, const float *b, int n)
{
    const int epoch = n / 16;
    int remain = n % 16;
    float s[16];
#pragma unroll
    for (int l = 0; l < 16; l++) s[l] = epoch > 0 ? __fmul_rn(a[l], b[l]) : 0.0f;
    for (int c = 1; c < epoch; c++)
#pragma unroll
        for (int l = 0; l < 16; l++) s[l] = __fmaf_rn(a[16 * c + l], b[16 * c + l], s[l]);
#pragma unroll
    for (int l = 0; l < 8; l++) s[l] = __fadd_rn(s[l + 8], s[l]);
#pragma unroll
    for (int l = 0; l < 4; l++) s[l] = __fadd_rn(s[l + 4], s[l]);
    float sum = __fadd_rn(__fadd_rn(s[0], s[2]), __fadd_rn(s[1], s[3]));
    a += 16 * epoch;
    b += 16 * epoch;
    if (remain >= 8) {
#pragma unroll
        for (int l = 0; l < 4; l++) s[l] = __fadd_rn(__fmul_rn(a[l + 4], b[l + 4]), __fmul_rn(a[l], b[l]));
        sum = __fadd_rn(sum, __fadd_rn(__fadd_rn(s[0], s[2]), __fadd_rn(s[1], s[3])));
        a += 8;
        b += 8;
        remain -= 8;
    }
    for (int i = 0; i < remain; i++) sum = __fmaf_rn(a[i], b[i], sum);
    return sum;
}

// floats.Dot by the 16 lanes of a half warp, lane l holding accumulator l; every lane of the warp calls it (on = false:
// the half warp has no vector and reads nothing).  The result is in the half warp's lane 0.
__device__ __forceinline__ float avx_dot16(const float *a, const float *b, int n, int l, bool on)
{
    const int epoch = n / 16;
    int remain = n % 16;
    float s = on && epoch > 0 ? __fmul_rn(a[l], b[l]) : 0.0f;
    if (on)
        for (int c = 1; c < epoch; c++) s = __fmaf_rn(a[16 * c + l], b[16 * c + l], s);
    s = __fadd_rn(__shfl_down_sync(FULL, s, 8, 16), s);
    s = __fadd_rn(__shfl_down_sync(FULL, s, 4, 16), s);
    s = __fadd_rn(s, __shfl_down_sync(FULL, s, 2, 16));   // lane 0: r4[0] + r4[2], lane 1: r4[1] + r4[3]
    float sum = __fadd_rn(s, __shfl_down_sync(FULL, s, 1, 16));
    a += 16 * epoch;
    b += 16 * epoch;
    const bool blk = remain >= 8;   // the same for the whole warp
    if (blk) {
        float p = on && l < 8 ? __fmul_rn(a[l], b[l]) : 0.0f;
        p = __fadd_rn(__shfl_down_sync(FULL, p, 4, 16), p);
        p = __fadd_rn(p, __shfl_down_sync(FULL, p, 2, 16));
        p = __fadd_rn(p, __shfl_down_sync(FULL, p, 1, 16));
        sum = __fadd_rn(sum, p);
        a += 8;
        b += 8;
        remain -= 8;
    }
    if (on && l == 0)
        for (int i = 0; i < remain; i++) sum = __fmaf_rn(a[i], b[i], sum);
    return sum;
}

// a row's values summed as Tensor.sum does: the first, then the rest added in order; v is lane-strided (c = c0 + lane)
__device__ __forceinline__ float row_sum_step(float sum, float v, int c0, int dim)
{
    const int cnt = min(32, dim - c0);
    for (int j = 0; j < cnt; j++) {
        const float x = __shfl_sync(FULL, v, j);
        sum = c0 + j == 0 ? x : __fadd_rn(sum, x);
    }
    return sum;
}

__global__ void __launch_bounds__(WARPS * 32) fm_fit_emb_hz_kernel(Group G, Slot S0, int k, const int32_t *emb_row, Batch T)
{
    Blk tb;
    if (!trial_block(G, tb)) return;
    const Slot S = slot_at(S0, tb.off);
    const int lane = threadIdx.x & 31, B = T.rows(), dim = S.dim;
    for (int b = tb.x * WARPS + (threadIdx.x >> 5); b < B; b += tb.nx * WARPS) {
        const int64_t row = emb_row[T.r0() + b];
        const bool present = row >= 0 && (!S.mask || S.mask[row * S.n_emb + S.s]);
        float *e = S.e + (int64_t)b * dim, *z = S.y + (int64_t)b * dim;
        for (int c = lane; c < dim; c += 32) e[c] = present ? __uint_as_float((uint32_t)S.table[row * dim + c] << 16) : 0.0f;
        __syncwarp();
        float h = 0.0f;
        if (lane < k) {
#pragma unroll 8
            for (int c = 0; c < dim; c++) h = __fmaf_rn(e[c], S.AW[c * k + lane], h);   // MatMul(e, AW)
            h = __fadd_rn(h, S.Ab[lane]);                                             // + Ab
            S.h[(int64_t)b * k + lane] = h;
            h = go_max(h, 0.0f);                                                      // ReLU
        }
        float mx = -INFINITY;   // Go's max is associative and commutative with -Inf as identity
        for (int c0 = 0; c0 < dim; c0 += 32) {
            const int c = c0 + lane;
            float zc = 0.0f;
            for (int f = 0; f < k; f++) {
                const float hf = __shfl_sync(FULL, h, f);
                if (c < dim) zc = __fmaf_rn(hf, S.H[f * dim + c], zc);                 // MatMul(., H)
            }
            if (c < dim) {
                z[c] = zc;
                mx = go_max(mx, zc);
            }
        }
        for (int o = 16; o; o >>= 1) mx = go_max(mx, __shfl_xor_sync(FULL, mx, o));
        if (lane == 0) S.zmax[b] = mx;
    }
}

__global__ void __launch_bounds__(WARPS * 32) fm_fit_emb_exp_kernel(Group G, Slot S0, Batch T)
{
    Blk tb;
    if (!trial_block(G, tb)) return;
    const Slot S = slot_at(S0, tb.off);
    const int lane = threadIdx.x & 31, B = T.rows(), dim = S.dim;
    for (int r = tb.x * WARPS + (threadIdx.x >> 5); r < B; r += tb.nx * WARPS) {
        float *y = S.y + (int64_t)r * dim;
        float sum = 0.0f;
        for (int c0 = 0; c0 < dim; c0 += 32) {
            const int c = c0 + lane;
            float v = 0.0f;
            if (c < dim) {
                v = fmx_expf(__fsub_rn(y[c], S.zmax[((int64_t)r * dim + c) % B]));   // x.sub(max): row (r dim + c) % B's
                y[c] = v;
            }
            sum = row_sum_step(sum, v, c0, dim);
        }
        if (lane == 0) S.rowsum[r] = sum;
    }
}

__global__ void __launch_bounds__(WARPS * 32, 1) fm_fit_emb_enc_kernel(Group G, Slot S0, int k, Batch T, const float *vx, float *p)
{
    Blk tb;
    if (!trial_block(G, tb)) return;
    const int64_t o = tb.off;   // the slot's pointers are offset where they are used
    const Slot &S = S0;
    vx = at(vx, o);
    p = at(p, o);
    const int lane = threadIdx.x & 31, B = T.rows(), dim = S.dim;
    for (int r = tb.x * WARPS + (threadIdx.x >> 5); r < B; r += tb.nx * WARPS) {
        float *y = at(S.y, o) + (int64_t)r * dim, *att = at(S.att, o) + (int64_t)r * dim;
        const float *e = at(S.e, o) + (int64_t)r * dim;
        for (int c = lane; c < dim; c += 32) {
            const float a = __fdiv_rn(y[c], at(S.rowsum, o)[((int64_t)r * dim + c) % B]);   // y.div(sum): row (r dim + c) % B's
            y[c] = a;
            att[c] = __fmul_rn(a, e[c]);                                              // Mul(softmax, e)
        }
        __syncwarp();
        float enc = 0.0f, v = 0.0f;
        if (lane < k) {
#pragma unroll 8
            for (int c = 0; c < dim; c++) enc = __fmaf_rn(att[c], at(S.EW, o)[c * k + lane], enc);   // MatMul(., EW)
            enc = __fadd_rn(enc, at(S.Eb, o)[lane]);                                                // + Eb
            at(S.enc, o)[(int64_t)r * k + lane] = enc;
            v = vx[(int64_t)r * k + lane];
        }
        float dot = 0.0f;
        for (int q = 0; q < k; q++) dot = __fmaf_rn(__shfl_sync(FULL, v, q), __shfl_sync(FULL, enc, q), dot);   // BMM(vx, enc)
        if (lane == 0) p[r] = __fadd_rn(p[r], dot);
    }
}

__global__ void __launch_bounds__(WARPS * 32) fm_fit_emb_datt_kernel(Group G, Slot S0, int k, Batch T, const float *vx, const float *g)
{
    Blk tb;
    if (!trial_block(G, tb)) return;
    const Slot S = slot_at(S0, tb.off);
    vx = at(vx, tb.off);
    g = at(g, tb.off);
    const int lane = threadIdx.x & 31, B = T.rows(), dim = S.dim;
    for (int r = tb.x * WARPS + (threadIdx.x >> 5); r < B; r += tb.nx * WARPS) {
        float *denc = S.denc + (int64_t)r * k, *gx = S.gx + (int64_t)r * dim;
        // Add(fmOutput, .): 0 + dp; BMM(vx, enc): denc = vx dp; Add(., Eb): a clone
        if (lane < k) denc[lane] = __fmaf_rn(vx[(int64_t)r * k + lane], __fadd_rn(0.0f, g[r]), 0.0f);
        __syncwarp();
        const float *y = S.y + (int64_t)r * dim, *e = S.e + (int64_t)r * dim;
        float sum = 0.0f;
        for (int c0 = 0; c0 < dim; c0 += 32) {
            const int c = c0 + lane;
            float v = 0.0f;
            if (c < dim) {
                const float datt = avx_dot(denc, S.EW + (int64_t)c * k, k);   // MatMul(att, EW): dx0 = dy EW^T
                v = __fmul_rn(y[c], __fmul_rn(datt, e[c]));                    // Mul: gx0 = dy e; Softmax: gx = y dy
                gx[c] = v;
            }
            sum = row_sum_step(sum, v, c0, dim);                               // gx.sum(1, true)
        }
        if (lane == 0) S.sumdx[r] = sum;
    }
}

__global__ void __launch_bounds__(WARPS * 32) fm_fit_emb_dh_kernel(Group G, Slot S0, int k, Batch T)
{
    Blk tb;
    if (!trial_block(G, tb)) return;
    const Slot S = slot_at(S0, tb.off);
    const int lane = threadIdx.x & 31, B = T.rows(), dim = S.dim;
    for (int r = tb.x * WARPS + (threadIdx.x >> 5); r < B; r += tb.nx * WARPS) {
        float *dz = S.gx + (int64_t)r * dim;
        const float *y = S.y + (int64_t)r * dim;
        // y.mul(sumdx) and gx.sub(y), sumdx indexed i % B: two roundings
        for (int c = lane; c < dim; c += 32) dz[c] = __fsub_rn(dz[c], __fmul_rn(y[c], S.sumdx[((int64_t)r * dim + c) % B]));
        __syncwarp();
        for (int f0 = 0; f0 < k; f0 += 2) {
            const int f = f0 + (lane >> 4);
            const float d = avx_dot16(dz, S.H + (int64_t)f * dim, dim, lane & 15, f < k);   // MatMul(ReLU(h), H): dx0 = dz H^T
            if (f < k && (lane & 15) == 0) {
                const float h = S.h[(int64_t)r * k + f];
                S.dh[(int64_t)r * k + f] = __fmul_rn(h > 0.0f ? 1.0f : 0.0f, d);            // ReLU: gt(h, 0) dy; Add(., Ab): a clone
            }
        }
    }
}

// dx1 = x0^T dy of the three MatMuls and the two biases' gx1[i % k] += dy[i]: per element one chain over the batch rows
__global__ void fm_fit_emb_wgrad_kernel(Group G, Slot S0, int k, Batch T)
{
    Blk tb;
    if (!trial_block(G, tb)) return;
    const Slot S = slot_at(S0, tb.off);
    const int B = T.rows(), dim = S.dim, dk = dim * k;
    for (int i = tb.x * blockDim.x + threadIdx.x; i < 2 * dk + 2 * k; i += tb.nx * blockDim.x) {
        if (i < dk) {                     // dEW = att^T denc and dAW = e^T dh, element (c, f)
            const int c = i / k, f = i % k;
            float ew = 0.0f, aw = 0.0f;
#pragma unroll 8
            for (int b = 0; b < B; b++) {
                ew = __fmaf_rn(S.att[(int64_t)b * dim + c], S.denc[(int64_t)b * k + f], ew);
                aw = __fmaf_rn(S.e[(int64_t)b * dim + c], S.dh[(int64_t)b * k + f], aw);
            }
            S.gEW[i] = ew;
            S.gAW[i] = aw;
        } else if (i < 2 * dk) {          // dH = ReLU(h)^T dz, element (f, c)
            const int j = i - dk, f = j / dim, c = j % dim;
            float acc = 0.0f;
#pragma unroll 8
            for (int b = 0; b < B; b++) acc = __fmaf_rn(go_max(S.h[(int64_t)b * k + f], 0.0f), S.gx[(int64_t)b * dim + c], acc);
            S.gH[j] = acc;
        } else {                          // dEb and dAb: from +0, every row's dy in order
            const int j = i - 2 * dk, f = j % k;
            const float *src = j < k ? S.denc : S.dh;
            float acc = 0.0f;
#pragma unroll 8
            for (int b = 0; b < B; b++) acc = __fadd_rn(acc, src[(int64_t)b * k + f]);
            (j < k ? S.gEb : S.gAb)[f] = acc;
        }
    }
}

// the forward of the slot-free part on a batch, kept for the slots: the rows' logits and vx
__global__ void __launch_bounds__(WARPS * 32) fm_fit_emb_base_kernel(Group G, const float *P, int64_t nf, int k, Rows R, Batch T, float *p, float *vx)
{
    Blk tb;
    if (!trial_block(G, tb)) return;
    P = at(P, tb.off);
    p = at(p, tb.off);
    vx = at(vx, tb.off);
    const int lane = threadIdx.x & 31, B = T.rows();
    for (int b = tb.x * WARPS + (threadIdx.x >> 5); b < B; b += tb.nx * WARPS) {
        float v;
        const float pb = row_forward(P, nf, k, R, T.r0() + b, lane, v);
        if (lane == 0) p[b] = pb;
        if (lane < k) vx[(int64_t)b * k + lane] = v;
    }
}
