// fm.cu -- batched FM ranking: gorse_b200_fm_create / _destroy / _rank.
//
// The worker ranks each user's candidates with the factorization machine when recommend.ranker.type = "fm"
// (worker/pipeline.go:257-264, rankByClickTroughRate :450-499): one AFM.BatchPredict call per user (model/ctr/fm.go:180-229)
// and a sort by score.  One gorse_b200_fm_rank call does that for many users.  The scores are the reference's bit for bit,
// because every kernel forms each value with the reference's operations in the reference's order (DESIGN §8.4):
//
//   fm_item_kernel   per slot, one warp per row of the call's item table: h = ReLU(e AW + Ab), z = h H and the row max of z.
//                    They depend on the item only (its embedding, or zeros when it has none).
//   fm_pair_kernel   groups of L lanes (L = n_factors rounded up to 8, 16 or 32), one (user, candidate) pair per group, one
//                    factor per lane: walks the pair's D_u features in the reference's order, padding included, and forms
//                    vx, the squared sums, the linear term and ((linear + 0.5 sum) + B).  Indices go through float32.
//   fm_attn_kernel   per slot, one CTA per chunk of batch_size candidates of one user (BatchInternalPredict's chunks,
//                    fm.go:168-176): the softmax's exp / row sum / divide, with element (r, c) using the max and the sum of
//                    row (r dim + c) % B, as the reference's Tensor.sub / Tensor.div broadcast does; then Mul(., e), E and
//                    the dot with vx, added to the score.
//   fm_sort_kernel   one CTA per user: the candidate positions by (score descending, position ascending), NaN last, with
//                    the recall's block_sort.
// The arithmetic is fp32 on the CUDA cores with explicit __fmaf_rn / __fmul_rn / __fadd_rn / __fsub_rn / __fdiv_rn: the
// reference's chains are sequential, which the tensor cores cannot reproduce.  The softmax's double exp is fm_exp.h.
#include <algorithm>

#include "fm.cuh"
#include "fm_exp.h"

namespace gb {
namespace fm {

// Go's max(a, b) on float32: NaN propagates, max(-0, +0) = +0
__device__ __forceinline__ float go_max(float a, float b)
{
    if (a != a) return a;
    if (b != b) return b;
    if (a == b) return __int_as_float(__float_as_int(a) & __float_as_int(b));
    return a > b ? a : b;
}

__device__ __forceinline__ float emb_at(const Slot &S, int64_t item, int c)
{
    if (S.mask && !S.mask[item * S.n_emb + S.s]) return 0.0f;
    return __uint_as_float((uint32_t)S.emb[item * S.dim + c] << 16);
}

__global__ void fm_item_kernel(Slot S, int k, int64_t n_items)
{
    const int lane = threadIdx.x & 31;
    const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t it = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); it < n_items; it += warps) {
        float h = 0.0f;
        if (lane < k) {
            for (int c = 0; c < S.dim; c++) h = __fmaf_rn(emb_at(S, it, c), S.AW[c * k + lane], h);   // MatMul(e, AW)
            h = go_max(__fadd_rn(h, S.Ab[lane]), 0.0f);                                            // + Ab, ReLU
        }
        // Go's max is associative and commutative (NaN absorbs, -0 < +0) with -Inf as identity, so lanes and a tree give
        // the row's sequential max (Tensor.max, tensor.go:658-695)
        float mx = -INFINITY;
        for (int c0 = 0; c0 < S.dim; c0 += 32) {
            const int c = c0 + lane;
            float z = 0.0f;
            for (int f = 0; f < k; f++) {
                const float hf = __shfl_sync(0xffffffffu, h, f);
                if (c < S.dim) z = __fmaf_rn(hf, S.H[f * S.dim + c], z);                           // MatMul(., H)
            }
            if (c < S.dim) {
                S.z[it * S.dim + c] = z;
                mx = go_max(mx, z);
            }
        }
        for (int o = 16; o; o >>= 1) mx = go_max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        if (lane == 0) S.zmax[it] = mx;
    }
}

template <int L>
__global__ void fm_pair_kernel(Model M, Feats U, Feats I, const int64_t *cand_off, const int32_t *cand_items, const int32_t *dims,
                               int64_t u0, int64_t u1, int64_t pair_base, float *score, float *vx_out)
{
    constexpr int G = 32 / L;
    const int lane = threadIdx.x & 31, g = lane / L, f = lane % L;
    const unsigned gmask = L == 32 ? 0xffffffffu : (((1u << L) - 1u) << (g * L));
    const int k = M.k;
    const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t u = u0 + (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); u < u1; u += warps) {
        const int64_t c0 = cand_off[u], n = cand_off[u + 1] - c0;
        const int32_t uf = U.feat[u];
        const int64_t ul0 = U.off[u], ul1 = U.off[u + 1];
        const int D = dims[u];
        for (int64_t t = g; t < n; t += G) {
            const int32_t it = cand_items[c0 + t];
            float vx = 0.0f, ss = 0.0f, lin = 0.0f;
            // one feature of the row: Embedding gathers row (int)(float32)index of V and W (op.go:662-685, fm.go:552)
            auto step = [&](int32_t idx, float x) {
                const int64_t r = (int64_t)__int2float_rn(idx);
                const float x2 = __fmul_rn(x, x);
                if (f < k) {
                    const float v = M.V[r * k + f];
                    vx = __fmaf_rn(v, x, vx);                       // BMM(v, x): V^T x
                    ss = __fmaf_rn(__fmul_rn(v, v), x2, ss);        // BMM(Square(v), Square(x))
                }
                lin = __fmaf_rn(M.W[r], x, lin);                    // BMM(w, x)
            };
            int l = 0;
            if (uf >= 0) { step(uf, 1.0f); l++; }
            const int32_t itf = I.feat[it];
            if (itf >= 0) { step(itf, 1.0f); l++; }
            for (int64_t j = ul0; j < ul1; j++, l++) step(U.idx[j], U.val[j]);
            for (int64_t j = I.off[it]; j < I.off[it + 1]; j++, l++) step(I.idx[j], I.val[j]);
            for (; l < D; l++) step(0, 0.0f);                       // convertToTensors' padding: index 0, value 0
            const float d = __fsub_rn(__fmul_rn(vx, vx), ss);      // Sub(Square(vx), squareSum)
            float s = 0.0f;
            for (int q = 0; q < k; q++) s = __fadd_rn(s, __shfl_sync(gmask, d, q, L));   // Sum(., 1), from 0 in factor order
            s = __fmul_rn(s, 0.5f);
            if (f == 0) score[c0 + t] = __fadd_rn(__fadd_rn(lin, s), M.bias);              // Add(linear, sum, B)
            if (vx_out && f < k) vx_out[(c0 + t - pair_base) * k + f] = vx;
        }
    }
}

// the softmax's numerator of element (r, c) of a chunk: exp(z[r][c] - max of row (r dim + c) % B)
__device__ __forceinline__ float numerator(const Slot &S, const int32_t *items, int r, int c, int B, const float *zr)
{
    const int32_t q = (int32_t)(((int64_t)r * S.dim + c) % B);
    return fmx_expf(__fsub_rn(zr[c], S.zmax[items[q]]));
}

__global__ void __launch_bounds__(ATTN_WARPS * 32) fm_attn_kernel(Slot S, int k, const int64_t *chunk_start, const int32_t *chunk_rows,
                                                                  int64_t ch0, int64_t ch1, const int32_t *cand_items, int64_t pair_base,
                                                                  const float *vx, float *rowsum, float *score)
{
    extern __shared__ float s_m[];   // [ATTN_WARPS][dim]
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    float *m = s_m + (size_t)w * S.dim;
    for (int64_t ch = ch0 + blockIdx.x; ch < ch1; ch += gridDim.x) {
        const int64_t p0 = chunk_start[ch];
        const int B = chunk_rows[ch];
        const int32_t *items = cand_items + p0;
        float *rs = rowsum + (p0 - pair_base);
        // exp and row sums: y.sum(1, true) starts at the row's first element and adds the rest in order
        for (int r = w; r < B; r += ATTN_WARPS) {
            const float *zr = S.z + (int64_t)items[r] * S.dim;
            float sum = 0.0f;
            for (int c0 = 0; c0 < S.dim; c0 += 32) {
                const float y = c0 + lane < S.dim ? numerator(S, items, r, c0 + lane, B, zr) : 0.0f;
                const int cnt = min(32, S.dim - c0);
                for (int j = 0; j < cnt; j++) {
                    const float v = __shfl_sync(0xffffffffu, y, j);
                    sum = c0 + j == 0 ? v : __fadd_rn(sum, v);
                }
            }
            if (lane == 0) rs[r] = sum;
        }
        __syncthreads();
        for (int r = w; r < B; r += ATTN_WARPS) {
            const int32_t it = items[r];
            const float *zr = S.z + (int64_t)it * S.dim;
            for (int c = lane; c < S.dim; c += 32) {
                const int32_t q = (int32_t)(((int64_t)r * S.dim + c) % B);
                const float a = __fdiv_rn(numerator(S, items, r, c, B, zr), rs[q]);   // y.div(sum): row (r dim + c) % B
                m[c] = __fmul_rn(a, emb_at(S, it, c));                                  // Mul(softmax, e)
            }
            __syncwarp();
            float enc = 0.0f, v = 0.0f;
            if (lane < k) {
                for (int c = 0; c < S.dim; c++) enc = __fmaf_rn(m[c], S.EW[c * k + lane], enc);   // MatMul(., EW)
                enc = __fadd_rn(enc, S.Eb[lane]);                                                // + Eb
                v = vx[(p0 - pair_base + r) * k + lane];
            }
            float dot = 0.0f;
            for (int q = 0; q < k; q++)
                dot = __fmaf_rn(__shfl_sync(0xffffffffu, v, q), __shfl_sync(0xffffffffu, enc, q), dot);   // BMM(vx, enc)
            if (lane == 0) score[p0 + r] = __fadd_rn(score[p0 + r], dot);
            __syncwarp();
        }
        __syncthreads();
    }
}

// ascending key = (descending score, position); -0 sorts with +0 and every NaN after every number
__device__ __forceinline__ uint64_t rank_key(float s, uint32_t pos)
{
    uint32_t hi;
    if (s != s) hi = 0xffffffffu;
    else {
        const uint32_t b = s == 0.0f ? 0u : __float_as_uint(s);
        hi = ~((b & 0x80000000u) ? ~b : (b | 0x80000000u));
    }
    return ((uint64_t)hi << 32) | pos;
}

__global__ void __launch_bounds__(SORT_THREADS) fm_sort_kernel(const int64_t *cand_off, int64_t u0, int64_t u1, const float *score,
                                                               int32_t *order, uint64_t *g_key, int32_t *g_val, int64_t g_stride)
{
    __shared__ uint64_t s_key[SORT_SMEM];
    __shared__ int32_t s_val[SORT_SMEM];
    for (int64_t u = u0 + blockIdx.x; u < u1; u += gridDim.x) {
        const int64_t c0 = cand_off[u];
        const int n = (int)(cand_off[u + 1] - c0);
        if (n == 0) continue;
        const int p = recall::pow2_at_least(n);
        uint64_t *key = p <= SORT_SMEM ? s_key : g_key + blockIdx.x * g_stride;
        int32_t *val = p <= SORT_SMEM ? s_val : g_val + blockIdx.x * g_stride;
        for (int i = threadIdx.x; i < p; i += SORT_THREADS) {
            key[i] = i < n ? rank_key(score[c0 + i], (uint32_t)i) : ~0ull;
            val[i] = i;
        }
        __syncthreads();
        recall::block_sort<SORT_THREADS>(key, val, p);
        for (int i = threadIdx.x; i < n; i += SORT_THREADS) order[c0 + i] = (int32_t)(uint32_t)key[i];
        __syncthreads();
    }
}

Model model(const gorse_b200_fm *m)
{
    const float *P = m->params.p;
    return Model{P + 1, P + 1 + (size_t)m->n_features * m->k, m->bias, m->k};
}

int32_t item_tables(gorse_b200_fm *m, int64_t n_items, bool masked, Slot *S)
{
    gorse_b200_ctx *ctx = m->ctx;
    const float *P = m->params.p;
    for (int s = 0; s < m->n_emb; s++) {
        const int d = m->dim[(size_t)s];
        GB_TRY(m->z[s].grow((size_t)std::max<int64_t>(n_items, 1) * d));
        GB_TRY(m->zmax[s].grow((size_t)std::max<int64_t>(n_items, 1)));
        const float *b = P + m->slot_off[(size_t)s];
        const size_t kd = (size_t)m->k * d;
        S[s] = Slot{b, b + kd, b + 2 * kd, b + 2 * kd + m->k, b + 3 * kd + m->k, m->emb[s].p, masked ? m->mask.p : nullptr,
                    m->n_emb, s, d, m->z[s].p, m->zmax[s].p};
        if (n_items == 0) continue;
        fm_item_kernel<<<(unsigned)std::min<int64_t>((n_items + 7) / 8, (int64_t)ctx->sm_count * 16), 256, 0, ctx->stream>>>(S[s], m->k, n_items);
        GB_LAUNCHED(ctx);
    }
    return GORSE_B200_OK;
}

int32_t rank_pass(gorse_b200_fm *m, const Feats &U, const Feats &I, const int64_t *c_off, const int32_t *cand, const int32_t *dims, int64_t u0,
                  int64_t u1, int64_t pair_base, const Slot *S, const int64_t *ch_start, const int32_t *ch_rows, int64_t ch0, int64_t ch1,
                  int64_t max_n, float *score, int32_t *order, bool *global_sort)
{
    gorse_b200_ctx *ctx = m->ctx;
    cudaStream_t st = ctx->stream;
    const Model M = model(m);
    const int n_emb = m->n_emb;
    const unsigned pg = (unsigned)std::min<int64_t>((u1 - u0 + 7) / 8, (int64_t)ctx->sm_count * 16);
    float *vx = n_emb > 0 ? m->vx.p : nullptr;
    if (m->k <= 8) fm_pair_kernel<8><<<pg, 256, 0, st>>>(M, U, I, c_off, cand, dims, u0, u1, pair_base, score, vx);
    else if (m->k <= 16) fm_pair_kernel<16><<<pg, 256, 0, st>>>(M, U, I, c_off, cand, dims, u0, u1, pair_base, score, vx);
    else fm_pair_kernel<32><<<pg, 256, 0, st>>>(M, U, I, c_off, cand, dims, u0, u1, pair_base, score, vx);
    GB_LAUNCHED(ctx);
    for (int s = 0; s < n_emb && ch1 > ch0; s++) {
        const size_t smem = (size_t)ATTN_WARPS * S[s].dim * sizeof(float);
        fm_attn_kernel<<<(unsigned)std::min<int64_t>(ch1 - ch0, (int64_t)ctx->sm_count * 16), ATTN_WARPS * 32, smem, st>>>(
            S[s], m->k, ch_start, ch_rows, ch0, ch1, cand, pair_base, m->vx.p, m->rowsum.p, score);
        GB_LAUNCHED(ctx);
    }
    int64_t sg = std::min<int64_t>(u1 - u0, (int64_t)ctx->sm_count * 8), stride = 0;
    const int64_t max_p = recall::pow2_at_least((int)std::max<int64_t>(max_n, 1));
    *global_sort = max_p > SORT_SMEM;
    if (*global_sort) {   // a global key / position buffer per CTA, at most 256 MB of them
        stride = max_p;
        sg = std::max<int64_t>(1, std::min<int64_t>(sg, (int64_t(256) << 20) / (max_p * 12)));
        GB_TRY(m->sort_key.grow((size_t)(sg * stride)));
        GB_TRY(m->sort_val.grow((size_t)(sg * stride)));
    }
    fm_sort_kernel<<<(unsigned)sg, SORT_THREADS, 0, st>>>(c_off, u0, u1, score, order, m->sort_key.p, m->sort_val.p, stride);
    GB_LAUNCHED(ctx);
    return GORSE_B200_OK;
}

}  // namespace fm
}  // namespace gb

using namespace gb;

extern "C" int32_t gorse_b200_fm_create(gorse_b200_ctx *ctx, int64_t n_features, int32_t n_factors, int32_t num_dimension, int32_t batch_size,
                                        int32_t n_emb, const int32_t *emb_dim, const float *params, int64_t n_params, gorse_b200_fm **out)
{
    GB_CHECK_ARG(ctx != nullptr && out != nullptr, "NULL ctx/out");
    *out = nullptr;
    GB_CHECK_ARG(n_features >= 1 && n_features <= INT32_MAX, "n_features = %lld is not in [1, 2^31)", (long long)n_features);
    GB_CHECK_ARG(n_factors >= 1 && num_dimension >= 0 && batch_size >= 1 && n_emb >= 0, "n_factors, batch_size >= 1 and num_dimension, n_emb >= 0");
    GB_CHECK_ARG(n_emb == 0 || emb_dim != nullptr, "emb_dim is NULL");
    GB_CHECK_ARG(params != nullptr, "params is NULL");
    int64_t want = 1 + n_features * (int64_t)n_factors + n_features;
    for (int s = 0; s < n_emb; s++) {
        GB_CHECK_ARG(emb_dim[s] >= 1, "embedding slot %d: dim %d", s, emb_dim[s]);
        want += 3 * (int64_t)n_factors * emb_dim[s] + 2 * (int64_t)n_factors;
    }
    GB_CHECK_ARG(n_params == want, "n_params = %lld, the model has %lld", (long long)n_params, (long long)want);
    if (n_factors > fm::MAX_FACTORS || n_emb > fm::MAX_SLOTS) {
        set_error("fm: n_factors %d (at most %d) or %d embedding slots (at most %d)", n_factors, fm::MAX_FACTORS, n_emb, fm::MAX_SLOTS);
        return GORSE_B200_ERR_UNSUPPORTED;
    }
    for (int s = 0; s < n_emb; s++)
        if (emb_dim[s] > fm::MAX_EMB_DIM) {
            set_error("fm: embedding slot %d has dim %d, at most %d", s, emb_dim[s], fm::MAX_EMB_DIM);
            return GORSE_B200_ERR_UNSUPPORTED;
        }
    ScopedDevice sd(ctx->device);
    gorse_b200_fm *m = new (std::nothrow) gorse_b200_fm();
    if (!m) { set_error("host allocation failed"); return GORSE_B200_ERR_OOM; }
    m->ctx = ctx; m->n_features = n_features; m->k = n_factors; m->num_dimension = num_dimension; m->batch_size = batch_size;
    m->n_emb = n_emb; m->bias = params[0];
    size_t o = 1 + (size_t)n_features * n_factors + (size_t)n_features;   // B, V, W, then the slots
    for (int s = 0; s < n_emb; s++) {
        m->dim.push_back(emb_dim[s]);
        m->slot_off.push_back(o);
        o += 3 * (size_t)n_factors * emb_dim[s] + 2 * (size_t)n_factors;
    }
    int32_t st = m->params.alloc((size_t)n_params);
    if (st == GORSE_B200_OK && cudaMemcpy(m->params.p, params, (size_t)n_params * sizeof(float), cudaMemcpyHostToDevice) != cudaSuccess) {
        set_error("fm: parameter upload failed");
        st = GORSE_B200_ERR_CUDA;
    }
    if (st) { delete m; return st; }
    *out = m;
    return GORSE_B200_OK;
}

extern "C" int32_t gorse_b200_fm_destroy(gorse_b200_fm *m)
{
    if (!m) return GORSE_B200_OK;
    ScopedDevice sd(m->ctx->device);
    delete m;
    return GORSE_B200_OK;
}

namespace gb {
namespace fm {
int32_t upload_feats(gorse_b200_fm *m, int64_t n_users, const int32_t *user_feat, const int64_t *user_lab_off, const int32_t *user_lab_idx,
                     const float *user_lab_val, int64_t n_items, const int32_t *item_feat, const int64_t *item_lab_off, const int32_t *item_lab_idx,
                     const float *item_lab_val, const uint16_t *const *item_emb, const uint8_t *item_emb_mask, Slot *S)
{
    const cudaStream_t st = m->ctx->stream;
    GB_TRY(m->u_feat.upload(user_feat, (size_t)n_users, st));
    GB_TRY(m->u_off.upload(user_lab_off, (size_t)n_users + 1, st));
    GB_TRY(m->u_idx.upload(user_lab_idx, (size_t)user_lab_off[n_users], st));
    GB_TRY(m->u_val.upload(user_lab_val, (size_t)user_lab_off[n_users], st));
    GB_TRY(m->i_feat.upload(item_feat, (size_t)n_items, st));
    GB_TRY(m->i_off.upload(item_lab_off, n_items ? (size_t)n_items + 1 : 0, st));
    GB_TRY(m->i_idx.upload(item_lab_idx, n_items ? (size_t)item_lab_off[n_items] : 0, st));
    GB_TRY(m->i_val.upload(item_lab_val, n_items ? (size_t)item_lab_off[n_items] : 0, st));
    if (m->n_emb == 0) return GORSE_B200_OK;
    if (item_emb_mask) GB_TRY(m->mask.upload(item_emb_mask, (size_t)n_items * m->n_emb, st));
    for (int s = 0; s < m->n_emb; s++) GB_TRY(m->emb[s].upload(n_items ? item_emb[s] : nullptr, (size_t)n_items * m->dim[(size_t)s], st));
    return item_tables(m, n_items, item_emb_mask != nullptr, S);
}
}  // namespace fm
}  // namespace gb

extern "C" int32_t gorse_b200_fm_rank(gorse_b200_fm *m, int64_t n_users, const int32_t *user_feat, const int64_t *user_lab_off,
                                      const int32_t *user_lab_idx, const float *user_lab_val, int64_t n_items, const int32_t *item_feat,
                                      const int64_t *item_lab_off, const int32_t *item_lab_idx, const float *item_lab_val,
                                      const uint16_t *const *item_emb, const uint8_t *item_emb_mask, const int64_t *cand_off,
                                      const int32_t *cand_items, float *scores_out, int32_t *order_out, int64_t *stats_out)
{
    using namespace gb::fm;
    GB_CHECK_ARG(m != nullptr, "fm handle is NULL");
    GB_CHECK_ARG(n_users >= 0 && n_items >= 0, "negative count");
    if (stats_out) std::fill(stats_out, stats_out + 4, 0);
    if (n_users == 0) return GORSE_B200_OK;
    GB_CHECK_ARG(cand_off != nullptr && cand_off[0] == 0, "cand_off is NULL or does not start at 0");
    for (int64_t u = 0; u < n_users; u++)
        GB_CHECK_ARG(cand_off[u + 1] >= cand_off[u] && cand_off[u + 1] - cand_off[u] <= INT32_MAX,
                     "user %lld: candidate offsets decrease or hold 2^31 or more", (long long)u);
    const int64_t total = cand_off[n_users];
    GB_CHECK_ARG(total == 0 || (cand_items != nullptr && scores_out != nullptr && order_out != nullptr), "NULL candidates or outputs");
    for (int64_t t = 0; t < total; t++)
        GB_CHECK_ARG(cand_items[t] >= 0 && cand_items[t] < n_items, "candidate %lld: item row %d is not in [0, %lld)", (long long)t,
                     cand_items[t], (long long)n_items);
    GB_TRY(check_feats("user", n_users, user_feat, user_lab_off, user_lab_idx, user_lab_val, m->n_features));
    GB_TRY(check_feats("item", n_items, item_feat, item_lab_off, item_lab_idx, item_lab_val, m->n_features));
    const int n_emb = m->n_emb;
    if (n_emb > 0 && n_items > 0) {
        GB_CHECK_ARG(item_emb != nullptr, "item_emb is NULL");
        for (int s = 0; s < n_emb; s++) GB_CHECK_ARG(item_emb[s] != nullptr, "item_emb[%d] is NULL", s);
    }
    if (total == 0) return GORSE_B200_OK;
    // D_u = max(numDimension, the longest row of the user's call) (convertToTensors, fm.go:536-539)
    std::vector<int32_t> dims((size_t)n_users);
    for (int64_t u = 0; u < n_users; u++) {
        int64_t longest = 0;
        for (int64_t t = cand_off[u]; t < cand_off[u + 1]; t++) {
            const int32_t it = cand_items[t];
            longest = std::max<int64_t>(longest, (item_feat[it] >= 0) + item_lab_off[it + 1] - item_lab_off[it]);
        }
        const int64_t d = std::max<int64_t>(m->num_dimension, (user_feat[u] >= 0) + user_lab_off[u + 1] - user_lab_off[u] + longest);
        GB_CHECK_ARG(d <= INT32_MAX, "user %lld: rows of 2^31 or more features", (long long)u);
        dims[(size_t)u] = (int32_t)d;
    }
    // BatchInternalPredict's chunks, user by user; each user's first chunk, for cutting the users into device passes
    std::vector<int64_t> ch_start, first_chunk((size_t)n_users + 1);
    std::vector<int32_t> ch_rows;
    for (int64_t u = 0; u < n_users; u++) {
        first_chunk[(size_t)u] = (int64_t)ch_start.size();
        if (n_emb == 0) continue;
        for (int64_t a = cand_off[u]; a < cand_off[u + 1]; a += m->batch_size) {
            ch_start.push_back(a);
            ch_rows.push_back((int32_t)std::min<int64_t>(m->batch_size, cand_off[u + 1] - a));
        }
    }
    first_chunk[(size_t)n_users] = (int64_t)ch_start.size();

    std::lock_guard<std::mutex> lk(m->mu);
    gorse_b200_ctx *ctx = m->ctx;
    ScopedDevice sd(ctx->device);
    cudaStream_t st = ctx->stream;
    Slot S[MAX_SLOTS];
    GB_TRY(upload_feats(m, n_users, user_feat, user_lab_off, user_lab_idx, user_lab_val, n_items, item_feat, item_lab_off, item_lab_idx,
                        item_lab_val, item_emb, item_emb_mask, S));
    GB_TRY(m->c_off.upload(cand_off, (size_t)n_users + 1, st));
    GB_TRY(m->cand.upload(cand_items, (size_t)total, st));
    GB_TRY(m->dims.upload(dims.data(), dims.size(), st));
    GB_TRY(m->score.grow((size_t)total));
    GB_TRY(m->order.grow((size_t)total));

    Feats U{m->u_feat.p, m->u_off.p, m->u_idx.p, m->u_val.p};
    Feats I{m->i_feat.p, m->i_off.p, m->i_idx.p, m->i_val.p};
    if (n_emb > 0) {
        GB_TRY(m->ch_start.upload(ch_start.data(), ch_start.size(), st));
        GB_TRY(m->ch_rows.upload(ch_rows.data(), ch_rows.size(), st));
    }
    // device passes over consecutive users holding at most GROUP_PAIRS pairs (or one user)
    int64_t passes = 0, global_sorts = 0;
    for (int64_t u0 = 0; u0 < n_users;) {
        int64_t u1 = u0 + 1;
        while (u1 < n_users && cand_off[u1 + 1] - cand_off[u0] <= GROUP_PAIRS) u1++;
        const int64_t pb = cand_off[u0], np = cand_off[u1] - pb;
        int64_t max_n = 0;
        for (int64_t u = u0; u < u1; u++) max_n = std::max<int64_t>(max_n, cand_off[u + 1] - cand_off[u]);
        if (np > 0) {
            passes++;
            if (n_emb > 0) {
                GB_TRY(m->vx.grow((size_t)np * m->k));
                GB_TRY(m->rowsum.grow((size_t)np));
            }
            bool global_sort = false;
            GB_TRY(rank_pass(m, U, I, m->c_off.p, m->cand.p, m->dims.p, u0, u1, pb, S, m->ch_start.p, m->ch_rows.p, first_chunk[(size_t)u0],
                             first_chunk[(size_t)u1], max_n, m->score.p, m->order.p, &global_sort));
            if (global_sort)
                for (int64_t u = u0; u < u1; u++) global_sorts += recall::pow2_at_least((int)(cand_off[u + 1] - cand_off[u])) > SORT_SMEM;
        }
        u0 = u1;
    }
    GB_CUDA(cudaMemcpyAsync(scores_out, m->score.p, (size_t)total * sizeof(float), cudaMemcpyDeviceToHost, st));
    GB_CUDA(cudaMemcpyAsync(order_out, m->order.p, (size_t)total * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    GB_CUDA(cudaStreamSynchronize(st));
    if (stats_out) {
        stats_out[0] = total;
        stats_out[1] = (int64_t)ch_start.size();
        stats_out[2] = passes;
        stats_out[3] = global_sorts;
    }
    return GORSE_B200_OK;
}
