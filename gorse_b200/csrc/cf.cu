// cf.cu -- CF model state: create/destroy, factor upload/download, normal init, batched Predict.
#include <algorithm>
#include <cstdlib>
#include <thread>

#include "cf.cuh"

namespace gb {

// N(mean, std) via Box-Muller on the counter RNG; element e of the (users ++ items) stream
__global__ void init_normal_kernel(float *dst, int64_t n, int64_t stream_off, uint64_t base, float mean, float stddev)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) {
        SStream s;
        s.x = mix64(base + (uint64_t)(stream_off + i));
        float u1 = ((float)(s.next32() >> 8) + 0.5f) * (1.0f / 16777216.0f);
        float u2 = ((float)(s.next32() >> 8) + 0.5f) * (1.0f / 16777216.0f);
        float r = sqrtf(-2.0f * logf(u1));
        float z = r * cospif(2.0f * u2);
        dst[i] = z * stddev + mean;  // float32(NormFloat64())*stdDev + mean, common/util/random.go:48
    }
}

// Predict for d % 16 == 0: one quad per (u, i) pair
__global__ void predict_quad_kernel(const float *P, const float *Q, int d, int32_t u_lo, const int32_t *users,
                                    const int32_t *items, int64_t n, float *out)
{
    int lane4 = threadIdx.x & 3;
    unsigned mask = quad_mask();
    int64_t g = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 2;
    int64_t ng = ((int64_t)gridDim.x * blockDim.x) >> 2;
    for (; g < n; g += ng) {
        float v = quad_dot_global(P + (int64_t)(users[g] - u_lo) * d, Q + (int64_t)items[g] * d, d / 16, lane4, mask);
        if (lane4 == 0) out[g] = v;
    }
}

__global__ void predict_any_kernel(const float *P, const float *Q, int d, int32_t u_lo, const int32_t *users,
                                   const int32_t *items, int64_t n, float *out)
{
    int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t ng = (int64_t)gridDim.x * blockDim.x;
    for (; g < n; g += ng) out[g] = dot_any(P + (int64_t)(users[g] - u_lo) * d, Q + (int64_t)items[g] * d, d);
}

// offsets may start anywhere (a rank's slice of a global CSR keeps its global offsets); everything is rebased to off[0]
static bool csr_valid(const int64_t *off, int32_t rows, const int32_t *idx, int32_t id_bound, const char *what)
{
    for (int32_t r = 0; r < rows; r++)
        if (off[r + 1] < off[r]) {
            set_error("%s_off is not non-decreasing at row %d", what, r);
            return false;
        }
    const int64_t nnz = off[rows] - off[0];
    const unsigned nt = nnz < (1 << 18) ? 1u : std::max(1u, std::min(16u, std::thread::hardware_concurrency()));
    std::vector<int64_t> bad(nt, -1);
    auto work = [&](unsigned t) {
        const int64_t t0 = nnz * t / nt, t1 = nnz * (t + 1) / nt;
        for (int64_t k = t0; k < t1; k++)
            if (idx[k] < 0 || idx[k] >= id_bound) { bad[t] = k; return; }
    };
    if (nt == 1) work(0);
    else {
        std::vector<std::thread> th;
        for (unsigned t = 0; t < nt; t++) th.emplace_back(work, t);
        for (auto &x : th) x.join();
    }
    for (unsigned t = 0; t < nt; t++)
        if (bad[t] >= 0) {
            set_error("%s index %d at position %lld out of range [0, %d)", what, idx[bad[t]], (long long)bad[t], id_bound);
            return false;
        }
    return true;
}

template <typename F>
static void parallel_rows(int32_t rows, int64_t nnz, F &&work)
{
    unsigned nt = std::max(1u, std::min(16u, std::thread::hardware_concurrency()));
    if (nnz < (1 << 16)) nt = 1;
    if (nt == 1) {
        work(0, rows, 0u);
        return;
    }
    std::vector<std::thread> th;
    for (unsigned t = 0; t < nt; t++)
        th.emplace_back(work, (int32_t)((int64_t)rows * t / nt), (int32_t)((int64_t)rows * (t + 1) / nt), t);
    for (auto &x : th) x.join();
}

}  // namespace gb

using namespace gb;

extern "C" {

int32_t gorse_b200_cf_create(gorse_b200_ctx *ctx, int32_t n_users, int32_t n_items, int32_t n_factors,
                             const int64_t *user_off, const int32_t *user_items,
                             const int64_t *item_off, const int32_t *item_users,
                             gorse_b200_cf **out)
{
    GB_CHECK_ARG(ctx != nullptr && out != nullptr, "NULL ctx/out");
    *out = nullptr;
    const bool multi = ctx->world > 1;
    // this rank's rows: users [u_lo, u_hi) and (ALS) items [i_lo, i_hi); everything when world = 1
    const int32_t u_lo = (int32_t)((int64_t)n_users * ctx->rank / ctx->world), u_hi = (int32_t)((int64_t)n_users * (ctx->rank + 1) / ctx->world);
    const int32_t i_lo = (int32_t)((int64_t)n_items * ctx->rank / ctx->world), i_hi = (int32_t)((int64_t)n_items * (ctx->rank + 1) / ctx->world);
    const int32_t nu = u_hi - u_lo, ni = i_hi - i_lo;
    const bool has_items = item_off != nullptr;
    // Validation never returns before the collective below in a distributed context: a rank with bad arguments
    // reports through the all-reduced failure count, so that the other ranks fail with it instead of hanging.
    int32_t vst = GORSE_B200_OK;
    auto validate = [&]() -> int32_t {
        GB_CHECK_ARG(n_users >= 0 && n_items >= 0, "negative table size");
        GB_CHECK_ARG(n_factors >= 1 && n_factors <= 4096, "n_factors %d out of range [1, 4096]", n_factors);
        GB_CHECK_ARG(user_off != nullptr, "user_off is NULL");
        GB_CHECK_ARG(user_off[nu] == user_off[0] || user_items != nullptr, "user_items is NULL");
        if (!csr_valid(user_off, nu, user_items, n_items, "user")) return GORSE_B200_ERR_ARG;
        if (has_items) {
            GB_CHECK_ARG(item_off[ni] == item_off[0] || item_users != nullptr, "item_users is NULL");
            if (!csr_valid(item_off, ni, item_users, n_users, "item")) return GORSE_B200_ERR_ARG;
            GB_CHECK_ARG(multi || item_off[ni] - item_off[0] == user_off[nu] - user_off[0], "user and item CSR disagree on feedback count");
        }
        if (user_off[nu] - user_off[0] >= (1ll << 38)) { set_error("more than 2^38 feedback entries are not supported"); return GORSE_B200_ERR_UNSUPPORTED; }
        return GORSE_B200_OK;
    };
    vst = validate();
    if (vst != GORSE_B200_OK && !multi) return vst;
    ScopedDevice sd(ctx->device);
    int64_t n_fb_local = vst == GORSE_B200_OK ? user_off[nu] - user_off[0] : 0, n_fb_global = n_fb_local;
    if (multi) {
        // one small collective: [ranks that failed validation, feedback by user rows, feedback by item rows]
        long long h[3] = {vst != GORSE_B200_OK, (long long)n_fb_local, vst == GORSE_B200_OK && has_items ? (long long)(item_off[ni] - item_off[0]) : 0};
        DevBuf<long long> dcnt;
        const std::string keep = gorse_b200_last_error();
        GB_NCCL_API(nc);
        GB_TRY(dcnt.alloc(3));
        cudaError_t e = cudaMemcpyAsync(dcnt.p, h, sizeof(h), cudaMemcpyHostToDevice, ctx->stream);
        ncclResult_t r = e == cudaSuccess ? nc->AllReduce(dcnt.p, dcnt.p, 3, ncclInt64, ncclSum, ctx->comm, ctx->stream) : ncclSuccess;
        if (e == cudaSuccess && r == ncclSuccess) e = cudaMemcpyAsync(h, dcnt.p, sizeof(h), cudaMemcpyDeviceToHost, ctx->stream);
        if (e == cudaSuccess && r == ncclSuccess) e = cudaStreamSynchronize(ctx->stream);
        dcnt.free();
        if (r != ncclSuccess) { set_error("cf_create: ncclAllReduce -> %s", nc->GetErrorString(r)); return GORSE_B200_ERR_NCCL; }
        if (e != cudaSuccess) { set_error("cf_create: %s", cudaGetErrorString(e)); return GORSE_B200_ERR_CUDA; }
        if (vst != GORSE_B200_OK) { set_error("%s", keep.c_str()); return vst; }
        if (h[0] != 0) { set_error("cf_create failed on %lld other rank(s)", h[0]); return GORSE_B200_ERR_STATE; }
        if (has_items && h[1] != h[2]) { set_error("user and item CSR disagree on the global feedback count (%lld vs %lld)", h[1], h[2]); return GORSE_B200_ERR_ARG; }
        n_fb_global = h[1];
    }
    gorse_b200_cf *cf = new (std::nothrow) gorse_b200_cf();
    if (!cf) {
        set_error("host allocation failed");
        return GORSE_B200_ERR_OOM;
    }
    cf->ctx = ctx;
    cf->n_users = n_users;
    cf->n_items = n_items;
    cf->d = n_factors;
    cf->u_lo = u_lo; cf->u_hi = u_hi; cf->i_lo = i_lo; cf->i_hi = i_hi;
    cf->n_feedback = n_fb_local;
    cf->n_feedback_global = n_fb_global;
    cf->has_item_csr = has_items;
    // rebased host copies of this rank's offsets (ALS bucketing)
    cf->h_user_off.resize((size_t)nu + 1);
    for (int32_t r = 0; r <= nu; r++) cf->h_user_off[(size_t)r] = user_off[r] - user_off[0];
    if (has_items) {
        cf->h_item_off.resize((size_t)ni + 1);
        for (int32_t r = 0; r <= ni; r++) cf->h_item_off[(size_t)r] = item_off[r] - item_off[0];
        cf->n_item_feedback = cf->h_item_off[(size_t)ni];
    }
    const std::vector<int64_t> &uoff = cf->h_user_off;

    int32_t st = GORSE_B200_OK;
    auto fail = [&](int32_t s) {
        gorse_b200_cf_destroy(cf);
        return s;
    };
    // per row: sort ascending (device copy only; sampling i ~ U(R_u) does not depend on the order), 64-bit Bloom signature
    std::vector<int32_t> sorted(user_items, user_items + n_fb_local);
    std::vector<UserMeta> meta((size_t)nu);
    std::vector<int32_t> too_long(16, -1);
    parallel_rows(nu, n_fb_local, [&](int32_t r0, int32_t r1, unsigned t) {
        for (int32_t r = r0; r < r1; r++) {
            const int64_t o = uoff[(size_t)r], len = uoff[(size_t)r + 1] - o;
            int32_t *b = sorted.data() + o, *e = b + len;
            if (!std::is_sorted(b, e)) std::sort(b, e);
            if (len >= (1ll << 26)) { too_long[t] = r; continue; }
            uint64_t bloom = 0;
            for (int64_t k = 0; k < len; k++) bloom |= UserMeta::bit(b[k]);
            meta[(size_t)r].off_len = (uint64_t)o | ((uint64_t)len << 38);
            meta[(size_t)r].bloom = bloom;
        }
    });
    for (int32_t r : too_long)
        if (r >= 0) { set_error("user %d has more than 2^26 feedback entries", u_lo + r); return fail(GORSE_B200_ERR_UNSUPPORTED); }
    std::vector<int32_t> active;
    for (int32_t r = 0; r < nu; r++)
        if (uoff[(size_t)r + 1] > uoff[(size_t)r]) active.push_back(u_lo + r);
    cf->n_active = (int32_t)active.size();
    cf->all_active = cf->n_active == nu;

    // multi-GPU exchange: expected updates of item i per local step.  The positive-sampling mass P(i) is proportional to
    // sum_{u in R_i} 1/|R_u| (user uniform, then item uniform in the row)
    std::vector<float> item_rate;
    if (multi) {
        // per-thread partial masses, added in thread order: deterministic for a given thread count
        std::vector<std::vector<double>> part(16);
        parallel_rows(nu, n_fb_local, [&](int32_t r0, int32_t r1, unsigned t) {
            std::vector<double> &m = part[t];
            m.assign((size_t)n_items, 0.0);
            for (int32_t r = r0; r < r1; r++) {
                const int64_t o = uoff[(size_t)r], len = uoff[(size_t)r + 1] - o;
                const double w = len ? 1.0 / (double)len : 0.0;
                for (int64_t k = 0; k < len; k++) m[(size_t)sorted[(size_t)(o + k)]] += w;
            }
        });
        std::vector<double> mass((size_t)n_items, 0.0);
        for (auto &m : part)
            if (!m.empty()) for (int32_t i = 0; i < n_items; i++) mass[(size_t)i] += m[(size_t)i];
        const double total = std::max(1, cf->n_active);
        // P(i is the positive) + P(i is the negative ~ uniform)
        item_rate.resize((size_t)n_items);
        for (int32_t i = 0; i < n_items; i++) item_rate[(size_t)i] = (float)(mass[(size_t)i] / total + 1.0 / (double)n_items);
    }
    if ((st = cf->P.alloc((size_t)nu * n_factors)) != 0) return fail(st);
    if ((st = cf->Q.alloc((size_t)n_items * n_factors)) != 0) return fail(st);
    if (multi) {
        if ((st = cf->Q0.alloc((size_t)n_items * n_factors)) != 0) return fail(st);
        if ((st = cf->item_rate.alloc((size_t)n_items)) != 0) return fail(st);
        if ((st = cf->xchg.alloc((size_t)2 * n_items + 4)) != 0) return fail(st);
    }
    if ((st = cf->user_off.alloc((size_t)nu + 1)) != 0) return fail(st);
    if ((st = cf->user_items.alloc((size_t)n_fb_local)) != 0) return fail(st);
    if ((st = cf->active.alloc(active.size())) != 0) return fail(st);
    if ((st = cf->user_meta.alloc((size_t)nu)) != 0) return fail(st);
    cudaStream_t s = ctx->stream;
    auto up = [&](void *dst, const void *src, size_t bytes) -> int32_t {
        if (bytes == 0) return GORSE_B200_OK;
        GB_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, s));
        return GORSE_B200_OK;
    };
    if ((st = up(cf->user_off.p, uoff.data(), sizeof(int64_t) * ((size_t)nu + 1))) != 0) return fail(st);
    if ((st = up(cf->user_items.p, sorted.data(), sizeof(int32_t) * (size_t)n_fb_local)) != 0) return fail(st);
    if ((st = up(cf->active.p, active.data(), sizeof(int32_t) * active.size())) != 0) return fail(st);
    if ((st = up(cf->user_meta.p, meta.data(), sizeof(UserMeta) * meta.size())) != 0) return fail(st);
    if ((st = up(cf->item_rate.p, item_rate.data(), sizeof(float) * item_rate.size())) != 0) return fail(st);
    if (has_items) {
        if ((st = cf->item_off.alloc((size_t)ni + 1)) != 0) return fail(st);
        if ((st = cf->item_users.alloc((size_t)cf->n_item_feedback)) != 0) return fail(st);
        if ((st = up(cf->item_off.p, cf->h_item_off.data(), sizeof(int64_t) * ((size_t)ni + 1))) != 0) return fail(st);
        if ((st = up(cf->item_users.p, item_users, sizeof(int32_t) * (size_t)cf->n_item_feedback)) != 0) return fail(st);
    }
    if (cf->P.n) cudaMemsetAsync(cf->P.p, 0, cf->P.n * sizeof(float), s);
    if (cf->Q.n) cudaMemsetAsync(cf->Q.p, 0, cf->Q.n * sizeof(float), s);
    cudaError_t e = cudaStreamSynchronize(s);  // host staging vectors die at return
    if (e != cudaSuccess) {
        set_error("cf_create: %s", cudaGetErrorString(e));
        return fail(GORSE_B200_ERR_CUDA);
    }
    *out = cf;
    return GORSE_B200_OK;
}

int32_t gorse_b200_cf_destroy(gorse_b200_cf *cf)
{
    if (!cf) return GORSE_B200_OK;
    ScopedDevice sd(cf->ctx->device);
    cudaStreamSynchronize(cf->ctx->stream);
    cf->P.free(); cf->Q.free(); cf->Q0.free(); cf->item_rate.free(); cf->xchg.free(); cf->P_all.free();
    cf->user_off.free(); cf->item_off.free();
    cf->user_items.free(); cf->item_users.free(); cf->active.free(); cf->user_meta.free();
    cf->gram.free();
    for (int a = 0; a < 2; a++) {
        for (int b = 0; b < 7; b++) cf->als_rows[a][b].free();
        cf->als_chunk_len[a].free(); cf->als_row_chunk0[a].free(); cf->als_chunk_begin[a].free();
        cf->als_s_rows[a].free(); cf->als_s_len[a].free(); cf->als_s_begin[a].free();
    }
    cf->als_partial.free(); cf->als_pred.free();
    delete cf;
    return GORSE_B200_OK;
}

int32_t gorse_b200_cf_set_factors(gorse_b200_cf *cf, const float *P, const float *Q)
{
    GB_CHECK_ARG(cf != nullptr, "cf is NULL");
    GB_CHECK_ARG((P != nullptr || cf->n_users == 0) && (Q != nullptr || cf->n_items == 0), "NULL factor table");
    ScopedDevice sd(cf->ctx->device);
    cudaStream_t s = cf->ctx->stream;
    if (cf->P.n)
        GB_CUDA(cudaMemcpyAsync(cf->P.p, P + (int64_t)cf->u_lo * cf->d, cf->P.n * sizeof(float), cudaMemcpyHostToDevice, s));
    if (cf->Q.n) GB_CUDA(cudaMemcpyAsync(cf->Q.p, Q, cf->Q.n * sizeof(float), cudaMemcpyHostToDevice, s));
    if (cf->Q0.n) GB_CUDA(cudaMemcpyAsync(cf->Q0.p, cf->Q.p, cf->Q.n * sizeof(float), cudaMemcpyDeviceToDevice, s));
    GB_CUDA(cudaStreamSynchronize(s));
    return GORSE_B200_OK;
}

int32_t gorse_b200_cf_get_factors(gorse_b200_cf *cf, float *P, float *Q)
{
    GB_CHECK_ARG(cf != nullptr, "cf is NULL");
    ScopedDevice sd(cf->ctx->device);
    cudaStream_t s = cf->ctx->stream;
    // in a distributed context each rank fills its own user rows of the shared host mirror
    if (P && cf->P.n)
        GB_CUDA(cudaMemcpyAsync(P + (int64_t)cf->u_lo * cf->d, cf->P.p, cf->P.n * sizeof(float), cudaMemcpyDeviceToHost, s));
    if (Q && cf->Q.n) GB_CUDA(cudaMemcpyAsync(Q, cf->Q.p, cf->Q.n * sizeof(float), cudaMemcpyDeviceToHost, s));
    GB_CUDA(cudaStreamSynchronize(s));
    return GORSE_B200_OK;
}

int32_t gorse_b200_cf_init_normal(gorse_b200_cf *cf, float mean, float stddev, uint64_t seed)
{
    GB_CHECK_ARG(cf != nullptr, "cf is NULL");
    ScopedDevice sd(cf->ctx->device);
    gorse_b200_ctx *c = cf->ctx;
    uint64_t base = mix64(seed ^ 0x6a09e667f3bcc908ull);
    // element index in the reference's stream order: users then items (model/cf/model.go:534-535)
    if (cf->P.n) {
        init_normal_kernel<<<c->sm_count * 8, 256, 0, c->stream>>>(cf->P.p, (int64_t)cf->P.n,
                                                                  (int64_t)cf->u_lo * cf->d, base, mean, stddev);
        GB_LAUNCHED(c);
    }
    if (cf->Q.n) {
        init_normal_kernel<<<c->sm_count * 8, 256, 0, c->stream>>>(cf->Q.p, (int64_t)cf->Q.n,
                                                                  (int64_t)cf->n_users * cf->d, base, mean, stddev);
        GB_LAUNCHED(c);
    }
    // every rank generates the same replicated Q; keep the epoch-start copy used by the delta exchange
    if (cf->Q0.n) GB_CUDA(cudaMemcpyAsync(cf->Q0.p, cf->Q.p, cf->Q.n * sizeof(float), cudaMemcpyDeviceToDevice, c->stream));
    return GORSE_B200_OK;
}

int32_t gorse_b200_cf_predict(gorse_b200_cf *cf, const int32_t *users, const int32_t *items, int64_t n, float *out)
{
    GB_CHECK_ARG(cf != nullptr, "cf is NULL");
    GB_CHECK_ARG(n >= 0, "negative n");
    if (n == 0) return GORSE_B200_OK;
    GB_CHECK_ARG(users && items && out, "NULL argument");
    for (int64_t t = 0; t < n; t++) {
        GB_CHECK_ARG(users[t] >= cf->u_lo && users[t] < cf->u_hi, "user %d outside this rank's shard [%d, %d)", users[t],
                     cf->u_lo, cf->u_hi);
        GB_CHECK_ARG(items[t] >= 0 && items[t] < cf->n_items, "item %d out of range", items[t]);
    }
    ScopedDevice sd(cf->ctx->device);
    gorse_b200_ctx *c = cf->ctx;
    DevBuf<int32_t> du, di;
    DevBuf<float> dout;
    int32_t st;
    if ((st = du.alloc(n)) || (st = di.alloc(n)) || (st = dout.alloc(n))) {
        du.free(); di.free(); dout.free();
        return st;
    }
    auto done = [&](int32_t s) {
        du.free(); di.free(); dout.free();
        return s;
    };
    cudaError_t e;
    if ((e = cudaMemcpyAsync(du.p, users, n * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream)) != cudaSuccess ||
        (e = cudaMemcpyAsync(di.p, items, n * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream)) != cudaSuccess) {
        set_error("predict upload: %s", cudaGetErrorString(e));
        return done(GORSE_B200_ERR_CUDA);
    }
    if (cf->d % 16 == 0) {
        int blocks = std::min<int64_t>(div_up(n * 4, 256), (int64_t)c->sm_count * 16);
        predict_quad_kernel<<<blocks, 256, 0, c->stream>>>(cf->P.p, cf->Q.p, cf->d, cf->u_lo, du.p, di.p, n, dout.p);
    } else {
        int blocks = std::min<int64_t>(div_up(n, 128), (int64_t)c->sm_count * 16);
        predict_any_kernel<<<blocks, 128, 0, c->stream>>>(cf->P.p, cf->Q.p, cf->d, cf->u_lo, du.p, di.p, n, dout.p);
    }
    c->launches++;
    if ((e = cudaGetLastError()) != cudaSuccess ||
        (e = cudaMemcpyAsync(out, dout.p, n * sizeof(float), cudaMemcpyDeviceToHost, c->stream)) != cudaSuccess ||
        (e = cudaStreamSynchronize(c->stream)) != cudaSuccess) {
        set_error("predict: %s", cudaGetErrorString(e));
        return done(GORSE_B200_ERR_CUDA);
    }
    return done(GORSE_B200_OK);
}

}  // extern "C"
