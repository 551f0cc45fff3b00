// evaluate.cu -- cf.Evaluate on device: model/cf/evaluator.go:35-72 with scorers NDCG, Precision, Recall.
// Kernel 1 scores every (user, candidate) pair with floats.Dot order (internalPredict); kernel 2 runs the
// reference's TopKFilter (Go container/heap, common/heap/filter.go:35-59) per user and the metrics;
// the host adds the per-user metrics in user order, which is the reference with Jobs = 1.
#include <cmath>

#include "cf.cuh"
#include "evaluate.cuh"
#include "tables.cuh"

namespace gb {

__global__ void eval_score_kernel(const float *P, const float *Q, int d, int32_t u_lo, const int32_t *cand_user,
                                  const int32_t *cand_item, int64_t n, float *score)
{
    if (d % 16 == 0) {
        int lane4 = threadIdx.x & 3;
        unsigned mask = quad_mask();
        int64_t g = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 2;
        int64_t ng = ((int64_t)gridDim.x * blockDim.x) >> 2;
        for (; g < n; g += ng) {
            float v = quad_dot_global(P + (int64_t)(cand_user[g] - u_lo) * d, Q + (int64_t)cand_item[g] * d, d / 16, lane4, mask);
            if (lane4 == 0) score[g] = v;
        }
    } else {
        int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
        int64_t ng = (int64_t)gridDim.x * blockDim.x;
        for (; g < n; g += ng) score[g] = dot_any(P + (int64_t)(cand_user[g] - u_lo) * d, Q + (int64_t)cand_item[g] * d, d);
    }
}

// Go container/heap on a min-heap of (value, weight): Less = strict weight compare (common/heap/pq.go:42-48)
struct GoMinHeap {
    int32_t v[GB_EVAL_MAX_TOPK + 1];
    float w[GB_EVAL_MAX_TOPK + 1];
    int n;
    __device__ void swap(int i, int j)
    {
        int32_t tv = v[i]; v[i] = v[j]; v[j] = tv;
        float tw = w[i]; w[i] = w[j]; w[j] = tw;
    }
    __device__ void up(int j)
    {
        for (;;) {
            int i = (j - 1) / 2;
            if (i == j || !(w[j] < w[i])) break;
            swap(i, j);
            j = i;
        }
    }
    __device__ void down(int i0, int nn)
    {
        int i = i0;
        for (;;) {
            int j1 = 2 * i + 1;
            if (j1 >= nn || j1 < 0) break;
            int j = j1, j2 = j1 + 1;
            if (j2 < nn && w[j2] < w[j1]) j = j2;
            if (!(w[j] < w[i])) break;
            swap(i, j);
            i = j;
        }
    }
    __device__ void push(int32_t val, float wt)
    {
        v[n] = val; w[n] = wt; n++;
        up(n - 1);
    }
    __device__ int32_t pop()
    {
        int nn = n - 1;
        swap(0, nn);
        down(0, nn);
        n--;
        return v[n];
    }
};

// one thread per user: Rank (evaluator.go:162-169) + NDCG/Precision/Recall (:75-116)
__global__ void eval_rank_kernel(const int64_t *cand_off, const int32_t *cand_item, const float *score,
                                 const int64_t *test_off, const int32_t *test_items, int32_t n_users, int32_t topk,
                                 const float *inv_log2, float *metrics /* n_users x 4: ndcg, prec, recall, valid */)
{
    int32_t u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= n_users) return;
    int64_t t0 = test_off[u], nt = test_off[u + 1] - t0;
    float *m = metrics + 4 * (int64_t)u;
    if (nt <= 0) { m[0] = m[1] = m[2] = m[3] = 0.f; return; }
    GoMinHeap h;
    h.n = 0;
    int64_t c0 = cand_off[u], nc = cand_off[u + 1] - c0;
    for (int64_t c = 0; c < nc; c++) {
        h.push(cand_item[c0 + c], score[c0 + c]);
        if (h.n > topk) (void)h.pop();
    }
    int nr = h.n;
    int32_t rank[GB_EVAL_MAX_TOPK];
    for (int i = nr - 1; i >= 0; i--) rank[i] = h.pop();  // PopAllValues: decreasing weight
    const int32_t *tgt = test_items + t0;
    // mapset cardinality = distinct test items
    int card = 0;
    for (int64_t a = 0; a < nt; a++) {
        bool dup = false;
        for (int64_t b = 0; b < a; b++) if (tgt[b] == tgt[a]) { dup = true; break; }
        if (!dup) card++;
    }
    float idcg = 0.f, dcg = 0.f, hit = 0.f;
    for (int i = 0; i < card && i < nr; i++) idcg = idcg + inv_log2[i];
    for (int i = 0; i < nr; i++) {
        bool in = false;
        for (int64_t a = 0; a < nt; a++) if (tgt[a] == rank[i]) { in = true; break; }
        if (in) { dcg = dcg + inv_log2[i]; hit = hit + 1.0f; }
    }
    m[0] = dcg / idcg;
    m[1] = hit / (float)nr;
    m[2] = hit / (float)card;
    m[3] = 1.f;
}

// math32.Log2 as restated in DESIGN.md (frexp, Log(frac) * (1/Ln2) + exp)
static float log2_math32(float x)
{
    int e;
    float frac = frexpf(x, &e);
    if (frac == 0.5f) return (float)(e - 1);
    volatile float l = logf(frac);
    volatile float inv = (float)(1.0 / 0.693147180559945309417232121458176568);
    volatile float p = l * inv;
    return p + (float)e;
}


// dataset.SampleUserNegatives (dataset/dataset.go:242-253) -> util.SampleInt32 (common/util/random.go:108-132) for one
// user per thread: n distinct items outside train(u) + test(u); when fewer than n + 1 remain, all of them, ascending.
// count_only: write only the number of negatives the user will get.  The Go math/rand stream is unreproducible (SURVEY F9):
// the draws come from the library's counter RNG (shared bit for bit with the oracle), the distribution is the reference's.
__global__ void eval_negatives_kernel(const int64_t *train_off, const int32_t *train_items, const int64_t *test_off,
                                      const int32_t *test_items, int32_t n_users, int32_t u_lo, int32_t n_items, int32_t n_cand,
                                      uint64_t base, bool count_only, int32_t *n_neg, const int64_t *neg_off, int32_t *neg_items)
{
    const int32_t u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= n_users) return;
    const int32_t *tr = train_items + train_off[u];
    const int64_t ntr = train_off[u + 1] - train_off[u];
    const int32_t *te = test_items + test_off[u];
    const int64_t nte = test_off[u + 1] - test_off[u];
    auto excluded = [&](int32_t v) {
        if (row_contains(tr, ntr, v)) return true;
        for (int64_t a = 0; a < nte; a++) if (te[a] == v) return true;
        return false;
    };
    if (count_only) {
        // cardinality of train(u) | test(u): train rows are sorted (duplicates adjacent)
        int64_t card = 0;
        for (int64_t a = 0; a < ntr; a++) if (a == 0 || tr[a] != tr[a - 1]) card++;
        for (int64_t a = 0; a < nte; a++) {
            bool dup = row_contains(tr, ntr, te[a]);
            for (int64_t b = 0; b < a && !dup; b++) dup = te[b] == te[a];
            if (!dup) card++;
        }
        n_neg[u] = (int32_t)((int64_t)n_cand >= (int64_t)n_items - card ? (int64_t)n_items - card : (int64_t)n_cand);
        return;
    }
    int32_t *out = neg_items + neg_off[u];
    const int32_t n = (int32_t)(neg_off[u + 1] - neg_off[u]);
    if (n < n_cand) {   // the "take everything that is left" branch (:116-122)
        int32_t k = 0;
        for (int32_t v = 0; v < n_items && k < n; v++) if (!excluded(v)) out[k++] = v;
        return;
    }
    SStream s;
    s.x = mix64(base + (uint64_t)(u_lo + u));
    int32_t k = 0;
    while (k < n) {
        const int32_t v = (int32_t)s.bounded((uint32_t)n_items);
        if (excluded(v)) continue;
        bool dup = false;
        for (int32_t b = 0; b < k && !dup; b++) dup = out[b] == v;
        if (!dup) out[k++] = v;
    }
}

// candidates of user u = test(u) ++ negatives(u) (evaluator.go:51-53); users without test items get none
__global__ void eval_candidates_kernel(const int64_t *test_off, const int32_t *test_items, const int64_t *neg_off,
                                       const int32_t *neg_items, int32_t n_users, int32_t u_lo, const int64_t *cand_off,
                                       int32_t *cand_user, int32_t *cand_item)
{
    const int32_t u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= n_users) return;
    int64_t p = cand_off[u];
    if (cand_off[u + 1] == p) return;
    for (int64_t a = test_off[u]; a < test_off[u + 1]; a++, p++) { cand_user[p] = u_lo + u; cand_item[p] = test_items[a]; }
    for (int64_t a = neg_off[u]; a < neg_off[u + 1]; a++, p++) { cand_user[p] = u_lo + u; cand_item[p] = neg_items[a]; }
}

void eval_inv_log2(int32_t topk, float *out)
{
    for (int i = 0; i < topk; i++) out[i] = 1.0f / log2_math32((float)i + 2.0f);
}

void launch_eval_rank(cudaStream_t s, const int64_t *cand_off, const int32_t *cand_item, const float *score, const int64_t *test_off,
                      const int32_t *test_items, int32_t n_users, int32_t topk, const float *inv_log2, float *metrics)
{
    if (n_users > 0)
        eval_rank_kernel<<<(n_users + 127) / 128, 128, 0, s>>>(cand_off, cand_item, score, test_off, test_items, n_users, topk, inv_log2, metrics);
}

void launch_eval_negatives(cudaStream_t s, const int64_t *excl_off, const int32_t *excl_items, const int64_t *test_off,
                           const int32_t *test_items, int32_t n_users, int32_t u_lo, int32_t n_items, int32_t n_cand, uint64_t base,
                           bool count_only, int32_t *n_neg, const int64_t *neg_off, int32_t *neg_items)
{
    if (n_users > 0)
        eval_negatives_kernel<<<(n_users + 127) / 128, 128, 0, s>>>(excl_off, excl_items, test_off, test_items, n_users, u_lo, n_items,
                                                                     n_cand, base, count_only, n_neg, neg_off, neg_items);
}

}  // namespace gb

using namespace gb;

// Evaluate's inputs resident in HBM (built once per Fit; the reference caches its negatives the same way, dataset.go:243)
struct gorse_b200_eval {
    gorse_b200_cf *cf = nullptr;
    int32_t U = 0, topk = 0;
    int64_t nc = 0, n_neg = 0;
    DevBuf<int64_t> test_off, neg_off, cand_off;
    DevBuf<int32_t> test_items, neg_items, cand_user, cand_item;
    DevBuf<float> score, inv, metrics;
    std::vector<float> h_metrics;
    std::vector<int64_t> h_neg_off;
};

int32_t gb::eval_run_tables(gorse_b200_eval *ev, const float *P, const float *Q, float *out)
{
    gorse_b200_cf *cf = ev->cf;
    gorse_b200_ctx *c = cf->ctx;
    const bool multi = c->world > 1;
    const int32_t U = ev->U;
    const int64_t nc = ev->nc;
    out[0] = out[1] = out[2] = 0.f;
    if (nc == 0 && !multi) { out[0] = out[1] = out[2] = NAN; return GORSE_B200_OK; }  // 0 * (1/0), like the reference
    ScopedDevice sd(c->device);
    cudaStream_t s = c->stream;
    cudaError_t e = cudaSuccess;
    if (nc > 0) {
        int threads = 256;
        int64_t work = cf->d % 16 == 0 ? nc * 4 : nc;
        int blocks = (int)std::max<int64_t>(1, std::min<int64_t>((work + threads - 1) / threads, (int64_t)c->sm_count * 16));
        eval_score_kernel<<<blocks, threads, 0, s>>>(P, Q, cf->d, cf->u_lo, ev->cand_user.p, ev->cand_item.p, nc, ev->score.p);
        c->launches++;
        eval_rank_kernel<<<(U + 127) / 128, 128, 0, s>>>(ev->cand_off.p, ev->cand_item.p, ev->score.p, ev->test_off.p, ev->test_items.p, U, ev->topk,
                                                         ev->inv.p, ev->metrics.p);
        c->launches++;
        if ((e = cudaGetLastError()) != cudaSuccess) { set_error("evaluate launch: %s", cudaGetErrorString(e)); return GORSE_B200_ERR_CUDA; }
        if ((e = cudaMemcpyAsync(ev->h_metrics.data(), ev->metrics.p, sizeof(float) * 4 * (size_t)U, cudaMemcpyDeviceToHost, s)) != cudaSuccess ||
            (e = cudaStreamSynchronize(s)) != cudaSuccess) {
            set_error("evaluate: %s", cudaGetErrorString(e));
            return GORSE_B200_ERR_CUDA;
        }
    }
    // evaluator.go:63-71 with one worker: fp32 sums in user order, then * (1/count)
    volatile float sum0 = 0.f, sum1 = 0.f, sum2 = 0.f, count = 0.f;
    if (nc > 0)
        for (int32_t u = 0; u < U; u++) {
            const float *m = ev->h_metrics.data() + 4 * (size_t)u;
            if (m[3] != 0.f) {
                count = count + 1.0f;
                sum0 = sum0 + m[0]; sum1 = sum1 + m[1]; sum2 = sum2 + m[2];
            }
        }
    if (multi) {
        // sum of the per-rank partial sums (the reference with Jobs = world: one partial sum per worker, evaluator.go:63-71)
        float h[4] = {sum0, sum1, sum2, count};
        DevBuf<float> dsum;
        GB_NCCL_API(nc_api);
        GB_TRY(dsum.alloc(4));
        e = cudaMemcpyAsync(dsum.p, h, sizeof(h), cudaMemcpyHostToDevice, s);
        ncclResult_t r = e == cudaSuccess ? nc_api->AllReduce(dsum.p, dsum.p, 4, ncclFloat32, ncclSum, c->comm, s) : ncclSuccess;
        if (e == cudaSuccess && r == ncclSuccess) e = cudaMemcpyAsync(h, dsum.p, sizeof(h), cudaMemcpyDeviceToHost, s);
        if (e == cudaSuccess && r == ncclSuccess) e = cudaStreamSynchronize(s);
        dsum.free();
        if (r != ncclSuccess) { set_error("evaluate: ncclAllReduce -> %s", nc_api->GetErrorString(r)); return GORSE_B200_ERR_NCCL; }
        if (e != cudaSuccess) { set_error("evaluate: %s", cudaGetErrorString(e)); return GORSE_B200_ERR_CUDA; }
        sum0 = h[0]; sum1 = h[1]; sum2 = h[2]; count = h[3];
    }
    volatile float inv = 1.0f / count;
    out[0] = sum0 * inv; out[1] = sum1 * inv; out[2] = sum2 * inv;
    return GORSE_B200_OK;
}

extern "C" {

int32_t gorse_b200_eval_destroy(gorse_b200_eval *ev)
{
    if (!ev) return GORSE_B200_OK;
    ScopedDevice sd(ev->cf->ctx->device);
    cudaStreamSynchronize(ev->cf->ctx->stream);
    ev->test_off.free(); ev->neg_off.free(); ev->cand_off.free();
    ev->test_items.free(); ev->neg_items.free(); ev->cand_user.free(); ev->cand_item.free();
    ev->score.free(); ev->inv.free(); ev->metrics.free();
    delete ev;
    return GORSE_B200_OK;
}

int32_t gorse_b200_eval_create(gorse_b200_cf *cf, const int64_t *test_off, const int32_t *test_items,
                               const int64_t *neg_off, const int32_t *neg_items, int32_t n_candidates, uint64_t seed,
                               int32_t topk, gorse_b200_eval **out)
{
    GB_CHECK_ARG(cf != nullptr && out != nullptr, "NULL cf/out");
    *out = nullptr;
    GB_CHECK_ARG(test_off != nullptr, "test_off is NULL");
    GB_CHECK_ARG(topk >= 1 && topk <= GB_EVAL_MAX_TOPK, "topk %d out of range [1, %d]", topk, GB_EVAL_MAX_TOPK);
    GB_CHECK_ARG(neg_off != nullptr || n_candidates >= 0, "negative n_candidates");
    // in a distributed context every rank passes the rows of ITS users [u_lo, u_hi)
    const int32_t U = cf->u_hi - cf->u_lo;
    const int64_t t0 = test_off[0], n_test = test_off[U] - t0;
    GB_CHECK_ARG(n_test == 0 || test_items != nullptr, "test_items is NULL");
    for (int32_t u = 0; u < U; u++) GB_CHECK_ARG(test_off[u + 1] >= test_off[u], "test_off not non-decreasing at user %d", u);
    for (int64_t a = 0; a < n_test; a++)
        GB_CHECK_ARG(test_items[a] >= 0 && test_items[a] < cf->n_items, "test item %d out of range", test_items[a]);
    int64_t n_neg = 0;
    if (neg_off) {
        n_neg = neg_off[U] - neg_off[0];
        GB_CHECK_ARG(n_neg == 0 || neg_items != nullptr, "neg_items is NULL");
        for (int32_t u = 0; u < U; u++) GB_CHECK_ARG(neg_off[u + 1] >= neg_off[u], "neg_off not non-decreasing at user %d", u);
        for (int64_t a = 0; a < n_neg; a++)
            GB_CHECK_ARG(neg_items[a] >= 0 && neg_items[a] < cf->n_items, "negative item %d out of range", neg_items[a]);
    }
    ScopedDevice sd(cf->ctx->device);
    gorse_b200_ctx *c = cf->ctx;
    cudaStream_t s = c->stream;
    gorse_b200_eval *ev = new (std::nothrow) gorse_b200_eval();
    if (!ev) { set_error("host allocation failed"); return GORSE_B200_ERR_OOM; }
    ev->cf = cf; ev->U = U; ev->topk = topk;
    int32_t st = GORSE_B200_OK;
    auto fail = [&](int32_t code) { gorse_b200_eval_destroy(ev); return code; };
    auto cuda_fail = [&](cudaError_t e) { set_error("eval_create: %s", cudaGetErrorString(e)); return fail(GORSE_B200_ERR_CUDA); };
    cudaError_t e = cudaSuccess;
    std::vector<int64_t> toff((size_t)U + 1), noff((size_t)U + 1, 0), coff((size_t)U + 1, 0);
    for (int32_t u = 0; u <= U; u++) toff[(size_t)u] = test_off[u] - t0;   // rebase (a slice of a global CSR is fine)
    if ((st = ev->test_off.alloc((size_t)U + 1)) || (st = ev->test_items.alloc((size_t)n_test)) || (st = ev->neg_off.alloc((size_t)U + 1)) ||
        (st = ev->cand_off.alloc((size_t)U + 1)) || (st = ev->inv.alloc((size_t)topk)) || (st = ev->metrics.alloc((size_t)4 * std::max(U, 1))))
        return fail(st);
    if ((e = cudaMemcpyAsync(ev->test_off.p, toff.data(), sizeof(int64_t) * ((size_t)U + 1), cudaMemcpyHostToDevice, s)) != cudaSuccess) return cuda_fail(e);
    if (n_test && (e = cudaMemcpyAsync(ev->test_items.p, test_items, sizeof(int32_t) * (size_t)n_test, cudaMemcpyHostToDevice, s)) != cudaSuccess) return cuda_fail(e);
    const int ub = std::max(1, (U + 127) / 128);
    if (neg_off) {
        for (int32_t u = 0; u <= U; u++) noff[(size_t)u] = neg_off[u] - neg_off[0];
        if ((st = ev->neg_items.alloc((size_t)n_neg))) return fail(st);
        if (n_neg && (e = cudaMemcpyAsync(ev->neg_items.p, neg_items, sizeof(int32_t) * (size_t)n_neg, cudaMemcpyHostToDevice, s)) != cudaSuccess) return cuda_fail(e);
    } else if (U > 0) {
        // sample on the device against the training rows that already live there
        DevBuf<int32_t> cnt;
        if ((st = cnt.alloc((size_t)U))) return fail(st);
        const uint64_t base = eval_negatives_base(seed);
        eval_negatives_kernel<<<ub, 128, 0, s>>>(cf->user_off.p, cf->user_items.p, ev->test_off.p, ev->test_items.p, U, cf->u_lo, cf->n_items,
                                                 n_candidates, base, true, cnt.p, nullptr, nullptr);
        c->launches++;
        std::vector<int32_t> hc((size_t)U);
        if ((e = cudaMemcpyAsync(hc.data(), cnt.p, sizeof(int32_t) * (size_t)U, cudaMemcpyDeviceToHost, s)) != cudaSuccess ||
            (e = cudaStreamSynchronize(s)) != cudaSuccess) { cnt.free(); return cuda_fail(e); }
        cnt.free();
        for (int32_t u = 0; u < U; u++) noff[(size_t)u + 1] = noff[(size_t)u] + hc[(size_t)u];
        n_neg = noff[(size_t)U];
        if ((st = ev->neg_items.alloc((size_t)n_neg))) return fail(st);
        if ((e = cudaMemcpyAsync(ev->neg_off.p, noff.data(), sizeof(int64_t) * ((size_t)U + 1), cudaMemcpyHostToDevice, s)) != cudaSuccess) return cuda_fail(e);
        eval_negatives_kernel<<<ub, 128, 0, s>>>(cf->user_off.p, cf->user_items.p, ev->test_off.p, ev->test_items.p, U, cf->u_lo, cf->n_items,
                                                 n_candidates, base, false, nullptr, ev->neg_off.p, ev->neg_items.p);
        c->launches++;
    }
    ev->n_neg = n_neg;
    ev->h_neg_off = noff;
    if ((e = cudaMemcpyAsync(ev->neg_off.p, noff.data(), sizeof(int64_t) * ((size_t)U + 1), cudaMemcpyHostToDevice, s)) != cudaSuccess) return cuda_fail(e);
    for (int32_t u = 0; u < U; u++) {
        const int64_t nt = toff[(size_t)u + 1] - toff[(size_t)u], nn = noff[(size_t)u + 1] - noff[(size_t)u];
        coff[(size_t)u + 1] = coff[(size_t)u] + (nt > 0 ? nt + nn : 0);
    }
    ev->nc = coff[(size_t)U];
    if ((st = ev->cand_user.alloc((size_t)ev->nc)) || (st = ev->cand_item.alloc((size_t)ev->nc)) || (st = ev->score.alloc((size_t)ev->nc))) return fail(st);
    if ((e = cudaMemcpyAsync(ev->cand_off.p, coff.data(), sizeof(int64_t) * ((size_t)U + 1), cudaMemcpyHostToDevice, s)) != cudaSuccess) return cuda_fail(e);
    if (ev->nc > 0) {
        eval_candidates_kernel<<<ub, 128, 0, s>>>(ev->test_off.p, ev->test_items.p, ev->neg_off.p, ev->neg_items.p, U, cf->u_lo, ev->cand_off.p,
                                                  ev->cand_user.p, ev->cand_item.p);
        c->launches++;
    }
    std::vector<float> inv_log2((size_t)topk);
    for (int i = 0; i < topk; i++) inv_log2[i] = 1.0f / log2_math32((float)i + 2.0f);
    if ((e = cudaMemcpyAsync(ev->inv.p, inv_log2.data(), sizeof(float) * (size_t)topk, cudaMemcpyHostToDevice, s)) != cudaSuccess) return cuda_fail(e);
    if ((e = cudaGetLastError()) != cudaSuccess || (e = cudaStreamSynchronize(s)) != cudaSuccess) return cuda_fail(e);   // host staging dies here
    ev->h_metrics.resize((size_t)4 * U);
    *out = ev;
    return GORSE_B200_OK;
}

int32_t gorse_b200_eval_negatives(gorse_b200_eval *ev, int64_t *neg_off_out, int32_t *neg_items_out)
{
    GB_CHECK_ARG(ev != nullptr && neg_off_out != nullptr, "NULL eval/neg_off_out");
    for (int32_t u = 0; u <= ev->U; u++) neg_off_out[u] = ev->h_neg_off[(size_t)u];
    if (neg_items_out && ev->n_neg) {
        ScopedDevice sd(ev->cf->ctx->device);
        GB_CUDA(cudaMemcpyAsync(neg_items_out, ev->neg_items.p, sizeof(int32_t) * (size_t)ev->n_neg, cudaMemcpyDeviceToHost, ev->cf->ctx->stream));
        GB_CUDA(cudaStreamSynchronize(ev->cf->ctx->stream));
    }
    return GORSE_B200_OK;
}

int32_t gorse_b200_eval_run(gorse_b200_eval *ev, float *out)
{
    GB_CHECK_ARG(ev != nullptr && out != nullptr, "NULL eval/out");
    return eval_run_tables(ev, ev->cf->P.p, ev->cf->Q.p, out);
}

int32_t gorse_b200_cf_evaluate(gorse_b200_cf *cf, const int64_t *test_off, const int32_t *test_items,
                               const int64_t *neg_off, const int32_t *neg_items, int32_t topk, float *out)
{
    GB_CHECK_ARG(cf != nullptr && out != nullptr, "NULL cf/out");
    GB_CHECK_ARG(test_off != nullptr && neg_off != nullptr, "NULL offsets");
    gorse_b200_eval *ev = nullptr;
    GB_TRY(gorse_b200_eval_create(cf, test_off, test_items, neg_off, neg_items, 0, 0, topk, &ev));
    const int32_t st = gorse_b200_eval_run(ev, out);
    gorse_b200_eval_destroy(ev);
    return st;
}

}  // extern "C"
