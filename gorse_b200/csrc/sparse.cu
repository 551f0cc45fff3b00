// sparse.cu -- brute-force search over SPARSE vectors with the Dot metric: what logics.item_to_item / user_to_user of the
// types "tags", "users" and "auto" ask their vector store for (storage/vectors/xvec.go:244-248 flat sparse index, :405
// query; vectors built by appendSparseVector, logics/vector_writer.go:200-209).  SURVEY 8f-1, the row after the dense index.
//
// First hardware run in round 2 (tests/test_sparse_gpu.py green).  The arithmetic it must reproduce: merge-join dot of two
// sparse vectors summed in ascending index order, fp32, multiply and add unfused (the test suite's CPU restatement).
//
// Layout: the vectors as CSR (row -> ascending feature indices + values) and the same entries as CSC (feature -> ascending
// rows + values, the posting lists).  The stored rows are cut into tiles of TILE rows; a work item is one (query, tile) pair and
// one CTA accumulates it in a shared-memory float per row of the tile, by one of two paths chosen per work item:
//   push  for every feature f of the query in ascending order, add v_qf * v_cf into acc[c] for the postings c of f inside the
//         tile (found by binary search: postings ascend by row); the threads take distinct rows and a barrier separates the
//         features.  Cost: one CTA round per feature with postings in the tile, plus the postings / threads.
//   pull  one warp per row c of the tile merge-joins the row's CSR against the query's features (a binary search per entry);
//         the matched products are added in entry order by a shuffle chain.  Cost: the tile's entries / 32 plus its rows,
//         spread over the warps, times the search depth.
// Either way every candidate's dot is summed in ascending feature order, fp32, multiply and add unfused -- the merge-join order
// of the oracle -- so both paths give the same bits.  Each work item keeps its tile's best k positive dots (order: dot
// descending, then row ascending) under the allow mask and self-exclusion; a merge kernel folds each query's tile lists into
// its answer.  Rows with dot <= 0 are never returned (the reference drops them right after the query,
// logics/item_to_item.go:73).  Work items are taken tile-major, so the queries of one tile run together and reuse the tile's
// posting ranges from L2, and a heavy query spreads over as many CTAs as it has tiles.
//
// k > 128 (the wide path): the lists do not stretch that far, so the same work items write each query's score row [n] instead
// (the dot of every candidate, NaN for every other row), and one CTA per query emits the answer in sorted rounds of at most
// 2048 with the dense exact kernel's emission (recall::emit_in_rounds).
#include <algorithm>

#include <cub/cub.cuh>

#include "recall.cuh"
#include "sparse.cuh"

using namespace gb;

namespace {

// (dist, idx) ordering of topk.cu: ascending distance (= descending dot), then ascending index
__device__ __forceinline__ bool before(float da, int32_t ia, float db, int32_t ib) { return da < db || (da == db && ia < ib); }

// topk.cu list_insert_warp: sorted insertion done by the whole warp; all arguments warp-uniform, k <= 128
__device__ __forceinline__ void list_insert_warp(float *ld, int32_t *li, int &len, int k, float dv, int32_t iv, int lane)
{
    if (len == k && !before(dv, iv, ld[k - 1], li[k - 1])) return;
    const int n = len;
    float od[4];
    int32_t oi[4];
    int pos = 0;
#pragma unroll
    for (int r = 0; r < 4; r++) {
        const int e = lane + 32 * r;
        const bool has = e < n;
        od[r] = has ? ld[e] : 0.f;
        oi[r] = has ? li[e] : 0;
        pos += __popc(__ballot_sync(0xffffffffu, has && before(od[r], oi[r], dv, iv)));
    }
    __syncwarp();
#pragma unroll
    for (int r = 0; r < 4; r++) {
        const int e = lane + 32 * r;
        if (e < n && e >= pos && e + 1 < k) { ld[e + 1] = od[r]; li[e + 1] = oi[r]; }
    }
    if (lane == 0) { ld[pos] = dv; li[pos] = iv; }
    if (len < k) len++;
    __syncwarp();
}

// merge two sorted lists (a: na, b: nb entries, all rows distinct) into the first min(k, na + nb) of out; one warp
__device__ __forceinline__ int count_before(const float *d, const int32_t *id, int n, float dv, int32_t iv)
{
    int lo = 0, hi = n;
    while (lo < hi) {
        const int m = (lo + hi) >> 1;
        if (before(d[m], id[m], dv, iv)) lo = m + 1;
        else hi = m;
    }
    return lo;
}
__device__ __forceinline__ int merge_warp(const float *ad, const int32_t *ai, int na, const float *bd, const int32_t *bi, int nb, float *od,
                                          int32_t *oi, int k, int lane)
{
    for (int e = lane; e < na; e += 32) {
        const int r = e + count_before(bd, bi, nb, ad[e], ai[e]);
        if (r < k) { od[r] = ad[e]; oi[r] = ai[e]; }
    }
    for (int e = lane; e < nb; e += 32) {
        const int r = e + count_before(ad, ai, na, bd[e], bi[e]);
        if (r < k) { od[r] = bd[e]; oi[r] = bi[e]; }
    }
    __syncwarp();
    return min(k, na + nb);
}

constexpr int TILE = 8192;              // rows per tile: a 32 KB accumulator, four CTAs per SM
constexpr int NT = 256, NW = NT / 32;   // threads / warps of a work item's CTA; NT features per batch of posting ranges
constexpr int MERGE_WARPS = 4;
constexpr int LIST_K = 128;            // the largest k the warps' lists hold; larger k take the wide path
constexpr int EMIT_THREADS = 256;

struct Stored {   // the index's device layouts
    const int64_t *off; const uint32_t *ind; const float *val;    // CSR
    const int64_t *foff; const int32_t *frow; const float *fval;  // CSC
    int64_t n; uint32_t n_features;
};
// the queries of one search: rows of an external device CSR (q_off != nullptr; vecdb.cu: QueryVectors passes the vector, not its
// id), the stored rows rows[q] (a device list, item_to_item.cu), or the stored rows q0 + q; stored query rows never return themselves
struct Queries {
    const int64_t *q_off; const uint32_t *q_ind; const float *q_val;
    const int64_t *rows; int64_t q0;
};

__device__ __forceinline__ int64_t lower_row(const int32_t *frow, int64_t a, int64_t b, int64_t x)
{
    while (a < b) {
        const int64_t m = (a + b) >> 1;
        if (frow[m] < x) a = m + 1;
        else b = m;
    }
    return a;
}

__device__ __forceinline__ int64_t block_sum(int64_t v, int64_t *red)
{
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    int64_t s = 0;
#pragma unroll
    for (int w = 0; w < NW; w++) s += red[w];
    __syncthreads();
    return s;
}

// one CTA per work item at a time, work items w = t * nqc + q (tile-major) taken from *next; paths[0] / [1] count the push /
// pull work items.  The list instance (k <= 128) writes the tile list of w to tl_dot / tl_idx [w * k ...] (negated dots, best
// first) and tl_cnt[w].  The wide instance writes the tile's segment of the query's score row sc[(q - qc0) * n ...]: the dot
// of every candidate (positive, allowed, not the query itself), NaN for every other row; it adds the candidates to have[q - qc0].
template <bool WIDE>
__global__ void __launch_bounds__(NT, 4)
sparse_tile_kernel(Stored S, Queries Q, int64_t qc0, int64_t nqc, int ntiles, int k, const uint8_t *allow, unsigned long long *next,
                   float *tl_dot, int32_t *tl_idx, int32_t *tl_cnt, unsigned long long *paths, float *sc, int32_t *have)
{
    extern __shared__ __align__(16) unsigned char sm_raw[];
    float *acc = reinterpret_cast<float *>(sm_raw);                        // [TILE], zero between work items
    uint32_t *bits = reinterpret_cast<uint32_t *>(acc + TILE);              // [TILE / 32] rows the push touched, zero between
    int64_t *r_lo = reinterpret_cast<int64_t *>(bits + TILE / 32);          // [NT] a batch of posting ranges and query values
    int64_t *r_hi = r_lo + NT;
    float *r_v = reinterpret_cast<float *>(r_hi + NT);
    float *ld = r_v + NT;                                                    // [2][NW][k] the warps' lists, two buffers (list instance)
    int32_t *li = reinterpret_cast<int32_t *>(ld + 2 * NW * k);
    __shared__ int64_t red[NW];
    __shared__ int lens[2][NW];
    __shared__ unsigned long long item;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    for (int i = tid; i < TILE; i += NT) acc[i] = 0.f;
    for (int i = tid; i < TILE / 32; i += NT) bits[i] = 0u;
    const unsigned long long total = (unsigned long long)nqc * ntiles;
    for (;;) {
        if (tid == 0) item = atomicAdd(next, 1ull);
        __syncthreads();
        const unsigned long long w = item;
        if (w >= total) return;
        const int64_t t = (int64_t)(w / nqc), q = qc0 + (int64_t)(w % nqc);
        const int64_t row = Q.q_off ? -1 : Q.rows ? Q.rows[q] : Q.q0 + q;
        const int64_t tb = Q.q_off ? Q.q_off[q] : S.off[row], te = Q.q_off ? Q.q_off[q + 1] : S.off[row + 1];
        const uint32_t *qi = Q.q_off ? Q.q_ind : S.ind;
        const float *qv = Q.q_off ? Q.q_val : S.val;
        const int64_t c0 = t * TILE, c1 = min(S.n, c0 + TILE);

        // the paths' costs in CTA rounds; the push's is counted until it passes the pull's
        int depth = 1;
        while ((1ll << depth) <= te - tb) depth++;
        const int64_t pull_cost = ((S.off[c1] - S.off[c0]) / 32 + (c1 - c0) + NW - 1) / NW * (depth + 1);
        int64_t push_cost = 0;
        for (int64_t b = tb; b < te && push_cost <= pull_cost; b += NT) {
            int64_t my = 0;
            if (b + tid < te) {
                const uint32_t f = qi[b + tid];
                if (f < S.n_features) {
                    const int64_t lo = lower_row(S.frow, S.foff[f], S.foff[f + 1], c0), hi = lower_row(S.frow, lo, S.foff[f + 1], c1);
                    if (hi > lo) my = 1 + (hi - lo + NT - 1) / NT;
                }
            }
            push_cost += block_sum(my, red);
        }
        float *wd = ld + wid * k;
        int32_t *wi = li + wid * k;
        int len = 0;   // this warp's list, warp-uniform
        float *out = sc + (q - qc0) * S.n;   // the wide instance's score row
        int64_t found = 0;                   // and this thread's candidates in it
        const bool pull = push_cost > pull_cost;
        if (push_cost == 0) {
            // the query shares no feature with the tile: nothing to add
        } else if (!pull) {
            for (int64_t b = tb; b < te; b += NT) {
                int64_t lo = 0, hi = 0;
                float v = 0.f;
                if (b + tid < te) {
                    const uint32_t f = qi[b + tid];
                    v = qv[b + tid];
                    if (f < S.n_features) {   // a feature no stored vector has adds nothing
                        lo = lower_row(S.frow, S.foff[f], S.foff[f + 1], c0);
                        hi = lower_row(S.frow, lo, S.foff[f + 1], c1);
                    }
                }
                r_lo[tid] = lo; r_hi[tid] = hi; r_v[tid] = v;
                __syncthreads();
                const int nb = (int)min((int64_t)NT, te - b);
                for (int x = 0; x < nb; x++) {
                    const int64_t plo = r_lo[x], phi = r_hi[x];
                    if (plo == phi) continue;   // block-uniform
                    const float fv = r_v[x];
                    for (int64_t p = plo + tid; p < phi; p += NT) {
                        const int c = S.frow[p] - (int)c0;
                        acc[c] = acc[c] + fv * S.fval[p];   // unfused multiply and add, like the oracle (-fmad=false)
                        if (!WIDE) atomicOr(&bits[c >> 5], 1u << (c & 31));
                    }
                    __syncthreads();   // the next feature adds after this one: each sum in ascending feature order
                }
                __syncthreads();
            }
            // thread tid owns bitmap word tid (TILE / 32 == NT): its touched rows, read and cleared
            uint32_t m = WIDE ? 0u : bits[tid];
            if (!WIDE) bits[tid] = 0u;
            while (__any_sync(0xffffffffu, m != 0u)) {
                float x = 0.f;
                int32_t c = -1;
                bool cand = false;
                if (m) {
                    const int i = tid * 32 + __ffs(m) - 1;
                    m &= m - 1;
                    x = acc[i];
                    acc[i] = 0.f;
                    c = (int32_t)(c0 + i);
                    cand = x > 0.f && c != row && (allow == nullptr || allow[c] != 0);
                }
                cand = cand && (len < k || before(-x, c, wd[k - 1], wi[k - 1]));
                unsigned bal = __ballot_sync(0xffffffffu, cand);
                while (bal) {
                    const int s = __ffs(bal) - 1;
                    bal &= bal - 1;
                    const float dd = __shfl_sync(0xffffffffu, -x, s);
                    const int32_t cc = __shfl_sync(0xffffffffu, c, s);
                    list_insert_warp(wd, wi, len, k, dd, cc, lane);
                }
            }
        } else {
            for (int64_t r = c0 + wid; r < c1; r += NW) {
                const int64_t a = S.off[r], e = S.off[r + 1];
                float s = 0.f;
                int64_t lo = tb;   // the query's features below lo are below every remaining entry of the row
                for (int64_t base = a; base < e && lo < te; base += 32) {
                    const int64_t p = base + lane;
                    float prod = 0.f;
                    bool hit = false;
                    int64_t pos = te;
                    if (p < e) {
                        const uint32_t g = S.ind[p];
                        int64_t x = lo, y = te;
                        while (x < y) {
                            const int64_t mid = (x + y) >> 1;
                            if (qi[mid] < g) x = mid + 1;
                            else y = mid;
                        }
                        pos = x;
                        if (x < te && qi[x] == g) { hit = true; prod = qv[x] * S.val[p]; }
                    }
                    unsigned hm = __ballot_sync(0xffffffffu, hit);
                    while (hm) {   // in entry order = ascending feature order
                        const int src = __ffs(hm) - 1;
                        hm &= hm - 1;
                        s = s + __shfl_sync(0xffffffffu, prod, src);
                    }
                    lo = __shfl_sync(0xffffffffu, pos, 31);
                }
                const bool cand = s > 0.f && r != row && (allow == nullptr || allow[r] != 0);
                if (WIDE) {
                    if (lane == 0) { out[r] = cand ? s : __int_as_float(0x7fffffff); found += cand; }
                } else if (cand && (len < k || before(-s, (int32_t)r, wd[k - 1], wi[k - 1]))) {
                    list_insert_warp(wd, wi, len, k, -s, (int32_t)r, lane);
                }
            }
        }
        if constexpr (WIDE) {
            if (!pull)   // the push (or no feature in common) left the tile's dots in acc: every row of the tile, acc cleared
                for (int i = tid; i < c1 - c0; i += NT) {
                    const float x = acc[i];
                    acc[i] = 0.f;
                    const int64_t c = c0 + i;
                    const bool cand = x > 0.f && c != row && (allow == nullptr || allow[c] != 0);
                    out[c] = cand ? x : __int_as_float(0x7fffffff);
                    found += cand;
                }
            found = block_sum(found, red);
            if (tid == 0) {
                atomicAdd(&have[q - qc0], (int32_t)found);
                if (push_cost) atomicAdd(&paths[pull], 1ull);
            }
            __syncthreads();   // acc and `item` are reused by the next work item
            continue;
        }
        // the warps' lists pairwise into one: NW -> NW / 2 -> ... -> 1, alternating buffers
        if (lane == 0) lens[0][wid] = len;
        __syncthreads();
        int src = 0, nl = NW;
        for (; nl > 1; nl >>= 1, src ^= 1) {
            if (wid < nl / 2) {
                const float *sd = ld + (size_t)src * NW * k;
                const int32_t *si = li + (size_t)src * NW * k;
                const int n = merge_warp(sd + 2 * wid * k, si + 2 * wid * k, lens[src][2 * wid], sd + (2 * wid + 1) * k, si + (2 * wid + 1) * k,
                                         lens[src][2 * wid + 1], ld + (size_t)(src ^ 1) * NW * k + wid * k,
                                         li + (size_t)(src ^ 1) * NW * k + wid * k, k, lane);
                if (lane == 0) lens[src ^ 1][wid] = n;
            }
            __syncthreads();
        }
        const int n = lens[src][0];
        for (int e = tid; e < n; e += NT) {
            tl_dot[w * k + e] = ld[(size_t)src * NW * k + e];
            tl_idx[w * k + e] = li[(size_t)src * NW * k + e];
        }
        if (tid == 0) {
            tl_cnt[w] = n;
            if (push_cost) atomicAdd(&paths[pull], 1ull);
        }
        __syncthreads();   // lens, the lists and `item` are reused by the next work item
    }
}

// one warp per query of the chunk: fold its tile lists into the answer out_*[(qc0 + q) * k ...], padded with -1 / 0
__global__ void __launch_bounds__(32 * MERGE_WARPS)
sparse_merge_kernel(int64_t qc0, int64_t nqc, int ntiles, int k, const float *tl_dot, const int32_t *tl_idx, const int32_t *tl_cnt,
                    int32_t *out_idx, float *out_dot, int32_t *out_cnt)
{
    extern __shared__ __align__(16) unsigned char sm_raw[];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    float *bd = reinterpret_cast<float *>(sm_raw) + (size_t)wid * 3 * k;   // [3][k]: two running lists and the tile list
    int32_t *bi = reinterpret_cast<int32_t *>(reinterpret_cast<float *>(sm_raw) + (size_t)MERGE_WARPS * 3 * k) + (size_t)wid * 3 * k;
    const int64_t q = (int64_t)blockIdx.x * MERGE_WARPS + wid;
    if (q >= nqc) return;
    int len = 0, cur = 0;
    for (int t = 0; t < ntiles; t++) {
        const int64_t w = (int64_t)t * nqc + q;
        const int nb = tl_cnt[w];
        if (nb == 0) continue;
        if (len == k && !before(tl_dot[w * k], tl_idx[w * k], bd[cur * k + k - 1], bi[cur * k + k - 1])) continue;
        float *td = bd + 2 * k;
        int32_t *ti = bi + 2 * k;
        for (int e = lane; e < nb; e += 32) { td[e] = tl_dot[w * k + e]; ti[e] = tl_idx[w * k + e]; }
        __syncwarp();
        len = merge_warp(bd + cur * k, bi + cur * k, len, td, ti, nb, bd + (cur ^ 1) * k, bi + (cur ^ 1) * k, k, lane);
        cur ^= 1;
    }
    const int64_t o = (qc0 + q) * k;
    for (int e = lane; e < k; e += 32) {
        const bool has = e < len;
        out_idx[o + e] = has ? bi[cur * k + e] : -1;
        out_dot[o + e] = has ? -bd[cur * k + e] : 0.f;
    }
    if (lane == 0) out_cnt[qc0 + q] = len;
}

// the wide path's answers: one CTA per query of the chunk emits the first min(k, have) entries of its score row in sorted
// rounds (recall::emit_in_rounds, the exact kernel's emission) into out_*[(qc0 + q) * k ...], padded with -1 / 0; out_cnt holds
// the chunk's candidate counts have[] on entry and the answers' lengths on exit
__global__ void __launch_bounds__(EMIT_THREADS)
sparse_emit_kernel(int64_t qc0, int64_t n, int k, float *sc, int32_t *out_idx, float *out_dot, int32_t *out_cnt)
{
    using namespace recall;
    constexpr int T = EMIT_THREADS;
    extern __shared__ __align__(16) unsigned char sm_raw[];
    uint64_t *s_key = reinterpret_cast<uint64_t *>(sm_raw);         // [SORT_CAP]
    float *s_val = reinterpret_cast<float *>(s_key + SORT_CAP);     // [SORT_CAP]
    int *hist = reinterpret_cast<int *>(s_val + SORT_CAP);          // [256]
    int *s_warp = hist + 256;                                       // [32]
    int *s_bc = s_warp + 32;                                        // [4]
    const int64_t q = qc0 + blockIdx.x, o = q * k;
    const int K = min(k, out_cnt[q]);
    __syncthreads();   // every thread has read out_cnt[q] before thread 0 overwrites it
    int written = 0;
    emit_in_rounds<T>(sc + (int64_t)blockIdx.x * n, n, K, s_key, s_val, hist, s_warp, s_bc, [&](int m) {
        for (int i = threadIdx.x; i < m; i += T) {
            out_idx[o + written + i] = (int32_t)(uint32_t)s_key[i];
            out_dot[o + written + i] = s_val[i];
        }
        written += m;
    });
    for (int e = K + threadIdx.x; e < k; e += T) { out_idx[o + e] = -1; out_dot[o + e] = 0.f; }
    if (threadIdx.x == 0) out_cnt[q] = K;
}

// ---- the CSC builder (csc_append): the postings of new rows, numbered above every stored row, go after the stored postings of
// their feature.  A stable radix sort by feature keeps the new postings of one feature in row order.
// pk[p] = (base + r) << 32 | bits(val[p]) for the entries p of row r: a posting's row and value in one sort value; one warp per row
__global__ void csc_pack_kernel(const int64_t *off, int64_t m, const float *val, int64_t base, uint64_t *pk)
{
    const int lane = threadIdx.x & 31;
    const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < m; r += nw)
        for (int64_t p = off[r] + lane; p < off[r + 1]; p += 32) pk[p] = (uint64_t)(base + r) << 32 | __float_as_uint(val[p]);
}
// for f in [0, F_new]: lb[f] = the new postings of features below f (keys: their features, sorted), foff_n[f] = foff[min(f, F_old)] + lb[f]
__global__ void csc_bounds_kernel(const uint32_t *keys, int64_t nnz, const int64_t *foff, uint32_t F_old, uint32_t F_new, int64_t *lb, int64_t *foff_n)
{
    const int64_t st = (int64_t)gridDim.x * blockDim.x;
    for (int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; f <= F_new; f += st) {
        int64_t a = 0, b = nnz;
        while (a < b) {
            const int64_t mid = (a + b) >> 1;
            if (keys[mid] < f) a = mid + 1;
            else b = mid;
        }
        lb[f] = a;
        foff_n[f] = (foff ? foff[min(f, (int64_t)F_old)] : 0) + a;
    }
}
// the stored postings of feature f move up by lb[f]; one warp per feature
__global__ void csc_old_kernel(const int64_t *foff, uint32_t F_old, const int32_t *frow, const float *fval, const int64_t *lb, int32_t *frow_n, float *fval_n)
{
    const int lane = threadIdx.x & 31;
    const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t f = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; f < F_old; f += nw)
        for (int64_t p = foff[f] + lane; p < foff[f + 1]; p += 32) { frow_n[p + lb[f]] = frow[p]; fval_n[p + lb[f]] = fval[p]; }
}
// the new posting s (sorted by feature) after every stored posting of its feature and the new ones before it:
// foff_n[f] + (stored of f) + (s - lb[f]) = foff[f + 1] + s
__global__ void csc_new_kernel(const uint32_t *keys, const uint64_t *pk, int64_t nnz, const int64_t *foff, uint32_t F_old, int32_t *frow_n, float *fval_n)
{
    const int64_t st = (int64_t)gridDim.x * blockDim.x;
    for (int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; s < nnz; s += st) {
        const int64_t to = (foff ? foff[min((int64_t)keys[s] + 1, (int64_t)F_old)] : 0) + s;
        frow_n[to] = (int32_t)(pk[s] >> 32);
        fval_n[to] = __uint_as_float((uint32_t)pk[s]);
    }
}

// the stored CSC (foff[F_old + 1] / frow / fval, nnz_old postings; foff == nullptr: none) with the postings of m new rows
// appended: the device CSR off[m + 1] from 0 / ind / val (nnz entries, every index < F_new), rows base .. base + m - 1, above
// every stored row.  Into foff_n[F_new + 1] / frow_n / fval_n (allocated here; F_new >= F_old), postings ascending by row within
// each feature.  Enqueued on the context's stream; its scratch is released before it returns.
int32_t csc_append(gorse_b200_ctx *c, const int64_t *off, const uint32_t *ind, const float *val, int64_t m, int64_t nnz, int64_t base,
                   const int64_t *foff, const int32_t *frow, const float *fval, uint32_t F_old, int64_t nnz_old, uint32_t F_new,
                   DevBuf<int64_t> &foff_n, DevBuf<int32_t> &frow_n, DevBuf<float> &fval_n)
{
    cudaStream_t s = c->stream;
    DevBuf<uint32_t> keys;
    DevBuf<uint64_t> pk, pk_s;
    DevBuf<int64_t> lb;
    DevBuf<uint8_t> tmp;
    StreamSync sync{s};
    int32_t st;
    if ((st = foff_n.alloc((size_t)F_new + 1)) || (st = frow_n.alloc((size_t)(nnz_old + nnz))) || (st = fval_n.alloc((size_t)(nnz_old + nnz))) ||
        (st = keys.alloc((size_t)nnz)) || (st = pk.alloc((size_t)nnz)) || (st = pk_s.alloc((size_t)nnz)) || (st = lb.alloc((size_t)F_new + 1)))
        return st;
    int end_bit = 1;   // every feature index is below F_new
    while (end_bit < 32 && ((uint64_t)F_new - 1) >> end_bit) end_bit++;
    const unsigned grid = (unsigned)c->sm_count * 8;
    cudaError_t e = cudaSuccess;
    if (nnz) {
        csc_pack_kernel<<<grid, 256, 0, s>>>(off, m, val, base, pk.p);
        c->launches++;
        size_t tmp_bytes = 0;
        e = cudaGetLastError();
        if (e == cudaSuccess) e = cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, ind, keys.p, pk.p, pk_s.p, nnz, 0, end_bit, s);
        if (e == cudaSuccess && (st = tmp.alloc(tmp_bytes))) return st;
        if (e == cudaSuccess) e = cub::DeviceRadixSort::SortPairs(tmp.p, tmp_bytes, ind, keys.p, pk.p, pk_s.p, nnz, 0, end_bit, s);
    }
    if (e == cudaSuccess) {
        csc_bounds_kernel<<<div_up((int64_t)F_new + 1, 256), 256, 0, s>>>(keys.p, nnz, foff, F_old, F_new, lb.p, foff_n.p);
        if (nnz_old) csc_old_kernel<<<grid, 256, 0, s>>>(foff, F_old, frow, fval, lb.p, frow_n.p, fval_n.p);
        if (nnz) csc_new_kernel<<<grid, 256, 0, s>>>(keys.p, pk_s.p, nnz, foff, F_old, frow_n.p, fval_n.p);
        c->launches += 3;
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) { set_error("sparse CSC: %s", cudaGetErrorString(e)); return e == cudaErrorMemoryAllocation ? GORSE_B200_ERR_OOM : GORSE_B200_ERR_CUDA; }
    return GORSE_B200_OK;
}

// the device layouts from the host CSR: the CSR is uploaded and the CSC built from it on the device
int32_t sync_device(gorse_b200_sparse_index *ix)
{
    if (!ix->dirty) return GORSE_B200_OK;
    gorse_b200_ctx *c = ix->ctx;
    const int64_t n = (int64_t)ix->h_off.size() - 1, nnz = (int64_t)ix->h_ind.size();
    GB_TRY(ix->off.alloc((size_t)n + 1));
    GB_TRY(ix->ind.alloc((size_t)nnz));
    GB_TRY(ix->val.alloc((size_t)nnz));
    cudaStream_t s = c->stream;
    GB_CUDA(cudaMemcpyAsync(ix->off.p, ix->h_off.data(), sizeof(int64_t) * ((size_t)n + 1), cudaMemcpyHostToDevice, s));
    if (nnz) {
        GB_CUDA(cudaMemcpyAsync(ix->ind.p, ix->h_ind.data(), sizeof(uint32_t) * (size_t)nnz, cudaMemcpyHostToDevice, s));
        GB_CUDA(cudaMemcpyAsync(ix->val.p, ix->h_val.data(), sizeof(float) * (size_t)nnz, cudaMemcpyHostToDevice, s));
    }
    GB_TRY(csc_append(c, ix->off.p, ix->ind.p, ix->val.p, n, nnz, 0, nullptr, nullptr, nullptr, 0, 0, ix->n_features, ix->foff, ix->frow, ix->fval));
    ix->dirty = false;
    return GORSE_B200_OK;
}

// ---- vectors from id rows (sparse_idf_rows): appendSparseVector of every row on the device.  The rows are merged (row r: its
// A ids, then its B ids), each merged row is sorted by key = part << 32 | (uint32)id, and the kept entries are scanned into place.
struct IdfPart {
    const int64_t *off; const int32_t *ids; const float *idf; int32_t n_idf; uint32_t offset;
};
// key[t] of merged entry t (m_off[n + 1]: the merged offsets), head[t] = 1 for the first entry of a row
__global__ void idf_gather_kernel(IdfPart A, IdfPart B, const int64_t *m_off, int64_t n, int64_t total, uint64_t *key, uint8_t *head)
{
    const int64_t st = (int64_t)gridDim.x * blockDim.x;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += st) {
        int64_t lo = 0, hi = n;   // m_off[lo] <= t < m_off[hi]: at the end, the (non-empty) row lo holds t
        while (hi - lo > 1) {
            const int64_t mid = (lo + hi) >> 1;
            if (m_off[mid] <= t) lo = mid;
            else hi = mid;
        }
        const int64_t j = t - m_off[lo], na = A.off[lo + 1] - A.off[lo];
        key[t] = j < na ? (uint64_t)(uint32_t)A.ids[A.off[lo] + j] : 1ull << 32 | (uint32_t)B.ids[B.off[lo] + j - na];
        head[t] = j == 0;
    }
}
// keep[t] = 1 for a sorted entry that enters its vector: an id in [0, n_idf) whose idf is not <= 0 (a NaN idf enters, and is
// refused by the scatter), not equal to the entry before it in its row; keep[total] = 0
__global__ void idf_keep_kernel(IdfPart A, IdfPart B, const uint64_t *key, const uint8_t *head, int64_t total, int64_t *keep)
{
    const int64_t st = (int64_t)gridDim.x * blockDim.x;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t <= total; t += st) {
        if (t == total) { keep[t] = 0; continue; }
        const uint64_t k = key[t];
        const bool b = k >> 32;
        const int32_t id = (int32_t)(uint32_t)k;
        keep[t] = id >= 0 && id < (b ? B.n_idf : A.n_idf) && !((b ? B.idf : A.idf)[id] <= 0.f) && (head[t] || key[t - 1] != k);
    }
}
// the kept entries to their scanned positions: index offset + id, value (float)sqrt((double)idf[id]).  err bit 1: a NaN value,
// bit 2: an index >= 0x7fffffff (what gorse_b200_sparse_index_add refuses); stat[1] = the largest index
__global__ void idf_scatter_kernel(IdfPart A, IdfPart B, const uint64_t *key, const int64_t *scan, int64_t total, uint32_t *ind, float *val,
                                   unsigned *stat)
{
    const int64_t st = (int64_t)gridDim.x * blockDim.x;
    unsigned err = 0, mx = 0;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += st) {
        const int64_t p = scan[t];
        if (scan[t + 1] == p) continue;
        const uint64_t k = key[t];
        const bool b = k >> 32;
        const int32_t id = (int32_t)(uint32_t)k;
        const uint32_t x = (b ? B.offset : A.offset) + (uint32_t)id;
        const float v = (float)sqrt((double)(b ? B.idf : A.idf)[id]);
        ind[p] = x;
        val[p] = v;
        err |= (v != v ? 1u : 0u) | (x >= 0x7fffffffu ? 2u : 0u);
        mx = max(mx, x);
    }
    err = __reduce_or_sync(0xffffffffu, err);
    mx = __reduce_max_sync(0xffffffffu, mx);
    if ((threadIdx.x & 31) == 0) {
        if (err) atomicOr(&stat[0], err);
        atomicMax(&stat[1], mx);
    }
}
// per row r: out_off[r] = its first entry in the built CSR, out_off[n] = the entries; err bit 4: the row's first B index does not
// exceed its last A index (a_off == m_off without a part B).  Each part's kept indices ascend unless one is >= 0x7fffffff.
__global__ void idf_rows_kernel(const int64_t *a_off, const int64_t *m_off, const int64_t *scan, int64_t n, const uint32_t *ind, int64_t *out_off,
                                unsigned *stat)
{
    const int64_t st = (int64_t)gridDim.x * blockDim.x;
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r <= n; r += st) {
        const int64_t a0 = scan[m_off[r]];
        out_off[r] = a0;
        if (r == n) continue;
        const int64_t ab = scan[m_off[r] + a_off[r + 1] - a_off[r]], b1 = scan[m_off[r + 1]];
        if (a0 < ab && ab < b1 && ind[ab] <= ind[ab - 1]) atomicOr(&stat[0], 4u);
    }
}

// ---- compaction (sparse_compact): `scan` is the exclusive sum of the rows' live flags, row r is live iff scan[r + 1] != scan[r]
// keep[t] = 1 for the CSR entries of live rows, keep[nnz] = 0; one warp per row
__global__ void sparse_row_keep_kernel(const int64_t *off, int64_t n, const int64_t *scan, int64_t *keep)
{
    const int lane = threadIdx.x & 31;
    const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < n; r += nw) {
        const int64_t k = scan[r + 1] != scan[r];
        for (int64_t t = off[r] + lane; t < off[r + 1]; t += 32) keep[t] = k;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) keep[off[n]] = 0;
}
// keep[p] = 1 for the CSC entries whose row is live, keep[nnz] = 0
__global__ void sparse_col_keep_kernel(const int32_t *frow, int64_t nnz, const int64_t *scan, int64_t *keep)
{
    const int64_t st = (int64_t)gridDim.x * blockDim.x;
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p <= nnz; p += st)
        keep[p] = p < nnz && scan[frow[p] + 1] != scan[frow[p]];
}
// entries are grouped by row (by feature), so a list's new offset is the entry scan read at its old one:
// off'[scan[r]] = e_scan[off[r]] for live r and off'[live] = e_scan[nnz]; rows == nullptr: every list is kept, out[i] = e_scan[in[i]]
__global__ void sparse_compact_off_kernel(const int64_t *in, int64_t m, const int64_t *rows, const int64_t *e_scan, int64_t *out)
{
    const int64_t st = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i <= m; i += st) {
        if (!rows) out[i] = e_scan[in[i]];
        else if (i == m) out[rows[m]] = e_scan[in[m]];
        else if (rows[i + 1] != rows[i]) out[rows[i]] = e_scan[in[i]];
    }
}
// the kept entries to their scanned positions; CSC rows are renamed through the row scan (monotone: lists stay ascending)
__global__ void sparse_compact_csr_kernel(const uint32_t *ind, const float *val, int64_t nnz, const int64_t *e_scan, uint32_t *ind_n, float *val_n)
{
    const int64_t st = (int64_t)gridDim.x * blockDim.x;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < nnz; t += st) {
        const int64_t to = e_scan[t];
        if (e_scan[t + 1] != to) { ind_n[to] = ind[t]; val_n[to] = val[t]; }
    }
}
__global__ void sparse_compact_csc_kernel(const int32_t *frow, const float *fval, int64_t nnz, const int64_t *e_scan, const int64_t *scan,
                                          int32_t *frow_n, float *fval_n)
{
    const int64_t st = (int64_t)gridDim.x * blockDim.x;
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < nnz; p += st) {
        const int64_t to = e_scan[p];
        if (e_scan[p + 1] != to) { frow_n[to] = (int32_t)scan[frow[p]]; fval_n[to] = fval[p]; }
    }
}

// the last search's device time into search_ms (every caller synchronises its stream before it returns, so this rarely waits)
void fold_time(gorse_b200_sparse_index *ix)
{
    if (!ix->ev_pending) return;
    float ms = 0.f;
    if (cudaEventSynchronize(ix->ev[1]) == cudaSuccess && cudaEventElapsedTime(&ms, ix->ev[0], ix->ev[1]) == cudaSuccess) ix->search_ms += ms;
    ix->ev_pending = false;
}

}  // namespace

extern "C" {

int32_t gorse_b200_sparse_index_create(gorse_b200_ctx *ctx, gorse_b200_sparse_index **out)
{
    GB_CHECK_ARG(ctx != nullptr && out != nullptr, "NULL argument");
    gorse_b200_sparse_index *ix = new gorse_b200_sparse_index();
    ix->ctx = ctx;
    *out = ix;
    return GORSE_B200_OK;
}

int32_t gorse_b200_sparse_index_destroy(gorse_b200_sparse_index *ix)
{
    if (!ix) return GORSE_B200_OK;
    ScopedDevice sd(ix->ctx->device);
    cudaStreamSynchronize(ix->ctx->stream);
    for (cudaEvent_t e : ix->ev)
        if (e) cudaEventDestroy(e);
    delete ix;
    return GORSE_B200_OK;
}

int32_t gorse_b200_sparse_index_add(gorse_b200_sparse_index *ix, const int64_t *off, const uint32_t *indices, const float *values,
                                    int64_t n, int64_t *count_out)
{
    GB_CHECK_ARG(ix != nullptr, "index is NULL");
    GB_CHECK_ARG(n >= 0, "negative n");
    std::lock_guard<std::mutex> lk(ix->mu);
    if (n > 0) {
        GB_CHECK_ARG(off != nullptr, "off is NULL");
        GB_CHECK_ARG(off[0] == 0, "off[0] must be 0");
        for (int64_t r = 0; r < n; r++) {
            GB_CHECK_ARG(off[r + 1] >= off[r], "offsets must not decrease (row %lld)", (long long)r);
            for (int64_t t = off[r]; t < off[r + 1]; t++) {
                GB_CHECK_ARG(indices != nullptr && values != nullptr, "NULL indices/values");
                GB_CHECK_ARG(t == off[r] || indices[t] > indices[t - 1], "indices of row %lld are not strictly ascending", (long long)r);
                GB_CHECK_ARG(values[t] == values[t], "NaN value in row %lld", (long long)r);
                GB_CHECK_ARG(indices[t] < 0x7fffffffu, "feature index too large");
            }
        }
        if ((int64_t)ix->h_off.size() - 1 + n >= (1ll << 31)) { set_error("more than 2^31 vectors"); return GORSE_B200_ERR_UNSUPPORTED; }
        const int64_t base = ix->h_off.back();
        for (int64_t r = 0; r < n; r++) ix->h_off.push_back(base + off[r + 1]);
        ix->h_ind.insert(ix->h_ind.end(), indices, indices + off[n]);
        ix->h_val.insert(ix->h_val.end(), values, values + off[n]);
        for (int64_t t = 0; t < off[n]; t++) ix->n_features = std::max(ix->n_features, indices[t] + 1);
        ix->dirty = true;
    }
    if (count_out) *count_out = (int64_t)ix->h_off.size() - 1;
    return GORSE_B200_OK;
}

int32_t gorse_b200_sparse_index_len(const gorse_b200_sparse_index *ix, int64_t *count_out)
{
    GB_CHECK_ARG(ix != nullptr && count_out != nullptr, "NULL argument");
    *count_out = (int64_t)ix->h_off.size() - 1;
    return GORSE_B200_OK;
}

int32_t gorse_b200_sparse_index_search_range(gorse_b200_sparse_index *ix, int64_t q0, int64_t q1, int32_t k, int32_t *idx_out,
                                             float *dot_out, int32_t *count_out)
{
    GB_CHECK_ARG(ix != nullptr, "index is NULL");
    GB_CHECK_ARG(k > 0, "k must be positive (got %d)", k);
    std::lock_guard<std::mutex> lk(ix->mu);
    const int64_t n = (int64_t)ix->h_off.size() - 1;
    if (q0 < 0 || q1 < q0 || q1 > n) {
        set_error("index out of range: [%lld, %lld)", (long long)q0, (long long)q1);
        return GORSE_B200_ERR_RANGE;
    }
    const int64_t nq = q1 - q0;
    if (nq == 0) return GORSE_B200_OK;
    GB_CHECK_ARG(idx_out != nullptr && dot_out != nullptr && count_out != nullptr, "NULL output");
    return gb::sparse_search_host(ix, q0, nq, nullptr, nullptr, nullptr, nullptr, k, idx_out, dot_out, count_out);
}

int32_t gorse_b200_sparse_index_stats(gorse_b200_sparse_index *ix, int64_t *push_items, int64_t *pull_items, int64_t *tiles, double *search_ms)
{
    GB_CHECK_ARG(ix != nullptr, "index is NULL");
    std::lock_guard<std::mutex> lk(ix->mu);
    ScopedDevice sd(ix->ctx->device);
    cudaStream_t s = ix->ctx->stream;
    fold_time(ix);
    unsigned long long h[2] = {0, 0};
    if (ix->paths.p) {
        GB_CUDA(cudaMemcpyAsync(h, ix->paths.p, sizeof(h), cudaMemcpyDeviceToHost, s));
        GB_CUDA(cudaMemsetAsync(ix->paths.p, 0, sizeof(h), s));
        GB_CUDA(cudaStreamSynchronize(s));
    }
    if (push_items) *push_items = (int64_t)h[0];
    if (pull_items) *pull_items = (int64_t)h[1];
    if (tiles) *tiles = ix->tiles;
    if (search_ms) *search_ms = ix->search_ms;
    ix->tiles = 0;
    ix->search_ms = 0.0;
    return GORSE_B200_OK;
}

}  // extern "C"

namespace gb {

// the tile lists (k <= 128) or the score rows (k > 128) of a chunk take at most this many bytes; larger searches run in chunks
// of queries, at least one query per chunk
static constexpr int64_t TILE_LIST_BYTES = 512ll << 20;

// the tiled search of nq queries (see the top of this file) into the device buffers d_idx / d_dot [nq x k] and d_cnt[nq],
// enqueued on the context's stream; the index holds at least one vector and its device layouts are current.  k <= 128: the
// work items keep tile lists and a merge kernel folds them.  k > 128 (the wide path): the work items write each query's score
// row [n], and one CTA per query emits its answer in sorted rounds.
static int32_t tiled_search(gorse_b200_sparse_index *ix, const Queries &Q, int64_t nq, const uint8_t *d_allow, int k, int32_t *d_idx,
                            float *d_dot, int32_t *d_cnt)
{
    gorse_b200_ctx *c = ix->ctx;
    cudaStream_t s = c->stream;
    const int64_t n = (int64_t)ix->h_off.size() - 1;
    const int ntiles = div_up(n, TILE);
    const bool wide = k > LIST_K;
    const int64_t per_query = wide ? (int64_t)sizeof(float) * n : (int64_t)ntiles * (8 * k + 4);
    const int64_t nqc_max = std::max<int64_t>(1, std::min<int64_t>(nq, TILE_LIST_BYTES / per_query));
    const int64_t chunks = (nq + nqc_max - 1) / nqc_max;
    const size_t lists = (size_t)nqc_max * ntiles;
    if (wide) {   // the score rows take the tile lists' dot buffer
        if (ix->tl_dot.n < (size_t)nqc_max * n) GB_TRY(ix->tl_dot.alloc((size_t)nqc_max * n));
    } else {
        if (ix->tl_cnt.n < lists) GB_TRY(ix->tl_cnt.alloc(lists));
        if (ix->tl_dot.n < lists * k) GB_TRY(ix->tl_dot.alloc(lists * k));
        if (ix->tl_idx.n < lists * k) GB_TRY(ix->tl_idx.alloc(lists * k));
    }
    if (ix->next.n < (size_t)chunks) GB_TRY(ix->next.alloc((size_t)chunks));
    if (!ix->paths.p) {
        GB_TRY(ix->paths.alloc(2));
        GB_CUDA(cudaMemsetAsync(ix->paths.p, 0, ix->paths.bytes(), s));
    }
    for (cudaEvent_t &e : ix->ev)
        if (!e) GB_CUDA(cudaEventCreate(&e));
    const size_t tile_smem = sizeof(float) * TILE + sizeof(uint32_t) * (TILE / 32) + (2 * sizeof(int64_t) + sizeof(float)) * NT +
                             (wide ? 0 : (size_t)2 * NW * k * (sizeof(float) + sizeof(int32_t)));
    const size_t merge_smem = (size_t)MERGE_WARPS * 3 * k * (sizeof(float) + sizeof(int32_t));
    const size_t emit_smem = (size_t)recall::SORT_CAP * (sizeof(uint64_t) + sizeof(float)) + (256 + 32 + 4) * sizeof(int);
    auto *tile_kernel = wide ? sparse_tile_kernel<true> : sparse_tile_kernel<false>;
    GB_CUDA(cudaFuncSetAttribute(tile_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tile_smem));
    int per_sm = 0;
    GB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, tile_kernel, NT, tile_smem));
    const int64_t grid = (int64_t)c->sm_count * std::max(1, per_sm);
    fold_time(ix);
    GB_CUDA(cudaMemsetAsync(ix->next.p, 0, sizeof(unsigned long long) * (size_t)chunks, s));
    if (wide) GB_CUDA(cudaMemsetAsync(d_cnt, 0, sizeof(int32_t) * (size_t)nq, s));   // the candidate counts
    GB_CUDA(cudaEventRecord(ix->ev[0], s));
    const Stored S{ix->off.p, ix->ind.p, ix->val.p, ix->foff.p, ix->frow.p, ix->fval.p, n, ix->n_features};
    for (int64_t ch = 0; ch < chunks; ch++) {
        const int64_t qc0 = ch * nqc_max, nqc = std::min(nqc_max, nq - qc0);
        tile_kernel<<<(unsigned)std::min<int64_t>(grid, nqc * ntiles), NT, tile_smem, s>>>(
            S, Q, qc0, nqc, ntiles, k, d_allow, ix->next.p + ch, ix->tl_dot.p, ix->tl_idx.p, ix->tl_cnt.p, ix->paths.p, ix->tl_dot.p, d_cnt + qc0);
        GB_LAUNCHED(c);
        if (wide)
            sparse_emit_kernel<<<(unsigned)nqc, EMIT_THREADS, emit_smem, s>>>(qc0, n, k, ix->tl_dot.p, d_idx, d_dot, d_cnt);
        else
            sparse_merge_kernel<<<div_up(nqc, MERGE_WARPS), 32 * MERGE_WARPS, merge_smem, s>>>(qc0, nqc, ntiles, k, ix->tl_dot.p, ix->tl_idx.p,
                                                                                             ix->tl_cnt.p, d_idx, d_dot, d_cnt);
        GB_LAUNCHED(c);
    }
    GB_CUDA(cudaEventRecord(ix->ev[1], s));
    ix->ev_pending = true;
    ix->tiles += ntiles * chunks;
    return GORSE_B200_OK;
}

int32_t sparse_search_rows(gorse_b200_sparse_index *ix, const int64_t *d_rows, int64_t nq, const uint8_t *d_allow, int32_t k, int32_t *d_idx,
                           float *d_dot, int32_t *d_cnt)
{
    GB_TRY(sync_device(ix));
    return tiled_search(ix, Queries{nullptr, nullptr, nullptr, d_rows, 0}, nq, d_allow, k, d_idx, d_dot, d_cnt);
}

// queries = stored rows [q0, q0 + nq) (q_off == nullptr) or nq rows of a HOST CSR (q_off/q_ind/q_val); allow = optional DEVICE
// per-row filter; results to host buffers.  The caller holds ix->mu.
int32_t sparse_search_host(gorse_b200_sparse_index *ix, int64_t q0, int64_t nq, const int64_t *q_off, const uint32_t *q_ind,
                           const float *q_val, const uint8_t *d_allow, int32_t k, int32_t *idx_out, float *dot_out, int32_t *count_out)
{
    const int64_t n = (int64_t)ix->h_off.size() - 1;
    gorse_b200_ctx *c = ix->ctx;
    ScopedDevice sd(c->device);
    GB_TRY(sync_device(ix));
    if (n == 0) {
        for (int64_t q = 0; q < nq; q++) count_out[q] = 0;
        return GORSE_B200_OK;
    }
    const int kc = (int)std::min<int64_t>(k, n);   // no answer is longer than n: the device holds kc columns, the host rows k
    DevBuf<int32_t> d_idx, d_cnt;
    DevBuf<float> d_dot, dq_val;
    DevBuf<int64_t> dq_off;
    DevBuf<uint32_t> dq_ind;
    StreamSync sync{c->stream};
    GB_TRY(d_idx.alloc((size_t)nq * kc));
    GB_TRY(d_dot.alloc((size_t)nq * kc));
    GB_TRY(d_cnt.alloc((size_t)nq));
    cudaError_t e = cudaSuccess;
    if (q_off) {
        const int64_t qn = q_off[nq];
        GB_TRY(dq_off.alloc((size_t)nq + 1));
        GB_TRY(dq_ind.alloc((size_t)qn));
        GB_TRY(dq_val.alloc((size_t)qn));
        e = cudaMemcpyAsync(dq_off.p, q_off, sizeof(int64_t) * ((size_t)nq + 1), cudaMemcpyHostToDevice, c->stream);
        if (e == cudaSuccess && qn) e = cudaMemcpyAsync(dq_ind.p, q_ind, sizeof(uint32_t) * (size_t)qn, cudaMemcpyHostToDevice, c->stream);
        if (e == cudaSuccess && qn) e = cudaMemcpyAsync(dq_val.p, q_val, sizeof(float) * (size_t)qn, cudaMemcpyHostToDevice, c->stream);
        if (e != cudaSuccess) { set_error("sparse search upload: %s", cudaGetErrorString(e)); return GORSE_B200_ERR_CUDA; }
    }
    const Queries Q = q_off ? Queries{dq_off.p, dq_ind.p, dq_val.p, nullptr, 0} : Queries{nullptr, nullptr, nullptr, nullptr, q0};
    GB_TRY(tiled_search(ix, Q, nq, d_allow, kc, d_idx.p, d_dot.p, d_cnt.p));
    if (kc == k) {
        e = cudaMemcpyAsync(idx_out, d_idx.p, sizeof(int32_t) * (size_t)nq * k, cudaMemcpyDeviceToHost, c->stream);
        if (e == cudaSuccess) e = cudaMemcpyAsync(dot_out, d_dot.p, sizeof(float) * (size_t)nq * k, cudaMemcpyDeviceToHost, c->stream);
    } else {
        e = cudaMemcpy2DAsync(idx_out, sizeof(int32_t) * k, d_idx.p, sizeof(int32_t) * kc, sizeof(int32_t) * kc, (size_t)nq, cudaMemcpyDeviceToHost,
                              c->stream);
        if (e == cudaSuccess)
            e = cudaMemcpy2DAsync(dot_out, sizeof(float) * k, d_dot.p, sizeof(float) * kc, sizeof(float) * kc, (size_t)nq, cudaMemcpyDeviceToHost, c->stream);
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(count_out, d_cnt.p, sizeof(int32_t) * (size_t)nq, cudaMemcpyDeviceToHost, c->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
    if (e != cudaSuccess) { set_error("sparse search: %s", cudaGetErrorString(e)); return GORSE_B200_ERR_CUDA; }
    for (int64_t q = 0; q < nq && kc < k; q++) {
        std::fill(idx_out + q * k + kc, idx_out + (q + 1) * k, -1);
        std::fill(dot_out + q * k + kc, dot_out + (q + 1) * k, 0.f);
    }
    return GORSE_B200_OK;
}

int32_t sparse_compact(gorse_b200_sparse_index *ix, const int64_t *scan, int64_t live)
{
    GB_TRY(sync_device(ix));
    gorse_b200_ctx *c = ix->ctx;
    cudaStream_t s = c->stream;
    const int64_t n = (int64_t)ix->h_off.size() - 1, nnz = (int64_t)ix->h_ind.size(), F = ix->n_features;
    int64_t live_nnz = 0;
    std::vector<int64_t> h_off((size_t)live + 1);   // the compacted host CSR
    std::vector<uint32_t> h_ind;
    std::vector<float> h_val;
    DevBuf<int64_t> rs, cs, off_n, foff_n;   // entry keep flags, scanned in place: CSR (rs) and CSC (cs)
    DevBuf<uint8_t> tmp;
    DevBuf<uint32_t> ind_n;
    DevBuf<float> val_n, fval_n;
    DevBuf<int32_t> frow_n;
    StreamSync sync{s};
    GB_TRY(rs.alloc((size_t)nnz + 1));
    GB_TRY(cs.alloc((size_t)nnz + 1));
    const unsigned grid = (unsigned)c->sm_count * 8;
    sparse_row_keep_kernel<<<grid, 256, 0, s>>>(ix->off.p, n, scan, rs.p);
    sparse_col_keep_kernel<<<grid, 256, 0, s>>>(ix->frow.p, nnz, scan, cs.p);
    c->launches += 2;
    size_t tmp_bytes = 0;
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, rs.p, nnz + 1, s);
    if (e != cudaSuccess) { set_error("sparse compact: %s", cudaGetErrorString(e)); return GORSE_B200_ERR_CUDA; }
    GB_TRY(tmp.alloc(tmp_bytes));
    e = cub::DeviceScan::ExclusiveSum(tmp.p, tmp_bytes, rs.p, nnz + 1, s);
    if (e == cudaSuccess) e = cub::DeviceScan::ExclusiveSum(tmp.p, tmp_bytes, cs.p, nnz + 1, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(&live_nnz, rs.p + nnz, sizeof(int64_t), cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) { set_error("sparse compact: %s", cudaGetErrorString(e)); return GORSE_B200_ERR_CUDA; }
    // every buffer of the compacted index, then the host CSR, before any state changes
    GB_TRY(off_n.alloc((size_t)live + 1));
    GB_TRY(foff_n.alloc((size_t)F + 1));
    GB_TRY(ind_n.alloc((size_t)live_nnz));
    GB_TRY(val_n.alloc((size_t)live_nnz));
    GB_TRY(frow_n.alloc((size_t)live_nnz));
    GB_TRY(fval_n.alloc((size_t)live_nnz));
    h_ind.resize((size_t)live_nnz);
    h_val.resize((size_t)live_nnz);
    sparse_compact_off_kernel<<<div_up(n + 1, 256), 256, 0, s>>>(ix->off.p, n, scan, rs.p, off_n.p);
    sparse_compact_off_kernel<<<div_up((int64_t)F + 1, 256), 256, 0, s>>>(ix->foff.p, F, nullptr, cs.p, foff_n.p);
    sparse_compact_csr_kernel<<<grid, 256, 0, s>>>(ix->ind.p, ix->val.p, nnz, rs.p, ind_n.p, val_n.p);
    sparse_compact_csc_kernel<<<grid, 256, 0, s>>>(ix->frow.p, ix->fval.p, nnz, cs.p, scan, frow_n.p, fval_n.p);
    c->launches += 4;
    e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaMemcpyAsync(h_off.data(), off_n.p, sizeof(int64_t) * h_off.size(), cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess && live_nnz) e = cudaMemcpyAsync(h_ind.data(), ind_n.p, sizeof(uint32_t) * h_ind.size(), cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess && live_nnz) e = cudaMemcpyAsync(h_val.data(), val_n.p, sizeof(float) * h_val.size(), cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) { set_error("sparse compact: %s", cudaGetErrorString(e)); return GORSE_B200_ERR_CUDA; }
    ix->off = std::move(off_n); ix->foff = std::move(foff_n); ix->ind = std::move(ind_n);
    ix->val = std::move(val_n); ix->frow = std::move(frow_n); ix->fval = std::move(fval_n);
    ix->h_off.swap(h_off); ix->h_ind.swap(h_ind); ix->h_val.swap(h_val);
    ix->tl_dot.free(); ix->tl_idx.free(); ix->tl_cnt.free(); ix->next.free();   // sized for the old N; the next search allocates them
    return GORSE_B200_OK;
}

int32_t sparse_idf_rows(gorse_b200_ctx *c, int64_t n, const int64_t *a_off, const int32_t *a_ids, const float *a_idf, int32_t a_n_idf,
                        uint32_t a_offset, const int64_t *b_off, const int32_t *b_ids, const float *b_idf, int32_t b_n_idf, uint32_t b_offset,
                        SparseRows &out)
{
    cudaStream_t s = c->stream;
    const int64_t total = a_off[n] + (b_off ? b_off[n] : 0);
    out = SparseRows();
    out.row_off.assign((size_t)n + 1, 0);
    out.off.assign(1, 0);
    if (total == 0) return GORSE_B200_OK;
    if (total > INT32_MAX || n > INT32_MAX) {
        set_error("%lld ids in %lld rows in one call (at most 2^31 - 1 of each)", (long long)total, (long long)n);
        return GORSE_B200_ERR_UNSUPPORTED;
    }
    std::vector<int64_t> m_off;
    if (b_off) {
        m_off.resize((size_t)n + 1);
        for (int64_t r = 0; r <= n; r++) m_off[(size_t)r] = a_off[r] + b_off[r];
    }
    DevBuf<int64_t> d_aoff, d_boff, d_moff, keep, d_out_off;
    DevBuf<int32_t> d_aids, d_bids;
    DevBuf<float> d_aidf, d_bidf;
    unsigned h_stat[2] = {0, 0};
    DevBuf<uint64_t> key, key_s;
    DevBuf<uint8_t> head, tmp;
    DevBuf<unsigned> stat;
    StreamSync sync{s};
    int32_t st;
    if ((st = d_aoff.alloc((size_t)n + 1)) || (st = d_aids.alloc((size_t)a_off[n])) || (st = d_aidf.alloc((size_t)a_n_idf)) ||
        (b_off && ((st = d_boff.alloc((size_t)n + 1)) || (st = d_moff.alloc((size_t)n + 1)) || (st = d_bids.alloc((size_t)b_off[n])) ||
                   (st = d_bidf.alloc((size_t)b_n_idf)))) ||
        (st = key.alloc((size_t)total)) || (st = key_s.alloc((size_t)total)) || (st = head.alloc((size_t)total)) || (st = keep.alloc((size_t)total + 1)) ||
        (st = d_out_off.alloc((size_t)n + 1)) || (st = stat.alloc(2)))
        return st;
    cudaError_t e = cudaMemcpyAsync(d_aoff.p, a_off, sizeof(int64_t) * ((size_t)n + 1), cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess && a_off[n]) e = cudaMemcpyAsync(d_aids.p, a_ids, sizeof(int32_t) * (size_t)a_off[n], cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess && a_n_idf) e = cudaMemcpyAsync(d_aidf.p, a_idf, sizeof(float) * (size_t)a_n_idf, cudaMemcpyHostToDevice, s);
    if (b_off) {
        if (e == cudaSuccess) e = cudaMemcpyAsync(d_boff.p, b_off, sizeof(int64_t) * ((size_t)n + 1), cudaMemcpyHostToDevice, s);
        if (e == cudaSuccess) e = cudaMemcpyAsync(d_moff.p, m_off.data(), sizeof(int64_t) * ((size_t)n + 1), cudaMemcpyHostToDevice, s);
        if (e == cudaSuccess && b_off[n]) e = cudaMemcpyAsync(d_bids.p, b_ids, sizeof(int32_t) * (size_t)b_off[n], cudaMemcpyHostToDevice, s);
        if (e == cudaSuccess && b_n_idf) e = cudaMemcpyAsync(d_bidf.p, b_idf, sizeof(float) * (size_t)b_n_idf, cudaMemcpyHostToDevice, s);
    }
    if (e == cudaSuccess) e = cudaMemsetAsync(stat.p, 0, stat.bytes(), s);
    const IdfPart A{d_aoff.p, d_aids.p, d_aidf.p, a_n_idf, a_offset};
    const IdfPart B{d_boff.p, d_bids.p, d_bidf.p, b_off ? b_n_idf : 0, b_offset};
    const int64_t *moff = b_off ? d_moff.p : d_aoff.p;
    const unsigned grid = (unsigned)c->sm_count * 8;
    size_t sort_bytes = 0, scan_bytes = 0;
    if (e == cudaSuccess) {
        idf_gather_kernel<<<grid, 256, 0, s>>>(A, B, moff, n, total, key.p, head.p);
        c->launches++;
        e = cudaGetLastError();
    }
    // each row sorted on its own: a few ids per row for most rows, hundreds of thousands for a head item
    if (e == cudaSuccess) e = cub::DeviceSegmentedSort::SortKeys(nullptr, sort_bytes, key.p, key_s.p, (int)total, (int)n, moff, moff + 1, s);
    if (e == cudaSuccess) e = cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, keep.p, total + 1, s);
    if (e == cudaSuccess && (st = tmp.alloc(std::max(sort_bytes, scan_bytes)))) return st;
    if (e == cudaSuccess) e = cub::DeviceSegmentedSort::SortKeys(tmp.p, sort_bytes, key.p, key_s.p, (int)total, (int)n, moff, moff + 1, s);
    if (e == cudaSuccess) {
        idf_keep_kernel<<<grid, 256, 0, s>>>(A, B, key_s.p, head.p, total, keep.p);
        c->launches++;
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cub::DeviceScan::ExclusiveSum(tmp.p, scan_bytes, keep.p, total + 1, s);
    int64_t nnz = 0;
    if (e == cudaSuccess) e = cudaMemcpyAsync(&nnz, keep.p + total, sizeof(int64_t), cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) { set_error("idf vectors: %s", cudaGetErrorString(e)); return GORSE_B200_ERR_CUDA; }
    GB_TRY(out.ind.alloc((size_t)nnz));
    GB_TRY(out.val.alloc((size_t)nnz));
    idf_scatter_kernel<<<grid, 256, 0, s>>>(A, B, key_s.p, keep.p, total, out.ind.p, out.val.p, stat.p);
    idf_rows_kernel<<<div_up(n + 1, 256), 256, 0, s>>>(d_aoff.p, moff, keep.p, n, out.ind.p, d_out_off.p, stat.p);
    c->launches += 2;
    e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaMemcpyAsync(out.row_off.data(), d_out_off.p, sizeof(int64_t) * ((size_t)n + 1), cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(h_stat, stat.p, sizeof(h_stat), cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) { set_error("idf vectors: %s", cudaGetErrorString(e)); return GORSE_B200_ERR_CUDA; }
    if (h_stat[0]) {
        set_error(h_stat[0] & 1u ? "NaN value (an idf entry in use is NaN)"
                  : h_stat[0] & 2u ? "feature index too large (offset + id >= 0x7fffffff)"
                                   : "indices of a row are not strictly ascending (part B's offset does not place it after part A)");
        return GORSE_B200_ERR_ARG;
    }
    // the CSR of the non-empty rows
    for (int64_t r = 0; r < n; r++)
        if (out.row_off[(size_t)r + 1] > out.row_off[(size_t)r]) out.off.push_back(out.row_off[(size_t)r + 1]);
    out.n_features = nnz ? h_stat[1] + 1 : 0;
    return GORSE_B200_OK;
}

int32_t sparse_append(gorse_b200_sparse_index *ix, const SparseRows &rows)
{
    GB_TRY(sync_device(ix));   // the device layouts hold every stored row
    gorse_b200_ctx *c = ix->ctx;
    cudaStream_t s = c->stream;
    const int64_t n = (int64_t)ix->h_off.size() - 1, nnz_old = (int64_t)ix->h_ind.size();
    const int64_t m = (int64_t)rows.off.size() - 1, nnz = rows.off.back();
    if (m == 0) return GORSE_B200_OK;
    if (n + m >= (1ll << 31)) { set_error("more than 2^31 vectors"); return GORSE_B200_ERR_UNSUPPORTED; }
    const uint32_t F = std::max(ix->n_features, rows.n_features);
    // the new rows' offsets in the index and on the device; their entries from the staging buffers
    std::vector<int64_t> h_off((size_t)m);
    for (int64_t j = 0; j < m; j++) h_off[(size_t)j] = nnz_old + rows.off[(size_t)j + 1];
    std::vector<uint32_t> h_ind((size_t)nnz);
    std::vector<float> h_val((size_t)nnz);
    DevBuf<int64_t> off_n, foff_n, d_off;
    DevBuf<uint32_t> ind_n;
    DevBuf<float> val_n, fval_n;
    DevBuf<int32_t> frow_n;
    StreamSync sync{s};
    GB_TRY(off_n.alloc((size_t)(n + m + 1)));
    GB_TRY(ind_n.alloc((size_t)(nnz_old + nnz)));
    GB_TRY(val_n.alloc((size_t)(nnz_old + nnz)));
    GB_TRY(d_off.alloc((size_t)m + 1));
    cudaError_t e = cudaMemcpyAsync(d_off.p, rows.off.data(), sizeof(int64_t) * ((size_t)m + 1), cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(off_n.p, ix->off.p, sizeof(int64_t) * (size_t)(n + 1), cudaMemcpyDeviceToDevice, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(off_n.p + n + 1, h_off.data(), sizeof(int64_t) * (size_t)m, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess && nnz_old) e = cudaMemcpyAsync(ind_n.p, ix->ind.p, sizeof(uint32_t) * (size_t)nnz_old, cudaMemcpyDeviceToDevice, s);
    if (e == cudaSuccess && nnz_old) e = cudaMemcpyAsync(val_n.p, ix->val.p, sizeof(float) * (size_t)nnz_old, cudaMemcpyDeviceToDevice, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(ind_n.p + nnz_old, rows.ind.p, sizeof(uint32_t) * (size_t)nnz, cudaMemcpyDeviceToDevice, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(val_n.p + nnz_old, rows.val.p, sizeof(float) * (size_t)nnz, cudaMemcpyDeviceToDevice, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(h_ind.data(), rows.ind.p, sizeof(uint32_t) * (size_t)nnz, cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(h_val.data(), rows.val.p, sizeof(float) * (size_t)nnz, cudaMemcpyDeviceToHost, s);
    if (e != cudaSuccess) { set_error("sparse append: %s", cudaGetErrorString(e)); return GORSE_B200_ERR_CUDA; }
    GB_TRY(csc_append(c, d_off.p, rows.ind.p, rows.val.p, m, nnz, n, ix->foff.p, ix->frow.p, ix->fval.p, ix->n_features, nnz_old, F, foff_n,
                      frow_n, fval_n));   // csc_append synchronised the stream: the host copies are complete
    ix->off = std::move(off_n); ix->foff = std::move(foff_n); ix->ind = std::move(ind_n);
    ix->val = std::move(val_n); ix->frow = std::move(frow_n); ix->fval = std::move(fval_n);
    ix->h_off.insert(ix->h_off.end(), h_off.begin(), h_off.end());
    ix->h_ind.insert(ix->h_ind.end(), h_ind.begin(), h_ind.end());
    ix->h_val.insert(ix->h_val.end(), h_val.begin(), h_val.end());
    ix->n_features = F;
    return GORSE_B200_OK;
}

int32_t sparse_sync_device(gorse_b200_sparse_index *ix) { return sync_device(ix); }

size_t sparse_bytes(const gorse_b200_sparse_index *ix)
{
    return ix->off.bytes() + ix->foff.bytes() + ix->ind.bytes() + ix->val.bytes() + ix->frow.bytes() + ix->fval.bytes() + ix->tl_dot.bytes() +
           ix->tl_idx.bytes() + ix->tl_cnt.bytes() + ix->next.bytes() + ix->paths.bytes();
}

}  // namespace gb
