// topk.cuh -- brute-force index state shared by topk.cu (the top-k pipeline) and topk_mma.cu (tensor-core stage 1).
#pragma once
#include <cuda_bf16.h>

#include "cf.cuh"
#include "common.cuh"

namespace gb {
// grow-only work buffers of the top-k pipeline (recall::recall_rows), kept with the index, and the host side of a chunk's
// row tables
struct RecallWork {
    DevBuf<float> q, scores, scratch;
    DevBuf<int64_t> ex_off, ex, out_off, rows, slots;
    DevBuf<int32_t> k, count, flags;
    std::vector<int32_t> h_k;
    std::vector<int64_t> h_exoff, h_outoff, h_rows;
    std::vector<int8_t> h_cls;
    size_t bytes() const
    {
        return q.bytes() + scores.bytes() + scratch.bytes() + ex_off.bytes() + ex.bytes() + out_off.bytes() + rows.bytes() + slots.bytes() +
               k.bytes() + count.bytes() + flags.bytes();
    }
};

// the stored rows of an index as a kernel reads them: fp32 values, or bf16 values kept as the high 16 bits of their fp32 bit
// patterns (uint16_t).  A launch picks its instantiation once, through with_rows; no kernel branches on the element type.
struct RowView {
    const void *p;
    bool bf16;
};
template <typename F>
inline auto with_rows(RowView v, F f)
{
    return v.bf16 ? f(static_cast<const uint16_t *>(v.p)) : f(static_cast<const float *>(v.p));
}
// the element type behind a row pointer of with_rows
template <typename P>
using row_elem_t = std::remove_const_t<std::remove_pointer_t<P>>;
// the 4-value vector of an element type: one 16-byte (fp32) or 8-byte (bf16) load
template <typename T>
struct row_quad_type { using type = float4; };
template <>
struct row_quad_type<uint16_t> { using type = uint2; };
}  // namespace gb

struct gorse_b200_index {
    gorse_b200_ctx *ctx = nullptr;
    int32_t d = 0, metric = 0;
    int64_t n = 0, cap = 0;
    // the vectors as added, [cap x d] row-major, in exactly one of X (value_bytes 4) and Xh (value_bytes 2; the exact re-rank reads
    // these).  The bare index is fp32.  A vector collection's index starts bf16 and stays so while every value it was given is
    // bf16-exact (low 16 bits zero); the first value that is not promotes it to fp32 for good (index_append, index_promote).
    gb::DevBuf<float> X;
    gb::DevBuf<uint16_t> Xh;
    int32_t value_bytes = 4;
    gb::DevBuf<float> stage;        // grow-only fp32 staging of a bf16 index's host uploads (at most APPEND_STAGE_BYTES)
    gb::DevBuf<int32_t> inexact;    // [1] the narrowing kernel's flag: a value was not bf16-exact
    gb::DevBuf<__nv_bfloat16> Xb;   // [n_pad x d] bf16 mirror feeding the tensor cores (built lazily)
    gb::DevBuf<float> norm;         // per-vector fp32 norms (+ max at [n], max |bf16(x) - x| at [n + 1]), built lazily
    gb::DevBuf<int32_t> perm;       // mirror row p holds vector perm[p] (random: the first columns are a uniform sample)
    float max_norm = 0.f;           // max |x| and max |bf16(x) - x| over the vectors: the per-row eps of stage 1 (topk_mma.cu)
    float max_dx = 0.f;
    bool mma_ready = false;
    float *dbg_scores = nullptr;    // tests only: dense stage-1 scores
    int64_t last_fallback_rows = 0; // rows of the last searches whose candidate set failed certification
    std::vector<cudaEvent_t> ev;    // CUDA event pairs around the stage-1 kernels of one call (bench.py roofline)
    double stage1_ms = 0.0, stage1_flop = 0.0; // accumulated since the last debug read
    // reusable work buffers of the tensor path (sized for w_cq query rows at mirror width w_kp)
    int64_t w_cq = 0;
    int w_kp = 0;
    gb::DevBuf<__nv_bfloat16> w_qb;
    gb::DevBuf<float> w_eps, w_cval, w_theta;
    gb::DevBuf<int32_t> w_ccol, w_ccnt;
    gb::RecallWork recall;
    // result staging of search_common (grow-only: a 120 MB cudaMalloc + cudaFree per all-pairs call otherwise)
    gb::DevBuf<int32_t> r_idx, r_count;
    gb::DevBuf<float> r_dist;
    std::mutex mu;
    gb::RowView rows() const { return value_bytes == 2 ? gb::RowView{Xh.p, true} : gb::RowView{X.p, false}; }
};

namespace gb {

// geometry of the tensor-core sweep (topk_mma.cu) and of its candidate lists
namespace mma {
constexpr int BM = 64, BN = 128, BK = 64;      // rows per consumer warpgroup (queries), tile columns (vectors), k-block (bf16)
constexpr int CONSUMERS = 2;                   // consumer warpgroups per CTA; both multiply every B tile
constexpr int GROUP_ROWS = CONSUMERS * BM;     // query rows of one CTA pass over all vectors
constexpr int MAX_KB = 3;                      // k-blocks per tile with the queries resident: Kp <= 192
constexpr int MAX_D = 4096;                    // the widest rows the sweep takes
constexpr int WIDE_MAX_KB = (MAX_D + 2 + BK - 1) / BK;   // k-blocks per tile of the wide sweep (both operands streamed): Kp <= 4160
                                               // with the two norm columns of Euclidean at d = 4096
constexpr int CAP = 2048;                      // candidate slots per query row
constexpr int PARTS = 4;                       // a row's columns are split over the 4 threads of an accumulator quad
constexpr int PART_CAP = CAP / PARTS;          // candidate slots per (row, part)
constexpr int R_TOP = 16;                      // sample order statistic that fixes the threshold
constexpr int THREADS = 128 * (1 + CONSUMERS); // warpgroup 0: warp 0 = TMA producer, warps 1-3 idle; then the consumers
constexpr uint32_t A_TILE_BYTES = BM * BK * 2; // one [64 x 64] bf16 k-block of queries = 8 KB
constexpr uint32_t B_TILE_BYTES = BN * BK * 2; // one [128 x 64] bf16 k-block of vectors = 16 KB
// a ring slot of the wide sweep: one k-block of both consumers' queries and of the vector tile = 32 KB.  6 slots (193 KB with
// the alignment and barriers) leave about as much L1 beside the 227 KB shared-memory budget as the narrow sweep's ring does.
constexpr uint32_t WIDE_STAGE_BYTES = CONSUMERS * A_TILE_BYTES + B_TILE_BYTES;
constexpr int WIDE_STAGES = 6;
static_assert(WIDE_STAGES * WIDE_STAGE_BYTES + 1024 + 256 <= 227 * 1024, "the wide ring fits the shared-memory budget");
}  // namespace mma

#ifdef __CUDACC__
// widening of stored bf16 values: bits << 16, exact (no flush of subnormals, NaN payloads kept); the fp32 forms are the identity
__device__ __forceinline__ float widen(float v) { return v; }
__device__ __forceinline__ float4 widen(float4 v) { return v; }
__device__ __forceinline__ float widen(uint16_t h) { return __uint_as_float((uint32_t)h << 16); }
__device__ __forceinline__ float4 widen(uint2 h)   // 4 bf16 values, little-endian: value 0 is the low half of h.x
{
    return make_float4(__uint_as_float(h.x << 16), __uint_as_float(h.x & 0xffff0000u), __uint_as_float(h.y << 16),
                       __uint_as_float(h.y & 0xffff0000u));
}
// the exact scan's arithmetic, shared by the index search (topk.cu) and the batched recall (recall.cu)
// exact distance by a quad, d % 16 == 0.  Euclidean: floats_avx512.c:374-441 (sub, mul, add: no fusing).
// T = float or uint16_t (bf16 rows): the lane's 4 values of a 16-value chunk are one 16- or 8-byte load either way.
template <typename T>
__device__ __forceinline__ float quad_dist(const float4 *q /* C regs, query chunk c at q[c] */, const T *x, int chunks,
                                           int lane4, unsigned mask, int metric, float qq)
{
    const auto *x4 = reinterpret_cast<const typename row_quad_type<T>::type *>(x) + lane4;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    if (metric == GORSE_B200_METRIC_COSINE) {   // 1 - q.x / (|q| |x|); the reference's arithmetic lives in its vector store (unpinned)
        float4 xx = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int c = 0; c < chunks; c++) {
            const float4 b = widen(__ldg(x4 + 4 * c));
            dot_chunk(acc, q[c], b, c == 0);
            dot_chunk(xx, b, b, c == 0);
        }
        const float dot = quad_tree(acc, mask), nx = quad_tree(xx, mask);
        return __fsub_rn(1.0f, __fdiv_rn(dot, __fmul_rn(__fsqrt_rn(qq), __fsqrt_rn(nx))));
    }
    if (metric == GORSE_B200_METRIC_NEG_DOT) {
        for (int c = 0; c < chunks; c++) dot_chunk(acc, q[c], widen(__ldg(x4 + 4 * c)), c == 0);
        return -quad_tree(acc, mask);
    }
    for (int c = 0; c < chunks; c++) {
        float4 b = widen(__ldg(x4 + 4 * c)), v;
        v.x = __fsub_rn(q[c].x, b.x); v.y = __fsub_rn(q[c].y, b.y); v.z = __fsub_rn(q[c].z, b.z); v.w = __fsub_rn(q[c].w, b.w);
        v.x = __fmul_rn(v.x, v.x); v.y = __fmul_rn(v.y, v.y); v.z = __fmul_rn(v.z, v.z); v.w = __fmul_rn(v.w, v.w);
        if (c == 0) acc = v;
        else { acc.x = __fadd_rn(v.x, acc.x); acc.y = __fadd_rn(v.y, acc.y); acc.z = __fadd_rn(v.z, acc.z); acc.w = __fadd_rn(v.w, acc.w); }
    }
    return __fsqrt_rn(quad_tree(acc, mask));
}

// any d, one thread (8-lane block + fused tails as in the reference); b = a stored row, T = float or uint16_t (bf16)
template <typename T>
__device__ inline float dist_any(const float *a, const T *b, int n, int metric, float qq)
{
    if (metric == GORSE_B200_METRIC_NEG_DOT) return -dot_any(a, b, n);
    if (metric == GORSE_B200_METRIC_COSINE)
        return __fsub_rn(1.0f, __fdiv_rn(dot_any(a, b, n), __fmul_rn(__fsqrt_rn(qq), __fsqrt_rn(dot_any(b, b, n)))));
    int epoch = n / 16, remain = n % 16;
    float s[16];
#pragma unroll
    for (int l = 0; l < 16; l++) s[l] = 0.f;
    if constexpr (std::is_same<T, uint16_t>::value) {   // bf16 rows: 16 values by two loads (row_chunk16)
        float bv[16];
        if (epoch > 0) {
            row_chunk16(b, bv);
#pragma unroll
            for (int l = 0; l < 16; l++) { float v = __fsub_rn(a[l], bv[l]); s[l] = __fmul_rn(v, v); }
        }
        for (int c = 1; c < epoch; c++) {
            row_chunk16(b + 16 * c, bv);
#pragma unroll
            for (int l = 0; l < 16; l++) { float v = __fsub_rn(a[16 * c + l], bv[l]); s[l] = __fadd_rn(__fmul_rn(v, v), s[l]); }
        }
    } else {
        if (epoch > 0) {
#pragma unroll
            for (int l = 0; l < 16; l++) { float v = __fsub_rn(a[l], row_val(b, l)); s[l] = __fmul_rn(v, v); }
        }
        for (int c = 1; c < epoch; c++) {
#pragma unroll
            for (int l = 0; l < 16; l++) { float v = __fsub_rn(a[16 * c + l], row_val(b, 16 * c + l)); s[l] = __fadd_rn(__fmul_rn(v, v), s[l]); }
        }
    }
    float r4[4];
#pragma unroll
    for (int l = 0; l < 4; l++) r4[l] = __fadd_rn(__fadd_rn(s[l + 12], s[l + 4]), __fadd_rn(s[l + 8], s[l]));
    float sum = __fadd_rn(__fadd_rn(r4[0], r4[2]), __fadd_rn(r4[1], r4[3]));
    a += 16 * epoch; b += 16 * epoch;
    if (remain >= 8) {
        float p[8];
#pragma unroll
        for (int l = 0; l < 8; l++) { float v = __fsub_rn(a[l], row_val(b, l)); p[l] = __fmul_rn(v, v); }
        float q4[4];
#pragma unroll
        for (int l = 0; l < 4; l++) q4[l] = __fadd_rn(p[l + 4], p[l]);
        sum = __fadd_rn(sum, __fadd_rn(__fadd_rn(q4[0], q4[2]), __fadd_rn(q4[1], q4[3])));
        a += 8; b += 8; remain -= 8;
    }
    for (int i = 0; i < remain; i++) { float v = __fsub_rn(a[i], row_val(b, i)); sum = __fmaf_rn(v, v, sum); }
    return __fsqrt_rn(sum);
}

// order-preserving 32-bit keys of fp32 scores (larger score = larger key)
__device__ __forceinline__ uint32_t float_key(float v)
{
    const uint32_t u = __float_as_uint(v);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_float(uint32_t k)
{
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}
#endif  // __CUDACC__

// make room for `need` vectors in the rows of the index's element type (amortised doubling); the caller holds ix->mu
int32_t index_reserve(gorse_b200_index *ix, int64_t need);
// the add path of every index: m rows, row s = src[(map ? map[s] : s) * d ..], src on the host (map == nullptr) or the device.
// A bf16 index narrows them (host rows through ix->stage, at most APPEND_STAGE_BYTES at a time) and promotes itself to fp32 before
// they land when one value is not bf16-exact.  On an error the index is exactly as it was.  The caller holds ix->mu.
int32_t index_append(gorse_b200_index *ix, const float *src, const int32_t *map, int64_t m, bool host);
constexpr int64_t APPEND_STAGE_BYTES = 64ll << 20;
// launches the narrowing of m fp32 device rows (row s = src[(map ? map[s] : s) * d ..]) into the bf16 rows dst on stream s;
// *inexact (device) becomes 1 when a value is not bf16-exact, and dst then holds its truncation
cudaError_t index_narrow(int d, gorse_b200_ctx *c, cudaStream_t s, const float *src, const int32_t *map, int64_t m, uint16_t *dst,
                         int32_t *inexact);
// promotion of a bf16 index: fp32 rows of capacity ix->cap, rows [0, rows) widened from Xh in one pass, Xh released.  One-way.
// On an error the index is unchanged.  The caller holds ix->mu.
int32_t index_promote(gorse_b200_index *ix, int64_t rows);
// out[i * d ..] (host) = the fp32 values of stored row rows[i] (host list), for every i with rows[i] >= 0; fp32 rows are copied
// one by one into out, bf16 rows one by one into a host buffer and widened there.  Ends with the stream synchronised.
int32_t index_download_rows(gorse_b200_index *ix, const int64_t *rows, int64_t n, float *out);
// compaction (gorse_b200_vecdb_compact): scan[n + 1] (device) is the exclusive sum of the live flags, so slot s is live iff
// scan[s + 1] != scan[s] and then moves to scan[s]; X becomes the live rows in order, live = scan[n] of them, with cap = live,
// and everything built from the old rows (mirror, norms, permutation, exact scratch, stage-1 counters) is dropped.  On an
// error the index is unchanged.  The caller holds ix->mu.
int32_t index_compact(gorse_b200_index *ix, const int64_t *scan, int64_t live);
// device bytes held by the index and its work buffers
size_t index_bytes(const gorse_b200_index *ix);
// the tensor-core candidate sweep (topk_mma.cu) of the top-k pipeline (recall_rows) and of the stage-1 test hook.
// mma_reserve: the bf16 mirror and the work buffers for up to cq query rows per sweep; GORSE_B200_ERR_OOM when they do not fit,
// with none of them held (the caller answers through the exact kernel).  mma_sample_tiles: the sample size
// that leaves about `cands` columns per row above its threshold.  mma_sweep: query rows (q_base, d_q, d_qidx, q0 as in
// build_queries_kernel) -> candidate lists in ix->w_ccol / w_cval / w_ccnt / w_theta, eps in ix->w_eps; ev0 / ev1 (may be
// nullptr) are recorded around the sweep kernel.
int32_t mma_reserve(gorse_b200_index *ix, int64_t cq);
int mma_sample_tiles(const gorse_b200_index *ix, double cands);
int32_t mma_sweep(gorse_b200_index *ix, RowView q_base, const float *d_q, const int64_t *d_qidx, int64_t q0, int64_t nq, int m_tiles,
                  cudaEvent_t ev0, cudaEvent_t ev1);
// the sweep serves Dot and Euclidean indexes of >= 32768 vectors, d <= 4096, for >= 64 rows; GORSE_B200_TOPK_EXACT=1 turns it off
bool mma_path_eligible(const gorse_b200_index *ix, int64_t nq);

namespace recall {
// A fixed-stride copy of the pipeline's answers (table_kernel): row q's entries at q * n, in order, with int32 slots; the
// value is the score, negated when negate (the index's distance); with positive only values > 0 are kept; the row is padded
// with slot -1 / value 0 and cnt[q] holds the kept entries.  h_*: host copies downloaded per chunk, or all nullptr.
struct Table {
    int32_t *slot;
    float *val;
    int32_t *cnt;
    bool negate, positive;
    int32_t *h_slot;
    float *h_val;
    int32_t *h_cnt;
};

// The dense top-k pipeline (topk.cu): routing, tensor-core sweep, window and exact kernels, for nq rows of the index.  Row q
// is a host query q_host[q * d ..] or, with q_host == nullptr, the stored vector of slot d_qslots[q] (a device list), which
// the row never returns.  allow (device, may be nullptr = every vector): 0 = never returned.  k_q = n + (excl_off[q + 1] -
// excl_off[q]); ex[ex_off[q] ..]: each row's exclusions sorted, -1 entries dropped; excl_off == nullptr: no exclusions, k_q = n
// (ex and ex_off are not read).  Row q's answer is the first k_q allowed
// vectors by (score desc, slot asc) minus its exclusions, score = -distance; it starts at q * n + excl_off[q] in
// ix->recall.slots / scores, count in ix->recall.count[q].  Every finished chunk is copied into `table` (may be nullptr) and
// downloaded to the host buffers slots_out / scores_out / count_out (may be nullptr) and the table's host copies while the
// next one computes.  *exact_rows_out (may be nullptr): rows the exact kernel answered.  The caller holds ix->mu; the call
// ends with both streams synchronised.
int32_t recall_rows(gorse_b200_index *ix, const uint8_t *allow, int64_t nq, const float *q_host, const int64_t *d_qslots, int32_t n,
                    const int64_t *excl_off, const int64_t *ex, const int64_t *ex_off, const Table *table, int64_t *slots_out,
                    float *scores_out, int32_t *count_out, int64_t *exact_rows_out);
}  // namespace recall

}  // namespace gb
