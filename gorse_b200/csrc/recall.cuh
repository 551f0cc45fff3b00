// recall.cuh -- block-wide selection and sorting helpers of the top-k pipeline (topk.cu), shared with the item-to-item
// aggregation (item_to_item.cu) and the sparse search (sparse.cu).
#pragma once
#include "common.cuh"
#include "topk.cuh"

namespace gb {
namespace recall {

constexpr int SORT_CAP = mma::CAP;   // entries one CTA sorts at a time (a window never holds more)

#ifdef __CUDACC__
// order key of a score: larger score = larger key; -0 and +0 are one score (the exact scan compares floats); NaN = 0 = no entry
__device__ __forceinline__ uint32_t rank_key(float s) { return s != s ? 0u : float_key(s == 0.f ? 0.f : s); }
// sort key: ascending order = score descending, then slot ascending
__device__ __forceinline__ uint64_t sort_key(uint32_t key, int64_t slot) { return ((uint64_t)~key << 32) | (uint32_t)slot; }

__device__ __forceinline__ bool contains(const int64_t *a, int64_t n, int64_t v)
{
    int64_t lo = 0, hi = n;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (a[mid] < v) lo = mid + 1;
        else hi = mid;
    }
    return lo < n && a[lo] == v;
}

// exclusive rank of f among the CTA's threads in thread order; total = how many are set.  Every thread calls it.
template <int NT>
__device__ __forceinline__ int block_rank(bool f, int *s_warp, int &total)
{
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const unsigned b = __ballot_sync(0xffffffffu, f);
    __syncthreads();   // s_warp is free again
    if (lane == 0) s_warp[w] = __popc(b);
    __syncthreads();
    int before = 0;
    total = 0;
#pragma unroll
    for (int i = 0; i < NT / 32; i++) {
        const int c = s_warp[i];
        before += i < w ? c : 0;
        total += c;
    }
    return before + __popc(b & ((1u << lane) - 1));
}

template <int NT>
__device__ __forceinline__ int block_sum(int v, int *s_warp)
{
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = v;
    __syncthreads();
    int t = 0;
#pragma unroll
    for (int i = 0; i < NT / 32; i++) t += s_warp[i];
    return t;
}

// the m-th largest non-zero key of key_at(0 .. n-1) (at least m of them are non-zero), 8 bits per pass; the key type
// (uint32_t or uint64_t) is what key_at returns.  *ties = how many entries equal to the result belong to the m largest.
template <int NT, typename KeyAt>
__device__ auto block_select(int64_t n, int m, KeyAt key_at, int *hist /* [256] */, int *s_bc /* [2] */, int *ties) -> decltype(key_at(0))
{
    using K = decltype(key_at(0));
    K prefix = 0, mask = 0;
    int need = m;
    const int lane = threadIdx.x & 31;
    for (int shift = 8 * (int)sizeof(K) - 8; shift >= 0; shift -= 8) {
        for (int b = threadIdx.x; b < 256; b += NT) hist[b] = 0;
        __syncthreads();
        for (int64_t i = threadIdx.x; i < n; i += NT) {
            const K k = key_at(i);
            if (k != 0u && (k & mask) == prefix) atomicAdd(&hist[(uint32_t)(k >> shift) & 255u], 1);
        }
        __syncthreads();
        if (threadIdx.x < 32) {
            // the bin holding the need-th largest key, from the top: lane l sums bins 255 - 8 l .. 248 - 8 l, a warp scan
            // gives the keys above each lane's bins, and the lane where the running count reaches need picks the bin (bins
            // 255 .. 1; bin 0 when they hold fewer than need keys)
            int sum = 0;
#pragma unroll
            for (int j = 0; j < 8; j++) sum += hist[255 - 8 * lane - j];
            int incl = sum;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int t = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += t;
            }
            int above = incl - sum, pick = -1;
#pragma unroll
            for (int j = 0; j < 8; j++) {
                const int b = 255 - 8 * lane - j;
                if (pick < 0 && b > 0 && above + hist[b] >= need) pick = b;
                if (pick < 0 && b > 0) above += hist[b];
            }
            const unsigned found = __ballot_sync(0xffffffffu, pick >= 0);
            const int src = found ? __ffs(found) - 1 : 31;   // none: bin 0, above = the keys of bins 255 .. 1
            const int b = __shfl_sync(0xffffffffu, pick >= 0 ? pick : 0, src);
            const int ab = __shfl_sync(0xffffffffu, above, src);
            if (lane == 0) {
                s_bc[0] = b;
                s_bc[1] = need - ab;
            }
        }
        __syncthreads();
        prefix |= (K)s_bc[0] << shift;
        mask |= (K)255u << shift;
        need = s_bc[1];
        __syncthreads();
    }
    *ties = need;
    return prefix;
}

// ascending bitonic sort of key[0, p) with a payload, p a power of two
template <int NT, typename Key, typename Val>
__device__ void block_sort(Key *key, Val *val, int p)
{
    for (int size = 2; size <= p; size <<= 1)
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            for (int i = threadIdx.x; i < p / 2; i += NT) {
                const int lo = 2 * i - (i & (stride - 1)), hi = lo + stride;
                const bool up = (lo & size) == 0;
                const Key a = key[lo], b = key[hi];
                if ((a > b) == up) {
                    key[lo] = b; key[hi] = a;
                    const Val t = val[lo]; val[lo] = val[hi]; val[hi] = t;
                }
            }
            __syncthreads();
        }
}

__host__ __device__ __forceinline__ int pow2_at_least(int m)
{
    int p = 1;
    while (p < m) p <<= 1;
    return p;
}

// The first K entries of the score row sc[0, N) by (score desc, slot asc), K <= its non-NaN entries, in sorted rounds of at
// most SORT_CAP: each round radix-selects its last key, gathers its entries into s_key / s_val [SORT_CAP] (those equal to the
// last key in slot order: the lowest slots win the tie), sorts them, hands them to emit(m) and retires them (sc = NaN).
// Every thread calls it.
template <int NT, typename Emit>
__device__ __forceinline__ void emit_in_rounds(float *sc, int64_t N, int K, uint64_t *s_key, float *s_val, int *hist, int *s_warp, int *s_bc,
                                               Emit emit)
{
    const float none = __int_as_float(0x7fffffff);   // NaN: rank_key 0
    for (int emitted = 0; emitted < K;) {
        const int m = min(SORT_CAP, K - emitted);
        int ties;
        const uint32_t t = block_select<NT>(N, m, [&](int64_t j) { return rank_key(sc[j]); }, hist, s_bc, &ties);
        if (threadIdx.x == 0) s_bc[2] = 0;
        int eq_taken = 0;   // entries equal to t go in slot order: the lowest slots win the tie
        __syncthreads();
        for (int64_t base = 0; base < N; base += NT) {
            const int64_t j = base + threadIdx.x;
            const uint32_t key = j < N ? rank_key(sc[j]) : 0u;
            int n_eq;
            const int er = block_rank<NT>(key == t, s_warp, n_eq);
            int pos = -1;
            if (key > t) pos = atomicAdd(&s_bc[2], 1);
            else if (key == t && eq_taken + er < ties) pos = m - ties + eq_taken + er;
            if (pos >= 0) { s_key[pos] = sort_key(key, j); s_val[pos] = sc[j]; }
            eq_taken += n_eq;
        }
        const int p2 = pow2_at_least(m);
        for (int j = m + threadIdx.x; j < p2; j += NT) s_key[j] = ~0ull;
        __syncthreads();
        block_sort<NT>(s_key, s_val, p2);
        emit(m);
        for (int j = threadIdx.x; j < m; j += NT) sc[(uint32_t)s_key[j]] = none;
        __syncthreads();
        emitted += m;
    }
}

#endif  // __CUDACC__

}  // namespace recall
}  // namespace gb
