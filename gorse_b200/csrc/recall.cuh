// recall.cuh -- block-wide selection and sorting helpers of the batched recall (recall.cu), shared with the item-to-item
// aggregation (item_to_item.cu), and the recall's chunked row pipeline.
#pragma once
#include <vector>

#include "vecdb.cuh"

namespace gb {
namespace recall {

#ifdef __CUDACC__
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
    for (int shift = 8 * (int)sizeof(K) - 8; shift >= 0; shift -= 8) {
        for (int b = threadIdx.x; b < 256; b += NT) hist[b] = 0;
        __syncthreads();
        for (int64_t i = threadIdx.x; i < n; i += NT) {
            const K k = key_at(i);
            if (k != 0u && (k & mask) == prefix) atomicAdd(&hist[(uint32_t)(k >> shift) & 255u], 1);
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            int above = 0, b = 255;
            for (; b > 0 && above + hist[b] < need; b--) above += hist[b];
            s_bc[0] = b;
            s_bc[1] = need - above;
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

#endif  // __CUDACC__

template <typename T>
int32_t grow(DevBuf<T> &b, size_t n)
{
    return b.n >= n ? GORSE_B200_OK : b.alloc(n);
}

// The chunked row pipeline of gorse_b200_vecdb_query_excluding (routing, tensor-core sweep, window and exact kernels), for
// nq rows of one collection whose allow mask is current.  Row q is a host query q_host[q * d ..] or, with q_host == nullptr,
// the stored vector of slot d_qslots[q] (a device list), gathered on the device.  k_q = n + (excl_off[q + 1] - excl_off[q]);
// ex / ex_off: each row's exclusions sorted, -1 entries dropped.  Row q's answer starts at q * n + excl_off[q] in
// db->recall.slots / scores, count in db->recall.count[q]; with slots_out != nullptr every finished chunk is also downloaded
// to the host buffers while the next one computes.  *exact_rows_out: rows the exact kernel answered.  The caller holds
// db->mu; the call ends with both streams synchronised.
int32_t recall_rows(gorse_b200_vecdb *db, int64_t nq, const float *q_host, const int64_t *d_qslots, int32_t n, const int64_t *excl_off,
                    const std::vector<int64_t> &ex, const std::vector<int64_t> &ex_off, int64_t *slots_out, float *scores_out,
                    int32_t *count_out, int64_t *exact_rows_out);

}  // namespace recall
}  // namespace gb
