// aggregate.cuh -- what the batched recommenders' two aggregation kernels share (i2i_aggregate_kernel in item_to_item.cu,
// for item-to-item and session; u2u_aggregate_kernel in user_to_user.cu): the neighbour score transform, the shared-memory
// layout of one aggregating CTA, the float64 sum per id, and the selection of the first n float64 sums by (sum descending,
// id ascending).
#pragma once
#include "recall.cuh"

namespace gb {
namespace agg {

using u128 = unsigned __int128;

constexpr int THREADS = 256;
constexpr int TABLE_CAP = 8192;                  // shared-memory table entries: int32 id + float64 sum, 96 KB
constexpr int TABLE_KEYS = TABLE_CAP / 4 * 3;    // a user takes the table when its adds are at most this (load <= 3/4)

// dynamic shared memory of one aggregating CTA for n results; `table`: with the open-addressing table
inline size_t smem_bytes(int n, bool table)
{
    const size_t p2 = (size_t)recall::pow2_at_least(n);
    return p2 * 24 + (256 + 32 + 4) * 4 + (table ? (size_t)TABLE_CAP * 12 : 0);
}

#ifdef __CUDACC__
struct Smem {
    u128 *s_key;      // [p2] sort keys: ~sum key, then id
    double *s_val;    // [p2]
    int *hist;        // [256]
    int *s_warp;      // [32]
    int *s_bc;        // [4]: [0..1] select, [2] gather fill, [3] distinct ids (the caller's)
    int32_t *t_key;   // table: [TABLE_CAP] id, -1 = empty
    double *t_val;    // table: [TABLE_CAP] sum
};

__device__ __forceinline__ Smem carve(uint8_t *sm, int p2)
{
    Smem S;
    S.s_key = reinterpret_cast<u128 *>(sm);
    S.s_val = reinterpret_cast<double *>(S.s_key + p2);
    S.hist = reinterpret_cast<int *>(S.s_val + p2);
    S.s_warp = S.hist + 256;
    S.s_bc = S.s_warp + 32;
    S.t_key = reinterpret_cast<int32_t *>(S.s_bc + 4);
    S.t_val = reinterpret_cast<double *>(S.t_key + TABLE_CAP);
    return S;
}

// order-preserving 64-bit key of a float64 sum (never 0: the sums are not NaN)
__device__ __forceinline__ uint64_t sum_key(double v)
{
    const uint64_t u = (uint64_t)__double_as_longlong(v);
    return (u >> 63) ? ~u : (u | (1ull << 63));
}

// QueryItemToItem's / QueryUserToUser's score (logics/item_to_item.go:76-79, logics/user_to_user.go:76-79), rounded step
// by step as Go does
__device__ __forceinline__ double neighbour_score(float raw, double scale, bool euclid)
{
    const double s = __dmul_rn((double)raw, scale);
    return euclid ? __ddiv_rn(1.0, __dsub_rn(1.0, s)) : s;
}

// sum[id] += s for one CTA's float64 sums, each starting at 0 + s as the reference's map does.  SHARED: the open-addressing
// table t_key / t_val of cap = 2^lg entries; else the global row acc with its flag row seen and the list touched of the ids
// set so far.  *distinct counts the ids.  Concurrent calls must add to distinct ids.
template <bool SHARED>
__device__ __forceinline__ void add_sum(int32_t id, double s, int32_t *t_key, double *t_val, int cap, int lg, double *acc, uint8_t *seen,
                                        int32_t *touched, int *distinct)
{
    if (SHARED) {
        uint32_t h = ((uint32_t)id * 0x9E3779B1u) >> (32 - lg);
        for (;;) {
            const int32_t k = t_key[h];
            if (k == id) { t_val[h] = __dadd_rn(t_val[h], s); break; }
            if (k < 0 && atomicCAS(&t_key[h], -1, id) == -1) {
                t_val[h] = __dadd_rn(0.0, s);
                atomicAdd(distinct, 1);
                break;
            }
            h = (h + 1) & (uint32_t)(cap - 1);
        }
    } else if (seen[id]) {
        acc[id] = __dadd_rn(acc[id], s);
    } else {
        seen[id] = 1;
        touched[atomicAdd(distinct, 1)] = id;
        acc[id] = __dadd_rn(0.0, s);
    }
}

// The first m = min(n, distinct) of the entries 0 .. range-1 by (sum descending, id ascending), sorted into S.s_key (low 32
// bits: the id) / S.s_val [0, m).  id_at(j) < 0 marks an empty entry; `distinct` entries are not empty.  The n-th largest
// sum key comes from an 8-bit radix select; when more sums equal it than the cut admits, a second 32-bit select keeps the
// lowest ids among them; the winners are bitonic-sorted on the 128-bit key.  Every thread of the CTA calls it; returns m.
template <int NT, typename IdAt, typename ValAt>
__device__ int select_first_n(int64_t range, int distinct, int n, int p2, IdAt id_at, ValAt val_at, const Smem &S)
{
    using namespace gb::recall;
    const int m = min(n, distinct);
    if (m == 0) return 0;
    auto key_at = [&](int64_t j) -> uint64_t { return id_at(j) >= 0 ? sum_key(val_at(j)) : 0ull; };
    int ties;
    const uint64_t K = block_select<NT>(range, m, key_at, S.hist, S.s_bc, &ties);
    // of the sums equal to the m-th, the `ties` lowest ids are kept
    int eq = 0;
    for (int64_t j = threadIdx.x; j < range; j += NT) eq += key_at(j) == K;
    eq = block_sum<NT>(eq, S.s_warp);
    uint32_t last = 0xffffffffu;
    if (eq > ties) {
        int t2;
        last = ~block_select<NT>(range, ties, [&](int64_t j) { return key_at(j) == K ? ~(uint32_t)id_at(j) : 0u; }, S.hist, S.s_bc, &t2);
    }
    if (threadIdx.x == 0) S.s_bc[2] = 0;
    __syncthreads();
    for (int64_t j = threadIdx.x; j < range; j += NT) {
        const uint64_t k = key_at(j);
        if (k > K || (k == K && (uint32_t)id_at(j) <= last)) {
            const int pos = atomicAdd(&S.s_bc[2], 1);
            S.s_key[pos] = ((u128)~k << 64) | (uint32_t)id_at(j);
            S.s_val[pos] = val_at(j);
        }
    }
    for (int j = m + threadIdx.x; j < p2; j += NT) S.s_key[j] = ~(u128)0;
    __syncthreads();
    block_sort<NT>(S.s_key, S.s_val, p2);
    return m;
}
#endif  // __CUDACC__

}  // namespace agg
}  // namespace gb
