// fm_gauc.cuh -- the per-user AUC of gorse_b200_fm_gauc (EvaluateAFM, cmd/gorse-bench/main.go:125-207; DESIGN §8.10).
// Included by fm_fit.cu inside gb::fmfit; the predictions come from Fit::predict, the trainer's list forward.
//
//   fm_gauc_keys_kernel  a thread per test row: key = user << 33 | (target <= 0) << 32 | the prediction's orderable bits
//   (one cub radix sort of the keys over the bits n_users needs: each user's positives ascending, then its negatives)
//   fm_gauc_user_kernel  a warp per scored user: per positive the negatives strictly below it, their sum as the reference's
//                        float32 chain forms it, and the AUC
#pragma once

struct GaucUser {                // a scored user's keys in the sorted list: positives [start, start + P), then N negatives
    int32_t start, P, N;
};

// a float's bits in an order that unsigned comparison shares with `<`: -0 folds into +0 so that they tie; a NaN lands above
// +Inf or below -Inf, so the key still tells it apart
__device__ __forceinline__ uint32_t ord_f32(float f)
{
    const uint32_t b = f == 0.0f ? 0u : __float_as_uint(f);
    return (b & 0x80000000u) ? ~b : b | 0x80000000u;
}

__device__ __forceinline__ bool ord_nan(uint32_t o) { return o > 0xff800000u || o < 0x007fffffu; }

// row_hi[r] = user << 1 | (target <= 0), from the host
__global__ void fm_gauc_keys_kernel(const float *pred, const uint32_t *row_hi, int64_t n, uint64_t *key)
{
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        key[i] = (uint64_t)row_hi[i] << 32 | ord_f32(pred[i]);
}

// AUC(pos, neg) (evaluator.go:136-153) of every scored user, comparing the keys' low halves (the orderable predictions; the
// high halves differ in the list bit).  Every count is at most N, so with P N <= 2^24 each partial sum of the reference's
// float32 chain is an integer below 2^24 and exact: the warp sums the counts as integers and converts once.  Above that one
// lane runs the reference's walk and chain.  A NaN prediction makes the AUC NaN (the reference's sort order is then unpinned).
__global__ void __launch_bounds__(WARPS * 32) fm_gauc_user_kernel(const uint64_t *key, const GaucUser *users, int64_t n_scored, float *auc)
{
    const int lane = threadIdx.x & 31;
    for (int64_t j = (int64_t)blockIdx.x * WARPS + (threadIdx.x >> 5); j < n_scored; j += (int64_t)gridDim.x * WARPS) {
        const GaucUser u = users[j];
        const uint64_t *pos = key + u.start, *neg = pos + u.P;
        bool nan = false;
        for (int32_t i = lane; i < u.P + u.N; i += 32) nan |= ord_nan((uint32_t)pos[i]);
        nan = __any_sync(FULL, nan);
        const int64_t pairs = (int64_t)u.P * u.N;
        float sum = 0.0f;
        if (pairs <= (1 << 24)) {
            long long c = 0;
            for (int32_t i = lane; i < u.P; i += 32) {
                const uint32_t p = (uint32_t)pos[i];
                int32_t lo = 0, hi = u.N;
                while (lo < hi) {
                    const int32_t mid = (int32_t)(((int64_t)lo + hi) >> 1);
                    if ((uint32_t)neg[mid] < p) lo = mid + 1;
                    else hi = mid;
                }
                c += lo;
            }
            for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(FULL, c, o);
            sum = (float)c;
        } else if (lane == 0) {
            int32_t below = 0;
            for (int32_t i = 0; i < u.P; i++) {
                while (below < u.N && (uint32_t)neg[below] < (uint32_t)pos[i]) below++;
                sum = __fadd_rn(sum, __int2float_rn(below));
            }
        }
        if (lane == 0) auc[j] = nan ? __int_as_float(0x7fffffff) : __fdiv_rn(sum, __ll2float_rn(pairs));
    }
}
