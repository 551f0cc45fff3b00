// als.cuh -- pieces of the eALS epoch that live in their own translation units.
#pragma once
#include <algorithm>

#include "cf.cuh"

namespace gb {

// floats between consecutive partial (G, h) blocks (d x d, then d), rounded up to a multiple of 4 so that every block is
// 16-byte aligned for float4 access: 16 512 at d = 128
constexpr __host__ __device__ inline int als_partial_stride(int d) { return (d * d + d + 3) & ~3; }

// als_thread.cu: one thread per row, rows with at most 4 entries, d in {32, 64, 96, 128}
int32_t als_thread_rows(gorse_b200_cf *cf, float *X, const float *Y, const int64_t *off, const int32_t *idx, float reg, float w,
                        const int32_t *rows, int32_t n_rows);

// als_gram_tc.cu: partial (G, h) of every chunk on the tensor cores (3xTF32), d = 128 only
int32_t als_chunk_gram_tc(gorse_b200_ctx *c, const float *Y, const int32_t *idx, const int64_t *chunk_begin, const int32_t *chunk_len,
                          int32_t n_chunks, float *partial);

}  // namespace gb
