// common.cuh -- shared plumbing of libgorse_b200.so (error handling, context, device buffers).
// sm_90a only; no CPU fallback anywhere: every entry point needs a CUDA device.
#pragma once
#include <cuda_runtime.h>
#include <nccl.h>

#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <new>
#include <string>
#include <vector>

#include "../../include/gorse_b200.h"

namespace gb {

void set_error(const char *fmt, ...);

#define GB_CHECK_ARG(cond, ...)                 \
    do {                                        \
        if (!(cond)) {                          \
            gb::set_error(__VA_ARGS__);         \
            return GORSE_B200_ERR_ARG;          \
        }                                       \
    } while (0)

#define GB_CUDA(call)                                                                            \
    do {                                                                                         \
        cudaError_t e_ = (call);                                                                 \
        if (e_ != cudaSuccess) {                                                                 \
            gb::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(e_)); \
            return e_ == cudaErrorMemoryAllocation ? GORSE_B200_ERR_OOM : GORSE_B200_ERR_CUDA;   \
        }                                                                                        \
    } while (0)

// NCCL is bound lazily with dlopen (libnccl.so.2): the library carries no link-time NCCL dependency, so a
// host process that brings its own NCCL (PyTorch bundles a newer one under the same soname) keeps it.
struct NcclApi {
    ncclResult_t (*GetUniqueId)(ncclUniqueId *);
    ncclResult_t (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int);
    ncclResult_t (*CommDestroy)(ncclComm_t);
    ncclResult_t (*AllReduce)(const void *, void *, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t);
    ncclResult_t (*AllGather)(const void *, void *, size_t, ncclDataType_t, ncclComm_t, cudaStream_t);
    const char *(*GetErrorString)(ncclResult_t);
    // optional (only the multi-rank eALS epoch uses them; nullptr when the loaded libnccl lacks them)
    ncclResult_t (*Broadcast)(const void *, void *, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t);
    ncclResult_t (*GroupStart)();
    ncclResult_t (*GroupEnd)();
};
const NcclApi *nccl();  // nullptr (and last_error set) when libnccl cannot be loaded

#define GB_NCCL_API(var)                              \
    const gb::NcclApi *var = gb::nccl();              \
    if (!var) return GORSE_B200_ERR_NCCL

#define GB_NCCL(api, call)                                                                            \
    do {                                                                                              \
        ncclResult_t r_ = (api)->call;                                                                \
        if (r_ != ncclSuccess) {                                                                      \
            gb::set_error("%s:%d: nccl%s -> %s", __FILE__, __LINE__, #call, (api)->GetErrorString(r_)); \
            return GORSE_B200_ERR_NCCL;                                                               \
        }                                                                                             \
    } while (0)

#define GB_TRY(call)                 \
    do {                             \
        int32_t s_ = (call);         \
        if (s_ != GORSE_B200_OK) return s_; \
    } while (0)

// check the launch that was just issued and count it
#define GB_LAUNCHED(ctx)                      \
    do {                                      \
        (ctx)->launches++;                    \
        GB_CUDA(cudaGetLastError());          \
    } while (0)

}  // namespace gb

struct gorse_b200_ctx {
    int device = 0;
    int sm_count = 132;
    int rank = 0, world = 1;
    cudaStream_t stream = nullptr;
    cudaStream_t copy_stream = nullptr;   // result downloads that overlap the next chunk's kernels (topk)
    cudaEvent_t copy_ev = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    ncclComm_t comm = nullptr;
    int64_t launches = 0;
    void *flush_buf = nullptr;
    size_t flush_bytes = 0;
    int *nccl_token = nullptr;
};

namespace gb {

// RAII-less device buffer (explicit free; objects live behind opaque handles)
template <typename T>
struct DevBuf {
    T *p = nullptr;
    size_t n = 0;
    int32_t alloc(size_t count)
    {
        free();
        if (count == 0) return GORSE_B200_OK;
        GB_CUDA(cudaMalloc((void **)&p, count * sizeof(T)));
        n = count;   // only a successful allocation has a size
        return GORSE_B200_OK;
    }
    void free()
    {
        if (p) cudaFree(p);
        p = nullptr;
        n = 0;
    }
};

struct ScopedDevice {
    int prev = -1;
    bool ok = true;
    explicit ScopedDevice(int dev)
    {
        if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
        if (prev != dev) ok = cudaSetDevice(dev) == cudaSuccess;
    }
    ~ScopedDevice()
    {
        if (prev >= 0) cudaSetDevice(prev);
    }
};

inline int div_up(int64_t a, int64_t b) { return (int)((a + b - 1) / b); }

}  // namespace gb
