// common.cuh -- shared plumbing of libgorse_b200.so (error handling, context, device buffers).
// sm_90a only; no CPU fallback anywhere: every entry point needs a CUDA device.
#pragma once
#include <cuda_runtime.h>
#include <nccl.h>

#include <algorithm>
#include <atomic>
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <new>
#include <string>
#include <type_traits>
#include <utility>
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

namespace gb {

// device bytes held by every DevBuf of the process (gorse_b200_device_bytes)
inline std::atomic<int64_t> g_device_bytes{0};

// owning device buffer: the destructor frees; moves leave the source empty, copies do not compile
template <typename T>
struct DevBuf {
    T *p = nullptr;
    size_t n = 0;
    DevBuf() = default;
    DevBuf(const DevBuf &) = delete;
    DevBuf &operator=(const DevBuf &) = delete;
    DevBuf(DevBuf &&o) noexcept : p(o.p), n(o.n)
    {
        o.p = nullptr;
        o.n = 0;
    }
    DevBuf &operator=(DevBuf &&o) noexcept
    {
        if (this != &o) {
            free();
            std::swap(p, o.p);
            std::swap(n, o.n);
        }
        return *this;
    }
    ~DevBuf() { free(); }
    int32_t alloc(size_t count)
    {
        free();
        if (count == 0) return GORSE_B200_OK;
        GB_CUDA(cudaMalloc((void **)&p, count * sizeof(T)));
        n = count;   // only a successful allocation has a size
        g_device_bytes += (int64_t)bytes();
        return GORSE_B200_OK;
    }
    void free()
    {
        if (p) {
            cudaFree(p);
            g_device_bytes -= (int64_t)bytes();
        }
        p = nullptr;
        n = 0;
    }
    // grow-only: reallocates (contents lost) when count exceeds the size
    int32_t grow(size_t count) { return n >= count ? GORSE_B200_OK : alloc(count); }
    // as grow; a new allocation is zeroed on stream s
    int32_t grow_zeroed(size_t count, cudaStream_t s)
    {
        if (n >= count) return GORSE_B200_OK;
        GB_TRY(alloc(count));
        GB_CUDA(cudaMemsetAsync(p, 0, sizeof(T) * count, s));
        return GORSE_B200_OK;
    }
    // grows to max(count, 1) and copies h[0, count) on stream s
    int32_t upload(const T *h, size_t count, cudaStream_t s)
    {
        GB_TRY(grow(std::max<size_t>(count, 1)));
        if (count) GB_CUDA(cudaMemcpyAsync(p, h, count * sizeof(T), cudaMemcpyHostToDevice, s));
        return GORSE_B200_OK;
    }
    size_t bytes() const { return n * sizeof(T); }
};
static_assert(!std::is_copy_constructible<DevBuf<int>>::value && !std::is_copy_assignable<DevBuf<int>>::value, "DevBuf owns its memory");
static_assert(std::is_nothrow_move_constructible<DevBuf<int>>::value, "std::vector<DevBuf> moves on growth");

// owning pinned host buffer (cudaHostAlloc), allocated once: the destructor frees; host memory, so not counted in
// g_device_bytes
template <typename T>
struct PinnedBuf {
    T *p = nullptr;
    PinnedBuf() = default;
    PinnedBuf(const PinnedBuf &) = delete;
    PinnedBuf &operator=(const PinnedBuf &) = delete;
    ~PinnedBuf()
    {
        if (p) cudaFreeHost(p);
    }
    int32_t alloc(size_t count)
    {
        GB_CUDA(cudaHostAlloc((void **)&p, count * sizeof(T), cudaHostAllocDefault));
        return GORSE_B200_OK;
    }
};

// synchronises its streams when destroyed: declare it after the buffers the enqueued work reads, so it is destroyed first
struct StreamSync {
    cudaStream_t a, b = nullptr;
    ~StreamSync()
    {
        cudaStreamSynchronize(a);
        if (b) cudaStreamSynchronize(b);
    }
};

// an owning CUDA event, without timing unless create() is asked for it; declare it before the StreamSync that waits for the
// work it records
struct Event {
    cudaEvent_t e = nullptr;
    Event() = default;
    Event(const Event &) = delete;
    Event &operator=(const Event &) = delete;
    ~Event()
    {
        if (e) cudaEventDestroy(e);
    }
    int32_t create(unsigned flags = cudaEventDisableTiming)
    {
        GB_CUDA(cudaEventCreateWithFlags(&e, flags));
        return GORSE_B200_OK;
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

namespace rec {
struct Work;
}  // namespace rec

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
    gb::DevBuf<float4> flush_buf;
    gb::DevBuf<int> nccl_token;
    gb::rec::Work *rec_work = nullptr;   // gorse_b200_recommend's grow-only device buffers (recommend.cu)
};

namespace gb {
void recommend_work_free(gorse_b200_ctx *ctx);   // deletes ctx->rec_work (recommend.cu)

inline int div_up(int64_t a, int64_t b) { return (int)((a + b - 1) / b); }

}  // namespace gb
