// ctx.cu -- context: one GPU, one stream, optional NCCL rank; measurement hooks.
#include <dlfcn.h>

#include <cstdlib>

#include "common.cuh"

namespace gb {

static thread_local char g_err[1024] = "";

void set_error(const char *fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

const NcclApi *nccl()
{
    static std::mutex mu;
    static NcclApi api;
    static bool ok = false;
    std::lock_guard<std::mutex> lk(mu);
    if (ok) return &api;
    const char *env = getenv("GORSE_B200_NCCL_LIB");
    const char *names[] = {env, "libnccl.so.2", "libnccl.so"};
    void *h = nullptr;
    for (const char *n : names) {
        if (!n || !*n) continue;
        if ((h = dlopen(n, RTLD_NOW | RTLD_LOCAL))) break;
    }
    if (!h) {
        set_error("cannot load libnccl.so.2 (set GORSE_B200_NCCL_LIB): %s", dlerror());
        return nullptr;
    }
    api.GetUniqueId = (decltype(api.GetUniqueId))dlsym(h, "ncclGetUniqueId");
    api.CommInitRank = (decltype(api.CommInitRank))dlsym(h, "ncclCommInitRank");
    api.CommDestroy = (decltype(api.CommDestroy))dlsym(h, "ncclCommDestroy");
    api.AllReduce = (decltype(api.AllReduce))dlsym(h, "ncclAllReduce");
    api.AllGather = (decltype(api.AllGather))dlsym(h, "ncclAllGather");
    api.GetErrorString = (decltype(api.GetErrorString))dlsym(h, "ncclGetErrorString");
    api.Broadcast = (decltype(api.Broadcast))dlsym(h, "ncclBroadcast");
    api.GroupStart = (decltype(api.GroupStart))dlsym(h, "ncclGroupStart");
    api.GroupEnd = (decltype(api.GroupEnd))dlsym(h, "ncclGroupEnd");
    if (!api.GetUniqueId || !api.CommInitRank || !api.CommDestroy || !api.AllReduce || !api.AllGather || !api.GetErrorString) {
        set_error("libnccl is missing a required symbol");
        return nullptr;
    }
    ok = true;
    return &api;
}

__global__ void flush_kernel(float4 *buf, size_t n4, float v)
{
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t stride = (size_t)gridDim.x * blockDim.x;
    for (; i < n4; i += stride) buf[i] = make_float4(v, v, v, v);
}

}  // namespace gb

extern "C" {

int32_t gorse_b200_version(void) { return GORSE_B200_ABI_VERSION; }

const char *gorse_b200_last_error(void) { return gb::g_err; }

int32_t gorse_b200_device_count(int32_t *count)
{
    GB_CHECK_ARG(count != nullptr, "count is NULL");
    int n = 0;
    GB_CUDA(cudaGetDeviceCount(&n));
    *count = n;
    return GORSE_B200_OK;
}

static int32_t ctx_create_common(int32_t device, gorse_b200_ctx **out)
{
    GB_CHECK_ARG(out != nullptr, "out is NULL");
    *out = nullptr;
    int n = 0;
    GB_CUDA(cudaGetDeviceCount(&n));
    GB_CHECK_ARG(device >= 0 && device < n, "device %d out of range (%d devices)", device, n);
    GB_CUDA(cudaSetDevice(device));
    cudaDeviceProp prop;
    GB_CUDA(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) {
        gb::set_error("device %d is sm_%d%d; this library is built for sm_90a (H100) only", device, prop.major,
                      prop.minor);
        return GORSE_B200_ERR_UNSUPPORTED;
    }
    gorse_b200_ctx *c = new (std::nothrow) gorse_b200_ctx();
    if (!c) {
        gb::set_error("host allocation failed");
        return GORSE_B200_ERR_OOM;
    }
    c->device = device;
    c->sm_count = prop.multiProcessorCount;
    GB_CUDA(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
    GB_CUDA(cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking));
    GB_CUDA(cudaEventCreateWithFlags(&c->copy_ev, cudaEventDisableTiming));
    GB_CUDA(cudaEventCreate(&c->ev0));
    GB_CUDA(cudaEventCreate(&c->ev1));
    *out = c;
    return GORSE_B200_OK;
}

int32_t gorse_b200_ctx_create(int32_t device, gorse_b200_ctx **out) { return ctx_create_common(device, out); }

int32_t gorse_b200_nccl_unique_id(void *id_out)
{
    GB_CHECK_ARG(id_out != nullptr, "id_out is NULL");
    static_assert(sizeof(ncclUniqueId) <= GORSE_B200_NCCL_ID_BYTES, "nccl id size");
    GB_NCCL_API(nc);
    ncclUniqueId id;
    GB_NCCL(nc, GetUniqueId(&id));
    memset(id_out, 0, GORSE_B200_NCCL_ID_BYTES);
    memcpy(id_out, &id, sizeof(id));
    return GORSE_B200_OK;
}

int32_t gorse_b200_ctx_create_dist(int32_t device, int32_t rank, int32_t world, const void *nccl_id,
                                   gorse_b200_ctx **out)
{
    GB_CHECK_ARG(world >= 1 && rank >= 0 && rank < world, "bad rank %d / world %d", rank, world);
    GB_CHECK_ARG(world == 1 || nccl_id != nullptr, "nccl_id is NULL");
    GB_TRY(ctx_create_common(device, out));
    gorse_b200_ctx *c = *out;
    c->rank = rank;
    c->world = world;
    if (world > 1) {
        GB_NCCL_API(nc);
        ncclUniqueId id;
        memcpy(&id, nccl_id, sizeof(id));
        GB_NCCL(nc, CommInitRank(&c->comm, world, id, rank));
        GB_TRY(c->nccl_token.alloc(1));
        GB_CUDA(cudaMemsetAsync(c->nccl_token.p, 0, sizeof(int), c->stream));
    }
    return GORSE_B200_OK;
}

int32_t gorse_b200_ctx_destroy(gorse_b200_ctx *ctx)
{
    if (!ctx) return GORSE_B200_OK;
    gb::ScopedDevice sd(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    if (ctx->comm && gb::nccl()) gb::nccl()->CommDestroy(ctx->comm);
    gb::recommend_work_free(ctx);
    cudaEventDestroy(ctx->ev0);
    cudaEventDestroy(ctx->ev1);
    cudaStreamDestroy(ctx->stream);
    if (ctx->copy_stream) cudaStreamDestroy(ctx->copy_stream);
    if (ctx->copy_ev) cudaEventDestroy(ctx->copy_ev);
    delete ctx;
    return GORSE_B200_OK;
}

int32_t gorse_b200_ctx_sync(gorse_b200_ctx *ctx)
{
    GB_CHECK_ARG(ctx != nullptr, "ctx is NULL");
    gb::ScopedDevice sd(ctx->device);
    GB_CUDA(cudaStreamSynchronize(ctx->stream));
    return GORSE_B200_OK;
}

int32_t gorse_b200_ctx_rank(const gorse_b200_ctx *ctx, int32_t *rank, int32_t *world)
{
    GB_CHECK_ARG(ctx != nullptr, "ctx is NULL");
    if (rank) *rank = ctx->rank;
    if (world) *world = ctx->world;
    return GORSE_B200_OK;
}

int32_t gorse_b200_ctx_timer_begin(gorse_b200_ctx *ctx)
{
    GB_CHECK_ARG(ctx != nullptr, "ctx is NULL");
    gb::ScopedDevice sd(ctx->device);
    GB_CUDA(cudaEventRecord(ctx->ev0, ctx->stream));
    return GORSE_B200_OK;
}

int32_t gorse_b200_ctx_timer_end(gorse_b200_ctx *ctx, float *ms_out)
{
    GB_CHECK_ARG(ctx != nullptr && ms_out != nullptr, "NULL argument");
    gb::ScopedDevice sd(ctx->device);
    GB_CUDA(cudaEventRecord(ctx->ev1, ctx->stream));
    GB_CUDA(cudaEventSynchronize(ctx->ev1));
    GB_CUDA(cudaEventElapsedTime(ms_out, ctx->ev0, ctx->ev1));
    return GORSE_B200_OK;
}

int32_t gorse_b200_ctx_launch_count(const gorse_b200_ctx *ctx, int64_t *count)
{
    GB_CHECK_ARG(ctx != nullptr && count != nullptr, "NULL argument");
    *count = ctx->launches;
    return GORSE_B200_OK;
}

int32_t gorse_b200_device_bytes(int64_t *bytes)
{
    GB_CHECK_ARG(bytes != nullptr, "bytes is NULL");
    *bytes = gb::g_device_bytes.load();
    return GORSE_B200_OK;
}

int32_t gorse_b200_ctx_flush_l2(gorse_b200_ctx *ctx)
{
    GB_CHECK_ARG(ctx != nullptr, "ctx is NULL");
    gb::ScopedDevice sd(ctx->device);
    if (!ctx->flush_buf.p) GB_TRY(ctx->flush_buf.alloc(((size_t)256 << 20) / sizeof(float4)));  // 5x the 50 MB L2
    gb::flush_kernel<<<ctx->sm_count * 4, 256, 0, ctx->stream>>>(ctx->flush_buf.p, ctx->flush_buf.n, (float)(ctx->launches & 7));
    GB_CUDA(cudaGetLastError());  // not counted: measurement hygiene, not the hot path
    return GORSE_B200_OK;
}

int32_t gorse_b200_host_alloc(size_t bytes, void **out)
{
    GB_CHECK_ARG(out != nullptr, "out is NULL");
    *out = nullptr;
    if (bytes == 0) return GORSE_B200_OK;
    GB_CUDA(cudaHostAlloc(out, bytes, cudaHostAllocPortable));
    return GORSE_B200_OK;
}

int32_t gorse_b200_host_free(void *p)
{
    if (p) GB_CUDA(cudaFreeHost(p));
    return GORSE_B200_OK;
}

int32_t gorse_b200_ctx_barrier(gorse_b200_ctx *ctx)
{
    GB_CHECK_ARG(ctx != nullptr, "ctx is NULL");
    gb::ScopedDevice sd(ctx->device);
    if (ctx->world > 1) {
        GB_NCCL_API(nc);
        GB_NCCL(nc, AllReduce(ctx->nccl_token.p, ctx->nccl_token.p, 1, ncclInt32, ncclSum, ctx->comm, ctx->stream));
    }
    GB_CUDA(cudaStreamSynchronize(ctx->stream));
    return GORSE_B200_OK;
}

}  // extern "C"
