// wgmma.cuh -- the few PTX wrappers the Hopper tensor-core kernels share (topk_mma.cu: bf16 candidate sweep; als_gram_tc.cu:
// 3xTF32 row Grams): mbarriers, TMA tile loads, shared-memory matrix descriptors, warpgroup MMA issue / commit / wait.
// Descriptor bit layout as in the PTX ISA, "Matrix Descriptor Format" of wgmma (sm_90a).
#pragma once
#include <cuda.h>

#include <cstdint>

namespace gb {
namespace mma {

__device__ __forceinline__ uint32_t s32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(s32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(s32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(s32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity)
{
    uint32_t done = 0;
    while (!done) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(s32(bar)), "r"(parity)
            : "memory");
    }
}
// the same wait for a warp that is not on the critical path of the SM's issue slots (the TMA producer): back off between polls
__device__ __forceinline__ void mbar_wait_backoff(uint64_t *bar, uint32_t parity)
{
    uint32_t done = 0;
    for (;;) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(s32(bar)), "r"(parity)
            : "memory");
        if (done) break;
        __nanosleep(40);
    }
}
__device__ __forceinline__ void tma_load_2d(void *dst, const CUtensorMap *map, int x, int y, uint64_t *bar)
{
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(s32(dst)),
                 "l"(map), "r"(s32(bar)), "r"(x), "r"(y)
                 : "memory");
}
// one lane of a converged warp (elect.sync)
__device__ __forceinline__ bool elect_one()
{
    uint32_t pred;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "elect.sync _|p, 0xffffffff;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(pred));
    return pred != 0;
}

// K-major operand in the 128-byte swizzle: rows of 128 bytes (the TMA box / the writer applies the swizzle: 16-byte chunk
// index ^= row % 8), 8-row groups SBO = 1024 bytes apart, LBO unused for this layout (1), layout type 1 = SWIZZLE_128B in
// bits 62-63.  The tile must start 1024-byte aligned; a K step inside the 128-byte row is a plain start-address advance.
__device__ __forceinline__ uint64_t wgmma_desc(uint32_t smem_addr)
{
    return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | (1ull << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait()
{
    asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}

#define GB_WGMMA_D64                                                                                                       \
    "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),  \
        "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), \
        "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), \
        "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), \
        "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), \
        "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), \
        "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
#define GB_WGMMA_REGS64                                                                    \
    "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "              \
    "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "     \
    "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "     \
    "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}"

// D[64 x 128] (fp32, registers) (+)= A[64 x 16] * B[128 x 16]^T, bf16, both operands K-major in shared memory.
// Accumulator fragment: thread t of the warpgroup holds rows 16 (t / 32) + (t % 32) / 4 (+ 8), columns 8 j + 2 (t % 4) + {0, 1}
// in d[4 j + {0, 1}] (+ 8 rows: d[4 j + {2, 3}]).
__device__ __forceinline__ void wgmma_m64n128k16_bf16(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 " GB_WGMMA_REGS64 ", %64, %65, p, 1, 1, 0, 0;\n\t}"
        : GB_WGMMA_D64
        : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
// the same shape with K = 8 tf32 operands (both K-major: the only layout wgmma takes for 32-bit operands)
__device__ __forceinline__ void wgmma_m64n128k8_tf32(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 " GB_WGMMA_REGS64 ", %64, %65, p, 1, 1;\n\t}"
        : GB_WGMMA_D64
        : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
#undef GB_WGMMA_REGS64
#undef GB_WGMMA_D64

}  // namespace mma
}  // namespace gb
