// gmma_common.cuh -- the few Hopper (sm_90a) primitives the tensor-core pruning kernel needs, hand-written as
// inline PTX: shared-memory matrix descriptors, warpgroup MMAs (wgmma.mma_async, kind tf32, FP32 accumulators in
// registers), mbarriers, 1-D bulk async copies (TMA engine).
//
// Shared-memory operand layout used throughout (K-major, no swizzle; "INTERLEAVE" canonical form):
// a tile X[R rows][Kp floats] is stored as 8-row x 16-byte core matrices,
//     byte_offset(r, j) = (j/4) * (R/8)*128  +  (r/8) * 128  +  (r%8) * 16  +  (j%4) * 4
// i.e. consecutive 8-row groups are 128 B apart (SBO) and consecutive 16-byte K chunks are
// (R/8)*128 B apart (LBO).  One wgmma of kind tf32 consumes K = 8 floats = two chunks.
#pragma once
#include <stdint.h>
#include <cuda_runtime.h>

namespace gmma {

__device__ __forceinline__ uint32_t smem_u32 (const void *p)
{
    return (uint32_t) __cvta_generic_to_shared (p);
}

// byte offset of element (r, j) in the canonical K-major layout of a tile with R rows
__device__ __forceinline__ uint32_t canon_off (int r, int j, int R)
{
    return (uint32_t)((j >> 2) * (R >> 3) * 128 + (r >> 3) * 128 + (r & 7) * 16 + (j & 3) * 4);
}

// 64-bit wgmma shared-memory matrix descriptor: [0,14) start>>4, [16,30) leading byte offset>>4 (K direction),
// [32,46) stride byte offset>>4 (8-row groups), [49,52) base offset = 0, [62,64) layout type = 0 (no swizzle)
__device__ __forceinline__ uint64_t make_desc (uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes)
{
    uint64_t d = 0;
    d |= (uint64_t)((saddr >> 4) & 0x3fff);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3fff) << 16;
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3fff) << 32;
    return d;
}

// ---- warpgroup MMA: D[64 x N] (+)= A[64 x 8] * B[N x 8]^T, tf32 operands from shared memory, FP32 accumulators in
// registers.  Issued by all 128 threads of a warpgroup; thread t of warp w holds, for every 8-column block j,
// d[4j + i] = D[16 w + t/4 + 8 (i/2)][8 j + 2 (t%4) + i%2].
#define GMMA_F4(b) "+f"(d[(b)]), "+f"(d[(b) + 1]), "+f"(d[(b) + 2]), "+f"(d[(b) + 3])
#define GMMA_F16(b) GMMA_F4 (b), GMMA_F4 ((b) + 4), GMMA_F4 ((b) + 8), GMMA_F4 ((b) + 12)

template <int N> __device__ __forceinline__ void mma_tf32 (float *d, uint64_t desc_a, uint64_t desc_b, bool accumulate);

template <> __device__ __forceinline__ void mma_tf32<32> (float *d, uint64_t desc_a, uint64_t desc_b, bool accumulate)
{
    asm volatile (
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n\t}\n"
        : GMMA_F16 (0)
        : "l"(desc_a), "l"(desc_b), "r"(accumulate ? 1u : 0u) : "memory");
}

template <> __device__ __forceinline__ void mma_tf32<64> (float *d, uint64_t desc_a, uint64_t desc_b, bool accumulate)
{
    asm volatile (
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
        "%24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t}\n"
        : GMMA_F16 (0), GMMA_F16 (16)
        : "l"(desc_a), "l"(desc_b), "r"(accumulate ? 1u : 0u) : "memory");
}

template <> __device__ __forceinline__ void mma_tf32<128> (float *d, uint64_t desc_a, uint64_t desc_b, bool accumulate)
{
    asm volatile (
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
        "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, "
        "%47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}\n"
        : GMMA_F16 (0), GMMA_F16 (16), GMMA_F16 (32), GMMA_F16 (48)
        : "l"(desc_a), "l"(desc_b), "r"(accumulate ? 1u : 0u) : "memory");
}
#undef GMMA_F16
#undef GMMA_F4

// the accumulator registers are about to be handed to wgmma (orders earlier register accesses before it)
__device__ __forceinline__ void mma_fence () { asm volatile ("wgmma.fence.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void mma_commit () { asm volatile ("wgmma.commit_group.sync.aligned;\n" ::: "memory"); }
// wait until every committed group has completed: accumulators final, shared-memory operands read
__device__ __forceinline__ void mma_wait_all () { asm volatile ("wgmma.wait_group.sync.aligned 0;\n" ::: "memory"); }
// keep the compiler from moving accumulator accesses across the asynchronous MMAs
__device__ __forceinline__ void fence_regs (float &r) { asm volatile ("" : "+f"(r) :: "memory"); }

// generic-proxy writes to shared memory -> visible to the async proxy (wgmma, bulk copies)
__device__ __forceinline__ void fence_async_smem ()  { asm volatile ("fence.proxy.async.shared::cta;\n" ::: "memory"); }

// ---- mbarrier ----
__device__ __forceinline__ void mbar_init (uint64_t *bar, int count)
{
    asm volatile ("mbarrier.init.shared::cta.b64 [%0], %1;\n" :: "r"(smem_u32 (bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init () { asm volatile ("fence.mbarrier_init.release.cluster;\n" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx (uint64_t *bar, uint32_t bytes)
{
    asm volatile ("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" :: "r"(smem_u32 (bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive (uint64_t *bar)
{
    asm volatile ("mbarrier.arrive.shared::cta.b64 _, [%0];\n" :: "r"(smem_u32 (bar)) : "memory");
}

// ---- 1-D bulk async copies (TMA engine; no tensor map needed for contiguous tiles) ----
__device__ __forceinline__ void bulk_g2s (void *smem_dst, const void *gsrc, uint32_t bytes, uint64_t *bar)
{
    asm volatile ("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n"
                  :: "r"(smem_u32 (smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32 (bar)) : "memory");
}

// round-to-nearest TF32 (10-bit mantissa) of an fp32 value, returned as fp32 bits
__device__ __forceinline__ float to_tf32 (float x)
{
    uint32_t r;
    asm ("cvt.rna.tf32.f32 %0, %1;\n" : "=r"(r) : "f"(x));
    return __uint_as_float (r);
}

} // namespace gmma
