// b200_tc_ptx.cuh — inline-PTX building blocks of the tensor-core GEMM (mmq_tc2.cu, sm_90a): mbarrier, TMA tensor copies,
// warpgroup MMA (wgmma) issue / commit / wait and its shared-memory descriptors, programmatic dependent launch.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <stdint.h>

namespace b200 {

__device__ __forceinline__ uint32_t tc_smem(const void * p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void tc_mbar_init(uint64_t * b, uint32_t c) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(tc_smem(b)), "r"(c) : "memory"); }
__device__ __forceinline__ void tc_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void tc_expect_tx(uint64_t * b, uint32_t bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(tc_smem(b)), "r"(bytes) : "memory"); }
__device__ __forceinline__ void tc_arrive(uint64_t * b) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(tc_smem(b)) : "memory"); }
__device__ __forceinline__ void tc_wait(uint64_t * b, uint32_t parity) {
    asm volatile(
        "{\n.reg .pred p;\nTC_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra TC_DONE;\nbra TC_WAIT;\nTC_DONE:\n}\n" ::"r"(tc_smem(b)), "r"(parity) : "memory");
}
__device__ __forceinline__ void tc_tma_2d(void * dst, const CUtensorMap * map, int c0, int c1, uint64_t * bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                 ::"r"(tc_smem(dst)), "l"(map), "r"(tc_smem(bar)), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tc_prefetch_map(const CUtensorMap * map) { asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory"); }
// generic-proxy stores to shared memory -> visible to the async proxy (the wgmma operand reads)
__device__ __forceinline__ void tc_fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- warpgroup MMA (all 128 threads of a warpgroup execute these together)
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across an asynchronous wgmma
__device__ __forceinline__ void wg_fence_operand(float & r) { asm volatile("" : "+f"(r)::"memory"); }
// D[64 x 64] (f32, registers) += A[64 x 16] . B[64 x 16]^T, A and B fp16 K-major in shared memory
__device__ __forceinline__ void wg_mma_m64n64k16(float (&d)[32], uint64_t adesc, uint64_t bdesc) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
        "%32, %33, p, 1, 1, 0, 0;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]),
          "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]),
          "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(adesc), "l"(bdesc), "r"(1));
}
// wgmma shared-memory descriptor: K-major, SWIZZLE_128B (128-byte rows, 8-row groups 1024 B apart; layout type 1 at bit 62)
__device__ __forceinline__ uint64_t tc_smem_desc(uint32_t saddr) {
    return (uint64_t)((saddr & 0x3FFFF) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}
__device__ __forceinline__ void tc_pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void tc_pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// host side (defined in mmq_tc.cu)
typedef CUresult (*encode_tiled_fn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *, const cuuint32_t *,
                                    const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
encode_tiled_fn tc_get_encode();
// activations f32 -> fp16 rows with an exact power-of-two scale per row (inv_scale[n] undoes it in the epilogue)
int tc_launch_x_to_f16(const float * x, size_t nb11, __half * xh, float * inv_scale, int64_t K, int64_t N, cudaStream_t st, bool pdl);

} // namespace b200
