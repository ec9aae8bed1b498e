// b200_internal.h — host-side plumbing shared by the kernel translation units (not part of the ABI).
#pragma once

#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <cstdio>

#include "../../include/ggml-b200.h"

namespace b200 {

extern std::atomic<uint64_t> g_launches;
void set_error(const char * fmt, ...);
int  sm_count();

// Per-device control block, zeroed once, in 4-byte words:
//   [0, 64)                    global control words of the mat-vec kernels
//   [64, 64 + 64 * 8)          64 per-launch scheduling slots of the mat-vec kernels (sb_next_slot)
//   [2048, 2048 + 64 * 256)    64 slots of 256 self-cleaning split-K flags of the GEMM (tc_flag_slot)
constexpr int CTL_SPLITK_FLAGS = 2048, TC_FLAG_SLOTS = 64, TC_FLAGS_PER_SLOT = 256;
unsigned int * control_block();   // nullptr on error (set_error called)

// Programmatic dependent launch: kernels launched through launch_pdl may become resident while their predecessor on the stream still
// runs; each one orders itself against it with griddepcontrol.wait.
template <typename... KArgs, typename... Args>
cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, const Args &... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}

// Raises Kernel's dynamic shared-memory limit to `bytes`.  The attribute is a per-device setting: it is set once per (kernel, device), so
// that a process that drives several GPUs through the backend (one ggml device per GPU) configures every one of them.  The flag is keyed
// on the kernel itself: instantiations that share a signature each need their own.
template <auto Kernel> cudaError_t set_max_dynamic_smem(int bytes) {
    static std::atomic<bool> done[64] = {};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) dev = 0;
    if (done[dev].load(std::memory_order_acquire)) return cudaSuccess;      // setting the attribute twice is harmless: no lock needed
    const cudaError_t e = cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e == cudaSuccess) done[dev].store(true, std::memory_order_release);
    return e;
}

#define B200_CUDA_TRY(...)   /* variadic: the expression may hold template-argument commas */                \
    do {                                                                                            \
        cudaError_t e_ = (__VA_ARGS__);                                                             \
        if (e_ != cudaSuccess) {                                                                    \
            ::b200::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #__VA_ARGS__, cudaGetErrorString(e_)); \
            return GGML_B200_ECUDA;                                                                 \
        }                                                                                           \
    } while (0)

#define B200_LAUNCH_CHECK()                                                                          \
    do {                                                                                            \
        ::b200::g_launches.fetch_add(1, std::memory_order_relaxed);                                 \
        B200_CUDA_TRY(cudaGetLastError());                                                          \
    } while (0)

// Kernel families: plan_X is true when family X can run the shape and fills the plan (types in b200_mm_plan.h); launch_X runs a plan
// plan_X made from the same arguments without planning again, and of the arguments checks only the workspace size.
struct tma_plan; struct sb_plan; struct mma_plan; struct tc2_plan; struct dense_plan; struct mmid_g_plan;

// mmvq.cu
int    launch_quantize_activations(int type, const float * x, int64_t K, int64_t n11, int64_t n12, int64_t n13,
                                   size_t nb11, size_t nb12, size_t nb13, void * recs, cudaStream_t st);
int    launch_mmvq_generic(const ggml_b200_mul_mat_args & a, cudaStream_t st);
size_t mmvq_generic_workspace(const ggml_b200_mul_mat_args & a);
bool   plan_tma(const ggml_b200_mul_mat_args & a, tma_plan & pl);
int    launch_tma(const ggml_b200_mul_mat_args & a, const tma_plan & pl, cudaStream_t st);
// mmvq_sb.cu (n = 1 bandwidth path)
bool   plan_sb(const ggml_b200_mul_mat_args & a, sb_plan & pl);
int    launch_sb(const ggml_b200_mul_mat_args & a, const sb_plan & pl, cudaStream_t st, const ggml_b200_gather * ga = nullptr, const ggml_b200_epilogue * ep = nullptr);
int    launch_gather_wait(const uint32_t * flags, int world, uint32_t epoch, cudaStream_t st);
unsigned int * sb_next_slot(unsigned int * ctl);   // the next of the 64 self-resetting scheduling slots
// bytes of W a dependent mat-vec launch (mmvq_sb and mmvq_mma) pulls into L2 ahead of its predecessor's output: 8 MB of the H100's 50 MB L2
// (scripts/gemv_sweep.py on an H100, sweeping the cap: q4_K n = 1 and n = 8 dependent launches 12-17 % faster than with 48 MB, within a few
// % of no prefetch)
constexpr int64_t L2_PREFETCH_CAP = (int64_t)8 << 20;

// mmvq_mma.cu (bandwidth path, int8 mma.sync consume phase: 2 <= n <= 8, n = 1 on request); workspace: the quantized activation records
bool   plan_mma(const ggml_b200_mul_mat_args & a, mma_plan & pl);
int    launch_mma(const ggml_b200_mul_mat_args & a, const mma_plan & pl, cudaStream_t st);

// mmq_tc2.cu (the wgmma GEMM kernel: quantized W with an operand decoder, n >= 5)
bool   plan_wgmma(const ggml_b200_mul_mat_args & a, tc2_plan & pl);
int    launch_wgmma(const ggml_b200_mul_mat_args & a, const tc2_plan & pl, cudaStream_t st);
bool   plan_dense(const ggml_b200_mul_mat_args & a, dense_plan & pl);   // n >= 9, formats without an operand decoder: dequantize to fp16 + the same GEMM
int    launch_dense(const ggml_b200_mul_mat_args & a, const dense_plan & pl, cudaStream_t st);
size_t mmq_f16w_workspace(int64_t M, int64_t N, int64_t K);         // dense fp16 weights, n >= 9 (0 = not eligible)
int    launch_mmq_f16w(const void * w, size_t nb01, const float * x, size_t nb11, float * y, int64_t M, int64_t N, int64_t K, void * ws, size_t ws_size, uint32_t flags, cudaStream_t st);
size_t mmq_f16f16_workspace(int64_t M, int64_t N, int64_t K);       // dense fp16 x fp16, n >= 9, K % 64 == 0 (0 = not eligible)
int    launch_mmq_f16f16(const void * w, size_t nb01, const void * x, size_t nb11, float * y, int64_t M, int64_t N, int64_t K, void * ws, size_t ws_size, uint32_t flags, cudaStream_t st);
// expert-grouped MUL_MAT_ID on the GEMM kernel (mmq_tc2.cu); the caller checks the workspace
bool   plan_mmid_grouped(const ggml_b200_mul_mat_id_args & a, mmid_g_plan & pl);
int    launch_mmid_grouped(const ggml_b200_mul_mat_id_args & a, const mmid_g_plan & pl, cudaStream_t st);

} // namespace b200
