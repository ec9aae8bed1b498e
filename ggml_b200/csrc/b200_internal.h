// b200_internal.h — host-side plumbing shared by the kernel translation units (not part of the ABI).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <cstdio>

#include "../../include/ggml-b200.h"

namespace b200 {

extern std::atomic<uint64_t> g_launches;
void set_error(const char * fmt, ...);
int  sm_count();

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) is a per-device setting: remember it per (kernel instantiation, device), so that a
// process that drives several GPUs through the backend (one ggml device per GPU) configures every one of them.
struct per_device_flag {
    std::atomic<bool> done[64] = {};
    static int dev() { int d = 0; if (cudaGetDevice(&d) != cudaSuccess || d < 0 || d >= 64) d = 0; return d; }
    bool test() const { return done[dev()].load(std::memory_order_acquire); }      // setting the attribute twice is harmless: no lock needed
    void set() { done[dev()].store(true, std::memory_order_release); }
};

#define B200_CUDA_TRY(expr)                                                                         \
    do {                                                                                            \
        cudaError_t e_ = (expr);                                                                    \
        if (e_ != cudaSuccess) {                                                                    \
            ::b200::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(e_)); \
            return GGML_B200_ECUDA;                                                                 \
        }                                                                                           \
    } while (0)

#define B200_LAUNCH_CHECK()                                                                          \
    do {                                                                                            \
        ::b200::g_launches.fetch_add(1, std::memory_order_relaxed);                                 \
        B200_CUDA_TRY(cudaGetLastError());                                                          \
    } while (0)

// mmvq.cu
int    launch_quantize_activations(int type, const float * x, int64_t K, int64_t n11, int64_t n12, int64_t n13,
                                   size_t nb11, size_t nb12, size_t nb13, void * recs, cudaStream_t st);
int    launch_mmvq_generic(const ggml_b200_mul_mat_args & a, cudaStream_t st);
bool   mmvq_tma_eligible(const ggml_b200_mul_mat_args & a);
int    launch_mmvq_tma(const ggml_b200_mul_mat_args & a, cudaStream_t st);
size_t mmvq_generic_workspace(const ggml_b200_mul_mat_args & a);
// mmvq_sb.cu (n = 1 bandwidth path)
bool   mmvq_sb_eligible(const ggml_b200_mul_mat_args & a);
int    launch_mmvq_sb(const ggml_b200_mul_mat_args & a, cudaStream_t st, const ggml_b200_gather * ga = nullptr, const ggml_b200_epilogue * ep = nullptr);
int    debug_read_trace(unsigned long long * out);
int    prepare_device();   // allocate the per-device control block (never inside a stream capture)
int    launch_gather_wait(const uint32_t * flags, int world, uint32_t epoch, cudaStream_t st);

// mmvq_mma.cu (bandwidth path, int8 mma.sync consume phase: 2 <= n <= 8, n = 1 on request)
bool   mmvq_mma_eligible(const ggml_b200_mul_mat_args & a);
int    launch_mmvq_mma(const ggml_b200_mul_mat_args & a, cudaStream_t st);
size_t mmvq_mma_workspace(const ggml_b200_mul_mat_args & a);   // the quantized activation records (written by the pre-kernel)

// mmq_tc.cu (tensor-core GEMM front end: activation conversion, dispatch)
bool   mmq_tc_eligible(const ggml_b200_mul_mat_args & a);
size_t mmq_tc_workspace(const ggml_b200_mul_mat_args & a);
bool   mmq_dense_eligible(const ggml_b200_mul_mat_args & a);   // n >= 9, formats without an operand decoder: dequantize to fp16 + the same GEMM (mmq_tc2.cu)
size_t mmq_dense_workspace(const ggml_b200_mul_mat_args & a);
int    launch_mmq_dense(const ggml_b200_mul_mat_args & a, cudaStream_t st);
size_t mmq_f16w_workspace(int64_t M, int64_t N, int64_t K);         // dense fp16 weights, n >= 9 (0 = not eligible)
int    launch_mmq_f16w(const void * w, size_t nb01, const float * x, size_t nb11, float * y, int64_t M, int64_t N, int64_t K, void * ws, size_t ws_size, uint32_t flags, cudaStream_t st);
bool   mmq_tc_eligible_small(const ggml_b200_mul_mat_args & a);   // 5 <= n <= 8 on the tensor-core path (shapes the mat-vec kernel would have to split)
int    launch_mmq_tc(const ggml_b200_mul_mat_args & a, cudaStream_t st);
// mmq_tc2.cu (the wgmma GEMM kernel)
bool   mmq_tc2_eligible(const ggml_b200_mul_mat_args & a);
size_t mmq_tc2_workspace(const ggml_b200_mul_mat_args & a);
int    launch_mmq_tc2(const ggml_b200_mul_mat_args & a, cudaStream_t st);
// expert-grouped MUL_MAT_ID on the GEMM kernel (mmq_tc2.cu)
bool   mmid_grouped_eligible(const ggml_b200_mul_mat_id_args & a);
size_t mmid_grouped_workspace(const ggml_b200_mul_mat_id_args & a);
int    launch_mmid_grouped(const ggml_b200_mul_mat_id_args & a, cudaStream_t st);
unsigned int * tc_flag_slot();   // a zeroed, self-cleaning block of split-K flags from the device's control block (nullptr on error)
int    tc_prepare_device();
int tc2_trace_read(unsigned long long * host_dst, int max_ctas);   // GEMM stamp trace: none is recorded (returns 0)

} // namespace b200
