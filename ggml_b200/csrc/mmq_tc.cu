// mmq_tc.cu — batched quantized mat-mul (n > 8, and 5 <= n <= 8 where the mat-vec kernels cannot take the shape) on the Hopper
// tensor cores: the front end of the GEMM.  Converts the activations to fp16 (x_to_f16_kernel), owns the tensor-map encoder, and sends
// the shape to the warpgroup-MMA kernel (mmq_tc2.cu), directly for the formats with an operand decoder, through an fp16 copy of W for
// the others (launch_mmq_dense).
//
// Replaces the reference's mul_mat_q (src/ggml-cuda/mmq.cuh:2499-2655: int8 mma.sync tiles + stream-k fix-up) and its
// cuBLAS fallback (dequantize_block_* -> cublasGemmEx, src/ggml-cuda/ggml-cuda.cu:1158-1300); computes GGML_OP_MUL_MAT
// for block-quantized src0 and f32 src1 as ggml_compute_forward_mul_mat does (src/ggml-cpu/ggml-cpu.c:7428).
//
// Per-block scales cannot be interposed in an accumulation that runs over the whole K loop, so the scales are folded into the
// operand: W tiles are dequantized to fp16 in shared memory (K-major SWIZZLE_128B layout), X is converted to fp16 once (each
// activation row pre-scaled by a power of two when its largest magnitude would leave the fp16 range; the epilogue undoes the scale,
// so nothing overflows and the scaling is exact), D accumulates in f32.  fp16 is chosen over bf16 because integer codes convert to
// fp16 with two packed-half instructions per two weights and carry 11 instead of 8 significant bits.  NMSE against the CPU backend
// ~1e-7 .. 1e-6 (the reference's gate is 5e-4, tests/test-backend-ops.cpp:1915-1917).
#include "b200_internal.h"
#include "b200_quants.cuh"
#include "b200_tc_dequant.cuh"   // h2u
#include "b200_ptx.cuh"

#include <mutex>

namespace b200 {

// ----------------------------------------------------------------------------- X -> fp16 prologue
// one CTA per activation row: largest magnitude -> exact power-of-two scale that puts it into [2^13, 2^14) (neither overflow nor
// a row of fp16 subnormals, whatever the row's magnitude), then the conversion.  inv_scale[n] is applied to column n of the
// result in the GEMM epilogue.
__global__ void __launch_bounds__(256) x_to_f16_kernel(const float * __restrict__ x, size_t nb11, __half * __restrict__ xh, float * __restrict__ inv_scale, int64_t K) {
    // programmatic dependent launch (no-ops for a plain launch): the GEMM that follows may start its prologue and its weight stream
    // now; this kernel itself waits for its predecessor (which may have produced x, and may still be reading the fp16 buffer)
    pdl_launch_dependents();
    pdl_wait();
    const int64_t n = blockIdx.x;
    const float * xr = (const float *)((const uint8_t *)x + n * nb11);
    __shared__ float s_max[8];
    float amax = 0.0f;
    for (int64_t k = (int64_t)threadIdx.x * 8; k < K; k += 256 * 8) {
        const float4 a = load_f4(xr + k), b = load_f4(xr + k + 4);
        amax = fmaxf(amax, fmaxf(fmaxf(fmaxf(fabsf(a.x), fabsf(a.y)), fmaxf(fabsf(a.z), fabsf(a.w))), fmaxf(fmaxf(fabsf(b.x), fabsf(b.y)), fmaxf(fabsf(b.z), fabsf(b.w)))));
    }
    amax = warp_max(amax);
    if ((threadIdx.x & 31) == 0) s_max[threadIdx.x >> 5] = amax;
    __syncthreads();
    amax = s_max[0];
#pragma unroll
    for (int i = 1; i < 8; ++i) amax = fmaxf(amax, s_max[i]);
    // e = exponent(amax) - 13 (finite non-zero amax only; zero / inf / nan rows keep scale 1 and propagate), |e| <= 100
    int e = 0;
    if (amax > 0.0f && amax <= 3.0e38f) e = max(-100, min(100, (int)((__float_as_uint(amax) >> 23) & 0xFF) - 127 - 13));
    const float sc = __uint_as_float((uint32_t)(127 - e) << 23);            // 2^-e, exact
    if (threadIdx.x == 0) inv_scale[n] = __uint_as_float((uint32_t)(127 + e) << 23);
    for (int64_t k = (int64_t)threadIdx.x * 8; k < K; k += 256 * 8) {
        const float4 a = load_f4(xr + k), b = load_f4(xr + k + 4);
        __half2 h0 = __floats2half2_rn(a.x * sc, a.y * sc), h1 = __floats2half2_rn(a.z * sc, a.w * sc);
        __half2 h2 = __floats2half2_rn(b.x * sc, b.y * sc), h3 = __floats2half2_rn(b.z * sc, b.w * sc);
        uint4 o; o.x = h2u(h0); o.y = h2u(h1); o.z = h2u(h2); o.w = h2u(h3);
        *(uint4 *)(xh + n * K + k) = o;
    }
}

// ----------------------------------------------------------------------------- host side
int tc_launch_x_to_f16(const float * x, size_t nb11, __half * xh, float * inv_scale, int64_t K, int64_t N, cudaStream_t st) {
    B200_CUDA_TRY(launch_pdl(x_to_f16_kernel, dim3((unsigned)N), dim3(256), 0, st, x, nb11, xh, inv_scale, K));
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

encode_tiled_fn tc_get_encode() {
    static encode_tiled_fn fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void * p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess) fn = (encode_tiled_fn)p;
        else cudaGetLastError();
    });
    return fn;
}

bool mmq_tc_eligible(const ggml_b200_mul_mat_args & a) { return a.N >= 9 && (mmq_tc2_eligible(a) || mmq_dense_eligible(a)); }
bool mmq_tc_eligible_small(const ggml_b200_mul_mat_args & a) { return a.N >= 5 && mmq_tc2_eligible(a); }
size_t mmq_tc_workspace(const ggml_b200_mul_mat_args & a) {
    if (mmq_dense_eligible(a)) return mmq_dense_workspace(a);
    return mmq_tc2_workspace(a);
}

int launch_mmq_tc(const ggml_b200_mul_mat_args & a, cudaStream_t st) {
    if (mmq_dense_eligible(a)) return launch_mmq_dense(a, st);             // formats without an operand decoder: fp16 copy + the same GEMM
    if (mmq_tc2_eligible(a)) return launch_mmq_tc2(a, st);
    set_error("mul_mat: shape not eligible for the tensor-core kernel");
    return GGML_B200_EUNSUPPORTED;
}

} // namespace b200
