// dequant.cu — bit-exact block-format conversion kernels for sm_90a.
//
// Replaces the reference's dequantize_block_* family (src/ggml-cuda/convert.cu:6-278, built there with
// -use_fast_math) by kernels whose every output is bit-identical to the CPU reference
// dequantize_row_q4_0 / q8_0 / q4_K / q5_K / q6_K (src/ggml-quants.c:255-273, 349-363, 1280-1302, 1482-1507,
// 1690-1719) and quantize_row_q4_0_ref / q8_0_ref (:31-66, :194-217): multiplies and subtracts are issued
// as separately rounded __fmul_rn / __fsub_rn (the reference's ggml-base is compiled without FMA).
// Each thread produces 4 consecutive outputs, so stores are coalesced 16-byte vectors.
#include "b200_internal.h"
#include "b200_quants.cuh"
#include "b200_dequant.cuh"

namespace b200 {

template <typename OUT> __device__ __forceinline__ void store4(OUT * dst, float a, float b, float c, float d);
template <> __device__ __forceinline__ void store4<float>(float * dst, float a, float b, float c, float d) {
    *(float4 *)dst = make_float4(a, b, c, d);
}
template <> __device__ __forceinline__ void store4<__half>(__half * dst, float a, float b, float c, float d) {
    __half2 lo = __halves2half2(__float2half_rn(a), __float2half_rn(b)), hi = __halves2half2(__float2half_rn(c), __float2half_rn(d));
    uint2 v; v.x = *(uint32_t *)&lo; v.y = *(uint32_t *)&hi;
    *(uint2 *)dst = v;
}

// one thread -> elements [4*t, 4*t+4) of the flat tensor
template <int T, typename OUT>
__global__ void __launch_bounds__(256) dequantize_kernel(const uint8_t * __restrict__ src, OUT * __restrict__ dst, int64_t n4) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n4) return;
    const int64_t e = t * 4;
    float o[4];
    dequant4<T>(src, e, o);
    store4<OUT>(dst + e, o[0], o[1], o[2], o[3]);
}

template <typename OUT> static int dequantize_dispatch(int type, const void * src, OUT * dst, int64_t n, cudaStream_t st) {
    const int64_t n4 = n / 4;
    const unsigned grid = (unsigned)((n4 + 255) / 256);
    const uint8_t * s = (const uint8_t *)src;
    if (!with_format(ALL_FORMATS(), type, [&](auto t) { dequantize_kernel<t, OUT><<<grid, 256, 0, st>>>(s, dst, n4); })) {
        set_error("dequantize: unsupported type %d", type);
        return GGML_B200_EUNSUPPORTED;
    }
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

// ------------------------------------------------------------------ f32 -> Q8_0 / Q4_0 (reference *_ref semantics)
// one thread per 32-block: the reference's serial scan order (first element of largest magnitude wins)
template <int T>
__global__ void __launch_bounds__(128) quantize_ref_kernel(const float * __restrict__ x, uint8_t * __restrict__ dst, int64_t nblocks) {
    const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nblocks) return;
    const float * xb = x + b * 32;
    float v[32];
#pragma unroll
    for (int i = 0; i < 8; ++i) { const float4 t = *(const float4 *)(xb + 4 * i); v[4 * i] = t.x; v[4 * i + 1] = t.y; v[4 * i + 2] = t.z; v[4 * i + 3] = t.w; }
    float amax = 0.0f, vmax = 0.0f;
#pragma unroll
    for (int i = 0; i < 32; ++i) if (amax < fabsf(v[i])) { amax = fabsf(v[i]); vmax = v[i]; }
    if constexpr (T == T_Q8_0) {
        uint8_t * o = dst + b * 34;
        const float d = __fdiv_rn(amax, 127.0f);
        const float id = d != 0.0f ? __fdiv_rn(1.0f, d) : 0.0f;
        *(__half *)o = __float2half_rn(d);
#pragma unroll
        for (int i = 0; i < 32; ++i) o[2 + i] = (uint8_t)(int8_t)roundf(__fmul_rn(v[i], id));
    } else {
        uint8_t * o = dst + b * 18;
        const float d = __fdiv_rn(vmax, -8.0f);
        const float id = d != 0.0f ? __fdiv_rn(1.0f, d) : 0.0f;
        *(__half *)o = __float2half_rn(d);
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            const int lo = min(15, (int)(int8_t)(int)__fadd_rn(__fmul_rn(v[i], id), 8.5f));
            const int hi = min(15, (int)(int8_t)(int)__fadd_rn(__fmul_rn(v[i + 16], id), 8.5f));
            o[2 + i] = (uint8_t)((lo & 0xFF) | (hi << 4));
        }
    }
}

} // namespace b200

using namespace b200;

extern "C" {

int ggml_b200_dequantize(int32_t type, const void * src, void * dst, int32_t dst_type, int64_t n, void * stream) {
    const int qk = type_qk(type);
    if (type_bytes(type) == 0) { set_error("dequantize: unsupported type %d", type); return GGML_B200_EUNSUPPORTED; }
    if (n < 0 || n % qk != 0 || (n > 0 && (!src || !dst))) { set_error("dequantize: bad arguments"); return GGML_B200_EINVAL; }
    if (n == 0) return GGML_B200_OK;
    cudaStream_t st = (cudaStream_t)stream;
    if (dst_type == T_F32) return dequantize_dispatch<float>(type, src, (float *)dst, n, st);
    if (dst_type == T_F16) return dequantize_dispatch<__half>(type, src, (__half *)dst, n, st);
    set_error("dequantize: unsupported destination type %d", dst_type);
    return GGML_B200_EUNSUPPORTED;
}

int ggml_b200_quantize(int32_t type, const float * src, void * dst, int64_t n, void * stream) {
    if (type != T_Q8_0 && type != T_Q4_0) { set_error("quantize: only Q8_0 / Q4_0 are produced on the device (got %d)", type); return GGML_B200_EUNSUPPORTED; }
    if (n < 0 || n % 32 != 0 || (n > 0 && (!src || !dst)) || ((uintptr_t)src & 15)) { set_error("quantize: bad arguments"); return GGML_B200_EINVAL; }
    if (n == 0) return GGML_B200_OK;
    const int64_t nb = n / 32;
    const unsigned grid = (unsigned)((nb + 127) / 128);
    cudaStream_t st = (cudaStream_t)stream;
    if (type == T_Q8_0) quantize_ref_kernel<T_Q8_0><<<grid, 128, 0, st>>>(src, (uint8_t *)dst, nb);
    else                quantize_ref_kernel<T_Q4_0><<<grid, 128, 0, st>>>(src, (uint8_t *)dst, nb);
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

} // extern "C"
