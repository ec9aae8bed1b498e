// ops.cu — the small device ops either side of the quantized mat-mul in the examples/gpt-2 graph
// (SURVEY.md §8f-1): GET_ROWS, ADD/MUL/SUB/DIV with broadcast, NORM / RMS_NORM, SCALE, DIAG_MASK_INF, SOFT_MAX,
// unary GELU/SILU/RELU/…, CPY/CONT/DUP (strided, f32/f16 and f32 -> Q8_0/Q4_0), the float (f32/f16 x f32)
// batched strided MUL_MAT used for KQ and KQV, and ROPE (the rotary position embedding of llama-family decoders).  They exist so
// that `gpt-2-backend` runs entirely on the device (it has no scheduler to fall back to the CPU).  Semantics follow the CPU
// backend (src/ggml-cpu/ggml-cpu.c):
//   get_rows :8560-8760   add/mul bcast :4660-5560   norm :8915-8975   rms_norm :8990-9050   scale :8300-8345
//   diag_mask :9745-9805  soft_max :9810-9925        gelu :6520-6570 (+ fp16 table, ggml-cpu.c:1355)   dup/cpy :3220-4300
//   rope :9157-9640       argsort :10746-10783       sum_rows :5663-5694 (+ ggml_vec_sum_f32 :2118)
//   concat :6097-6157     ssm_conv :11379-11445      ssm_scan :11449-11537
//   rwkv_wkv6 :11865-12044                           gated_linear_attn :12067-12235   im2col :9875-10041
//   pool_2d :10305-10377  upscale :10503-10540       leaky_relu :6689-6717            repeat :5901-6015
//   win_part :11541-11582 win_unpart :11604-11640    get_rel_pos :11737-11760         add_rel_pos :11784-11842
//   conv_transpose_2d :10140-10230                   sin / cos :1733-1734
//   out_prod :7788-7905   cross_entropy_loss :12449-12525                    cross_entropy_loss_back :12545-12605
//   opt_step_adamw :12626-12685                      argmax :5773-5795          count_equal :5821-5878   sum :5537-5565
//   repeat_back :6019-6075                           step :1737
// IM2COL is the first node of ggml_conv_1d / ggml_conv_2d (the convolutional front end of Whisper-style encoders); POOL_2D, UPSCALE,
// LEAKY_RELU and REPEAT (the batch norm's per-channel vectors) are the ops around the convs of YOLO-style networks.  WIN_PART / WIN_UNPART
// (windowed attention), GET_REL_POS / ADD_REL_POS (the decomposed relative-position bias), CONV_TRANSPOSE_2D (the mask decoder's output
// upscaling) and SIN / COS (the random-Fourier positional encoding) are the ops of Segment-Anything-style image encoders and mask decoders.
// OUT_PROD (the gradient of MUL_MAT), CROSS_ENTROPY_LOSS and its gradient, OPT_STEP_ADAMW, ARGMAX, COUNT_EQUAL, SUM, REPEAT_BACK (the
// gradient of a broadcast ADD / MUL) and STEP (the gradient of RELU) are the ops ggml_opt's backward and optimizer graphs add.
// ARGSORT and SUM_ROWS are the mixture-of-experts router's top-k and weight normalisation; CONCAT, SSM_CONV and SSM_SCAN are the
// rolling conv state, the causal depthwise convolution and the selective scan of the Mamba-1 layer; RWKV_WKV6 and GATED_LINEAR_ATTN are
// the recurrences of the RWKV-6 time mix and of its gated (RWKV6-Qwen2) form.
// They replace the reference's getrows.cu, binbcast.cu, norm.cu, scale.cu, diagmask.cu, softmax.cu, unary.cu, cpy.cu, mmv.cu, argsort.cu,
// sumrows.cu, concat.cu, wkv6.cu, gla.cu (the reference has no SSM kernels).
#include "b200_internal.h"
#include "b200_op_checks.h"
#include "b200_conv.cuh"
#include "b200_pool.cuh"
#include "b200_sam.cuh"
#include "b200_train.cuh"
#include "b200_quants.cuh"
#include "b200_dequant.cuh"
#include "b200_ptx.cuh"
#include "b200_rope.cuh"
#include "b200_sort.cuh"
#include "b200_ssm.cuh"
#include "b200_wkv.cuh"

#include <cfloat>

namespace b200 {

// Programmatic dependent launch for every small op: each kernel is launched with the programmatic-serialization attribute (launch_pdl),
// so it becomes resident while its predecessor still runs (the launch latency of a ~2 us kernel chain is hidden), waits for the
// predecessor's completion before touching any global memory (griddepcontrol.wait: completion stays transitive along the stream),
// and only then lets ITS successor launch -- a one-kernel lookahead.  A quantized mat-vec launched after one of these small ops starts
// its weight prefetch while the small op runs and waits for this kernel's results before reading them.
__device__ __forceinline__ void pdl_trigger() {
    pdl_wait();
    pdl_launch_dependents();
}

struct tdesc {      // device-side copy of ggml_b200_tensor
    uint8_t * data; int32_t type; int64_t ne[4]; size_t nb[4];
};
static inline tdesc T(const ggml_b200_tensor * t) {
    tdesc d; d.data = (uint8_t *)t->data; d.type = t->type;
    for (int i = 0; i < 4; ++i) { d.ne[i] = t->ne[i]; d.nb[i] = t->nb[i]; }
    return d;
}
static inline int64_t nelem(const tdesc & t) { return t.ne[0] * t.ne[1] * t.ne[2] * t.ne[3]; }
static inline int64_t nrows(const tdesc & t) { return t.ne[1] * t.ne[2] * t.ne[3]; }

// block-wide reduce (blockDim multiple of 32, <= 1024); result broadcast to all threads
template <bool MAX> __device__ __forceinline__ float block_reduce(float v, float * sh) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    v = MAX ? warp_max(v) : warp_sum(v);
    if (nw == 1) return v;
    __syncthreads();
    if (lane == 0) sh[warp] = v;
    __syncthreads();
    float r = lane < nw ? sh[lane] : (MAX ? -INFINITY : 0.0f);
    r = MAX ? warp_max(r) : warp_sum(r);
    return r;
}

// ------------------------------------------------------------------ dequantize one element (bit-exact, as dequant.cu)
template <int T> __device__ __forceinline__ float elem_via_dequant4(const uint8_t * row, int64_t i) {
    float o[4];
    dequant4<T>(row, i & ~(int64_t)3, o);
    return o[i & 3];
}
__device__ __forceinline__ float load_elem(const uint8_t * row, int type, int64_t i) {
    switch (type) {
        case T_F32: return ((const float *)row)[i];
        case T_F16: return __half2float(((const __half *)row)[i]);
        case T_Q4_0: {
            const uint8_t * b = row + (i / 32) * 18; const int j = (int)(i % 32);
            const int q = j < 16 ? (b[2 + j] & 0x0F) : (b[2 + j - 16] >> 4);
            return __fmul_rn((float)(q - 8), h2f(load_u16(b)));
        }
        case T_Q8_0: {
            const uint8_t * b = row + (i / 32) * 34;
            return __fmul_rn((float)(int8_t)b[2 + (i % 32)], h2f(load_u16(b)));
        }
        case T_Q4_K: case T_Q5_K: {
            const int BY = type == T_Q4_K ? 144 : 176;
            const uint8_t * b = row + (i / 256) * BY;
            const int w = (int)(i % 256), c = w / 64, l = w % 32, hi = (w % 64) / 32, j = 2 * c + hi;
            const uint8_t * s = b + 4;
            int sc, mn;
            if (j < 4) { sc = s[j] & 63; mn = s[j + 4] & 63; }
            else       { sc = (s[j + 4] & 0x0F) | ((s[j - 4] >> 6) << 4); mn = (s[j + 4] >> 4) | ((s[j] >> 6) << 4); }
            const uint8_t qb = b[(type == T_Q5_K ? 48 : 16) + 32 * c + l];
            int v = hi ? (qb >> 4) : (qb & 0x0F);
            if (type == T_Q5_K) v += ((b[16 + l] >> j) & 1) << 4;
            return __fsub_rn(__fmul_rn(__fmul_rn(h2f(load_u16(b)), (float)sc), (float)v), __fmul_rn(h2f(load_u16(b + 2)), (float)mn));
        }
        case T_Q6_K: {
            const uint8_t * b = row + (i / 256) * 210;
            const int w = (int)(i % 256), h = w / 128, pos = (w % 128) / 32, l = w % 32;
            const uint8_t ql = b[64 * h + (pos & 1) * 32 + l], qh = b[128 + 32 * h + l];
            const int lo = pos >= 2 ? (ql >> 4) : (ql & 0x0F);
            const int v = (int)(int8_t)(lo | (((qh >> (2 * pos)) & 3) << 4)) - 32;
            const int sc = (int)(int8_t)b[192 + 8 * h + l / 16 + 2 * pos];
            return __fmul_rn(__fmul_rn(h2f(load_u16(b + 208)), (float)sc), (float)v);
        }
        // every other block format: through the element decoders of b200_dequant.cuh (four consecutive weights, pick one)
        case T_Q4_1:   return elem_via_dequant4<T_Q4_1>(row, i);
        case T_Q5_0:   return elem_via_dequant4<T_Q5_0>(row, i);
        case T_Q5_1:   return elem_via_dequant4<T_Q5_1>(row, i);
        case T_Q2_K:   return elem_via_dequant4<T_Q2_K>(row, i);
        case T_Q3_K:   return elem_via_dequant4<T_Q3_K>(row, i);
        case T_IQ4_NL: return elem_via_dequant4<T_IQ4_NL>(row, i);
        case T_IQ4_XS: return elem_via_dequant4<T_IQ4_XS>(row, i);
        case T_IQ2_XXS: return elem_via_dequant4<T_IQ2_XXS>(row, i);
        case T_IQ3_XXS: return elem_via_dequant4<T_IQ3_XXS>(row, i);
        case T_IQ1_S:  return elem_via_dequant4<T_IQ1_S>(row, i);
        case T_IQ2_XS: return elem_via_dequant4<T_IQ2_XS>(row, i);
        case T_IQ2_S: return elem_via_dequant4<T_IQ2_S>(row, i);
        case T_IQ3_S: return elem_via_dequant4<T_IQ3_S>(row, i);
        case T_IQ1_M: return elem_via_dequant4<T_IQ1_M>(row, i);
        case T_TQ1_0: return elem_via_dequant4<T_TQ1_0>(row, i);
        case T_TQ2_0: return elem_via_dequant4<T_TQ2_0>(row, i);
        default: return __int_as_float(0x7fc00000);          // unreachable (check_get_rows rejects unknown types): NaN, never a silent 0
    }
}

// ------------------------------------------------------------------ GET_ROWS
__global__ void get_rows_kernel(tdesc src, tdesc ids, tdesc dst) {
    pdl_trigger();
    // one CTA per destination row (i10, i11, i12)
    const int64_t r = blockIdx.x;
    const int64_t i10 = r % ids.ne[0], i11 = (r / ids.ne[0]) % ids.ne[1], i12 = r / (ids.ne[0] * ids.ne[1]);
    const int32_t i01 = *(const int32_t *)(ids.data + i10 * ids.nb[0] + i11 * ids.nb[1] + i12 * ids.nb[2]);
    const uint8_t * srow = src.data + (int64_t)i01 * src.nb[1] + i11 * src.nb[2] + i12 * src.nb[3];
    float * drow = (float *)(dst.data + i10 * dst.nb[1] + i11 * dst.nb[2] + i12 * dst.nb[3]);
    for (int64_t i = threadIdx.x; i < src.ne[0]; i += blockDim.x) drow[i] = load_elem(srow, src.type, i);
}

// ------------------------------------------------------------------ binary ops with broadcast (f32)
template <int OP> __device__ __forceinline__ float bin_op(float a, float b) {
    if (OP == 0) return a + b;
    if (OP == 1) return a * b;
    if (OP == 2) return a - b;
    return a / b;
}
template <int OP> __global__ void bin_bcast_kernel(tdesc a, tdesc b, tdesc d, int64_t n) {
    pdl_trigger();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int64_t i0 = i % d.ne[0], i1 = (i / d.ne[0]) % d.ne[1], i2 = (i / (d.ne[0] * d.ne[1])) % d.ne[2], i3 = i / (d.ne[0] * d.ne[1] * d.ne[2]);
    const float x = *(const float *)(a.data + i0 * a.nb[0] + i1 * a.nb[1] + i2 * a.nb[2] + i3 * a.nb[3]);
    const float y = *(const float *)(b.data + (i0 % b.ne[0]) * b.nb[0] + (i1 % b.ne[1]) * b.nb[1] + (i2 % b.ne[2]) * b.nb[2] + (i3 % b.ne[3]) * b.nb[3]);
    *(float *)(d.data + i0 * d.nb[0] + i1 * d.nb[1] + i2 * d.nb[2] + i3 * d.nb[3]) = bin_op<OP>(x, y);
}

// ------------------------------------------------------------------ NORM / RMS_NORM (rows contiguous along dim 0)
// block-wide sum of one double per thread (blockDim multiple of 32, <= 1024); result broadcast to all threads
__device__ __forceinline__ double block_sum_f64(double v, double * sh) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (nw == 1) return v;
    __syncthreads();
    if (lane == 0) sh[warp] = v;
    __syncthreads();
    double r = lane < nw ? sh[lane] : 0.0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) r += __shfl_xor_sync(0xffffffffu, r, o);
    return r;
}

// A row's mean (0 for RMS_NORM) and scale as ggml-cpu computes them (ggml_compute_forward_norm_f32 / _rms_norm_f32): the sums of x and of
// the f32 squares in double, the mean and the variance rounded to f32, scale = 1.0f / sqrtf(variance + eps).  Sums in f32 put rows with a
// common offset of 30 .. 1e4 up to 4340x (in NMSE against f64) further from the true result than ggml-cpu's.
template <bool RMS> __device__ __forceinline__ void norm_row_stats(const float * x, int64_t n, float eps, double * sh, float & mean, float & scale) {
    mean = 0.0f;
    if (!RMS) {
        double sum = 0.0;
        for (int64_t i = threadIdx.x; i < n; i += blockDim.x) sum += (double)x[i];
        mean = (float)(block_sum_f64(sum, sh) / (double)n);
    }
    double sq = 0.0;
    for (int64_t i = threadIdx.x; i < n; i += blockDim.x) { const float v = x[i] - mean; sq += (double)(v * v); }
    const float var = (float)(block_sum_f64(sq, sh) / (double)n);
    scale = 1.0f / sqrtf(var + eps);
}

template <bool RMS> __global__ void norm_kernel(tdesc s, tdesc d, float eps) {
    pdl_trigger();
    __shared__ double sh[32];
    const int64_t r = blockIdx.x;
    const int64_t i1 = r % s.ne[1], i2 = (r / s.ne[1]) % s.ne[2], i3 = r / (s.ne[1] * s.ne[2]);
    const float * x = (const float *)(s.data + i1 * s.nb[1] + i2 * s.nb[2] + i3 * s.nb[3]);
    float * y = (float *)(d.data + i1 * d.nb[1] + i2 * d.nb[2] + i3 * d.nb[3]);
    const int64_t n = s.ne[0];
    float mean, scale;
    norm_row_stats<RMS>(x, n, eps, sh, mean, scale);
    for (int64_t i = threadIdx.x; i < n; i += blockDim.x) y[i] = (x[i] - mean) * scale;
}

// NORM -> MUL(gain) -> ADD(bias) in one pass; every intermediate tensor of the three ggml nodes is still written
template <bool RMS> __global__ void norm_affine_kernel(tdesc s, tdesc d1, const float * gain, tdesc d2, const float * bias, tdesc d3, float eps) {
    pdl_trigger();
    __shared__ double sh[32];
    const int64_t r = blockIdx.x;
    const int64_t i1 = r % s.ne[1], i2 = (r / s.ne[1]) % s.ne[2], i3 = r / (s.ne[1] * s.ne[2]);
    const float * x = (const float *)(s.data + i1 * s.nb[1] + i2 * s.nb[2] + i3 * s.nb[3]);
    float * y1 = (float *)(d1.data + i1 * d1.nb[1] + i2 * d1.nb[2] + i3 * d1.nb[3]);
    float * y2 = (float *)(d2.data + i1 * d2.nb[1] + i2 * d2.nb[2] + i3 * d2.nb[3]);
    float * y3 = (float *)(d3.data + i1 * d3.nb[1] + i2 * d3.nb[2] + i3 * d3.nb[3]);
    const int64_t n = s.ne[0];
    float mean, scale;
    norm_row_stats<RMS>(x, n, eps, sh, mean, scale);
    for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
        const float a = (x[i] - mean) * scale, b = __fmul_rn(a, gain[i]), c = __fadd_rn(b, bias[i]);   // separately rounded, like the three ggml ops
        y1[i] = a; y2[i] = b; y3[i] = c;
    }
}

// ------------------------------------------------------------------ SCALE, DIAG_MASK_INF, unary
__global__ void scale_kernel(const float * x, float * y, float s, int64_t n) {
    pdl_trigger();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) y[i] = x[i] * s;
}
__global__ void diag_mask_inf_kernel(const float * x, float * y, int64_t ne0, int64_t ne1, int n_past, int64_t n) {
    pdl_trigger();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int64_t c = i % ne0, r = (i / ne0) % ne1;
    y[i] = c > n_past + r ? -INFINITY : x[i];
}
enum { U_GELU = 0, U_SILU = 1, U_RELU = 2, U_TANH = 3, U_NEG = 4, U_ABS = 5, U_GELU_QUICK = 6, U_SIGMOID = 7, U_EXP = 8, U_SQR = 9, U_SQRT = 10,
       U_SIN = 11, U_COS = 12, U_STEP = 13 };
__global__ void unary_kernel(int uop, const float * x, float * y, int64_t n) {
    pdl_trigger();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float v = x[i];
    float r;
    switch (uop) {
        case U_GELU: r = gelu_ggml(v); break;
        case U_SILU: r = v / (1.0f + expf(-v)); break;
        case U_RELU: r = fmaxf(v, 0.0f); break;
        case U_TANH: r = tanhf(v); break;
        case U_NEG: r = -v; break;
        case U_ABS: r = fabsf(v); break;
        case U_GELU_QUICK: r = gelu_quick_ggml(v); break;
        case U_SIGMOID: r = 1.0f / (1.0f + expf(-v)); break;
        case U_EXP: r = expf(v); break;
        case U_SQR: r = v * v; break;
        case U_SQRT: r = sqrtf(v); break;
        // the library sinf / cosf (within 2 ulp everywhere), never the __sinf / __cosf intrinsics
        case U_SIN: r = sinf(v); break;
        case U_COS: r = cosf(v); break;
        default: r = step_value(v); break;
    }
    y[i] = r;
}

// ------------------------------------------------------------------ SOFT_MAX (rows contiguous): softmax(x*scale + mask*slope)
// diag_n_past >= 0 folds a preceding GGML_OP_DIAG_MASK_INF (and, through `scale`, a preceding GGML_OP_SCALE) into the row pass:
// element i0 of row i1 is -inf where i0 > diag_n_past + i1 (ggml_compute_forward_diag_mask_f32, src/ggml-cpu/ggml-cpu.c)
__global__ void soft_max_kernel(const float * x, const uint8_t * mask, int mask_type, float * y, int64_t ne0, int64_t ne1, int64_t ne2,
                                float scale, float max_bias, float m0, float m1, uint32_t n_head_log2, int diag_n_past) {
    pdl_trigger();
    __shared__ float sh[32];
    const int64_t r = blockIdx.x;                 // row = i1 + ne1 * (i2 + ne2 * i3)
    const int64_t i1 = r % ne1;
    const float * xr = x + r * ne0;
    float * yr = y + r * ne0;
    float slope = 1.0f;
    if (max_bias > 0.0f) {
        const uint32_t h = (uint32_t)((r / ne1) % ne2);
        slope = h < n_head_log2 ? powf(m0, (float)(h + 1)) : powf(m1, (float)(2 * (h - n_head_log2) + 1));
    }
    const uint8_t * mr = mask ? mask + (size_t)i1 * ne0 * (mask_type == T_F16 ? 2 : 4) : nullptr;
    auto val = [&](int64_t i) {
        float v = xr[i] * scale;
        if (diag_n_past >= 0 && i > (int64_t)diag_n_past + i1) v = -INFINITY;
        if (mr) v += slope * (mask_type == T_F16 ? __half2float(((const __half *)mr)[i]) : ((const float *)mr)[i]);
        return v;
    };
    float mx = -INFINITY;
    for (int64_t i = threadIdx.x; i < ne0; i += blockDim.x) mx = fmaxf(mx, val(i));
    mx = block_reduce<true>(mx, sh);
    float sum = 0.0f;
    for (int64_t i = threadIdx.x; i < ne0; i += blockDim.x) { const float e = expf(val(i) - mx); yr[i] = e; sum += e; }
    sum = block_reduce<false>(sum, sh);
    const float inv = 1.0f / sum;
    for (int64_t i = threadIdx.x; i < ne0; i += blockDim.x) yr[i] *= inv;
}

// ------------------------------------------------------------------ CPY / CONT / DUP (same element count, any strides)
__device__ __forceinline__ size_t offset_of(const tdesc & t, int64_t i) {    // i = linear element index in t's logical order
    const int64_t i0 = i % t.ne[0], i1 = (i / t.ne[0]) % t.ne[1], i2 = (i / (t.ne[0] * t.ne[1])) % t.ne[2], i3 = i / (t.ne[0] * t.ne[1] * t.ne[2]);
    return i0 * t.nb[0] + i1 * t.nb[1] + i2 * t.nb[2] + i3 * t.nb[3];
}
// blockIdx.y selects one of two independent copies of the same size (the K and V cache updates of a layer: one launch)
__global__ void cpy_kernel(tdesc s, tdesc d, tdesc s2, tdesc d2, int64_t n) {
    pdl_trigger();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (blockIdx.y) { s = s2; d = d2; }
    const uint8_t * sp = s.data + offset_of(s, i);
    uint8_t * dp = d.data + offset_of(d, i);
    const float v = s.type == T_F32 ? *(const float *)sp : __half2float(*(const __half *)sp);
    if (d.type == T_F32) *(float *)dp = v;
    else if (s.type == T_F16) *(__half *)dp = *(const __half *)sp;
    else *(__half *)dp = __float2half_rn(v);
}
// f32 (strided, dim-0 contiguous) -> Q8_0 / Q4_0 rows (dst rows contiguous blocks); one thread per 32-block
template <int QT> __global__ void cpy_f32_q_kernel(tdesc s, tdesc d, int64_t nblocks) {
    pdl_trigger();
    const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nblocks) return;
    const int64_t e = b * 32;                                   // linear element index of the block start
    const float * x = (const float *)(s.data + offset_of(s, e));
    const int64_t bpr = d.ne[0] / 32;                           // dst blocks per row
    const int64_t drow = b / bpr, dblk = b % bpr;
    const int64_t i1 = drow % d.ne[1], i2 = (drow / d.ne[1]) % d.ne[2], i3 = drow / (d.ne[1] * d.ne[2]);
    uint8_t * o = d.data + i1 * d.nb[1] + i2 * d.nb[2] + i3 * d.nb[3] + dblk * (QT == T_Q8_0 ? 34 : 18);
    float amax = 0.0f, vmax = 0.0f;
    for (int i = 0; i < 32; ++i) if (amax < fabsf(x[i])) { amax = fabsf(x[i]); vmax = x[i]; }
    if (QT == T_Q8_0) {
        // what ggml-cpu's CPY writes on x86 (quantize_row_q8_0, AVX branch, src/ggml-cpu/ggml-cpu-quants.c:786-830): id = 127 / amax, codes
        // rounded half to even.  The _ref formula (id = 1 / d, roundf) differs in a few codes per million, more on half-integer inputs.
        const float dd = __fdiv_rn(amax, 127.0f), id = amax != 0.0f ? __fdiv_rn(127.0f, amax) : 0.0f;
        *(__half *)o = __float2half_rn(dd);
        for (int i = 0; i < 32; ++i) o[2 + i] = (uint8_t)(int8_t)__float2int_rn(__fmul_rn(x[i], id));
    } else {                                                    // Q4_0: quantize_row_q4_0_ref, which ggml-cpu's CPY calls as well
        const float dd = __fdiv_rn(vmax, -8.0f), id = dd != 0.0f ? __fdiv_rn(1.0f, dd) : 0.0f;
        *(__half *)o = __float2half_rn(dd);
        for (int i = 0; i < 16; ++i) {
            const int lo = min(15, (int)(int8_t)(int)__fadd_rn(__fmul_rn(x[i], id), 8.5f));
            const int hi = min(15, (int)(int8_t)(int)__fadd_rn(__fmul_rn(x[i + 16], id), 8.5f));
            o[2 + i] = (uint8_t)((lo & 0xFF) | (hi << 4));
        }
    }
}

// ------------------------------------------------------------------ float MUL_MAT (f32 / f16 weights x f32), batched + strided
// one warp per output element; the CPU rounds src1 to f16 when src0 is f16 (vec_dot_type, ggml-cpu.c:262-268)
__global__ void __launch_bounds__(128) mul_mat_f_kernel(tdesc a, tdesc b, tdesc d, int64_t nout) {
    pdl_trigger();
    const int lane = threadIdx.x & 31;
    const int64_t o = (int64_t)blockIdx.x * 4 + (threadIdx.x >> 5);
    if (o >= nout) return;
    const int64_t m = o % d.ne[0], n = (o / d.ne[0]) % d.ne[1], i12 = (o / (d.ne[0] * d.ne[1])) % d.ne[2], i13 = o / (d.ne[0] * d.ne[1] * d.ne[2]);
    const int64_t i02 = i12 / (b.ne[2] / a.ne[2]), i03 = i13 / (b.ne[3] / a.ne[3]);
    const uint8_t * ar = a.data + m * a.nb[1] + i02 * a.nb[2] + i03 * a.nb[3];
    const uint8_t * br = b.data + n * b.nb[1] + i12 * b.nb[2] + i13 * b.nb[3];
    float acc = 0.0f;
    if (a.type == T_F32) {
        for (int64_t k = lane; k < a.ne[0]; k += 32) acc += *(const float *)(ar + k * a.nb[0]) * *(const float *)(br + k * b.nb[0]);
    } else if (b.type == T_F16) {                                // f16 x f16 (the conv mat-mul of ggml_conv_1d / _2d): src1 read as is
        for (int64_t k = lane; k < a.ne[0]; k += 32)
            acc += __half2float(*(const __half *)(ar + k * a.nb[0])) * __half2float(*(const __half *)(br + k * b.nb[0]));
    } else {
        for (int64_t k = lane; k < a.ne[0]; k += 32)
            acc += __half2float(*(const __half *)(ar + k * a.nb[0])) * __half2float(__float2half_rn(*(const float *)(br + k * b.nb[0])));
    }
    acc = warp_sum(acc);
    if (lane == 0) *(float *)(d.data + m * d.nb[0] + n * d.nb[1] + i12 * d.nb[2] + i13 * d.nb[3]) = acc;
}

// ------------------------------------------------------------------ FLASH_ATTN_EXT (f32 Q; f16 / f32 / block-quantized K and V; f16 mask)
// What ggml_compute_forward_flash_attn_ext_f16 computes (src/ggml-cpu/ggml-cpu.c:10805-10990): per (query row, head, batch) an online-softmax
// pass over the KV positions, dst[d, head, q, b] = sum_kv softmax(scale * K.q [softcap] + slope * mask) V.  One CTA per query row and head;
// its four warps take the KV positions round-robin, each lane owns the elements lane, lane + 32, ... of the head dimension (<= 256), K and V
// rows are decoded on the fly (any advertised block format: quantized KV caches), the four partial (max, sum, accumulator) triples are
// merged through shared memory.  Accumulation is f32 (the CPU keeps an f16 accumulator for f16 V; the reference's own gate is NMSE 5e-4).
// Replaces src/ggml-cuda/fattn*.cu for correctness; this is the bandwidth-shaped decode form, not a tensor-core prefill kernel.
struct fa_params {
    tdesc q, k, v, mask, dst;
    float scale, max_bias, softcap, m0, m1;
    uint32_t n_head_log2;
};
__global__ void __launch_bounds__(128) flash_attn_ext_kernel(fa_params p) {
    pdl_trigger();
    __shared__ float s_m[4], s_s[4], s_acc[4][256];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t iq1 = blockIdx.x, iq2 = blockIdx.y, iq3 = blockIdx.z;
    const int D = (int)p.q.ne[0];
    const int64_t nkv = p.k.ne[1];
    const int64_t ik2 = iq2 / (p.q.ne[2] / p.k.ne[2]), ik3 = iq3 / (p.q.ne[3] / p.k.ne[3]);
    const int64_t iv2 = iq2 / (p.q.ne[2] / p.v.ne[2]), iv3 = iq3 / (p.q.ne[3] / p.v.ne[3]);
    const float * pq = (const float *)(p.q.data + iq1 * p.q.nb[1] + iq2 * p.q.nb[2] + iq3 * p.q.nb[3]);
    float qv[8], acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) { const int d = lane + 32 * i; qv[i] = d < D ? pq[d] : 0.0f; acc[i] = 0.0f; }
    float slope = 1.0f;
    if (p.max_bias > 0.0f) {
        const uint32_t h = (uint32_t)iq2;
        slope = h < p.n_head_log2 ? powf(p.m0, (float)(h + 1)) : powf(p.m1, (float)(2 * (h - p.n_head_log2) + 1));
    }
    const __half * mp = p.mask.data ? (const __half *)(p.mask.data + iq1 * p.mask.nb[1]) : nullptr;
    float M = -INFINITY, S = 0.0f;
    for (int64_t ic = warp; ic < nkv; ic += 4) {
        const float mv = mp ? slope * __half2float(mp[ic]) : 0.0f;
        if (mv == -INFINITY) continue;                                          // warp-uniform
        const uint8_t * krow = p.k.data + ic * p.k.nb[1] + ik2 * p.k.nb[2] + ik3 * p.k.nb[3];
        float part = 0.0f;
#pragma unroll
        for (int i = 0; i < 8; ++i) { const int d = lane + 32 * i; if (d < D) part += qv[i] * load_elem(krow, p.k.type, d); }
        float sc = warp_sum(part) * p.scale;
        if (p.softcap != 0.0f) sc = p.softcap * tanhf(sc);
        sc += mv;
        float vs = 1.0f;
        if (sc > M) {
            const float ms = expf(M - sc);                                      // 0 on the first position (M = -inf)
            M = sc;
#pragma unroll
            for (int i = 0; i < 8; ++i) acc[i] *= ms;
            S = S * ms + 1.0f;
        } else {
            vs = expf(sc - M);
            S += vs;
        }
        const uint8_t * vrow = p.v.data + ic * p.v.nb[1] + iv2 * p.v.nb[2] + iv3 * p.v.nb[3];
#pragma unroll
        for (int i = 0; i < 8; ++i) { const int d = lane + 32 * i; if (d < D) acc[i] += vs * load_elem(vrow, p.v.type, d); }
    }
    if (lane == 0) { s_m[warp] = M; s_s[warp] = S; }
#pragma unroll
    for (int i = 0; i < 8; ++i) { const int d = lane + 32 * i; if (d < D) s_acc[warp][d] = acc[i]; }
    __syncthreads();
    if (warp == 0) {
        const float Mx = fmaxf(fmaxf(s_m[0], s_m[1]), fmaxf(s_m[2], s_m[3]));
        float f[4], St = 0.0f;
#pragma unroll
        for (int w = 0; w < 4; ++w) { f[w] = s_m[w] == -INFINITY ? 0.0f : expf(s_m[w] - Mx); St += s_s[w] * f[w]; }
        const float inv = 1.0f / St;
        float * out = (float *)(p.dst.data + iq2 * p.dst.nb[1] + iq1 * p.dst.nb[2] + iq3 * p.dst.nb[3]);
        for (int d = lane; d < D; d += 32)
            out[d] = (s_acc[0][d] * f[0] + s_acc[1][d] * f[1] + s_acc[2][d] * f[2] + s_acc[3][d] * f[3]) * inv;
    }
}

// ------------------------------------------------------------------ ROPE (forward; f32 -> f32, f16 -> f16; any row strides; dst may alias src)
// One CTA per (position i2, block of heads, i3): the cos/sin of every pair at that position is computed once into shared memory (b200_rope.cuh,
// the CPU's sequential theta product), then applied to each head of the block.  Each thread owns whole pairs (item q of a row: two elements)
// and reads both before writing either, so the in-place form is safe.  Positions (and freq factors) are read on the device.
template <typename T> __device__ __forceinline__ float rope_ld(const uint8_t * p) {
    if constexpr (sizeof(T) == 4) return *(const float *)p; else return __half2float(*(const __half *)p);
}
template <typename T> __device__ __forceinline__ void rope_st(uint8_t * p, float v) {
    if constexpr (sizeof(T) == 4) *(float *)p = v; else *(__half *)p = __float2half_rn(v);
}
template <typename T> __global__ void __launch_bounds__(128) rope_kernel(tdesc s, const int32_t * pos, const float * ff, tdesc d, rope_consts c, int heads_per_cta) {
    pdl_trigger();
    __shared__ float2 cache[ROPE_MAX_CACHE];
    const int64_t i2 = blockIdx.x, i3 = blockIdx.z, ne2 = s.ne[2];
    float p[4];
    p[0] = (float)pos[i2];
    if (c.mode & ROPE_MROPE) { p[1] = (float)pos[i2 + ne2]; p[2] = (float)pos[i2 + 2 * ne2]; p[3] = (float)pos[i2 + 3 * ne2]; }
    else p[1] = p[2] = p[3] = 0.0f;
    const int ncache = rope_n_cache(c);
    for (int j = threadIdx.x; j < ncache; j += blockDim.x) {
        float cs, sn;
        rope_cos_sin(c, rope_theta(c, p, j), ff ? ff[j] : 1.0f, j, cs, sn);
        cache[j] = make_float2(cs, sn);
    }
    __syncthreads();
    const int64_t ppr = s.ne[0] / 2, h0 = (int64_t)blockIdx.y * heads_per_cta;
    const int64_t nh = min((int64_t)heads_per_cta, s.ne[1] - h0);
    for (int64_t it = threadIdx.x; it < nh * ppr; it += blockDim.x) {
        const int64_t i1 = h0 + it / ppr, q = it % ppr;
        const uint8_t * sr = s.data + i1 * s.nb[1] + i2 * s.nb[2] + i3 * s.nb[3];
        uint8_t * dr = d.data + i1 * d.nb[1] + i2 * d.nb[2] + i3 * d.nb[3];
        int64_t e0, e1;
        const int slot = rope_item(c, q, e0, e1);
        if (slot < 0) {                                        // tail beyond n_dims: copied bit for bit
            const T a = *(const T *)(sr + e0 * sizeof(T)), b = *(const T *)(sr + e1 * sizeof(T));
            *(T *)(dr + e0 * sizeof(T)) = a; *(T *)(dr + e1 * sizeof(T)) = b;
            continue;
        }
        const float x0 = rope_ld<T>(sr + e0 * sizeof(T)), x1 = rope_ld<T>(sr + e1 * sizeof(T));
        float y0, y1;
        rope_rotate(x0, x1, cache[slot].x, cache[slot].y, y0, y1);
        rope_st<T>(dr + e0 * sizeof(T), y0); rope_st<T>(dr + e1 * sizeof(T), y1);
    }
}

// ------------------------------------------------------------------ IM2COL (f32 input -> f32 / f16 columns, dst packed)
// One thread per dst element, in dst's order, so the stores coalesce; b200_conv.cuh locates the input element (or the padding) of each.
template <typename T> __global__ void im2col_kernel(im2col_geom g, const uint8_t * __restrict__ src1, T * __restrict__ dst, int64_t n) {
    pdl_trigger();
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n) return;
    const float v = im2col_value(g, src1, e);
    if constexpr (sizeof(T) == 4) dst[e] = v; else dst[e] = __float2half_rn(v);
}

// ------------------------------------------------------------------ POOL_2D, UPSCALE, LEAKY_RELU, REPEAT (around the convs of YOLO-style nets)
// One thread per dst element, in dst's order, so the stores coalesce; b200_pool.cuh holds each element's logic.
__global__ void pool2d_kernel(pool2d_geom g, const uint8_t * __restrict__ src, float * __restrict__ dst, int64_t n) {
    pdl_trigger();
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n) return;
    dst[e] = pool2d_value(g, src, e);
}

__global__ void upscale_kernel(upscale_geom g, const uint8_t * __restrict__ src, uint8_t * __restrict__ dst, int64_t n) {
    pdl_trigger();
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n) return;
    int64_t dofs;
    const int64_t sofs = upscale_offsets(g, e, dofs);
    *(float *)(dst + dofs) = *(const float *)(src + sofs);
}

// in place when dst is src: each thread reads its element before it writes it
__global__ void leaky_relu_kernel(tdesc s, tdesc d, float slope, int64_t n) {
    pdl_trigger();
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n) return;
    const int64_t i0 = e % d.ne[0], i1 = (e / d.ne[0]) % d.ne[1], i2 = (e / (d.ne[0] * d.ne[1])) % d.ne[2], i3 = e / (d.ne[0] * d.ne[1] * d.ne[2]);
    const float x = *(const float *)(s.data + i0 * 4 + i1 * s.nb[1] + i2 * s.nb[2] + i3 * s.nb[3]);
    *(float *)(d.data + i0 * 4 + i1 * d.nb[1] + i2 * d.nb[2] + i3 * d.nb[3]) = leaky_relu_value(x, slope);
}

// W: the element as a raw word (uint32_t: f32 / i32, uint16_t: f16 / bf16 / i16), never converted
template <typename W> __global__ void repeat_kernel(repeat_geom g, const uint8_t * __restrict__ src, uint8_t * __restrict__ dst, int64_t n) {
    pdl_trigger();
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n) return;
    int64_t dofs;
    const int64_t sofs = repeat_offsets(g, e, dofs);
    *(W *)(dst + dofs) = *(const W *)(src + sofs);
}

// ------------------------------------------------------------------ WIN_PART, WIN_UNPART, GET_REL_POS, ADD_REL_POS (SAM-style image encoders)
// One row of threads per dst row of ne0 words: the row on grid x, blocks of the row on grid y.  The row's source is decided once per thread
// in 32-bit arithmetic (b200_sam.cuh), and loads and stores coalesce along dim 0.  The data ops move raw words.
__global__ void win_part_kernel(win_geom g, const uint32_t * __restrict__ src, uint32_t * __restrict__ dst, int64_t ne0) {
    pdl_trigger();
    const int64_t i0 = (int64_t)blockIdx.y * blockDim.x + threadIdx.x;
    if (i0 >= ne0) return;
    const int32_t sr = win_part_src_row(g, blockIdx.x);
    dst[(int64_t)blockIdx.x * ne0 + i0] = sr < 0 ? 0u : src[(int64_t)sr * ne0 + i0];          // 0u: the +0.0f ggml-cpu writes
}

__global__ void win_unpart_kernel(win_geom g, const uint32_t * __restrict__ src, uint32_t * __restrict__ dst, int64_t ne0) {
    pdl_trigger();
    const int64_t i0 = (int64_t)blockIdx.y * blockDim.x + threadIdx.x;
    if (i0 >= ne0) return;
    dst[(int64_t)blockIdx.x * ne0 + i0] = src[(int64_t)win_unpart_src_row(g, blockIdx.x) * ne0 + i0];
}

__global__ void get_rel_pos_kernel(uint32_t w, const uint16_t * __restrict__ src, uint16_t * __restrict__ dst, int64_t ne0) {
    pdl_trigger();
    const int64_t i0 = (int64_t)blockIdx.y * blockDim.x + threadIdx.x;
    if (i0 >= ne0) return;
    dst[(int64_t)blockIdx.x * ne0 + i0] = src[(int64_t)get_rel_pos_src_row(w, blockIdx.x) * ne0 + i0];
}

// V consecutive keys per thread (V = 4: float4 loads and stores, when L L % 4 == 0 and src / dst are 16-byte aligned).  In place when dst is
// src: each thread reads its elements before it writes them.
template <int V> __global__ void add_rel_pos_kernel(const float * src, const float * __restrict__ pw, const float * __restrict__ ph, float * dst,
                                                    uint32_t L, uint32_t LL) {
    pdl_trigger();
    const uint32_t c0 = (blockIdx.y * blockDim.x + threadIdx.x) * V;
    if (c0 >= LL) return;
    const int64_t r = blockIdx.x, e = r * LL + c0;
    const float * pwr = pw + r * L, * phr = ph + r * L;
    float v[V];
    if constexpr (V == 4) { const float4 t = *(const float4 *)(src + e); v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w; }
    else v[0] = src[e];
    uint32_t kh = c0 / L, kw = c0 - kh * L;
#pragma unroll
    for (int j = 0; j < V; ++j) {
        v[j] = add_rel_pos_value(v[j], pwr[kw], phr[kh], kh, kw);
        if (++kw == L) { kw = 0; ++kh; }
    }
    if constexpr (V == 4) *(float4 *)(dst + e) = make_float4(v[0], v[1], v[2], v[3]);
    else dst[e] = v[0];
}

// ------------------------------------------------------------------ CONV_TRANSPOSE_2D (the mask decoder's output upscaling)
// Output (ox, oy) = (px + s qx, py + s qy) of stride phase (px, py) takes taps kx = px + s mx, ky = py + s my from input (qx - mx, qy - my):
// every output of one phase has the same taps.  A CTA owns CT2D_TQX x CT2D_TQY outputs (qx, qy) of the phase blockIdx.z and CT2D_CO output
// channels; each thread one output pixel x CT2D_COT channels, accumulated in f32 registers.  The taps run in descending (my, mx), which is
// ascending input row, then column: ggml-cpu's order.  For each tap the dot over Cin runs in chunks of CT2D_CI channels, each staged in shared
// memory as the fp16-rounded input tile and the kernel slice (as f32).  No workspace; every output is written once (phases without taps,
// s > K, write +0).  Three CTAs per SM: 80 registers without spills (a bare 256-thread bound lets ptxas squeeze to 64 and spill).
__global__ void __launch_bounds__(CT2D_THREADS, 3) ct2d_kernel(ct2d_geom g, const uint8_t * __restrict__ k, const uint8_t * __restrict__ x,
                                                            float * __restrict__ dst) {
    pdl_trigger();
    constexpr int NP = CT2D_TQX * CT2D_TQY;
    __shared__ float sx[CT2D_CI][NP];
    __shared__ __align__(16) float sk[CT2D_CI][CT2D_CO];
    const int s = g.s, py = (int)blockIdx.z / s, px = (int)blockIdx.z - py * s;
    const int nqx = px < g.OW ? (g.OW - px + s - 1) / s : 0, nqy = py < g.OH ? (g.OH - py + s - 1) / s : 0;   // this phase's outputs
    const int tiles_x = ((g.OW + s - 1) / s + CT2D_TQX - 1) / CT2D_TQX;
    const int ty = (int)blockIdx.x / tiles_x, tx = (int)blockIdx.x - ty * tiles_x;
    const int qx0 = tx * CT2D_TQX, qy0 = ty * CT2D_TQY;
    if (qx0 >= nqx || qy0 >= nqy) return;                                   // the whole CTA: a tile beyond this phase's outputs
    const int p = threadIdx.x % NP, grp = threadIdx.x / NP;                 // grp is warp-uniform: sk reads broadcast
    const int qx = qx0 + p % CT2D_TQX, qy = qy0 + p / CT2D_TQX;
    const int co0 = blockIdx.y * CT2D_CO;
    const int Mx = px < g.Kw ? (g.Kw - px + s - 1) / s : 0, My = py < g.Kh ? (g.Kh - py + s - 1) / s : 0;
    float out[CT2D_COT];
#pragma unroll
    for (int j = 0; j < CT2D_COT; ++j) out[j] = 0.0f;
    for (int my = My - 1; my >= 0; --my) {
        for (int mx = Mx - 1; mx >= 0; --mx) {
            const int ky = py + my * s, kx = px + mx * s;
            float dot[CT2D_COT];
#pragma unroll
            for (int j = 0; j < CT2D_COT; ++j) dot[j] = 0.0f;
            for (int ci0 = 0; ci0 < g.Cin; ci0 += CT2D_CI) {
                const int n = min(CT2D_CI, g.Cin - ci0);
                __syncthreads();                                            // the previous chunk's readers are done
                for (int i = threadIdx.x; i < CT2D_CI * NP; i += CT2D_THREADS) {
                    const int c = i / NP, pp = i % NP;
                    const int ix = qx0 + pp % CT2D_TQX - mx, iy = qy0 + pp / CT2D_TQX - my;
                    sx[c][pp] = c < n && ix >= 0 && ix < g.W && iy >= 0 && iy < g.H ? ct2d_input(g, x, ix, iy, ci0 + c) : 0.0f;
                }
                for (int i = threadIdx.x; i < CT2D_CI * CT2D_CO; i += CT2D_THREADS) {
                    const int c = i / CT2D_CO, o = i % CT2D_CO;
                    sk[c][o] = c < n && co0 + o < g.Cout ? ct2d_kernel(g, k, kx, ky, co0 + o, ci0 + c) : 0.0f;
                }
                __syncthreads();
                for (int c = 0; c < n; ++c) {
                    const float xv = sx[c][p];
#pragma unroll
                    for (int j = 0; j < CT2D_COT; ++j) dot[j] = ct2d_dot_step(dot[j], xv, sk[c][grp * CT2D_COT + j]);
                }
            }
            const int ix = qx - mx, iy = qy - my;
            if (ix >= 0 && ix < g.W && iy >= 0 && iy < g.H) {               // a tap ggml-cpu has: add it
#pragma unroll
                for (int j = 0; j < CT2D_COT; ++j) out[j] = pool_add(out[j], dot[j]);
            }
        }
    }
    if (qx >= nqx || qy >= nqy) return;
    const int64_t ox = px + (int64_t)s * qx, oy = py + (int64_t)s * qy;
#pragma unroll
    for (int j = 0; j < CT2D_COT; ++j) {
        const int co = co0 + grp * CT2D_COT + j;
        if (co < g.Cout) dst[((int64_t)co * g.OH + oy) * g.OW + ox] = out[j];
    }
}

// ------------------------------------------------------------------ OUT_PROD (the gradient of MUL_MAT): a tiled FP32 SIMT GEMM
// dst[i0, i1] = sum_k a[i0, k] b[i1, k] for one (i2, i3) per grid z.  A CTA owns OP_BM x OP_BN outputs and walks K in slices of OP_BK:
// each slice of a (coalesced along i0) and of b (coalesced along whichever of i1 / k is contiguous, b_k_contig) is staged in shared
// memory, then every thread updates its OP_TM x OP_TN accumulators with one fused multiply-add per term, in ascending k (b200_train.cuh).
// A thread's outputs are two groups of 4 along i0 (tx*4 and 64 + tx*4) by two of 4 along i1, so its shared-memory reads are float4s
// without bank conflicts and a warp's stores cover 64 consecutive i0.  No workspace; K == 0 writes zeros.
struct out_prod_geom {
    int64_t M, N, K;                // dst ne0, ne1; the shared dim
    int64_t ne2, dps2, dps3;        // dst ne2; dst per src0 along dims 2 and 3
    int64_t anb1, anb2, anb3;       // src0 strides (nb0 == 4), bytes
    int64_t bnb0, bnb1, bnb2, bnb3; // src1 strides, bytes
    int64_t dnb1, dnb2, dnb3;       // dst strides, bytes
    int b_k_contig;                 // src1 is contiguous along k (ggml_transpose(grad)): stage it k-fastest
};

__global__ void __launch_bounds__(OP_THREADS, 1) out_prod_kernel(out_prod_geom g, const uint8_t * __restrict__ a, const uint8_t * __restrict__ b,
                                                                 uint8_t * __restrict__ dst) {
    pdl_trigger();
    __shared__ __align__(16) float sa[OP_BK][OP_BM];
    __shared__ __align__(16) float sb[OP_BK][OP_BN + 4];       // +4: the k-fastest staging writes without bank conflicts
    const int tid = threadIdx.x, tx = tid % 16, ty = tid / 16;
    const int64_t m0 = (int64_t)blockIdx.x * OP_BM, n0 = (int64_t)blockIdx.y * OP_BN;
    const int64_t i2 = blockIdx.z % g.ne2, i3 = blockIdx.z / g.ne2;
    const uint8_t * ab = a + (i2 / g.dps2) * g.anb2 + (i3 / g.dps3) * g.anb3;
    const uint8_t * bb = b + i2 * g.bnb2 + i3 * g.bnb3;
    float acc[OP_TM][OP_TN];
#pragma unroll
    for (int r = 0; r < OP_TM; ++r)
#pragma unroll
        for (int c = 0; c < OP_TN; ++c) acc[r][c] = 0.0f;
    for (int64_t k0 = 0; k0 < g.K; k0 += OP_BK) {
        const int kn = (int)min((int64_t)OP_BK, g.K - k0);
#pragma unroll
        for (int j = 0; j < OP_BK * OP_BM / OP_THREADS; ++j) {
            const int e = tid + j * OP_THREADS, k = e / OP_BM, m = e % OP_BM;
            sa[k][m] = k < kn && m0 + m < g.M ? *(const float *)(ab + (m0 + m) * 4 + (k0 + k) * g.anb1) : 0.0f;
        }
#pragma unroll
        for (int j = 0; j < OP_BK * OP_BN / OP_THREADS; ++j) {
            const int e = tid + j * OP_THREADS;
            const int k = g.b_k_contig ? e % OP_BK : e / OP_BN, n = g.b_k_contig ? e / OP_BK : e % OP_BN;
            sb[k][n] = k < kn && n0 + n < g.N ? *(const float *)(bb + (n0 + n) * g.bnb0 + (k0 + k) * g.bnb1) : 0.0f;
        }
        __syncthreads();
        if (kn == OP_BK) {
#pragma unroll
            for (int k = 0; k < OP_BK; ++k) {
                const float4 a0 = *(const float4 *)&sa[k][tx * 4], a1 = *(const float4 *)&sa[k][64 + tx * 4];
                const float4 b0 = *(const float4 *)&sb[k][ty * 4], b1 = *(const float4 *)&sb[k][64 + ty * 4];
                const float av[OP_TM] = { a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w };
                const float bv[OP_TN] = { b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w };
#pragma unroll
                for (int r = 0; r < OP_TM; ++r)
#pragma unroll
                    for (int c = 0; c < OP_TN; ++c) acc[r][c] = out_prod_step(acc[r][c], av[r], bv[c]);
            }
        } else {                                              // the last, partial slice: only the kn terms K has
            for (int k = 0; k < kn; ++k) {
                const float4 a0 = *(const float4 *)&sa[k][tx * 4], a1 = *(const float4 *)&sa[k][64 + tx * 4];
                const float4 b0 = *(const float4 *)&sb[k][ty * 4], b1 = *(const float4 *)&sb[k][64 + ty * 4];
                const float av[OP_TM] = { a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w };
                const float bv[OP_TN] = { b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w };
#pragma unroll
                for (int r = 0; r < OP_TM; ++r)
#pragma unroll
                    for (int c = 0; c < OP_TN; ++c) acc[r][c] = out_prod_step(acc[r][c], av[r], bv[c]);
            }
        }
        __syncthreads();
    }
    uint8_t * db = dst + i2 * g.dnb2 + i3 * g.dnb3;
#pragma unroll
    for (int c = 0; c < OP_TN; ++c) {
        const int64_t n = n0 + (c < 4 ? ty * 4 + c : 64 + ty * 4 + c - 4);
        if (n >= g.N) continue;
#pragma unroll
        for (int r = 0; r < OP_TM; ++r) {
            const int64_t m = m0 + (r < 4 ? tx * 4 + r : 64 + tx * 4 + r - 4);
            if (m < g.M) *(float *)(db + n * g.dnb1 + m * 4) = acc[r][c];
        }
    }
}

// ------------------------------------------------------------------ reductions of one CTA (CROSS_ENTROPY_LOSS, SUM, COUNT_EQUAL)
// A block-wide sum of doubles / int64s in one fixed order: lane-strided butterflies, then the warp partials in warp order.  Every thread
// gets the result.  blockDim is a multiple of 32.
template <typename V> __device__ __forceinline__ V block_sum_fixed(V v, V * sh) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    __syncthreads();
    if (lane == 0) sh[warp] = v;
    __syncthreads();
    V r = 0;
    for (int w = 0; w < nw; ++w) r += sh[w];
    return r;
}

// CROSS_ENTROPY_LOSS: warp w takes rows w, w + nw, ...; per row the max and the double sum of expf(x - max) by the warp, then the row's
// value (b200_train.cuh, ce_term) summed in double across the lanes and rounded to f32 as ggml_vec_sum_f32 rounds it.  Each warp adds its
// row values in double in row order, the warps' sums are added in warp order and the total is rounded once: a fixed order, no atomics.
__global__ void __launch_bounds__(RED_THREADS) cross_entropy_loss_kernel(tdesc x, tdesc l, float * dst) {
    pdl_trigger();
    __shared__ double sh[RED_THREADS / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    const int64_t nc = x.ne[0], nr = x.ne[1] * x.ne[2] * x.ne[3];
    double wsum = 0.0;
    for (int64_t r = warp; r < nr; r += nw) {
        const int64_t i1 = r % x.ne[1], i2 = (r / x.ne[1]) % x.ne[2], i3 = r / (x.ne[1] * x.ne[2]);
        const float * xr = (const float *)(x.data + i1 * x.nb[1] + i2 * x.nb[2] + i3 * x.nb[3]);
        const float * lr = (const float *)(l.data + i1 * l.nb[1] + i2 * l.nb[2] + i3 * l.nb[3]);
        float mx = -INFINITY;
        for (int64_t i = lane; i < nc; i += 32) mx = fmaxf(mx, xr[i]);
        mx = warp_max(mx);
        double se = 0.0;
        for (int64_t i = lane; i < nc; i += 32) se += (double)expf(pool_add(xr[i], -mx));
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) se += __shfl_xor_sync(0xffffffffu, se, o);
        const float neg_lse = -logf((float)se);
        double rs = 0.0;
        for (int64_t i = lane; i < nc; i += 32) rs += (double)ce_term(xr[i], mx, neg_lse, lr[i]);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) rs += __shfl_xor_sync(0xffffffffu, rs, o);
        wsum += (double)(float)rs;
    }
    const double total = block_sum_fixed(lane == 0 ? wsum : 0.0, sh);         // every lane holds its warp's sum: count it once
    if (threadIdx.x == 0) *dst = pool_mul((float)total, -1.0f / (float)nr);
}

// SUM: each thread adds its elements (lane-strided along dim 0, rows in order) in double; the block adds the threads' sums in a fixed order
// and rounds once, as ggml-cpu's one double accumulator rounds once.
__global__ void __launch_bounds__(RED_THREADS) sum_kernel(tdesc s, float * dst) {
    pdl_trigger();
    __shared__ double sh[RED_THREADS / 32];
    const int64_t ne0 = s.ne[0], nr = s.ne[1] * s.ne[2] * s.ne[3];
    double acc = 0.0;
    if (ne0 >= 32) {
        for (int64_t r = threadIdx.x >> 5; r < nr; r += blockDim.x >> 5) {          // a warp per row
            const int64_t i1 = r % s.ne[1], i2 = (r / s.ne[1]) % s.ne[2], i3 = r / (s.ne[1] * s.ne[2]);
            const float * xr = (const float *)(s.data + i1 * s.nb[1] + i2 * s.nb[2] + i3 * s.nb[3]);
            for (int64_t i = threadIdx.x & 31; i < ne0; i += 32) acc += (double)xr[i];
        }
    } else {                                                                         // short rows: a thread per element
        for (int64_t e = threadIdx.x; e < ne0 * nr; e += blockDim.x) {
            const int64_t i0 = e % ne0, r = e / ne0, i1 = r % s.ne[1], i2 = (r / s.ne[1]) % s.ne[2], i3 = r / (s.ne[1] * s.ne[2]);
            acc += (double)*(const float *)(s.data + i0 * 4 + i1 * s.nb[1] + i2 * s.nb[2] + i3 * s.nb[3]);
        }
    }
    const double total = block_sum_fixed(acc, sh);
    if (threadIdx.x == 0) *dst = (float)total;
}

// COUNT_EQUAL (ne2 == ne3 == 1): the number of equal i32 pairs, counted per thread and added in a fixed order
__global__ void __launch_bounds__(RED_THREADS) count_equal_kernel(tdesc a, tdesc b, int64_t * dst) {
    pdl_trigger();
    __shared__ long long sh[RED_THREADS / 32];
    const int64_t ne0 = a.ne[0], n = ne0 * a.ne[1];
    long long cnt = 0;
    for (int64_t e = threadIdx.x; e < n; e += blockDim.x) {
        const int64_t i0 = e % ne0, i1 = e / ne0;
        cnt += *(const int32_t *)(a.data + i0 * a.nb[0] + i1 * a.nb[1]) == *(const int32_t *)(b.data + i0 * b.nb[0] + i1 * b.nb[1]);
    }
    const long long total = block_sum_fixed(cnt, sh);
    if (threadIdx.x == 0) *dst = (int64_t)total;
}

// ------------------------------------------------------------------ CROSS_ENTROPY_LOSS_BACK (packed rows): one CTA per row
// max, then s = the double sum of e = expf(x - max), inv = (float)(1.0 / s), and dst = (e inv - l) grad[0] / nr (b200_train.cuh).  grad is
// read on the device.
__global__ void cross_entropy_loss_back_kernel(const float * grad, const float * x, const float * l, float * dst, int64_t nc, int64_t nr) {
    pdl_trigger();
    __shared__ float shf[32];
    __shared__ double shd[32];
    const int64_t r = blockIdx.x;
    const float * xr = x + r * nc, * lr = l + r * nc;
    float * yr = dst + r * nc;
    float mx = -INFINITY;
    for (int64_t i = threadIdx.x; i < nc; i += blockDim.x) mx = fmaxf(mx, xr[i]);
    mx = block_reduce<true>(mx, shf);
    double se = 0.0;
    for (int64_t i = threadIdx.x; i < nc; i += blockDim.x) se += (double)expf(pool_add(xr[i], -mx));
    se = block_sum_fixed(se, shd);
    const float inv = (float)(1.0 / se), d_by_nr = pool_div(*grad, (float)nr);
    for (int64_t i = threadIdx.x; i < nc; i += blockDim.x) yr[i] = ce_back_value(expf(pool_add(xr[i], -mx)), inv, lr[i], d_by_nr);
}

// ------------------------------------------------------------------ OPT_STEP_ADAMW (packed, in place): one thread per element
// The seven hyper-parameters are read from device memory by every thread: a captured graph replays with the values of its step.
__global__ void opt_step_adamw_kernel(float * __restrict__ w, const float * __restrict__ g, float * __restrict__ m, float * __restrict__ v,
                                      const float * __restrict__ params, int64_t n) {
    pdl_trigger();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float p[ADAMW_NPARAMS];
#pragma unroll
    for (int j = 0; j < ADAMW_NPARAMS; ++j) p[j] = params[j];
    float wi = w[i], mi = m[i], vi = v[i];
    adamw_update(wi, g[i], mi, vi, p);
    w[i] = wi; m[i] = mi; v[i] = vi;
}

// ------------------------------------------------------------------ ARGMAX (f32 rows -> i32): one CTA per row, the closed form of
// b200_train.cuh in three block-wide passes: the last element that is not NaN, the last NaN before it, then the last-tie argmax between.
__device__ __forceinline__ int32_t block_max_i32(int32_t v, int32_t * sh) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = max(v, __shfl_xor_sync(0xffffffffu, v, o));
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    __syncthreads();
    if (lane == 0) sh[warp] = v;
    __syncthreads();
    int32_t r = -1;
    for (int k = 0; k < nw; ++k) r = max(r, sh[k]);
    return r;
}

__global__ void __launch_bounds__(256) argmax_kernel(const uint8_t * __restrict__ src, int64_t nb1, int32_t * __restrict__ dst, int64_t dnb0_words,
                                                     int32_t ne0) {
    pdl_trigger();
    __shared__ int32_t shi[8];
    __shared__ float shv[8];
    const float * x = (const float *)(src + (int64_t)blockIdx.x * nb1);
    int32_t last = -1;
    for (int32_t i = threadIdx.x; i < ne0; i += blockDim.x) if (!isnan(x[i])) last = i;
    last = block_max_i32(last, shi);
    int32_t nan_before = -1;
    for (int32_t i = threadIdx.x; i < last; i += blockDim.x) if (isnan(x[i])) nan_before = i;
    nan_before = block_max_i32(nan_before, shi);
    float bv = 0.0f;
    int32_t bi = -1;
    for (int32_t i = nan_before + 1 + threadIdx.x; i <= last; i += blockDim.x) if (argmax_beats(x[i], i, bv, bi)) { bv = x[i]; bi = i; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
        const int32_t oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (argmax_beats(ov, oi, bv, bi)) { bv = ov; bi = oi; }
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    __syncthreads();
    if (lane == 0) { shv[warp] = bv; shi[warp] = bi; }
    __syncthreads();
    if (threadIdx.x == 0) {
        float rv = shv[0];
        int32_t ri = shi[0];
        for (int k = 1; k < nw; ++k) if (argmax_beats(shv[k], shi[k], rv, ri)) { rv = shv[k]; ri = shi[k]; }
        dst[(int64_t)blockIdx.x * dnb0_words] = last < 0 ? 0 : ri;
    }
}

// ------------------------------------------------------------------ REPEAT_BACK (f32): one thread per dst element, the repeats in
// ggml-cpu's order (b200_train.cuh)
__global__ void repeat_back_kernel(repeat_back_geom g, const uint8_t * __restrict__ src, uint8_t * __restrict__ dst, int64_t n) {
    pdl_trigger();
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n) return;
    float v;
    const int64_t off = repeat_back_value(g, src, e, &v);
    *(float *)(dst + off) = v;
}

// ------------------------------------------------------------------ ARGSORT (f32 rows of ne0 <= 1024 -> i32 indices, dst contiguous)
// One CTA per row: the row's (key, index) items (b200_sort.cuh), padded to P = the next power of two, are sorted by the bitonic network in
// shared memory, one compare-exchange per thread and step.  The order is a strict total order (ties by index, NaNs last), so each output
// row is a permutation of 0 .. ne0-1: MUL_MAT_ID and GET_ROWS can index with it whatever the router produced.
__global__ void __launch_bounds__(512) argsort_kernel(tdesc s, int32_t * dst, int P, int order) {
    pdl_trigger();
    __shared__ uint64_t items[SORT_MAX_COLS];
    const int64_t r = blockIdx.x, ne0 = s.ne[0];
    const int64_t i1 = r % s.ne[1], i2 = (r / s.ne[1]) % s.ne[2], i3 = r / (s.ne[1] * s.ne[2]);
    const float * x = (const float *)(s.data + i1 * s.nb[1] + i2 * s.nb[2] + i3 * s.nb[3]);
    for (int i = threadIdx.x; i < P; i += blockDim.x) items[i] = i < ne0 ? sort_item(x[i], i, order) : sort_pad(i);
    __syncthreads();
    for (int k = 2; k <= P; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int t = threadIdx.x; t < P / 2; t += blockDim.x) sort_step(items, k, j, t);
            __syncthreads();
        }
    int32_t * d = dst + r * ne0;
    for (int i = threadIdx.x; i < ne0; i += blockDim.x) d[i] = (int32_t)(uint32_t)items[i];
}

// ------------------------------------------------------------------ SUM_ROWS (f32 rows, any strides -> f32 [1, ne1, ne2, ne3])
// One warp per row.  Like ggml_vec_sum_f32 each row is accumulated in double and rounded once to f32; only the order of the f64 additions
// differs (lane-strided partial sums, then a butterfly), so the result equals the CPU's whenever the f64 sum is exact and is otherwise
// at most one f32 ulp apart.
__global__ void __launch_bounds__(128) sum_rows_kernel(tdesc s, tdesc d, int64_t rows) {
    pdl_trigger();
    const int lane = threadIdx.x & 31;
    const int64_t r = (int64_t)blockIdx.x * 4 + (threadIdx.x >> 5);
    if (r >= rows) return;
    const int64_t i1 = r % s.ne[1], i2 = (r / s.ne[1]) % s.ne[2], i3 = r / (s.ne[1] * s.ne[2]);
    const float * x = (const float *)(s.data + i1 * s.nb[1] + i2 * s.nb[2] + i3 * s.nb[3]);
    double acc = 0.0;
    for (int64_t i = lane; i < s.ne[0]; i += 32) acc += (double)x[i];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) *(float *)(d.data + i1 * d.nb[1] + i2 * d.nb[2] + i3 * d.nb[3]) = (float)acc;
}

// ------------------------------------------------------------------ CONCAT (f32 / i32, any dim; src0 dim 0 contiguous, src1 and dst any strides)
// One thread per dst element, in dst's logical order; each copies one 4-byte word, so the result is bit-identical whatever the values.
// In the Mamba layer src1 is TRANSPOSE(x): its nb0 is a row stride.
__global__ void concat_kernel(tdesc a, tdesc b, tdesc d, int dim, int64_t n) {
    pdl_trigger();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int64_t i0 = i % d.ne[0], i1 = (i / d.ne[0]) % d.ne[1], i2 = (i / (d.ne[0] * d.ne[1])) % d.ne[2], i3 = i / (d.ne[0] * d.ne[1] * d.ne[2]);
    const uint8_t * sp;
    if (i0 < a.ne[0] && i1 < a.ne[1] && i2 < a.ne[2] && i3 < a.ne[3]) {
        sp = a.data + i0 * a.nb[0] + i1 * a.nb[1] + i2 * a.nb[2] + i3 * a.nb[3];
    } else {                                                    // src1, shifted back by src0's extent along dim
        sp = b.data + (i0 - (dim == 0 ? a.ne[0] : 0)) * b.nb[0] + (i1 - (dim == 1 ? a.ne[1] : 0)) * b.nb[1] +
                      (i2 - (dim == 2 ? a.ne[2] : 0)) * b.nb[2] + (i3 - (dim == 3 ? a.ne[3] : 0)) * b.nb[3];
    }
    *(uint32_t *)(d.data + i0 * d.nb[0] + i1 * d.nb[1] + i2 * d.nb[2] + i3 * d.nb[3]) = *(const uint32_t *)sp;
}

// ------------------------------------------------------------------ SSM_CONV (conv_x f32 [d_conv - 1 + n_t, d_inner, n_s], rows contiguous)
// One thread per output dst[i1, t, s] (i1 fastest, so the stores coalesce): the d_conv-wide window of conv_x row (i1, s) starting at column
// t, dotted with row i1 of the conv1d weight c [d_conv, d_inner] (b200_ssm.cuh: separately rounded, ascending i0, as ggml-cpu).
__global__ void ssm_conv_kernel(tdesc sx, tdesc c, tdesc d, int64_t n) {
    pdl_trigger();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int64_t i1 = i % d.ne[0], t = (i / d.ne[0]) % d.ne[1], s = i / (d.ne[0] * d.ne[1]);
    const float * win = (const float *)(sx.data + i1 * sx.nb[1] + s * sx.nb[2]) + t;
    const float * w = (const float *)(c.data + i1 * c.nb[1]);
    *(float *)(d.data + i1 * d.nb[0] + t * d.nb[1] + s * d.nb[2]) = ssm_conv_dot(win, w, c.ne[0]);
}

// ------------------------------------------------------------------ SSM_SCAN (the selective scan of Mamba-1)
// One thread per (row i1, sequence s) walks the n_t tokens in order; for each it runs the d_state recurrence of b200_ssm.cuh and writes
// y[i1, t, s] and the row's state, which is read back for the next token (as on the CPU: dst's state part is the running state).  The
// sum over d_state stays a sequential loop in ascending i0 -- spreading it over lanes would change the summation order.  dst holds
// y [d_inner, n_t, n_s] (x's layout) and then, from byte offset x.nb[3], the final states [d_state, d_inner, n_s] (s0's layout).
__global__ void __launch_bounds__(128) ssm_scan_kernel(tdesc s0, tdesc x, tdesc dt, tdesc A, tdesc B, tdesc C, uint8_t * dst) {
    pdl_trigger();
    const int64_t i1 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, s = blockIdx.y;
    if (i1 >= x.ne[0]) return;
    const int64_t nc = s0.ne[0];
    const float * a = (const float *)(A.data + i1 * A.nb[1]);
    const float * prev = (const float *)(s0.data + i1 * s0.nb[1] + s * s0.nb[2]);
    float * st = (float *)(dst + x.nb[3] + i1 * s0.nb[1] + s * s0.nb[2]);
    for (int64_t t = 0; t < x.ne[1]; ++t) {
        const float xv = *(const float *)(x.data + i1 * x.nb[0] + t * x.nb[1] + s * x.nb[2]);
        const float dv = *(const float *)(dt.data + i1 * dt.nb[0] + t * dt.nb[1] + s * dt.nb[2]);
        const float * b = (const float *)(B.data + t * B.nb[1] + s * B.nb[2]);
        const float * cc = (const float *)(C.data + t * C.nb[1] + s * C.nb[2]);
        *(float *)(dst + i1 * x.nb[0] + t * x.nb[1] + s * x.nb[2]) = ssm_scan_token(prev, st, a, b, cc, xv, dv, nc);
        prev = st;
    }
}

// ------------------------------------------------------------------ RWKV_WKV6 / GATED_LINEAR_ATTN (the RWKV-6 recurrence and its gated form)
// One CTA per (block of WKV_COLS state columns, head h, sequence s); one lane per column j walks the S rows i in order (b200_wkv.cuh), so y[j]
// keeps the CPU's summation order with no reduction.  The CTA's columns of the state stay in shared memory across the sequence's tokens,
// lane j touching only column j (conflict-free: the block is stored S x WKV_COLS); it is read from s0 before the first token and written
// to dst's state part after the last.  The token's k, r / q', td / g are staged in shared memory once per token; the next token's are
// loaded into registers while the current one is computed.  Each sequence owns n_seq_tok consecutive tokens, as on the CPU.
// All tensors are packed (check_wkv_common): token t, head h, element i at t * C + h * S + i; state[i][j] of (s, h) at
// ((s * H + h) * S + i) * S + j; dst: y [C, T], then the final states from T * C.
template <bool GLA>
__global__ void __launch_bounds__(WKV_COLS) wkv_kernel(const float * __restrict__ k, const float * __restrict__ v, const float * __restrict__ a,
                                                       const float * __restrict__ b, const float * __restrict__ tf, const float * __restrict__ s0,
                                                       float * __restrict__ dst, int S, int H, int64_t T, int64_t n_seq_tok, float scale) {
    extern __shared__ float wkv_sh[];
    pdl_trigger();
    constexpr int PER = WKV_MAX_HEAD / WKV_COLS;                // staged values per lane and vector
    const int lane = threadIdx.x, j = blockIdx.x * WKV_COLS + lane, h = blockIdx.y, s = blockIdx.z;
    const bool live = j < S;
    const int64_t C = (int64_t)S * H;
    float * st = wkv_sh;                                         // [S][WKV_COLS]
    float * sk = st + (size_t)S * WKV_COLS, * sa = sk + S, * sb = sa + S, * sf = sb + S;

    const int64_t head_state = ((int64_t)s * H + h) * S * S;
    for (int i0 = 0; i0 < S; i0 += WKV_COLS) {                  // WKV_COLS rows' loads in flight at once (a decode step is one token)
        float row[WKV_COLS];
#pragma unroll
        for (int u = 0; u < WKV_COLS; ++u) row[u] = live && i0 + u < S ? s0[head_state + (int64_t)(i0 + u) * S + j] : 0.0f;
#pragma unroll
        for (int u = 0; u < WKV_COLS; ++u) if (i0 + u < S) st[(i0 + u) * WKV_COLS + lane] = row[u];
    }
    if (!GLA) for (int i = lane; i < S; i += WKV_COLS) sf[i] = tf[(int64_t)h * S + i];

    float nk[PER], na[PER], nb[PER], nv = 0.0f;
    auto fetch = [&](int64_t t) {
        const int64_t base = t * C + (int64_t)h * S;
#pragma unroll
        for (int m = 0; m < PER; ++m) {
            const int i = lane + m * WKV_COLS;
            if (i < S) { nk[m] = k[base + i]; na[m] = a[base + i]; nb[m] = b[base + i]; }
        }
        if (live) nv = v[base + j];
    };
    const int64_t t0 = (int64_t)s * n_seq_tok, t1 = t0 + n_seq_tok;
    fetch(t0);
    for (int64_t t = t0; t < t1; ++t) {
        __syncthreads();                                         // the previous token's k / a / b are no longer read
#pragma unroll
        for (int m = 0; m < PER; ++m) {
            const int i = lane + m * WKV_COLS;
            if (i < S) { sk[i] = nk[m]; sa[i] = GLA ? gla_scaled_q(na[m], scale) : na[m]; sb[i] = nb[m]; }
        }
        const float vj = nv;
        __syncthreads();
        if (t + 1 < t1) fetch(t + 1);
        if (live) {
            float * col = st + lane;
            const float y = GLA ? gla_column(sk, sa, sb, vj, col, col, WKV_COLS, S) : wkv6_column(sk, sa, sf, sb, vj, col, col, WKV_COLS, S);
            dst[t * C + (int64_t)h * S + j] = y;
        }
    }
    if (!live) return;
    float * out = dst + T * C + head_state;
    for (int i = 0; i < S; ++i) out[(int64_t)i * S + j] = st[i * WKV_COLS + lane];
}

static inline unsigned blocks_for(int64_t n, int per) { return (unsigned)((n + per - 1) / per); }

} // namespace b200

using namespace b200;

// every launcher below first applies its acceptance rule from b200_op_checks.h (the one supports_op asks)
#define CHECK_ARGS(check) do { const op_check r_ = (check); if (!r_.ok()) { set_error("%s: %s", __func__, r_.reason); return r_.code; } } while (0)

extern "C" {

int ggml_b200_op_get_rows(const ggml_b200_tensor * src0, const ggml_b200_tensor * ids, const ggml_b200_tensor * dst, void * stream) {
    CHECK_ARGS(check_get_rows(src0, ids, dst));
    const tdesc s = T(src0), i = T(ids), d = T(dst);
    const int64_t rows = i.ne[0] * i.ne[1] * i.ne[2];
    if (rows == 0 || s.ne[0] == 0) return GGML_B200_OK;
    B200_CUDA_TRY(launch_pdl(get_rows_kernel, dim3((unsigned)rows), dim3(256), 0, (cudaStream_t)stream, s, i, d));
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

int ggml_b200_op_bin_bcast(int32_t op, const ggml_b200_tensor * src0, const ggml_b200_tensor * src1, const ggml_b200_tensor * dst, void * stream) {
    CHECK_ARGS(check_bin_bcast(op, src0, src1, dst));
    const tdesc a = T(src0), b = T(src1), d = T(dst);
    const int64_t n = nelem(d);
    if (n == 0) return GGML_B200_OK;
    static void (* const kernel[4])(tdesc, tdesc, tdesc, int64_t) = { bin_bcast_kernel<0>, bin_bcast_kernel<1>, bin_bcast_kernel<2>, bin_bcast_kernel<3> };
    B200_CUDA_TRY(launch_pdl(kernel[op], dim3(blocks_for(n, 256)), dim3(256), 0, (cudaStream_t)stream, a, b, d, n));
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

int ggml_b200_op_norm(int32_t rms, const ggml_b200_tensor * src, const ggml_b200_tensor * dst, float eps, void * stream) {
    CHECK_ARGS(check_norm(src, dst));
    const tdesc s = T(src), d = T(dst);
    const int64_t rows = nrows(s);
    if (rows == 0 || s.ne[0] == 0) return GGML_B200_OK;
    const int threads = s.ne[0] >= 1024 ? 256 : s.ne[0] >= 256 ? 128 : 32;
    if (rms) B200_CUDA_TRY(launch_pdl(norm_kernel<true>, dim3((unsigned)rows), dim3(threads), 0, (cudaStream_t)stream, s, d, eps));
    else     B200_CUDA_TRY(launch_pdl(norm_kernel<false>, dim3((unsigned)rows), dim3(threads), 0, (cudaStream_t)stream, s, d, eps));
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

int ggml_b200_op_norm_affine(int32_t rms, const ggml_b200_tensor * src, const ggml_b200_tensor * dst_norm, const ggml_b200_tensor * gain_t,
                             const ggml_b200_tensor * dst_mul, const ggml_b200_tensor * bias_t, const ggml_b200_tensor * dst_add, float eps, void * stream) {
    CHECK_ARGS(check_norm_affine(src, dst_norm, gain_t, dst_mul, bias_t, dst_add));
    const tdesc s = T(src), d1 = T(dst_norm), d2 = T(dst_mul), d3 = T(dst_add);
    const float * gain = (const float *) gain_t->data, * bias = (const float *) bias_t->data;
    const int64_t rows = nrows(s);
    if (rows == 0 || s.ne[0] == 0) return GGML_B200_OK;
    const int threads = s.ne[0] >= 1024 ? 256 : s.ne[0] >= 256 ? 128 : 32;
    if (rms) B200_CUDA_TRY(launch_pdl(norm_affine_kernel<true>, dim3((unsigned)rows), dim3(threads), 0, (cudaStream_t)stream, s, d1, gain, d2, bias, d3, eps));
    else     B200_CUDA_TRY(launch_pdl(norm_affine_kernel<false>, dim3((unsigned)rows), dim3(threads), 0, (cudaStream_t)stream, s, d1, gain, d2, bias, d3, eps));
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

int ggml_b200_op_scale(const ggml_b200_tensor * src, const ggml_b200_tensor * dst, float s, void * stream) {
    CHECK_ARGS(check_scale(src, dst));
    const int64_t n = nelem(*dst);
    if (n == 0) return GGML_B200_OK;
    B200_CUDA_TRY(launch_pdl(scale_kernel, dim3(blocks_for(n, 256)), dim3(256), 0, (cudaStream_t)stream, (const float *)src->data, (float *)dst->data, s, n));
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

int ggml_b200_op_diag_mask_inf(const ggml_b200_tensor * src, const ggml_b200_tensor * dst, int32_t n_past, void * stream) {
    CHECK_ARGS(check_diag_mask_inf(src, dst));
    const int64_t n = nelem(*dst);
    if (n == 0) return GGML_B200_OK;
    B200_CUDA_TRY(launch_pdl(diag_mask_inf_kernel, dim3(blocks_for(n, 256)), dim3(256), 0, (cudaStream_t)stream, (const float *)src->data, (float *)dst->data,
                             dst->ne[0], dst->ne[1], n_past, n));
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

int ggml_b200_op_unary(int32_t uop, const ggml_b200_tensor * src, const ggml_b200_tensor * dst, void * stream) {
    CHECK_ARGS(check_unary(uop, src, dst));
    const int64_t n = nelem(*dst);
    if (n == 0) return GGML_B200_OK;
    B200_CUDA_TRY(launch_pdl(unary_kernel, dim3(blocks_for(n, 256)), dim3(256), 0, (cudaStream_t)stream, uop, (const float *)src->data, (float *)dst->data, n));
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

int ggml_b200_op_soft_max(const ggml_b200_tensor * src, const ggml_b200_tensor * mask, const ggml_b200_tensor * dst, float scale, float max_bias,
                          int32_t diag_n_past, void * stream) {
    CHECK_ARGS(check_soft_max(src, mask, dst));
    const int64_t ne0 = src->ne[0], ne1 = src->ne[1], ne2 = src->ne[2], rows = nrows(*src);
    if (rows == 0 || ne0 == 0) return GGML_B200_OK;
    const uint32_t n_head = (uint32_t)ne2;
    uint32_t n_head_log2 = 1; while (n_head_log2 * 2 <= n_head) n_head_log2 *= 2;
    const float m0 = powf(2.0f, -(max_bias) / n_head_log2), m1 = powf(2.0f, -(max_bias / 2.0f) / n_head_log2);
    const int threads = ne0 >= 1024 ? 256 : ne0 >= 128 ? 128 : 32;
    const uint8_t * mp = mask ? (const uint8_t *)mask->data : nullptr;
    const int mask_type = mask ? mask->type : 0;
    B200_CUDA_TRY(launch_pdl(soft_max_kernel, dim3((unsigned)rows), dim3(threads), 0, (cudaStream_t)stream, (const float *)src->data, mp, mask_type,
                             (float *)dst->data, ne0, ne1, ne2, scale, max_bias, m0, m1, n_head_log2, (int)diag_n_past));
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

int ggml_b200_op_cpy(const ggml_b200_tensor * src, const ggml_b200_tensor * dst, void * stream) {
    CHECK_ARGS(check_cpy(src, dst));
    const tdesc s = T(src), d = T(dst);
    const int64_t n = nelem(s);
    if (n == 0) return GGML_B200_OK;
    cudaStream_t st = (cudaStream_t)stream;
    if (d.type == T_F32 || d.type == T_F16) {
        B200_CUDA_TRY(launch_pdl(cpy_kernel, dim3(blocks_for(n, 256)), dim3(256), 0, st, s, d, s, d, n));
    } else {                                                    // f32 -> Q8_0 / Q4_0
        const int64_t nb = n / 32;
        if (d.type == T_Q8_0) B200_CUDA_TRY(launch_pdl(cpy_f32_q_kernel<T_Q8_0>, dim3(blocks_for(nb, 128)), dim3(128), 0, st, s, d, nb));
        else                  B200_CUDA_TRY(launch_pdl(cpy_f32_q_kernel<T_Q4_0>, dim3(blocks_for(nb, 128)), dim3(128), 0, st, s, d, nb));
    }
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

int ggml_b200_op_cpy2(const ggml_b200_tensor * src_a, const ggml_b200_tensor * dst_a, const ggml_b200_tensor * src_b, const ggml_b200_tensor * dst_b, void * stream) {
    CHECK_ARGS(check_cpy2(src_a, dst_a, src_b, dst_b));
    const tdesc s = T(src_a), d = T(dst_a), s2 = T(src_b), d2 = T(dst_b);
    const int64_t n = nelem(s);
    if (n == 0) return GGML_B200_OK;
    B200_CUDA_TRY(launch_pdl(cpy_kernel, dim3(blocks_for(n, 256), 2), dim3(256), 0, (cudaStream_t)stream, s, d, s2, d2, n));
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

int ggml_b200_op_flash_attn_ext(const ggml_b200_tensor * q, const ggml_b200_tensor * k, const ggml_b200_tensor * v, const ggml_b200_tensor * mask,
                                const ggml_b200_tensor * dst, float scale, float max_bias, float logit_softcap, void * stream) {
    CHECK_ARGS(check_flash_attn_ext(q, k, v, mask, dst));
    fa_params p;
    p.q = T(q); p.k = T(k); p.v = T(v); p.dst = T(dst);
    if (mask) p.mask = T(mask); else { p.mask = tdesc{}; p.mask.data = nullptr; }
    if (p.q.ne[1] == 0 || p.q.ne[2] == 0 || p.q.ne[3] == 0) return GGML_B200_OK;
    p.scale = scale; p.max_bias = max_bias; p.softcap = logit_softcap;
    if (logit_softcap != 0.0f) p.scale /= logit_softcap;
    const uint32_t n_head = (uint32_t)p.q.ne[2];
    uint32_t n_head_log2 = 1; while (n_head_log2 * 2 <= n_head) n_head_log2 *= 2;
    p.n_head_log2 = n_head_log2;
    p.m0 = powf(2.0f, -(max_bias) / n_head_log2); p.m1 = powf(2.0f, -(max_bias / 2.0f) / n_head_log2);
    B200_CUDA_TRY(launch_pdl(flash_attn_ext_kernel, dim3((unsigned)p.q.ne[1], (unsigned)p.q.ne[2], (unsigned)p.q.ne[3]), dim3(128), 0, (cudaStream_t)stream, p));
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

int ggml_b200_op_mul_mat_f(const ggml_b200_tensor * src0, const ggml_b200_tensor * src1, const ggml_b200_tensor * dst, void * stream) {
    CHECK_ARGS(check_mul_mat_f(src0, src1, dst));
    const tdesc a = T(src0), b = T(src1), d = T(dst);
    const int64_t nout = nelem(d);
    if (nout == 0) return GGML_B200_OK;
    B200_CUDA_TRY(launch_pdl(mul_mat_f_kernel, dim3(blocks_for(nout, 4)), dim3(128), 0, (cudaStream_t)stream, a, b, d, nout));
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

int ggml_b200_op_rope(const ggml_b200_tensor * src, const ggml_b200_tensor * pos, const ggml_b200_tensor * freq_factors, const ggml_b200_tensor * dst,
                      const ggml_b200_rope_params * params, void * stream) {
    CHECK_ARGS(check_rope(src, pos, freq_factors, dst, params));
    const tdesc s = T(src), p = T(pos), d = T(dst);
    const rope_consts & c = *params;
    const float * ff = freq_factors ? (const float *)freq_factors->data : nullptr;
    if (s.ne[0] == 0 || s.ne[1] == 0 || s.ne[2] == 0 || s.ne[3] == 0) return GGML_B200_OK;
    const int heads_per_cta = rope_heads_per_cta(s.ne[0]);
    const int64_t hb = (s.ne[1] + heads_per_cta - 1) / heads_per_cta;
    const dim3 grid((unsigned)s.ne[2], (unsigned)hb, (unsigned)s.ne[3]);
    if (s.type == T_F32) B200_CUDA_TRY(launch_pdl(rope_kernel<float>, grid, dim3(128), 0, (cudaStream_t)stream, s, (const int32_t *)p.data, ff, d, c, heads_per_cta));
    else                 B200_CUDA_TRY(launch_pdl(rope_kernel<__half>, grid, dim3(128), 0, (cudaStream_t)stream, s, (const int32_t *)p.data, ff, d, c, heads_per_cta));
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

int ggml_b200_op_im2col(const ggml_b200_tensor * src0, const ggml_b200_tensor * src1, const ggml_b200_tensor * dst, const ggml_b200_im2col_params * params,
                        void * stream) {
    CHECK_ARGS(check_im2col(src0, src1, dst, params));
    const int64_t n = nelem(*dst);
    if (n == 0) return GGML_B200_OK;
    const im2col_geom g = im2col_geometry(*src0, *src1, *dst, *params);
    const uint8_t * x = (const uint8_t *)src1->data;
    if (dst->type == T_F32) B200_CUDA_TRY(launch_pdl(im2col_kernel<float>, dim3(blocks_for(n, 256)), dim3(256), 0, (cudaStream_t)stream, g, x, (float *)dst->data, n));
    else                    B200_CUDA_TRY(launch_pdl(im2col_kernel<__half>, dim3(blocks_for(n, 256)), dim3(256), 0, (cudaStream_t)stream, g, x, (__half *)dst->data, n));
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

int ggml_b200_op_pool_2d(const ggml_b200_tensor * src, const ggml_b200_tensor * dst, const ggml_b200_pool_params * params, void * stream) {
    CHECK_ARGS(check_pool_2d(src, dst, params));
    const int64_t n = nelem(*dst);
    if (n == 0) return GGML_B200_OK;
    const pool2d_geom g = pool2d_geometry(*src, *dst, *params);
    B200_CUDA_TRY(launch_pdl(pool2d_kernel, dim3(blocks_for(n, 256)), dim3(256), 0, (cudaStream_t)stream, g, (const uint8_t *)src->data, (float *)dst->data, n));
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

int ggml_b200_op_upscale(const ggml_b200_tensor * src, const ggml_b200_tensor * dst, void * stream) {
    CHECK_ARGS(check_upscale(src, dst));
    const int64_t n = nelem(*dst);
    if (n == 0) return GGML_B200_OK;
    const upscale_geom g = upscale_geometry(*src, *dst);
    B200_CUDA_TRY(launch_pdl(upscale_kernel, dim3(blocks_for(n, 256)), dim3(256), 0, (cudaStream_t)stream, g, (const uint8_t *)src->data, (uint8_t *)dst->data, n));
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

int ggml_b200_op_leaky_relu(const ggml_b200_tensor * src, const ggml_b200_tensor * dst, float slope, void * stream) {
    CHECK_ARGS(check_leaky_relu(src, dst));
    const tdesc s = T(src), d = T(dst);
    const int64_t n = nelem(d);
    if (n == 0) return GGML_B200_OK;
    B200_CUDA_TRY(launch_pdl(leaky_relu_kernel, dim3(blocks_for(n, 256)), dim3(256), 0, (cudaStream_t)stream, s, d, slope, n));
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

int ggml_b200_op_repeat(const ggml_b200_tensor * src, const ggml_b200_tensor * dst, void * stream) {
    CHECK_ARGS(check_repeat(src, dst));
    const int64_t n = nelem(*dst);
    if (n == 0) return GGML_B200_OK;
    const repeat_geom g = repeat_geometry(*src, *dst);
    const uint8_t * s = (const uint8_t *)src->data;
    uint8_t * d = (uint8_t *)dst->data;
    if (repeat_elem_size(src->type) == 4) B200_CUDA_TRY(launch_pdl(repeat_kernel<uint32_t>, dim3(blocks_for(n, 256)), dim3(256), 0, (cudaStream_t)stream, g, s, d, n));
    else                                  B200_CUDA_TRY(launch_pdl(repeat_kernel<uint16_t>, dim3(blocks_for(n, 256)), dim3(256), 0, (cudaStream_t)stream, g, s, d, n));
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

// the row kernels' block: ne0 threads rounded up to a warp, at most 256 (the checks bound the row's blocks by 65535)
static inline int row_threads(int64_t ne0) { return (int)std::min<int64_t>(256, (ne0 + 31) / 32 * 32); }

int ggml_b200_op_win_part(const ggml_b200_tensor * src, const ggml_b200_tensor * dst, int32_t npx, int32_t npy, int32_t w, void * stream) {
    CHECK_ARGS(check_win_part(src, dst, npx, npy, w));
    if (nelem(*dst) == 0) return GGML_B200_OK;
    const win_geom g{ w, npx, (int32_t)src->ne[1], (int32_t)src->ne[2] };
    const int64_t ne0 = dst->ne[0];
    const int th = row_threads(ne0);
    B200_CUDA_TRY(launch_pdl(win_part_kernel, dim3((unsigned)nrows(*dst), blocks_for(ne0, th)), dim3(th), 0, (cudaStream_t)stream, g,
                             (const uint32_t *)src->data, (uint32_t *)dst->data, ne0));
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

int ggml_b200_op_win_unpart(const ggml_b200_tensor * src, const ggml_b200_tensor * dst, int32_t w, void * stream) {
    CHECK_ARGS(check_win_unpart(src, dst, w));
    if (nelem(*dst) == 0) return GGML_B200_OK;
    const win_geom g{ w, (int32_t)((dst->ne[1] + w - 1) / w), (int32_t)dst->ne[1], (int32_t)dst->ne[2] };
    const int64_t ne0 = dst->ne[0];
    const int th = row_threads(ne0);
    B200_CUDA_TRY(launch_pdl(win_unpart_kernel, dim3((unsigned)nrows(*dst), blocks_for(ne0, th)), dim3(th), 0, (cudaStream_t)stream, g,
                             (const uint32_t *)src->data, (uint32_t *)dst->data, ne0));
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

int ggml_b200_op_get_rel_pos(const ggml_b200_tensor * src, const ggml_b200_tensor * dst, void * stream) {
    CHECK_ARGS(check_get_rel_pos(src, dst));
    if (nelem(*dst) == 0) return GGML_B200_OK;
    const int64_t ne0 = dst->ne[0];
    const int th = row_threads(ne0);
    B200_CUDA_TRY(launch_pdl(get_rel_pos_kernel, dim3((unsigned)nrows(*dst), blocks_for(ne0, th)), dim3(th), 0, (cudaStream_t)stream,
                             (uint32_t)dst->ne[1], (const uint16_t *)src->data, (uint16_t *)dst->data, ne0));
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

int ggml_b200_op_add_rel_pos(const ggml_b200_tensor * src0, const ggml_b200_tensor * pw, const ggml_b200_tensor * ph, const ggml_b200_tensor * dst,
                             void * stream) {
    CHECK_ARGS(check_add_rel_pos(src0, pw, ph, dst));
    if (nelem(*dst) == 0) return GGML_B200_OK;
    const uint32_t L = (uint32_t)pw->ne[0], LL = (uint32_t)dst->ne[0];
    const float * s = (const float *)src0->data, * w = (const float *)pw->data, * h = (const float *)ph->data;
    float * d = (float *)dst->data;
    const dim3 rows((unsigned)nrows(*dst));
    cudaStream_t st = (cudaStream_t)stream;
    if (LL % 4 == 0 && ((uintptr_t)s % 16) == 0 && ((uintptr_t)d % 16) == 0) {
        const int th = row_threads(LL / 4);
        B200_CUDA_TRY(launch_pdl(add_rel_pos_kernel<4>, dim3(rows.x, blocks_for(LL / 4, th)), dim3(th), 0, st, s, w, h, d, L, LL));
    } else {
        const int th = row_threads(LL);
        B200_CUDA_TRY(launch_pdl(add_rel_pos_kernel<1>, dim3(rows.x, blocks_for(LL, th)), dim3(th), 0, st, s, w, h, d, L, LL));
    }
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

int ggml_b200_op_conv_transpose_2d(const ggml_b200_tensor * kernel, const ggml_b200_tensor * input, const ggml_b200_tensor * dst, int32_t stride,
                                   void * stream) {
    CHECK_ARGS(check_conv_transpose_2d(kernel, input, dst, stride));
    if (nelem(*dst) == 0) return GGML_B200_OK;
    const ct2d_geom g = ct2d_geometry(*kernel, *input, *dst, stride);
    const int64_t nq_x = (g.OW + stride - 1) / stride, nq_y = (g.OH + stride - 1) / stride;      // outputs of the largest phase
    const unsigned tiles = blocks_for(nq_x, CT2D_TQX) * blocks_for(nq_y, CT2D_TQY);
    const dim3 grid(tiles, blocks_for(g.Cout, CT2D_CO), (unsigned)(stride * stride));
    B200_CUDA_TRY(launch_pdl(ct2d_kernel, grid, dim3(CT2D_THREADS), 0, (cudaStream_t)stream, g, (const uint8_t *)kernel->data,
                             (const uint8_t *)input->data, (float *)dst->data));
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

int ggml_b200_op_argsort(const ggml_b200_tensor * src, const ggml_b200_tensor * dst, int32_t order, void * stream) {
    CHECK_ARGS(check_argsort(src, dst, order));
    const tdesc s = T(src), d = T(dst);
    const int64_t rows = nrows(s);
    if (rows == 0 || s.ne[0] == 0) return GGML_B200_OK;
    const int P = sort_width((int)s.ne[0]);
    const int threads = std::max(32, std::min(512, P / 2));
    B200_CUDA_TRY(launch_pdl(argsort_kernel, dim3((unsigned)rows), dim3(threads), 0, (cudaStream_t)stream, s, (int32_t *)d.data, P, (int)order));
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

int ggml_b200_op_sum_rows(const ggml_b200_tensor * src, const ggml_b200_tensor * dst, void * stream) {
    CHECK_ARGS(check_sum_rows(src, dst));
    const tdesc s = T(src), d = T(dst);
    const int64_t rows = nrows(s);
    if (rows == 0) return GGML_B200_OK;
    B200_CUDA_TRY(launch_pdl(sum_rows_kernel, dim3(blocks_for(rows, 4)), dim3(128), 0, (cudaStream_t)stream, s, d, rows));
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

int ggml_b200_op_concat(const ggml_b200_tensor * src0, const ggml_b200_tensor * src1, const ggml_b200_tensor * dst, int32_t dim, void * stream) {
    CHECK_ARGS(check_concat(src0, src1, dst, dim));
    const tdesc a = T(src0), b = T(src1), d = T(dst);
    const int64_t n = nelem(d);
    if (n == 0) return GGML_B200_OK;
    B200_CUDA_TRY(launch_pdl(concat_kernel, dim3(blocks_for(n, 256)), dim3(256), 0, (cudaStream_t)stream, a, b, d, (int)dim, n));
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

int ggml_b200_op_ssm_conv(const ggml_b200_tensor * sx, const ggml_b200_tensor * c, const ggml_b200_tensor * dst, void * stream) {
    CHECK_ARGS(check_ssm_conv(sx, c, dst));
    const tdesc x = T(sx), w = T(c), d = T(dst);
    const int64_t n = nelem(d);
    if (n == 0) return GGML_B200_OK;
    B200_CUDA_TRY(launch_pdl(ssm_conv_kernel, dim3(blocks_for(n, 256)), dim3(256), 0, (cudaStream_t)stream, x, w, d, n));
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

int ggml_b200_op_ssm_scan(const ggml_b200_tensor * s, const ggml_b200_tensor * x, const ggml_b200_tensor * dt, const ggml_b200_tensor * A,
                          const ggml_b200_tensor * B, const ggml_b200_tensor * C, const ggml_b200_tensor * dst, void * stream) {
    CHECK_ARGS(check_ssm_scan(s, x, dt, A, B, C, dst));
    const tdesc ts = T(s), tx = T(x), tdt = T(dt), ta = T(A), tb = T(B), tc = T(C), d = T(dst);
    const int64_t d_inner = ts.ne[1], n_s = ts.ne[2];
    if (d_inner == 0 || n_s == 0) return GGML_B200_OK;
    B200_CUDA_TRY(launch_pdl(ssm_scan_kernel, dim3(blocks_for(d_inner, 128), (unsigned)n_s), dim3(128), 0, (cudaStream_t)stream, ts, tx, tdt, ta, tb, tc,
                             (uint8_t *)d.data));
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

} // extern "C"

// the one launch of RWKV_WKV6 (GLA false: a = r, b = td) and GATED_LINEAR_ATTN (GLA true: a = q, b = g, tf unused), after their check
template <bool GLA>
static int launch_wkv(const ggml_b200_tensor * k, const ggml_b200_tensor * v, const ggml_b200_tensor * a, const ggml_b200_tensor * b,
                      const ggml_b200_tensor * tf, const ggml_b200_tensor * s, const ggml_b200_tensor * dst, float scale, void * stream) {
    const int64_t S = k->ne[0], H = k->ne[1], T = k->ne[2], n_seqs = s->ne[1];
    if (T == 0 || S == 0) return GGML_B200_OK;
    const dim3 grid(blocks_for(S, WKV_COLS), (unsigned)H, (unsigned)n_seqs);
    B200_CUDA_TRY(launch_pdl(wkv_kernel<GLA>, grid, dim3(WKV_COLS), wkv_smem_bytes(S), (cudaStream_t)stream, (const float *)k->data, (const float *)v->data,
                             (const float *)a->data, (const float *)b->data, tf ? (const float *)tf->data : nullptr, (const float *)s->data, (float *)dst->data,
                             (int)S, (int)H, T, T / n_seqs, scale));
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

extern "C" {

int ggml_b200_op_rwkv_wkv6(const ggml_b200_tensor * k, const ggml_b200_tensor * v, const ggml_b200_tensor * r, const ggml_b200_tensor * tf,
                           const ggml_b200_tensor * td, const ggml_b200_tensor * s, const ggml_b200_tensor * dst, void * stream) {
    CHECK_ARGS(check_rwkv_wkv6(k, v, r, tf, td, s, dst));
    return launch_wkv<false>(k, v, r, td, tf, s, dst, 1.0f, stream);
}

int ggml_b200_op_gated_linear_attn(const ggml_b200_tensor * k, const ggml_b200_tensor * v, const ggml_b200_tensor * q, const ggml_b200_tensor * g,
                                   const ggml_b200_tensor * s, const ggml_b200_tensor * dst, float scale, void * stream) {
    CHECK_ARGS(check_gated_linear_attn(k, v, q, g, s, dst));
    return launch_wkv<true>(k, v, q, g, nullptr, s, dst, scale, stream);
}

// ------------------------------------------------------------------ the ops of ggml_opt's backward and optimizer graphs
int ggml_b200_op_out_prod(const ggml_b200_tensor * src0, const ggml_b200_tensor * src1, const ggml_b200_tensor * dst, void * stream) {
    CHECK_ARGS(check_out_prod(src0, src1, dst));
    if (nelem(*dst) == 0) return GGML_B200_OK;
    out_prod_geom g;
    g.M = dst->ne[0]; g.N = dst->ne[1]; g.K = src0->ne[1];
    g.ne2 = dst->ne[2]; g.dps2 = dst->ne[2] / src0->ne[2]; g.dps3 = dst->ne[3] / src0->ne[3];
    g.anb1 = (int64_t)src0->nb[1]; g.anb2 = (int64_t)src0->nb[2]; g.anb3 = (int64_t)src0->nb[3];
    g.bnb0 = (int64_t)src1->nb[0]; g.bnb1 = (int64_t)src1->nb[1]; g.bnb2 = (int64_t)src1->nb[2]; g.bnb3 = (int64_t)src1->nb[3];
    g.dnb1 = (int64_t)dst->nb[1]; g.dnb2 = (int64_t)dst->nb[2]; g.dnb3 = (int64_t)dst->nb[3];
    g.b_k_contig = src1->nb[0] != 4 && src1->nb[1] == 4;
    const dim3 grid(blocks_for(g.M, OP_BM), blocks_for(g.N, OP_BN), (unsigned)(dst->ne[2] * dst->ne[3]));
    B200_CUDA_TRY(launch_pdl(out_prod_kernel, grid, dim3(OP_THREADS), 0, (cudaStream_t)stream, g, (const uint8_t *)src0->data,
                             (const uint8_t *)src1->data, (uint8_t *)dst->data));
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

int ggml_b200_op_cross_entropy_loss(const ggml_b200_tensor * logits, const ggml_b200_tensor * labels, const ggml_b200_tensor * dst, void * stream) {
    CHECK_ARGS(check_cross_entropy_loss(logits, labels, dst));
    B200_CUDA_TRY(launch_pdl(cross_entropy_loss_kernel, dim3(1), dim3(RED_THREADS), 0, (cudaStream_t)stream, T(logits), T(labels), (float *)dst->data));
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

int ggml_b200_op_cross_entropy_loss_back(const ggml_b200_tensor * grad, const ggml_b200_tensor * logits, const ggml_b200_tensor * labels,
                                         const ggml_b200_tensor * dst, void * stream) {
    CHECK_ARGS(check_cross_entropy_loss_back(grad, logits, labels, dst));
    if (nelem(*dst) == 0) return GGML_B200_OK;
    const int64_t nc = dst->ne[0], nr = nrows(*dst);
    const int threads = (int)std::min<int64_t>(1024, std::max<int64_t>(32, (nc + 31) / 32 * 32));
    B200_CUDA_TRY(launch_pdl(cross_entropy_loss_back_kernel, dim3((unsigned)nr), dim3(threads), 0, (cudaStream_t)stream, (const float *)grad->data,
                             (const float *)logits->data, (const float *)labels->data, (float *)dst->data, nc, nr));
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

int ggml_b200_op_opt_step_adamw(const ggml_b200_tensor * w, const ggml_b200_tensor * g, const ggml_b200_tensor * m, const ggml_b200_tensor * v,
                                const ggml_b200_tensor * params, void * stream) {
    CHECK_ARGS(check_opt_step_adamw(w, g, m, v, params));
    const int64_t n = nelem(*w);
    if (n == 0) return GGML_B200_OK;
    B200_CUDA_TRY(launch_pdl(opt_step_adamw_kernel, dim3(blocks_for(n, 256)), dim3(256), 0, (cudaStream_t)stream, (float *)w->data,
                             (const float *)g->data, (float *)m->data, (float *)v->data, (const float *)params->data, n));
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

int ggml_b200_op_argmax(const ggml_b200_tensor * src, const ggml_b200_tensor * dst, void * stream) {
    CHECK_ARGS(check_argmax(src, dst));
    if (src->ne[1] == 0) return GGML_B200_OK;
    B200_CUDA_TRY(launch_pdl(argmax_kernel, dim3((unsigned)src->ne[1]), dim3(256), 0, (cudaStream_t)stream, (const uint8_t *)src->data,
                             (int64_t)src->nb[1], (int32_t *)dst->data, (int64_t)(dst->nb[0] / 4), (int32_t)src->ne[0]));
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

int ggml_b200_op_count_equal(const ggml_b200_tensor * src0, const ggml_b200_tensor * src1, const ggml_b200_tensor * dst, void * stream) {
    CHECK_ARGS(check_count_equal(src0, src1, dst));
    B200_CUDA_TRY(launch_pdl(count_equal_kernel, dim3(1), dim3(RED_THREADS), 0, (cudaStream_t)stream, T(src0), T(src1), (int64_t *)dst->data));
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

int ggml_b200_op_sum(const ggml_b200_tensor * src, const ggml_b200_tensor * dst, void * stream) {
    CHECK_ARGS(check_sum(src, dst));
    B200_CUDA_TRY(launch_pdl(sum_kernel, dim3(1), dim3(RED_THREADS), 0, (cudaStream_t)stream, T(src), (float *)dst->data));
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

int ggml_b200_op_repeat_back(const ggml_b200_tensor * src, const ggml_b200_tensor * dst, void * stream) {
    CHECK_ARGS(check_repeat_back(src, dst));
    const int64_t n = nelem(*dst);
    if (n == 0) return GGML_B200_OK;
    B200_CUDA_TRY(launch_pdl(repeat_back_kernel, dim3(blocks_for(n, 256)), dim3(256), 0, (cudaStream_t)stream, repeat_back_geometry(*src, *dst),
                             (const uint8_t *)src->data, (uint8_t *)dst->data, n));
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

} // extern "C"
