// mmid.cu — GGML_OP_MUL_MAT_ID (mixture-of-experts mat-mul) for sm_90a.
//
// Computes what ggml_compute_forward_mul_mat_id (reference src/ggml-cpu/ggml-cpu.c:7609-7784) computes and
// replaces ggml_cuda_mul_mat_id (src/ggml-cuda/ggml-cuda.cu:1955-2090), which copies `ids` to the host and
// synchronises the stream to build per-expert row lists.  Here routing stays on the device: every output
// vector dst[t][e][:] = as[ids[t][e]] . b[t][e % nb1cols] is an independent quantized mat-vec whose expert
// index is read by the kernel itself, so the op is one quantize launch + one mat-vec launch, no host sync.
#include "b200_internal.h"
#include "b200_quants.cuh"
#include "b200_iq.cuh"

namespace b200 {

struct mmid_params {
    const uint8_t * w; const uint8_t * recs; const uint8_t * ids; float * y;
    int64_t K, M, n_expert, n_used, nb1cols, n_tok;
    size_t  nb01, nb02, ids_nb1;
    act_layout L;
    int64_t nrg;
};

__device__ __forceinline__ float warp_sum_id(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

template <int T>
__global__ void __launch_bounds__(128) mmid_kernel(mmid_params p) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t rg = blockIdx.x % p.nrg, pair = blockIdx.x / p.nrg;     // pair = t * n_used + e
    const int64_t m = rg * 4 + warp;
    if (m >= p.M) return;
    const int64_t t = pair / p.n_used, e = pair % p.n_used;
    const int32_t x = *(const int32_t *)(p.ids + t * p.ids_nb1 + e * 4);
    float acc = 0.0f;
    if (x >= 0 && x < p.n_expert) {      // the reference asserts this; an invalid id yields 0 instead of a fault
        const uint8_t * row = p.w + (size_t)x * p.nb02 + m * p.nb01;
        const uint8_t * rec = p.recs + (size_t)(t * p.nb1cols + (e % p.nb1cols)) * p.L.bytes;
        const int nunits = (int)(p.K / 64);
        for (int u = lane; u < nunits; u += 32) {
            unit_act A;
            load_unit_act<T>(rec, p.L, u, A);
            acc += unit_dot<T>(row, u, A);
        }
        if constexpr (fmt<T>::QK == 32) {
            if ((p.K & 63) != 0 && lane == 0) acc += tail_block_dot<T>(row + (size_t)nunits * 2 * fmt<T>::BYTES, rec, p.L, nunits * 2);
        }
    }
    acc = warp_sum_id(acc);
    if (lane == 0) p.y[(size_t)pair * p.M + m] = acc;
}

} // namespace b200

using namespace b200;

extern "C" {

size_t ggml_b200_mul_mat_id_workspace_size(const ggml_b200_mul_mat_id_args * a) {
    if (!a || type_bytes(a->type) == 0 || a->K <= 0) return 0;
    if (mmid_grouped_eligible(*a)) return mmid_grouped_workspace(*a);
    return (size_t)make_act_layout(a->K, type_is_kquant(a->type)).bytes * (size_t)(a->nb1cols * a->n_tok) + 64;
}

int ggml_b200_mul_mat_id(const ggml_b200_mul_mat_id_args * a, void * stream) {
    if (!a) { set_error("mul_mat_id: NULL args"); return GGML_B200_EINVAL; }
    if (type_bytes(a->type) == 0) { set_error("mul_mat_id: unsupported weight type %d", a->type); return GGML_B200_EUNSUPPORTED; }
    if (a->K <= 0 || a->K % type_qk(a->type) != 0 || a->M < 0 || a->n_expert < 1 || a->n_used < 1 || a->nb1cols < 1 || a->n_tok < 0) { set_error("mul_mat_id: bad shape"); return GGML_B200_EINVAL; }
    if (a->M == 0 || a->n_tok == 0) return GGML_B200_OK;
    if (!a->src0 || !a->src1 || !a->ids || !a->dst) { set_error("mul_mat_id: NULL tensor pointer"); return GGML_B200_EINVAL; }
    if ((a->nb11 & 3) || (a->nb12 & 3) || (a->ids_nb1 & 3) || (a->nb01 & 1) || (a->nb02 & 1)) { set_error("mul_mat_id: bad strides"); return GGML_B200_EINVAL; }
    if ((a->type == T_Q4_K || a->type == T_Q5_K) && (((uintptr_t)a->src0 | a->nb01 | a->nb02) & 15)) { set_error("mul_mat_id: Q4_K/Q5_K rows must be 16-byte aligned"); return GGML_B200_EINVAL; }
    const size_t need = ggml_b200_mul_mat_id_workspace_size(a);
    if (!a->workspace || a->workspace_size < need) { set_error("mul_mat_id: workspace %zu < %zu", a->workspace_size, need); return GGML_B200_EWORKSPACE; }
    cudaStream_t st = (cudaStream_t)stream;
    if (mmid_grouped_eligible(*a)) return launch_mmid_grouped(*a, st);      // batched tokens: rows grouped per expert on the device, tensor cores
    // b[K, nb1cols, n_tok] -> records indexed t * nb1cols + c
    int rc = launch_quantize_activations(a->type, a->src1, a->K, a->nb1cols, a->n_tok, 1, a->nb11, a->nb12, 0, a->workspace, st);
    if (rc != GGML_B200_OK) return rc;
    mmid_params p;
    p.w = (const uint8_t *)a->src0; p.recs = (const uint8_t *)a->workspace; p.ids = (const uint8_t *)a->ids; p.y = a->dst;
    p.K = a->K; p.M = a->M; p.n_expert = a->n_expert; p.n_used = a->n_used; p.nb1cols = a->nb1cols; p.n_tok = a->n_tok;
    p.nb01 = a->nb01; p.nb02 = a->nb02; p.ids_nb1 = a->ids_nb1;
    p.L = make_act_layout(a->K, type_is_kquant(a->type));
    p.nrg = (a->M + 3) / 4;
    const int64_t nblk = p.nrg * a->n_used * a->n_tok;
    if (nblk > 0x7fffffffLL) { set_error("mul_mat_id: grid too large"); return GGML_B200_EUNSUPPORTED; }
    switch (a->type) {
        case T_Q4_0: mmid_kernel<T_Q4_0><<<(unsigned)nblk, 128, 0, st>>>(p); break;
        case T_Q8_0: mmid_kernel<T_Q8_0><<<(unsigned)nblk, 128, 0, st>>>(p); break;
        case T_Q4_K: mmid_kernel<T_Q4_K><<<(unsigned)nblk, 128, 0, st>>>(p); break;
        case T_Q5_K: mmid_kernel<T_Q5_K><<<(unsigned)nblk, 128, 0, st>>>(p); break;
        case T_Q6_K: mmid_kernel<T_Q6_K><<<(unsigned)nblk, 128, 0, st>>>(p); break;
        case T_Q4_1: mmid_kernel<T_Q4_1><<<(unsigned)nblk, 128, 0, st>>>(p); break;
        case T_Q5_0: mmid_kernel<T_Q5_0><<<(unsigned)nblk, 128, 0, st>>>(p); break;
        case T_Q5_1: mmid_kernel<T_Q5_1><<<(unsigned)nblk, 128, 0, st>>>(p); break;
        case T_Q2_K: mmid_kernel<T_Q2_K><<<(unsigned)nblk, 128, 0, st>>>(p); break;
        case T_Q3_K: mmid_kernel<T_Q3_K><<<(unsigned)nblk, 128, 0, st>>>(p); break;
        case T_IQ4_NL: mmid_kernel<T_IQ4_NL><<<(unsigned)nblk, 128, 0, st>>>(p); break;
        case T_IQ4_XS: mmid_kernel<T_IQ4_XS><<<(unsigned)nblk, 128, 0, st>>>(p); break;
        case T_IQ2_XXS: mmid_kernel<T_IQ2_XXS><<<(unsigned)nblk, 128, 0, st>>>(p); break;
        case T_IQ3_XXS: mmid_kernel<T_IQ3_XXS><<<(unsigned)nblk, 128, 0, st>>>(p); break;
        case T_IQ1_S: mmid_kernel<T_IQ1_S><<<(unsigned)nblk, 128, 0, st>>>(p); break;
        case T_IQ2_XS: mmid_kernel<T_IQ2_XS><<<(unsigned)nblk, 128, 0, st>>>(p); break;
        case T_IQ2_S: mmid_kernel<T_IQ2_S><<<(unsigned)nblk, 128, 0, st>>>(p); break;
        case T_IQ3_S: mmid_kernel<T_IQ3_S><<<(unsigned)nblk, 128, 0, st>>>(p); break;
        case T_IQ1_M: mmid_kernel<T_IQ1_M><<<(unsigned)nblk, 128, 0, st>>>(p); break;
        case T_TQ1_0: mmid_kernel<T_TQ1_0><<<(unsigned)nblk, 128, 0, st>>>(p); break;
        case T_TQ2_0: mmid_kernel<T_TQ2_0><<<(unsigned)nblk, 128, 0, st>>>(p); break;
        default: return GGML_B200_EUNSUPPORTED;
    }
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

} // extern "C"
