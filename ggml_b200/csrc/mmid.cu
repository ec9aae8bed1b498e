// mmid.cu — GGML_OP_MUL_MAT_ID (mixture-of-experts mat-mul) for sm_90a.
//
// Computes what ggml_compute_forward_mul_mat_id (reference src/ggml-cpu/ggml-cpu.c:7609-7784) computes and
// replaces ggml_cuda_mul_mat_id (src/ggml-cuda/ggml-cuda.cu:1955-2090), which copies `ids` to the host and
// synchronises the stream to build per-expert row lists.  Here routing stays on the device: every output
// vector dst[t][e][:] = as[ids[t][e]] . b[t][e % nb1cols] is an independent quantized mat-vec whose expert
// index is read by the kernel itself, so the op is one quantize launch + one mat-vec launch, no host sync.
#include "b200_internal.h"
#include "b200_mm_plan.h"
#include "b200_quants.cuh"
#include "b200_iq.cuh"
#include "b200_ptx.cuh"

namespace b200 {

struct mmid_params {
    const uint8_t * w; const uint8_t * recs; const uint8_t * ids; float * y;
    int64_t K, M, n_expert, n_used, nb1cols, n_tok;
    size_t  nb01, nb02, ids_nb1;
    act_layout L;
    int64_t nrg;
};

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
    acc = warp_sum(acc);
    if (lane == 0) p.y[(size_t)pair * p.M + m] = acc;
}

// The form a MUL_MAT_ID call runs and the workspace it requires: expert-grouped on the GEMM kernel (batched tokens), else one
// quantized mat-vec per (token, slot) pair over activation records b[K, nb1cols, n_tok] -> record t * nb1cols + c.
struct mmid_plan { bool grouped; mmid_g_plan g; size_t workspace; };

static mmid_plan plan_mmid(const ggml_b200_mul_mat_id_args & a) {
    mmid_plan pl;
    pl.grouped = plan_mmid_grouped(a, pl.g);
    pl.workspace = pl.grouped ? pl.g.workspace : (size_t)make_act_layout(a.K, type_is_kquant(a.type)).bytes * (size_t)(a.nb1cols * a.n_tok) + 64;
    return pl;
}

} // namespace b200

using namespace b200;

extern "C" {

size_t ggml_b200_mul_mat_id_workspace_size(const ggml_b200_mul_mat_id_args * a) {
    if (!a || type_bytes(a->type) == 0 || a->K <= 0) return 0;
    return plan_mmid(*a).workspace;
}

int ggml_b200_mul_mat_id(const ggml_b200_mul_mat_id_args * a, void * stream) {
    if (!a) { set_error("mul_mat_id: NULL args"); return GGML_B200_EINVAL; }
    if (type_bytes(a->type) == 0) { set_error("mul_mat_id: unsupported weight type %d", a->type); return GGML_B200_EUNSUPPORTED; }
    if (a->K <= 0 || a->K % type_qk(a->type) != 0 || a->M < 0 || a->n_expert < 1 || a->n_used < 1 || a->nb1cols < 1 || a->n_tok < 0) { set_error("mul_mat_id: bad shape"); return GGML_B200_EINVAL; }
    if (a->M == 0 || a->n_tok == 0) return GGML_B200_OK;
    if (!a->src0 || !a->src1 || !a->ids || !a->dst) { set_error("mul_mat_id: NULL tensor pointer"); return GGML_B200_EINVAL; }
    if ((a->nb11 & 3) || (a->nb12 & 3) || (a->ids_nb1 & 3) || (a->nb01 & 1) || (a->nb02 & 1)) { set_error("mul_mat_id: bad strides"); return GGML_B200_EINVAL; }
    if ((a->type == T_Q4_K || a->type == T_Q5_K) && (((uintptr_t)a->src0 | a->nb01 | a->nb02) & 15)) { set_error("mul_mat_id: Q4_K/Q5_K rows must be 16-byte aligned"); return GGML_B200_EINVAL; }
    const mmid_plan pl = plan_mmid(*a);
    if (!a->workspace || a->workspace_size < pl.workspace) { set_error("mul_mat_id: workspace %zu < %zu", a->workspace_size, pl.workspace); return GGML_B200_EWORKSPACE; }
    cudaStream_t st = (cudaStream_t)stream;
    if (pl.grouped) return launch_mmid_grouped(*a, pl.g, st);
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
    if (!with_format(ALL_FORMATS(), a->type, [&](auto t) { mmid_kernel<t><<<(unsigned)nblk, 128, 0, st>>>(p); })) return GGML_B200_EUNSUPPORTED;
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

} // extern "C"
