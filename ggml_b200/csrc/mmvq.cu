// mmvq.cu — quantized mat-vec kernels (n <= 8 activation columns) for sm_90a.
//
// Replaces the reference's mul_mat_vec_q (src/ggml-cuda/mmvq.cu:50-130) + quantize_q8_1
// (src/ggml-cuda/quantize.cu:4-38) and computes what ggml_compute_forward_mul_mat
// (src/ggml-cpu/ggml-cpu.c:7428-7605) computes: int8-quantized activations, integer block dots,
// f32 scaling.  Weights are read in the packed block_q* layout, once.
//
//   mmvq_tma_kernel     bandwidth path.  Persistent CTAs; each owns a contiguous range of weight rows and
//                       streams it through a ring of shared-memory stages filled by TMA bulk copies
//                       (cp.async.bulk + mbarrier complete_tx), so the copy is coalesced and 16-byte
//                       granular whatever the block size (18/34/210-byte blocks are only 2-byte aligned).
//                       The CTA quantizes the activation vector(s) itself while the first stages are in
//                       flight (no separate launch); warps decode 64-weight units from shared memory in
//                       registers, dp4a against the int8 activations, reduce with warp shuffles.
//   mmvq_generic_kernel any K / strides / batch / broadcast: one warp per output element straight from
//                       global memory, activations pre-quantized by quantize_act_kernel.
#include "b200_internal.h"
#include "b200_quants.cuh"
#include "b200_iq.cuh"

#include <cstdlib>

namespace b200 {

// =============================================================================== PTX helpers
__device__ __forceinline__ uint32_t smem_u32(const void * p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t * bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t * bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t * bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "B200_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra B200_DONE;\n"
        "bra B200_WAIT;\n"
        "B200_DONE:\n"
        "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
// TMA bulk copy global -> shared, completion signalled on an mbarrier (SASS: UBLKCP)
__device__ __forceinline__ void tma_bulk_g2s(void * dst_smem, const void * src_gmem, uint32_t bytes, uint64_t * bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// =============================================================================== activation quantizer
template <bool KQ>
__global__ void __launch_bounds__(256) quantize_act_kernel(const float * __restrict__ x, int64_t K, int64_t n11, int64_t n12,
                                                           size_t nb11, size_t nb12, size_t nb13, uint8_t * __restrict__ recs, act_layout L) {
    const int64_t r = blockIdx.x;
    const int64_t i11 = r % n11, i12 = (r / n11) % n12, i13 = r / (n11 * n12);
    const float * xr = (const float *)((const uint8_t *)x + i11 * nb11 + i12 * nb12 + i13 * nb13);
    cta_quantize_row<KQ>(xr, K, recs + (size_t)r * L.bytes, L);
}

int launch_quantize_activations(int type, const float * x, int64_t K, int64_t n11, int64_t n12, int64_t n13,
                                size_t nb11, size_t nb12, size_t nb13, void * recs, cudaStream_t st) {
    const bool kq = type_is_kquant(type);
    const act_layout L = make_act_layout(K, kq);
    const int64_t rows = n11 * n12 * n13;
    if (rows <= 0) return GGML_B200_OK;
    const int warps = (int)((K + 255) / 256 < 8 ? (K + 255) / 256 : 8);
    if (kq) quantize_act_kernel<true><<<(unsigned)rows, 32 * warps, 0, st>>>(x, K, n11, n12, nb11, nb12, nb13, (uint8_t *)recs, L);
    else    quantize_act_kernel<false><<<(unsigned)rows, 32 * warps, 0, st>>>(x, K, n11, n12, nb11, nb12, nb13, (uint8_t *)recs, L);
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

// =============================================================================== generic kernel
struct generic_params {
    const uint8_t * w; const uint8_t * recs; float * y;
    int64_t K, M, N, ne02, ne03, ne12, ne13;
    size_t  nb01, nb02, nb03;
    act_layout L;
    int64_t nrg;      // row groups = ceil(M / warps per CTA)
};

template <int T>
__global__ void __launch_bounds__(128) mmvq_generic_kernel(generic_params p) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t rg = blockIdx.x % p.nrg, col = blockIdx.x / p.nrg;
    const int64_t m = rg * 4 + warp;
    if (m >= p.M) return;
    const int64_t i12 = (col / p.N) % p.ne12, i13 = col / (p.N * p.ne12);
    const int64_t i02 = i12 / (p.ne12 / p.ne02), i03 = i13 / (p.ne13 / p.ne03);
    const uint8_t * row = p.w + m * p.nb01 + i02 * p.nb02 + i03 * p.nb03;
    const uint8_t * rec = p.recs + (size_t)col * p.L.bytes;
    const int nunits = (int)(p.K / 64);
    float acc = 0.0f;
    for (int u = lane; u < nunits; u += 32) {
        unit_act A;
        load_unit_act<T>(rec, p.L, u, A);
        acc += unit_dot<T>(row, u, A);
    }
    if constexpr (fmt<T>::QK == 32) {
        if ((p.K & 63) != 0 && lane == 0) acc += tail_block_dot<T>(row + (size_t)nunits * 2 * fmt<T>::BYTES, rec, p.L, nunits * 2);
    }
    acc = warp_sum(acc);
    if (lane == 0) p.y[(size_t)col * p.M + m] = acc;
}

size_t mmvq_generic_workspace(const ggml_b200_mul_mat_args & a) {
    const act_layout L = make_act_layout(a.K, type_is_kquant(a.type));
    return (size_t)L.bytes * (size_t)(a.N * a.ne12 * a.ne13) + 64;
}

int launch_mmvq_generic(const ggml_b200_mul_mat_args & a, cudaStream_t st) {
    const size_t need = mmvq_generic_workspace(a);
    if (a.workspace == nullptr || a.workspace_size < need) { set_error("mul_mat: workspace %zu < %zu", a.workspace_size, need); return GGML_B200_EWORKSPACE; }
    int rc = launch_quantize_activations(a.type, a.src1, a.K, a.N, a.ne12, a.ne13, a.nb11, a.nb12, a.nb13, a.workspace, st);
    if (rc != GGML_B200_OK) return rc;
    generic_params p;
    p.w = (const uint8_t *)a.src0; p.recs = (const uint8_t *)a.workspace; p.y = a.dst;
    p.K = a.K; p.M = a.M; p.N = a.N; p.ne02 = a.ne02; p.ne03 = a.ne03; p.ne12 = a.ne12; p.ne13 = a.ne13;
    p.nb01 = a.nb01; p.nb02 = a.nb02; p.nb03 = a.nb03;
    p.L = make_act_layout(a.K, type_is_kquant(a.type));
    p.nrg = (a.M + 3) / 4;
    const int64_t cols = a.N * a.ne12 * a.ne13;
    const int64_t nblk = p.nrg * cols;
    if (nblk <= 0) return GGML_B200_OK;
    if (nblk > 0x7fffffffLL) { set_error("mul_mat: grid too large"); return GGML_B200_EUNSUPPORTED; }
    switch (a.type) {
        case T_Q4_0: mmvq_generic_kernel<T_Q4_0><<<(unsigned)nblk, 128, 0, st>>>(p); break;
        case T_Q8_0: mmvq_generic_kernel<T_Q8_0><<<(unsigned)nblk, 128, 0, st>>>(p); break;
        case T_Q4_K: mmvq_generic_kernel<T_Q4_K><<<(unsigned)nblk, 128, 0, st>>>(p); break;
        case T_Q5_K: mmvq_generic_kernel<T_Q5_K><<<(unsigned)nblk, 128, 0, st>>>(p); break;
        case T_Q6_K: mmvq_generic_kernel<T_Q6_K><<<(unsigned)nblk, 128, 0, st>>>(p); break;
        case T_Q4_1: mmvq_generic_kernel<T_Q4_1><<<(unsigned)nblk, 128, 0, st>>>(p); break;
        case T_Q5_0: mmvq_generic_kernel<T_Q5_0><<<(unsigned)nblk, 128, 0, st>>>(p); break;
        case T_Q5_1: mmvq_generic_kernel<T_Q5_1><<<(unsigned)nblk, 128, 0, st>>>(p); break;
        case T_Q2_K: mmvq_generic_kernel<T_Q2_K><<<(unsigned)nblk, 128, 0, st>>>(p); break;
        case T_Q3_K: mmvq_generic_kernel<T_Q3_K><<<(unsigned)nblk, 128, 0, st>>>(p); break;
        case T_IQ4_NL: mmvq_generic_kernel<T_IQ4_NL><<<(unsigned)nblk, 128, 0, st>>>(p); break;
        case T_IQ4_XS: mmvq_generic_kernel<T_IQ4_XS><<<(unsigned)nblk, 128, 0, st>>>(p); break;
        case T_IQ2_XXS: mmvq_generic_kernel<T_IQ2_XXS><<<(unsigned)nblk, 128, 0, st>>>(p); break;
        case T_IQ3_XXS: mmvq_generic_kernel<T_IQ3_XXS><<<(unsigned)nblk, 128, 0, st>>>(p); break;
        case T_IQ1_S: mmvq_generic_kernel<T_IQ1_S><<<(unsigned)nblk, 128, 0, st>>>(p); break;
        case T_IQ2_XS: mmvq_generic_kernel<T_IQ2_XS><<<(unsigned)nblk, 128, 0, st>>>(p); break;
        case T_IQ2_S: mmvq_generic_kernel<T_IQ2_S><<<(unsigned)nblk, 128, 0, st>>>(p); break;
        case T_IQ3_S: mmvq_generic_kernel<T_IQ3_S><<<(unsigned)nblk, 128, 0, st>>>(p); break;
        case T_IQ1_M: mmvq_generic_kernel<T_IQ1_M><<<(unsigned)nblk, 128, 0, st>>>(p); break;
        case T_TQ1_0: mmvq_generic_kernel<T_TQ1_0><<<(unsigned)nblk, 128, 0, st>>>(p); break;
        case T_TQ2_0: mmvq_generic_kernel<T_TQ2_0><<<(unsigned)nblk, 128, 0, st>>>(p); break;
        default: set_error("mul_mat: unsupported weight type %d", a.type); return GGML_B200_EUNSUPPORTED;
    }
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

// =============================================================================== TMA-staged bandwidth kernel
constexpr int TMA_MAX_STAGES = 8;

struct tma_params {
    const uint8_t * w;        // row 0, 16-byte aligned, rows contiguous (nb01 == row_bytes)
    const float *   x;        // activation columns
    float *         y;        // [N][M]
    size_t          nb11;     // activation column stride (bytes)
    int64_t         M, K;
    int32_t         N;        // valid columns (<= NC)
    int32_t         row_bytes;
    int32_t         RB;       // rows per stage
    int32_t         P, G;     // warps = G row-groups x P k-parts
    int32_t         nchunks;  // ceil(M / RB)
    int32_t         stage_bytes;   // RB * row_bytes rounded up to 128
    int32_t         nstages;
    act_layout      L;
};

// transposing shuffle reduction of 4 per-lane values: returns, in every lane, the full sum of value
// number ((lane >> 3) & 3); 6 shuffles instead of 20
__device__ __forceinline__ float warp_sum4(float v0, float v1, float v2, float v3, int lane) {
    const bool hi16 = lane & 16;
    float a = hi16 ? v2 : v0, sa = hi16 ? v0 : v2;
    float b = hi16 ? v3 : v1, sb = hi16 ? v1 : v3;
    a += __shfl_xor_sync(0xffffffffu, sa, 16);
    b += __shfl_xor_sync(0xffffffffu, sb, 16);
    const bool hi8 = lane & 8;
    float c = hi8 ? b : a, sc = hi8 ? a : b;
    c += __shfl_xor_sync(0xffffffffu, sc, 8);
    c += __shfl_xor_sync(0xffffffffu, c, 4);
    c += __shfl_xor_sync(0xffffffffu, c, 2);
    c += __shfl_xor_sync(0xffffffffu, c, 1);
    return c;
}

template <int T, int NC, int R>
__global__ void __launch_bounds__(256) mmvq_tma_kernel(const tma_params p) {
    extern __shared__ __align__(128) uint8_t smem[];
    // layout: [stages] [act records NC] [red 2 x RB x NC x P floats] [mbarriers]
    uint8_t * stages = smem;
    uint8_t * recs   = stages + (size_t)p.nstages * p.stage_bytes;
    float *   red    = (float *)(recs + (size_t)NC * p.L.bytes);
    uint64_t * full  = (uint64_t *)(red + 2 * p.RB * NC * p.P);   // TMA_MAX_STAGES barriers

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = warp / p.P, kp = warp % p.P;

    // contiguous, balanced chunk range of this CTA
    const int per = p.nchunks / gridDim.x, rem = p.nchunks % gridDim.x;
    const int first = blockIdx.x * per + min((int)blockIdx.x, rem);
    const int mine  = per + ((int)blockIdx.x < rem ? 1 : 0);

    auto issue = [&](int it) {
        const int s = it % p.nstages;
        const int64_t row0 = (int64_t)(first + it) * p.RB;
        const int rows = (int)min((int64_t)p.RB, p.M - row0);
        const uint32_t bytes = (uint32_t)rows * (uint32_t)p.row_bytes;      // multiple of 16 by construction
        mbar_arrive_expect_tx(&full[s], bytes);
        tma_bulk_g2s(stages + (size_t)s * p.stage_bytes, p.w + (size_t)row0 * p.row_bytes, bytes, &full[s]);
    };

    if (tid == 0) {
        for (int s = 0; s < p.nstages; ++s) mbar_init(&full[s], 1);
        fence_mbar_init();
        for (int it = 0; it < p.nstages && it < mine; ++it) issue(it);
    }
    // quantize the activation column(s) while the first stages are in flight
#pragma unroll
    for (int c = 0; c < NC; ++c)
        if (c < p.N) cta_quantize_row<fmt<T>::ACT_K != 0>((const float *)((const uint8_t *)p.x + c * p.nb11), p.K, recs + (size_t)c * p.L.bytes, p.L);
    __syncthreads();

    const int nunits = (int)(p.K / 64);
    for (int it = 0; it < mine; ++it) {
        const int s = it % p.nstages;
        const int64_t row0 = (int64_t)(first + it) * p.RB;
        const int rows = (int)min((int64_t)p.RB, p.M - row0);
        const uint8_t * st = stages + (size_t)s * p.stage_bytes;
        float * redb = red + (size_t)(it & 1) * p.RB * NC * p.P;
        mbar_wait(&full[s], (uint32_t)(it / p.nstages) & 1u);

        for (int r0 = g * R; r0 < rows; r0 += p.G * R) {
            float acc[R][NC];
#pragma unroll
            for (int i = 0; i < R; ++i)
#pragma unroll
                for (int c = 0; c < NC; ++c) acc[i][c] = 0.0f;
            for (int u = kp * 32 + lane; u < nunits; u += p.P * 32) {
#pragma unroll
                for (int c = 0; c < NC; ++c) {
                    if (c < p.N) {
                        unit_act A;
                        load_unit_act<T>(recs + (size_t)c * p.L.bytes, p.L, u, A);
#pragma unroll
                        for (int i = 0; i < R; ++i)
                            if (r0 + i < rows) acc[i][c] += unit_dot<T>(st + (size_t)(r0 + i) * p.row_bytes, u, A);
                    }
                }
            }
            if constexpr (R == 4 && NC == 1) {
                const float v = warp_sum4(acc[0][0], acc[1][0], acc[2][0], acc[3][0], lane);
                const int i = (lane >> 3) & 3;
                if ((lane & 7) == 0 && r0 + i < rows) redb[(r0 + i) * p.P + kp] = v;
            } else {
#pragma unroll
                for (int i = 0; i < R; ++i)
#pragma unroll
                    for (int c = 0; c < NC; ++c) {
                        const float v = warp_sum(acc[i][c]);
                        if (lane == 0 && r0 + i < rows && c < p.N) redb[((r0 + i) * NC + c) * p.P + kp] = v;
                    }
            }
        }
        __syncthreads();     // stage s fully consumed, partial sums visible
        if (tid == 0 && it + p.nstages < mine) issue(it + p.nstages);
        for (int o = tid; o < rows * NC; o += blockDim.x) {
            const int r = o / NC, c = o % NC;
            if (c < p.N) {
                float v = 0.0f;
                for (int q = 0; q < p.P; ++q) v += redb[o * p.P + q];
                p.y[(size_t)c * p.M + row0 + r] = v;
            }
        }
    }
}

struct tma_plan {
    tma_params p;
    int grid, block, smem, nc, r;
};

static bool make_tma_plan(const ggml_b200_mul_mat_args & a, tma_plan & pl) {
    if (a.type != T_Q4_0 && a.type != T_Q8_0 && a.type != T_Q4_K && a.type != T_Q5_K && a.type != T_Q6_K) return false;   // the other formats: generic kernel
    if (a.N < 1 || a.N > 8 || a.ne02 != 1 || a.ne03 != 1 || a.ne12 != 1 || a.ne13 != 1) return false;
    if (a.K % 64 != 0 || a.K < 64 || a.M < 1) return false;                 // whole units; Q4_0/Q8_0 pairs 4-byte aligned
    const size_t rb = row_bytes(a.type, a.K);
    if (rb == 0 || a.nb01 != rb) return false;                              // rows must be contiguous for bulk copies
    if (((uintptr_t)a.src0 & 15) != 0 || ((uintptr_t)a.src1 & 3) != 0) return false;
    if ((a.M * rb) % 16 != 0) return false;                                 // last chunk must end on a 16-byte boundary
    if (rb > 48 * 1024) return false;
    const bool kq = type_is_kquant(a.type);
    const act_layout L = make_act_layout(a.K, kq);

    const int nc = a.N == 1 ? 1 : a.N == 2 ? 2 : a.N <= 4 ? 4 : 8;
    const int nunits = (int)(a.K / 64);
    int P = (nunits + 31) / 32; if (P > 8) P = 8;
    // tunables (env, for sweeps): stage size target, ring depth, CTAs per SM
    static const int env_stage_kb = getenv("GGML_B200_GEMV_STAGE_KB") ? atoi(getenv("GGML_B200_GEMV_STAGE_KB")) : 18;
    static const int env_stages   = getenv("GGML_B200_GEMV_STAGES")   ? atoi(getenv("GGML_B200_GEMV_STAGES"))   : 3;
    static const int env_per_sm   = getenv("GGML_B200_GEMV_CTAS")     ? atoi(getenv("GGML_B200_GEMV_CTAS"))     : 0;
    static const int env_warps    = getenv("GGML_B200_GEMV_WARPS")    ? atoi(getenv("GGML_B200_GEMV_WARPS"))    : 4;
    const size_t target = (size_t)env_stage_kb * 1024;
    int granule = 1; while ((granule * rb) % 16 != 0) granule *= 2;
    // rows per tile pass: G row-groups x R rows (register blocking); pick the largest G*R that fits the stage target
    const int rpref = nc == 1 ? 4 : nc == 2 ? 2 : 1;
    int gmax = env_warps / P; if (gmax < 1) gmax = 1;
    int G = 1, r = 1;
    for (int rr = rpref; rr >= 1; rr >>= 1)
        for (int gg = gmax; gg >= 1; --gg)
            if ((size_t)gg * rr * rb <= target + target / 4 && gg * rr > G * r) { G = gg; r = rr; }
    int step = G * r; while (step % granule != 0) step += G * r;
    int RB = (int)(target / rb) / step * step; if (RB < step) RB = step;
    if ((size_t)RB * rb > 56 * 1024) return false;
    int nstages = env_stages < 2 ? 2 : env_stages > TMA_MAX_STAGES ? TMA_MAX_STAGES : env_stages;

    tma_params & p = pl.p;
    p.w = (const uint8_t *)a.src0; p.x = a.src1; p.y = a.dst; p.nb11 = a.nb11; p.M = a.M; p.K = a.K; p.N = (int)a.N;
    p.row_bytes = (int)rb; p.RB = RB; p.P = P; p.G = G;
    p.nchunks = (int)((a.M + RB - 1) / RB);
    p.stage_bytes = (int)(((size_t)RB * rb + 127) & ~(size_t)127);
    p.L = L; p.nstages = nstages;
    pl.nc = nc; pl.r = r;
    pl.block = 32 * P * G;
    pl.smem = p.nstages * p.stage_bytes + nc * L.bytes + 2 * RB * nc * P * 4 + TMA_MAX_STAGES * 8 + 16;
    while (pl.smem > 200 * 1024 && p.nstages > 2) { p.nstages--; pl.smem -= p.stage_bytes; }
    if (pl.smem > 200 * 1024) return false;
    int per_sm = (224 * 1024) / (pl.smem + 1024); if (per_sm < 1) per_sm = 1; if (per_sm > 8) per_sm = 8;
    if (env_per_sm > 0 && env_per_sm < per_sm) per_sm = env_per_sm;
    if (per_sm * pl.block > 2048) per_sm = 2048 / pl.block;
    int grid = sm_count() * per_sm;
    if (grid > p.nchunks) grid = p.nchunks;
    pl.grid = grid;
    return true;
}

bool mmvq_tma_eligible(const ggml_b200_mul_mat_args & a) {
    tma_plan pl;
    return make_tma_plan(a, pl);
}

template <int T, int NC, int R> static int launch_tma_inst(const tma_plan & pl, cudaStream_t st) {
    static per_device_flag attr_set;   // per instantiation and device
    if (!attr_set.test()) {
        B200_CUDA_TRY(cudaFuncSetAttribute(mmvq_tma_kernel<T, NC, R>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        attr_set.set();
    }
    mmvq_tma_kernel<T, NC, R><<<pl.grid, pl.block, pl.smem, st>>>(pl.p);
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

template <int T> static int launch_tma_type(const tma_plan & pl, cudaStream_t st) {
    switch (pl.nc) {
        case 1: return pl.r == 4 ? launch_tma_inst<T, 1, 4>(pl, st) : pl.r == 2 ? launch_tma_inst<T, 1, 2>(pl, st) : launch_tma_inst<T, 1, 1>(pl, st);
        case 2: return pl.r == 2 ? launch_tma_inst<T, 2, 2>(pl, st) : launch_tma_inst<T, 2, 1>(pl, st);
        case 4: return launch_tma_inst<T, 4, 1>(pl, st);
        default: return launch_tma_inst<T, 8, 1>(pl, st);
    }
}

int launch_mmvq_tma(const ggml_b200_mul_mat_args & a, cudaStream_t st) {
    tma_plan pl;
    if (!make_tma_plan(a, pl)) { set_error("mul_mat: shape not eligible for the TMA mat-vec kernel"); return GGML_B200_EUNSUPPORTED; }
    switch (a.type) {
        case T_Q4_0: return launch_tma_type<T_Q4_0>(pl, st);
        case T_Q8_0: return launch_tma_type<T_Q8_0>(pl, st);
        case T_Q4_K: return launch_tma_type<T_Q4_K>(pl, st);
        case T_Q5_K: return launch_tma_type<T_Q5_K>(pl, st);
        case T_Q6_K: return launch_tma_type<T_Q6_K>(pl, st);
        default: set_error("mul_mat: unsupported weight type %d", a.type); return GGML_B200_EUNSUPPORTED;
    }
}

} // namespace b200
