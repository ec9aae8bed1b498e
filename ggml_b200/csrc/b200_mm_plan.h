// b200_mm_plan.h — launch plans of the mat-mul kernel families (host side, not part of the ABI).
//
// A family's planner (plan_X, b200_internal.h) decides whether the family can run a shape and computes everything its launcher needs,
// the workspace bytes included; the launcher (launch_X) runs the plan as it is.  Planning is pure: scheduling slots, split-K flags and
// the control block are taken at launch, so a plan made when the route is chosen is the plan that launches.
#pragma once

#include "b200_internal.h"
#include "b200_quants.cuh"
#include "b200_sb_tasks.cuh"
#include "b200_sb_mma.cuh"

namespace b200 {

// ----------------------------------------------------------------------------- first-generation TMA mat-vec (mmvq.cu)
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

struct tma_plan {
    tma_params p;
    int grid, block, smem, nc, r;
};

// ----------------------------------------------------------------------------- superblock mat-vec (mmvq_sb.cu)
struct sb_params {
    const uint8_t * w; const float * x; float * y;
    int64_t M, K;
    int32_t row_bytes, rows_per_chunk, nchunks, stage_bytes, nstages, ntasks_row;
    unsigned int * counters;      // this launch's scheduling slot: [0] next chunk, [1] finished producers, [2] finished CTAs (all return to 0)
    unsigned int * ctl;           // device-global control words: [0] exchange epoch
    int32_t ncols; int64_t x_stride;   // activation columns (1..8) and the distance between them in floats; y is [ncols][M]
    int32_t src1_static;          // activations are not produced by the preceding kernel either: never wait for it (independent ops overlap)
    int32_t src0_static;          // weights are not produced by the preceding kernel: prefetch them before griddepcontrol.wait
    int32_t static_chunks;        // chunks dealt round-robin instead of by the atomic counter
    int64_t l2_prefetch_bytes;    // dependent launches: bytes of W every CTA's share of which is pulled into L2 while the previous kernel still runs (0 = off)
    // row-sharded multi-GPU: every result is stored straight into each peer's full-length y over NVLink (world == 0: off)
    // fused epilogue (bias add and GELU of the following ggml nodes): y2 = y + bias, y3 = gelu(y2); null = off
    const float * ep_bias; float * ep_y2; float * ep_y3; const float * ep_res;    // ep_res: y3 = y2 + residual instead of gelu(y2)
    int32_t world, rank;
    int64_t row_offset;
    uint32_t epoch;
    float *    y_peers[8];
    uint32_t * flag_peers[8];
    sb_act A;
};

// w, x and y are bound at launch: the plan of one column group serves every group of its width
struct sb_plan { sb_params p; int grid, smem, nw, nc; bool two, act_regs; };

// ----------------------------------------------------------------------------- int8 mma.sync mat-vec (mmvq_mma.cu)
struct mma_params {
    const uint8_t * w; const float * x; float * y;
    int64_t M, K;
    int32_t row_bytes, ntiles, nslices, ks, ntask_row, pitch, stage_bytes, nstages;
    int32_t ncols; int64_t x_stride;
    int32_t src1_static, src0_static;
    int64_t l2_prefetch_bytes;
    const uint8_t * rec_global;   // ncols planar records written by mma_quantize_kernel (workspace)
    mma_act A;
};

struct mma_plan { mma_params p; int grid, smem; size_t workspace; };

// ----------------------------------------------------------------------------- wgmma GEMM (mmq_tc2.cu)
struct tc2_plan {
    int BN, m_tiles, n_tiles, splitk, chunks, nstages, smem, grid;
    size_t xb_bytes, partial_bytes, scale_bytes, workspace;
};

// formats without an operand decoder: W dequantized to fp16 in the workspace, then the GEMM on `b`, the same shape with fp16 weights
struct dense_plan { ggml_b200_mul_mat_args b; size_t wbytes; tc2_plan tc; size_t workspace; };

// expert-grouped MUL_MAT_ID on the GEMM kernel
struct mmid_g_plan { int BN, m_tiles, max_tiles, chunks, nstages, smem; size_t xb_bytes, scale_bytes, tab_bytes, perm_bytes, workspace; int64_t n_pairs; };

// ----------------------------------------------------------------------------- the kernel one mul_mat call runs (api.cu::route)
enum route_kind {
    R_GENERIC,     // one warp per output (mmvq.cu): any shape
    R_TMA,         // first-generation 64-weight-unit mat-vec (mmvq.cu)
    R_TMA_UNFIT,   // GEMV_V1 without FORCE_GEMV where only the superblock kernel takes the shape: a mat-vec route whose launch fails
    R_SB,          // superblock mat-vec (mmvq_sb.cu), all columns in one launch
    R_SB_GROUPS,   // superblock mat-vec in column groups of `group`
    R_MMA,         // int8 mma.sync mat-vec (mmvq_mma.cu)
    R_WGMMA,       // warpgroup-MMA GEMM (mmq_tc2.cu)
    R_DENSE,       // W dequantized to fp16, then the same GEMM (mmq_tc2.cu)
};

// Only the member of the chosen family is meaningful.  R_SB_GROUPS: `sb` is the plan of a group of `group` columns, `sb_tail` that of
// the narrower last group when `group` does not divide n.
struct mm_plan {
    route_kind kind;
    int64_t group;
    size_t workspace;             // bytes the launch requires
    tma_plan tma;
    sb_plan sb, sb_tail;
    mma_plan mma;
    tc2_plan wgmma;
    dense_plan dense;
};

} // namespace b200
