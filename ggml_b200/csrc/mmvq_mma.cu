// mmvq_mma.cu — the bandwidth-path quantized mat-mul for small batches (2 <= n <= 8; n = 1 on request) on int8 mma.sync.
//
// Same streaming skeleton as mmvq_sb.cu (persistent CTAs, one TMA producer warp, a ring of bulk-copy stages with full / empty
// mbarriers, programmatic dependent launch, weights read once from HBM in the reference's packed layout), different consume phase
// (b200_sb_mma.cuh):
//   * a chunk is a TILE of 16 weight rows, dealt to the CTAs round-robin; the eight consumer warps split the tile's K range by
//     256-weight task (task i of a slice goes to warp i mod 8), each multiplying its 16 x 256 weights with all (<= 8) activation
//     columns on the tensor cores (m16n8k32, int8 x int8 -> int32, exactly the integer block dots of ggml-cpu) and keeping 4 f32
//     partial outputs per lane;
//   * rows too long for a ring of whole-row stages are streamed in K slices of KS tasks (consecutive stages of the same tile, the
//     accumulators stay in registers across them);
//   * every row of a stage is its own bulk copy into a padded pitch (= 32 mod 128 bytes), so that the 8-byte fragment loads of the
//     four row groups of a half-warp fall into distinct bank groups;
//   * at the end of a tile the warps' partial fragments meet in shared memory (double-buffered, one named barrier per tile) and are
//     summed in a fixed order: results are bitwise repeatable.
// Activations: quantized ONCE per launch by a small pre-kernel (mma_quantize_kernel, chained with programmatic dependent launch) into
// planar per-column records (int8 codes + block sums + scales, as ggml-cpu quantizes them) in the workspace; every CTA of the main
// kernel pulls them into shared memory with one bulk copy per column while its first weight stages are in flight.  (First version:
// every CTA quantized all columns itself, on the critical path of every CTA.)
#include "b200_internal.h"
#include "b200_mm_plan.h"
#include "b200_quants.cuh"
#include "b200_ptx.cuh"
#include "b200_sb_mma.cuh"

#include <algorithm>

namespace b200 {

constexpr int MMA_MAX_STAGES = 8;
constexpr int MMA_TILE = 16;             // rows per tile (the m of m16n8k32)
constexpr int MMA_GROUP_WARPS = 8;       // consumer warps per CTA

// one act-task (256 activations of one column) per half-warp.  Always waits for the preceding kernel: it may have produced x, and the
// records live in the launch-shared workspace that the previous mat-mul's CTAs may still be reading.
template <bool KQ, bool S16, bool S81>
__global__ void __launch_bounds__(256) mma_quantize_kernel(const float * __restrict__ x, int64_t x_stride, int ncols, const mma_act A, uint8_t * __restrict__ rec) {
    pdl_launch_dependents();
    pdl_wait();
    const int i = (int)blockIdx.x * 16 + (int)(threadIdx.x >> 4);
    const bool ok = i < ncols * A.ntask;
    const int c = ok ? i / A.ntask : 0, t = ok ? i % A.ntask : 0;
    mma_quantize_task_h<KQ, S16, S81>(x + (size_t)c * x_stride, ok, rec + (size_t)c * A.col_bytes, A, t);
}

// 8 consumer warps and one producer warp with its stage ring.  Tiles are dealt round-robin (b, b + grid, ...): a dynamic hand-out (one
// global atomic per tile) gained nothing, with a few tiles per CTA the atomic's round trip sits between consecutive stages of the ring.
template <int T>
__global__ void __launch_bounds__((MMA_GROUP_WARPS + 1) * 32, 1) mmvq_mma_kernel(const mma_params p) {
    using F = mmafmt<T>;
    constexpr int GW = MMA_GROUP_WARPS;
    extern __shared__ __align__(128) uint8_t smem[];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;                  // warp GW is the producer
    uint8_t * stages = smem;                                                        // p.nstages stages
    uint8_t * rec    = smem + (size_t)p.nstages * p.stage_bytes;                    // ncols planar records
    float * partial  = (float *)(rec + (size_t)p.ncols * p.A.col_bytes);            // [2][GW][128]
    uint64_t * full  = (uint64_t *)(partial + 2 * GW * 128);
    uint64_t * empty = full + MMA_MAX_STAGES;
    uint64_t * rec_full = full + 2 * MMA_MAX_STAGES;                                // the activation records have landed
    int2 * unit_of   = (int2 *)(rec_full + 2);                                      // (tile, slice) held by each stage; tile < 0 = end

    pdl_launch_dependents();
    if (tid == 0) {
        for (int s = 0; s < p.nstages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], GW); }
        mbar_init(rec_full, 1);
        mbar_fence_init();
    }
    __syncthreads();

    if (warp == GW) {
        // ===== producer warp: lane r copies row r of the tile (slice) — sixteen bulk copies per stage, one barrier
        if (!p.src0_static) pdl_wait();
        int s = 0; uint32_t par = 0; bool wrapped = false;        // ring position: stage, parity of the round, past the first round
        int tile = (int)blockIdx.x;
        bool first = true;
        while (true) {
            const bool valid = tile < p.ntiles;
            const int nsl = valid ? p.nslices : 1;
            for (int sl = 0; sl < nsl; ++sl) {
                if (wrapped) mbar_wait(&empty[s], par ^ 1u);
                if (valid) {
                    const int64_t row0 = (int64_t)tile * MMA_TILE;
                    const int rows = (int)min((int64_t)MMA_TILE, p.M - row0);
                    const int nt = min(p.ks, p.ntask_row - sl * p.ks);
                    const uint32_t seg = (uint32_t)nt * (uint32_t)F::TASK_B;
                    if (lane == 0) { unit_of[s] = make_int2(tile, sl); mbar_expect_tx(&full[s], (uint32_t)rows * seg); }
                    __syncwarp();
                    if (lane < rows)
                        bulk_g2s(stages + (size_t)s * p.stage_bytes + (size_t)lane * p.pitch,
                                   p.w + (size_t)(row0 + lane) * p.row_bytes + (size_t)sl * p.ks * F::TASK_B, seg, &full[s]);
                } else if (lane == 0) {
                    unit_of[s] = make_int2(-1, 0);
                    mbar_arrive(&full[s]);                       // publish the end marker
                }
                if (++s == p.nstages) { s = 0; par ^= 1u; wrapped = true; }
            }
            if (first && p.l2_prefetch_bytes > 0 && lane == 0) {
                // a dependent launch cannot consume before its predecessor's output is visible, but HBM need not idle meanwhile:
                // CTA b pulls slice b of the matrix into L2, the rings then stream from L2
                const int64_t per = ((p.l2_prefetch_bytes + gridDim.x - 1) / gridDim.x + 15) & ~(int64_t)15;
                const int64_t lo = (int64_t)blockIdx.x * per;
                const int64_t hi = min(lo + per, p.l2_prefetch_bytes & ~(int64_t)15);
                for (int64_t o = lo; o < hi; o += 32768) bulk_prefetch_l2(p.w + o, (uint32_t)min((int64_t)32768, hi - o));
            }
            first = false;
            if (!valid) break;
            tile += (int)gridDim.x;
        }
        return;
    }

    // ===== consumers: the quantized activation columns (written by the pre-kernel just before this one) -> shared memory
    if (tid == 0) {
        pdl_wait();
        mbar_expect_tx(rec_full, (uint32_t)p.ncols * (uint32_t)p.A.col_bytes);
        for (int c = 0; c < p.ncols; ++c)
            bulk_g2s(rec + (size_t)c * p.A.col_bytes, p.rec_global + (size_t)c * p.A.col_bytes, (uint32_t)p.A.col_bytes, rec_full);
    }
    mbar_wait(rec_full, 0u);

    const int g = lane >> 2, t = lane & 3;
    mma_cols C;
    C.b  = rec + (size_t)min(g, p.ncols - 1) * p.A.col_bytes;                       // columns beyond n repeat the last one (results discarded)
    C.c0 = rec + (size_t)min(2 * t, p.ncols - 1) * p.A.col_bytes;
    C.c1 = rec + (size_t)min(2 * t + 1, p.ncols - 1) * p.A.col_bytes;
    float facc[4] = { 0.0f, 0.0f, 0.0f, 0.0f };
    int buf = 0;
    int s = 0; uint32_t par = 0;                                                    // ring position: stage, parity of the round
    for (;;) {
        mbar_wait(&full[s], par);
        const int2 unit = unit_of[s];
        if (unit.x < 0) break;
        const int nt = min(p.ks, p.ntask_row - unit.y * p.ks);
        const uint8_t * st = stages + (size_t)s * p.stage_bytes + (size_t)g * p.pitch;
        for (int i = warp; i < nt; i += GW)
            mma_task<T>(st + (size_t)i * F::TASK_B, st + (size_t)i * F::TASK_B + (size_t)8 * p.pitch, C, p.A, unit.y * p.ks + i, t, facc);
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[s]);
        if (++s == p.nstages) { s = 0; par ^= 1u; }
        if (unit.y == p.nslices - 1) {
            // tile finished: the eight partial fragments meet in shared memory and are summed in warp order
            float * part = partial + buf * (GW * 128);
            *(float4 *)(part + warp * 128 + lane * 4) = make_float4(facc[0], facc[1], facc[2], facc[3]);
            facc[0] = facc[1] = facc[2] = facc[3] = 0.0f;
            asm volatile("bar.sync 1, %0;" ::"n"(GW * 32) : "memory");                  // consumers only
            if (tid < 128) {
                // thread o writes (column o / 16, row o % 16): consecutive threads, consecutive rows of one column
                const int col = tid >> 4, row = tid & 15;
                const int src = ((row & 7) * 4 + (col >> 1)) * 4 + (row >> 3) * 2 + (col & 1);
                float sum = part[src];
#pragma unroll
                for (int w = 1; w < GW; ++w) sum += part[w * 128 + src];
                const int64_t grow = (int64_t)unit.x * MMA_TILE + row;
                if (col < p.ncols && grow < p.M) p.y[(size_t)col * p.M + grow] = sum;
            }
            buf ^= 1;
        }
    }
}

template <int T> static bool make_mma_plan(const ggml_b200_mul_mat_args & a, mma_plan & pl) {
    using F = mmafmt<T>;
    if (a.N < 1 || a.N > 8 || a.ne02 != 1 || a.ne03 != 1 || a.ne12 != 1 || a.ne13 != 1) return false;
    if (a.N > 1 && ((a.nb11 & 3) != 0 || a.nb11 < (size_t)a.K * 4)) return false;
    if (a.K % 256 != 0 || a.K < 2048 || a.M < MMA_TILE || a.K > 65536) return false;      // shorter rows leave most consumer warps without a task
    const size_t rb = row_bytes(a.type, a.K);
    if (a.nb01 != rb || (rb & 15) != 0 || ((uintptr_t)a.src0 & 15) != 0 || ((uintptr_t)a.src1 & 15) != 0 || (a.nb11 & 15) != 0) return false;
    mma_params & p = pl.p;
    p.w = (const uint8_t *)a.src0; p.x = a.src1; p.y = a.dst; p.M = a.M; p.K = a.K;
    p.row_bytes = (int)rb;
    p.ntiles = (int)((a.M + MMA_TILE - 1) / MMA_TILE);
    p.ntask_row = (int)(a.K / 256);
    p.A = make_mma_act(a.K, F::KQ, F::S16, F::RESIDUE, mma_s81<T>::value);
    p.ncols = (int32_t)a.N; p.x_stride = a.N > 1 ? (int64_t)(a.nb11 / 4) : 0;
    p.rec_global = nullptr;
    p.src0_static = (a.flags & GGML_B200_MM_SRC0_STATIC) ? 1 : 0;
    p.src1_static = (a.flags & GGML_B200_MM_SRC1_STATIC) ? 1 : 0;
    p.l2_prefetch_bytes = p.src0_static ? (int64_t)std::min<size_t>((size_t)a.M * rb, (size_t)L2_PREFETCH_CAP) : 0;
    // the records, the partial fragments [2][GW][128], the full / empty barriers, the records' barrier, the (tile, slice) of each stage
    const size_t budget = 226 * 1024;
    const size_t fixed = (size_t)p.ncols * p.A.col_bytes + (size_t)2 * MMA_GROUP_WARPS * 128 * 4 + (size_t)2 * MMA_MAX_STAGES * 8 + 16
                       + (size_t)MMA_MAX_STAGES * 8 + 128;
    if (fixed + (size_t)2 * 8 * F::TASK_B * MMA_TILE > budget) return false;
    // slices of KS tasks (a multiple of the warp count): whole rows when at least three such stages fit next to the records
    auto geometry = [&](int ks) {
        p.ks = ks;
        p.nslices = (p.ntask_row + ks - 1) / ks;
        int pitch = std::min(ks, p.ntask_row) * F::TASK_B;
        pitch = (pitch + 15) & ~15;
        while ((pitch & 127) != F::RESIDUE) pitch += 16;
        p.pitch = pitch;
        p.stage_bytes = (pitch * MMA_TILE + 127) & ~127;
        return (int)std::min<size_t>((budget - fixed) / p.stage_bytes, MMA_MAX_STAGES);
    };
    int ks = std::min(16, p.ntask_row);                  // 16 tasks x 16 rows: 36 KB (Q4_K) .. 70 KB (Q8_0) per stage
    int nst = geometry(ks);
    while (nst < 3 && ks > 8) { ks = std::max(8, ks / 2); nst = geometry(ks); }
    if (nst < 2) return false;
    p.nstages = nst;
    pl.smem = (int)(fixed + (size_t)p.nstages * p.stage_bytes);
    pl.grid = std::min(sm_count(), p.ntiles);
    pl.workspace = (size_t)p.ncols * p.A.col_bytes + 256;       // the activation records, 256-byte aligned
    return true;
}

template <int T> static int launch_mma_t(const ggml_b200_mul_mat_args & a, mma_plan pl, cudaStream_t st) {
    using F = mmafmt<T>;
    if (!a.workspace || a.workspace_size < pl.workspace) { set_error("mul_mat: workspace %zu < %zu", a.workspace_size, pl.workspace); return GGML_B200_EWORKSPACE; }
    uint8_t * rec = (uint8_t *)(((uintptr_t)a.workspace + 255) & ~(uintptr_t)255);
    pl.p.rec_global = rec;
    B200_CUDA_TRY(launch_pdl(mma_quantize_kernel<F::KQ, F::S16, mma_s81<T>::value>, dim3((unsigned)((pl.p.ncols * pl.p.A.ntask + 15) / 16)), dim3(256), 0, st,
                             a.src1, pl.p.x_stride, (int)pl.p.ncols, pl.p.A, rec));
    B200_LAUNCH_CHECK();
    B200_CUDA_TRY(set_max_dynamic_smem<mmvq_mma_kernel<T>>(227 * 1024));
    B200_CUDA_TRY(launch_pdl(mmvq_mma_kernel<T>, dim3(pl.grid), dim3((MMA_GROUP_WARPS + 1) * 32), pl.smem, st, pl.p));
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

bool plan_mma(const ggml_b200_mul_mat_args & a, mma_plan & pl) {
    bool ok = false;
    with_format(TC_FORMATS(), a.type, [&](auto t) { ok = make_mma_plan<t>(a, pl); });
    return ok;
}

int launch_mma(const ggml_b200_mul_mat_args & a, const mma_plan & pl, cudaStream_t st) {
    int rc = GGML_B200_EUNSUPPORTED;                                 // plan_mma accepts TC_FORMATS only
    with_format(TC_FORMATS(), a.type, [&](auto t) { rc = launch_mma_t<t>(a, pl, st); });
    return rc;
}

} // namespace b200
