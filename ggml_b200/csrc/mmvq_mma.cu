// mmvq_mma.cu — the bandwidth-path quantized mat-mul for small batches (2 <= n <= 8; n = 1 on request) on int8 mma.sync.
//
// Same streaming skeleton as mmvq_sb.cu (persistent CTAs, one TMA producer warp, a ring of bulk-copy stages with full / empty
// mbarriers, chunks handed out by a self-resetting atomic slot, programmatic dependent launch, weights read once from HBM in the
// reference's packed layout), different consume phase (b200_sb_mma.cuh):
//   * a chunk is a TILE of 16 weight rows; the eight consumer warps of a group split the tile's K range by 256-weight task (task i of a
//     slice goes to warp i mod 8), each multiplying its 16 x 256 weights with all (<= 8) activation columns on the tensor cores
//     (m16n8k32, int8 x int8 -> int32, exactly the integer block dots of ggml-cpu) and keeping 4 f32 partial outputs per lane;
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
#include "b200_quants.cuh"
#include "b200_sb_ptx.cuh"
#include "b200_sb_mma.cuh"

#include <algorithm>
#include <cstdlib>

namespace b200 {

constexpr int MMA_MAX_STAGES = 8;
constexpr int MMA_TILE = 16;             // rows per tile (the m of m16n8k32)
constexpr int MMA_GROUP_WARPS = 8;       // consumer warps per group

struct mma_params {
    const uint8_t * w; const float * x; float * y;
    int64_t M, K;
    int32_t row_bytes, ntiles, nslices, ks, ntask_row, pitch, stage_bytes, nstages;
    unsigned int * counters;      // null: tiles dealt round-robin; else this launch's scheduling slot: [0] next tile, [1] finished producers
    int32_t ncols; int64_t x_stride;
    int32_t src1_static, src0_static;
    int64_t l2_prefetch_bytes;
    const uint8_t * rec_global;   // ncols planar records written by mma_quantize_kernel (workspace)
    mma_act A;
};

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

// NG consumer groups per CTA, each = 8 consumer warps + its own producer warp, stage ring, barriers and tile sequence (group v of the
// NG * grid "virtual CTAs" takes tiles v, v + NG * grid, ...); the groups share the activation records.  Two groups drift out of phase, so one
// group's fragment loads overlap the other's mma / scaling arithmetic, and a tile round costs a group-time instead of a CTA-time.
template <int T, int NG>
__global__ void __launch_bounds__(NG * (MMA_GROUP_WARPS + 1) * 32, 1) mmvq_mma_kernel(const mma_params p) {
    using F = mmafmt<T>;
    constexpr int GW = MMA_GROUP_WARPS;
    extern __shared__ __align__(128) uint8_t smem[];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int grp = warp / (GW + 1), wg = warp - grp * (GW + 1);                    // group, warp within the group (GW = the producer)
    uint8_t * stages = smem + (size_t)grp * p.nstages * p.stage_bytes;              // this group's ring (p.nstages stages per group)
    uint8_t * rec    = smem + (size_t)NG * p.nstages * p.stage_bytes;               // ncols planar records
    float * partial  = (float *)(rec + (size_t)p.ncols * p.A.col_bytes) + grp * (2 * GW * 128);   // per group [2][GW][128]
    uint64_t * bars  = (uint64_t *)((float *)(rec + (size_t)p.ncols * p.A.col_bytes) + NG * (2 * GW * 128));
    uint64_t * full  = bars + grp * (2 * MMA_MAX_STAGES);
    uint64_t * empty = full + MMA_MAX_STAGES;
    uint64_t * rec_full = bars + NG * (2 * MMA_MAX_STAGES);                         // the activation records have landed
    int2 * unit_of   = (int2 *)(rec_full + 2) + grp * MMA_MAX_STAGES;               // (tile, slice) held by each stage; tile < 0 = end

    pdl_launch_dependents();
    if (wg == 0 && lane == 0) {
        for (int s = 0; s < p.nstages; ++s) { sb_mbar_init(&full[s], 1); sb_mbar_init(&empty[s], GW); }
        if (grp == 0) sb_mbar_init(rec_full, 1);
        sb_fence_mbar_init();
    }
    __syncthreads();
    const int vcta = (int)blockIdx.x * NG + grp, vgrid = (int)gridDim.x * NG;

    if (wg == GW) {
        // ===== producer warp: lane r copies row r of the tile (slice) — sixteen bulk copies per stage, one barrier
        if (!p.src0_static) pdl_wait();
        int s = 0; uint32_t par = 0; bool wrapped = false;        // ring position: stage, parity of the round, past the first round
        int tile = vcta;
        bool first = true;
        while (true) {
            const bool valid = tile < p.ntiles;
            // Tiles are dealt round-robin (v, v + vgrid, ...) unless p.counters is set.  Dynamic hand-out (one global atomic per tile) gained
            // nothing here: with a few tiles per group the atomic's round trip sits between consecutive stages of the ring.
            int next = tile + vgrid;
            if (p.counters && valid && lane == 0) next = (int)atomicAdd(&p.counters[0], 1u) + vgrid;
            const int nsl = valid ? p.nslices : 1;
            for (int sl = 0; sl < nsl; ++sl) {
                if (wrapped) sb_mbar_wait(&empty[s], par ^ 1u);
                if (valid) {
                    const int64_t row0 = (int64_t)tile * MMA_TILE;
                    const int rows = (int)min((int64_t)MMA_TILE, p.M - row0);
                    const int nt = min(p.ks, p.ntask_row - sl * p.ks);
                    const uint32_t seg = (uint32_t)nt * (uint32_t)F::TASK_B;
                    if (lane == 0) { unit_of[s] = make_int2(tile, sl); sb_mbar_expect_tx(&full[s], (uint32_t)rows * seg); }
                    __syncwarp();
                    if (lane < rows)
                        sb_tma_g2s(stages + (size_t)s * p.stage_bytes + (size_t)lane * p.pitch,
                                   p.w + (size_t)(row0 + lane) * p.row_bytes + (size_t)sl * p.ks * F::TASK_B, seg, &full[s]);
                } else if (lane == 0) {
                    unit_of[s] = make_int2(-1, 0);
                    sb_mbar_arrive(&full[s]);                       // publish the end marker
                }
                if (++s == p.nstages) { s = 0; par ^= 1u; wrapped = true; }
            }
            if (first && p.l2_prefetch_bytes > 0 && lane == 0) {
                // a dependent launch cannot consume before its predecessor's output is visible, but HBM need not idle meanwhile:
                // virtual CTA v pulls slice v of the matrix into L2, the rings then stream from L2
                const int64_t per = ((p.l2_prefetch_bytes + vgrid - 1) / vgrid + 15) & ~(int64_t)15;
                const int64_t lo = (int64_t)vcta * per;
                const int64_t hi = min(lo + per, p.l2_prefetch_bytes & ~(int64_t)15);
                for (int64_t o = lo; o < hi; o += 32768) sb_prefetch_l2(p.w + o, (uint32_t)min((int64_t)32768, hi - o));
            }
            first = false;
            if (!valid) break;
            tile = p.counters ? __shfl_sync(0xffffffffu, next, 0) : next;
        }
        if (p.counters && lane == 0) {
            // last producer to finish its scheduling resets the counters for the next launch
            __threadfence();
            if (atomicAdd(&p.counters[1], 1u) == (unsigned)vgrid - 1) { p.counters[0] = 0; p.counters[1] = 0; __threadfence(); }
        }
        return;
    }

    // ===== consumers: the quantized activation columns (written by the pre-kernel just before this one) -> shared memory
    if (tid == 0) {
        pdl_wait();
        sb_mbar_expect_tx(rec_full, (uint32_t)p.ncols * (uint32_t)p.A.col_bytes);
        for (int c = 0; c < p.ncols; ++c)
            sb_tma_g2s(rec + (size_t)c * p.A.col_bytes, p.rec_global + (size_t)c * p.A.col_bytes, (uint32_t)p.A.col_bytes, rec_full);
    }
    sb_mbar_wait(rec_full, 0u);

    const int g = lane >> 2, t = lane & 3;
    const int gtid = wg * 32 + lane;                                                // thread index within the group's consumers
    mma_cols C;
    C.b  = rec + (size_t)min(g, p.ncols - 1) * p.A.col_bytes;                       // columns beyond n repeat the last one (results discarded)
    C.c0 = rec + (size_t)min(2 * t, p.ncols - 1) * p.A.col_bytes;
    C.c1 = rec + (size_t)min(2 * t + 1, p.ncols - 1) * p.A.col_bytes;
    float facc[4] = { 0.0f, 0.0f, 0.0f, 0.0f };
    int buf = 0;
    int s = 0; uint32_t par = 0;                                                    // ring position: stage, parity of the round
    for (;;) {
        sb_mbar_wait(&full[s], par);
        const int2 unit = unit_of[s];
        if (unit.x < 0) break;
        const int nt = min(p.ks, p.ntask_row - unit.y * p.ks);
        const uint8_t * st = stages + (size_t)s * p.stage_bytes + (size_t)g * p.pitch;
        for (int i = wg; i < nt; i += GW)
            mma_task<T>(st + (size_t)i * F::TASK_B, st + (size_t)i * F::TASK_B + (size_t)8 * p.pitch, C, p.A, unit.y * p.ks + i, t, facc);
        __syncwarp();
        if (lane == 0) sb_mbar_arrive(&empty[s]);
        if (++s == p.nstages) { s = 0; par ^= 1u; }
        if (unit.y == p.nslices - 1) {
            // tile finished: the group's eight partial fragments meet in shared memory and are summed in warp order
            float * part = partial + buf * (GW * 128);
            *(float4 *)(part + wg * 128 + lane * 4) = make_float4(facc[0], facc[1], facc[2], facc[3]);
            facc[0] = facc[1] = facc[2] = facc[3] = 0.0f;
            asm volatile("bar.sync %0, %1;" ::"r"(1 + grp), "n"(GW * 32) : "memory");   // this group's consumers only
            if (gtid < 128) {
                // thread o writes (column o / 16, row o % 16): consecutive threads, consecutive rows of one column
                const int col = gtid >> 4, row = gtid & 15;
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

struct mma_plan { mma_params p; int grid, smem, ng; };

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
    p.counters = nullptr; p.rec_global = nullptr;
    p.src0_static = (a.flags & GGML_B200_MM_SRC0_STATIC) ? 1 : 0;
    p.src1_static = (a.flags & GGML_B200_MM_SRC1_STATIC) ? 1 : 0;
    static const int e_l2_mb = getenv("GGML_B200_SB_L2_MB") ? atoi(getenv("GGML_B200_SB_L2_MB")) : 8;      // L2 prefetch cap: see mmvq_sb.cu
    p.l2_prefetch_bytes = (p.src0_static && e_l2_mb > 0) ? (int64_t)std::min<size_t>((size_t)a.M * rb, (size_t)e_l2_mb << 20) : 0;
    // slices of KS tasks (a multiple of the warp count): whole rows when at least three such stages fit next to the records
    static const int e_ks = getenv("GGML_B200_MMA_KS") ? atoi(getenv("GGML_B200_MMA_KS")) : 0;
    static const int e_stages = getenv("GGML_B200_MMA_STAGES") ? atoi(getenv("GGML_B200_MMA_STAGES")) : 0;
    // consumer groups per CTA: 1 by default, GGML_B200_MMA_GROUPS = 2 for two independent groups (the consume phase is bound by a per-SM
    // rate, not by latency, so more warps on one tile do not help).
    static const int e_groups = getenv("GGML_B200_MMA_GROUPS") ? atoi(getenv("GGML_B200_MMA_GROUPS")) : 1;
    const size_t budget = 226 * 1024;
    for (int ng = e_groups == 2 ? 2 : 1; ng >= 1; --ng) {            // two groups when each gets a ring of >= 2 stages next to the records
        pl.ng = ng;
        const size_t fixed = (size_t)p.ncols * p.A.col_bytes + (size_t)ng * 2 * MMA_GROUP_WARPS * 128 * 4 + (size_t)ng * 2 * MMA_MAX_STAGES * 8 + 16
                           + (size_t)ng * MMA_MAX_STAGES * 8 + 128;
        if (fixed + (size_t)ng * 2 * 8 * F::TASK_B * MMA_TILE > budget) continue;
        auto geometry = [&](int ks) {
            p.ks = ks;
            p.nslices = (p.ntask_row + ks - 1) / ks;
            int pitch = std::min(ks, p.ntask_row) * F::TASK_B;
            pitch = (pitch + 15) & ~15;
            while ((pitch & 127) != F::RESIDUE) pitch += 16;
            p.pitch = pitch;
            p.stage_bytes = (pitch * MMA_TILE + 127) & ~127;
            return (int)std::min<size_t>((budget - fixed) / p.stage_bytes / ng, MMA_MAX_STAGES);   // stages per group
        };
        int ks = e_ks > 0 ? e_ks : 16;                   // 16 tasks x 16 rows: 36 KB (Q4_K) .. 70 KB (Q8_0) per stage
        if (ks > p.ntask_row) ks = p.ntask_row;
        int nst = geometry(ks);
        while (nst < (ng == 1 ? 3 : 2) && ks > 8) { ks = std::max(8, ks / 2); nst = geometry(ks); }
        if (nst < 2) continue;
        if (e_stages >= 2 && e_stages <= nst) nst = e_stages;
        p.nstages = nst;
        pl.smem = (int)(fixed + (size_t)ng * p.nstages * p.stage_bytes);
        pl.grid = std::min(sm_count(), (p.ntiles + ng - 1) / ng);
        return true;
    }
    return false;
}

static size_t mma_rec_bytes(const mma_plan & pl) { return (size_t)pl.p.ncols * pl.p.A.col_bytes; }

template <int T, int NG> static int launch_mma_ng(const mma_plan & pl, cudaStream_t st, const cudaLaunchAttribute * attr, int nattr) {
    static per_device_flag attr_set;
    if (!attr_set.test()) {
        B200_CUDA_TRY(cudaFuncSetAttribute(mmvq_mma_kernel<T, NG>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        attr_set.set();
    }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(pl.grid); cfg.blockDim = dim3(NG * (MMA_GROUP_WARPS + 1) * 32); cfg.dynamicSmemBytes = pl.smem; cfg.stream = st;
    cfg.attrs = const_cast<cudaLaunchAttribute *>(attr); cfg.numAttrs = nattr;
    B200_CUDA_TRY(cudaLaunchKernelEx(&cfg, mmvq_mma_kernel<T, NG>, pl.p));
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

template <int T> static int launch_mma(const ggml_b200_mul_mat_args & a, cudaStream_t st) {
    using F = mmafmt<T>;
    mma_plan pl;
    if (!make_mma_plan<T>(a, pl)) { set_error("mul_mat: shape not eligible for the mma small-batch kernel"); return GGML_B200_EUNSUPPORTED; }
    const size_t need = mma_rec_bytes(pl) + 256;
    if (!a.workspace || a.workspace_size < need) { set_error("mul_mat: workspace %zu < %zu", a.workspace_size, need); return GGML_B200_EWORKSPACE; }
    uint8_t * rec = (uint8_t *)(((uintptr_t)a.workspace + 255) & ~(uintptr_t)255);
    pl.p.rec_global = rec;
    unsigned int * ctl = sb_control_block();
    if (!ctl) return GGML_B200_ECUDA;
    static const bool e_dynamic = getenv("GGML_B200_MMA_DYNAMIC") && atoi(getenv("GGML_B200_MMA_DYNAMIC")) != 0;
    pl.p.counters = e_dynamic ? sb_next_slot(ctl) : nullptr;
    static const bool use_pdl = !(getenv("GGML_B200_NO_PDL") && atoi(getenv("GGML_B200_NO_PDL")) != 0);
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    {
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3((unsigned)((pl.p.ncols * pl.p.A.ntask + 15) / 16)); cfg.blockDim = dim3(256); cfg.dynamicSmemBytes = 0; cfg.stream = st;
        cfg.attrs = attr; cfg.numAttrs = use_pdl ? 1 : 0;
        B200_CUDA_TRY(cudaLaunchKernelEx(&cfg, mma_quantize_kernel<F::KQ, F::S16, mma_s81<T>::value>, a.src1, pl.p.x_stride, (int)pl.p.ncols, pl.p.A, rec));
        B200_LAUNCH_CHECK();
    }
    return pl.ng == 1 ? launch_mma_ng<T, 1>(pl, st, attr, use_pdl ? 1 : 0) : launch_mma_ng<T, 2>(pl, st, attr, use_pdl ? 1 : 0);
}

size_t mmvq_mma_workspace(const ggml_b200_mul_mat_args & a) {
    mma_plan pl;
    bool ok = false;
    switch (a.type) {
        case T_Q4_0: ok = make_mma_plan<T_Q4_0>(a, pl); break;
        case T_Q8_0: ok = make_mma_plan<T_Q8_0>(a, pl); break;
        case T_Q4_K: ok = make_mma_plan<T_Q4_K>(a, pl); break;
        case T_Q5_K: ok = make_mma_plan<T_Q5_K>(a, pl); break;
        case T_Q6_K: ok = make_mma_plan<T_Q6_K>(a, pl); break;
        case T_Q5_0: ok = make_mma_plan<T_Q5_0>(a, pl); break;
        case T_Q4_1: ok = make_mma_plan<T_Q4_1>(a, pl); break;
        case T_Q5_1: ok = make_mma_plan<T_Q5_1>(a, pl); break;
        case T_IQ4_NL: ok = make_mma_plan<T_IQ4_NL>(a, pl); break;
        case T_IQ4_XS: ok = make_mma_plan<T_IQ4_XS>(a, pl); break;
        case T_Q2_K: ok = make_mma_plan<T_Q2_K>(a, pl); break;
        case T_Q3_K: ok = make_mma_plan<T_Q3_K>(a, pl); break;
        default: break;
    }
    return ok ? mma_rec_bytes(pl) + 256 : 0;
}

bool mmvq_mma_eligible(const ggml_b200_mul_mat_args & a) {
    mma_plan pl;
    switch (a.type) {
        case T_Q4_0: return make_mma_plan<T_Q4_0>(a, pl);
        case T_Q8_0: return make_mma_plan<T_Q8_0>(a, pl);
        case T_Q4_K: return make_mma_plan<T_Q4_K>(a, pl);
        case T_Q5_K: return make_mma_plan<T_Q5_K>(a, pl);
        case T_Q6_K: return make_mma_plan<T_Q6_K>(a, pl);
        case T_Q5_0: return make_mma_plan<T_Q5_0>(a, pl);
        case T_Q4_1: return make_mma_plan<T_Q4_1>(a, pl);
        case T_Q5_1: return make_mma_plan<T_Q5_1>(a, pl);
        case T_IQ4_NL: return make_mma_plan<T_IQ4_NL>(a, pl);
        case T_IQ4_XS: return make_mma_plan<T_IQ4_XS>(a, pl);
        case T_Q2_K: return make_mma_plan<T_Q2_K>(a, pl);
        case T_Q3_K: return make_mma_plan<T_Q3_K>(a, pl);
        default: return false;
    }
}

int launch_mmvq_mma(const ggml_b200_mul_mat_args & a, cudaStream_t st) {
    switch (a.type) {
        case T_Q4_0: return launch_mma<T_Q4_0>(a, st);
        case T_Q8_0: return launch_mma<T_Q8_0>(a, st);
        case T_Q4_K: return launch_mma<T_Q4_K>(a, st);
        case T_Q5_K: return launch_mma<T_Q5_K>(a, st);
        case T_Q6_K: return launch_mma<T_Q6_K>(a, st);
        case T_Q5_0: return launch_mma<T_Q5_0>(a, st);
        case T_Q4_1: return launch_mma<T_Q4_1>(a, st);
        case T_Q5_1: return launch_mma<T_Q5_1>(a, st);
        case T_IQ4_NL: return launch_mma<T_IQ4_NL>(a, st);
        case T_IQ4_XS: return launch_mma<T_IQ4_XS>(a, st);
        case T_Q2_K: return launch_mma<T_Q2_K>(a, st);
        case T_Q3_K: return launch_mma<T_Q3_K>(a, st);
        default: set_error("mul_mat: unsupported weight type %d for the mma kernel", a.type); return GGML_B200_EUNSUPPORTED;
    }
}

} // namespace b200
