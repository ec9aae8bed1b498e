// mmvq_sb.cu — the bandwidth-path quantized mat-vec (1 <= n <= 8), second generation: "one lane per 256-weight task".
//
// Why: the first TMA kernel moved exactly the algorithmic bytes from DRAM but spent
// 5.0 M warp-instructions on a 45 M-weight matrix (6-bit scale decode repeated per 64 weights with a run-time
// sub-block index, activation quantization repeated by 444 small CTAs on their critical path, 12 warps per SM),
// i.e. it was issue/latency-bound at 30 % of the HBM roofline.  Here:
//   * a lane owns a whole TASK = 256 consecutive weights of one row (a K-quant superblock, or 8 Q4_0 / 4 Q8_0
//     blocks): the 12-byte scale pack is decoded four sub-blocks at a time with packed-byte arithmetic, the mins are
//     applied with dp2a against int16 activation sums, the high nibbles are used in place (u8 dp4a of q & 0xF0 = 16 x
//     the nibble dot), every shared-memory load is "base + immediate" -> ~1.1 instructions per weight;
//   * LPR lanes cooperate on a row (tasks strided by LPR), so a row's dot product is finished by 4-5 shuffles inside
//     a (half-)warp and written straight to y: no cross-warp reduction, no block-wide barrier per stage;
//   * the activation vector is quantized once per CTA (one 256-value act-task per half-warp) while the first TMA
//     stages are in flight, into per-task records whose 368-byte pitch makes every LDS.128 bank-conflict-free;
//   * a dedicated producer warp keeps a ring of TMA bulk copies (cp.async.bulk + mbarrier complete_tx) in flight;
//     consumers release stages through per-stage "empty" mbarriers; chunks after the first are handed out by an
//     atomic counter (self-resetting, one slot per launch), so SMs stay balanced to one chunk, or round-robin for
//     independent launches with at most 16 chunks per CTA (no atomic round trip before a refill);
//   * programmatic dependent launch: an independent launch (SRC0|SRC1_STATIC) runs as 4-warp CTAs of which four
//     launches share an SM -- a pipeline across launches; a dependent launch runs 8-warp CTAs, prefetches its first
//     stages and pulls W into L2 while its predecessor still runs, and only then waits for the predecessor's output;
//   * 2 <= n <= 8: one activation record per column, the weights of a task are decoded once and dotted with every
//     column (bit-identical, column by column, to the n = 1 result);
//   * Q4_K / Q5_K at n = 1 with K <= 4096 (at most 16 tasks per row), 4-warp CTAs: a warp covers a whole row, so each lane's task is
//     fixed for the launch; lane pairs split a task in halves whose activations stay in registers (q45_rows_regs, 2 rows per warp
//     and pass), and the consumers read each stage byte from shared memory once instead of re-reading the activation record for
//     every row (bit-identical results).
// Weights are read once from HBM in the reference's packed layout.  Numerics are those of b200_quants.cuh
// (int8 activations quantized as ggml-cpu does, integer dots, f32 scaling); only the f32 summation order differs.
#include "b200_internal.h"
#include "b200_mm_plan.h"
#include "b200_quants.cuh"
#include "b200_ptx.cuh"
#include "b200_sb_tasks.cuh"   // dp4a_us, task geometry, activation-record layout, task dot products (also compiled for the host by tests/hostemu)

#include <atomic>
#include <cstdlib>

namespace b200 {

// ----------------------------------------------------------------------------- kernel
constexpr int SB_MAX_STAGES = 6;

// how the consumer lanes split a stage: a task per lane (every format), or, for Q4_K / Q5_K at n = 1, two rows per lane group
// sharing each activation load, or activations held in registers (a lane's task fixed for the launch, K <= 4096)
enum sb_consume { SB_TASKS = 0, SB_TWO_ROWS = 1, SB_ACT_REGS = 2 };

template <int T, int NW, int NC, int CM = SB_TASKS>
__global__ void __launch_bounds__((NW + 1) * 32, NC > 1 ? 1 : NW == 8 ? 2 : 4) mmvq_sb_kernel(const sb_params p) {
    using F = sbfmt<T>;
    constexpr int SB_CONSUMER_WARPS = NW;
    constexpr int LPR = F::LPR, RPW = 32 / LPR;                 // rows per warp pass
    extern __shared__ __align__(128) uint8_t smem[];
    uint8_t * stages = smem;
    uint8_t * rec    = stages + (size_t)p.nstages * p.stage_bytes;
    uint64_t * full  = (uint64_t *)(rec + NC * p.A.bytes);      // NC activation records (one per column)
    uint64_t * empty = full + SB_MAX_STAGES;
    int * chunk_of   = (int *)(empty + SB_MAX_STAGES);          // chunk id held by each stage (-1 = end)

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    pdl_launch_dependents();

    if (tid == 0) {
        for (int s = 0; s < p.nstages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], SB_CONSUMER_WARPS); }
        mbar_fence_init();
    }
    __syncthreads();

    auto issue = [&](int s, int chunk) {
        chunk_of[s] = chunk < p.nchunks ? chunk : -1;
        if (chunk < p.nchunks) {
            const int64_t row0 = (int64_t)chunk * p.rows_per_chunk;
            const int rows = (int)min((int64_t)p.rows_per_chunk, p.M - row0);
            const uint32_t bytes = (uint32_t)rows * (uint32_t)p.row_bytes;
            mbar_expect_tx(&full[s], bytes);
            bulk_g2s(stages + (size_t)s * p.stage_bytes, p.w + (size_t)row0 * p.row_bytes, bytes, &full[s]);
        } else {
            mbar_arrive(&full[s]);                             // publish the end marker
        }
    };

    if (warp == SB_CONSUMER_WARPS) {
        // ===== producer warp: weights do not depend on the previous kernel, start streaming immediately
        if (lane == 0) {
            if (!p.src0_static) pdl_wait();
            issue(0, (int)blockIdx.x);                            // first chunk is static
            if (p.l2_prefetch_bytes > 0) {
                // this launch cannot consume before the previous kernel's output is visible, but HBM need not idle meanwhile:
                // CTA b pulls slice b of the matrix into L2 (whoever ends up consuming it), the ring then streams from L2
                const int64_t per = ((p.l2_prefetch_bytes + gridDim.x - 1) / gridDim.x + 15) & ~(int64_t)15;
                const int64_t lo = (int64_t)blockIdx.x * per;
                const int64_t hi = min(lo + per, p.l2_prefetch_bytes & ~(int64_t)15);
                for (int64_t o = lo; o < hi; o += 32768) bulk_prefetch_l2(p.w + o, (uint32_t)min((int64_t)32768, hi - o));
            }
            // (the scheduling counters are per launch slot, so the producer never has to wait for the previous grid on their account)
            // the next chunk index is fetched (one global atomic round trip) BEFORE waiting for a free stage, so the atomic's
            // latency overlaps the consumers' work instead of delaying the refill
            int it = 1;
            bool done = (int)blockIdx.x >= p.nchunks;
            if (p.static_chunks) {
                // chunks dealt round-robin (b, b + grid, ...): no atomic round trip (~1 us) between consecutive stages of this CTA's ring
                while (!done) {
                    const int s = it % p.nstages;
                    const int chunk = (int)blockIdx.x + it * (int)gridDim.x;
                    if (it >= p.nstages) mbar_wait(&empty[s], (uint32_t)((it / p.nstages) - 1) & 1u);
                    issue(s, chunk);
                    done = chunk >= p.nchunks;
                    ++it;
                }
                return;
            }
            while (!done) {
                const int s = it % p.nstages;
                const int chunk = (int)atomicAdd(&p.counters[0], 1u) + (int)gridDim.x;
                if (it >= p.nstages) mbar_wait(&empty[s], (uint32_t)((it / p.nstages) - 1) & 1u);
                issue(s, chunk);
                done = chunk >= p.nchunks;
                ++it;
            }
            // last CTA to finish its scheduling resets the counters for the next launch
            __threadfence();
            if (atomicAdd(&p.counters[1], 1u) == gridDim.x - 1) { p.counters[0] = 0; p.counters[1] = 0; __threadfence(); }
        }
        return;
    }

    // ===== consumers: quantize the activation vector (needs the previous kernel's output)
    if (!p.src1_static) pdl_wait();
    // one act-task per half-warp per round (this phase is on the critical path of a dependent launch: it can only start once
    // the previous kernel's output is visible)
    for (int i0 = 2 * warp; i0 < p.ncols * p.A.ntask; i0 += 2 * SB_CONSUMER_WARPS) {
        const int i = i0 + (lane >> 4);
        const bool ok = i < p.ncols * p.A.ntask;
        const int c = NC == 1 ? 0 : (ok ? i / p.A.ntask : 0), t = NC == 1 ? i : (ok ? i % p.A.ntask : 0);
        sb_quantize_task_h<F::KQ != 0, needs_s<T>::value>(p.x + (size_t)c * p.x_stride, ok, rec + c * p.A.bytes, t);
    }
    asm volatile("bar.sync 1, %0;" ::"n"(SB_CONSUMER_WARPS * 32) : "memory");        // consumers only

    // rows per warp and pass of the activation-stationary form (0: not used)
    constexpr int AR = NC == 1 && (T == T_Q4_K || T == T_Q5_K) && CM == SB_ACT_REGS ? 2 : 0;
    q45_acts acts;                                                // this lane's half of its act-task, loaded once
    if constexpr (AR > 0) { if ((lane >> 1) < p.ntasks_row) q45_load_acts(rec, lane >> 1, lane & 1, acts); }

    const int sub = lane / LPR, l = lane % LPR;
    for (int it = 0;; ++it) {
        const int s = it % p.nstages;
        mbar_wait(&full[s], (uint32_t)(it / p.nstages) & 1u);
        const int chunk = chunk_of[s];
        if (chunk < 0) break;                                     // last stage done
        const int64_t row0 = (int64_t)chunk * p.rows_per_chunk;
        const int rows = (int)min((int64_t)p.rows_per_chunk, p.M - row0);
        const uint8_t * st = stages + (size_t)s * p.stage_bytes;
        auto store_row = [&](int64_t grow, float acc) {
            if (p.world == 0) {
                p.y[grow] = acc;
                if (p.ep_bias) {
                    const float v2 = acc + p.ep_bias[grow];
                    p.ep_y2[grow] = v2;
                    if (p.ep_y3) p.ep_y3[grow] = p.ep_res ? v2 + p.ep_res[grow] : gelu_ggml(v2);
                }
            } else {
                // row-sharded multi-GPU: straight into the gathered y of every rank (own one included) over NVLink
                const int64_t gi = p.row_offset + grow;
#pragma unroll
                for (int q = 0; q < 8; ++q) if (q < p.world) p.y_peers[q][gi] = acc;
            }
        };
        if constexpr (AR > 0) {
            // AR rows per warp and pass, the activations already in registers: only weights are read from shared memory
            for (int r0 = warp * AR; r0 < rows; r0 += SB_CONSUMER_WARPS * AR) {
                const uint8_t * rp[AR];
#pragma unroll
                for (int j = 0; j < AR; ++j) rp[j] = st + (size_t)min(r0 + j, rows - 1) * p.row_bytes;    // past the end: repeat the last row (not stored)
                const float acc = q45_rows_regs<T == T_Q5_K, AR>(rp, acts, lane, p.ntasks_row);
                const int r = r0 + lane / (32 / AR);
                if (lane % (32 / AR) == 0 && r < rows) store_row(row0 + r, acc);
            }
        } else if constexpr (CM == SB_TWO_ROWS && NC == 1 && (T == T_Q4_K || T == T_Q5_K)) {
            // two rows per lane group and pass, sharing every activation load (each row's operations and their order are those of the
            // one-row path: bit-identical results); halves the activation traffic out of shared memory
            for (int r0 = warp * RPW * 2; r0 < rows; r0 += SB_CONSUMER_WARPS * RPW * 2) {
                const int r = r0 + 2 * sub;
                float a0 = 0.0f, a1 = 0.0f;
                if (r < rows) {
                    const uint8_t * ra = st + (size_t)r * p.row_bytes, * rb = r + 1 < rows ? ra + p.row_bytes : ra;
                    for (int t = l; t < p.ntasks_row; t += LPR) {
                        float x0, x1;
                        q45_task2<T == T_Q5_K>(ra + (size_t)t * F::TASK_B, rb + (size_t)t * F::TASK_B, rec, t, x0, x1);
                        a0 += x0; a1 += x1;
                    }
                }
#pragma unroll
                for (int o = LPR / 2; o > 0; o >>= 1) { a0 += __shfl_xor_sync(0xffffffffu, a0, o); a1 += __shfl_xor_sync(0xffffffffu, a1, o); }
                if (l == 0 && r < rows) { store_row(row0 + r, a0); if (r + 1 < rows) store_row(row0 + r + 1, a1); }
            }
        } else {
            // the row loop is warp-uniform (both half-warps iterate together): the shuffles below use the full mask
            for (int r0 = warp * RPW; r0 < rows; r0 += SB_CONSUMER_WARPS * RPW) {
                const int r = r0 + sub;
                if constexpr (NC > 1) {
                    float accn[NC];
#pragma unroll
                    for (int c = 0; c < NC; ++c) accn[c] = 0.0f;
                    if (r < rows) {
                        const uint8_t * row = st + (size_t)r * p.row_bytes;
                        for (int t = l; t < p.ntasks_row; t += LPR) task_dot_nc<T, NC>(row + (size_t)t * F::TASK_B, rec, p.A.bytes, t, p.ncols, accn);
                    }
#pragma unroll
                    for (int c = 0; c < NC; ++c) {
#pragma unroll
                        for (int o = LPR / 2; o > 0; o >>= 1) accn[c] += __shfl_xor_sync(0xffffffffu, accn[c], o);
                    }
                    if (l == 0 && r < rows) {
#pragma unroll
                        for (int c = 0; c < NC; ++c) if (c < p.ncols) p.y[(size_t)c * p.M + row0 + r] = accn[c];
                    }
                    continue;
                }
                float acc = 0.0f;
                if (r < rows) {
                    const uint8_t * row = st + (size_t)r * p.row_bytes;
                    for (int t = l; t < p.ntasks_row; t += LPR) acc += task_dot<T>(row + (size_t)t * F::TASK_B, rec, t);
                }
#pragma unroll
                for (int o = LPR / 2; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
                if (l == 0 && r < rows) store_row(row0 + r, acc);
            }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[s]);
    }
    // Completion must stay transitive along the stream (a later kernel's griddepcontrol.wait covers only ITS predecessor): a launch
    // whose consumers did not wait for the preceding grid (SRC1_STATIC) does so before it retires, holding no work back.
    if (p.src1_static && tid == 0) pdl_wait();
    if (p.world > 0) {
        // fused gather, publication: every row was already stored into every rank's gathered y by the lane that finished it (the row
        // loop above), so the exchange traffic is spread over all SMs and overlaps the streaming of the remaining rows.  Here each
        // thread makes its own remote stores visible system-wide, the CTA counts itself done, and the CTA that finishes last raises
        // this rank's epoch in every peer's flag array (stores -> fence.sys -> counter -> fence.sys -> release flag: causally ordered).
        // The griddepcontrol.wait above keeps the publications of overlapping launches in launch order.
        __threadfence_system();
        asm volatile("bar.sync 1, %0;" ::"n"(SB_CONSUMER_WARPS * 32) : "memory");
        if (tid == 0 && atomicAdd(&p.counters[2], 1u) == gridDim.x - 1) {
            p.counters[2] = 0;
            // the exchange epoch lives on the device (ctl[0]) so that a CUDA graph can replay the launch; the flags only ever grow
            const uint32_t e = p.epoch ? p.epoch : atomicAdd(&p.ctl[0], 1u) + 1u;
            __threadfence_system();
            for (int q = 0; q < p.world; ++q)
                asm volatile("red.release.sys.global.max.u32 [%0], %1;" ::"l"(p.flag_peers[q] + p.rank), "r"(e) : "memory");
        }
    }
}

// wait until every rank has published `epoch` in this rank's flag array (one warp)
__global__ void gather_wait_kernel(const uint32_t * flags, int world, uint32_t epoch, const unsigned int * ctl) {
    const int q = threadIdx.x;
    if (epoch == 0) epoch = ctl[0];          // the epoch this rank published with its last fused mat-vec
    if (q < world) {
        uint32_t v;
        do {
            asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(flags + q) : "memory");
        } while ((int32_t)(v - epoch) < 0);
    }
    __syncwarp();
    __threadfence_system();
}

static std::atomic<unsigned> g_sb_slot_seq{0};
unsigned int * sb_next_slot(unsigned int * ctl) { return ctl + 64 + (g_sb_slot_seq.fetch_add(1, std::memory_order_relaxed) % 64u) * 8; }

template <int T> static bool make_sb_plan(const ggml_b200_mul_mat_args & a, sb_plan & pl) {
    using F = sbfmt<T>;
    if (a.N < 1 || a.N > 8 || a.ne02 != 1 || a.ne03 != 1 || a.ne12 != 1 || a.ne13 != 1) return false;
    if (a.N > 1 && ((a.nb11 & 3) != 0 || a.nb11 < (size_t)a.K * 4)) return false;
    const int nc = a.N == 1 ? 1 : a.N == 2 ? 2 : a.N <= 4 ? 4 : 8;       // kernel instantiation (columns beyond N are skipped)
    pl.nc = nc;
    if (a.K % 256 != 0 || a.K < 256 || a.M < 1 || a.K > 32768) return false;
    const size_t rb = row_bytes(a.type, a.K);
    if (a.nb01 != rb || ((uintptr_t)a.src0 & 15) != 0 || ((uintptr_t)a.src1 & 3) != 0) return false;
    if ((a.M * rb) % 16 != 0) return false;
    // Two operating points: launches flagged independent of their predecessor (SRC1_STATIC) run as
    // small CTAs (4 consumer warps, 18 KB stages) of which four launches share an SM, a deep pipeline ACROSS launches; a dependent
    // launch wants its prologue short and its prefetch deep: 8 consumer warps, 36 KB stages, two launches per SM, W pulled into L2.
    const bool ind = (a.flags & GGML_B200_MM_SRC1_STATIC) != 0 && a.N == 1;
    const int stage_kb = ind ? 18 : 36;
    const int SB_CONSUMER_WARPS = ind ? 4 : 8;
    pl.nw = SB_CONSUMER_WARPS;
    constexpr int RPW = 32 / F::LPR;
    // two rows per lane group sharing the activation loads (Q4_K / Q5_K, n = 1): faster on dependent launches (the consume phase is bounded by
    // shared-memory traffic, most of it activation reads), slower for independent launches (fewer co-resident CTAs): used for DEPENDENT
    // launches with enough tasks per row, which always run 8-warp CTAs
    pl.two = nc == 1 && (T == T_Q4_K || T == T_Q5_K) && !ind && a.K >= 2048 && a.M >= 2048 && (size_t)(SB_CONSUMER_WARPS * RPW * 2) * rb <= 100 * 1024;
    // activations held in registers (Q4_K / Q5_K, n = 1, at most 16 tasks per row) in the 4-warp kernel of independent launches: each stage
    // byte is read from shared memory once instead of with a re-read activation record (faster on an H100 at 400 W; the 8-warp kernel of
    // dependent launches, where it measured slower than the two-row form, keeps the shared-memory paths).  The chunk geometry is unchanged.
    // GGML_B200_SB_ACT_REGS = 0 keeps the shared-memory consume paths everywhere
    static const int e_areg = getenv("GGML_B200_SB_ACT_REGS") ? atoi(getenv("GGML_B200_SB_ACT_REGS")) : 1;
    pl.act_regs = e_areg != 0 && nc == 1 && (T == T_Q4_K || T == T_Q5_K) && a.K <= 16 * 256 && SB_CONSUMER_WARPS == 4;
    int granule = 1; while ((granule * rb) % 16 != 0) granule *= 2;
    int step = SB_CONSUMER_WARPS * RPW * (pl.two ? 2 : 1); while (step % granule != 0) step *= 2;
    int rpc = (int)(((size_t)stage_kb * 1024) / rb) / step * step; if (rpc < step) rpc = step;
    if ((size_t)rpc * rb > 100 * 1024) {                         // very long rows: fewer rows per chunk than one full pass
        rpc = granule; while ((size_t)(rpc + granule) * rb <= 48 * 1024) rpc += granule;
        if ((size_t)rpc * rb > 100 * 1024) return false;
    }
    sb_params & p = pl.p;
    p.M = a.M; p.K = a.K;
    p.row_bytes = (int)rb; p.rows_per_chunk = rpc; p.nchunks = (int)((a.M + rpc - 1) / rpc);
    p.stage_bytes = (int)(((size_t)rpc * rb + 127) & ~(size_t)127);
    p.ntasks_row = (int)(a.K / F::TASK_W);
    p.A = make_sb_act(a.K);
    p.w = nullptr; p.x = nullptr; p.y = nullptr;                 // bound at launch (launch_sb_t)
    p.ctl = nullptr; p.counters = nullptr;                       // assigned at launch (assign_sb_slot): planning has no side effects
    p.src0_static = (a.flags & GGML_B200_MM_SRC0_STATIC) ? 1 : 0;
    p.l2_prefetch_bytes = (!ind && p.src0_static) ? (int64_t)std::min<size_t>((size_t)a.M * rb, (size_t)L2_PREFETCH_CAP) : 0;
    p.world = 0; p.rank = 0; p.row_offset = 0; p.epoch = 0;
    p.ep_bias = nullptr; p.ep_y2 = nullptr; p.ep_y3 = nullptr; p.ep_res = nullptr;
    p.src1_static = (a.flags & GGML_B200_MM_SRC1_STATIC) ? 1 : 0;
    p.ncols = (int32_t)a.N; p.x_stride = a.N > 1 ? (int64_t)(a.nb11 / 4) : 0;
    for (int q = 0; q < 8; ++q) { p.y_peers[q] = nullptr; p.flag_peers[q] = nullptr; }
    auto smem_of = [&]() { return p.nstages * p.stage_bytes + nc * p.A.bytes + 2 * SB_MAX_STAGES * 8 + SB_MAX_STAGES * 4 + 64; };
    const int max_res = nc > 1 ? 1 : SB_CONSUMER_WARPS == 8 ? 2 : 4;                       // register-limited residency (__launch_bounds__)
    const int resident = std::min(ind ? 4 : 2, max_res);
    // deepest ring that still lets `resident` CTAs (of consecutive launches) share an SM, so that programmatic dependent
    // launch can overlap the next mat-vec's prologue and first TMA round trip with this one's tail
    p.nstages = 4;
    while (p.nstages > 2 && smem_of() * resident > 226 * 1024) p.nstages--;
    while (smem_of() > 222 * 1024 && p.nstages > 2) p.nstages--;
    if (smem_of() > 222 * 1024) return false;
    pl.smem = smem_of();
    pl.grid = std::min(sm_count(), p.nchunks);
    // Independent launches with at most 16 chunks per CTA take them round-robin: the producer's atomic round trip before each refill is
    // not hidden by two stages, and the co-resident launches absorb the imbalance of a few chunks.  With more chunks per CTA the SMs'
    // speed differences add up and the atomic counter balances better.  Measured on an H100 at 700 W: Q4_K 4096 -> 11008 (10 chunks per
    // CTA) 3164 instead of 3144 GB/s, Q4_0 4096 x 4096 (4) 2937 instead of 2792; Q4_K / Q8_0 4096 -> 32000 (30 / 61) 2.5 / 3.8 % slower
    // round-robin.  Dependent launches keep the atomic counter.
    p.static_chunks = (ind && p.nchunks <= 16 * pl.grid) ? 1 : 0;
    return true;
}

// a launch takes the next of the 64 scheduling slots of this device's control block (self-resetting counters: a slot is free again
// when its launch has finished scheduling, and 64 launches never overlap on one device)
static int assign_sb_slot(sb_params & p) {
    p.ctl = control_block();
    if (!p.ctl) return GGML_B200_ECUDA;
    p.counters = sb_next_slot(p.ctl);
    return GGML_B200_OK;
}

template <int T, int NW, int NC, int CM = SB_TASKS> static int launch_sb_nw(sb_plan & pl, cudaStream_t st) {
    B200_CUDA_TRY(set_max_dynamic_smem<mmvq_sb_kernel<T, NW, NC, CM>>(222 * 1024));
    B200_CUDA_TRY(launch_pdl(mmvq_sb_kernel<T, NW, NC, CM>, dim3(pl.grid), dim3((NW + 1) * 32), pl.smem, st, pl.p));
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

template <int T> static int launch_sb_t(const ggml_b200_mul_mat_args & a, sb_plan pl, const ggml_b200_gather * ga, cudaStream_t st, const ggml_b200_epilogue * ep) {
    pl.p.w = (const uint8_t *)a.src0; pl.p.x = a.src1; pl.p.y = a.dst;
    { const int rc = assign_sb_slot(pl.p); if (rc != GGML_B200_OK) return rc; }
    if (ep && ep->bias) {
        pl.p.ep_bias = ep->bias; pl.p.ep_y2 = ep->dst_bias; pl.p.ep_y3 = ep->unary != 0 ? ep->dst_unary : nullptr;
        pl.p.ep_res = ep->unary == 2 ? ep->residual : nullptr;
    }
    if (ga) {
        pl.p.world = ga->world; pl.p.rank = ga->rank; pl.p.row_offset = ga->row_offset; pl.p.epoch = ga->epoch;
        for (int q = 0; q < ga->world; ++q) { pl.p.y_peers[q] = ga->y_peers[q]; pl.p.flag_peers[q] = ga->flag_peers[q]; }
    }
    if (pl.nc > 1 && (ga || (ep && ep->bias))) { set_error("mul_mat: the fused epilogue / gather exist for n = 1 only"); return GGML_B200_EUNSUPPORTED; }
    switch (pl.nc) {
        case 1:
            if constexpr (T == T_Q4_K || T == T_Q5_K) {
                if (pl.act_regs) return launch_sb_nw<T, 4, 1, SB_ACT_REGS>(pl, st);
                if (pl.two) return launch_sb_nw<T, 8, 1, SB_TWO_ROWS>(pl, st);
            }
            return pl.nw == 4 ? launch_sb_nw<T, 4, 1>(pl, st) : launch_sb_nw<T, 8, 1>(pl, st);
        case 2:  return launch_sb_nw<T, 8, 2>(pl, st);
        case 4:  return launch_sb_nw<T, 8, 4>(pl, st);
        default: return launch_sb_nw<T, 8, 8>(pl, st);
    }
}

bool plan_sb(const ggml_b200_mul_mat_args & a, sb_plan & pl) {
    bool ok = false;
    with_format(TC_FORMATS(), a.type, [&](auto t) { ok = make_sb_plan<t>(a, pl); });
    return ok;
}

int launch_sb(const ggml_b200_mul_mat_args & a, const sb_plan & pl, cudaStream_t st, const ggml_b200_gather * ga, const ggml_b200_epilogue * ep) {
    int rc = GGML_B200_EUNSUPPORTED;                                 // plan_sb accepts TC_FORMATS only
    with_format(TC_FORMATS(), a.type, [&](auto t) { rc = launch_sb_t<t>(a, pl, ga, st, ep); });
    return rc;
}

int launch_gather_wait(const uint32_t * flags, int world, uint32_t epoch, cudaStream_t st) {
    gather_wait_kernel<<<1, 32, 0, st>>>(flags, world, epoch, control_block());
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

} // namespace b200
