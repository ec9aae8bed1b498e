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
//     atomic counter (self-resetting, one slot per launch), so SMs stay balanced to one chunk;
//   * programmatic dependent launch: an independent launch (SRC0|SRC1_STATIC) runs as 4-warp CTAs of which four
//     launches share an SM -- a pipeline across launches; a dependent launch runs 8-warp CTAs, prefetches its first
//     stages and pulls W into L2 while its predecessor still runs, and only then waits for the predecessor's output;
//   * 2 <= n <= 8: one activation record per column, the weights of a task are decoded once and dotted with every
//     column (bit-identical, column by column, to the n = 1 result).
// Weights are read once from HBM in the reference's packed layout.  Numerics are those of b200_quants.cuh
// (int8 activations quantized as ggml-cpu does, integer dots, f32 scaling); only the f32 summation order differs.
#include "b200_internal.h"
#include "b200_quants.cuh"
#include "b200_sb_ptx.cuh"
#include "b200_sb_tasks.cuh"   // dp4a_us, task geometry, activation-record layout, task dot products (also compiled for the host by tests/hostemu)

#include <atomic>
#include <cstdlib>
#include <mutex>

namespace b200 {

// ----------------------------------------------------------------------------- kernel
constexpr int SB_MAX_STAGES = 6;

struct sb_params {
    const uint8_t * w; const float * x; float * y;
    int64_t M, K;
    int32_t row_bytes, rows_per_chunk, nchunks, stage_bytes, nstages, ntasks_row;
    unsigned int * counters;      // this launch's scheduling slot: [0] next chunk, [1] finished producers, [2] finished CTAs (all return to 0)
    unsigned int * ctl;           // device-global control words: [0] exchange epoch, [1] trace launch index
    int32_t ncols; int64_t x_stride;   // activation columns (1..8) and the distance between them in floats; y is [ncols][M]
    int32_t src1_static;          // activations are not produced by the preceding kernel either: never wait for it (independent ops overlap)
    int32_t src0_static;          // weights are not produced by the preceding kernel: prefetch them before griddepcontrol.wait
    int32_t static_chunks;        // chunks dealt round-robin instead of by the atomic counter
    int64_t l2_prefetch_bytes;    // dependent launches: bytes of W every CTA's share of which is pulled into L2 while the previous kernel still runs (0 = off)
    // row-sharded multi-GPU: every result is stored straight into each peer's full-length y over NVLink (world == 0: off)
    // fused epilogue (bias add and GELU of the following ggml nodes): y2 = y + bias, y3 = gelu(y2); null = off
    const float * ep_bias; float * ep_y2; float * ep_y3; const float * ep_res;    // ep_res: y3 = y2 + residual instead of gelu(y2)
    unsigned long long * dbg;     // optional %globaltimer trace (GGML_B200_SB_DEBUG=1): 32 launches x 8 stamps
    int32_t world, rank;
    int64_t row_offset;
    uint32_t epoch;
    float *    y_peers[8];
    uint32_t * flag_peers[8];
    sb_act A;
};

template <int T, int NW, int NC, bool TWO = false>
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
    // trace slot of this launch (host-chosen): CTA 0 stamps [0..5]; every CTA folds its own times into [6] (latest exit) and
    // [7] (latest consumer release from griddepcontrol.wait)
    unsigned long long * dbg = nullptr, * dbg_all = p.dbg;
    if (p.dbg && blockIdx.x == 0) {
        dbg = p.dbg;
        if (tid == 0) dbg[0] = gtime();                          // CTA 0 entry
    }

    if (tid == 0) {
        for (int s = 0; s < p.nstages; ++s) { sb_mbar_init(&full[s], 1); sb_mbar_init(&empty[s], SB_CONSUMER_WARPS); }
        sb_fence_mbar_init();
    }
    __syncthreads();

    auto issue = [&](int s, int chunk) {
        chunk_of[s] = chunk < p.nchunks ? chunk : -1;
        if (chunk < p.nchunks) {
            const int64_t row0 = (int64_t)chunk * p.rows_per_chunk;
            const int rows = (int)min((int64_t)p.rows_per_chunk, p.M - row0);
            const uint32_t bytes = (uint32_t)rows * (uint32_t)p.row_bytes;
            sb_mbar_expect_tx(&full[s], bytes);
            sb_tma_g2s(stages + (size_t)s * p.stage_bytes, p.w + (size_t)row0 * p.row_bytes, bytes, &full[s]);
        } else {
            sb_mbar_arrive(&full[s]);                             // publish the end marker
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
                for (int64_t o = lo; o < hi; o += 32768) sb_prefetch_l2(p.w + o, (uint32_t)min((int64_t)32768, hi - o));
            }
            if (dbg) dbg[1] = gtime();                            // first TMA issued
            // (the scheduling counters are per launch slot, so the producer never has to wait for the previous grid on their account)
            if (dbg) dbg[2] = gtime();                            // producer past griddepcontrol.wait                                           // the chunk counter belongs to the previous launch until it completes
            // the next chunk index is fetched (one global atomic round trip) BEFORE waiting for a free stage, so the atomic's
            // latency overlaps the consumers' work instead of delaying the refill
            int it = 1;
            bool done = (int)blockIdx.x >= p.nchunks;
            if (p.static_chunks) {
                // chunks dealt round-robin (b, b + grid, ...): no atomic round trip (~1 us) between consecutive stages of this CTA's ring
                while (!done) {
                    const int s = it % p.nstages;
                    const int chunk = (int)blockIdx.x + it * (int)gridDim.x;
                    if (it >= p.nstages) sb_mbar_wait(&empty[s], (uint32_t)((it / p.nstages) - 1) & 1u);
                    issue(s, chunk);
                    done = chunk >= p.nchunks;
                    ++it;
                }
                return;
            }
            while (!done) {
                const int s = it % p.nstages;
                const int chunk = (int)atomicAdd(&p.counters[0], 1u) + (int)gridDim.x;
                if (it >= p.nstages) sb_mbar_wait(&empty[s], (uint32_t)((it / p.nstages) - 1) & 1u);
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
    if (dbg && tid == 0) dbg[3] = gtime();                       // consumers past griddepcontrol.wait
    if (dbg_all && tid == 0) atomicMax(dbg_all + 7, gtime());
    // one act-task per half-warp per round (this phase is on the critical path of a dependent launch: it can only start once
    // the previous kernel's output is visible)
    for (int i0 = 2 * warp; i0 < p.ncols * p.A.ntask; i0 += 2 * SB_CONSUMER_WARPS) {
        const int i = i0 + (lane >> 4);
        const bool ok = i < p.ncols * p.A.ntask;
        const int c = NC == 1 ? 0 : (ok ? i / p.A.ntask : 0), t = NC == 1 ? i : (ok ? i % p.A.ntask : 0);
        sb_quantize_task_h<F::KQ != 0, needs_s<T>::value>(p.x + (size_t)c * p.x_stride, ok, rec + c * p.A.bytes, t);
    }
    asm volatile("bar.sync 1, %0;" ::"n"(SB_CONSUMER_WARPS * 32) : "memory");        // consumers only

    const int sub = lane / LPR, l = lane % LPR;
    for (int it = 0;; ++it) {
        const int s = it % p.nstages;
        sb_mbar_wait(&full[s], (uint32_t)(it / p.nstages) & 1u);
        if (dbg && tid == 0 && it == 0) dbg[4] = gtime();        // first stage landed
        const int chunk = chunk_of[s];
        if (chunk < 0) { if (dbg && tid == 0) dbg[5] = gtime(); if (dbg_all && tid == 0) atomicMax(dbg_all + 6, gtime()); break; }   // last stage done
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
        if constexpr (TWO && NC == 1 && (T == T_Q4_K || T == T_Q5_K)) {
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
            __syncwarp();
            if (lane == 0) sb_mbar_arrive(&empty[s]);
            continue;
        }
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
        __syncwarp();
        if (lane == 0) sb_mbar_arrive(&empty[s]);
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

struct sb_plan { sb_params p; int grid, smem, nw, nc; bool two; };

// device control block: [0,64) global control words, [64, 64 + 64*8) 64 per-launch scheduling slots, byte 4096.. trace.
// One per device, allocated on first use under a mutex (or ahead of time by ggml_b200_prepare, which the backend calls at
// device initialisation so that no allocation can fall inside a stream capture) and kept for the life of the process.
static unsigned int * sb_counters() {
    static unsigned int * ptr[64] = { nullptr };
    static std::mutex mu;
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) { set_error("control block: cudaGetDevice failed"); return nullptr; }
    std::lock_guard<std::mutex> lock(mu);
    if (!ptr[dev]) {
        unsigned int * p = nullptr;
        cudaError_t e = cudaMalloc(&p, 8192);
        if (e == cudaSuccess) e = cudaMemset(p, 0, 8192);
        if (e == cudaSuccess) e = cudaDeviceSynchronize();
        if (e != cudaSuccess) {
            set_error("control block: %s", cudaGetErrorString(e));
            cudaGetLastError();
            if (p) cudaFree(p);
            return nullptr;
        }
        ptr[dev] = p;
    }
    return ptr[dev];
}

int prepare_device() { return sb_counters() ? GGML_B200_OK : GGML_B200_ECUDA; }
unsigned int * sb_control_block() { return sb_counters(); }
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
    static const int e_stage_kb = getenv("GGML_B200_SB_STAGE_KB") ? atoi(getenv("GGML_B200_SB_STAGE_KB")) : 0;
    static const int env_stages = getenv("GGML_B200_SB_STAGES")   ? atoi(getenv("GGML_B200_SB_STAGES"))   : 0;
    static const int env_ctas   = getenv("GGML_B200_SB_CTAS")     ? atoi(getenv("GGML_B200_SB_CTAS"))     : 1;
    static const int e_warps    = getenv("GGML_B200_SB_WARPS")    ? atoi(getenv("GGML_B200_SB_WARPS"))    : 0;
    static const int e_resident = getenv("GGML_B200_SB_RESIDENT") ? atoi(getenv("GGML_B200_SB_RESIDENT")) : 0;
    // L2 prefetch cap of dependent launches: 8 MB of the H100's 50 MB L2 (GGML_B200_SB_L2_MB=<MB> python scripts/gemv_sweep.py on an H100:
    // q4_K n = 1 and n = 8 dependent launches 12-17 % faster than with 48 MB, within a few % of no prefetch)
    static const int e_l2_mb    = getenv("GGML_B200_SB_L2_MB")    ? atoi(getenv("GGML_B200_SB_L2_MB"))    : 8;
    const int env_warps    = e_warps    ? e_warps    : (ind ? 4 : 8);
    const int env_resident = e_resident ? e_resident : (ind ? 4 : 2);
    const int env_stage_kb = e_stage_kb ? e_stage_kb : (ind ? 18 : 36);
    const int SB_CONSUMER_WARPS = (env_warps == 4 && nc == 1) ? 4 : 8;
    pl.nw = SB_CONSUMER_WARPS;
    constexpr int RPW = 32 / F::LPR;
    // two rows per lane group sharing the activation loads (Q4_K / Q5_K, n = 1): faster on dependent launches (the consume phase is bounded by
    // shared-memory traffic, most of it activation reads), slower for independent launches (fewer co-resident CTAs): default for DEPENDENT
    // launches with enough tasks per row.  GGML_B200_SB_TWOROW = 0 off, 1 always
    static const int e_two = getenv("GGML_B200_SB_TWOROW") ? atoi(getenv("GGML_B200_SB_TWOROW")) : 2;
    pl.two = nc == 1 && (T == T_Q4_K || T == T_Q5_K) && (e_two == 1 || (e_two == 2 && !ind && a.K >= 2048 && a.M >= 2048 && (size_t)(SB_CONSUMER_WARPS * RPW * 2) * rb <= 100 * 1024));
    int granule = 1; while ((granule * rb) % 16 != 0) granule *= 2;
    int step = SB_CONSUMER_WARPS * RPW * (pl.two ? 2 : 1); while (step % granule != 0) step *= 2;
    int rpc = (int)(((size_t)env_stage_kb * 1024) / rb) / step * step; if (rpc < step) rpc = step;
    if ((size_t)rpc * rb > 100 * 1024) {                         // very long rows: fewer rows per chunk than one full pass
        rpc = granule; while ((size_t)(rpc + granule) * rb <= 48 * 1024) rpc += granule;
        if ((size_t)rpc * rb > 100 * 1024) return false;
    }
    sb_params & p = pl.p;
    p.w = (const uint8_t *)a.src0; p.x = a.src1; p.y = a.dst; p.M = a.M; p.K = a.K;
    p.row_bytes = (int)rb; p.rows_per_chunk = rpc; p.nchunks = (int)((a.M + rpc - 1) / rpc);
    p.stage_bytes = (int)(((size_t)rpc * rb + 127) & ~(size_t)127);
    p.nstages = env_stages;       // 0 = automatic (below)
    p.ntasks_row = (int)(a.K / F::TASK_W);
    p.A = make_sb_act(a.K);
    p.ctl = nullptr; p.counters = nullptr; p.dbg = nullptr;      // assigned at launch (assign_sb_slot): planning has no side effects
    p.src0_static = (a.flags & GGML_B200_MM_SRC0_STATIC) ? 1 : 0;
    p.l2_prefetch_bytes = (!ind && p.src0_static && e_l2_mb > 0) ? (int64_t)std::min<size_t>((size_t)a.M * rb, (size_t)e_l2_mb << 20) : 0;
    p.world = 0; p.rank = 0; p.row_offset = 0; p.epoch = 0;
    p.ep_bias = nullptr; p.ep_y2 = nullptr; p.ep_y3 = nullptr; p.ep_res = nullptr;
    p.src1_static = (a.flags & GGML_B200_MM_SRC1_STATIC) ? 1 : 0;
    // GGML_B200_SB_STATIC: 0 = dynamic hand-out everywhere, 1 = round-robin everywhere, 2 = round-robin for dependent launches only
    static const int e_static = getenv("GGML_B200_SB_STATIC") ? atoi(getenv("GGML_B200_SB_STATIC")) : 0;
    p.static_chunks = (e_static == 1 || (e_static == 2 && !ind)) ? 1 : 0;
    p.ncols = (int32_t)a.N; p.x_stride = a.N > 1 ? (int64_t)(a.nb11 / 4) : 0;
    for (int q = 0; q < 8; ++q) { p.y_peers[q] = nullptr; p.flag_peers[q] = nullptr; }
    auto smem_of = [&]() { return p.nstages * p.stage_bytes + nc * p.A.bytes + 2 * SB_MAX_STAGES * 8 + SB_MAX_STAGES * 4 + 64; };
    const int max_res = nc > 1 ? 1 : SB_CONSUMER_WARPS == 8 ? 2 : 4;                       // register-limited residency (__launch_bounds__)
    int ctas = env_ctas < 1 ? 1 : env_ctas > max_res ? max_res : env_ctas;
    int resident = env_resident < ctas ? ctas : env_resident > max_res ? max_res : env_resident;
    if (p.nstages <= 0) {
        // deepest ring that still lets `resident` CTAs (of consecutive launches) share an SM, so that programmatic dependent
        // launch can overlap the next mat-vec's prologue and first TMA round trip with this one's tail
        p.nstages = 4;
        while (p.nstages > 2 && smem_of() * resident > 226 * 1024) p.nstages--;
    }
    if (p.nstages < 2) p.nstages = 2;
    if (p.nstages > SB_MAX_STAGES) p.nstages = SB_MAX_STAGES;
    while (smem_of() * ctas > 222 * 1024 && p.nstages > 2) p.nstages--;
    while (smem_of() * ctas > 222 * 1024 && ctas > 1) ctas--;
    if (smem_of() > 222 * 1024) return false;
    pl.smem = smem_of();
    pl.grid = sm_count() * ctas;
    if (pl.grid > p.nchunks) pl.grid = p.nchunks;
    return true;
}

// a launch takes the next of the 64 scheduling slots of this device's control block (self-resetting counters: a slot is free again
// when its launch has finished scheduling, and 64 launches never overlap on one device) and, in trace mode, the next trace record
static int assign_sb_slot(sb_params & p) {
    p.ctl = sb_counters();
    if (!p.ctl) return GGML_B200_ECUDA;
    p.counters = sb_next_slot(p.ctl);
    static const bool env_dbg = getenv("GGML_B200_SB_DEBUG") && atoi(getenv("GGML_B200_SB_DEBUG")) != 0;
    static std::atomic<unsigned> dbg_seq{0};
    p.dbg = env_dbg ? (unsigned long long *)(p.ctl + 1024) + (dbg_seq.fetch_add(1, std::memory_order_relaxed) % 32u) * 8 : nullptr;
    return GGML_B200_OK;
}

template <int T, int NW, int NC, bool TWO = false> static int launch_sb_nw(sb_plan & pl, cudaStream_t st) {
    static per_device_flag attr_set;
    if (!attr_set.test()) {
        B200_CUDA_TRY(cudaFuncSetAttribute(mmvq_sb_kernel<T, NW, NC, TWO>, cudaFuncAttributeMaxDynamicSharedMemorySize, 222 * 1024));
        attr_set.set();
    }
    static const bool use_pdl = !(getenv("GGML_B200_NO_PDL") && atoi(getenv("GGML_B200_NO_PDL")) != 0);
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(pl.grid); cfg.blockDim = dim3((NW + 1) * 32); cfg.dynamicSmemBytes = pl.smem; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = use_pdl ? 1 : 0;
    B200_CUDA_TRY(cudaLaunchKernelEx(&cfg, mmvq_sb_kernel<T, NW, NC, TWO>, pl.p));
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

template <int T> static int launch_sb(const ggml_b200_mul_mat_args & a, const ggml_b200_gather * ga, cudaStream_t st, const ggml_b200_epilogue * ep = nullptr) {
    sb_plan pl;
    if (!make_sb_plan<T>(a, pl)) { set_error("mul_mat: shape not eligible for the superblock mat-vec kernel"); return GGML_B200_EUNSUPPORTED; }
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
            if constexpr (T == T_Q4_K || T == T_Q5_K) { if (pl.two) return pl.nw == 4 ? launch_sb_nw<T, 4, 1, true>(pl, st) : launch_sb_nw<T, 8, 1, true>(pl, st); }
            return pl.nw == 4 ? launch_sb_nw<T, 4, 1>(pl, st) : launch_sb_nw<T, 8, 1>(pl, st);
        case 2:  return launch_sb_nw<T, 8, 2>(pl, st);
        case 4:  return launch_sb_nw<T, 8, 4>(pl, st);
        default: return launch_sb_nw<T, 8, 8>(pl, st);
    }
}

bool mmvq_sb_eligible(const ggml_b200_mul_mat_args & a) {
    sb_plan pl;
    switch (a.type) {
        case T_Q4_0: return make_sb_plan<T_Q4_0>(a, pl);
        case T_Q8_0: return make_sb_plan<T_Q8_0>(a, pl);
        case T_Q4_K: return make_sb_plan<T_Q4_K>(a, pl);
        case T_Q5_K: return make_sb_plan<T_Q5_K>(a, pl);
        case T_Q6_K: return make_sb_plan<T_Q6_K>(a, pl);
        // next formats (host-verified task dots and quantizer; GPU check: tests/test_gpu_next_formats.py)
        case T_Q4_1: return make_sb_plan<T_Q4_1>(a, pl);
        case T_Q5_1: return make_sb_plan<T_Q5_1>(a, pl);
        case T_Q5_0: return make_sb_plan<T_Q5_0>(a, pl);
        case T_IQ4_NL: return make_sb_plan<T_IQ4_NL>(a, pl);
        case T_IQ4_XS: return make_sb_plan<T_IQ4_XS>(a, pl);
        case T_Q2_K: return make_sb_plan<T_Q2_K>(a, pl);
        case T_Q3_K: return make_sb_plan<T_Q3_K>(a, pl);
        default: return false;
    }
}

int launch_mmvq_sb(const ggml_b200_mul_mat_args & a, cudaStream_t st, const ggml_b200_gather * ga, const ggml_b200_epilogue * ep) {
    switch (a.type) {
        case T_Q4_0: return launch_sb<T_Q4_0>(a, ga, st, ep);
        case T_Q8_0: return launch_sb<T_Q8_0>(a, ga, st, ep);
        case T_Q4_K: return launch_sb<T_Q4_K>(a, ga, st, ep);
        case T_Q5_K: return launch_sb<T_Q5_K>(a, ga, st, ep);
        case T_Q6_K: return launch_sb<T_Q6_K>(a, ga, st, ep);
        case T_Q4_1: return launch_sb<T_Q4_1>(a, ga, st, ep);
        case T_Q5_1: return launch_sb<T_Q5_1>(a, ga, st, ep);
        case T_Q5_0: return launch_sb<T_Q5_0>(a, ga, st, ep);
        case T_IQ4_NL: return launch_sb<T_IQ4_NL>(a, ga, st, ep);
        case T_IQ4_XS: return launch_sb<T_IQ4_XS>(a, ga, st, ep);
        case T_Q2_K: return launch_sb<T_Q2_K>(a, ga, st, ep);
        case T_Q3_K: return launch_sb<T_Q3_K>(a, ga, st, ep);
        default: set_error("mul_mat: unsupported weight type %d", a.type); return GGML_B200_EUNSUPPORTED;
    }
}

int debug_read_trace(unsigned long long * out) {
    unsigned int * c = sb_counters();
    if (!c) return GGML_B200_ECUDA;
    B200_CUDA_TRY(cudaDeviceSynchronize());
    B200_CUDA_TRY(cudaMemcpy(out, c + 1024, 32 * 8 * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    return GGML_B200_OK;
}

int launch_gather_wait(const uint32_t * flags, int world, uint32_t epoch, cudaStream_t st) {
    gather_wait_kernel<<<1, 32, 0, st>>>(flags, world, epoch, sb_counters());
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

} // namespace b200
