// mmq_tc2.cu — the tensor-core GEMM kernel (sm_90a): one 256 (W rows) x BN (activation rows) output tile per CTA over a K range,
// fp16 operands in shared memory, f32 accumulation in registers by warpgroup MMA (wgmma.mma_async m64n64k16).
//
// Operands: W is dequantized to fp16 in shared memory (K-major SWIZZLE_128B, the layout the wgmma descriptors read), X was converted
// to fp16 once by mmq_tc.cu with an exact power-of-two row scale (undone in the epilogue).  T_F16: the A operand already is fp16
// (dense f16 weights, or a format without an operand decoder dequantized into the workspace first) and arrives by TMA like X.
//
// Warp roles (12 warps, three warpgroups; setmaxnreg moves the producer's registers to the consumers):
//   warps 0-7   two consumer warpgroups; thread t owns W row t of the tile.  Per K-step (64 weights) each thread dequantizes its
//               row into the stage (generic-proxy stores + fence.proxy.async, then a warpgroup barrier), the warpgroup waits for the
//               stage's activation tile and issues 4 x (2 x BN/64) wgmma over its 128 rows.  The MMAs of a step run while the next
//               step is dequantized (wgmma.wait_group 1); a finished step releases its stage to the producer.
//   warp 8      TMA producer (warps 9-11 idle): raw W units of the 256 rows (packed bytes of UNIT_KSTEPS x 64 weights per row) into a 2-deep raw ring,
//               one unit ahead, and the BN x 64 activation tile of every K-step into the operand ring (for T_F16 also the A tile).
// Split-K when the tiles alone do not fill the GPU: partial producers (ks > 0) are scheduled first and hand their accumulators to
// the tile owner through the workspace (flag per tile in a self-cleaning per-device block), so the owner's wait cannot deadlock.
// The activation conversion kernel and this kernel are chained with programmatic dependent launch: barrier set-up, tensor-map
// prefetch and (static weights) the first raw W unit run while the conversion is still in flight.
//
// Replaces the reference's mul_mat_q (src/ggml-cuda/mmq.cuh:2499-2655) and its dequantize + cuBLAS route for the shapes make_tc2_plan
// accepts.
#include "b200_internal.h"
#include "b200_quants.cuh"
#include "b200_tc_dequant.cuh"
#include "b200_tc_ptx.cuh"

#include <cstdlib>
#include <mutex>

namespace b200 {

constexpr int T2_BM = 256;                    // W rows per CTA (128 per consumer warpgroup)
constexpr int T2_BK = 64;
constexpr int T2_CONSUMERS = 256, T2_THREADS = T2_CONSUMERS + 128;     // + the producer warpgroup
constexpr int T2_MAX_STAGES = 6;

// raw-unit geometry (b200_tc_dequant.cuh); T_F16: no raw ring, one K-step per "unit"
template <int T> struct tc2fmt : tcfmt<T> {};
template <> struct tc2fmt<T_F16> { static constexpr int RAW = 0, STRIDE_WORDS = 0, UNIT_WORDS = 1, UNIT_KSTEPS = 1, ODD_BACK_WORDS = 0, LOAD_BYTES = 16; };

struct tc2_params {
    float * y; float * partials; unsigned int * flags; const float * inv_scale;
    int64_t M, N;
    int32_t BN, m_tiles, n_tiles, splitk, units_total, nstages, w_static;
    // grouped mode (MUL_MAT_ID, expert-grouped): the activation rows are SORTED by expert (position -> (token, slot) pair in `perm`), n-tiles are
    // enumerated per expert (tile_base: prefix of tiles per expert, off: prefix of positions per expert, both n_expert + 1 long, device-resident:
    // no host synchronisation); W is the [n_expert x M] row stack; y rows are scattered back through perm
    const int32_t * g_off; const int32_t * g_tile_base; const int32_t * g_perm;
    int32_t n_expert;
};

// one K-step of A: the thread's 64 weights of its row, converted into the swizzled stage row (KS: K-step within the unit)
template <int T>
__device__ __forceinline__ void tc2_dequant(int ks, const uint32_t (&u)[tc2fmt<T>::UNIT_WORDS], uint8_t * dst, uint32_t sw) {
    if constexpr (T != T_F16) {
        if (ks == 0) dq64<T, 0>(u, dst, sw);
        else if (ks == 1) dq64<T, 1>(u, dst, sw);
        if constexpr (tc2fmt<T>::UNIT_KSTEPS == 4) {
            if (ks == 2) dq64<T, 2>(u, dst, sw);
            else if (ks == 3) dq64<T, 3>(u, dst, sw);
        }
    }
}

template <int T, bool GROUPED = false>
__global__ void __launch_bounds__(T2_THREADS, 1)
mmq_tc2_kernel(const __grid_constant__ CUtensorMap map_w, const __grid_constant__ CUtensorMap map_x, const tc2_params p) {
    constexpr int RAW = tc2fmt<T>::RAW, UK = tc2fmt<T>::UNIT_KSTEPS;
    constexpr bool DENSE = T == T_F16;                            // fp16 A tiles by TMA: no raw ring, no dequantizers
    extern __shared__ uint8_t smem_raw[];
    // [ring: nstages x (A: 256 x 128 B | B: BN x 128 B)][raw: 2 x 256 x RAW][barriers][inv_scale of the tile's columns]
    uint8_t * smem = (uint8_t *)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);      // SWIZZLE_128B tiles: 1024-byte aligned
    constexpr int a_bytes = T2_BM * T2_BK * 2;
    const int b_bytes = p.BN * T2_BK * 2, stage_bytes = a_bytes + b_bytes;
    uint8_t * ring = smem;
    uint8_t * raw  = ring + p.nstages * stage_bytes;
    uint64_t * bars = (uint64_t *)(raw + 2 * T2_BM * RAW);
    uint64_t * full = bars, * empty = bars + T2_MAX_STAGES, * raw_full = bars + 2 * T2_MAX_STAGES, * raw_empty = raw_full + 2;
    float * s_inv = (float *)(raw_empty + 2);

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    tc_pdl_launch_dependents();
    // work item: partial producers (ks > 0) first, tile owners (ks == 0) last
    const int tiles = p.m_tiles * p.n_tiles;
    const int ks = p.splitk - 1 - (int)blockIdx.x / tiles;
    const int tile = (int)blockIdx.x % tiles, tm = tile % p.m_tiles, tn = tile / p.m_tiles;
    const int ubeg = (int)((int64_t)p.units_total * ks / p.splitk), uend = (int)((int64_t)p.units_total * (ks + 1) / p.splitk);
    const int nunits = uend - ubeg;
    // grouped mode: n-tile tn of the enumeration belongs to expert gx, covers sorted positions [gn0, gn0 + gcols); tiles past the last one
    // (the grid is sized for the worst case) retire at once
    int gx = 0, gn0 = 0, gcols = 0;
    if constexpr (GROUPED) {
        if (tn >= p.g_tile_base[p.n_expert]) return;
        int lo = 0, hi = p.n_expert;                              // largest x with tile_base[x] <= tn
        while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (p.g_tile_base[mid] <= tn) lo = mid; else hi = mid; }
        gx = lo;
        gn0 = p.g_off[gx] + (tn - p.g_tile_base[gx]) * p.BN;
        gcols = min(p.BN, p.g_off[gx + 1] - gn0);
    }
    const int64_t row_base = (int64_t)tm * T2_BM;                 // first W row of the tile (within the expert's matrix)
    const int64_t w_row0 = GROUPED ? (int64_t)gx * p.M + row_base : row_base;       // row in the [n_expert x M] stack
    const int x_row0 = GROUPED ? gn0 : tn * p.BN;

    if (tid == 0) {
        for (int s = 0; s < p.nstages; ++s) { tc_mbar_init(&full[s], 1); tc_mbar_init(&empty[s], 2); }     // producer's expect_tx; one release per warpgroup
        for (int s = 0; s < 2; ++s) { tc_mbar_init(&raw_full[s], 1); tc_mbar_init(&raw_empty[s], T2_CONSUMERS / 32); }
        tc_fence_init();
        tc_prefetch_map(&map_w); tc_prefetch_map(&map_x);
    }
    __syncthreads();

    if (warp >= T2_CONSUMERS / 32) {
        // ===================== TMA producer
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
        if (warp == T2_CONSUMERS / 32 && lane == 0) {
            auto issue_raw = [&](int u) {
                const int rs = u & 1;
                tc_expect_tx(&raw_full[rs], T2_BM * RAW);
                int coord;                                        // first 4-byte word of the box: 16-byte aligned start at or below the unit
                if constexpr (tc2fmt<T>::LOAD_BYTES == 2) coord = (((ubeg + u) * tc2fmt<T>::UNIT_BYTES) & ~15) >> 2;   // unaligned units: lead bytes in front of the payload
                else                        coord = (ubeg + u) * tc2fmt<T>::STRIDE_WORDS - ((ubeg + u) & 1) * tc2fmt<T>::ODD_BACK_WORDS;
                tc_tma_2d(raw + rs * T2_BM * RAW, &map_w, coord, (int)w_row0, &raw_full[rs]);
            };
            if (!DENSE && p.w_static) issue_raw(0);               // static weights: the first unit streams while the conversion kernel runs
            tc_pdl_wait();                                        // the fp16 activations (and non-static W) are written by the preceding kernels
            if (!DENSE && !p.w_static) issue_raw(0);
            for (int u = 0; u < nunits; ++u) {
                if (!DENSE && u + 1 < nunits) {
                    if (u + 1 >= 2) tc_wait(&raw_empty[(u + 1) & 1], (uint32_t)(((u + 1) >> 1) - 1) & 1u);
                    issue_raw(u + 1);
                }
                for (int q = 0; q < UK; ++q) {
                    const int step = UK * u + q, s = step % p.nstages;
                    if (step >= p.nstages) tc_wait(&empty[s], (uint32_t)((step / p.nstages) - 1) & 1u);
                    const int kc = ((ubeg + u) * UK + q) * T2_BK;
                    uint8_t * st = ring + s * stage_bytes;
                    if constexpr (DENSE) {
                        tc_expect_tx(&full[s], (uint32_t)(a_bytes + b_bytes));
                        tc_tma_2d(st, &map_w, kc, (int)w_row0, &full[s]);
                    } else {
                        tc_expect_tx(&full[s], (uint32_t)b_bytes);
                    }
                    tc_tma_2d(st + a_bytes, &map_x, kc, x_row0, &full[s]);
                }
            }
        }
        return;
    }

    // ===================== consumers: thread tid owns W row tid of the tile; warpgroup wg multiplies rows 128 wg .. 128 wg + 127
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");        // 128 accumulators + a raw unit + addressing per thread
    const int wg = tid >> 7, row = tid;
    const uint32_t sw = (uint32_t)(row & 7);
    const int a_row_off = (row >> 3) * 1024 + (row & 7) * 128;
    const bool two_n = p.BN == 128;
    float acc[2][2][32];
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
        for (int nj = 0; nj < 2; ++nj)
#pragma unroll
            for (int i = 0; i < 32; ++i) acc[mi][nj][i] = 0.0f;
    uint32_t ub[tc2fmt<T>::UNIT_WORDS];
    for (int u = 0; u < nunits; ++u) {
        if constexpr (!DENSE) {
            const int rs = u & 1;
            tc_wait(&raw_full[rs], (uint32_t)(u >> 1) & 1u);
            int lead;                                             // bytes between the box start and the unit's first byte
            if constexpr (tc2fmt<T>::LOAD_BYTES == 2) lead = ((ubeg + u) * tc2fmt<T>::UNIT_BYTES) & 15;
            else                        lead = ((ubeg + u) & 1) * (4 * tc2fmt<T>::ODD_BACK_WORDS);
            tc_load_unit<T>(raw + rs * T2_BM * RAW + row * RAW + lead, ub);
            // the unit is in registers: the buffer can be refilled.  The refill is a TMA write (async proxy) after these generic-proxy reads,
            // so every reader fences before its warp releases the buffer; without the fence, Q8_0 tiles (the fastest raw-ring turnover) read
            // units that were already being overwritten whenever the release came from the last busy warp.
            tc_fence_async_smem();
            __syncwarp();
            if (lane == 0) tc_arrive(&raw_empty[rs]);
        }
#pragma unroll
        for (int q = 0; q < UK; ++q) {
            const int step = UK * u + q, s = step % p.nstages;
            uint8_t * st = ring + s * stage_bytes;
            if constexpr (!DENSE) {
                // this warpgroup's rows of the stage were last read by its own MMAs of step - nstages <= step - 2: complete (wait_group 1 below)
                if (row < p.M - row_base) tc2_dequant<T>(q, ub, st + a_row_off, sw);     // rows past M: zero-filled box, results never stored
                tc_fence_async_smem();
                asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");
            }
            tc_wait(&full[s], (uint32_t)(step / p.nstages) & 1u);
            wg_fence();
            const uint64_t ad = tc_smem_desc(tc_smem(st + wg * (128 * 128)));
            const uint64_t bd = tc_smem_desc(tc_smem(st + a_bytes));
#pragma unroll
            for (int k = 0; k < T2_BK / 16; ++k) {               // +32 bytes per K = 16; +8 KB per 64 rows (A) / 64 columns (B)
#pragma unroll
                for (int mi = 0; mi < 2; ++mi) {
                    wg_mma_m64n64k16(acc[mi][0], ad + (uint64_t)(2 * k + mi * 512), bd + (uint64_t)(2 * k));
                    if (two_n) wg_mma_m64n64k16(acc[mi][1], ad + (uint64_t)(2 * k + mi * 512), bd + (uint64_t)(2 * k + 512));
                }
            }
            wg_commit();
            wg_wait<1>();                                         // the MMAs of step - 1 are complete: release its stage
            if (step > 0 && (tid & 127) == 0) tc_arrive(&empty[(step - 1) % p.nstages]);
        }
    }
    wg_wait<0>();
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
        for (int nj = 0; nj < 2; ++nj)
#pragma unroll
            for (int i = 0; i < 32; ++i) wg_fence_operand(acc[mi][nj][i]);

    // ===================== epilogue.  wgmma m64nN fragment: warp w of the warpgroup holds rows 16 w + lane / 4 (+ 8), register 4 j + 2 h + e
    // is row + 8 h, column 8 j + 2 (lane % 4) + e
    tc_pdl_wait();                                                // inv_scale comes from the conversion kernel
    const int r0 = wg * 128 + ((tid & 127) >> 5) * 16 + (lane >> 2), c0 = 2 * (lane & 3);
    const int nregs = (two_n ? 2 : 1) * 64;                       // accumulator registers per thread (partials layout: [register][thread])
    auto consumers_sync = [] { asm volatile("bar.sync 3, %0;" ::"n"(T2_CONSUMERS) : "memory"); };
    float * part = p.partials ? p.partials + (size_t)tile * (p.splitk - 1) * (size_t)(p.BN * T2_BM) : nullptr;
    if (ks > 0) {
        float * dst = part + (size_t)(ks - 1) * (p.BN * T2_BM);
#pragma unroll
        for (int mi = 0; mi < 2; ++mi)
#pragma unroll
            for (int nj = 0; nj < 2; ++nj)
                if (nj == 0 || two_n) {
#pragma unroll
                    for (int i = 0; i < 32; ++i) __stcg(&dst[(size_t)(mi * (nregs / 2) + nj * 32 + i) * T2_CONSUMERS + tid], acc[mi][nj][i]);
                }
        __threadfence();
        consumers_sync();
        if (tid == 0) atomicAdd(&p.flags[tile], 1u);
        return;
    }
    // inv_scale of the tile's columns -> shared memory
    for (int c = tid; c < p.BN; c += T2_CONSUMERS) {
        const int64_t n = GROUPED ? (int64_t)gn0 + c : (int64_t)tn * p.BN + c;
        s_inv[c] = (GROUPED ? c < gcols : n < p.N) ? __ldcg(p.inv_scale + n) : 0.0f;
    }
    if (p.splitk > 1 && tid == 0) { while (atomicAdd(&p.flags[tile], 0u) < (unsigned)(p.splitk - 1)) __nanosleep(64); __threadfence(); }
    consumers_sync();
    for (int j = 1; j < p.splitk; ++j) {
        const float * src = part + (size_t)(j - 1) * (p.BN * T2_BM);
#pragma unroll
        for (int mi = 0; mi < 2; ++mi)
#pragma unroll
            for (int nj = 0; nj < 2; ++nj)
                if (nj == 0 || two_n) {
#pragma unroll
                    for (int i = 0; i < 32; ++i) acc[mi][nj][i] += __ldcg(&src[(size_t)(mi * (nregs / 2) + nj * 32 + i) * T2_CONSUMERS + tid]);
                }
    }
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
        for (int nj = 0; nj < 2; ++nj) {
            if (nj == 1 && !two_n) continue;
#pragma unroll
            for (int i = 0; i < 32; ++i) {
                const int rl = r0 + mi * 64 + ((i >> 1) & 1) * 8, c = nj * 64 + (i >> 2) * 8 + c0 + (i & 1);
                const int64_t m = row_base + rl;
                if (m >= p.M) continue;
                const float v = acc[mi][nj][i] * s_inv[c];
                if constexpr (GROUPED) {
                    if (c < gcols) p.y[(size_t)__ldg(p.g_perm + gn0 + c) * p.M + m] = v;
                } else {
                    const int64_t n = (int64_t)tn * p.BN + c;
                    if (n < p.N) p.y[(size_t)n * p.M + m] = v;
                }
            }
        }
    if (p.splitk > 1) {
        consumers_sync();
        if (tid == 0) p.flags[tile] = 0;                          // leave the flag clean for the next launch that gets this slot
    }
}

// ----------------------------------------------------------------------------- split-K flags: persistent, zero-initialised, self-cleaning
constexpr int T2_FLAG_SLOTS = 64, T2_FLAGS_PER_SLOT = 256;
static unsigned int * tc_flag_block() {
    static unsigned int * ptr[64] = { nullptr };
    static std::mutex mu;
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) { set_error("tc flags: cudaGetDevice failed"); return nullptr; }
    std::lock_guard<std::mutex> lock(mu);
    if (!ptr[dev]) {
        unsigned int * p = nullptr;
        const size_t bytes = (size_t)T2_FLAG_SLOTS * T2_FLAGS_PER_SLOT * sizeof(unsigned int);
        cudaError_t e = cudaMalloc(&p, bytes);
        if (e == cudaSuccess) e = cudaMemset(p, 0, bytes);
        if (e == cudaSuccess) e = cudaDeviceSynchronize();
        if (e != cudaSuccess) { set_error("tc flags: %s", cudaGetErrorString(e)); cudaGetLastError(); if (p) cudaFree(p); return nullptr; }
        ptr[dev] = p;
    }
    return ptr[dev];
}
int tc_prepare_device() { return tc_flag_block() ? GGML_B200_OK : GGML_B200_ECUDA; }
unsigned int * tc_flag_slot() {
    unsigned int * b = tc_flag_block();
    if (!b) return nullptr;
    static std::atomic<unsigned> seq{0};
    return b + (size_t)(seq.fetch_add(1, std::memory_order_relaxed) % T2_FLAG_SLOTS) * T2_FLAGS_PER_SLOT;
}

// this kernel records no per-CTA stamp trace
int tc2_trace_read(unsigned long long * host_dst, int max_ctas) { (void)host_dst; (void)max_ctas; return 0; }

// ----------------------------------------------------------------------------- host side
struct tc2_plan {
    int BN, m_tiles, n_tiles, splitk, chunks, nstages, smem, grid;
    size_t xb_bytes, partial_bytes, scale_bytes;
};

static int tc2_raw_bytes(int type) {                                // tcfmt<T>::RAW
    switch (type) {
        case T_F16: return 0;
        case T_Q5_K: case T_Q5_0: return 176;
        case T_Q6_K: return 224;
        case T_Q4_1: return 160;
        case T_Q5_1: return 192;
        case T_Q2_K: return 96;
        case T_Q3_K: return 128;
        default: return 144;                                         // Q4_0, Q8_0 (half units), Q4_K, IQ4_NL, IQ4_XS
    }
}
static int tc2_unit_ksteps(int type) { return type == T_F16 ? 1 : type == T_Q8_0 ? 2 : 4; }     // tc2fmt<T>::UNIT_KSTEPS

// shared memory: the raw ring (2 units of 256 rows) first, then as many operand stages (>= 2: a stage is rewritten two steps after
// its MMAs were issued, and wait_group 1 has completed them by then) as fit the 227 KB an H100 block may use
static bool tc2_smem_plan(int BN, int raw, int & nstages, int & smem) {
    static const int env_stages = getenv("GGML_B200_TC2_STAGES") ? atoi(getenv("GGML_B200_TC2_STAGES")) : 0;
    const int stage = T2_BM * T2_BK * 2 + BN * T2_BK * 2;
    const int tail = 2 * T2_BM * raw + (2 * T2_MAX_STAGES + 4) * 8 + BN * 4 + 1024;       // + 1024: alignment of the ring
    int ns = (227 * 1024 - tail) / stage;
    if (ns > T2_MAX_STAGES) ns = T2_MAX_STAGES;
    if (env_stages >= 2 && env_stages < ns) ns = env_stages;
    if (ns < 2) return false;
    nstages = ns; smem = ns * stage + tail;
    return true;
}

static bool make_tc2_plan(const ggml_b200_mul_mat_args & a, tc2_plan & pl) {
    const bool dense = a.type == T_F16;                            // fp16 A tiles (launch_mmq_dense / launch_mmq_f16w)
    switch (a.type) {
        case T_Q4_0: case T_Q8_0: case T_Q4_K: case T_Q5_K: case T_Q6_K: case T_Q4_1: case T_Q5_0: case T_Q5_1: case T_IQ4_NL: case T_IQ4_XS: case T_Q2_K: case T_Q3_K: break;
        case T_F16: break;
        default: return false;
    }
    if (a.ne02 != 1 || a.ne03 != 1 || a.ne12 != 1 || a.ne13 != 1) return false;
    // n >= 9: every batch the mat-vec kernels do not take (the reference's mul_mat_q threshold, ggml-cuda.cu:1852-1875); also 5 <= n <= 8
    // when the mat-vec kernel cannot hold that many activation records next to its weight stages (very long rows: api.cu decides);
    // columns beyond n in the 64-wide minimum tile are zero-filled by the TMA box and never stored
    if (a.N < (dense ? 9 : 5) || a.M < 1 || a.K % 256 != 0 || a.K < 256) return false;
    const size_t rb = dense ? (size_t)a.K * 2 : row_bytes(a.type, a.K);
    if ((dense ? (a.nb01 < rb || (a.nb01 % 16) != 0) : a.nb01 != rb) || (rb % 16) != 0 || ((uintptr_t)a.src0 & 15) != 0 || ((uintptr_t)a.src1 & 3) != 0 || (a.nb11 & 3) != 0) return false;
    if (a.M >= (1ll << 31) || a.N >= (1ll << 31) || rb >= (1ull << 31)) return false;
    if (!tc_get_encode()) return false;
    static const int env_bn = getenv("GGML_B200_TC2_BN") ? atoi(getenv("GGML_B200_TC2_BN")) : 0;
    int BN = a.N > 64 ? 128 : 64;                                  // 2 x 128 rows x 128 columns of f32 accumulators: 128 registers per thread
    if (env_bn == 64 || env_bn == 128) BN = env_bn;
    pl.BN = BN;
    pl.n_tiles = (int)((a.N + BN - 1) / BN);
    pl.m_tiles = (int)((a.M + T2_BM - 1) / T2_BM);
    pl.chunks = (int)(a.K / (T2_BK * tc2_unit_ksteps(a.type)));  // units along K
    const int tiles = pl.m_tiles * pl.n_tiles;
    int splitk = sm_count() / tiles; if (splitk < 1) splitk = 1; if (splitk > 8) splitk = 8; if (splitk > pl.chunks) splitk = pl.chunks;
    static const int env_splitk = getenv("GGML_B200_TC_SPLITK") ? atoi(getenv("GGML_B200_TC_SPLITK")) : 0;
    if (env_splitk > 0 && env_splitk <= pl.chunks) splitk = env_splitk;
    if (splitk > 1 && tiles > T2_FLAGS_PER_SLOT) splitk = 1;
    pl.splitk = splitk;
    if (!tc2_smem_plan(BN, tc2_raw_bytes(a.type), pl.nstages, pl.smem)) return false;
    pl.grid = tiles * splitk;
    pl.xb_bytes = ((size_t)a.N * a.K * 2 + 255) & ~(size_t)255;
    pl.partial_bytes = splitk > 1 ? (size_t)tiles * (splitk - 1) * BN * T2_BM * 4 : 0;
    pl.scale_bytes = ((size_t)a.N * 4 + 255) & ~(size_t)255;
    return true;
}

bool mmq_tc2_eligible(const ggml_b200_mul_mat_args & a) { tc2_plan pl; return make_tc2_plan(a, pl); }
size_t mmq_tc2_workspace(const ggml_b200_mul_mat_args & a) {
    tc2_plan pl;
    if (!make_tc2_plan(a, pl)) return 0;
    return pl.xb_bytes + pl.partial_bytes + pl.scale_bytes + 1024;
}

template <int T> static int launch_tc2(const ggml_b200_mul_mat_args & a, const tc2_plan & pl, cudaStream_t st) {
    const size_t need = pl.xb_bytes + pl.partial_bytes + pl.scale_bytes + 1024;
    if (!a.workspace || a.workspace_size < need) { set_error("mul_mat: workspace %zu < %zu", a.workspace_size, need); return GGML_B200_EWORKSPACE; }
    uint8_t * ws = (uint8_t *)(((uintptr_t)a.workspace + 255) & ~(uintptr_t)255);
    __half * xb = (__half *)ws;
    float * partials = pl.partial_bytes ? (float *)(ws + pl.xb_bytes) : nullptr;
    float * inv_scale = (float *)(ws + pl.xb_bytes + pl.partial_bytes);
    unsigned int * flags = tc_flag_slot();
    if (!flags) return GGML_B200_ECUDA;
    static const bool use_pdl = !(getenv("GGML_B200_NO_PDL") && atoi(getenv("GGML_B200_NO_PDL")) != 0);

    { const int rc = tc_launch_x_to_f16(a.src1, a.nb11, xb, inv_scale, a.K, a.N, st, use_pdl); if (rc != GGML_B200_OK) return rc; }
    const size_t rb = T == T_F16 ? (size_t)a.K * 2 : row_bytes(a.type, a.K);
    alignas(64) CUtensorMap map_w, map_x;
    if constexpr (T == T_F16) {
        // fp16 weights [M][K]: 256 x 64 tiles straight into the swizzled operand ring
        const cuuint64_t dims[2] = { (cuuint64_t)a.K, (cuuint64_t)a.M };
        const cuuint64_t strides[1] = { (cuuint64_t)a.nb01 };
        const cuuint32_t box[2] = { (cuuint32_t)T2_BK, (cuuint32_t)T2_BM };
        const cuuint32_t es[2] = { 1, 1 };
        CUresult r = tc_get_encode()(&map_w, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, (void *)a.src0, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(W fp16) failed: %d", (int)r); return GGML_B200_ECUDA; }
    } else {
        const cuuint64_t dims[2] = { (cuuint64_t)(rb / 4), (cuuint64_t)a.M };
        const cuuint64_t strides[1] = { (cuuint64_t)rb };
        const cuuint32_t box[2] = { (cuuint32_t)(tc2fmt<T>::RAW / 4), (cuuint32_t)T2_BM };
        const cuuint32_t es[2] = { 1, 1 };
        CUresult r = tc_get_encode()(&map_w, CU_TENSOR_MAP_DATA_TYPE_UINT32, 2, (void *)a.src0, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                     CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(W) failed: %d", (int)r); return GGML_B200_ECUDA; }
    }
    {
        const cuuint64_t dims[2] = { (cuuint64_t)a.K, (cuuint64_t)a.N };
        const cuuint64_t strides[1] = { (cuuint64_t)a.K * 2 };
        const cuuint32_t box[2] = { (cuuint32_t)T2_BK, (cuuint32_t)pl.BN };
        const cuuint32_t es[2] = { 1, 1 };
        CUresult r = tc_get_encode()(&map_x, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, (void *)xb, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(X) failed: %d", (int)r); return GGML_B200_ECUDA; }
    }
    tc2_params p{};
    p.y = a.dst; p.partials = partials; p.flags = flags; p.inv_scale = inv_scale; p.M = a.M; p.N = a.N;
    p.BN = pl.BN; p.m_tiles = pl.m_tiles; p.n_tiles = pl.n_tiles; p.splitk = pl.splitk; p.units_total = pl.chunks; p.nstages = pl.nstages;
    p.w_static = (a.flags & GGML_B200_MM_SRC0_STATIC) ? 1 : 0;
    static per_device_flag attr_set;
    if (!attr_set.test()) { B200_CUDA_TRY(cudaFuncSetAttribute(mmq_tc2_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024)); attr_set.set(); }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)pl.grid); cfg.blockDim = dim3(T2_THREADS); cfg.dynamicSmemBytes = (size_t)pl.smem; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = use_pdl ? 1 : 0;
    B200_CUDA_TRY(cudaLaunchKernelEx(&cfg, mmq_tc2_kernel<T>, map_w, map_x, p));
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

int launch_mmq_tc2(const ggml_b200_mul_mat_args & a, cudaStream_t st) {
    tc2_plan pl;
    if (!make_tc2_plan(a, pl)) { set_error("mul_mat: shape not eligible for the tensor-core kernel"); return GGML_B200_EUNSUPPORTED; }
    switch (a.type) {
        case T_Q4_0:   return launch_tc2<T_Q4_0>(a, pl, st);
        case T_Q8_0:   return launch_tc2<T_Q8_0>(a, pl, st);
        case T_Q4_K:   return launch_tc2<T_Q4_K>(a, pl, st);
        case T_Q5_K:   return launch_tc2<T_Q5_K>(a, pl, st);
        case T_Q6_K:   return launch_tc2<T_Q6_K>(a, pl, st);
        case T_Q4_1:   return launch_tc2<T_Q4_1>(a, pl, st);
        case T_Q5_0:   return launch_tc2<T_Q5_0>(a, pl, st);
        case T_Q5_1:   return launch_tc2<T_Q5_1>(a, pl, st);
        case T_IQ4_NL: return launch_tc2<T_IQ4_NL>(a, pl, st);
        case T_IQ4_XS: return launch_tc2<T_IQ4_XS>(a, pl, st);
        case T_Q2_K:   return launch_tc2<T_Q2_K>(a, pl, st);
        case T_Q3_K:   return launch_tc2<T_Q3_K>(a, pl, st);
        default: set_error("mul_mat: unsupported weight type %d for the tensor-core kernel", a.type); return GGML_B200_EUNSUPPORTED;
    }
}

// ----------------------------------------------------------------------------- formats without an operand decoder (grid i-quants, ternary): n >= 9
// W is dequantized to fp16 into the workspace by the bit-exact conversion kernel (dequant.cu) and the same GEMM runs with plain fp16 A tiles.
// One extra pass over W (2 bytes per weight written, then read N / BN times), against the generic kernel's one warp per output element.
// Replaces the reference's dequantize + cuBLAS route
// (src/ggml-cuda/ggml-cuda.cu:1158-1300) for these formats.
static bool dense_source_type(int t) {
    switch (t) {
        case T_IQ2_XXS: case T_IQ2_XS: case T_IQ2_S: case T_IQ3_XXS: case T_IQ3_S: case T_IQ1_S: case T_IQ1_M: case T_TQ1_0: case T_TQ2_0: return true;
        default: return false;
    }
}
static bool make_dense_args(const ggml_b200_mul_mat_args & a, ggml_b200_mul_mat_args & b, size_t & wbytes) {
    static const bool env_off = getenv("GGML_B200_TC_DENSE") && atoi(getenv("GGML_B200_TC_DENSE")) == 0;
    if (env_off || !dense_source_type(a.type) || a.N < 9 || a.K % 256 != 0) return false;
    if (a.ne02 != 1 || a.ne03 != 1 || a.ne12 != 1 || a.ne13 != 1 || a.nb01 != row_bytes(a.type, a.K)) return false;
    wbytes = ((size_t)a.M * (size_t)a.K * 2 + 255) & ~(size_t)255;
    b = a;
    b.type = T_F16; b.nb01 = (size_t)a.K * 2; b.nb02 = b.nb01 * (size_t)a.M; b.nb03 = b.nb02;
    b.src0 = (const void *)(uintptr_t)256;                           // placeholder with the alignment of the real buffer (plan only looks at alignment)
    b.flags &= ~(uint32_t)GGML_B200_MM_SRC0_STATIC;                   // the fp16 copy is produced by the kernel in front of the GEMM
    return true;
}
bool mmq_dense_eligible(const ggml_b200_mul_mat_args & a) {
    ggml_b200_mul_mat_args b; size_t wbytes; tc2_plan pl;
    return make_dense_args(a, b, wbytes) && make_tc2_plan(b, pl);
}
size_t mmq_dense_workspace(const ggml_b200_mul_mat_args & a) {
    ggml_b200_mul_mat_args b; size_t wbytes; tc2_plan pl;
    if (!make_dense_args(a, b, wbytes) || !make_tc2_plan(b, pl)) return 0;
    return wbytes + 256 + pl.xb_bytes + pl.partial_bytes + pl.scale_bytes + 1024;
}
int launch_mmq_dense(const ggml_b200_mul_mat_args & a, cudaStream_t st) {
    ggml_b200_mul_mat_args b; size_t wbytes; tc2_plan pl;
    if (!make_dense_args(a, b, wbytes) || !make_tc2_plan(b, pl)) { set_error("mul_mat: shape not eligible for the dequantize + fp16 tensor-core path"); return GGML_B200_EUNSUPPORTED; }
    const size_t need = wbytes + 256 + pl.xb_bytes + pl.partial_bytes + pl.scale_bytes + 1024;
    if (!a.workspace || a.workspace_size < need) { set_error("mul_mat: workspace %zu < %zu", a.workspace_size, need); return GGML_B200_EWORKSPACE; }
    uint8_t * ws = (uint8_t *)(((uintptr_t)a.workspace + 255) & ~(uintptr_t)255);
    const int rc = ggml_b200_dequantize(a.type, a.src0, ws, T_F16, a.M * a.K, (void *)st);
    if (rc != GGML_B200_OK) return rc;
    b.src0 = ws;
    b.workspace = ws + wbytes;
    b.workspace_size = a.workspace_size - (size_t)((ws + wbytes) - (uint8_t *)a.workspace);
    return launch_tc2<T_F16>(b, pl, st);
}

// dense fp16 weights x f32 activations, n >= 9 (the reference: cuBLAS, ggml-cuda.cu:1158-1300): straight onto the fp16 A path
static bool make_f16w_args(const void * w, size_t nb01, const float * x, size_t nb11, float * y, int64_t M, int64_t N, int64_t K, uint32_t flags, ggml_b200_mul_mat_args & b) {
    b = ggml_b200_mul_mat_args{};
    b.type = T_F16; b.M = M; b.N = N; b.K = K; b.ne02 = b.ne03 = b.ne12 = b.ne13 = 1;
    b.nb01 = nb01; b.nb02 = nb01 * (size_t)M; b.nb03 = b.nb02; b.nb11 = nb11; b.nb12 = nb11 * (size_t)N; b.nb13 = b.nb12;
    b.src0 = w; b.src1 = x; b.dst = y; b.flags = flags;
    return w && x && y && M > 0 && N > 0 && K > 0;
}
size_t mmq_f16w_workspace(int64_t M, int64_t N, int64_t K) {
    ggml_b200_mul_mat_args b; tc2_plan pl;
    make_f16w_args((const void *)(uintptr_t)256, (size_t)K * 2, (const float *)(uintptr_t)256, (size_t)K * 4, (float *)(uintptr_t)256, M, N, K, 0, b);
    if (!make_tc2_plan(b, pl)) return 0;
    return pl.xb_bytes + pl.partial_bytes + pl.scale_bytes + 1024;
}
int launch_mmq_f16w(const void * w, size_t nb01, const float * x, size_t nb11, float * y, int64_t M, int64_t N, int64_t K, void * ws, size_t ws_size, uint32_t flags, cudaStream_t st) {
    ggml_b200_mul_mat_args b; tc2_plan pl;
    if (!make_f16w_args(w, nb01, x, nb11, y, M, N, K, flags, b) || !make_tc2_plan(b, pl)) { set_error("mul_mat_f16: shape not eligible for the tensor-core path"); return GGML_B200_EUNSUPPORTED; }
    b.workspace = ws; b.workspace_size = ws_size;
    return launch_tc2<T_F16>(b, pl, st);
}

// ----------------------------------------------------------------------------- MUL_MAT_ID, expert-grouped (batched tokens)
// The reference groups the rows per expert on the HOST (ids copied back, stream synchronised: src/ggml-cuda/ggml-cuda.cu:1975-2090; the CPU
// backend builds matrix_rows the same way, src/ggml-cpu/ggml-cpu.c:7679-7694).  Here the grouping stays on the device: one small kernel counts
// the (token, slot) pairs per expert, scans, and scatters the pair indices into a position list sorted by expert; the activation conversion
// writes row `position`; the GEMM runs over a worst-case tile grid whose tiles look their expert / position range up in the device
// tables, streaming every expert's weights once per 256-row tile instead of once per pair.  No host synchronisation anywhere.
constexpr int MMID_MAX_EXPERTS = 1024;
__global__ void __launch_bounds__(1024) mmid_group_kernel(const uint8_t * ids, size_t ids_nb1, int n_tok, int n_used, int n_expert, int BN,
                                                          int32_t * off, int32_t * tile_base, int32_t * perm) {
    __shared__ int hist[MMID_MAX_EXPERTS], cursor[MMID_MAX_EXPERTS];
    const int n_pairs = n_tok * n_used;
    for (int x = threadIdx.x; x < n_expert; x += blockDim.x) { hist[x] = 0; cursor[x] = 0; }
    __syncthreads();
    for (int pr = threadIdx.x; pr < n_pairs; pr += blockDim.x) {
        const int x = *(const int32_t *)(ids + (size_t)(pr / n_used) * ids_nb1 + (size_t)(pr % n_used) * 4);
        if (x >= 0 && x < n_expert) atomicAdd(&hist[x], 1);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int o = 0, tb = 0;
        for (int x = 0; x < n_expert; ++x) { off[x] = o; tile_base[x] = tb; o += hist[x]; tb += (hist[x] + BN - 1) / BN; }
        off[n_expert] = o; tile_base[n_expert] = tb;
    }
    __syncthreads();
    for (int pr = threadIdx.x; pr < n_pairs; pr += blockDim.x) {
        const int x = *(const int32_t *)(ids + (size_t)(pr / n_used) * ids_nb1 + (size_t)(pr % n_used) * 4);
        if (x >= 0 && x < n_expert) perm[off[x] + atomicAdd(&cursor[x], 1)] = pr;
    }
}

// activation row of sorted position `pos` = b[t][e % nb1cols] of pair perm[pos] -> fp16 row pos with its exact power-of-two scale
__global__ void __launch_bounds__(256) mmid_x_to_f16_kernel(const uint8_t * __restrict__ b, size_t nb11, size_t nb12, int n_used, int nb1cols, const int32_t * __restrict__ off,
                                                            const int32_t * __restrict__ perm, int n_expert, __half * __restrict__ xh, float * __restrict__ inv_scale, int64_t K) {
    const int pos = blockIdx.x;
    if (pos >= off[n_expert]) return;                            // positions past the valid pairs (invalid expert ids) stay unused
    const int pr = perm[pos], t = pr / n_used, e = pr % n_used;
    const float * xr = (const float *)(b + (size_t)t * nb12 + (size_t)(e % nb1cols) * nb11);
    __shared__ float s_max[8];
    float amax = 0.0f;
    for (int64_t k = (int64_t)threadIdx.x * 8; k < K; k += 256 * 8) {
        const float4 a = load_f4(xr + k), c = load_f4(xr + k + 4);
        amax = fmaxf(amax, fmaxf(fmaxf(fmaxf(fabsf(a.x), fabsf(a.y)), fmaxf(fabsf(a.z), fabsf(a.w))), fmaxf(fmaxf(fabsf(c.x), fabsf(c.y)), fmaxf(fabsf(c.z), fabsf(c.w)))));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    if ((threadIdx.x & 31) == 0) s_max[threadIdx.x >> 5] = amax;
    __syncthreads();
    amax = s_max[0];
#pragma unroll
    for (int i = 1; i < 8; ++i) amax = fmaxf(amax, s_max[i]);
    int ex = 0;
    if (amax > 0.0f && amax <= 3.0e38f) ex = max(-100, min(100, (int)((__float_as_uint(amax) >> 23) & 0xFF) - 127 - 13));
    const float sc = __uint_as_float((uint32_t)(127 - ex) << 23);
    if (threadIdx.x == 0) inv_scale[pos] = __uint_as_float((uint32_t)(127 + ex) << 23);
    for (int64_t k = (int64_t)threadIdx.x * 8; k < K; k += 256 * 8) {
        const float4 a = load_f4(xr + k), c = load_f4(xr + k + 4);
        __half2 h0 = __floats2half2_rn(a.x * sc, a.y * sc), h1 = __floats2half2_rn(a.z * sc, a.w * sc);
        __half2 h2 = __floats2half2_rn(c.x * sc, c.y * sc), h3 = __floats2half2_rn(c.z * sc, c.w * sc);
        uint4 o; o.x = h2u(h0); o.y = h2u(h1); o.z = h2u(h2); o.w = h2u(h3);
        *(uint4 *)(xh + (size_t)pos * K + k) = o;
    }
}

struct mmid_g_plan { int BN, m_tiles, max_tiles, chunks, nstages, smem; size_t xb_bytes, scale_bytes, tab_bytes, perm_bytes; int64_t n_pairs; };

static bool make_mmid_g_plan(const ggml_b200_mul_mat_id_args & a, mmid_g_plan & pl) {
    static const int env_on = getenv("GGML_B200_MMID_GROUPED") ? atoi(getenv("GGML_B200_MMID_GROUPED")) : 0;      // opt-in until the reference's whole MUL_MAT_ID sweep has run with it (tests/gpu_mmid_grouped_check.py checks it)
    if (!env_on) return false;
    switch (a.type) {
        case T_Q4_0: case T_Q8_0: case T_Q4_K: case T_Q5_K: case T_Q6_K: case T_Q4_1: case T_Q5_0: case T_Q5_1: case T_IQ4_NL: case T_IQ4_XS: case T_Q2_K: case T_Q3_K: break;
        default: return false;
    }
    const int64_t n_pairs = a.n_used * a.n_tok;
    if (n_pairs < 32 || a.n_expert > MMID_MAX_EXPERTS || a.M < 128 || a.K % 256 != 0 || a.K < 256) return false;
    const size_t rb = row_bytes(a.type, a.K);
    if (a.nb01 != rb || a.nb02 != rb * (size_t)a.M || (rb % 16) != 0 || ((uintptr_t)a.src0 & 15) != 0) return false;
    if ((a.nb11 & 15) != 0 || (a.nb12 & 15) != 0 || ((uintptr_t)a.src1 & 15) != 0) return false;                 // 16-byte row loads in the conversion kernel
    if (a.n_expert * a.M >= (1ll << 31) || n_pairs >= (1ll << 30) || !tc_get_encode()) return false;
    // tile width: the average group size decides (Mixtral-like 8 x 2 at 512 tokens -> 128 per expert)
    const int64_t avg = n_pairs / (a.n_expert > 0 ? a.n_expert : 1);
    pl.BN = avg > 80 ? 128 : 64;
    pl.m_tiles = (int)((a.M + T2_BM - 1) / T2_BM);
    pl.max_tiles = (int)((n_pairs + pl.BN - 1) / pl.BN + a.n_expert);
    pl.chunks = (int)(a.K / (T2_BK * tc2_unit_ksteps(a.type)));
    if (!tc2_smem_plan(pl.BN, tc2_raw_bytes(a.type), pl.nstages, pl.smem)) return false;
    if ((int64_t)pl.m_tiles * pl.max_tiles > 0x7fffffffLL) return false;
    pl.n_pairs = n_pairs;
    pl.xb_bytes = ((size_t)(n_pairs + pl.BN) * a.K * 2 + 255) & ~(size_t)255;        // + one tile of slack rows (read past the last position, never used)
    pl.scale_bytes = ((size_t)(n_pairs + pl.BN) * 4 + 255) & ~(size_t)255;
    pl.tab_bytes = ((size_t)(2 * (a.n_expert + 1)) * 4 + 255) & ~(size_t)255;
    pl.perm_bytes = ((size_t)(n_pairs + pl.BN) * 4 + 255) & ~(size_t)255;
    return true;
}

bool mmid_grouped_eligible(const ggml_b200_mul_mat_id_args & a) { mmid_g_plan pl; return make_mmid_g_plan(a, pl); }
size_t mmid_grouped_workspace(const ggml_b200_mul_mat_id_args & a) {
    mmid_g_plan pl;
    if (!make_mmid_g_plan(a, pl)) return 0;
    return pl.xb_bytes + pl.scale_bytes + pl.tab_bytes + pl.perm_bytes + 1024;
}

template <int T> static int launch_mmid_g(const ggml_b200_mul_mat_id_args & a, const mmid_g_plan & pl, cudaStream_t st) {
    const size_t need = pl.xb_bytes + pl.scale_bytes + pl.tab_bytes + pl.perm_bytes + 1024;
    if (!a.workspace || a.workspace_size < need) { set_error("mul_mat_id: workspace %zu < %zu", a.workspace_size, need); return GGML_B200_EWORKSPACE; }
    uint8_t * ws = (uint8_t *)(((uintptr_t)a.workspace + 255) & ~(uintptr_t)255);
    __half * xb = (__half *)ws;
    float * inv_scale = (float *)(ws + pl.xb_bytes);
    int32_t * off = (int32_t *)(ws + pl.xb_bytes + pl.scale_bytes), * tile_base = off + (a.n_expert + 1);
    int32_t * perm = (int32_t *)(ws + pl.xb_bytes + pl.scale_bytes + pl.tab_bytes);
    mmid_group_kernel<<<1, 1024, 0, st>>>((const uint8_t *)a.ids, a.ids_nb1, (int)a.n_tok, (int)a.n_used, (int)a.n_expert, pl.BN, off, tile_base, perm);
    B200_LAUNCH_CHECK();
    mmid_x_to_f16_kernel<<<(unsigned)pl.n_pairs, 256, 0, st>>>((const uint8_t *)a.src1, a.nb11, a.nb12, (int)a.n_used, (int)a.nb1cols, off, perm, (int)a.n_expert, xb, inv_scale, a.K);
    B200_LAUNCH_CHECK();
    const size_t rb = row_bytes(a.type, a.K);
    alignas(64) CUtensorMap map_w, map_x;
    {
        const cuuint64_t dims[2] = { (cuuint64_t)(rb / 4), (cuuint64_t)(a.n_expert * a.M) };
        const cuuint64_t strides[1] = { (cuuint64_t)rb };
        const cuuint32_t box[2] = { (cuuint32_t)(tc2fmt<T>::RAW / 4), (cuuint32_t)T2_BM };
        const cuuint32_t es[2] = { 1, 1 };
        CUresult r = tc_get_encode()(&map_w, CU_TENSOR_MAP_DATA_TYPE_UINT32, 2, (void *)a.src0, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                     CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(W experts) failed: %d", (int)r); return GGML_B200_ECUDA; }
    }
    {
        const cuuint64_t dims[2] = { (cuuint64_t)a.K, (cuuint64_t)(pl.n_pairs + pl.BN) };
        const cuuint64_t strides[1] = { (cuuint64_t)a.K * 2 };
        const cuuint32_t box[2] = { (cuuint32_t)T2_BK, (cuuint32_t)pl.BN };
        const cuuint32_t es[2] = { 1, 1 };
        CUresult r = tc_get_encode()(&map_x, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, (void *)xb, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(X sorted) failed: %d", (int)r); return GGML_B200_ECUDA; }
    }
    tc2_params p{};
    p.y = a.dst; p.partials = nullptr; p.flags = nullptr; p.inv_scale = inv_scale; p.M = a.M; p.N = pl.n_pairs;
    p.BN = pl.BN; p.m_tiles = pl.m_tiles; p.n_tiles = pl.max_tiles; p.splitk = 1; p.units_total = pl.chunks; p.nstages = pl.nstages; p.w_static = 0;
    p.g_off = off; p.g_tile_base = tile_base; p.g_perm = perm; p.n_expert = (int32_t)a.n_expert;
    static per_device_flag attr_set;
    if (!attr_set.test()) { B200_CUDA_TRY(cudaFuncSetAttribute(mmq_tc2_kernel<T, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024)); attr_set.set(); }
    // plain launch (no programmatic dependency): the tile tables are read at kernel entry and must be complete
    mmq_tc2_kernel<T, true><<<(unsigned)(pl.m_tiles * pl.max_tiles), T2_THREADS, (size_t)pl.smem, st>>>(map_w, map_x, p);
    B200_LAUNCH_CHECK();
    return GGML_B200_OK;
}

int launch_mmid_grouped(const ggml_b200_mul_mat_id_args & a, cudaStream_t st) {
    mmid_g_plan pl;
    if (!make_mmid_g_plan(a, pl)) { set_error("mul_mat_id: shape not eligible for the grouped tensor-core path"); return GGML_B200_EUNSUPPORTED; }
    switch (a.type) {
        case T_Q4_0:   return launch_mmid_g<T_Q4_0>(a, pl, st);
        case T_Q8_0:   return launch_mmid_g<T_Q8_0>(a, pl, st);
        case T_Q4_K:   return launch_mmid_g<T_Q4_K>(a, pl, st);
        case T_Q5_K:   return launch_mmid_g<T_Q5_K>(a, pl, st);
        case T_Q6_K:   return launch_mmid_g<T_Q6_K>(a, pl, st);
        case T_Q4_1:   return launch_mmid_g<T_Q4_1>(a, pl, st);
        case T_Q5_0:   return launch_mmid_g<T_Q5_0>(a, pl, st);
        case T_Q5_1:   return launch_mmid_g<T_Q5_1>(a, pl, st);
        case T_IQ4_NL: return launch_mmid_g<T_IQ4_NL>(a, pl, st);
        case T_IQ4_XS: return launch_mmid_g<T_IQ4_XS>(a, pl, st);
        case T_Q2_K:   return launch_mmid_g<T_Q2_K>(a, pl, st);
        case T_Q3_K:   return launch_mmid_g<T_Q3_K>(a, pl, st);
        default: return GGML_B200_EUNSUPPORTED;
    }
}

} // namespace b200
