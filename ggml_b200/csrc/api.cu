// api.cu — extern "C" kernel-launch shim (include/ggml-b200.h, layer 1): argument validation, kernel selection, workspace
// accounting.  route() picks the kernel of a mul_mat call and keeps the plan it made for it (b200_mm_plan.h): the workspace query
// reports that plan's workspace and the launch runs that plan.  No CPU fallback anywhere: unsupported combinations return an error code.
#include "b200_internal.h"
#include "b200_mm_plan.h"
#include "b200_quants.cuh"

#include <algorithm>
#include <cstdarg>
#include <cstdlib>
#include <cstring>
#include <mutex>

namespace b200 {

std::atomic<uint64_t> g_launches{0};
static thread_local char g_err[512] = "";

void set_error(const char * fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int sm_count() {
    static int cached[64] = {0};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
    if (cached[dev] == 0) {
        int n = 0;
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
        cached[dev] = n;
    }
    return cached[dev];
}

// One per device, allocated on first use under a mutex (or ahead of time by ggml_b200_prepare, which the backend calls at device
// initialisation so that no allocation can fall inside a stream capture) and kept for the life of the process.
unsigned int * control_block() {
    static unsigned int * ptr[64] = { nullptr };
    static std::mutex mu;
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) { set_error("control block: cudaGetDevice failed"); return nullptr; }
    std::lock_guard<std::mutex> lock(mu);
    if (!ptr[dev]) {
        unsigned int * p = nullptr;
        const size_t bytes = (CTL_SPLITK_FLAGS + (size_t)TC_FLAG_SLOTS * TC_FLAGS_PER_SLOT) * sizeof(unsigned int);
        cudaError_t e = cudaMalloc(&p, bytes);
        if (e == cudaSuccess) e = cudaMemset(p, 0, bytes);
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

static int validate(const ggml_b200_mul_mat_args * a) {
    if (!a) { set_error("mul_mat: NULL args"); return GGML_B200_EINVAL; }
    if (type_bytes(a->type) == 0) { set_error("mul_mat: unsupported weight type %d", a->type); return GGML_B200_EUNSUPPORTED; }
    if (a->K <= 0 || a->M < 0 || a->N < 0 || a->ne02 < 1 || a->ne03 < 1 || a->ne12 < 1 || a->ne13 < 1) { set_error("mul_mat: bad shape"); return GGML_B200_EINVAL; }
    if (a->K % type_qk(a->type) != 0) { set_error("mul_mat: K=%lld is not a multiple of the block size %d", (long long)a->K, type_qk(a->type)); return GGML_B200_EINVAL; }
    if (a->ne12 % a->ne02 != 0 || a->ne13 % a->ne03 != 0) { set_error("mul_mat: batch dims do not broadcast"); return GGML_B200_EINVAL; }
    if (a->M > 0 && a->N > 0 && (!a->src0 || !a->src1 || !a->dst)) { set_error("mul_mat: NULL tensor pointer"); return GGML_B200_EINVAL; }
    if (a->nb01 < row_bytes(a->type, a->K) || (a->nb01 & 1) || (a->nb02 & 1) || (a->nb03 & 1) || ((uintptr_t)a->src0 & 1)) { set_error("mul_mat: bad src0 strides/alignment"); return GGML_B200_EINVAL; }
    if ((a->nb11 & 3) || (a->nb12 & 3) || (a->nb13 & 3) || ((uintptr_t)a->src1 & 3)) { set_error("mul_mat: src1 must be 4-byte aligned"); return GGML_B200_EINVAL; }
    // Q4_K / Q5_K headers are read as 16-byte vectors
    if ((a->type == T_Q4_K || a->type == T_Q5_K) && (((uintptr_t)a->src0 | a->nb01 | a->nb02 | a->nb03) & 15)) { set_error("mul_mat: Q4_K/Q5_K rows must be 16-byte aligned"); return GGML_B200_EINVAL; }
    return GGML_B200_OK;
}

// the int8 mma.sync consume path (mmvq_mma.cu): default for 2 <= n <= 8, and for n = 1 when the rows are very long (K >= 12288: the dp4a kernel's
// chunks shrink to a few rows there; at K = 8192 the dp4a kernel is still the faster one; threshold chosen on a Blackwell part, not re-measured
// on the H100).  Per call GGML_B200_MM_GEMV_MMA / GGML_B200_MM_GEMV_DP4A select explicitly.
static bool mma_wanted(const ggml_b200_mul_mat_args & a, mma_plan & pl) {
    if (a.flags & (GGML_B200_MM_GEMV_V1 | GGML_B200_MM_GEMV_DP4A)) return false;
    if (!(a.flags & GGML_B200_MM_GEMV_MMA) && a.N < 2 && a.K < 12288) return false;
    return plan_mma(a, pl);
}

// columns [c0, c0 + g) of a, or to the last column
static ggml_b200_mul_mat_args column_group(const ggml_b200_mul_mat_args & a, int64_t c0, int64_t g) {
    ggml_b200_mul_mat_args sub = a;
    sub.N = std::min<int64_t>(g, a.N - c0);
    sub.src1 = (const float *)((const char *)a.src1 + (size_t)c0 * a.nb11);
    sub.dst = a.dst + (size_t)c0 * a.M;
    return sub;
}

static int chosen(mm_plan & pl, route_kind kind, size_t workspace) {
    pl.kind = kind;
    pl.workspace = workspace;
    return GGML_B200_OK;
}

// The kernel one mul_mat call runs, with its plan.  The workspace query, the launch and the fused entry point all read it from route(),
// so they cannot disagree.  GGML_B200_EUNSUPPORTED when a forced family cannot run the shape, or when the last of the column groups
// cannot be planned; sets no error message.
static int route(const ggml_b200_mul_mat_args & a, mm_plan & pl) {
    static const bool env_generic = getenv("GGML_B200_FORCE_GENERIC") && atoi(getenv("GGML_B200_FORCE_GENERIC")) != 0;   // debugging aid
    pl.group = 0;
    if (env_generic || (a.flags & GGML_B200_MM_FORCE_GENERIC)) return chosen(pl, R_GENERIC, mmvq_generic_workspace(a));
    const bool force_gemv = (a.flags & GGML_B200_MM_FORCE_GEMV) != 0;
    if (!force_gemv && ((a.flags & GGML_B200_MM_FORCE_GEMM) || a.N > 8)) {
        if (plan_dense(a, pl.dense)) return chosen(pl, R_DENSE, pl.dense.workspace);     // formats without an operand decoder (n >= 9 only)
        if (plan_wgmma(a, pl.wgmma)) return chosen(pl, R_WGMMA, pl.wgmma.workspace);     // n >= 5 only
        if (a.flags & GGML_B200_MM_FORCE_GEMM) return GGML_B200_EUNSUPPORTED;
        return chosen(pl, R_GENERIC, mmvq_generic_workspace(a));
    }
    // the mat-vec family: forced, or n <= 8
    if (mma_wanted(a, pl.mma)) return chosen(pl, R_MMA, pl.mma.workspace);   // never under GEMV_V1
    const bool sb = plan_sb(a, pl.sb);
    // 5..8 columns of very long rows: the superblock kernel would need two column-group launches (each re-streaming W, issue-bound); the
    // tensor-core kernel takes them in one pass (fp16-operand tolerance instead of the integer-exact dot: DESIGN.md section 3)
    if (!force_gemv && a.N >= 5 && !sb && plan_wgmma(a, pl.wgmma)) return chosen(pl, R_WGMMA, pl.wgmma.workspace);
    const bool v1 = (a.flags & GGML_B200_MM_GEMV_V1) != 0;      // the first-generation kernel whenever the family is the mat-vec one
    if (sb && !v1) return chosen(pl, R_SB, 0);
    const bool tma = plan_tma(a, pl.tma);
    if (!tma && (force_gemv || !sb)) return force_gemv ? GGML_B200_EUNSUPPORTED : chosen(pl, R_GENERIC, mmvq_generic_workspace(a));
    if (!tma) return chosen(pl, R_TMA_UNFIT, 0);                // v1 and sb here
    if (v1) return chosen(pl, R_TMA, 0);
    // long rows x many columns: the activation records of all columns do not fit next to the weight stages.  Column groups of 4 / 2 / 1
    // on the same kernel re-stream W per group, which is far cheaper than leaving the bandwidth kernel (columns are independent: results
    // are bit-identical to the one-launch form).  This form is only reached when the first-generation kernel is eligible for the whole
    // shape (checked above), so a format it does not take (Q4_1, for one) goes to the generic kernel instead, even where the superblock
    // kernel would take its column groups.
    if (a.N > 1 && a.ne02 == 1 && a.ne03 == 1 && a.ne12 == 1 && a.ne13 == 1) {
        for (int64_t g = 4; g >= 1; g >>= 1) {
            if (g < a.N && plan_sb(column_group(a, 0, g), pl.sb)) {
                // every group is planned before the first one launches
                if (a.N % g != 0 && !plan_sb(column_group(a, a.N - a.N % g, g), pl.sb_tail)) return GGML_B200_EUNSUPPORTED;
                pl.group = g;
                return chosen(pl, R_SB_GROUPS, 0);
            }
        }
    }
    return chosen(pl, R_TMA, 0);
}

static int family(int rc, const mm_plan & r) {
    if (rc != GGML_B200_OK) return rc;
    switch (r.kind) {
        case R_GENERIC: return GGML_B200_MM_FORCE_GENERIC;
        case R_WGMMA: case R_DENSE: return GGML_B200_MM_FORCE_GEMM;
        default: return GGML_B200_MM_FORCE_GEMV;
    }
}

} // namespace b200

using namespace b200;

extern "C" {

const char * ggml_b200_last_error(void) { return g_err; }
const char * ggml_b200_version(void) { return "ggml-b200 0.1 (sm_90a)"; }
uint64_t ggml_b200_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }
int ggml_b200_sm_count(void) { return sm_count(); }
int ggml_b200_prepare(void) { return control_block() ? GGML_B200_OK : GGML_B200_ECUDA; }
int ggml_b200_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

size_t ggml_b200_row_size(int32_t type, int64_t k) {
    if (type == T_F32) return (size_t)k * 4;
    if (type == T_F16) return (size_t)k * 2;
    return row_bytes(type, k);
}

size_t ggml_b200_act_record_size(int32_t weight_type, int64_t K) {
    return (size_t)make_act_layout(K, type_is_kquant(weight_type)).bytes;
}

int ggml_b200_quantize_activations(int32_t weight_type, const float * src, size_t row_stride_bytes, int64_t nrows, int64_t K,
                                   void * dst_records, void * stream) {
    if (type_bytes(weight_type) == 0 || K <= 0 || K % type_qk(weight_type) != 0 || nrows < 0 || (row_stride_bytes & 3)) { set_error("quantize_activations: bad arguments"); return GGML_B200_EINVAL; }
    return launch_quantize_activations(weight_type, src, K, nrows, 1, 1, row_stride_bytes, 0, 0, dst_records, (cudaStream_t)stream);
}

int ggml_b200_mul_mat_plan(const ggml_b200_mul_mat_args * args) {
    const int rc = validate(args);
    if (rc != GGML_B200_OK) return rc;
    mm_plan pl;
    return family(route(*args, pl), pl);
}

size_t ggml_b200_mul_mat_workspace_size(const ggml_b200_mul_mat_args * args) {
    if (validate(args) != GGML_B200_OK) return 0;
    mm_plan pl;
    return route(*args, pl) == GGML_B200_OK ? pl.workspace : mmvq_generic_workspace(*args);
}

int ggml_b200_mul_mat(const ggml_b200_mul_mat_args * args, void * stream) {
    int rc = validate(args);
    if (rc != GGML_B200_OK) return rc;
    if (args->M == 0 || args->N == 0) return GGML_B200_OK;
    cudaStream_t st = (cudaStream_t)stream;
    mm_plan pl;
    if (route(*args, pl) != GGML_B200_OK) { set_error("mul_mat: the forced kernel family cannot run this shape"); return GGML_B200_EUNSUPPORTED; }
    switch (pl.kind) {
        case R_TMA:   return launch_tma(*args, pl.tma, st);
        case R_TMA_UNFIT: set_error("mul_mat: shape not eligible for the TMA mat-vec kernel"); return GGML_B200_EUNSUPPORTED;
        case R_SB:    return launch_sb(*args, pl.sb, st);
        case R_MMA:   return launch_mma(*args, pl.mma, st);
        case R_WGMMA: return launch_wgmma(*args, pl.wgmma, st);
        case R_DENSE: return launch_dense(*args, pl.dense, st);
        case R_SB_GROUPS:
            for (int64_t c0 = 0; c0 < args->N; c0 += pl.group) {
                const ggml_b200_mul_mat_args sub = column_group(*args, c0, pl.group);
                rc = launch_sb(sub, sub.N == pl.group ? pl.sb : pl.sb_tail, st);
                if (rc != GGML_B200_OK) return rc;
            }
            return GGML_B200_OK;
        default:      return launch_mmvq_generic(*args, st);
    }
}

size_t ggml_b200_mul_mat_f16_workspace_size(int64_t M, int64_t N, int64_t K) { return mmq_f16w_workspace(M, N, K); }
int ggml_b200_mul_mat_f16(const void * w, size_t nb01, const float * x, size_t nb11, float * y, int64_t M, int64_t N, int64_t K, void * workspace, size_t workspace_size,
                          uint32_t flags, void * stream) {
    if (M == 0 || N == 0) return GGML_B200_OK;
    return launch_mmq_f16w(w, nb01, x, nb11, y, M, N, K, workspace, workspace_size, flags, (cudaStream_t)stream);
}

size_t ggml_b200_mul_mat_f16_f16_workspace_size(int64_t M, int64_t N, int64_t K) { return mmq_f16f16_workspace(M, N, K); }
int ggml_b200_mul_mat_f16_f16(const void * w, size_t nb01, const void * x, size_t nb11, float * y, int64_t M, int64_t N, int64_t K, void * workspace, size_t workspace_size,
                              uint32_t flags, void * stream) {
    if (M == 0 || N == 0) return GGML_B200_OK;
    return launch_mmq_f16f16(w, nb01, x, nb11, y, M, N, K, workspace, workspace_size, flags, (cudaStream_t)stream);
}

int ggml_b200_mul_mat_fused(const ggml_b200_mul_mat_args * args, const ggml_b200_epilogue * ep, void * stream) {
    int rc = validate(args);
    if (rc != GGML_B200_OK) return rc;
    if (!ep || !ep->bias || !ep->dst_bias || (ep->unary < 0 || ep->unary > 2) || (ep->unary != 0 && !ep->dst_unary) || (ep->unary == 2 && !ep->residual)) { set_error("mul_mat_fused: bad epilogue"); return GGML_B200_EINVAL; }
    // also where the unfused route is the mma kernel (n = 1, very long rows): the epilogue exists on the superblock kernel only
    mm_plan r;
    sb_plan pl;
    if (args->N != 1 || family(route(*args, r), r) != GGML_B200_MM_FORCE_GEMV || !plan_sb(*args, pl)) { set_error("mul_mat_fused: only the n = 1 mat-vec kernel has the fused epilogue"); return GGML_B200_EUNSUPPORTED; }
    if (args->M == 0) return GGML_B200_OK;
    return launch_sb(*args, pl, (cudaStream_t)stream, nullptr, ep);
}

int ggml_b200_mul_mat_gather(const ggml_b200_mul_mat_args * args, const ggml_b200_gather * ga, void * stream) {
    int rc = validate(args);
    if (rc != GGML_B200_OK) return rc;
    if (!ga || ga->world < 1 || ga->world > 8 || ga->rank < 0 || ga->rank >= ga->world) { set_error("mul_mat_gather: bad gather descriptor"); return GGML_B200_EINVAL; }
    for (int q = 0; q < ga->world; ++q) if (!ga->y_peers[q] || !ga->flag_peers[q]) { set_error("mul_mat_gather: NULL peer pointer"); return GGML_B200_EINVAL; }
    sb_plan pl;
    if (args->N != 1 || !plan_sb(*args, pl)) { set_error("mul_mat_gather: only the n = 1 mat-vec path supports the fused gather"); return GGML_B200_EUNSUPPORTED; }
    return launch_sb(*args, pl, (cudaStream_t)stream, ga);
}

int ggml_b200_mul_mat_gather_supported(const ggml_b200_mul_mat_args * args) {
    sb_plan pl;
    return validate(args) == GGML_B200_OK && args->N == 1 && plan_sb(*args, pl) ? 1 : 0;
}

int ggml_b200_gather_wait(const uint32_t * flags_local, int32_t world, uint32_t epoch, void * stream) {
    if (!flags_local || world < 1 || world > 8) { set_error("gather_wait: bad arguments"); return GGML_B200_EINVAL; }
    return launch_gather_wait(flags_local, world, epoch, (cudaStream_t)stream);
}

int ggml_b200_ipc_alloc(size_t bytes, void ** dev_ptr, void * handle64) {
    if (!dev_ptr || !handle64 || bytes == 0) { set_error("ipc_alloc: bad arguments"); return GGML_B200_EINVAL; }
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "handle size");
    B200_CUDA_TRY(cudaMalloc(dev_ptr, bytes));
    B200_CUDA_TRY(cudaMemset(*dev_ptr, 0, bytes));
    B200_CUDA_TRY(cudaDeviceSynchronize());
    B200_CUDA_TRY(cudaIpcGetMemHandle((cudaIpcMemHandle_t *)handle64, *dev_ptr));
    return GGML_B200_OK;
}
int ggml_b200_ipc_free(void * dev_ptr) { B200_CUDA_TRY(cudaFree(dev_ptr)); return GGML_B200_OK; }
int ggml_b200_ipc_open(const void * handle64, void ** dev_ptr) {
    if (!dev_ptr || !handle64) { set_error("ipc_open: bad arguments"); return GGML_B200_EINVAL; }
    cudaIpcMemHandle_t h;
    memcpy(&h, handle64, sizeof(h));
    B200_CUDA_TRY(cudaIpcOpenMemHandle(dev_ptr, h, cudaIpcMemLazyEnablePeerAccess));
    return GGML_B200_OK;
}
int ggml_b200_ipc_close(void * dev_ptr) { B200_CUDA_TRY(cudaIpcCloseMemHandle(dev_ptr)); return GGML_B200_OK; }

int ggml_b200_mul_mat_host(const ggml_b200_mul_mat_args * args, const float * host_src1, float * host_dst, void * stream) {
    int rc = validate(args);
    if (rc != GGML_B200_OK) return rc;
    if (!host_src1 || !host_dst) { set_error("mul_mat_host: NULL host pointer"); return GGML_B200_EINVAL; }
    if (args->nb11 != (size_t)args->K * 4 || args->nb12 != args->nb11 * (size_t)args->N || args->nb13 != args->nb12 * (size_t)args->ne12) { set_error("mul_mat_host: device staging for src1 must be contiguous"); return GGML_B200_EINVAL; }
    cudaStream_t st = (cudaStream_t)stream;
    const size_t xin = (size_t)args->K * args->N * args->ne12 * args->ne13 * 4, yout = (size_t)args->M * args->N * args->ne12 * args->ne13 * 4;
    B200_CUDA_TRY(cudaMemcpyAsync((void *)args->src1, host_src1, xin, cudaMemcpyHostToDevice, st));
    rc = ggml_b200_mul_mat(args, stream);
    if (rc != GGML_B200_OK) return rc;
    B200_CUDA_TRY(cudaMemcpyAsync(host_dst, args->dst, yout, cudaMemcpyDeviceToHost, st));
    B200_CUDA_TRY(cudaStreamSynchronize(st));
    return GGML_B200_OK;
}

int ggml_b200_mul_mat_host_batch(const ggml_b200_mul_mat_args * args, int32_t n, const float * host_src1, float * const * host_dst, void * stream) {
    if (!args || n < 1 || !host_src1 || !host_dst) { set_error("mul_mat_host_batch: bad arguments"); return GGML_B200_EINVAL; }
    cudaStream_t st = (cudaStream_t)stream;
    for (int i = 0; i < n; ++i) {
        int rc = validate(&args[i]);
        if (rc != GGML_B200_OK) return rc;
        if (args[i].src1 != args[0].src1 || args[i].K != args[0].K || args[i].N != args[0].N || args[i].ne12 != 1 || args[i].ne13 != 1 ||
            args[i].nb11 != (size_t)args[i].K * 4) { set_error("mul_mat_host_batch: all ops must share one contiguous src1 staging buffer"); return GGML_B200_EINVAL; }
    }
    B200_CUDA_TRY(cudaMemcpyAsync((void *)args[0].src1, host_src1, (size_t)args[0].K * args[0].N * 4, cudaMemcpyHostToDevice, st));
    for (int i = 0; i < n; ++i) {
        int rc = ggml_b200_mul_mat(&args[i], stream);
        if (rc != GGML_B200_OK) return rc;
    }
    for (int i = 0; i < n; ++i)
        B200_CUDA_TRY(cudaMemcpyAsync(host_dst[i], args[i].dst, (size_t)args[i].M * args[i].N * 4, cudaMemcpyDeviceToHost, st));
    B200_CUDA_TRY(cudaStreamSynchronize(st));
    return GGML_B200_OK;
}

} // extern "C"
