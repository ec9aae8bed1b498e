// api.cu — extern "C" kernel-launch shim (include/ggml-b200.h, layer 1): argument validation, kernel-family
// selection, workspace accounting.  No CPU fallback anywhere: unsupported combinations return an error code.
#include "b200_internal.h"
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
// on the H100).
// GGML_B200_MMA = 0 never, 2 always; per call GGML_B200_MM_GEMV_MMA / GGML_B200_MM_GEMV_DP4A select explicitly
static bool mma_wanted(const ggml_b200_mul_mat_args & a) {
    static const int env = getenv("GGML_B200_MMA") ? atoi(getenv("GGML_B200_MMA")) : 1;
    if (a.flags & (GGML_B200_MM_GEMV_V1 | GGML_B200_MM_GEMV_DP4A)) return false;
    if (!(a.flags & GGML_B200_MM_GEMV_MMA) && (env == 0 || (a.N < 2 && env != 2 && a.K < 12288))) return false;
    return mmvq_mma_eligible(a);
}

static int plan(const ggml_b200_mul_mat_args & a) {
    static const bool env_generic = getenv("GGML_B200_FORCE_GENERIC") && atoi(getenv("GGML_B200_FORCE_GENERIC")) != 0;   // debugging aid
    if (env_generic) return GGML_B200_MM_FORCE_GENERIC;
    if (a.flags & GGML_B200_MM_FORCE_GENERIC) return GGML_B200_MM_FORCE_GENERIC;
    if (a.flags & GGML_B200_MM_FORCE_GEMV) {
        const bool ok = (a.flags & GGML_B200_MM_GEMV_V1) ? mmvq_tma_eligible(a) : (mma_wanted(a) || mmvq_sb_eligible(a) || mmvq_tma_eligible(a));
        return ok ? GGML_B200_MM_FORCE_GEMV : GGML_B200_EUNSUPPORTED;
    }
    if (a.flags & GGML_B200_MM_FORCE_GEMM) return (mmq_tc_eligible(a) || mmq_tc_eligible_small(a)) ? GGML_B200_MM_FORCE_GEMM : GGML_B200_EUNSUPPORTED;
    // 5..8 columns of very long rows: the superblock kernel would need two column-group launches (each re-streaming W, issue-bound); the
    // tensor-core kernel takes them in one pass (fp16-operand tolerance instead of the integer-exact dot: DESIGN.md section 3)
    if (a.N <= 8 && mma_wanted(a)) return GGML_B200_MM_FORCE_GEMV;
    if (a.N >= 5 && a.N <= 8 && !mmvq_sb_eligible(a) && mmq_tc_eligible_small(a)) return GGML_B200_MM_FORCE_GEMM;
    if (a.N <= 8 && (mmvq_sb_eligible(a) || mmvq_tma_eligible(a))) return GGML_B200_MM_FORCE_GEMV;
    if (a.N > 8 && mmq_tc_eligible(a)) return GGML_B200_MM_FORCE_GEMM;
    return GGML_B200_MM_FORCE_GENERIC;
}

} // namespace b200

using namespace b200;

extern "C" {

const char * ggml_b200_last_error(void) { return g_err; }
const char * ggml_b200_version(void) { return "ggml-b200 0.1 (sm_90a)"; }
uint64_t ggml_b200_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }
int ggml_b200_sm_count(void) { return sm_count(); }
int ggml_b200_prepare(void) { const int rc = prepare_device(); return rc != GGML_B200_OK ? rc : tc_prepare_device(); }
int ggml_b200_debug_gemm_trace(uint64_t * host_dst, int32_t max_ctas) { return tc2_trace_read((unsigned long long *)host_dst, max_ctas); }
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
    return plan(*args);
}

size_t ggml_b200_mul_mat_workspace_size(const ggml_b200_mul_mat_args * args) {
    if (validate(args) != GGML_B200_OK) return 0;
    switch (plan(*args)) {
        case GGML_B200_MM_FORCE_GEMV: return mma_wanted(*args) ? mmvq_mma_workspace(*args) : 0;
        case GGML_B200_MM_FORCE_GEMM: return mmq_tc_workspace(*args);
        default: return mmvq_generic_workspace(*args);
    }
}

int ggml_b200_mul_mat(const ggml_b200_mul_mat_args * args, void * stream) {
    int rc = validate(args);
    if (rc != GGML_B200_OK) return rc;
    if (args->M == 0 || args->N == 0) return GGML_B200_OK;
    cudaStream_t st = (cudaStream_t)stream;
    switch (plan(*args)) {
        case GGML_B200_MM_FORCE_GEMV:
            // the superblock kernel (mmvq_sb.cu) for 1 <= n <= 8; the first-generation unit kernel (mmvq.cu) on request or as the last resort
            if (!(args->flags & GGML_B200_MM_GEMV_V1)) {
                if (mma_wanted(*args)) return launch_mmvq_mma(*args, st);
                if (mmvq_sb_eligible(*args)) return launch_mmvq_sb(*args, st);
                // long rows x many columns: the activation records of all columns do not fit next to the weight stages.  Column groups of
                // 4 / 2 / 1 on the same kernel re-stream W per group, which is far cheaper than leaving the bandwidth kernel
                // (columns are independent: results are bit-identical to the one-launch form)
                if (args->N > 1 && args->ne02 == 1 && args->ne03 == 1 && args->ne12 == 1 && args->ne13 == 1) {
                    for (int64_t g = 4; g >= 1; g >>= 1) {
                        if (g >= args->N) continue;
                        ggml_b200_mul_mat_args sub = *args;
                        sub.N = g;
                        if (!mmvq_sb_eligible(sub)) continue;
                        for (int64_t c0 = 0; c0 < args->N; c0 += g) {
                            sub.N = std::min<int64_t>(g, args->N - c0);
                            sub.src1 = (const float *)((const char *)args->src1 + (size_t)c0 * args->nb11);
                            sub.dst = args->dst + (size_t)c0 * args->M;
                            if (!mmvq_sb_eligible(sub)) { set_error("mul_mat: column group not eligible"); return GGML_B200_EUNSUPPORTED; }
                            rc = launch_mmvq_sb(sub, st);
                            if (rc != GGML_B200_OK) return rc;
                        }
                        return GGML_B200_OK;
                    }
                }
            }
            return launch_mmvq_tma(*args, st);
        case GGML_B200_MM_FORCE_GEMM:    return launch_mmq_tc(*args, st);
        case GGML_B200_MM_FORCE_GENERIC: return launch_mmvq_generic(*args, st);
        default: set_error("mul_mat: the forced kernel family cannot run this shape"); return GGML_B200_EUNSUPPORTED;
    }
}

size_t ggml_b200_mul_mat_f16_workspace_size(int64_t M, int64_t N, int64_t K) { return mmq_f16w_workspace(M, N, K); }
int ggml_b200_mul_mat_f16(const void * w, size_t nb01, const float * x, size_t nb11, float * y, int64_t M, int64_t N, int64_t K, void * workspace, size_t workspace_size,
                          uint32_t flags, void * stream) {
    if (M == 0 || N == 0) return GGML_B200_OK;
    return launch_mmq_f16w(w, nb01, x, nb11, y, M, N, K, workspace, workspace_size, flags, (cudaStream_t)stream);
}

int ggml_b200_mul_mat_fused(const ggml_b200_mul_mat_args * args, const ggml_b200_epilogue * ep, void * stream) {
    int rc = validate(args);
    if (rc != GGML_B200_OK) return rc;
    if (!ep || !ep->bias || !ep->dst_bias || (ep->unary < 0 || ep->unary > 2) || (ep->unary != 0 && !ep->dst_unary) || (ep->unary == 2 && !ep->residual)) { set_error("mul_mat_fused: bad epilogue"); return GGML_B200_EINVAL; }
    if (args->N != 1 || plan(*args) != GGML_B200_MM_FORCE_GEMV || !mmvq_sb_eligible(*args)) { set_error("mul_mat_fused: only the n = 1 mat-vec kernel has the fused epilogue"); return GGML_B200_EUNSUPPORTED; }
    if (args->M == 0) return GGML_B200_OK;
    return launch_mmvq_sb(*args, (cudaStream_t)stream, nullptr, ep);
}

int ggml_b200_mul_mat_gather(const ggml_b200_mul_mat_args * args, const ggml_b200_gather * ga, void * stream) {
    int rc = validate(args);
    if (rc != GGML_B200_OK) return rc;
    if (!ga || ga->world < 1 || ga->world > 8 || ga->rank < 0 || ga->rank >= ga->world) { set_error("mul_mat_gather: bad gather descriptor"); return GGML_B200_EINVAL; }
    for (int q = 0; q < ga->world; ++q) if (!ga->y_peers[q] || !ga->flag_peers[q]) { set_error("mul_mat_gather: NULL peer pointer"); return GGML_B200_EINVAL; }
    if (args->N != 1 || !mmvq_sb_eligible(*args)) { set_error("mul_mat_gather: only the n = 1 mat-vec path supports the fused gather"); return GGML_B200_EUNSUPPORTED; }
    return launch_mmvq_sb(*args, (cudaStream_t)stream, ga);
}

int ggml_b200_mul_mat_gather_supported(const ggml_b200_mul_mat_args * args) {
    return validate(args) == GGML_B200_OK && args->N == 1 && mmvq_sb_eligible(*args) ? 1 : 0;
}

int ggml_b200_debug_trace(unsigned long long * out256) { return debug_read_trace(out256); }

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
