// ggml-b200.cpp — the ggml backend plug-in (include/ggml-b200.h, layer 2).
//
// Implements the reference's backend SPI (src/ggml-backend-impl.h:17-207) for NVIDIA H100 (sm_90a):
//   ggml_backend_reg_i          -> "B200" registry entry, one device per visible GPU
//   ggml_backend_device_i       -> B200<i>: memory, props, supports_op / supports_buft / offload_op, events
//   ggml_backend_buffer_type_i  -> device memory (cudaMalloc), alignment 128; pinned host buffer type
//   ggml_backend_buffer_i       -> set/get/memset/cpy/clear with synchronous semantics
//   ggml_backend_i              -> one CUDA stream; graph_compute walks cgraph->nodes and launches the kernels
//                                  of libggml-b200-kernels.so through its extern "C" shim
// so that ggml_backend_sched, tests/test-backend-ops and examples/gpt-2 drive it unmodified.  This file is what
// would live in src/ggml-b200/ of the ggml tree; it is host-side C++ only (no kernels) and is compiled against
// the reference's headers.  It replaces the vtable glue of src/ggml-cuda/ggml-cuda.cu:480-3438.
//
// supports_op is exact: anything it accepts is executed on the device, there is no CPU fallback in here
// (unsupported nodes reaching graph_compute abort, as in the reference, ggml-cuda.cu:2655-2659).  Each op has one binding (bound_op) that
// builds its launcher's arguments from the node; supports_op and graph_compute both go through it, the first to ask the launcher's own
// check (ggml_b200/csrc/b200_op_checks.h) plus what the launcher cannot see, the second to launch, so the check sees the descriptors the
// launch passes.  The quantized MUL_MAT / MUL_MAT_ID decide in supports_mul_mat*; mul_mat_route picks a MUL_MAT node's kernel family and
// scratch, for the pre-capture sizing and the launch alike.

#include "ggml.h"
#include "ggml-backend.h"
#include "ggml-backend-impl.h"
#include "ggml-impl.h"
#include "ggml-cuda.h"          // the C ABI we additionally provide for programs built with -DGGML_USE_CUDA

#include "ggml-b200.h"
#include "ggml-b200-backend.h"
#include "b200_op_checks.h"

#include <cuda_runtime.h>

#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <string>
#include <unordered_set>
#include <vector>

#define B200_MAX_DEVICES 16

#define CUDA_OK(expr)                                                                                          \
    do {                                                                                                       \
        cudaError_t err_ = (expr);                                                                             \
        if (err_ != cudaSuccess) {                                                                             \
            GGML_LOG_ERROR("ggml-b200: %s failed: %s (%s:%d)\n", #expr, cudaGetErrorString(err_), __FILE__, __LINE__); \
            GGML_ABORT("CUDA error");                                                                          \
        }                                                                                                      \
    } while (0)

#define SHIM_OK(expr)                                                                                          \
    do {                                                                                                       \
        int rc_ = (expr);                                                                                      \
        if (rc_ != GGML_B200_OK) {                                                                             \
            GGML_LOG_ERROR("ggml-b200: %s failed (%d): %s\n", #expr, rc_, ggml_b200_last_error());             \
            GGML_ABORT("kernel shim error");                                                                   \
        }                                                                                                      \
    } while (0)

namespace {

struct device_ctx {
    int         index = 0;
    std::string name;          // "B2000", "B2001", ...
    std::string description;   // cudaDeviceProp.name
    ggml_backend_buffer_type buft{};        // device memory
    std::string buft_name;
};

struct backend_ctx {
    int          device = 0;
    cudaStream_t stream = nullptr;
    void *       workspace = nullptr;   // stream-ordered scratch for the kernel shim
    size_t       workspace_size = 0;
    std::string  name;
    cudaEvent_t  copy_event = nullptr;  // orders cross-backend copies (cpy_tensor_async)
    // CUDA-graph replay of whole ggml graphs (like the reference, src/ggml-cuda/ggml-cuda.cu:2696-2767): the node loop is
    // stream-captured and launched as one executable graph per graph_compute.
    // A small cache of instantiated graphs keyed on the exact node properties (ops, shapes, strides, data pointers, parameters,
    // sources): an unchanged ggml graph is replayed without being re-captured; a changed one is captured and the executable
    // graph of matching topology is updated in place (cudaGraphExecUpdate), re-instantiated only if that fails.
    struct cached_graph { std::vector<uint64_t> sig; cudaGraphExec_t exec = nullptr; uint64_t last_use = 0; };
    std::vector<cached_graph> graphs;
    uint64_t        graph_clock = 0;
    // a graph that changes on every call (token-by-token decoding: shapes and offsets move with n_past) costs more to re-capture and
    // update than to launch directly: after a few consecutive misses the nodes are launched eagerly (every kernel is PDL-chained), until
    // the same graph is seen twice in a row again.  The reference does the same (ggml-cuda.cu: disable_due_to_too_many_updates).
    int             consecutive_updates = 0;
    std::vector<uint64_t> last_sig;
    int             graph_calls = 0;      // the first graph_compute runs eagerly (one-time attribute / allocation work)
    bool            capturing = false;
    std::unordered_set<const ggml_tensor *> written;   // roots whose memory some node of the current cgraph writes through a view
    bool            first_real_node = true;
    // GGML_B200_PROFILE=1: host time spent in graph_compute per mode (printed when the backend is freed)
    struct host_profile { uint64_t calls[4] = {0,0,0,0}; double us[4] = {0,0,0,0}; uint64_t nodes[4] = {0,0,0,0}; } prof;   // 0 replay, 1 capture+update, 2 eager, 3 small/first
    // split-buffer mat-muls: one auxiliary stream per other device (+ staging for the activations, the n > 1 result, kernel scratch)
    struct split_peer {
        cudaStream_t stream = nullptr; cudaEvent_t done = nullptr;
        void * x_stage = nullptr; size_t x_cap = 0; void * y_stage = nullptr; size_t y_cap = 0; void * ws = nullptr; size_t ws_cap = 0;
        bool peer_access = false;
    };
    split_peer   peers[B200_MAX_DEVICES];
    cudaEvent_t  split_fork = nullptr;
    uint32_t *   split_flags = nullptr;      // on this device: one arrival flag per participating device (fused gather)
    uint32_t     split_epoch = 0;

    void * scratch(size_t need) {
        if (need <= workspace_size) return workspace;
        GGML_ASSERT(!capturing && "scratch must be sized before stream capture");
        // the kernels of every cached executable graph hold the old pool address (it is not part of the node signature): a later replay
        // would write through a freed pointer.  Graphs still in flight finish first (cudaGraphExecDestroy defers, cudaFreeAsync is stream-ordered).
        if (workspace) {
            for (auto & g : graphs) if (g.exec) CUDA_OK(cudaGraphExecDestroy(g.exec));
            graphs.clear();
            CUDA_OK(cudaFreeAsync(workspace, stream));
        }
        size_t sz = need + need / 4;
        sz = (sz + (1u << 20) - 1) & ~(size_t)((1u << 20) - 1);
        CUDA_OK(cudaMallocAsync(&workspace, sz, stream));
        workspace_size = sz;
        return workspace;
    }
};

struct buffer_ctx {
    int    device = 0;
    void * base = nullptr;
};

struct scoped_device {
    int prev = -1;
    explicit scoped_device(int dev) {
        CUDA_OK(cudaGetDevice(&prev));
        if (prev != dev) CUDA_OK(cudaSetDevice(dev)); else prev = -1;
    }
    ~scoped_device() { if (prev >= 0) cudaSetDevice(prev); }
};

ggml_backend_reg_t b200_reg();
ggml_guid_t b200_guid() {
    static ggml_guid guid = { 0xb2, 0x00, 0x5a, 0x10, 0x0a, 0x67, 0x67, 0x6d, 0x6c, 0x2d, 0x62, 0x32, 0x30, 0x30, 0x01, 0x00 };
    return &guid;
}

// ------------------------------------------------------------------------------------------ buffers
bool buft_is_b200(ggml_backend_buffer_type_t buft);
bool buffer_is_b200(ggml_backend_buffer_t buffer);

void buffer_free(ggml_backend_buffer_t buffer) {
    buffer_ctx * ctx = (buffer_ctx *) buffer->context;
    scoped_device sd(ctx->device);
    CUDA_OK(cudaFree(ctx->base));
    delete ctx;
}
void * buffer_get_base(ggml_backend_buffer_t buffer) { return ((buffer_ctx *) buffer->context)->base; }

void buffer_memset_tensor(ggml_backend_buffer_t buffer, ggml_tensor * tensor, uint8_t value, size_t offset, size_t size) {
    buffer_ctx * ctx = (buffer_ctx *) buffer->context;
    scoped_device sd(ctx->device);
    CUDA_OK(cudaMemsetAsync((char *) tensor->data + offset, value, size, cudaStreamPerThread));
    CUDA_OK(cudaStreamSynchronize(cudaStreamPerThread));
}
// GGML_B200_PROFILE=1: host time in the synchronous tensor transfers and in backend synchronize (printed with the graph_compute profile)
struct io_profile { std::atomic<uint64_t> calls[3]; std::atomic<uint64_t> ns[3]; };      // 0 set_tensor, 1 get_tensor, 2 synchronize
io_profile g_io_prof;
bool profile_on() { static const bool on = getenv("GGML_B200_PROFILE") && atoi(getenv("GGML_B200_PROFILE")) != 0; return on; }
struct io_timer {
    int k; std::chrono::steady_clock::time_point t0;
    explicit io_timer(int kind) : k(profile_on() ? kind : -1) { if (k >= 0) t0 = std::chrono::steady_clock::now(); }
    ~io_timer() { if (k >= 0) { g_io_prof.calls[k]++; g_io_prof.ns[k] += (uint64_t) std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t0).count(); } }
};

void buffer_set_tensor(ggml_backend_buffer_t buffer, ggml_tensor * tensor, const void * data, size_t offset, size_t size) {
    buffer_ctx * ctx = (buffer_ctx *) buffer->context;
    scoped_device sd(ctx->device);
    io_timer tm(0);
    CUDA_OK(cudaMemcpyAsync((char *) tensor->data + offset, data, size, cudaMemcpyHostToDevice, cudaStreamPerThread));
    CUDA_OK(cudaStreamSynchronize(cudaStreamPerThread));
}
void buffer_get_tensor(ggml_backend_buffer_t buffer, const ggml_tensor * tensor, void * data, size_t offset, size_t size) {
    buffer_ctx * ctx = (buffer_ctx *) buffer->context;
    scoped_device sd(ctx->device);
    io_timer tm(1);
    CUDA_OK(cudaMemcpyAsync(data, (const char *) tensor->data + offset, size, cudaMemcpyDeviceToHost, cudaStreamPerThread));
    CUDA_OK(cudaStreamSynchronize(cudaStreamPerThread));
}
bool buffer_cpy_tensor(ggml_backend_buffer_t buffer, const ggml_tensor * src, ggml_tensor * dst) {
    ggml_backend_buffer_t sbuf = src->view_src ? src->view_src->buffer : src->buffer;
    if (!sbuf || !buffer_is_b200(sbuf)) return false;
    buffer_ctx * sctx = (buffer_ctx *) sbuf->context;
    buffer_ctx * dctx = (buffer_ctx *) buffer->context;
    scoped_device sd(dctx->device);
    if (sctx->device == dctx->device) CUDA_OK(cudaMemcpyAsync(dst->data, src->data, ggml_nbytes(src), cudaMemcpyDeviceToDevice, cudaStreamPerThread));
    else                              CUDA_OK(cudaMemcpyPeerAsync(dst->data, dctx->device, src->data, sctx->device, ggml_nbytes(src), cudaStreamPerThread));
    CUDA_OK(cudaStreamSynchronize(cudaStreamPerThread));
    return true;
}
void buffer_clear(ggml_backend_buffer_t buffer, uint8_t value) {
    buffer_ctx * ctx = (buffer_ctx *) buffer->context;
    scoped_device sd(ctx->device);
    CUDA_OK(cudaDeviceSynchronize());
    CUDA_OK(cudaMemset(ctx->base, value, buffer->size));
    CUDA_OK(cudaDeviceSynchronize());
}

const ggml_backend_buffer_i k_buffer_iface = {
    /* .free_buffer   = */ buffer_free,
    /* .get_base      = */ buffer_get_base,
    /* .init_tensor   = */ nullptr,
    /* .memset_tensor = */ buffer_memset_tensor,
    /* .set_tensor    = */ buffer_set_tensor,
    /* .get_tensor    = */ buffer_get_tensor,
    /* .cpy_tensor    = */ buffer_cpy_tensor,
    /* .clear         = */ buffer_clear,
    /* .reset         = */ nullptr,
};

const char * buft_get_name(ggml_backend_buffer_type_t buft) { return ((device_ctx *) buft->device->context)->buft_name.c_str(); }
ggml_backend_buffer_t buft_alloc_buffer(ggml_backend_buffer_type_t buft, size_t size) {
    device_ctx * dctx = (device_ctx *) buft->device->context;
    scoped_device sd(dctx->index);
    void * ptr = nullptr;
    // +256: the mat-vec kernels read packed 2-byte-aligned blocks through aligned 32-bit words, which may touch
    // up to 2 bytes past the last block of the last tensor
    cudaError_t err = cudaMalloc(&ptr, size + 256);
    if (err != cudaSuccess) {
        cudaGetLastError();
        GGML_LOG_ERROR("ggml-b200: allocating %.2f MiB on device %d failed: %s\n", size / 1048576.0, dctx->index, cudaGetErrorString(err));
        return nullptr;
    }
    buffer_ctx * ctx = new buffer_ctx{ dctx->index, ptr };
    return ggml_backend_buffer_init(buft, k_buffer_iface, ctx, size);
}
size_t buft_get_alignment(ggml_backend_buffer_type_t) { return 128; }
size_t buft_get_alloc_size(ggml_backend_buffer_type_t, const ggml_tensor * tensor) { return ggml_nbytes(tensor); }

const ggml_backend_buffer_type_i k_buft_iface = {
    /* .get_name       = */ buft_get_name,
    /* .alloc_buffer   = */ buft_alloc_buffer,
    /* .get_alignment  = */ buft_get_alignment,
    /* .get_max_size   = */ nullptr,
    /* .get_alloc_size = */ buft_get_alloc_size,
    /* .is_host        = */ nullptr,
};

bool buft_is_b200(ggml_backend_buffer_type_t buft) { return buft && buft->iface.get_name == buft_get_name; }
bool buffer_is_b200(ggml_backend_buffer_t buffer) { return buffer && buft_is_b200(buffer->buft); }

// pinned host buffers: a CPU buffer (so the CPU backend can use it) whose memory is cudaMallocHost'ed
const char * host_buft_get_name(ggml_backend_buffer_type_t) { return "B200_Host"; }
void host_buffer_free(ggml_backend_buffer_t buffer) { CUDA_OK(cudaFreeHost(buffer->context)); }
ggml_backend_buffer_t host_buft_alloc_buffer(ggml_backend_buffer_type_t buft, size_t size) {
    void * ptr = nullptr;
    if (cudaMallocHost(&ptr, size) != cudaSuccess) {
        cudaGetLastError();
        GGML_LOG_WARN("ggml-b200: failed to allocate %.2f MiB of pinned memory, using pageable memory\n", size / 1048576.0);
        return ggml_backend_buft_alloc_buffer(ggml_backend_cpu_buffer_type(), size);
    }
    ggml_backend_buffer_t buffer = ggml_backend_cpu_buffer_from_ptr(ptr, size);
    buffer->buft = buft;
    buffer->iface.free_buffer = host_buffer_free;
    return buffer;
}
size_t host_buft_get_alignment(ggml_backend_buffer_type_t) { return 64; }
bool   host_buft_is_host(ggml_backend_buffer_type_t) { return true; }

int registry_device_count();
ggml_backend_buffer_type_t host_buffer_type() {
    if (registry_device_count() == 0) return nullptr;        // no supported GPU visible: there is no device to hang the buffer type on (reg_get_device would assert)
    static ggml_backend_buffer_type buft = {
        /* .iface   = */ { host_buft_get_name, host_buft_alloc_buffer, host_buft_get_alignment, nullptr, nullptr, host_buft_is_host },
        /* .device  = */ ggml_backend_reg_dev_get(b200_reg(), 0),
        /* .context = */ nullptr,
    };
    return &buft;
}


// ------------------------------------------------------------------------------------------ split buffers (row-sharded weights)
// The reference's multi-GPU entry (src/ggml-cuda/ggml-cuda.cu:716-1040): a buffer type whose 2-D weight tensors are split by ROWS over the
// visible devices according to `tensor_split`; only MUL_MAT may consume them.  One process drives every device.  Each device's shard is
// allocated in init_tensor; set_tensor / get_tensor scatter / gather the row ranges.  The mat-mul itself (compute_mul_mat_split below):
// every device computes its rows on its own stream and the mat-vec kernel stores them straight into the main device's dst over NVLink
// (the fused gather of ggml-b200.h, here with the main device as the only "peer"), flags instead of events; batches (n > 1) go through a
// per-device staging buffer and a strided peer copy, ordered with events like the reference (:1333-1351, 1621-1647).
constexpr int64_t SPLIT_ROW_ROUNDING = 64;      // shard boundaries: multiples of 64 rows (every block format then starts 16-byte aligned)

struct split_buft_ctx {
    int         main_device = 0;
    float       split[B200_MAX_DEVICES] = {};   // cumulative start fractions per device index (position in the registry), like the reference
    std::string name;
};

struct split_tensor_extra {
    void *  data[B200_MAX_DEVICES] = {};        // row shard on registry device i (nullptr: no rows)
    int64_t row_low[B200_MAX_DEVICES] = {}, row_high[B200_MAX_DEVICES] = {};
};

struct split_buffer_ctx {
    std::vector<split_tensor_extra *> extras;
    ~split_buffer_ctx();
};

int registry_device_index(int i);               // CUDA ordinal of registry device i

split_buffer_ctx::~split_buffer_ctx() {
    for (split_tensor_extra * e : extras) {
        for (int i = 0; i < registry_device_count(); ++i)
            if (e->data[i]) { scoped_device sd(registry_device_index(i)); cudaFree(e->data[i]); }
        delete e;
    }
}

void split_rows(const split_buft_ctx * bc, const ggml_tensor * t, int i, int64_t * lo, int64_t * hi) {
    const int n = registry_device_count();
    const int64_t nrows = ggml_nrows(t);
    int64_t l = i == 0 ? 0 : (int64_t)(nrows * bc->split[i]);
    l -= l % SPLIT_ROW_ROUNDING;
    int64_t h;
    if (i == n - 1) h = nrows;
    else { h = (int64_t)(nrows * bc->split[i + 1]); h -= h % SPLIT_ROW_ROUNDING; }
    if (h < l) h = l;
    *lo = l; *hi = h;
}

const char * split_buft_get_name(ggml_backend_buffer_type_t buft) { return ((split_buft_ctx *) buft->context)->name.c_str(); }
bool buft_is_b200_split(ggml_backend_buffer_type_t buft) { return buft && buft->iface.get_name == split_buft_get_name; }
bool tensor_in_split_buffer(const ggml_tensor * t) { return t && t->buffer && buft_is_b200_split(t->buffer->buft); }

void split_buffer_free(ggml_backend_buffer_t buffer) { delete (split_buffer_ctx *) buffer->context; }
void * split_buffer_get_base(ggml_backend_buffer_t) { return (void *) 0x1000; }    // never dereferenced: the shards hang off tensor->extra

void split_buffer_init_tensor(ggml_backend_buffer_t buffer, ggml_tensor * tensor) {
    GGML_ASSERT(tensor->view_src == nullptr && "views of split tensors are not supported");
    split_buffer_ctx * ctx = (split_buffer_ctx *) buffer->context;
    const split_buft_ctx * bc = (const split_buft_ctx *) buffer->buft->context;
    split_tensor_extra * e = new split_tensor_extra;
    ctx->extras.push_back(e);
    for (int i = 0; i < registry_device_count(); ++i) {
        split_rows(bc, tensor, i, &e->row_low[i], &e->row_high[i]);
        const int64_t rows = e->row_high[i] - e->row_low[i];
        if (rows == 0) continue;
        scoped_device sd(registry_device_index(i));
        const size_t size = (size_t) rows * ggml_row_size(tensor->type, tensor->ne[0]);
        CUDA_OK(cudaMalloc(&e->data[i], size + 256));          // + 256: see buft_alloc_buffer
        CUDA_OK(cudaMemset((char *) e->data[i] + size, 0, 256));
    }
    tensor->extra = e;
}

void split_buffer_set_tensor(ggml_backend_buffer_t buffer, ggml_tensor * tensor, const void * data, size_t offset, size_t size) {
    GGML_ASSERT(offset == 0 && size == ggml_nbytes(tensor) && "split tensors are set in their entirety");
    (void) buffer;
    const split_tensor_extra * e = (const split_tensor_extra *) tensor->extra;
    const size_t rb = ggml_row_size(tensor->type, tensor->ne[0]);
    for (int i = 0; i < registry_device_count(); ++i) {
        if (!e->data[i]) continue;
        scoped_device sd(registry_device_index(i));
        CUDA_OK(cudaMemcpyAsync(e->data[i], (const char *) data + e->row_low[i] * rb, (size_t)(e->row_high[i] - e->row_low[i]) * rb, cudaMemcpyHostToDevice, cudaStreamPerThread));
    }
    for (int i = 0; i < registry_device_count(); ++i) {
        if (!e->data[i]) continue;
        scoped_device sd(registry_device_index(i));
        CUDA_OK(cudaStreamSynchronize(cudaStreamPerThread));
    }
}

void split_buffer_get_tensor(ggml_backend_buffer_t buffer, const ggml_tensor * tensor, void * data, size_t offset, size_t size) {
    GGML_ASSERT(offset == 0 && size == ggml_nbytes(tensor) && "split tensors are read in their entirety");
    (void) buffer;
    const split_tensor_extra * e = (const split_tensor_extra *) tensor->extra;
    const size_t rb = ggml_row_size(tensor->type, tensor->ne[0]);
    for (int i = 0; i < registry_device_count(); ++i) {
        if (!e->data[i]) continue;
        scoped_device sd(registry_device_index(i));
        CUDA_OK(cudaMemcpyAsync((char *) data + e->row_low[i] * rb, e->data[i], (size_t)(e->row_high[i] - e->row_low[i]) * rb, cudaMemcpyDeviceToHost, cudaStreamPerThread));
    }
    for (int i = 0; i < registry_device_count(); ++i) {
        if (!e->data[i]) continue;
        scoped_device sd(registry_device_index(i));
        CUDA_OK(cudaStreamSynchronize(cudaStreamPerThread));
    }
}
void split_buffer_clear(ggml_backend_buffer_t, uint8_t) {}

const ggml_backend_buffer_i k_split_buffer_iface = {
    /* .free_buffer   = */ split_buffer_free,
    /* .get_base      = */ split_buffer_get_base,
    /* .init_tensor   = */ split_buffer_init_tensor,
    /* .memset_tensor = */ nullptr,
    /* .set_tensor    = */ split_buffer_set_tensor,
    /* .get_tensor    = */ split_buffer_get_tensor,
    /* .cpy_tensor    = */ nullptr,
    /* .clear         = */ split_buffer_clear,
    /* .reset         = */ nullptr,
};

ggml_backend_buffer_t split_buft_alloc_buffer(ggml_backend_buffer_type_t buft, size_t size) {
    // the exact split is only known per tensor (rounding): the shards are allocated in init_tensor; `size` is the cumulative bound
    // that ggml-alloc enforces through get_alloc_size
    return ggml_backend_buffer_init(buft, k_split_buffer_iface, new split_buffer_ctx, size);
}
size_t split_buft_get_alloc_size(ggml_backend_buffer_type_t buft, const ggml_tensor * tensor) {
    const split_buft_ctx * bc = (const split_buft_ctx *) buft->context;
    size_t total = 0;
    for (int i = 0; i < registry_device_count(); ++i) {
        int64_t lo, hi;
        split_rows(bc, tensor, i, &lo, &hi);
        total += (size_t)(hi - lo) * ggml_row_size(tensor->type, tensor->ne[0]);
    }
    return total;
}
bool split_buft_is_host(ggml_backend_buffer_type_t) { return false; }

ggml_backend_buffer_type_t split_buffer_type(int main_device, const float * tensor_split) {
    static std::mutex mu;
    std::lock_guard<std::mutex> lock(mu);
    static std::vector<ggml_backend_buffer_type *> bufts;      // never freed, like every buffer type
    const int n = registry_device_count();
    if (n == 0) return nullptr;
    int main_index = -1;
    for (int i = 0; i < n; ++i) if (registry_device_index(i) == main_device) main_index = i;
    if (main_index < 0) { GGML_LOG_ERROR("ggml-b200: split buffer type: invalid main device %d\n", main_device); return nullptr; }
    float split[B200_MAX_DEVICES] = {};
    bool all_zero = tensor_split == nullptr;
    if (!all_zero) { all_zero = true; for (int i = 0; i < n; ++i) if (tensor_split[i] != 0.0f) all_zero = false; }
    if (all_zero) { for (int i = 0; i < n; ++i) split[i] = (float) i / (float) n; }          // B200s are identical: equal shares
    else {
        float sum = 0.0f;
        for (int i = 0; i < n; ++i) { split[i] = sum; sum += tensor_split[i]; }
        for (int i = 0; i < n; ++i) split[i] /= sum;
    }
    for (auto * b : bufts) {
        const split_buft_ctx * c = (const split_buft_ctx *) b->context;
        if (c->main_device == main_device && memcmp(c->split, split, sizeof(split)) == 0) return b;
    }
    split_buft_ctx * c = new split_buft_ctx;
    c->main_device = main_device;
    memcpy(c->split, split, sizeof(split));
    c->name = "B200" + std::to_string(main_device) + "_Split";
    ggml_backend_buffer_type * b = new ggml_backend_buffer_type{
        { split_buft_get_name, split_buft_alloc_buffer, buft_get_alignment, nullptr, split_buft_get_alloc_size, split_buft_is_host },
        ggml_backend_reg_dev_get(b200_reg(), (size_t) main_index), c };
    bufts.push_back(b);
    return b;
}

// ------------------------------------------------------------------------------------------ op support
bool is_b200_weight_type(ggml_type t) { return b200::is_block_type((int32_t) t); }

bool tensor_on_device(const ggml_tensor * t, int device) {
    ggml_backend_buffer_t buf = t->view_src ? t->view_src->buffer : t->buffer;
    if (!buf) return true;                       // not allocated yet: the scheduler decides placement
    if (!buffer_is_b200(buf)) return false;
    return ((buffer_ctx *) buf->context)->device == device;
}

bool supports_mul_mat(const ggml_tensor * op) {
    const ggml_tensor * a = op->src[0], * b = op->src[1];
    if (!is_b200_weight_type(a->type) || b->type != GGML_TYPE_F32 || op->type != GGML_TYPE_F32) return false;
    if (a->nb[0] != ggml_type_size(a->type) || b->nb[0] != sizeof(float)) return false;   // K is the contiguous dim
    if (!ggml_is_contiguous(op)) return false;
    if ((a->type == GGML_TYPE_Q4_K || a->type == GGML_TYPE_Q5_K) && ((a->nb[1] | a->nb[2] | a->nb[3]) & 15)) return false;
    if ((b->nb[1] | b->nb[2] | b->nb[3]) & 3) return false;
    return true;
}

bool supports_mul_mat_id(const ggml_tensor * op) {
    const ggml_tensor * as = op->src[0], * b = op->src[1], * ids = op->src[2];
    if (!is_b200_weight_type(as->type) || b->type != GGML_TYPE_F32 || ids->type != GGML_TYPE_I32 || op->type != GGML_TYPE_F32) return false;
    if (as->nb[0] != ggml_type_size(as->type) || b->nb[0] != sizeof(float) || ids->nb[0] != sizeof(int32_t)) return false;
    if (as->ne[3] != 1 || b->ne[3] != 1 || !ggml_is_contiguous(op)) return false;
    if ((as->type == GGML_TYPE_Q4_K || as->type == GGML_TYPE_Q5_K) && ((as->nb[1] | as->nb[2]) & 15)) return false;
    return true;
}

bool is_f32_contig(const ggml_tensor * t) { return t->type == GGML_TYPE_F32 && ggml_is_contiguous(t); }

ggml_b200_tensor desc(const ggml_tensor * t) {
    ggml_b200_tensor d;
    d.data = t->data; d.type = (int32_t) t->type;
    for (int i = 0; i < 4; ++i) { d.ne[i] = t->ne[i]; d.nb[i] = t->nb[i]; }
    return d;
}

int32_t bin_bcast_op(ggml_op op) { return op == GGML_OP_ADD ? 0 : op == GGML_OP_MUL ? 1 : op == GGML_OP_SUB ? 2 : 3; }

// the kernel constants of a ROPE node: op_params as ggml_rope_impl writes them (read back at ggml-cpu.c:9267-9279), derived with the CPU's
// own expressions
ggml_b200_rope_params rope_params(const ggml_tensor * node) {
    const int32_t * ip = (const int32_t *) node->op_params;
    float freq_base, freq_scale, ext_factor, attn_factor, beta_fast, beta_slow;
    memcpy(&freq_base, ip + 5, sizeof(float));   memcpy(&freq_scale, ip + 6, sizeof(float));
    memcpy(&ext_factor, ip + 7, sizeof(float));  memcpy(&attn_factor, ip + 8, sizeof(float));
    memcpy(&beta_fast, ip + 9, sizeof(float));   memcpy(&beta_slow, ip + 10, sizeof(float));
    ggml_b200_rope_params rp{};
    rp.n_dims = ip[1]; rp.mode = ip[2];
    memcpy(rp.sections, ip + 11, sizeof(rp.sections));
    rp.freq_scale = freq_scale; rp.ext_factor = ext_factor;
    rp.theta_scale = powf(freq_base, -2.0f / rp.n_dims);
    ggml_rope_yarn_corr_dims(rp.n_dims, ip[4], freq_base, beta_fast, beta_slow, rp.corr_dims);
    rp.mscale = attn_factor;
    if (ext_factor != 0.0f) rp.mscale *= 1.0f + 0.1f * logf(1.0f / freq_scale);
    return rp;
}

// the strides, paddings, dilations and form of an IM2COL node: op_params as ggml_im2col writes them (read back at ggml-cpu.c:9886-9892)
ggml_b200_im2col_params im2col_params(const ggml_tensor * node) {
    const int32_t * ip = (const int32_t *) node->op_params;
    ggml_b200_im2col_params p;
    p.s0 = ip[0]; p.s1 = ip[1]; p.p0 = ip[2]; p.p1 = ip[3]; p.d0 = ip[4]; p.d1 = ip[5]; p.is_2D = ip[6];
    return p;
}

// the kernel library's code for a UNARY node's function, -1 where it has no kernel
int unary_code(const ggml_tensor * node) {
    switch (ggml_get_unary_op(node)) {
        case GGML_UNARY_OP_GELU:       return GGML_B200_UNARY_GELU;
        case GGML_UNARY_OP_SILU:       return GGML_B200_UNARY_SILU;
        case GGML_UNARY_OP_RELU:       return GGML_B200_UNARY_RELU;
        case GGML_UNARY_OP_TANH:       return GGML_B200_UNARY_TANH;
        case GGML_UNARY_OP_NEG:        return GGML_B200_UNARY_NEG;
        case GGML_UNARY_OP_ABS:        return GGML_B200_UNARY_ABS;
        case GGML_UNARY_OP_GELU_QUICK: return GGML_B200_UNARY_GELU_QUICK;
        case GGML_UNARY_OP_SIGMOID:    return GGML_B200_UNARY_SIGMOID;
        case GGML_UNARY_OP_EXP:        return GGML_B200_UNARY_EXP;
        case GGML_UNARY_OP_STEP:       return GGML_B200_UNARY_STEP;
        default:                       return -1;
    }
}

// How each node becomes its launcher's arguments (every op but the quantized MUL_MAT / MUL_MAT_ID and the tensor-core f16 MUL_MAT, whose
// arguments are mul_mat_args / mul_mat_id_args / mul_mat_route below).  launch == false: only ask, for supports_op: the launcher's own check
// on these descriptors, plus what the launcher cannot see (ggml-cpu's own layout rules, and the layout of the bare pointers some launchers
// take); launch == true: launch on `stream`.  Returns the check's / the launcher's status code.
int bound_op(const ggml_tensor * node, bool launch, void * stream) {
    const ggml_tensor * a = node->src[0], * b = node->src[1];
    const auto verdict = [](bool ok) { return ok ? GGML_B200_OK : GGML_B200_EUNSUPPORTED; };
    if (!launch && !a) return GGML_B200_EUNSUPPORTED;      // every op below has a src0 (ARANGE and the like have none)
    switch (node->op) {
        case GGML_OP_GET_ROWS: {
            // the kernel reads src0's rows as packed elements; the C ABI leaves nb0 to its callers, a ggml view may permute dim 0
            if (!launch && a->nb[0] != ggml_type_size(a->type)) return GGML_B200_EUNSUPPORTED;
            const auto x = desc(a), i = desc(b), d = desc(node);
            return launch ? ggml_b200_op_get_rows(&x, &i, &d, stream) : b200::check_get_rows(&x, &i, &d).code;
        }
        case GGML_OP_ADD: case GGML_OP_MUL: case GGML_OP_SUB: case GGML_OP_DIV: {
            // the kernel wraps any src1 index; ggml-cpu broadcasts only whole repeats of src1
            if (!launch && !ggml_can_repeat(b, a)) return GGML_B200_EUNSUPPORTED;
            const auto x = desc(a), y = desc(b), d = desc(node);
            const int32_t op = bin_bcast_op(node->op);
            return launch ? ggml_b200_op_bin_bcast(op, &x, &y, &d, stream) : b200::check_bin_bcast(op, &x, &y, &d).code;
        }
        case GGML_OP_NORM: case GGML_OP_RMS_NORM: {
            const auto x = desc(a), d = desc(node);
            return launch ? ggml_b200_op_norm(node->op == GGML_OP_RMS_NORM, &x, &d, ggml_get_op_params_f32(node, 0), stream) : b200::check_norm(&x, &d).code;
        }
        case GGML_OP_CPY: case GGML_OP_CONT: case GGML_OP_DUP: {
            const ggml_tensor * dt = node->op == GGML_OP_CPY ? b : node;
            // ggml-cpu quantizes only into a contiguous destination
            if (!launch && (dt->type == GGML_TYPE_Q8_0 || dt->type == GGML_TYPE_Q4_0) && !ggml_is_contiguous(dt)) return GGML_B200_EUNSUPPORTED;
            const auto x = desc(a), y = desc(dt);
            return launch ? ggml_b200_op_cpy(&x, &y, stream) : b200::check_cpy(&x, &y).code;
        }
        case GGML_OP_FLASH_ATTN_EXT: {
            const ggml_tensor * k = node->src[1], * v = node->src[2], * mask = node->src[3];
            // the kernel reads K and V rows as packed elements; the C ABI leaves nb0 to its callers
            if (!launch && (k->nb[0] != ggml_type_size(k->type) || v->nb[0] != ggml_type_size(v->type))) return GGML_B200_EUNSUPPORTED;
            const auto q = desc(a), tk = desc(k), tv = desc(v), d = desc(node), tm = mask ? desc(mask) : ggml_b200_tensor{};
            if (!launch) return b200::check_flash_attn_ext(&q, &tk, &tv, mask ? &tm : nullptr, &d).code;
            return ggml_b200_op_flash_attn_ext(&q, &tk, &tv, mask ? &tm : nullptr, &d, ggml_get_op_params_f32(node, 0), ggml_get_op_params_f32(node, 1),
                                               ggml_get_op_params_f32(node, 2), stream);
        }
        case GGML_OP_MUL_MAT: {                            // the plain float kernel: mul_mat_route says which MUL_MAT nodes take it
            const auto x = desc(a), y = desc(b), d = desc(node);
            return launch ? ggml_b200_op_mul_mat_f(&x, &y, &d, stream) : b200::check_mul_mat_f(&x, &y, &d).code;
        }
        case GGML_OP_ROPE: {                               // GGML_OP_ROPE_BACK (training) stays declined
            const ggml_tensor * ff = node->src[2];
            const ggml_b200_rope_params rp = rope_params(node);
            const auto x = desc(a), p = desc(b), d = desc(node), f = ff ? desc(ff) : ggml_b200_tensor{};
            return launch ? ggml_b200_op_rope(&x, &p, ff ? &f : nullptr, &d, &rp, stream) : b200::check_rope(&x, &p, ff ? &f : nullptr, &d, &rp).code;
        }
        case GGML_OP_ARGSORT: {
            // ggml-cpu reads row i at i*nb01 (ggml-cpu.c:10765): only evenly spaced rows mean the same data on both backends
            if (!launch && (a->nb[2] != a->ne[1] * a->nb[1] || a->nb[3] != a->ne[2] * a->nb[2])) return GGML_B200_EUNSUPPORTED;
            const auto x = desc(a), d = desc(node);
            const int32_t order = ggml_get_op_params_i32(node, 0);
            return launch ? ggml_b200_op_argsort(&x, &d, order, stream) : b200::check_argsort(&x, &d, order).code;
        }
        case GGML_OP_SUM_ROWS: {
            const auto x = desc(a), d = desc(node);
            return launch ? ggml_b200_op_sum_rows(&x, &d, stream) : b200::check_sum_rows(&x, &d).code;
        }
        case GGML_OP_CONCAT: {
            const auto x = desc(a), y = desc(b), d = desc(node);
            const int32_t dim = ggml_get_op_params_i32(node, 0);
            return launch ? ggml_b200_op_concat(&x, &y, &d, dim, stream) : b200::check_concat(&x, &y, &d, dim).code;
        }
        case GGML_OP_SSM_CONV: {
            const auto x = desc(a), c = desc(b), d = desc(node);
            return launch ? ggml_b200_op_ssm_conv(&x, &c, &d, stream) : b200::check_ssm_conv(&x, &c, &d).code;
        }
        case GGML_OP_IM2COL: {                             // GGML_OP_IM2COL_BACK (training) stays declined
            const auto k = desc(a), x = desc(b), d = desc(node);
            const ggml_b200_im2col_params p = im2col_params(node);
            return launch ? ggml_b200_op_im2col(&k, &x, &d, &p, stream) : b200::check_im2col(&k, &x, &d, &p).code;
        }
        case GGML_OP_POOL_2D: {                            // GGML_OP_POOL_2D_BACK (training) stays declined
            // ggml-cpu steps from plane to plane by nb2 until ggml_nbytes(src) is used up (ggml-cpu.c:10336-10375): it reads the planes
            // the descriptors name only when they are evenly spaced and a plane's rows end within nb2
            if (!launch && ggml_nelements(a) > 0 && ((a->ne[3] > 1 && a->nb[3] != a->ne[2] * a->nb[2]) ||
                                                     (a->ne[1] - 1) * (int64_t) a->nb[1] + a->ne[0] * (int64_t) sizeof(float) > (int64_t) a->nb[2]))
                return GGML_B200_EUNSUPPORTED;
            const int32_t * ip = (const int32_t *) node->op_params;
            const ggml_b200_pool_params p = { ip[0], ip[1], ip[2], ip[3], ip[4], ip[5], ip[6] };
            const auto x = desc(a), d = desc(node);
            return launch ? ggml_b200_op_pool_2d(&x, &d, &p, stream) : b200::check_pool_2d(&x, &d, &p).code;
        }
        case GGML_OP_UPSCALE: {
            const auto x = desc(a), d = desc(node);
            return launch ? ggml_b200_op_upscale(&x, &d, stream) : b200::check_upscale(&x, &d).code;
        }
        case GGML_OP_LEAKY_RELU: {
            // ggml-cpu walks nrows rows at i*nb1 (ggml-cpu.c:6712-6716): only evenly spaced rows mean the same data on both backends
            if (!launch && (a->nb[2] != a->ne[1] * a->nb[1] || a->nb[3] != a->ne[2] * a->nb[2] ||
                            node->nb[2] != node->ne[1] * node->nb[1] || node->nb[3] != node->ne[2] * node->nb[2])) return GGML_B200_EUNSUPPORTED;
            const auto x = desc(a), d = desc(node);
            return launch ? ggml_b200_op_leaky_relu(&x, &d, ggml_get_op_params_f32(node, 0), stream) : b200::check_leaky_relu(&x, &d).code;
        }
        case GGML_OP_REPEAT: {
            const auto x = desc(a), d = desc(node);
            return launch ? ggml_b200_op_repeat(&x, &d, stream) : b200::check_repeat(&x, &d).code;
        }
        // the ops of SAM-style image encoders and mask decoders; ggml-cpu indexes all their operands as packed, and the checks require it
        case GGML_OP_WIN_PART: {
            const int32_t * ip = (const int32_t *) node->op_params;            // npx, npy, w (ggml_win_part)
            const auto x = desc(a), d = desc(node);
            return launch ? ggml_b200_op_win_part(&x, &d, ip[0], ip[1], ip[2], stream) : b200::check_win_part(&x, &d, ip[0], ip[1], ip[2]).code;
        }
        case GGML_OP_WIN_UNPART: {
            const int32_t w = ggml_get_op_params_i32(node, 0);
            const auto x = desc(a), d = desc(node);
            return launch ? ggml_b200_op_win_unpart(&x, &d, w, stream) : b200::check_win_unpart(&x, &d, w).code;
        }
        case GGML_OP_GET_REL_POS: {
            const auto x = desc(a), d = desc(node);
            return launch ? ggml_b200_op_get_rel_pos(&x, &d, stream) : b200::check_get_rel_pos(&x, &d).code;
        }
        case GGML_OP_ADD_REL_POS: {                        // sources: a, pw, ph; in place (op_params[0]) dst is a view of a
            const ggml_tensor * ph = node->src[2];
            if (!launch && (!b || !ph)) return GGML_B200_EUNSUPPORTED;
            const auto x = desc(a), w = desc(b), h = desc(ph), d = desc(node);
            return launch ? ggml_b200_op_add_rel_pos(&x, &w, &h, &d, stream) : b200::check_add_rel_pos(&x, &w, &h, &d).code;
        }
        case GGML_OP_CONV_TRANSPOSE_2D: {                  // sources: the kernel, the input; op_params[0] = stride
            if (!launch && !b) return GGML_B200_EUNSUPPORTED;
            const int32_t s = ggml_get_op_params_i32(node, 0);
            const auto k = desc(a), x = desc(b), d = desc(node);
            return launch ? ggml_b200_op_conv_transpose_2d(&k, &x, &d, s, stream) : b200::check_conv_transpose_2d(&k, &x, &d, s).code;
        }
        // the ops of ggml_opt's backward and optimizer graphs
        case GGML_OP_OUT_PROD: {
            if (!launch && !b) return GGML_B200_EUNSUPPORTED;
            const auto x = desc(a), y = desc(b), d = desc(node);
            return launch ? ggml_b200_op_out_prod(&x, &y, &d, stream) : b200::check_out_prod(&x, &y, &d).code;
        }
        case GGML_OP_CROSS_ENTROPY_LOSS: {
            // ggml-cpu walks nrows rows at i*nb1 (ggml-cpu.c:12484-12486): only evenly spaced rows mean the same data on both backends
            if (!launch && (!b || a->nb[2] != a->ne[1] * a->nb[1] || a->nb[3] != a->ne[2] * a->nb[2] ||
                            b->nb[2] != b->ne[1] * b->nb[1] || b->nb[3] != b->ne[2] * b->nb[2])) return GGML_B200_EUNSUPPORTED;
            const auto x = desc(a), l = desc(b), d = desc(node);
            return launch ? ggml_b200_op_cross_entropy_loss(&x, &l, &d, stream) : b200::check_cross_entropy_loss(&x, &l, &d).code;
        }
        case GGML_OP_CROSS_ENTROPY_LOSS_BACK: {            // sources: the loss's gradient, the logits, the labels
            const ggml_tensor * c = node->src[2];
            if (!launch && (!b || !c)) return GGML_B200_EUNSUPPORTED;
            const auto gr = desc(a), x = desc(b), l = desc(c), d = desc(node);
            return launch ? ggml_b200_op_cross_entropy_loss_back(&gr, &x, &l, &d, stream) : b200::check_cross_entropy_loss_back(&gr, &x, &l, &d).code;
        }
        case GGML_OP_OPT_STEP_ADAMW: {                     // sources: w, grad, m, v, params; dst is a view of w, updated in place
            const ggml_tensor * m = node->src[2], * v = node->src[3], * pr = node->src[4];
            if (!launch && (!b || !m || !v || !pr)) return GGML_B200_EUNSUPPORTED;
            // the kernel reads the hyper-parameters on the device: a source still in a host buffer (device_supports_op lets one through for
            // the scheduler to copy in) is an error here, never a read of a host pointer
            if (launch && !buffer_is_b200(pr->view_src ? pr->view_src->buffer : pr->buffer)) {
                GGML_LOG_ERROR("ggml-b200: OPT_STEP_ADAMW's hyper-parameters (%s) are not in a device buffer\n", pr->name);
                return GGML_B200_EINVAL;
            }
            const auto w = desc(node), gr = desc(b), tm = desc(m), tv = desc(v), tp = desc(pr);
            return launch ? ggml_b200_op_opt_step_adamw(&w, &gr, &tm, &tv, &tp, stream) : b200::check_opt_step_adamw(&w, &gr, &tm, &tv, &tp).code;
        }
        case GGML_OP_ARGMAX: {
            const auto x = desc(a), d = desc(node);
            return launch ? ggml_b200_op_argmax(&x, &d, stream) : b200::check_argmax(&x, &d).code;
        }
        case GGML_OP_COUNT_EQUAL: {
            if (!launch && !b) return GGML_B200_EUNSUPPORTED;
            const auto x = desc(a), y = desc(b), d = desc(node);
            return launch ? ggml_b200_op_count_equal(&x, &y, &d, stream) : b200::check_count_equal(&x, &y, &d).code;
        }
        case GGML_OP_SUM: {
            const auto x = desc(a), d = desc(node);
            return launch ? ggml_b200_op_sum(&x, &d, stream) : b200::check_sum(&x, &d).code;
        }
        case GGML_OP_REPEAT_BACK: {
            const auto x = desc(a), d = desc(node);
            return launch ? ggml_b200_op_repeat_back(&x, &d, stream) : b200::check_repeat_back(&x, &d).code;
        }
        case GGML_OP_SSM_SCAN: {
            // sources: s, x, dt, A, B, C (ggml_ssm_scan); dst = y, then the final states
            ggml_b200_tensor t[6];
            for (int k = 0; k < 6; ++k) t[k] = desc(node->src[k]);
            const auto d = desc(node);
            return launch ? ggml_b200_op_ssm_scan(&t[0], &t[1], &t[2], &t[3], &t[4], &t[5], &d, stream) : b200::check_ssm_scan(&t[0], &t[1], &t[2], &t[3], &t[4], &t[5], &d).code;
        }
        case GGML_OP_RWKV_WKV6: {
            // sources: k, v, r, tf, td, state (ggml_rwkv_wkv6); dst = y, then the final states
            ggml_b200_tensor t[6];
            for (int k = 0; k < 6; ++k) t[k] = desc(node->src[k]);
            const auto d = desc(node);
            return launch ? ggml_b200_op_rwkv_wkv6(&t[0], &t[1], &t[2], &t[3], &t[4], &t[5], &d, stream) : b200::check_rwkv_wkv6(&t[0], &t[1], &t[2], &t[3], &t[4], &t[5], &d).code;
        }
        case GGML_OP_GATED_LINEAR_ATTN: {
            // sources: k, v, q, g, state (ggml_gated_linear_attn); op_params[0] = scale
            ggml_b200_tensor t[5];
            for (int k = 0; k < 5; ++k) t[k] = desc(node->src[k]);
            const auto d = desc(node);
            if (!launch) return b200::check_gated_linear_attn(&t[0], &t[1], &t[2], &t[3], &t[4], &d).code;
            return ggml_b200_op_gated_linear_attn(&t[0], &t[1], &t[2], &t[3], &t[4], &d, ggml_get_op_params_f32(node, 0), stream);
        }
        // the launchers that take bare pointers: their layout conditions are the caller's
        case GGML_OP_SCALE:
            if (!launch) return verdict(is_f32_contig(a) && is_f32_contig(node));
            return ggml_b200_op_scale((const float *) a->data, (float *) node->data, ggml_get_op_params_f32(node, 0), ggml_nelements(node), stream);
        case GGML_OP_DIAG_MASK_INF:
            if (!launch) return verdict(is_f32_contig(a) && is_f32_contig(node));
            return ggml_b200_op_diag_mask_inf((const float *) a->data, (float *) node->data, node->ne[0], node->ne[1], ggml_nelements(node), ggml_get_op_params_i32(node, 0), stream);
        case GGML_OP_SOFT_MAX:
            if (!launch) return verdict(is_f32_contig(a) && is_f32_contig(node) && (!b || ((b->type == GGML_TYPE_F32 || b->type == GGML_TYPE_F16) && ggml_is_contiguous(b))));
            return ggml_b200_op_soft_max((const float *) a->data, b ? b->data : nullptr, b ? (int32_t) b->type : 0, (float *) node->data,
                                         node->ne[0], node->ne[1], node->ne[2], node->ne[3], ggml_get_op_params_f32(node, 0), ggml_get_op_params_f32(node, 1), stream);
        // SQR and SQRT: x * x and sqrtf, correctly rounded on both backends: bit-identical to ggml-cpu.  SIN and COS: the device's sinf / cosf
        // (within 2 ulp), not bit-identical to glibc's
        case GGML_OP_UNARY: case GGML_OP_SQR: case GGML_OP_SQRT: case GGML_OP_SIN: case GGML_OP_COS: {
            const int u = node->op == GGML_OP_SQR ? GGML_B200_UNARY_SQR : node->op == GGML_OP_SQRT ? GGML_B200_UNARY_SQRT
                        : node->op == GGML_OP_SIN ? GGML_B200_UNARY_SIN : node->op == GGML_OP_COS ? GGML_B200_UNARY_COS : unary_code(node);
            if (!launch) return verdict(u >= 0 && is_f32_contig(a) && is_f32_contig(node));
            return ggml_b200_op_unary(u, (const float *) a->data, (float *) node->data, ggml_nelements(node), stream);
        }
        default:
            if (!launch) return GGML_B200_EUNSUPPORTED;
            GGML_LOG_ERROR("ggml-b200: op %s is not supported (supports_op must have declined it)\n", ggml_op_desc(node));
            GGML_ABORT("unsupported op");
    }
}

bool device_supports_op(ggml_backend_dev_t dev, const ggml_tensor * op) {
    const int device = ((device_ctx *) dev->context)->index;
    // split buffers can only be used with GGML_OP_MUL_MAT (src0), on the buffer type's main device (ggml-cuda.cu:2944-2951)
    for (int i = 0; i < GGML_MAX_SRC; ++i) {
        if (!tensor_in_split_buffer(op->src[i])) continue;
        if (op->op != GGML_OP_MUL_MAT || i != 0) return false;
        if (((const split_buft_ctx *) op->src[i]->buffer->buft->context)->main_device != device) return false;
        const ggml_tensor * a = op->src[0], * b = op->src[1];
        if (a->ne[2] != 1 || a->ne[3] != 1 || b->ne[2] != 1 || b->ne[3] != 1 || !ggml_is_contiguous(a)) return false;
        return supports_mul_mat(op) && tensor_on_device(b, device);
    }
    // OPT_STEP_ADAMW's hyper-parameters live in a host buffer (ggml_opt rewrites them every step): ggml_backend_sched copies such a source
    // into this device before the split runs.  Only a host buffer is let through; a graph computed on this backend directly must hold them
    // on the device (the launch refuses a host tensor, bound_op)
    for (int i = 0; i < GGML_MAX_SRC; ++i) {
        if (!op->src[i] || tensor_on_device(op->src[i], device)) continue;
        const ggml_tensor * s = op->src[i]->view_src ? op->src[i]->view_src : op->src[i];
        if (!(op->op == GGML_OP_OPT_STEP_ADAMW && i == 4 && ggml_backend_buffer_is_host(s->buffer))) return false;
    }
    switch (op->op) {
        case GGML_OP_NONE: case GGML_OP_RESHAPE: case GGML_OP_VIEW: case GGML_OP_PERMUTE: case GGML_OP_TRANSPOSE:
            return true;
        // the quantized rule, else the float launcher's check.  Which float kernel runs (tensor cores or plain) is chosen at compute time
        // from the real pointers (mul_mat_route); acceptance cannot depend on `data`, which may not be allocated yet, and need not:
        // a node the tensor-core kernels do not take runs on the plain one
        case GGML_OP_MUL_MAT:    return supports_mul_mat(op) || bound_op(op, false, nullptr) == GGML_B200_OK;
        case GGML_OP_MUL_MAT_ID: return supports_mul_mat_id(op);
        default:                 return bound_op(op, false, nullptr) == GGML_B200_OK;
    }
}

bool device_supports_buft(ggml_backend_dev_t dev, ggml_backend_buffer_type_t buft) {
    if (buft_is_b200(buft) || buft_is_b200_split(buft)) return buft->device == dev;
    return false;
}

// the scheduler asks whether an op whose weights live in host memory is worth shipping over (ggml-cuda.cu:3241-3247)
bool device_offload_op(ggml_backend_dev_t, const ggml_tensor * op) {
    const int min_batch = 32;
    return (op->op == GGML_OP_MUL_MAT && op->ne[1] >= min_batch) || (op->op == GGML_OP_MUL_MAT_ID && op->ne[2] >= min_batch);
}

// ------------------------------------------------------------------------------------------ compute
bool is_noop(ggml_op op) { return op == GGML_OP_NONE || op == GGML_OP_RESHAPE || op == GGML_OP_VIEW || op == GGML_OP_PERMUTE || op == GGML_OP_TRANSPOSE; }

// May the mat-vec kernel start fetching src0 before the preceding kernel on the stream has finished?  Only for tensors that
// nothing in flight writes: a graph leaf that owns its memory, that no node of this cgraph writes through a view (ggml_cpy into it,
// in-place ops: their results are views whose view_src is the leaf), and, outside CUDA-graph capture, not for the first kernel of a
// cgraph (its predecessor on the stream belongs to an earlier graph_compute that may have written anything).  Buffers marked as
// weights by the application (ggml_backend_buffer_set_usage) qualify regardless of the position.
int src0_flags(const backend_ctx * ctx, const ggml_tensor * a) {
    if (a->op != GGML_OP_NONE || a->view_src != nullptr) return GGML_B200_MM_AUTO;
    if (ctx->written.count(a)) return GGML_B200_MM_AUTO;
    const bool weights = a->buffer && ggml_backend_buffer_get_usage(a->buffer) == GGML_BACKEND_BUFFER_USAGE_WEIGHTS;
    if (!weights && !ctx->capturing && ctx->first_real_node) return GGML_B200_MM_AUTO;
    return GGML_B200_MM_SRC0_STATIC;
}

// the kernel arguments of a MUL_MAT node (no workspace yet); the workspace query before a capture and the launch see the same shape
ggml_b200_mul_mat_args mul_mat_args(const ggml_tensor * node, int32_t flags) {
    const ggml_tensor * a = node->src[0], * b = node->src[1];
    ggml_b200_mul_mat_args args{};
    args.type = (int32_t) a->type;
    args.flags = flags;
    args.K = a->ne[0]; args.M = a->ne[1]; args.N = b->ne[1];
    args.ne02 = a->ne[2]; args.ne03 = a->ne[3]; args.ne12 = b->ne[2]; args.ne13 = b->ne[3];
    args.nb01 = a->nb[1]; args.nb02 = a->nb[2]; args.nb03 = a->nb[3];
    args.nb11 = b->nb[1]; args.nb12 = b->nb[2]; args.nb13 = b->nb[3];
    args.src0 = a->data; args.src1 = (const float *) b->data; args.dst = (float *) node->data;
    return args;
}

// the kernel arguments of a MUL_MAT_ID node (no workspace yet)
ggml_b200_mul_mat_id_args mul_mat_id_args(const ggml_tensor * node) {
    const ggml_tensor * as = node->src[0], * b = node->src[1], * ids = node->src[2];
    ggml_b200_mul_mat_id_args args{};
    args.type = (int32_t) as->type;
    args.K = as->ne[0]; args.M = as->ne[1]; args.n_expert = as->ne[2];
    args.n_used = ids->ne[0]; args.nb1cols = b->ne[1]; args.n_tok = b->ne[2];
    args.nb01 = as->nb[1]; args.nb02 = as->nb[2];
    args.nb11 = b->nb[1]; args.nb12 = b->nb[2];
    args.ids_nb1 = ids->nb[1];
    args.src0 = as->data; args.src1 = (const float *) b->data; args.ids = (const int32_t *) ids->data; args.dst = (float *) node->data;
    return args;
}

void compute_mul_mat(backend_ctx * ctx, const ggml_tensor * dst, size_t need) {
    ggml_b200_mul_mat_args args = mul_mat_args(dst, src0_flags(ctx, dst->src[0]));
    args.workspace = ctx->scratch(need);
    args.workspace_size = ctx->workspace_size;
    SHIM_OK(ggml_b200_mul_mat(&args, ctx->stream));
}

void compute_mul_mat_id(backend_ctx * ctx, const ggml_tensor * dst) {
    ggml_b200_mul_mat_id_args args = mul_mat_id_args(dst);
    const size_t need = ggml_b200_mul_mat_id_workspace_size(&args);
    args.workspace = ctx->scratch(need);
    args.workspace_size = ctx->workspace_size;
    SHIM_OK(ggml_b200_mul_mat_id(&args, ctx->stream));
}


// grow-only device allocation on the current device (split path only: never inside a stream capture)
void grow(void ** ptr, size_t * cap, size_t need) {
    if (need <= *cap) return;
    if (*ptr) CUDA_OK(cudaFree(*ptr));
    const size_t sz = (need + need / 4 + 4095) & ~(size_t) 4095;
    CUDA_OK(cudaMalloc(ptr, sz));
    *cap = sz;
}

// MUL_MAT whose weights live in a split buffer: every device computes its row range concurrently and delivers it into dst on the main
// device.  n = 1: the mat-vec kernel stores its rows into dst over NVLink itself and raises a flag (ggml_b200_mul_mat_gather with the
// main device as the only peer); the main stream then waits for the flags of all participating devices.  n > 1: result staged on the
// computing device, strided peer copy into dst, event.  Replaces ggml_cuda_op_mul_mat's split path (src/ggml-cuda/ggml-cuda.cu:1333-1647).
void compute_mul_mat_split(backend_ctx * ctx, const ggml_tensor * dst) {
    const ggml_tensor * a = dst->src[0], * b = dst->src[1];
    const split_tensor_extra * e = (const split_tensor_extra *) a->extra;
    GGML_ASSERT(e && "split tensor without shards (init_tensor not called?)");
    const int64_t K = a->ne[0], M = a->ne[1], N = b->ne[1];
    const size_t rb = ggml_row_size(a->type, K);
    const int ndev = registry_device_count();
    if (!ctx->split_fork) CUDA_OK(cudaEventCreateWithFlags(&ctx->split_fork, cudaEventDisableTiming));
    if (!ctx->split_flags) { CUDA_OK(cudaMalloc((void **) &ctx->split_flags, 256)); CUDA_OK(cudaMemset(ctx->split_flags, 0, 256)); CUDA_OK(cudaDeviceSynchronize()); }
    CUDA_OK(cudaEventRecord(ctx->split_fork, ctx->stream));           // everything dst / src1 depend on is ordered before this point

    const uint32_t epoch = ++ctx->split_epoch;
    auto shard_args = [&](int i) {
        ggml_b200_mul_mat_args args{};
        const int64_t rows = e->row_high[i] - e->row_low[i];
        args.type = (int32_t) a->type; args.flags = GGML_B200_MM_AUTO;
        args.K = K; args.M = rows; args.N = N;
        args.ne02 = args.ne03 = args.ne12 = args.ne13 = 1;
        args.nb01 = rb; args.nb02 = rb * rows; args.nb03 = rb * rows;
        args.src0 = e->data[i]; args.src1 = (const float *) b->data; args.dst = (float *) dst->data;
        args.nb11 = b->nb[1]; args.nb12 = b->nb[1] * N; args.nb13 = b->nb[1] * N;
        return args;
    };
    // fused delivery (n = 1) for all shards or for none: decided before anything is launched
    bool fused_all = N == 1;
    for (int i = 0; i < ndev && fused_all; ++i) {
        if (!e->data[i]) continue;
        ggml_b200_mul_mat_args args = shard_args(i);
        fused_all = ggml_b200_mul_mat_gather_supported(&args) != 0;
    }
    int j = 0;
    // other devices first (they fork off the main stream), the main device's own shard last
    for (int pass = 0; pass < 2; ++pass) {
        for (int i = 0; i < ndev; ++i) {
            if (!e->data[i]) continue;
            const int d = registry_device_index(i);
            const bool is_main = d == ctx->device;
            if ((pass == 0) == is_main) continue;
            const int64_t lo = e->row_low[i], rows = e->row_high[i] - lo;
            backend_ctx::split_peer & pr = ctx->peers[i];
            scoped_device sd(d);
            cudaStream_t st = ctx->stream;
            const float * x = (const float *) b->data;
            size_t nb11 = b->nb[1];
            if (!is_main) {
                if (!pr.stream) {
                    CUDA_OK(cudaStreamCreateWithFlags(&pr.stream, cudaStreamNonBlocking));
                    CUDA_OK(cudaEventCreateWithFlags(&pr.done, cudaEventDisableTiming));
                    SHIM_OK(ggml_b200_prepare());
                }
                if (!pr.peer_access) {
                    cudaError_t pe = cudaDeviceEnablePeerAccess(ctx->device, 0);                       // d -> main (dst, flags, src1)
                    if (pe != cudaSuccess && pe != cudaErrorPeerAccessAlreadyEnabled) CUDA_OK(pe);
                    cudaGetLastError();
                    { scoped_device sm(ctx->device); pe = cudaDeviceEnablePeerAccess(d, 0); if (pe != cudaSuccess && pe != cudaErrorPeerAccessAlreadyEnabled) CUDA_OK(pe); cudaGetLastError(); }
                    pr.peer_access = true;
                }
                st = pr.stream;
                CUDA_OK(cudaStreamWaitEvent(st, ctx->split_fork, 0));
                grow(&pr.x_stage, &pr.x_cap, (size_t) N * K * sizeof(float));
                CUDA_OK(cudaMemcpy2DAsync(pr.x_stage, (size_t) K * sizeof(float), b->data, b->nb[1], (size_t) K * sizeof(float), (size_t) N, cudaMemcpyDeviceToDevice, st));
                x = (const float *) pr.x_stage; nb11 = (size_t) K * sizeof(float);
            }
            ggml_b200_mul_mat_args args = shard_args(i);
            args.src1 = x; args.nb11 = nb11; args.nb12 = nb11 * N; args.nb13 = nb11 * N;
            if (fused_all) {
                ggml_b200_gather ga{};
                ga.world = 1; ga.rank = 0; ga.row_offset = lo; ga.epoch = epoch;
                ga.y_peers[0] = (float *) dst->data; ga.flag_peers[0] = ctx->split_flags + j;
                SHIM_OK(ggml_b200_mul_mat_gather(&args, &ga, st));
            } else {
                void ** ysp = &pr.y_stage; size_t * ycp = &pr.y_cap;
                grow(ysp, ycp, (size_t) N * rows * sizeof(float));
                args.dst = (float *) *ysp;
                const size_t need = ggml_b200_mul_mat_workspace_size(&args);
                if (is_main) { args.workspace = ctx->scratch(need); args.workspace_size = ctx->workspace_size; }
                else { grow(&pr.ws, &pr.ws_cap, need); args.workspace = pr.ws; args.workspace_size = pr.ws_cap; }
                SHIM_OK(ggml_b200_mul_mat(&args, st));
                CUDA_OK(cudaMemcpy2DAsync((float *) dst->data + lo, (size_t) M * sizeof(float), *ysp, (size_t) rows * sizeof(float), (size_t) rows * sizeof(float), (size_t) N,
                                          cudaMemcpyDeviceToDevice, st));
                if (!is_main) {
                    CUDA_OK(cudaEventRecord(pr.done, st));
                    scoped_device sm(ctx->device);
                    CUDA_OK(cudaStreamWaitEvent(ctx->stream, pr.done, 0));
                }
            }
            ++j;
        }
    }
    if (fused_all) {
        scoped_device sm(ctx->device);
        SHIM_OK(ggml_b200_gather_wait(ctx->split_flags, j, epoch, ctx->stream));        // every participating device has delivered its rows
    }
}

// ------------------------------------------------------------------------------------------ backend (stream)
const char * backend_get_name(ggml_backend_t backend) { return ((backend_ctx *) backend->context)->name.c_str(); }

void backend_free(ggml_backend_t backend) {
    backend_ctx * ctx = (backend_ctx *) backend->context;
    if (ctx->prof.calls[0] + ctx->prof.calls[1] + ctx->prof.calls[2] + ctx->prof.calls[3]) {
        static const char * mode_name[4] = { "replay", "capture+update", "eager", "uncached" };
        for (int m = 0; m < 4; ++m)
            if (ctx->prof.calls[m])
                fprintf(stderr, "ggml-b200 profile [%s] %-14s: %llu graph_compute calls, %.1f us host time per call, %.1f nodes per call\n", ctx->name.c_str(), mode_name[m],
                        (unsigned long long) ctx->prof.calls[m], ctx->prof.us[m] / (double) ctx->prof.calls[m], (double) ctx->prof.nodes[m] / (double) ctx->prof.calls[m]);
        static const char * io_name[3] = { "set_tensor", "get_tensor", "synchronize" };
        for (int k = 0; k < 3; ++k)
            if (g_io_prof.calls[k])
                fprintf(stderr, "ggml-b200 profile %-12s: %llu calls, %.1f us host time per call\n", io_name[k], (unsigned long long) g_io_prof.calls[k].load(),
                        (double) g_io_prof.ns[k].load() / 1e3 / (double) g_io_prof.calls[k].load());
    }
    {
        scoped_device sd(ctx->device);
        cudaStreamSynchronize(ctx->stream);
        for (auto & g : ctx->graphs) if (g.exec) cudaGraphExecDestroy(g.exec);
        if (ctx->copy_event) cudaEventDestroy(ctx->copy_event);
        if (ctx->split_fork) cudaEventDestroy(ctx->split_fork);
        if (ctx->split_flags) cudaFree(ctx->split_flags);
        for (int i = 0; i < B200_MAX_DEVICES; ++i) {
            backend_ctx::split_peer & pr = ctx->peers[i];
            if (!pr.stream && !pr.y_stage) continue;
            scoped_device sp(i < registry_device_count() ? registry_device_index(i) : ctx->device);
            if (pr.stream) { cudaStreamSynchronize(pr.stream); cudaStreamDestroy(pr.stream); }
            if (pr.done) cudaEventDestroy(pr.done);
            if (pr.x_stage) cudaFree(pr.x_stage);
            if (pr.y_stage) cudaFree(pr.y_stage);
            if (pr.ws) cudaFree(pr.ws);
        }
        if (ctx->workspace) cudaFreeAsync(ctx->workspace, ctx->stream);
        cudaStreamSynchronize(ctx->stream);
        cudaStreamDestroy(ctx->stream);
    }
    delete ctx;
    delete backend;
}

void backend_set_tensor_async(ggml_backend_t backend, ggml_tensor * tensor, const void * data, size_t offset, size_t size) {
    backend_ctx * ctx = (backend_ctx *) backend->context;
    scoped_device sd(ctx->device);
    CUDA_OK(cudaMemcpyAsync((char *) tensor->data + offset, data, size, cudaMemcpyHostToDevice, ctx->stream));
}
void backend_get_tensor_async(ggml_backend_t backend, const ggml_tensor * tensor, void * data, size_t offset, size_t size) {
    backend_ctx * ctx = (backend_ctx *) backend->context;
    scoped_device sd(ctx->device);
    CUDA_OK(cudaMemcpyAsync(data, (const char *) tensor->data + offset, size, cudaMemcpyDeviceToHost, ctx->stream));
}
// device-to-device copy between two B200 backends (same or different GPUs), asynchronous on both streams like the reference's
// (src/ggml-cuda/ggml-cuda.cu:2353-2414): enqueue on the source stream, make the destination stream wait for it
bool backend_cpy_tensor_async(ggml_backend_t backend_src, ggml_backend_t backend_dst, const ggml_tensor * src, ggml_tensor * dst) {
    if (!ggml_backend_is_b200(backend_src) || !ggml_backend_is_b200(backend_dst)) return false;
    ggml_backend_buffer_t sbuf = src->view_src ? src->view_src->buffer : src->buffer;
    ggml_backend_buffer_t dbuf = dst->view_src ? dst->view_src->buffer : dst->buffer;
    if (!buffer_is_b200(sbuf) || !buffer_is_b200(dbuf)) return false;
    backend_ctx * sctx = (backend_ctx *) backend_src->context, * dctx = (backend_ctx *) backend_dst->context;
    if (((buffer_ctx *) sbuf->context)->device != sctx->device || ((buffer_ctx *) dbuf->context)->device != dctx->device) return false;
    if (backend_src == backend_dst) {
        scoped_device sd(sctx->device);
        CUDA_OK(cudaMemcpyAsync(dst->data, src->data, ggml_nbytes(dst), cudaMemcpyDeviceToDevice, sctx->stream));
        return true;
    }
    {
        scoped_device sd(sctx->device);
        if (sctx->device == dctx->device) CUDA_OK(cudaMemcpyAsync(dst->data, src->data, ggml_nbytes(dst), cudaMemcpyDeviceToDevice, sctx->stream));
        else                              CUDA_OK(cudaMemcpyPeerAsync(dst->data, dctx->device, src->data, sctx->device, ggml_nbytes(dst), sctx->stream));
        if (!sctx->copy_event) CUDA_OK(cudaEventCreateWithFlags(&sctx->copy_event, cudaEventDisableTiming));
        CUDA_OK(cudaEventRecord(sctx->copy_event, sctx->stream));
    }
    scoped_device sd(dctx->device);
    CUDA_OK(cudaStreamWaitEvent(dctx->stream, sctx->copy_event, 0));
    return true;
}

void backend_synchronize(ggml_backend_t backend) {
    backend_ctx * ctx = (backend_ctx *) backend->context;
    scoped_device sd(ctx->device);
    io_timer tm(2);
    CUDA_OK(cudaStreamSynchronize(ctx->stream));
}

// Dense f16 weights with a batch on the tensor-core kernel (plain 2-D operands, rows 16-byte aligned): its workspace, 0 when the node is not
// one it takes.  src1 f32: the kernel's fp16 path.  src1 f16 (the conv mat-mul of ggml_conv_1d / _2d: src0 the IM2COL result, src1 the
// conv kernel): both operands read by TMA, so src1 too is 16-byte aligned with rows that do not overlap, and K % 64 == 0.
size_t f16_tensor_core_workspace(const ggml_tensor * node) {
    const ggml_tensor * a = node->src[0], * b = node->src[1];
    const bool tma_b = b->type == GGML_TYPE_F16;
    if (a->type != GGML_TYPE_F16 || (b->type != GGML_TYPE_F32 && !tma_b) || node->type != GGML_TYPE_F32) return 0;
    if (a->ne[2] != 1 || a->ne[3] != 1 || b->ne[2] != 1 || b->ne[3] != 1 || b->ne[1] < 9) return 0;
    if (a->nb[0] != 2 || b->nb[0] != (tma_b ? 2u : 4u) || (a->nb[1] % 16) != 0 || (b->nb[1] % (tma_b ? 16 : 4)) != 0) return 0;
    if (((uintptr_t) a->data % 16) != 0 || !ggml_is_contiguous(node)) return 0;
    if (tma_b && (a->nb[1] < 2 * (size_t) a->ne[0] || b->nb[1] < 2 * (size_t) b->ne[0] || ((uintptr_t) b->data % 16) != 0)) return 0;
    return tma_b ? ggml_b200_mul_mat_f16_f16_workspace_size(a->ne[1], b->ne[1], a->ne[0]) : ggml_b200_mul_mat_f16_workspace_size(a->ne[1], b->ne[1], a->ne[0]);
}

// The kernel family a MUL_MAT node runs on, first match in this order, and the scratch it needs.  Sizing the pool before a capture and the
// launch inside it read the same answer.  The tensor-core routes depend on the real data pointers: see device_supports_op.
enum class mm_route { split, quantized, f16_tc, f16_f16_tc, plain_f };
struct mm_choice { mm_route route; size_t workspace; };
mm_choice mul_mat_route(const ggml_tensor * node) {
    const ggml_tensor * a = node->src[0];
    if (tensor_in_split_buffer(a)) return { mm_route::split, 0 };             // per-device scratch: compute_mul_mat_split
    if (is_b200_weight_type(a->type)) {
        // the flags the launch will pass (SRC0_STATIC) select neither the kernel nor the workspace size
        const ggml_b200_mul_mat_args args = mul_mat_args(node, GGML_B200_MM_AUTO);
        return { mm_route::quantized, ggml_b200_mul_mat_workspace_size(&args) };
    }
    if (const size_t ws = f16_tensor_core_workspace(node)) return { node->src[1]->type == GGML_TYPE_F16 ? mm_route::f16_f16_tc : mm_route::f16_tc, ws };
    return { mm_route::plain_f, 0 };
}

size_t node_scratch_need(const ggml_tensor * node) {
    if (node->op == GGML_OP_MUL_MAT) return mul_mat_route(node).workspace;
    if (node->op == GGML_OP_MUL_MAT_ID) {
        const ggml_b200_mul_mat_id_args args = mul_mat_id_args(node);
        return ggml_b200_mul_mat_id_workspace_size(&args);
    }
    return 0;
}

bool is_row_vector_f32(const ggml_tensor * t, int64_t n) {      // a contiguous f32 [n] (bias / gain) tensor
    return t && t->type == GGML_TYPE_F32 && t->ne[0] == n && ggml_nelements(t) == n && t->nb[0] == sizeof(float);
}

// MUL_MAT (n = 1, quantized) [+ ADD bias [+ GELU]] -> one launch; returns the number of extra nodes consumed (0 = not fused)
int try_fuse_mul_mat(backend_ctx * ctx, ggml_cgraph * cgraph, int i) {
    ggml_tensor * mm = cgraph->nodes[i];
    if (i + 1 >= cgraph->n_nodes || mm->src[1]->ne[1] != 1 || ggml_nelements(mm) != mm->ne[0]) return 0;
    ggml_tensor * add = cgraph->nodes[i + 1];
    if (add->op != GGML_OP_ADD || add->src[0] != mm || !is_row_vector_f32(add->src[1], mm->ne[0]) || !is_f32_contig(add) || !ggml_are_same_shape(add, mm)) return 0;
    ggml_b200_epilogue ep{};
    ep.bias = (const float *) add->src[1]->data; ep.dst_bias = (float *) add->data;
    int consumed = 1;
    if (i + 2 < cgraph->n_nodes) {
        ggml_tensor * un = cgraph->nodes[i + 2];
        if (un->op == GGML_OP_UNARY && ggml_get_unary_op(un) == GGML_UNARY_OP_GELU && un->src[0] == add && is_f32_contig(un)) {
            ep.unary = 1; ep.dst_unary = (float *) un->data; consumed = 2;
        } else if (un->op == GGML_OP_ADD && is_f32_contig(un) && ggml_are_same_shape(un, mm) &&
                   ((un->src[0] == add && is_f32_contig(un->src[1]) && ggml_are_same_shape(un->src[1], mm)) ||
                    (un->src[1] == add && is_f32_contig(un->src[0]) && ggml_are_same_shape(un->src[0], mm)))) {
            // the skip connection: cur = (W.x + bias) + residual  (f32 addition commutes exactly)
            ep.unary = 2; ep.dst_unary = (float *) un->data; consumed = 2;
            ep.residual = (const float *) (un->src[0] == add ? un->src[1] : un->src[0])->data;
        }
    }
    const ggml_tensor * a = mm->src[0], * b = mm->src[1];
    // the fused kernel writes the ADD / GELU outputs while other CTAs may still be reading src1: if the allocator placed one of them
    // on src1's (already dead, when unfused) memory, the nodes must run one by one
    {
        const char * x0 = (const char *) b->data, * x1 = x0 + ggml_nbytes(b);
        auto overlaps = [&](const void * p) { const char * y0 = (const char *) p, * y1 = y0 + mm->ne[0] * sizeof(float); return p && y0 < x1 && x0 < y1; };
        if (overlaps(ep.dst_bias) || overlaps(ep.dst_unary) || overlaps(mm->data)) return 0;
    }
    const ggml_b200_mul_mat_args args = mul_mat_args(mm, src0_flags(ctx, a));
    const int rc = ggml_b200_mul_mat_fused(&args, &ep, ctx->stream);
    if (rc == GGML_B200_EUNSUPPORTED) return 0;              // shape not on the mat-vec kernel: run the nodes one by one
    SHIM_OK(rc);
    return consumed;
}

// NORM / RMS_NORM -> MUL(gain) -> ADD(bias) -> one launch
int try_fuse_norm(backend_ctx * ctx, ggml_cgraph * cgraph, int i) {
    ggml_tensor * nm = cgraph->nodes[i];
    if (i + 2 >= cgraph->n_nodes) return 0;
    ggml_tensor * mul = cgraph->nodes[i + 1], * add = cgraph->nodes[i + 2];
    const int64_t n = nm->ne[0];
    if (mul->op != GGML_OP_MUL || mul->src[0] != nm || !is_row_vector_f32(mul->src[1], n) || !ggml_are_same_shape(mul, nm)) return 0;
    if (add->op != GGML_OP_ADD || add->src[0] != mul || !is_row_vector_f32(add->src[1], n) || !ggml_are_same_shape(add, nm)) return 0;
    auto s = desc(nm->src[0]), d1 = desc(nm), d2 = desc(mul), d3 = desc(add);
    const float * gain = (const float *) mul->src[1]->data, * bias = (const float *) add->src[1]->data;
    if (!b200::check_norm_affine(&s, &d1, gain, &d2, bias, &d3).ok()) return 0;
    SHIM_OK(ggml_b200_op_norm_affine(nm->op == GGML_OP_RMS_NORM, &s, &d1, gain, &d2, bias, &d3, ggml_get_op_params_f32(nm, 0), ctx->stream));
    return 2;
}

// does any node other than `except` consume `t` (as a source or through a view)?
bool has_other_consumer(const ggml_cgraph * cgraph, const ggml_tensor * t, const ggml_tensor * except) {
    if (t->flags & GGML_TENSOR_FLAG_OUTPUT) return true;
    for (int j = 0; j < cgraph->n_nodes; ++j) {
        const ggml_tensor * n = cgraph->nodes[j];
        if (n == except) continue;
        if (n->view_src == t) return true;
        for (int k = 0; k < GGML_MAX_SRC; ++k) if (n->src[k] == t) return true;
    }
    return false;
}

// SCALE -> DIAG_MASK_INF -> SOFT_MAX (the attention-score chain of examples/gpt-2, main-backend.cpp:574-584) in one row pass.  The two
// intermediates are NOT materialised, so the chain is only fused when nothing else reads them.
int try_fuse_soft_max(backend_ctx * ctx, ggml_cgraph * cgraph, int i) {
    if (i + 2 >= cgraph->n_nodes) return 0;
    ggml_tensor * sc = cgraph->nodes[i], * dm = cgraph->nodes[i + 1], * sm = cgraph->nodes[i + 2];
    if (dm->op != GGML_OP_DIAG_MASK_INF || dm->src[0] != sc || sm->op != GGML_OP_SOFT_MAX || sm->src[0] != dm || sm->src[1] != nullptr) return 0;
    if (!is_f32_contig(sc->src[0]) || !is_f32_contig(sc) || !is_f32_contig(dm) || !is_f32_contig(sm)) return 0;
    if (ggml_get_op_params_f32(sm, 0) != 1.0f || ggml_get_op_params_f32(sm, 1) != 0.0f) return 0;
    const int n_past = ggml_get_op_params_i32(dm, 0);
    if (n_past < 0) return 0;
    if (has_other_consumer(cgraph, sc, dm) || has_other_consumer(cgraph, dm, sm)) return 0;
    SHIM_OK(ggml_b200_op_soft_max_diag((const float *) sc->src[0]->data, nullptr, 0, (float *) sm->data, sm->ne[0], sm->ne[1], sm->ne[2], sm->ne[3],
                                       ggml_get_op_params_f32(sc, 0), 0.0f, n_past, ctx->stream));
    return 2;
}

// two consecutive float CPY nodes of the same size (the K and V cache updates of a layer) -> one launch
int try_fuse_cpy2(backend_ctx * ctx, ggml_cgraph * cgraph, int i) {
    if (i + 1 >= cgraph->n_nodes) return 0;
    ggml_tensor * c0 = cgraph->nodes[i], * c1 = cgraph->nodes[i + 1];
    if (c1->op != GGML_OP_CPY) return 0;
    auto s0 = desc(c0->src[0]), d0 = desc(c0->src[1]), s1 = desc(c1->src[0]), d1 = desc(c1->src[1]);
    if (!b200::check_cpy2(&s0, &d0, &s1, &d1).ok()) return 0;
    // independent: the second copy must neither read nor write what the first writes (byte spans of the possibly strided views)
    auto overlap = [](const ggml_tensor * a, const ggml_tensor * b) {
        const char * a0 = (const char *) a->data, * b0 = (const char *) b->data;
        return a0 < b0 + ggml_nbytes(b) && b0 < a0 + ggml_nbytes(a);
    };
    if (overlap(c1->src[0], c0->src[1]) || overlap(c1->src[1], c0->src[1]) || overlap(c1->src[1], c0->src[0])) return 0;
    SHIM_OK(ggml_b200_op_cpy2(&s0, &d0, &s1, &d1, ctx->stream));
    return 1;
}

// the multi-node launch that starts at node i, if there is one: returns the number of extra nodes consumed (0 = launch node i on its own)
int try_fuse(backend_ctx * ctx, ggml_cgraph * cgraph, int i) {
    static const bool fuse = !(getenv("GGML_B200_DISABLE_FUSION") && atoi(getenv("GGML_B200_DISABLE_FUSION")) != 0);
    if (!fuse) return 0;
    const ggml_tensor * node = cgraph->nodes[i];
    switch (node->op) {
        case GGML_OP_MUL_MAT:                       // only the quantized mat-vec has an epilogue
            return !tensor_in_split_buffer(node->src[0]) && is_b200_weight_type(node->src[0]->type) ? try_fuse_mul_mat(ctx, cgraph, i) : 0;
        case GGML_OP_NORM: case GGML_OP_RMS_NORM: return try_fuse_norm(ctx, cgraph, i);
        case GGML_OP_SCALE:                       return try_fuse_soft_max(ctx, cgraph, i);
        case GGML_OP_CPY:                         return try_fuse_cpy2(ctx, cgraph, i);
        default:                                  return 0;
    }
}

void compute_nodes(backend_ctx * ctx, ggml_cgraph * cgraph) {
    ctx->written.clear();
    for (int i = 0; i < cgraph->n_nodes; ++i) {
        const ggml_tensor * node = cgraph->nodes[i];
        if (node->view_src && !is_noop(node->op)) ctx->written.insert(node->view_src);
    }
    ctx->first_real_node = true;
    for (int i = 0; i < cgraph->n_nodes; ++i) {
        ggml_tensor * node = cgraph->nodes[i];
        if (ggml_is_empty(node)) continue;
        if (is_noop(node->op)) continue;
        struct not_first { backend_ctx * c; ~not_first() { c->first_real_node = false; } } nf{ ctx };
        const int extra = try_fuse(ctx, cgraph, i);
        if (extra > 0) { i += extra; continue; }
        switch (node->op) {
            case GGML_OP_MUL_MAT: {
                const ggml_tensor * a = node->src[0], * b = node->src[1];
                const mm_choice mm = mul_mat_route(node);
                switch (mm.route) {
                    case mm_route::split:     compute_mul_mat_split(ctx, node); break;
                    case mm_route::quantized: compute_mul_mat(ctx, node, mm.workspace); break;
                    case mm_route::f16_tc: {
                        void * ws = ctx->scratch(mm.workspace);
                        SHIM_OK(ggml_b200_mul_mat_f16(a->data, a->nb[1], (const float *) b->data, b->nb[1], (float *) node->data, a->ne[1], b->ne[1], a->ne[0], ws, ctx->workspace_size,
                                                      src0_flags(ctx, a), ctx->stream));
                    } break;
                    case mm_route::f16_f16_tc: {
                        void * ws = ctx->scratch(mm.workspace);
                        SHIM_OK(ggml_b200_mul_mat_f16_f16(a->data, a->nb[1], b->data, b->nb[1], (float *) node->data, a->ne[1], b->ne[1], a->ne[0], ws, ctx->workspace_size,
                                                          src0_flags(ctx, a), ctx->stream));
                    } break;
                    case mm_route::plain_f:   SHIM_OK(bound_op(node, true, ctx->stream)); break;
                }
            } break;
            case GGML_OP_MUL_MAT_ID: compute_mul_mat_id(ctx, node); break;
            default: SHIM_OK(bound_op(node, true, ctx->stream)); break;
        }
    }
}

// everything a captured launch sequence depends on: per node the op, type, shape, strides, data pointer, op parameters and the
// same for its sources (a changed source pointer or view offset changes the kernels' arguments)
void graph_signature(const ggml_cgraph * cgraph, std::vector<uint64_t> & sig) {
    sig.clear();
    sig.reserve((size_t) cgraph->n_nodes * 24);
    auto put_tensor = [&](const ggml_tensor * t) {
        sig.push_back(((uint64_t) t->op << 32) | (uint64_t) t->type);
        sig.push_back((uint64_t)(uintptr_t) t->data);
        for (int d = 0; d < 4; ++d) { sig.push_back((uint64_t) t->ne[d]); sig.push_back((uint64_t) t->nb[d]); }
    };
    for (int i = 0; i < cgraph->n_nodes; ++i) {
        const ggml_tensor * node = cgraph->nodes[i];
        if (is_noop(node->op)) continue;
        put_tensor(node);
        sig.push_back((uint64_t)(uintptr_t) node->view_src);
        const uint64_t * op = (const uint64_t *) node->op_params;
        for (size_t w = 0; w < sizeof(node->op_params) / sizeof(uint64_t); ++w) sig.push_back(op[w]);
        for (int j = 0; j < GGML_MAX_SRC; ++j) {
            if (!node->src[j]) { sig.push_back(0); continue; }
            put_tensor(node->src[j]);
            // weights marked by the application change the launch flags (src0_flags)
            sig.push_back(node->src[j]->buffer ? (uint64_t) ggml_backend_buffer_get_usage(node->src[j]->buffer) : 0);
        }
    }
}

static ggml_status graph_compute_impl(backend_ctx * ctx, ggml_cgraph * cgraph, int & mode, int & n_real_out) {
    static const bool graphs_off = getenv("GGML_B200_DISABLE_GRAPHS") && atoi(getenv("GGML_B200_DISABLE_GRAPHS")) != 0;
    int n_real = 0;
    bool has_split = false;        // multi-device work is not captured (the reference disables CUDA graphs for split buffers too, ggml-cuda.cu:2620)
    for (int i = 0; i < cgraph->n_nodes; ++i) {
        n_real += !is_noop(cgraph->nodes[i]->op);
        has_split = has_split || tensor_in_split_buffer(cgraph->nodes[i]->src[0]);
    }
    n_real_out = n_real;
    const bool use_graph = !graphs_off && !has_split && n_real >= 8 && ctx->graph_calls++ > 0;
    if (!use_graph) {
        mode = 3;
        compute_nodes(ctx, cgraph);
        return GGML_STATUS_SUCCESS;
    }
    constexpr size_t MAX_CACHED = 4;
    static thread_local std::vector<uint64_t> sig;
    graph_signature(cgraph, sig);
    ctx->graph_clock++;
    for (auto & g : ctx->graphs) {
        if (g.sig == sig) {                                        // unchanged graph: replay, no capture
            g.last_use = ctx->graph_clock;
            ctx->consecutive_updates = 0;
            ctx->last_sig = sig;
            mode = 0;
            CUDA_OK(cudaGraphLaunch(g.exec, ctx->stream));
            return GGML_STATUS_SUCCESS;
        }
    }
    static const int max_updates = getenv("GGML_B200_GRAPH_MAX_UPDATES") ? atoi(getenv("GGML_B200_GRAPH_MAX_UPDATES")) : 3;
    const bool repeated = sig == ctx->last_sig;                    // the same graph twice in a row: worth capturing (again)
    ctx->last_sig = sig;
    if (repeated) ctx->consecutive_updates = 0;
    else if (++ctx->consecutive_updates > max_updates) {
        mode = 2;
        compute_nodes(ctx, cgraph);                                // ever-changing graph: direct launches
        return GGML_STATUS_SUCCESS;
    }
    mode = 1;
    // size the scratch pool before capturing (allocation is not part of the graph)
    size_t need = 0;
    for (int i = 0; i < cgraph->n_nodes; ++i) { const size_t n = node_scratch_need(cgraph->nodes[i]); if (n > need) need = n; }
    ctx->scratch(need);
    cudaGraph_t graph = nullptr;
    // relaxed mode, as the reference (ggml-cuda.cu:2700): other threads of the process may call unrelated CUDA APIs meanwhile
    CUDA_OK(cudaStreamBeginCapture(ctx->stream, cudaStreamCaptureModeRelaxed));
    ctx->capturing = true;
    compute_nodes(ctx, cgraph);
    ctx->capturing = false;
    CUDA_OK(cudaStreamEndCapture(ctx->stream, &graph));
    // victim: a free slot, else the least recently used entry; prefer updating an executable graph of the same length in place
    backend_ctx::cached_graph * slot = nullptr;
    for (auto & g : ctx->graphs) if (g.sig.size() == sig.size() && (!slot || g.last_use < slot->last_use)) slot = &g;
    if (!slot && ctx->graphs.size() < MAX_CACHED) { ctx->graphs.emplace_back(); slot = &ctx->graphs.back(); }
    if (!slot) for (auto & g : ctx->graphs) if (!slot || g.last_use < slot->last_use) slot = &g;
    // a same-length entry is only overwritten when the cache is full or it is the token-by-token case (one live graph per shape)
    if (slot->exec) {
        cudaGraphExecUpdateResultInfo info;
        if (cudaGraphExecUpdate(slot->exec, graph, &info) != cudaSuccess) {              // topology changed: re-instantiate
            cudaGetLastError();
            CUDA_OK(cudaGraphExecDestroy(slot->exec));
            slot->exec = nullptr;
        }
    }
    if (!slot->exec) CUDA_OK(cudaGraphInstantiate(&slot->exec, graph, 0));
    CUDA_OK(cudaGraphDestroy(graph));
    slot->sig = sig;
    slot->last_use = ctx->graph_clock;
    CUDA_OK(cudaGraphLaunch(slot->exec, ctx->stream));
    return GGML_STATUS_SUCCESS;
}

ggml_status backend_graph_compute(ggml_backend_t backend, ggml_cgraph * cgraph) {
    backend_ctx * ctx = (backend_ctx *) backend->context;
    scoped_device sd(ctx->device);
    int mode = 3, n_real = 0;
    if (!profile_on()) return graph_compute_impl(ctx, cgraph, mode, n_real);
    const auto t0 = std::chrono::steady_clock::now();
    const ggml_status st = graph_compute_impl(ctx, cgraph, mode, n_real);
    const double us = std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - t0).count();
    ctx->prof.calls[mode]++; ctx->prof.us[mode] += us; ctx->prof.nodes[mode] += (uint64_t) n_real;
    return st;
}

void backend_event_record(ggml_backend_t backend, ggml_backend_event_t event) {
    backend_ctx * ctx = (backend_ctx *) backend->context;
    scoped_device sd(ctx->device);
    CUDA_OK(cudaEventRecord((cudaEvent_t) event->context, ctx->stream));
}
void backend_event_wait(ggml_backend_t backend, ggml_backend_event_t event) {
    backend_ctx * ctx = (backend_ctx *) backend->context;
    scoped_device sd(ctx->device);
    CUDA_OK(cudaStreamWaitEvent(ctx->stream, (cudaEvent_t) event->context, 0));
}

const ggml_backend_i k_backend_iface = {
    /* .get_name           = */ backend_get_name,
    /* .free               = */ backend_free,
    /* .set_tensor_async   = */ backend_set_tensor_async,
    /* .get_tensor_async   = */ backend_get_tensor_async,
    /* .cpy_tensor_async   = */ backend_cpy_tensor_async,
    /* .synchronize        = */ backend_synchronize,
    /* .graph_plan_create  = */ nullptr,
    /* .graph_plan_free    = */ nullptr,
    /* .graph_plan_update  = */ nullptr,
    /* .graph_plan_compute = */ nullptr,
    /* .graph_compute      = */ backend_graph_compute,
    /* .event_record       = */ backend_event_record,
    /* .event_wait         = */ backend_event_wait,
};

// ------------------------------------------------------------------------------------------ device
const char * device_get_name(ggml_backend_dev_t dev) { return ((device_ctx *) dev->context)->name.c_str(); }
const char * device_get_description(ggml_backend_dev_t dev) { return ((device_ctx *) dev->context)->description.c_str(); }
void device_get_memory(ggml_backend_dev_t dev, size_t * free, size_t * total) {
    scoped_device sd(((device_ctx *) dev->context)->index);
    CUDA_OK(cudaMemGetInfo(free, total));
}
enum ggml_backend_dev_type device_get_type(ggml_backend_dev_t) { return GGML_BACKEND_DEVICE_TYPE_GPU; }
void device_get_props(ggml_backend_dev_t dev, ggml_backend_dev_props * props) {
    props->name = device_get_name(dev);
    props->description = device_get_description(dev);
    props->type = GGML_BACKEND_DEVICE_TYPE_GPU;
    device_get_memory(dev, &props->memory_free, &props->memory_total);
    props->caps = { /* .async = */ true, /* .host_buffer = */ true, /* .buffer_from_host_ptr = */ false, /* .events = */ true };
}
ggml_backend_t device_init_backend(ggml_backend_dev_t dev, const char *) {
    return ggml_backend_b200_init(((device_ctx *) dev->context)->index);
}
ggml_backend_buffer_type_t device_get_buffer_type(ggml_backend_dev_t dev) { return &((device_ctx *) dev->context)->buft; }
ggml_backend_buffer_type_t device_get_host_buffer_type(ggml_backend_dev_t) { return host_buffer_type(); }

ggml_backend_event_t device_event_new(ggml_backend_dev_t dev) {
    scoped_device sd(((device_ctx *) dev->context)->index);
    cudaEvent_t ev;
    CUDA_OK(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    return new ggml_backend_event{ dev, ev };
}
void device_event_free(ggml_backend_dev_t, ggml_backend_event_t event) {
    CUDA_OK(cudaEventDestroy((cudaEvent_t) event->context));
    delete event;
}
void device_event_synchronize(ggml_backend_dev_t, ggml_backend_event_t event) { CUDA_OK(cudaEventSynchronize((cudaEvent_t) event->context)); }

const ggml_backend_device_i k_device_iface = {
    /* .get_name             = */ device_get_name,
    /* .get_description      = */ device_get_description,
    /* .get_memory           = */ device_get_memory,
    /* .get_type             = */ device_get_type,
    /* .get_props            = */ device_get_props,
    /* .init_backend         = */ device_init_backend,
    /* .get_buffer_type      = */ device_get_buffer_type,
    /* .get_host_buffer_type = */ device_get_host_buffer_type,
    /* .buffer_from_host_ptr = */ nullptr,
    /* .supports_op          = */ device_supports_op,
    /* .supports_buft        = */ device_supports_buft,
    /* .offload_op           = */ device_offload_op,
    /* .event_new            = */ device_event_new,
    /* .event_free           = */ device_event_free,
    /* .event_synchronize    = */ device_event_synchronize,
};

// ------------------------------------------------------------------------------------------ registry
struct reg_ctx {
    std::vector<ggml_backend_device *> devices;
};

const char * reg_get_name(ggml_backend_reg_t) { return "B200"; }
size_t reg_get_device_count(ggml_backend_reg_t reg) { return ((reg_ctx *) reg->context)->devices.size(); }
ggml_backend_dev_t reg_get_device(ggml_backend_reg_t reg, size_t index) {
    reg_ctx * ctx = (reg_ctx *) reg->context;
    GGML_ASSERT(index < ctx->devices.size());
    return ctx->devices[index];
}
ggml_backend_buffer_type_t split_buffer_type_entry(int main_device, const float * tensor_split) { return split_buffer_type(main_device, tensor_split); }
void * reg_get_proc_address(ggml_backend_reg_t, const char * name) {
    // the well-known name llama.cpp-style callers look up (include/ggml-backend.h:187-200; reference: ggml-cuda.cu:3374-3380)
    if (strcmp(name, "ggml_backend_split_buffer_type") == 0) return (void *) split_buffer_type_entry;
    if (strcmp(name, "ggml_backend_b200_launch_count") == 0) return (void *) ggml_b200_launch_count;
    return nullptr;
}

ggml_backend_reg_t b200_reg() {
    static ggml_backend_reg reg;
    static std::once_flag once;
    std::call_once(once, [] {
        reg_ctx * ctx = new reg_ctx;
        int n = 0;
        if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); n = 0; }
        if (n > B200_MAX_DEVICES) n = B200_MAX_DEVICES;
        for (int i = 0; i < n; ++i) {
            cudaDeviceProp prop;
            if (cudaGetDeviceProperties(&prop, i) != cudaSuccess) { cudaGetLastError(); continue; }
            if (prop.major != 9) {    // sm_90a binaries only load on Hopper (H100 / H200)
                GGML_LOG_WARN("ggml-b200: skipping device %d (%s, sm_%d%d): kernels are built for sm_90a\n", i, prop.name, prop.major, prop.minor);
                continue;
            }
            device_ctx * dctx = new device_ctx;
            dctx->index = i;
            dctx->name = "B200" + std::to_string(i);
            dctx->description = prop.name;
            dctx->buft_name = dctx->name;
            ggml_backend_device * dev = new ggml_backend_device{ k_device_iface, &reg, dctx };
            dctx->buft = ggml_backend_buffer_type{ k_buft_iface, dev, nullptr };
            ctx->devices.push_back(dev);
        }
        reg = ggml_backend_reg{ GGML_BACKEND_API_VERSION, { reg_get_name, reg_get_device_count, reg_get_device, reg_get_proc_address }, ctx };
    });
    return &reg;
}

int registry_device_count() { return (int) ((reg_ctx *) b200_reg()->context)->devices.size(); }
int registry_device_index(int i) { return ((device_ctx *) ((reg_ctx *) b200_reg()->context)->devices[(size_t) i]->context)->index; }

} // namespace

// ============================================================================================ exported C ABI
extern "C" {

GGML_B200_API ggml_backend_reg_t ggml_backend_b200_reg(void) { return b200_reg(); }

GGML_B200_API ggml_backend_t ggml_backend_b200_init(int device) {
    ggml_backend_reg_t reg = b200_reg();
    reg_ctx * rctx = (reg_ctx *) reg->context;
    ggml_backend_device * dev = nullptr;
    for (auto * d : rctx->devices) if (((device_ctx *) d->context)->index == device) dev = d;
    if (!dev) {
        GGML_LOG_ERROR("ggml-b200: invalid device %d\n", device);
        return nullptr;
    }
    backend_ctx * ctx = new backend_ctx;
    ctx->device = device;
    ctx->name = ((device_ctx *) dev->context)->name;
    {
        scoped_device sd(device);
        CUDA_OK(cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking));
        SHIM_OK(ggml_b200_prepare());       // per-device control block of the kernels: allocated here, never inside a stream capture
    }
    return new ggml_backend{ b200_guid(), k_backend_iface, dev, ctx };
}

GGML_B200_API bool ggml_backend_is_b200(ggml_backend_t backend) { return backend != nullptr && ggml_guid_matches(backend->guid, b200_guid()); }
GGML_B200_API ggml_backend_buffer_type_t ggml_backend_b200_buffer_type(int device) {
    reg_ctx * rctx = (reg_ctx *) b200_reg()->context;
    for (auto * d : rctx->devices) if (((device_ctx *) d->context)->index == device) return &((device_ctx *) d->context)->buft;
    return nullptr;
}
GGML_B200_API ggml_backend_buffer_type_t ggml_backend_b200_host_buffer_type(void) { return host_buffer_type(); }
GGML_B200_API int ggml_backend_b200_get_device_count(void) { return (int) ((reg_ctx *) b200_reg()->context)->devices.size(); }

// dynamic loading (src/ggml-backend-reg.cpp:220-263): ggml_backend_load(path) / $GGML_BACKEND_PATH
GGML_B200_API ggml_backend_reg_t ggml_backend_init(void) { return b200_reg(); }
GGML_B200_API int ggml_backend_score(void) { return ggml_backend_b200_get_device_count() > 0 ? 100 : 0; }

// include/ggml-cuda.h:23-45 — the symbols the examples bind when compiled with -DGGML_USE_CUDA
// (examples/gpt-2/main-backend.cpp:203-211, main-sched.cpp:115-123, tests/test-mul-mat.cpp:50-58)
GGML_B200_API ggml_backend_t ggml_backend_cuda_init(int device) { return ggml_backend_b200_init(device); }
GGML_B200_API bool ggml_backend_is_cuda(ggml_backend_t backend) { return ggml_backend_is_b200(backend); }
GGML_B200_API ggml_backend_buffer_type_t ggml_backend_cuda_buffer_type(int device) { return ggml_backend_b200_buffer_type(device); }
GGML_B200_API ggml_backend_buffer_type_t ggml_backend_b200_split_buffer_type(int main_device, const float * tensor_split) { return split_buffer_type(main_device, tensor_split); }
GGML_B200_API ggml_backend_buffer_type_t ggml_backend_cuda_split_buffer_type(int main_device, const float * tensor_split) { return split_buffer_type(main_device, tensor_split); }
GGML_B200_API ggml_backend_buffer_type_t ggml_backend_cuda_host_buffer_type(void) { return host_buffer_type(); }
GGML_B200_API int ggml_backend_cuda_get_device_count(void) { return ggml_backend_b200_get_device_count(); }
GGML_B200_API void ggml_backend_cuda_get_device_description(int device, char * description, size_t description_size) {
    cudaDeviceProp prop;
    CUDA_OK(cudaGetDeviceProperties(&prop, device));
    snprintf(description, description_size, "%s", prop.name);
}
GGML_B200_API void ggml_backend_cuda_get_device_memory(int device, size_t * free, size_t * total) {
    scoped_device sd(device);
    CUDA_OK(cudaMemGetInfo(free, total));
}
GGML_B200_API bool ggml_backend_cuda_register_host_buffer(void * buffer, size_t size) {
    if (cudaHostRegister(buffer, size, cudaHostRegisterPortable | cudaHostRegisterReadOnly) != cudaSuccess) { cudaGetLastError(); return false; }
    return true;
}
GGML_B200_API void ggml_backend_cuda_unregister_host_buffer(void * buffer) {
    if (cudaHostUnregister(buffer) != cudaSuccess) cudaGetLastError();
}
GGML_B200_API ggml_backend_reg_t ggml_backend_cuda_reg(void) { return b200_reg(); }

} // extern "C"
