// oracle/probe_harness.h — TEST INFRASTRUCTURE ONLY.
//
// What the op probes (attn_probe.cpp, conv_probe.cpp, core_probe.cpp, grad_probe.cpp, moe_probe.cpp, pool_probe.cpp, rope_probe.cpp,
// sam_probe.cpp, ssm_probe.cpp, train_probe.cpp, wkv_probe.cpp) share: the context their graph lives in, the view-of-a-parent source of
// oracle/pool.py's Source, and the run of that graph on a named device.  A probe builds its tensors in probe_ctx(), then hands the context to probe_run, which frees it.
#pragma once

#include "ggml.h"
#include "ggml-alloc.h"
#include "ggml-backend.h"
#include "ggml-cpu.h"

#include <utility>
#include <vector>

using probe_uploads = std::vector<std::pair<ggml_tensor *, const void *>>;     // (tensor, its ggml_nbytes of input)
using probe_reads   = std::vector<std::pair<ggml_tensor *, void *>>;           // (tensor, where its ggml_nbytes go)

// a no-alloc context with room for every probe's tensors (24) and its graph
inline ggml_context * probe_ctx() {
    ggml_init_params ip = { ggml_tensor_overhead() * 24 + ggml_graph_overhead(), nullptr, true };
    return ggml_init(ip);
}

// A source read through a view of its own parent, *parent.  spec (int64), oracle/pool.py's Source.spec(): type, the parent's ne[4], the
// view's ne[4], its nb1, nb2, nb3 (bytes), its byte offset, and 1 to read the view transposed (dims 0 and 1 swapped, ggml_transpose)
inline ggml_tensor * probe_view_source(ggml_context * ctx, const int64_t * spec, ggml_tensor ** parent) {
    ggml_tensor * p = ggml_new_tensor(ctx, (ggml_type) spec[0], 4, spec + 1);
    *parent = p;
    ggml_tensor * v = ggml_view_4d(ctx, p, spec[5], spec[6], spec[7], spec[8], (size_t) spec[9], (size_t) spec[10], (size_t) spec[11], (size_t) spec[12]);
    return spec[13] ? ggml_transpose(ctx, v) : v;
}

// Build the graph of `result` and run it on device `dev` (ggml-cpu with cpu_threads threads).  Every node must be supported but those that
// compute nothing (NONE, RESHAPE, VIEW, PERMUTE, TRANSPOSE: the plug-in's no-ops).  Each upload whose tensor is not null fills it; after
// the compute each read receives its tensor.  Frees ctx.
// Returns 0, -1 (no such device), -2 (the device declines a node), -3 (allocation failed) or -4 (compute failed; nothing is read back).
inline int probe_run(const char * dev, ggml_context * ctx, ggml_tensor * result, const probe_uploads & uploads, const probe_reads & reads,
                     int cpu_threads = 4) {
    ggml_backend_dev_t d = ggml_backend_dev_by_name(dev);
    ggml_backend_t be = d ? ggml_backend_dev_init(d, nullptr) : nullptr;
    if (!be) { ggml_free(ctx); return -1; }
    if (ggml_backend_is_cpu(be)) ggml_backend_cpu_set_n_threads(be, cpu_threads);
    ggml_cgraph * gf = ggml_new_graph(ctx);
    ggml_build_forward_expand(gf, result);
    int rc = 0;
    for (int i = 0; i < ggml_graph_n_nodes(gf); ++i) {
        const ggml_tensor * n = ggml_graph_node(gf, i);
        switch (n->op) {
            case GGML_OP_NONE: case GGML_OP_RESHAPE: case GGML_OP_VIEW: case GGML_OP_PERMUTE: case GGML_OP_TRANSPOSE: break;
            default: if (!ggml_backend_supports_op(be, n)) rc = -2;
        }
    }
    ggml_backend_buffer_t buf = nullptr;
    if (rc == 0 && !(buf = ggml_backend_alloc_ctx_tensors(ctx, be))) rc = -3;
    if (rc == 0) {
        for (const auto & u : uploads) if (u.first) ggml_backend_tensor_set(u.first, u.second, 0, ggml_nbytes(u.first));
        if (ggml_backend_graph_compute(be, gf) != GGML_STATUS_SUCCESS) rc = -4;
        else for (const auto & r : reads) ggml_backend_tensor_get(r.first, r.second, 0, ggml_nbytes(r.first));
    }
    if (buf) ggml_backend_buffer_free(buf);
    ggml_free(ctx);
    ggml_backend_free(be);
    return rc;
}
