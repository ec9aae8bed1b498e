// oracle/yolo_graph.cpp — TEST INFRASTRUCTURE ONLY.
//
// A synthetic YOLOv3-tiny detector built in memory on the reference's public API (ggml.h, ggml-alloc.h, ggml-backend.h, gguf.h): the
// network of the reference's examples/yolo program, with weights from fixed seeds instead of a converted checkpoint.
//   13 conv layers, each ggml_conv_2d (IM2COL with f16 columns, then an f16 x f16 MUL_MAT, then CONT of a permute), stride 1, padding 1
//   for 3 x 3 kernels and 0 for 1 x 1; then, except in the two linear layers 9 and 12, the batch norm (x - mean) / sqrt(var) * scale of
//   REPEATed per-channel vectors; + REPEATed bias; LEAKY_RELU(0.1) in place, again except in 9 and 12.
//     conv0 3->16, pool; conv1 16->32, pool; conv2 32->64, pool; conv3 64->128, pool; conv4 128->256 (= layer_8), pool;
//     conv5 256->512, pool k2 s1 p0.5; conv6 512->1024; conv7 1x1 1024->256 (= layer_13); conv8 256->512; conv9 1x1 512->255 = "layer_15";
//     conv10 1x1 layer_13 256->128, UPSCALE x2, CONCAT with layer_8 along channels; conv11 384->256; conv12 1x1 256->255 = "layer_22".
//   The five k2 s2 pools and the k2 s1 pool with ggml_pool_2d's float padding 0.5 are MAX pools.
// Weights: conv kernels f16 [k, k, in, out] ~ N(0, 1/K) (K = k k in, so activations stay O(1) through the 13 layers); biases, scales,
// means f32 [1, 1, C, 1]; variances positive (0.5 + 0.5 |N(0, 1)|), so SQRT stays finite.  The input image comes from a seed.
//
// Presets:
//   tiny    the example's network: one 416 x 416 x 3 image; heads [13, 13, 255] and [26, 26, 255]
//   batch2  the same network on two 320 x 320 x 3 images, so IM2COL, POOL_2D, UPSCALE, REPEAT and CONCAT all see ne3 = 2
//
// usage: yolo-graph PRESET compare DEVICE [sync]
//          ggml_backend_compare_graph_backend of ggml-cpu against DEVICE with decoder_harness.h's node comparison: "node image INDEX OP NAME
//          [ne] nmse E" per contiguous f32 node, then "summary image sync|free nodes_over_1e-9 N worst W first_over INDEX OP logits -1".
//          With "sync" the device copy of each node result is replaced by the CPU's after the comparison (identical inputs per node).
//        yolo-graph PRESET run DEVICE REPS OUT
//          ggml_backend_sched over [DEVICE, CPU] (DEVICE = CPU: the CPU alone), weights in DEVICE's buffer: one warm-up pass, then REPS
//          passes.  Writes the heads of the last pass (layer_15, then layer_22, f32) to OUT and prints "n_splits S", "cpu_nodes C",
//          "passes_identical 0|1" (every pass's heads equal the first's bit for bit) and "ms_per_pass M" (host clock around compute and the
//          read-back of both heads).
//        yolo-graph PRESET write-gguf PATH
//          the preset's weights as a GGUF file under the example's tensor names: l{i}_weights f16 [k, k, in, out]; l{i}_biases, and for the
//          batch-normalised layers l{i}_scales, l{i}_rolling_mean, l{i}_rolling_variance, f32 [1, 1, C, 1].
// Each graph built also prints "ops im2col I pool_2d P upscale U leaky_relu L repeat R concat C" (its node counts per op).
// Exit codes: 2 usage or unknown preset, 3 unknown device, 4 model allocation, 5 graph copy, 6 file, 7 scheduler allocation, 8 compute.

#include "decoder_harness.h"
#include "gguf.h"

#include <cmath>

namespace {

struct conv_layer {
    int k, in, out;
    bool bn;                                                   // batch norm and LEAKY_RELU (false: the linear layers 9 and 12)
    ggml_tensor * w = nullptr, * b = nullptr, * scale = nullptr, * mean = nullptr, * var = nullptr;
};

struct model {
    int size = 416, batch = 1;
    std::vector<conv_layer> conv;
    ggml_context * ctx = nullptr;
    ggml_backend_buffer_t buf = nullptr;
};

void setup(model & m, const std::string & preset) {
    if (preset == "batch2") { m.size = 320; m.batch = 2; }
    else if (preset != "tiny") { fprintf(stderr, "unknown preset %s (tiny | batch2)\n", preset.c_str()); exit(2); }
    // {kernel, in, out, batch-normalised}
    const int spec[13][4] = { {3, 3, 16, 1}, {3, 16, 32, 1}, {3, 32, 64, 1}, {3, 64, 128, 1}, {3, 128, 256, 1}, {3, 256, 512, 1},
                              {3, 512, 1024, 1}, {1, 1024, 256, 1}, {3, 256, 512, 1}, {1, 512, 255, 0}, {1, 256, 128, 1}, {3, 384, 256, 1},
                              {1, 256, 255, 0} };
    for (const auto & s : spec) m.conv.push_back(conv_layer{ s[0], s[1], s[2], s[3] != 0 });
}

// kind 1: a positive variance
float special(int, int64_t, int64_t, std::mt19937 & rng) {
    std::normal_distribution<float> nd(0.0f, 1.0f);
    return 0.5f + 0.5f * fabsf(nd(rng));
}

void build_model(model & m, ggml_backend_buffer_type_t bt) {
    ggml_init_params ip = { ggml_tensor_overhead() * 5 * m.conv.size(), nullptr, true };
    m.ctx = ggml_init(ip);
    weight_fill w;
    char name[64];
    for (size_t i = 0; i < m.conv.size(); ++i) {
        conv_layer & l = m.conv[i];
        auto vec = [&](const char * what, float scale, float offset, int kind) {
            ggml_tensor * t = ggml_new_tensor_4d(m.ctx, GGML_TYPE_F32, 1, 1, l.out, 1);
            snprintf(name, sizeof(name), "l%zu_%s", i, what);
            ggml_set_name(t, name);
            return w(t, scale, offset, kind);
        };
        l.w = ggml_new_tensor_4d(m.ctx, GGML_TYPE_F16, l.k, l.k, l.in, l.out);
        snprintf(name, sizeof(name), "l%zu_weights", i);
        ggml_set_name(l.w, name);
        w(l.w, 1.0f / sqrtf((float) (l.k * l.k * l.in)), 0.0f);
        l.b = vec("biases", 0.1f, 0.0f, 0);
        if (l.bn) {
            l.scale = vec("scales", 0.1f, 1.0f, 0);
            l.mean = vec("rolling_mean", 0.1f, 0.0f, 0);
            l.var = vec("rolling_variance", 0.0f, 0.0f, 1);
        }
    }
    m.buf = ggml_backend_alloc_ctx_tensors_from_buft(m.ctx, bt);
    if (!m.buf) { fprintf(stderr, "model allocation failed\n"); exit(4); }
    ggml_backend_buffer_set_usage(m.buf, GGML_BACKEND_BUFFER_USAGE_WEIGHTS);
    w.run(20241117u, special);
}

void free_model(model & m) {
    ggml_backend_buffer_free(m.buf);
    ggml_free(m.ctx);
}

ggml_tensor * conv(ggml_context * ctx, ggml_tensor * x, const conv_layer & l) {
    ggml_tensor * y = ggml_conv_2d(ctx, l.w, x, 1, 1, l.k / 2, l.k / 2, 1, 1);
    if (l.bn) {
        y = ggml_sub(ctx, y, ggml_repeat(ctx, l.mean, y));
        y = ggml_div(ctx, y, ggml_sqrt(ctx, ggml_repeat(ctx, l.var, y)));
        y = ggml_mul(ctx, y, ggml_repeat(ctx, l.scale, y));
    }
    y = ggml_add(ctx, y, ggml_repeat(ctx, l.b, y));
    return l.bn ? ggml_leaky_relu(ctx, y, 0.1f, true) : y;
}

ggml_tensor * max_pool(ggml_context * ctx, ggml_tensor * x, int s, float p) { return ggml_pool_2d(ctx, x, GGML_OP_POOL_MAX, 2, 2, s, s, p, p); }

// input "input" [size, size, 3, batch]; outputs "layer_15" and "layer_22"
ggml_cgraph * build_graph(const model & m, ggml_context * ctx) {
    ggml_cgraph * gf = ggml_new_graph_custom(ctx, 1024, false);
    ggml_tensor * x = ggml_new_tensor_4d(ctx, GGML_TYPE_F32, m.size, m.size, 3, m.batch);
    ggml_set_name(x, "input"); ggml_set_input(x);
    const std::vector<conv_layer> & c = m.conv;
    x = max_pool(ctx, conv(ctx, x, c[0]), 2, 0.0f);
    x = max_pool(ctx, conv(ctx, x, c[1]), 2, 0.0f);
    x = max_pool(ctx, conv(ctx, x, c[2]), 2, 0.0f);
    x = max_pool(ctx, conv(ctx, x, c[3]), 2, 0.0f);
    ggml_tensor * layer_8 = conv(ctx, x, c[4]);
    x = max_pool(ctx, layer_8, 2, 0.0f);
    x = max_pool(ctx, conv(ctx, x, c[5]), 1, 0.5f);
    ggml_tensor * layer_13 = conv(ctx, conv(ctx, x, c[6]), c[7]);
    ggml_tensor * layer_15 = conv(ctx, conv(ctx, layer_13, c[8]), c[9]);
    ggml_set_name(layer_15, "layer_15"); ggml_set_output(layer_15);
    x = ggml_concat(ctx, ggml_upscale(ctx, conv(ctx, layer_13, c[10]), 2), layer_8, 2);
    ggml_tensor * layer_22 = conv(ctx, conv(ctx, x, c[11]), c[12]);
    ggml_set_name(layer_22, "layer_22"); ggml_set_output(layer_22);
    ggml_build_forward_expand(gf, layer_15);
    ggml_build_forward_expand(gf, layer_22);
    int n[6] = { 0, 0, 0, 0, 0, 0 };
    const ggml_op ops[6] = { GGML_OP_IM2COL, GGML_OP_POOL_2D, GGML_OP_UPSCALE, GGML_OP_LEAKY_RELU, GGML_OP_REPEAT, GGML_OP_CONCAT };
    for (int i = 0; i < ggml_graph_n_nodes(gf); ++i)
        for (int k = 0; k < 6; ++k) n[k] += ggml_graph_node(gf, i)->op == ops[k];
    printf("ops im2col %d pool_2d %d upscale %d leaky_relu %d repeat %d concat %d\n", n[0], n[1], n[2], n[3], n[4], n[5]);
    return gf;
}

// an image's range, [0, 1], smooth along rows, from a fixed seed
void set_input(const model & m, ggml_cgraph * gf) {
    ggml_tensor * t = ggml_graph_get_tensor(gf, "input");
    std::mt19937 rng(5489u);
    std::uniform_real_distribution<float> ud(0.0f, 1.0f);
    std::vector<float> img((size_t) ggml_nelements(t));
    float prev = 0.5f;
    for (float & v : img) { prev = 0.7f * prev + 0.3f * ud(rng); v = prev; }
    ggml_backend_tensor_set(t, img.data(), 0, ggml_nbytes(t));
}

ggml_context * graph_ctx() {
    ggml_init_params ip = { ggml_tensor_overhead() * 1024 + ggml_graph_overhead_custom(1024, false), nullptr, true };
    return ggml_init(ip);
}

int run_compare(const model & m, ggml_backend_t cpu, ggml_backend_t dev, bool sync) {
    ggml_context * ctx = graph_ctx();
    ggml_cgraph * gf = build_graph(m, ctx);
    ggml_gallocr_t allocr = ggml_gallocr_new(ggml_backend_get_default_buffer_type(cpu));
    ggml_gallocr_alloc_graph(allocr, gf);
    set_input(m, gf);
    const decoder none;
    cmp_state st{ &none, "image", sync, 0, 0.0, -1, "", -1.0 };
    int rc = 0;
    if (!ggml_backend_compare_graph_backend(cpu, dev, gf, on_node, &st)) { fprintf(stderr, "graph copy failed\n"); rc = 5; }
    printf("summary %s %s nodes_over_1e-9 %d worst %.3e first_over %d %s logits %.3e\n", st.tag, sync ? "sync" : "free", st.n_bad, st.worst, st.first_bad,
           st.first_bad_op[0] ? st.first_bad_op : "-", st.logits);
    ggml_gallocr_free(allocr);
    ggml_free(ctx);
    return rc;
}

int run_passes(const model & m, ggml_backend_t dev, ggml_backend_t cpu, int reps, const char * out_path) {
    ggml_backend_t backends[2] = { dev, cpu };
    const int n_be = dev == cpu ? 1 : 2;
    ggml_backend_sched_t sched = ggml_backend_sched_new(backends, nullptr, n_be, 1024, false);
    ggml_context * ctx = graph_ctx();
    ggml_cgraph * gf = build_graph(m, ctx);
    if (!ggml_backend_sched_alloc_graph(sched, gf)) { fprintf(stderr, "sched alloc failed\n"); return 7; }
    ggml_tensor * heads[2] = { ggml_graph_get_tensor(gf, "layer_15"), ggml_graph_get_tensor(gf, "layer_22") };
    const size_t n15 = (size_t) ggml_nelements(heads[0]), n22 = (size_t) ggml_nelements(heads[1]);
    std::vector<float> out(n15 + n22), first;
    bool identical = true;
    double total_s = 0.0;
    for (int pass = 0; pass <= reps; ++pass) {                 // pass 0: warm-up
        set_input(m, gf);
        const auto t0 = std::chrono::steady_clock::now();
        if (ggml_backend_sched_graph_compute(sched, gf) != GGML_STATUS_SUCCESS) { fprintf(stderr, "compute failed\n"); return 8; }
        ggml_backend_tensor_get(heads[0], out.data(), 0, n15 * sizeof(float));
        ggml_backend_tensor_get(heads[1], out.data() + n15, 0, n22 * sizeof(float));
        const double dt = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
        if (pass == 0) { first = out; continue; }
        total_s += dt;
        identical = identical && memcmp(first.data(), out.data(), out.size() * sizeof(float)) == 0;
    }
    int cpu_nodes = 0;
    for (int i = 0; i < ggml_graph_n_nodes(gf); ++i)
        if (n_be == 2 && ggml_backend_sched_get_tensor_backend(sched, ggml_graph_node(gf, i)) == cpu) ++cpu_nodes;
    FILE * f = fopen(out_path, "wb");
    if (!f) { fprintf(stderr, "cannot open %s\n", out_path); return 6; }
    fwrite(out.data(), sizeof(float), out.size(), f);
    fclose(f);
    printf("n_splits %d\ncpu_nodes %d\npasses_identical %d\nms_per_pass %.4f\n", ggml_backend_sched_get_n_splits(sched), cpu_nodes, identical ? 1 : 0,
           reps > 0 ? 1e3 * total_s / reps : -1.0);
    ggml_backend_sched_free(sched);
    ggml_free(ctx);
    return 0;
}

int write_gguf(const model & m, const char * path) {
    gguf_context * g = gguf_init_empty();
    for (const conv_layer & l : m.conv)
        for (ggml_tensor * t : { l.w, l.b, l.scale, l.mean, l.var })
            if (t) gguf_add_tensor(g, t);
    const bool ok = gguf_write_to_file(g, path, false);
    gguf_free(g);
    if (!ok) { fprintf(stderr, "cannot write %s\n", path); return 6; }
    return 0;
}

} // namespace

int main(int argc, char ** argv) {
    if (argc < 4) {
        fprintf(stderr, "usage: %s PRESET compare DEVICE [sync]\n       %s PRESET run DEVICE REPS OUT\n       %s PRESET write-gguf PATH\n", argv[0], argv[0], argv[0]);
        return 2;
    }
    model m;
    setup(m, argv[1]);
    const std::string mode = argv[2];
    ggml_backend_load_all();
    ggml_backend_t cpu = ggml_backend_init_by_type(GGML_BACKEND_DEVICE_TYPE_CPU, nullptr);
    ggml_backend_cpu_set_n_threads(cpu, 8);
    if (mode == "write-gguf") {
        build_model(m, ggml_backend_get_default_buffer_type(cpu));        // host memory: gguf_add_tensor reads the data in place
        const int rc = write_gguf(m, argv[3]);
        free_model(m);
        ggml_backend_free(cpu);
        return rc;
    }
    ggml_backend_t dev = cpu;
    if (strcmp(argv[3], "CPU") != 0) {
        ggml_backend_dev_t dd = ggml_backend_dev_by_name(argv[3]);
        if (!dd) { fprintf(stderr, "no device %s\n", argv[3]); return 3; }
        dev = ggml_backend_dev_init(dd, nullptr);
    }
    int rc;
    if (mode == "compare") {
        build_model(m, ggml_backend_get_default_buffer_type(cpu));
        rc = run_compare(m, cpu, dev, argc > 4 && strcmp(argv[4], "sync") == 0);
    } else if (mode == "run" && argc >= 6) {
        build_model(m, ggml_backend_get_default_buffer_type(dev));
        rc = run_passes(m, dev, cpu, atoi(argv[4]), argv[5]);
    } else {
        fprintf(stderr, "unknown mode %s\n", mode.c_str());
        return 2;
    }
    free_model(m);
    if (dev != cpu) ggml_backend_free(dev);
    ggml_backend_free(cpu);
    return rc;
}
