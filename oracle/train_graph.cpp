// oracle/train_graph.cpp — TEST INFRASTRUCTURE ONLY.
//
// A synthetic trainer of this repository's own on the reference's public training API (ggml-opt.h): a 784-500-10 classifier with RELU,
// trained through ggml_opt_forward_backward on ggml_backend_sched over [DEVICE, CPU], so that ggml_opt builds its forward graph,
// ggml_build_backward_expand's backward graph and one OPT_STEP_ADAMW node per parameter, with the AdamW hyper-parameters in ggml_opt's own
// host buffer.
//
// usage: PROGRAM PRESET run DEVICE STEPS OUT
//   PRESET  fc   cross-entropy loss (GGML_OPT_LOSS_TYPE_CROSS_ENTROPY), physical batch 500, opt_period 2 (gb_grad and gb_opt alternate)
//           mse  the same network and batches with GGML_OPT_LOSS_TYPE_MEAN_SQUARED_ERROR (which brings in SUM)
//   STEPS   forward_backward calls (each one physical batch; an optimizer step every opt_period calls)
//   Prints "graph grad|opt n_splits S cpu_nodes C [OP ...]" for the first call of each graph (the ops of the nodes the scheduler put on the
//   CPU), "loss I L" per call (the batch's loss, %.9g), "accuracy A" of the last batch and "ms_per_call M" (host clock around each call
//   after the first two, which ends in reading the loss back), and writes the final weights (fc1 weight, fc1 bias, fc2 weight, fc2 bias,
//   f32) to OUT.  DEVICE = CPU: the CPU alone, 8 threads.
// Data: each class is a seeded random template plus seeded noise, so that the task is learnable; the batch of call i is drawn from a
// generator seeded with i, so every device sees the same batches.  Devices from $GGML_BACKEND_PATH are loaded with ggml_backend_load_all.
// Exit codes: 2 usage, 3 unknown device, 6 file.
#include "ggml.h"
#include "ggml-alloc.h"
#include "ggml-backend.h"
#include "ggml-cpu.h"
#include "ggml-opt.h"

#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <string>
#include <vector>

namespace {

constexpr int NIN = 784, NHID = 500, NOUT = 10, NBATCH = 500, OPT_PERIOD = 2;

struct observe {
    ggml_backend_sched_t sched;
    ggml_backend_t cpu;
    int cpu_nodes = 0;
    std::string ops;
};

// the scheduler's eval callback, set for one call only: counts the nodes it computes on the CPU; never asks to see a result, so every
// split is still computed whole
bool on_node(ggml_tensor * t, bool ask, void * ud) {
    observe * o = (observe *) ud;
    if (ask && ggml_backend_sched_get_tensor_backend(o->sched, t) == o->cpu) {
        ++o->cpu_nodes;
        o->ops += std::string(" ") + ggml_op_desc(t);
    }
    return false;
}

void fill_normal(ggml_tensor * t, float scale, unsigned seed) {
    std::mt19937 rng(seed);
    std::normal_distribution<float> nd(0.0f, 1.0f);
    std::vector<float> v((size_t) ggml_nelements(t));
    for (float & x : v) x = scale * nd(rng);
    ggml_backend_tensor_set(t, v.data(), 0, ggml_nbytes(t));
}

// batch `i`: NBATCH images of class c = template c + 0.6 N(0, 1), and their one-hot labels
void make_batch(int i, const std::vector<float> & templates, std::vector<float> & x, std::vector<float> & y, std::vector<int> & cls) {
    std::mt19937 rng(1000u + (unsigned) i);
    std::uniform_int_distribution<int> ud(0, NOUT - 1);
    std::normal_distribution<float> nd(0.0f, 1.0f);
    x.assign((size_t) NIN * NBATCH, 0.0f);
    y.assign((size_t) NOUT * NBATCH, 0.0f);
    cls.assign(NBATCH, 0);
    for (int b = 0; b < NBATCH; ++b) {
        const int c = ud(rng);
        cls[b] = c;
        y[(size_t) b * NOUT + c] = 1.0f;
        for (int k = 0; k < NIN; ++k) x[(size_t) b * NIN + k] = templates[(size_t) c * NIN + k] + 0.6f * nd(rng);
    }
}

} // namespace

int main(int argc, char ** argv) {
    if (argc < 6 || strcmp(argv[2], "run") != 0) {
        fprintf(stderr, "usage: %s fc|mse run DEVICE STEPS OUT\n", argv[0]);
        return 2;
    }
    const std::string preset = argv[1];
    if (preset != "fc" && preset != "mse") { fprintf(stderr, "unknown preset %s\n", argv[1]); return 2; }
    const int steps = atoi(argv[4]);
    ggml_backend_load_all();
    ggml_backend_t cpu = ggml_backend_init_by_type(GGML_BACKEND_DEVICE_TYPE_CPU, nullptr);
    ggml_backend_cpu_set_n_threads(cpu, 8);
    ggml_backend_t dev = cpu;
    if (strcmp(argv[3], "CPU") != 0) {
        ggml_backend_dev_t dd = ggml_backend_dev_by_name(argv[3]);
        if (!dd) { fprintf(stderr, "no device %s\n", argv[3]); return 3; }
        dev = ggml_backend_dev_init(dd, nullptr);
    }
    ggml_backend_t backends[2] = { dev, cpu };
    const int n_be = dev == cpu ? 1 : 2;
    ggml_backend_sched_t sched = ggml_backend_sched_new(backends, nullptr, n_be, GGML_DEFAULT_GRAPH_SIZE, false);

    // the weights and the images, statically in DEVICE's buffer (as examples/mnist keeps them)
    ggml_init_params sp = { 8 * ggml_tensor_overhead(), nullptr, true };
    ggml_context * ctx_static = ggml_init(sp);
    ggml_tensor * w1 = ggml_new_tensor_2d(ctx_static, GGML_TYPE_F32, NIN, NHID);
    ggml_tensor * b1 = ggml_new_tensor_1d(ctx_static, GGML_TYPE_F32, NHID);
    ggml_tensor * w2 = ggml_new_tensor_2d(ctx_static, GGML_TYPE_F32, NHID, NOUT);
    ggml_tensor * b2 = ggml_new_tensor_1d(ctx_static, GGML_TYPE_F32, NOUT);
    ggml_tensor * images = ggml_new_tensor_2d(ctx_static, GGML_TYPE_F32, NIN, NBATCH);
    ggml_set_input(images);
    ggml_backend_buffer_t buf = ggml_backend_alloc_ctx_tensors(ctx_static, dev);
    fill_normal(w1, 1.0f / sqrtf((float) NIN), 1);
    fill_normal(b1, 0.01f, 2);
    fill_normal(w2, 1.0f / sqrtf((float) NHID), 3);
    fill_normal(b2, 0.01f, 4);

    ggml_init_params cp = { 1024 * ggml_tensor_overhead() + 3 * ggml_graph_overhead_custom(GGML_DEFAULT_GRAPH_SIZE, true), nullptr, true };
    ggml_context * ctx_compute = ggml_init(cp);
    for (ggml_tensor * p : { w1, b1, w2, b2 }) ggml_set_param(ctx_compute, p);
    ggml_tensor * h = ggml_relu(ctx_compute, ggml_add(ctx_compute, ggml_mul_mat(ctx_compute, w1, images), b1));
    ggml_tensor * logits = ggml_add(ctx_compute, ggml_mul_mat(ctx_compute, w2, h), b2);

    ggml_opt_params op = ggml_opt_default_params(sched, ctx_compute, images, logits,
                                                 preset == "fc" ? GGML_OPT_LOSS_TYPE_CROSS_ENTROPY : GGML_OPT_LOSS_TYPE_MEAN_SQUARED_ERROR);
    op.opt_period = OPT_PERIOD;
    ggml_opt_context_t opt = ggml_opt_init(op);

    std::vector<float> templates((size_t) NOUT * NIN);
    {
        std::mt19937 rng(7);
        std::uniform_real_distribution<float> ud(-1.0f, 1.0f);
        for (float & v : templates) v = ud(rng);
    }
    std::vector<float> x, y;
    std::vector<int> cls;
    double total_s = 0.0;
    int timed = 0;
    double accuracy = 0.0;
    for (int i = 0; i < steps; ++i) {
        make_batch(i, templates, x, y, cls);
        ggml_backend_tensor_set(images, x.data(), 0, ggml_nbytes(images));
        ggml_backend_tensor_set(ggml_opt_labels(opt), y.data(), 0, ggml_nbytes(ggml_opt_labels(opt)));
        observe ob{ sched, cpu };
        const bool first = i < OPT_PERIOD;                     // call 0 evaluates gb_grad, call 1 gb_opt
        if (first) ggml_backend_sched_set_eval_callback(sched, on_node, &ob);
        ggml_opt_result_t res = ggml_opt_result_init();
        const auto t0 = std::chrono::steady_clock::now();
        ggml_opt_forward_backward(opt, res);
        const double dt = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
        if (first) {
            ggml_backend_sched_set_eval_callback(sched, nullptr, nullptr);
            printf("graph %s n_splits %d cpu_nodes %d%s\n", (i + 1) % OPT_PERIOD == 0 ? "opt" : "grad", ggml_backend_sched_get_n_splits(sched),
                   n_be == 2 ? ob.cpu_nodes : 0, n_be == 2 ? ob.ops.c_str() : "");
        } else {
            total_s += dt;
            ++timed;
        }
        double loss, unc;
        ggml_opt_result_loss(res, &loss, &unc);
        printf("loss %d %.9g\n", i, loss);
        if (i == steps - 1) {
            std::vector<int32_t> pred(NBATCH);
            ggml_opt_result_pred(res, pred.data());
            int ok = 0;
            for (int b = 0; b < NBATCH; ++b) ok += pred[b] == cls[b];
            accuracy = (double) ok / NBATCH;
        }
        ggml_opt_result_free(res);
    }
    printf("accuracy %.4f\nms_per_call %.4f\n", accuracy, timed ? 1e3 * total_s / timed : -1.0);

    int rc = 0;
    FILE * f = fopen(argv[5], "wb");
    if (!f) { fprintf(stderr, "cannot open %s\n", argv[5]); rc = 6; }
    else {
        for (ggml_tensor * p : { w1, b1, w2, b2 }) {
            std::vector<float> v((size_t) ggml_nelements(p));
            ggml_backend_tensor_get(p, v.data(), 0, ggml_nbytes(p));
            fwrite(v.data(), sizeof(float), v.size(), f);
        }
        fclose(f);
    }
    ggml_opt_free(opt);
    ggml_free(ctx_compute);
    ggml_backend_buffer_free(buf);
    ggml_free(ctx_static);
    ggml_backend_sched_free(sched);
    if (dev != cpu) ggml_backend_free(dev);
    ggml_backend_free(cpu);
    return rc;
}
