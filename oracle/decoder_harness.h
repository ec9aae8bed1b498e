// oracle/decoder_harness.h — TEST INFRASTRUCTURE ONLY.
//
// What the synthetic decoders (llama_graph.cpp, moe_graph.cpp, mamba_graph.cpp, rwkv_graph.cpp) share: the command line, the node-by-node
// comparison, the scheduler decode loop and the parallel weight fill.  A driver describes its model in a `decoder` and calls decoder_main.
//
// usage: PROGRAM PRESET compare DEVICE [sync]
//          ggml_backend_compare_graph_backend of ggml-cpu against DEVICE over the prompt and one decode step (token 99 + 11 s for sequence
//          s).  Prints "node PHASE INDEX OP NAME [ne] nmse E" per contiguous f32 node, "inode PHASE INDEX OP NAME [ne] mismatches M" per
//          contiguous i32 node (M: positions that differ), then per phase
//          "summary PHASE sync|free nodes_over_1e-9 N worst W first_over INDEX OP logits L" (L: NMSE of the logits node).
//          With "sync" the device copy of each node result is replaced by the CPU's after the comparison (identical inputs per node).
//        PROGRAM PRESET run DEVICE STEPS LOGITS_OUT [FORCE_TOKENS]
//          ggml_backend_sched over [DEVICE, CPU] (DEVICE = CPU: the CPU alone), weights and caches in DEVICE's buffer, full-graph
//          compute: the prompt, then STEPS - 1 decode steps, greedy (or teacher-forced by the i32 tokens in FORCE_TOKENS).  Writes per
//          step the logits of each sequence's last token (STEPS x n_seqs rows of n_vocab f32) to LOGITS_OUT and prints "n_splits S",
//          "cpu_nodes C", "tokens t0 t1 ..." (step-major, one per sequence and step; FORCE_TOKENS is read in the same order) and
//          "decode_ms_per_step M" (host clock around each decode step, which ends in reading the logits back).
// Devices from $GGML_BACKEND_PATH are loaded with ggml_backend_load_all.  Exit codes: 2 usage, unknown preset or STEPS beyond the context,
// 3 unknown device, 4 model allocation, 5 graph copy, 6 file, 7 scheduler allocation, 8 compute.
#pragma once

#include "ggml.h"
#include "ggml-alloc.h"
#include "ggml-backend.h"
#include "ggml-cpu.h"

#include <chrono>
#include <cinttypes>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <random>
#include <string>
#include <thread>
#include <vector>

struct decoder {
    int n_seqs = 1, n_vocab = 0, graph_size = 4096;
    int n_ctx = 0;                                         // the KV-cache length run mode must not exceed; 0: no limit
    std::vector<int32_t> prompt;                           // sequence-major, n_seqs x the prompt length
    std::function<void(ggml_backend_buffer_type_t)> build_model;       // weights and caches in buffers of this type
    std::function<void()> free_model;
    // the graph of n_t tokens per sequence at positions n_past .. n_past + n_t - 1; logits in "result_output", sequence-major rows
    std::function<ggml_cgraph *(ggml_context *, int n_past, int n_t)> build_graph;
    std::function<void(ggml_cgraph *, int n_past, const std::vector<int32_t> & toks)> set_inputs;
    // optional, compare mode without sync: an i32 node whose result differs from the CPU's (cpu, dev: the two results)
    std::function<void(const char * phase, int index, ggml_tensor * t_cpu, ggml_tensor * t_dev, const std::vector<int32_t> & cpu,
                       const std::vector<int32_t> & dev)> on_i32_mismatch;
};

// The weights of a model, filled on 8 threads: tensor j is drawn from its own generator (seed + j), so the fill is deterministic.
// Kind 0 is offset + scale * N(0, 1); a driver's other kinds come from `special(kind, element, row length, generator)`.
struct weight_fill {
    struct job { ggml_tensor * t; float scale, offset; int kind; };
    std::vector<job> jobs;

    ggml_tensor * operator()(ggml_tensor * t, float scale, float offset, int kind = 0) { jobs.push_back({ t, scale, offset, kind }); return t; }

    void run(unsigned seed, float (*special)(int kind, int64_t i, int64_t k, std::mt19937 & rng) = nullptr) const {
        std::vector<std::vector<uint8_t>> bytes(jobs.size());
        auto fill = [&](size_t j) {
            const ggml_tensor * t = jobs[j].t;
            std::mt19937 rng(seed + (unsigned) j);
            std::normal_distribution<float> nd(0.0f, 1.0f);
            const int64_t n = ggml_nelements(t), k = t->ne[0];
            std::vector<float> x((size_t) n);
            for (int64_t i = 0; i < n; ++i)
                x[(size_t) i] = jobs[j].kind ? special(jobs[j].kind, i, k, rng) : jobs[j].offset + jobs[j].scale * nd(rng);
            bytes[j].resize(ggml_nbytes(t));
            if (t->type == GGML_TYPE_F32) memcpy(bytes[j].data(), x.data(), bytes[j].size());
            else ggml_quantize_chunk(t->type, x.data(), bytes[j].data(), 0, n / k, k, nullptr);
        };
        std::vector<std::thread> pool;
        const size_t n_th = 8;
        for (size_t th = 0; th < n_th; ++th)
            pool.emplace_back([&, th] { for (size_t j = th; j < jobs.size(); j += n_th) fill(j); });
        for (std::thread & t : pool) t.join();
        for (size_t j = 0; j < jobs.size(); ++j) ggml_backend_tensor_set(jobs[j].t, bytes[j].data(), 0, bytes[j].size());
    }
};

// ------------------------------------------------------------------ compare
struct cmp_state { const decoder * d; const char * tag; bool sync; int n_bad; double worst; int first_bad; char first_bad_op[64]; double logits; };

static double nmse_f32(const float * a, const float * b, size_t n) {       // as tests/test-backend-ops.cpp computes it (a = device, b = cpu)
    double num = 0.0, den = 0.0;
    for (size_t i = 0; i < n; ++i) { const double d = (double) a[i] - (double) b[i]; num += d * d; den += (double) a[i] * (double) a[i]; }
    return den > 0.0 ? num / den : num;
}

// t1: CPU, t2: device; a / b: the device's / the CPU's result
static bool on_node(int index, ggml_tensor * t1, ggml_tensor * t2, void * ud) {
    cmp_state * st = (cmp_state *) ud;
    if (!ggml_is_contiguous(t1)) return true;                                       // views / f16 cache writes: compared through their consumers
    char ne[96];
    snprintf(ne, sizeof(ne), "[%" PRId64 ",%" PRId64 ",%" PRId64 ",%" PRId64 "]", t1->ne[0], t1->ne[1], t1->ne[2], t1->ne[3]);
    const size_t n = (size_t) ggml_nelements(t1);
    if (t1->type == GGML_TYPE_I32) {
        std::vector<int32_t> a(n), b(n);
        ggml_backend_tensor_get(t1, b.data(), 0, n * sizeof(int32_t));
        ggml_backend_tensor_get(t2, a.data(), 0, n * sizeof(int32_t));
        size_t mism = 0;
        for (size_t i = 0; i < n; ++i) mism += a[i] != b[i];
        printf("inode %s %d %s %s %s mismatches %zu\n", st->tag, index, ggml_op_desc(t1), t1->name, ne, mism);
        if (!st->sync && mism && st->d->on_i32_mismatch) st->d->on_i32_mismatch(st->tag, index, t1, t2, b, a);
        if (st->sync) ggml_backend_tensor_set(t2, b.data(), 0, n * sizeof(int32_t));
        return true;
    }
    if (t1->type != GGML_TYPE_F32) return true;
    std::vector<float> a(n), b(n);
    ggml_backend_tensor_get(t1, b.data(), 0, n * sizeof(float));
    ggml_backend_tensor_get(t2, a.data(), 0, n * sizeof(float));
    const double e = nmse_f32(a.data(), b.data(), n);
    if (e > st->worst) st->worst = e;
    if (e > 1e-9) { if (st->n_bad == 0) { st->first_bad = index; snprintf(st->first_bad_op, sizeof(st->first_bad_op), "%s", ggml_op_desc(t1)); } st->n_bad++; }
    if (strcmp(t1->name, "result_output") == 0) st->logits = e;
    if (st->sync) ggml_backend_tensor_set(t2, b.data(), 0, n * sizeof(float));
    printf("node %s %d %s %s %s nmse %.3e\n", st->tag, index, ggml_op_desc(t1), t1->name, ne, e);
    return true;
}

static ggml_context * graph_context(const decoder & d) {
    ggml_init_params ip = { ggml_tensor_overhead() * d.graph_size + ggml_graph_overhead_custom(d.graph_size, false), nullptr, true };
    return ggml_init(ip);
}

static int run_compare(const decoder & d, ggml_backend_t cpu, ggml_backend_t dev, bool sync) {
    const int prompt_len = (int) d.prompt.size() / d.n_seqs;
    ggml_gallocr_t allocr = ggml_gallocr_new(ggml_backend_get_default_buffer_type(cpu));
    int rc = 0;
    for (int phase = 0; phase < 2 && rc == 0; ++phase) {
        const int n_past = phase == 0 ? 0 : prompt_len, n_t = phase == 0 ? prompt_len : 1;
        std::vector<int32_t> toks = d.prompt;
        if (phase == 1) { toks.clear(); for (int s = 0; s < d.n_seqs; ++s) toks.push_back(99 + 11 * s); }
        ggml_context * ctx = graph_context(d);
        ggml_cgraph * gf = d.build_graph(ctx, n_past, n_t);
        ggml_gallocr_alloc_graph(allocr, gf);
        d.set_inputs(gf, n_past, toks);
        cmp_state st{ &d, phase == 0 ? "prompt" : "decode", sync, 0, 0.0, -1, "", -1.0 };
        // the CPU evaluation also advances the CPU-side caches (KV or state) that the decode phase copies over
        if (!ggml_backend_compare_graph_backend(cpu, dev, gf, on_node, &st)) { fprintf(stderr, "graph copy failed\n"); rc = 5; }
        printf("summary %s %s nodes_over_1e-9 %d worst %.3e first_over %d %s logits %.3e\n", st.tag, sync ? "sync" : "free", st.n_bad, st.worst, st.first_bad,
               st.first_bad_op[0] ? st.first_bad_op : "-", st.logits);
        ggml_free(ctx);
    }
    ggml_gallocr_free(allocr);
    return rc;
}

// ------------------------------------------------------------------ run
static int run_decode(const decoder & d, ggml_backend_t dev, ggml_backend_t cpu, int steps, const char * out_path, const char * force_path) {
    std::vector<int32_t> force;
    if (force_path) {
        FILE * f = fopen(force_path, "rb");
        if (!f) { fprintf(stderr, "cannot open %s\n", force_path); return 6; }
        int32_t t;
        while (fread(&t, sizeof(t), 1, f) == 1) force.push_back(t);
        fclose(f);
    }
    const int prompt_len = (int) d.prompt.size() / d.n_seqs;
    if (d.n_ctx && prompt_len + steps > d.n_ctx) { fprintf(stderr, "STEPS too large for n_ctx %d\n", d.n_ctx); return 2; }
    ggml_backend_t backends[2] = { dev, cpu };
    const int n_be = dev == cpu ? 1 : 2;
    ggml_backend_sched_t sched = ggml_backend_sched_new(backends, nullptr, n_be, d.graph_size, false);
    FILE * out = fopen(out_path, "wb");
    if (!out) { fprintf(stderr, "cannot open %s\n", out_path); return 6; }
    std::vector<float> logits((size_t) d.n_seqs * d.n_vocab);
    std::vector<int32_t> generated;
    int n_past = 0, max_splits = 0, max_cpu_nodes = 0;
    double decode_s = 0.0;
    int n_decode = 0;
    std::vector<int32_t> toks = d.prompt;
    for (int step = 0; step < steps; ++step) {
        const int n_t = step == 0 ? prompt_len : 1;
        ggml_context * ctx = graph_context(d);
        ggml_cgraph * gf = d.build_graph(ctx, n_past, n_t);
        ggml_backend_sched_reset(sched);
        if (!ggml_backend_sched_alloc_graph(sched, gf)) { fprintf(stderr, "sched alloc failed\n"); return 7; }
        d.set_inputs(gf, n_past, toks);
        const auto t0 = std::chrono::steady_clock::now();
        if (ggml_backend_sched_graph_compute(sched, gf) != GGML_STATUS_SUCCESS) { fprintf(stderr, "compute failed\n"); return 8; }
        ggml_tensor * res = ggml_graph_get_tensor(gf, "result_output");
        for (int s = 0; s < d.n_seqs; ++s) {
            const size_t row = (size_t) s * n_t + n_t - 1;                         // each sequence's last token
            ggml_backend_tensor_get(res, logits.data() + (size_t) s * d.n_vocab, row * d.n_vocab * sizeof(float), d.n_vocab * sizeof(float));
        }
        const double dt = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
        if (step >= 2) { decode_s += dt; ++n_decode; }                       // step 0: prompt; step 1: first decode (warm-up)
        int cpu_nodes = 0;
        for (int i = 0; i < ggml_graph_n_nodes(gf); ++i)
            if (n_be == 2 && ggml_backend_sched_get_tensor_backend(sched, ggml_graph_node(gf, i)) == cpu) ++cpu_nodes;
        if (ggml_backend_sched_get_n_splits(sched) > max_splits) max_splits = ggml_backend_sched_get_n_splits(sched);
        if (cpu_nodes > max_cpu_nodes) max_cpu_nodes = cpu_nodes;
        fwrite(logits.data(), sizeof(float), logits.size(), out);
        toks.resize(d.n_seqs);
        for (int s = 0; s < d.n_seqs; ++s) {
            const float * l = logits.data() + (size_t) s * d.n_vocab;
            int32_t best = 0;
            for (int i = 1; i < d.n_vocab; ++i) if (l[i] > l[best]) best = i;
            const size_t k = (size_t) step * d.n_seqs + s;
            toks[s] = k < force.size() ? force[k] : best;
        }
        generated.insert(generated.end(), toks.begin(), toks.end());
        n_past += n_t;
        ggml_free(ctx);
    }
    fclose(out);
    printf("n_splits %d\ncpu_nodes %d\ntokens", max_splits, max_cpu_nodes);
    for (int32_t t : generated) printf(" %d", t);
    printf("\ndecode_ms_per_step %.4f\n", n_decode ? 1e3 * decode_s / n_decode : -1.0);
    ggml_backend_sched_free(sched);
    return 0;
}

// setup(PRESET) selects the preset (exit(2) on an unknown one) and describes the model
static int decoder_main(int argc, char ** argv, const std::function<decoder(const std::string & preset)> & setup) {
    if (argc < 4) {
        fprintf(stderr, "usage: %s PRESET compare DEVICE [sync]\n       %s PRESET run DEVICE STEPS LOGITS_OUT [FORCE_TOKENS]\n", argv[0], argv[0]);
        return 2;
    }
    ggml_backend_load_all();
    const decoder d = setup(argv[1]);
    const std::string mode = argv[2];
    ggml_backend_t cpu = ggml_backend_init_by_type(GGML_BACKEND_DEVICE_TYPE_CPU, nullptr);
    // no more than the head count of the RWKV presets: ggml-cpu's WKV6 / GLA return before an internal barrier on threads ith >= H
    ggml_backend_cpu_set_n_threads(cpu, 8);
    ggml_backend_t dev = cpu;
    if (strcmp(argv[3], "CPU") != 0) {
        ggml_backend_dev_t dd = ggml_backend_dev_by_name(argv[3]);
        if (!dd) { fprintf(stderr, "no device %s\n", argv[3]); return 3; }
        dev = ggml_backend_dev_init(dd, nullptr);
    }
    int rc;
    if (mode == "compare") {
        d.build_model(ggml_backend_get_default_buffer_type(cpu));
        rc = run_compare(d, cpu, dev, argc > 4 && strcmp(argv[4], "sync") == 0);
    } else if (mode == "run" && argc >= 6) {
        d.build_model(ggml_backend_get_default_buffer_type(dev));
        rc = run_decode(d, dev, cpu, atoi(argv[4]), argv[5], argc > 6 ? argv[6] : nullptr);
    } else {
        fprintf(stderr, "unknown mode %s\n", mode.c_str());
        return 2;
    }
    d.free_model();
    if (dev != cpu) ggml_backend_free(dev);
    ggml_backend_free(cpu);
    return rc;
}
