// oracle/llama_graph.cpp — TEST INFRASTRUCTURE ONLY.
//
// A synthetic llama-architecture decoder built in memory on the reference's public API (ggml.h, ggml-alloc.h, ggml-backend.h): token
// embedding (Q4_K) -> n_layer x [RMS_NORM * gain -> Q/K/V projections (Q4_K, grouped-query: fewer K/V heads) -> ROPE of Q and K ->
// CPY of K and V (f16) into views of the KV cache -> attention -> output projection -> residual ADD -> RMS_NORM * gain -> SwiGLU FFN
// (SILU(gate) * up, Q4_K; down Q6_K) -> residual ADD] -> RMS_NORM * gain -> lm_head (Q6_K).  Weights come from a fixed seed and are
// quantized with ggml_quantize_chunk; the norm gains are close to 1.
//
// Presets:
//   norm  RoPE mode 0 over the whole head; attention as MUL_MAT(K, Q) -> SOFT_MAX_EXT(mask, scale) -> MUL_MAT(V^T, KQ)
//   neox  RoPE mode 2 over n_rot = 32 of 64 dims, with freq factors and YaRN (ext_factor 0.5, freq_scale 0.25, n_ctx_orig 512);
//         attention through FLASH_ATTN_EXT (f16 mask padded to GGML_KQ_MASK_PAD)
//
// usage: llama-graph PRESET compare DEVICE [sync]
//          ggml_backend_compare_graph_backend of ggml-cpu against DEVICE over a 7-token prompt and one decode step.  Prints
//          "node PHASE INDEX OP NAME [ne] nmse E" per f32 node and
//          "summary PHASE sync|free nodes_over_1e-9 N worst W first_over INDEX OP logits L" per phase (L: NMSE of the logits node).
//          With "sync" the device copy of each node result is replaced by the CPU's after the comparison (identical inputs per node).
//        llama-graph PRESET run DEVICE STEPS LOGITS_OUT [FORCE_TOKENS]
//          ggml_backend_sched over [DEVICE, CPU] (DEVICE = CPU: the CPU alone), weights and KV cache in DEVICE's buffer, full-graph
//          compute: the prompt, then STEPS - 1 decode steps, greedy (or teacher-forced by the i32 tokens in FORCE_TOKENS).  Writes STEPS
//          rows of n_vocab f32 logits (the last position of each step) to LOGITS_OUT and prints "n_splits S", "cpu_nodes C",
//          "tokens t0 t1 ..." and "decode_ms_per_step M" (host clock around each decode step, which ends in reading the logits back).
// Devices from $GGML_BACKEND_PATH are loaded with ggml_backend_load_all.

#include "ggml.h"
#include "ggml-alloc.h"
#include "ggml-backend.h"
#include "ggml-cpu.h"

#include <chrono>
#include <cinttypes>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <string>
#include <vector>

namespace {

struct hparams {
    int n_embd = 1024, n_head = 16, n_head_kv = 4, head_dim = 64, n_ff = 2816, n_layer = 4, n_vocab = 4096, n_ctx = 64;
    float eps = 1e-5f, freq_base = 10000.0f;
    // rope
    int n_rot = 64, mode = 0, n_ctx_orig = 512;
    float freq_scale = 1.0f, ext_factor = 0.0f, attn_factor = 1.0f, beta_fast = 32.0f, beta_slow = 1.0f;
    bool freq_factors = false, flash_attn = false;
    int n_embd_gqa() const { return n_head_kv * head_dim; }
};

struct layer {
    ggml_tensor * attn_norm, * wq, * wk, * wv, * wo, * ffn_norm, * w_gate, * w_up, * w_down;
    ggml_tensor * k, * v;                                      // KV cache, f16 [n_embd_gqa * n_ctx]
};

struct model {
    hparams hp;
    ggml_context * ctx_w = nullptr, * ctx_kv = nullptr;
    ggml_backend_buffer_t buf_w = nullptr, buf_kv = nullptr;
    ggml_tensor * tok_embd, * out_norm, * lm_head, * rope_ff = nullptr;
    std::vector<layer> layers;
};

hparams preset(const std::string & name) {
    hparams hp;
    if (name == "neox") {
        hp.mode = GGML_ROPE_TYPE_NEOX; hp.n_rot = 32; hp.freq_factors = true; hp.ext_factor = 0.5f; hp.freq_scale = 0.25f; hp.flash_attn = true;
    } else if (name != "norm") {
        fprintf(stderr, "unknown preset %s (norm | neox)\n", name.c_str());
        exit(2);
    }
    return hp;
}

// create the tensors of the model in ctx_w / ctx_kv, allocate them in buffers of `bt`, fill the weights from a fixed seed
void build_model(model & m, ggml_backend_buffer_type_t bt) {
    const hparams & hp = m.hp;
    const size_t n_t = 4 + 11 * (size_t) hp.n_layer;
    ggml_init_params ip = { ggml_tensor_overhead() * n_t, nullptr, true };
    m.ctx_w = ggml_init(ip);
    m.ctx_kv = ggml_init(ip);
    ggml_context * c = m.ctx_w;
    m.tok_embd = ggml_new_tensor_2d(c, GGML_TYPE_Q4_K, hp.n_embd, hp.n_vocab);
    m.out_norm = ggml_new_tensor_1d(c, GGML_TYPE_F32, hp.n_embd);
    m.lm_head = ggml_new_tensor_2d(c, GGML_TYPE_Q6_K, hp.n_embd, hp.n_vocab);
    if (hp.freq_factors) m.rope_ff = ggml_new_tensor_1d(c, GGML_TYPE_F32, hp.n_rot / 2);
    m.layers.resize(hp.n_layer);
    for (layer & l : m.layers) {
        l.attn_norm = ggml_new_tensor_1d(c, GGML_TYPE_F32, hp.n_embd);
        l.wq = ggml_new_tensor_2d(c, GGML_TYPE_Q4_K, hp.n_embd, hp.n_embd);
        l.wk = ggml_new_tensor_2d(c, GGML_TYPE_Q4_K, hp.n_embd, hp.n_embd_gqa());
        l.wv = ggml_new_tensor_2d(c, GGML_TYPE_Q4_K, hp.n_embd, hp.n_embd_gqa());
        l.wo = ggml_new_tensor_2d(c, GGML_TYPE_Q4_K, hp.n_embd, hp.n_embd);
        l.ffn_norm = ggml_new_tensor_1d(c, GGML_TYPE_F32, hp.n_embd);
        l.w_gate = ggml_new_tensor_2d(c, GGML_TYPE_Q4_K, hp.n_embd, hp.n_ff);
        l.w_up = ggml_new_tensor_2d(c, GGML_TYPE_Q4_K, hp.n_embd, hp.n_ff);
        l.w_down = ggml_new_tensor_2d(c, GGML_TYPE_Q6_K, hp.n_ff, hp.n_embd);
        l.k = ggml_new_tensor_1d(m.ctx_kv, GGML_TYPE_F16, (int64_t) hp.n_embd_gqa() * hp.n_ctx);
        l.v = ggml_new_tensor_1d(m.ctx_kv, GGML_TYPE_F16, (int64_t) hp.n_embd_gqa() * hp.n_ctx);
    }
    m.buf_w = ggml_backend_alloc_ctx_tensors_from_buft(m.ctx_w, bt);
    m.buf_kv = ggml_backend_alloc_ctx_tensors_from_buft(m.ctx_kv, bt);
    if (!m.buf_w || !m.buf_kv) { fprintf(stderr, "model allocation failed\n"); exit(4); }
    ggml_backend_buffer_set_usage(m.buf_w, GGML_BACKEND_BUFFER_USAGE_WEIGHTS);
    ggml_backend_buffer_clear(m.buf_kv, 0);

    std::mt19937 rng(20240611);
    std::normal_distribution<float> nd(0.0f, 1.0f);
    auto fill = [&](ggml_tensor * t, float scale, float offset) {
        const int64_t n = ggml_nelements(t), k = t->ne[0];
        std::vector<float> x((size_t) n);
        for (float & v : x) v = offset + scale * nd(rng);
        if (t->type == GGML_TYPE_F32) { ggml_backend_tensor_set(t, x.data(), 0, ggml_nbytes(t)); return; }
        std::vector<uint8_t> q(ggml_nbytes(t));
        ggml_quantize_chunk(t->type, x.data(), q.data(), 0, n / k, k, nullptr);
        ggml_backend_tensor_set(t, q.data(), 0, q.size());
    };
    fill(m.tok_embd, 1.0f, 0.0f);
    fill(m.out_norm, 0.05f, 1.0f);
    fill(m.lm_head, 1.0f / sqrtf((float) hp.n_embd), 0.0f);
    if (m.rope_ff) {
        std::vector<float> ff(hp.n_rot / 2);
        for (size_t i = 0; i < ff.size(); ++i) ff[i] = 1.0f + (float) (i % 4) * 0.75f;        // long-context style factors in [1, 3.25]
        ggml_backend_tensor_set(m.rope_ff, ff.data(), 0, ggml_nbytes(m.rope_ff));
    }
    for (layer & l : m.layers) {
        fill(l.attn_norm, 0.05f, 1.0f);
        fill(l.wq, 1.0f / sqrtf((float) hp.n_embd), 0.0f);
        fill(l.wk, 1.0f / sqrtf((float) hp.n_embd), 0.0f);
        fill(l.wv, 1.0f / sqrtf((float) hp.n_embd), 0.0f);
        fill(l.wo, 1.0f / sqrtf((float) hp.n_embd), 0.0f);
        fill(l.ffn_norm, 0.05f, 1.0f);
        fill(l.w_gate, 1.0f / sqrtf((float) hp.n_embd), 0.0f);
        fill(l.w_up, 1.0f / sqrtf((float) hp.n_embd), 0.0f);
        fill(l.w_down, 1.0f / sqrtf((float) hp.n_ff), 0.0f);
    }
}

// the token graph for N tokens at positions n_past .. n_past + N - 1; inputs "inp_tokens", "inp_pos", "kq_mask"; output "result_output"
ggml_cgraph * build_graph(const model & m, ggml_context * ctx, int n_past, int N) {
    const hparams & hp = m.hp;
    const int n_kv = n_past + N, hd = hp.head_dim, ngqa = hp.n_embd_gqa();
    const size_t es = ggml_type_size(GGML_TYPE_F16);
    ggml_cgraph * gf = ggml_new_graph_custom(ctx, 4096, false);
    ggml_tensor * tok = ggml_new_tensor_1d(ctx, GGML_TYPE_I32, N);
    ggml_set_name(tok, "inp_tokens"); ggml_set_input(tok);
    ggml_tensor * pos = ggml_new_tensor_1d(ctx, GGML_TYPE_I32, N);
    ggml_set_name(pos, "inp_pos"); ggml_set_input(pos);
    ggml_tensor * mask = hp.flash_attn ? ggml_new_tensor_2d(ctx, GGML_TYPE_F16, n_kv, GGML_PAD(N, GGML_KQ_MASK_PAD))
                                       : ggml_new_tensor_2d(ctx, GGML_TYPE_F32, n_kv, N);
    ggml_set_name(mask, "kq_mask"); ggml_set_input(mask);
    const float kq_scale = 1.0f / sqrtf((float) hd);
    auto rope = [&](ggml_tensor * x) {
        return ggml_rope_ext(ctx, x, pos, m.rope_ff, hp.n_rot, hp.mode, hp.n_ctx_orig, hp.freq_base, hp.freq_scale, hp.ext_factor, hp.attn_factor,
                             hp.beta_fast, hp.beta_slow);
    };

    ggml_tensor * inpL = ggml_get_rows(ctx, m.tok_embd, tok);
    for (int il = 0; il < hp.n_layer; ++il) {
        const layer & l = m.layers[il];
        ggml_tensor * cur = ggml_mul(ctx, ggml_rms_norm(ctx, inpL, hp.eps), l.attn_norm);
        ggml_tensor * q = rope(ggml_reshape_3d(ctx, ggml_mul_mat(ctx, l.wq, cur), hd, hp.n_head, N));
        ggml_tensor * k = rope(ggml_reshape_3d(ctx, ggml_mul_mat(ctx, l.wk, cur), hd, hp.n_head_kv, N));
        ggml_tensor * v = ggml_mul_mat(ctx, l.wv, cur);                                          // [ngqa, N]
        ggml_set_name(q, ("q_rope-" + std::to_string(il)).c_str());
        ggml_set_name(k, ("k_rope-" + std::to_string(il)).c_str());
        // KV cache update: K rows at n_past; V rows (flash attention) or V transposed (columns at n_past)
        ggml_build_forward_expand(gf, ggml_cpy(ctx, k, ggml_view_1d(ctx, l.k, (int64_t) N * ngqa, es * ngqa * n_past)));
        if (hp.flash_attn) {
            ggml_build_forward_expand(gf, ggml_cpy(ctx, v, ggml_view_1d(ctx, l.v, (int64_t) N * ngqa, es * ngqa * n_past)));
        } else {
            ggml_tensor * vt = ggml_view_2d(ctx, l.v, N, ngqa, es * hp.n_ctx, es * n_past);
            ggml_build_forward_expand(gf, ggml_cpy(ctx, ggml_transpose(ctx, v), vt));
        }
        ggml_tensor * Q = ggml_permute(ctx, q, 0, 2, 1, 3);                                        // [hd, N, n_head]
        ggml_tensor * K = ggml_view_3d(ctx, l.k, hd, n_kv, hp.n_head_kv, es * ngqa, es * hd, 0);
        if (hp.flash_attn) {
            ggml_tensor * V = ggml_view_3d(ctx, l.v, hd, n_kv, hp.n_head_kv, es * ngqa, es * hd, 0);
            cur = ggml_flash_attn_ext(ctx, Q, K, V, mask, kq_scale, 0.0f, 0.0f);                   // [hd, n_head, N]
            cur = ggml_reshape_2d(ctx, cur, hp.n_embd, N);
        } else {
            ggml_tensor * kq = ggml_soft_max_ext(ctx, ggml_mul_mat(ctx, K, Q), mask, kq_scale, 0.0f);  // [n_kv, N, n_head]
            ggml_tensor * V = ggml_view_3d(ctx, l.v, n_kv, hd, hp.n_head_kv, es * hp.n_ctx, es * hp.n_ctx * hd, 0);
            ggml_tensor * kqv = ggml_mul_mat(ctx, V, kq);                                          // [hd, N, n_head]
            cur = ggml_cont_2d(ctx, ggml_permute(ctx, kqv, 0, 2, 1, 3), hp.n_embd, N);
        }
        cur = ggml_mul_mat(ctx, l.wo, cur);
        ggml_tensor * ffn_inp = ggml_add(ctx, cur, inpL);
        cur = ggml_mul(ctx, ggml_rms_norm(ctx, ffn_inp, hp.eps), l.ffn_norm);
        ggml_tensor * gate = ggml_silu(ctx, ggml_mul_mat(ctx, l.w_gate, cur));
        cur = ggml_mul(ctx, gate, ggml_mul_mat(ctx, l.w_up, cur));
        cur = ggml_mul_mat(ctx, l.w_down, cur);
        inpL = ggml_add(ctx, cur, ffn_inp);
    }
    ggml_tensor * cur = ggml_mul(ctx, ggml_rms_norm(ctx, inpL, hp.eps), m.out_norm);
    cur = ggml_mul_mat(ctx, m.lm_head, cur);
    ggml_set_name(cur, "result_output"); ggml_set_output(cur);
    ggml_build_forward_expand(gf, cur);
    return gf;
}

void set_inputs(const model & m, ggml_cgraph * gf, int n_past, const std::vector<int32_t> & toks) {
    const int N = (int) toks.size(), n_kv = n_past + N;
    ggml_backend_tensor_set(ggml_graph_get_tensor(gf, "inp_tokens"), toks.data(), 0, N * sizeof(int32_t));
    std::vector<int32_t> pos(N);
    for (int i = 0; i < N; ++i) pos[i] = n_past + i;
    ggml_backend_tensor_set(ggml_graph_get_tensor(gf, "inp_pos"), pos.data(), 0, N * sizeof(int32_t));
    ggml_tensor * mask = ggml_graph_get_tensor(gf, "kq_mask");
    const int64_t rows = mask->ne[1];
    std::vector<float> mf((size_t) n_kv * rows);
    for (int64_t i = 0; i < rows; ++i)
        for (int j = 0; j < n_kv; ++j) mf[(size_t) i * n_kv + j] = (i < N && j <= n_past + i) ? 0.0f : -INFINITY;
    if (mask->type == GGML_TYPE_F32) { ggml_backend_tensor_set(mask, mf.data(), 0, ggml_nbytes(mask)); return; }
    std::vector<ggml_fp16_t> mh(mf.size());
    ggml_fp32_to_fp16_row(mf.data(), mh.data(), (int64_t) mf.size());
    ggml_backend_tensor_set(mask, mh.data(), 0, ggml_nbytes(mask));
}

std::vector<int32_t> prompt_tokens() { return { 1, 417, 2093, 58, 3001, 777, 12 }; }

// ------------------------------------------------------------------ compare
struct cmp_state { const char * tag; int n_bad; double worst; bool sync; int first_bad; char first_bad_op[64]; double logits; };

double nmse_f32(const float * a, const float * b, size_t n) {       // as tests/test-backend-ops.cpp computes it (a = device, b = cpu)
    double num = 0.0, den = 0.0;
    for (size_t i = 0; i < n; ++i) { const double d = (double) a[i] - (double) b[i]; num += d * d; den += (double) a[i] * (double) a[i]; }
    return den > 0.0 ? num / den : num;
}

bool on_node(int index, ggml_tensor * t1, ggml_tensor * t2, void * ud) {
    cmp_state * st = (cmp_state *) ud;
    if (t1->type != GGML_TYPE_F32 || !ggml_is_contiguous(t1)) return true;            // views / f16 cache writes: compared through their consumers
    const size_t n = (size_t) ggml_nelements(t1);
    std::vector<float> a(n), b(n);
    ggml_backend_tensor_get(t1, b.data(), 0, n * sizeof(float));                    // t1: CPU
    ggml_backend_tensor_get(t2, a.data(), 0, n * sizeof(float));                    // t2: device
    const double e = nmse_f32(a.data(), b.data(), n);
    if (e > st->worst) st->worst = e;
    if (e > 1e-9) { if (st->n_bad == 0) { st->first_bad = index; snprintf(st->first_bad_op, sizeof(st->first_bad_op), "%s", ggml_op_desc(t1)); } st->n_bad++; }
    if (strcmp(t1->name, "result_output") == 0) st->logits = e;
    if (st->sync) ggml_backend_tensor_set(t2, b.data(), 0, n * sizeof(float));
    printf("node %s %d %s %s [%" PRId64 ",%" PRId64 ",%" PRId64 ",%" PRId64 "] nmse %.3e\n", st->tag, index, ggml_op_desc(t1), t1->name, t1->ne[0], t1->ne[1], t1->ne[2], t1->ne[3], e);
    return true;
}

int run_compare(model & m, ggml_backend_t cpu, ggml_backend_t dev, bool sync) {
    const std::vector<int32_t> prompt = prompt_tokens();
    ggml_gallocr_t allocr = ggml_gallocr_new(ggml_backend_get_default_buffer_type(cpu));
    int rc = 0;
    for (int phase = 0; phase < 2 && rc == 0; ++phase) {
        const int n_past = phase == 0 ? 0 : (int) prompt.size();
        const std::vector<int32_t> toks = phase == 0 ? prompt : std::vector<int32_t>{ 99 };
        ggml_init_params ip = { ggml_tensor_overhead() * 4096 + ggml_graph_overhead_custom(4096, false), nullptr, true };
        ggml_context * ctx = ggml_init(ip);
        ggml_cgraph * gf = build_graph(m, ctx, n_past, (int) toks.size());
        ggml_gallocr_alloc_graph(allocr, gf);
        set_inputs(m, gf, n_past, toks);
        cmp_state st{ phase == 0 ? "prompt" : "decode", 0, 0.0, sync, -1, "", -1.0 };
        // the CPU evaluation also fills the CPU-side KV cache that the decode phase copies over
        if (!ggml_backend_compare_graph_backend(cpu, dev, gf, on_node, &st)) { fprintf(stderr, "graph copy failed\n"); rc = 5; }
        printf("summary %s %s nodes_over_1e-9 %d worst %.3e first_over %d %s logits %.3e\n", st.tag, sync ? "sync" : "free", st.n_bad, st.worst, st.first_bad,
               st.first_bad_op[0] ? st.first_bad_op : "-", st.logits);
        ggml_free(ctx);
    }
    ggml_gallocr_free(allocr);
    return rc;
}

// ------------------------------------------------------------------ run
int run_decode(model & m, ggml_backend_t dev, ggml_backend_t cpu, int steps, const char * out_path, const char * force_path) {
    const hparams & hp = m.hp;
    std::vector<int32_t> force;
    if (force_path) {
        FILE * f = fopen(force_path, "rb");
        if (!f) { fprintf(stderr, "cannot open %s\n", force_path); return 6; }
        int32_t t;
        while (fread(&t, sizeof(t), 1, f) == 1) force.push_back(t);
        fclose(f);
    }
    const std::vector<int32_t> prompt = prompt_tokens();
    if ((int) prompt.size() + steps > hp.n_ctx) { fprintf(stderr, "STEPS too large for n_ctx %d\n", hp.n_ctx); return 2; }
    ggml_backend_t backends[2] = { dev, cpu };
    const int n_be = dev == cpu ? 1 : 2;
    ggml_backend_sched_t sched = ggml_backend_sched_new(backends, nullptr, n_be, 4096, false);
    FILE * out = fopen(out_path, "wb");
    if (!out) { fprintf(stderr, "cannot open %s\n", out_path); return 6; }
    std::vector<float> logits(hp.n_vocab);
    std::vector<int32_t> generated;
    int n_past = 0, max_splits = 0, max_cpu_nodes = 0;
    double decode_s = 0.0;
    int n_decode = 0;
    std::vector<int32_t> toks = prompt;
    for (int step = 0; step < steps; ++step) {
        ggml_init_params ip = { ggml_tensor_overhead() * 4096 + ggml_graph_overhead_custom(4096, false), nullptr, true };
        ggml_context * ctx = ggml_init(ip);
        ggml_cgraph * gf = build_graph(m, ctx, n_past, (int) toks.size());
        ggml_backend_sched_reset(sched);
        if (!ggml_backend_sched_alloc_graph(sched, gf)) { fprintf(stderr, "sched alloc failed\n"); return 7; }
        set_inputs(m, gf, n_past, toks);
        const auto t0 = std::chrono::steady_clock::now();
        if (ggml_backend_sched_graph_compute(sched, gf) != GGML_STATUS_SUCCESS) { fprintf(stderr, "compute failed\n"); return 8; }
        ggml_tensor * res = ggml_graph_get_tensor(gf, "result_output");
        ggml_backend_tensor_get(res, logits.data(), (size_t) (toks.size() - 1) * hp.n_vocab * sizeof(float), hp.n_vocab * sizeof(float));
        const double dt = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
        if (step >= 2) { decode_s += dt; ++n_decode; }                       // step 0: prompt; step 1: first decode (warm-up)
        int cpu_nodes = 0;
        for (int i = 0; i < ggml_graph_n_nodes(gf); ++i)
            if (n_be == 2 && ggml_backend_sched_get_tensor_backend(sched, ggml_graph_node(gf, i)) == cpu) ++cpu_nodes;
        if (ggml_backend_sched_get_n_splits(sched) > max_splits) max_splits = ggml_backend_sched_get_n_splits(sched);
        if (cpu_nodes > max_cpu_nodes) max_cpu_nodes = cpu_nodes;
        fwrite(logits.data(), sizeof(float), logits.size(), out);
        int32_t next = 0;
        for (int i = 1; i < hp.n_vocab; ++i) if (logits[i] > logits[next]) next = i;
        if (step < (int) force.size()) next = force[step];
        generated.push_back(next);
        n_past += (int) toks.size();
        toks = { next };
        ggml_free(ctx);
    }
    fclose(out);
    printf("n_splits %d\ncpu_nodes %d\ntokens", max_splits, max_cpu_nodes);
    for (int32_t t : generated) printf(" %d", t);
    printf("\ndecode_ms_per_step %.4f\n", n_decode ? 1e3 * decode_s / n_decode : -1.0);
    ggml_backend_sched_free(sched);
    return 0;
}

} // namespace

int main(int argc, char ** argv) {
    if (argc < 4) {
        fprintf(stderr, "usage: %s PRESET compare DEVICE [sync]\n       %s PRESET run DEVICE STEPS LOGITS_OUT [FORCE_TOKENS]\n", argv[0], argv[0]);
        return 2;
    }
    ggml_backend_load_all();
    model m;
    m.hp = preset(argv[1]);
    const std::string mode = argv[2];
    ggml_backend_t cpu = ggml_backend_init_by_type(GGML_BACKEND_DEVICE_TYPE_CPU, nullptr);
    ggml_backend_cpu_set_n_threads(cpu, 8);
    ggml_backend_t dev = cpu;
    if (strcmp(argv[3], "CPU") != 0) {
        ggml_backend_dev_t d = ggml_backend_dev_by_name(argv[3]);
        if (!d) { fprintf(stderr, "no device %s\n", argv[3]); return 3; }
        dev = ggml_backend_dev_init(d, nullptr);
    }
    int rc;
    if (mode == "compare") {
        build_model(m, ggml_backend_get_default_buffer_type(cpu));
        rc = run_compare(m, cpu, dev, argc > 4 && strcmp(argv[4], "sync") == 0);
    } else if (mode == "run" && argc >= 6) {
        build_model(m, ggml_backend_get_default_buffer_type(dev));
        rc = run_decode(m, dev, cpu, atoi(argv[4]), argv[5], argc > 6 ? argv[6] : nullptr);
    } else {
        fprintf(stderr, "unknown mode %s\n", mode.c_str());
        return 2;
    }
    ggml_backend_buffer_free(m.buf_w);
    ggml_backend_buffer_free(m.buf_kv);
    ggml_free(m.ctx_w);
    ggml_free(m.ctx_kv);
    if (dev != cpu) ggml_backend_free(dev);
    ggml_backend_free(cpu);
    return rc;
}
