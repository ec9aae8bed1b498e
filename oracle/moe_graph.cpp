// oracle/moe_graph.cpp — TEST INFRASTRUCTURE ONLY.
//
// A synthetic mixture-of-experts decoder built in memory on the reference's public API (ggml.h, ggml-alloc.h, ggml-backend.h).  The
// attention block is oracle/llama_graph.cpp's `norm` preset (Q4_K projections, grouped-query attention, RoPE mode 0, f16 KV cache written
// by CPY into views, MUL_MAT(K, Q) -> SOFT_MAX_EXT -> MUL_MAT(V^T, KQ)); the FFN is llama.cpp's MoE form:
//   probs    = SOFT_MAX(MUL_MAT(gate_inp, cur))                           [n_expert, N], gate_inp f32
//   selected = ggml_top_k(probs, n_used)                                  ARGSORT (descending) + a view of its first n_used columns
//   weights  = GET_ROWS(reshape_3d(probs, 1, n_expert, N), selected)      [1, n_used, N]
//   weights  = DIV(weights, SUM_ROWS(weights))                            (normalised presets)
//   experts  = MUL_MAT_ID(down_exps, SILU(MUL_MAT_ID(gate_exps, cur)) * MUL_MAT_ID(up_exps, cur)) * weights   Q4_K gate/up, Q6_K down
//   moe_out  = ADD over ggml_view_2d(experts, n_embd, N, nb[2], i * nb[1]), i < n_used
// Weights come from fixed seeds (one per tensor, filled in parallel) and are quantized with ggml_quantize_chunk.
//
// Presets:
//   moe    Mixtral-like: 8 experts of n_ff_exp 1024, top-2, weights normalised (SUM_ROWS + DIV)
//   moe60  Qwen-MoE-like: 60 experts of n_ff_exp 256 (a non-power-of-two sort), top-4, no normalisation, plus a dense shared expert
//          (SwiGLU, n_ff 1024) gated by SIGMOID(MUL_MAT(gate_inp_shexp, cur)) and added to moe_out
//
// usage: moe-graph PRESET compare DEVICE [sync]
//          ggml_backend_compare_graph_backend of ggml-cpu against DEVICE over a 7-token prompt and one decode step.  Prints
//          "node PHASE INDEX OP NAME [ne] nmse E" per f32 node, "inode PHASE INDEX OP NAME [ne] mismatches M" per i32 node (M: index
//          positions that differ), and per ARGSORT row whose top-n_used set differs from the CPU's
//          "topk PHASE INDEX ROW margin D rms R" (D: the CPU's gap between its n_used-th and (n_used+1)-th probability; R: the RMS
//          deviation of the device's probabilities from the CPU's over the whole router node), then per phase
//          "summary PHASE sync|free nodes_over_1e-9 N worst W first_over INDEX OP logits L".
//          With "sync" the device copy of each node result (f32 and i32) is replaced by the CPU's after the comparison.
//        moe-graph PRESET run DEVICE STEPS LOGITS_OUT [FORCE_TOKENS]
//          as llama-graph's run mode: ggml_backend_sched over [DEVICE, CPU], the prompt, then STEPS - 1 decode steps; writes the logits
//          and prints "n_splits S", "cpu_nodes C", "tokens t0 t1 ..." and "decode_ms_per_step M".
// Devices from $GGML_BACKEND_PATH are loaded with ggml_backend_load_all.

#include "ggml.h"
#include "ggml-alloc.h"
#include "ggml-backend.h"
#include "ggml-cpu.h"

#include <algorithm>
#include <chrono>
#include <cinttypes>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <string>
#include <thread>
#include <vector>

namespace {

struct hparams {
    int n_embd = 1024, n_head = 16, n_head_kv = 4, head_dim = 64, n_layer = 4, n_vocab = 4096, n_ctx = 64;
    int n_expert = 8, n_used = 2, n_ff_exp = 1024, n_ff_shexp = 0;
    bool norm_w = true;
    float eps = 1e-5f, freq_base = 10000.0f;
    int n_embd_gqa() const { return n_head_kv * head_dim; }
};

struct layer {
    ggml_tensor * attn_norm, * wq, * wk, * wv, * wo, * ffn_norm;
    ggml_tensor * gate_inp, * gate_exps, * up_exps, * down_exps;
    ggml_tensor * gate_inp_shexp = nullptr, * gate_shexp = nullptr, * up_shexp = nullptr, * down_shexp = nullptr;
    ggml_tensor * k, * v;                                      // KV cache, f16 [n_embd_gqa * n_ctx]
};

struct model {
    hparams hp;
    ggml_context * ctx_w = nullptr, * ctx_kv = nullptr;
    ggml_backend_buffer_t buf_w = nullptr, buf_kv = nullptr;
    ggml_tensor * tok_embd, * out_norm, * lm_head;
    std::vector<layer> layers;
};

hparams preset(const std::string & name) {
    hparams hp;
    if (name == "moe60") {
        hp.n_expert = 60; hp.n_used = 4; hp.n_ff_exp = 256; hp.n_ff_shexp = 1024; hp.norm_w = false;
    } else if (name != "moe") {
        fprintf(stderr, "unknown preset %s (moe | moe60)\n", name.c_str());
        exit(2);
    }
    return hp;
}

// create the tensors of the model in ctx_w / ctx_kv, allocate them in buffers of `bt`, fill the weights from fixed seeds
void build_model(model & m, ggml_backend_buffer_type_t bt) {
    const hparams & hp = m.hp;
    const size_t n_t = 4 + 16 * (size_t) hp.n_layer;
    ggml_init_params ip = { ggml_tensor_overhead() * n_t, nullptr, true };
    m.ctx_w = ggml_init(ip);
    m.ctx_kv = ggml_init(ip);
    ggml_context * c = m.ctx_w;
    struct fill_job { ggml_tensor * t; float scale, offset; };
    std::vector<fill_job> jobs;
    auto w = [&](ggml_tensor * t, float scale, float offset) { jobs.push_back({ t, scale, offset }); return t; };
    const float se = 1.0f / sqrtf((float) hp.n_embd);
    m.tok_embd = w(ggml_new_tensor_2d(c, GGML_TYPE_Q4_K, hp.n_embd, hp.n_vocab), 1.0f, 0.0f);
    m.out_norm = w(ggml_new_tensor_1d(c, GGML_TYPE_F32, hp.n_embd), 0.05f, 1.0f);
    m.lm_head = w(ggml_new_tensor_2d(c, GGML_TYPE_Q6_K, hp.n_embd, hp.n_vocab), se, 0.0f);
    m.layers.resize(hp.n_layer);
    for (layer & l : m.layers) {
        l.attn_norm = w(ggml_new_tensor_1d(c, GGML_TYPE_F32, hp.n_embd), 0.05f, 1.0f);
        l.wq = w(ggml_new_tensor_2d(c, GGML_TYPE_Q4_K, hp.n_embd, hp.n_embd), se, 0.0f);
        l.wk = w(ggml_new_tensor_2d(c, GGML_TYPE_Q4_K, hp.n_embd, hp.n_embd_gqa()), se, 0.0f);
        l.wv = w(ggml_new_tensor_2d(c, GGML_TYPE_Q4_K, hp.n_embd, hp.n_embd_gqa()), se, 0.0f);
        l.wo = w(ggml_new_tensor_2d(c, GGML_TYPE_Q4_K, hp.n_embd, hp.n_embd), se, 0.0f);
        l.ffn_norm = w(ggml_new_tensor_1d(c, GGML_TYPE_F32, hp.n_embd), 0.05f, 1.0f);
        l.gate_inp = w(ggml_new_tensor_2d(c, GGML_TYPE_F32, hp.n_embd, hp.n_expert), se, 0.0f);
        l.gate_exps = w(ggml_new_tensor_3d(c, GGML_TYPE_Q4_K, hp.n_embd, hp.n_ff_exp, hp.n_expert), se, 0.0f);
        l.up_exps = w(ggml_new_tensor_3d(c, GGML_TYPE_Q4_K, hp.n_embd, hp.n_ff_exp, hp.n_expert), se, 0.0f);
        l.down_exps = w(ggml_new_tensor_3d(c, GGML_TYPE_Q6_K, hp.n_ff_exp, hp.n_embd, hp.n_expert), 1.0f / sqrtf((float) hp.n_ff_exp), 0.0f);
        if (hp.n_ff_shexp) {
            l.gate_inp_shexp = w(ggml_new_tensor_1d(c, GGML_TYPE_F32, hp.n_embd), se, 0.0f);
            l.gate_shexp = w(ggml_new_tensor_2d(c, GGML_TYPE_Q4_K, hp.n_embd, hp.n_ff_shexp), se, 0.0f);
            l.up_shexp = w(ggml_new_tensor_2d(c, GGML_TYPE_Q4_K, hp.n_embd, hp.n_ff_shexp), se, 0.0f);
            l.down_shexp = w(ggml_new_tensor_2d(c, GGML_TYPE_Q6_K, hp.n_ff_shexp, hp.n_embd), 1.0f / sqrtf((float) hp.n_ff_shexp), 0.0f);
        }
        l.k = ggml_new_tensor_1d(m.ctx_kv, GGML_TYPE_F16, (int64_t) hp.n_embd_gqa() * hp.n_ctx);
        l.v = ggml_new_tensor_1d(m.ctx_kv, GGML_TYPE_F16, (int64_t) hp.n_embd_gqa() * hp.n_ctx);
    }
    m.buf_w = ggml_backend_alloc_ctx_tensors_from_buft(m.ctx_w, bt);
    m.buf_kv = ggml_backend_alloc_ctx_tensors_from_buft(m.ctx_kv, bt);
    if (!m.buf_w || !m.buf_kv) { fprintf(stderr, "model allocation failed\n"); exit(4); }
    ggml_backend_buffer_set_usage(m.buf_w, GGML_BACKEND_BUFFER_USAGE_WEIGHTS);
    ggml_backend_buffer_clear(m.buf_kv, 0);

    // tensor j is drawn from its own generator (seed 20240611 + j), so the parallel fill is deterministic
    std::vector<std::vector<uint8_t>> bytes(jobs.size());
    auto fill = [&](size_t j) {
        const ggml_tensor * t = jobs[j].t;
        std::mt19937 rng(20240611u + (unsigned) j);
        std::normal_distribution<float> nd(0.0f, 1.0f);
        const int64_t n = ggml_nelements(t), k = t->ne[0];
        std::vector<float> x((size_t) n);
        for (float & v : x) v = jobs[j].offset + jobs[j].scale * nd(rng);
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

// the MoE FFN of layer l on cur [n_embd, N] (llama.cpp's build_moe_ffn with softmax gating and SILU experts)
ggml_tensor * moe_ffn(const hparams & hp, const layer & l, ggml_context * ctx, ggml_tensor * cur, int il, int N) {
    const std::string sfx = "-" + std::to_string(il);
    ggml_tensor * probs = ggml_soft_max(ctx, ggml_mul_mat(ctx, l.gate_inp, cur));                     // [n_expert, N]
    ggml_set_name(probs, ("ffn_moe_probs" + sfx).c_str());
    ggml_tensor * selected = ggml_top_k(ctx, probs, hp.n_used);                                        // [n_used, N]
    ggml_set_name(selected->view_src, ("ffn_moe_argsort" + sfx).c_str());
    ggml_tensor * weights = ggml_get_rows(ctx, ggml_reshape_3d(ctx, probs, 1, hp.n_expert, N), selected);   // [1, n_used, N]
    if (hp.norm_w) {
        weights = ggml_reshape_2d(ctx, weights, hp.n_used, N);
        ggml_tensor * sum = ggml_sum_rows(ctx, weights);                                                // [1, N]
        ggml_set_name(sum, ("ffn_moe_weights_sum" + sfx).c_str());
        weights = ggml_reshape_3d(ctx, ggml_div(ctx, weights, sum), 1, hp.n_used, N);
    }
    ggml_tensor * x = ggml_reshape_3d(ctx, cur, hp.n_embd, 1, N);
    ggml_tensor * up = ggml_mul_mat_id(ctx, l.up_exps, x, selected);                                  // [n_ff_exp, n_used, N]
    ggml_tensor * gate = ggml_silu(ctx, ggml_mul_mat_id(ctx, l.gate_exps, x, selected));
    ggml_tensor * experts = ggml_mul_mat_id(ctx, l.down_exps, ggml_mul(ctx, up, gate), selected);      // [n_embd, n_used, N]
    experts = ggml_mul(ctx, experts, weights);
    ggml_tensor * out = ggml_view_2d(ctx, experts, hp.n_embd, N, experts->nb[2], 0);
    for (int i = 1; i < hp.n_used; ++i)
        out = ggml_add(ctx, out, ggml_view_2d(ctx, experts, hp.n_embd, N, experts->nb[2], i * experts->nb[1]));
    if (hp.n_ff_shexp) {
        ggml_tensor * g = ggml_sigmoid(ctx, ggml_mul_mat(ctx, l.gate_inp_shexp, cur));                  // [1, N]
        ggml_tensor * sh = ggml_mul(ctx, ggml_silu(ctx, ggml_mul_mat(ctx, l.gate_shexp, cur)), ggml_mul_mat(ctx, l.up_shexp, cur));
        sh = ggml_mul(ctx, ggml_mul_mat(ctx, l.down_shexp, sh), g);
        out = ggml_add(ctx, out, sh);
    }
    return out;
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
    ggml_tensor * mask = ggml_new_tensor_2d(ctx, GGML_TYPE_F32, n_kv, N);
    ggml_set_name(mask, "kq_mask"); ggml_set_input(mask);
    const float kq_scale = 1.0f / sqrtf((float) hd);
    auto rope = [&](ggml_tensor * x) { return ggml_rope_ext(ctx, x, pos, nullptr, hd, 0, 512, hp.freq_base, 1.0f, 0.0f, 1.0f, 32.0f, 1.0f); };

    ggml_tensor * inpL = ggml_get_rows(ctx, m.tok_embd, tok);
    for (int il = 0; il < hp.n_layer; ++il) {
        const layer & l = m.layers[il];
        ggml_tensor * cur = ggml_mul(ctx, ggml_rms_norm(ctx, inpL, hp.eps), l.attn_norm);
        ggml_tensor * q = rope(ggml_reshape_3d(ctx, ggml_mul_mat(ctx, l.wq, cur), hd, hp.n_head, N));
        ggml_tensor * k = rope(ggml_reshape_3d(ctx, ggml_mul_mat(ctx, l.wk, cur), hd, hp.n_head_kv, N));
        ggml_tensor * v = ggml_mul_mat(ctx, l.wv, cur);                                          // [ngqa, N]
        ggml_build_forward_expand(gf, ggml_cpy(ctx, k, ggml_view_1d(ctx, l.k, (int64_t) N * ngqa, es * ngqa * n_past)));
        ggml_tensor * vt = ggml_view_2d(ctx, l.v, N, ngqa, es * hp.n_ctx, es * n_past);
        ggml_build_forward_expand(gf, ggml_cpy(ctx, ggml_transpose(ctx, v), vt));
        ggml_tensor * Q = ggml_permute(ctx, q, 0, 2, 1, 3);                                        // [hd, N, n_head]
        ggml_tensor * K = ggml_view_3d(ctx, l.k, hd, n_kv, hp.n_head_kv, es * ngqa, es * hd, 0);
        ggml_tensor * kq = ggml_soft_max_ext(ctx, ggml_mul_mat(ctx, K, Q), mask, kq_scale, 0.0f);  // [n_kv, N, n_head]
        ggml_tensor * V = ggml_view_3d(ctx, l.v, n_kv, hd, hp.n_head_kv, es * hp.n_ctx, es * hp.n_ctx * hd, 0);
        cur = ggml_cont_2d(ctx, ggml_permute(ctx, ggml_mul_mat(ctx, V, kq), 0, 2, 1, 3), hp.n_embd, N);
        cur = ggml_mul_mat(ctx, l.wo, cur);
        ggml_tensor * ffn_inp = ggml_add(ctx, cur, inpL);
        cur = ggml_mul(ctx, ggml_rms_norm(ctx, ffn_inp, hp.eps), l.ffn_norm);
        inpL = ggml_add(ctx, moe_ffn(hp, l, ctx, cur, il, N), ffn_inp);
    }
    ggml_tensor * cur = ggml_mul(ctx, ggml_rms_norm(ctx, inpL, hp.eps), m.out_norm);
    cur = ggml_mul_mat(ctx, m.lm_head, cur);
    ggml_set_name(cur, "result_output"); ggml_set_output(cur);
    ggml_build_forward_expand(gf, cur);
    return gf;
}

void set_inputs(ggml_cgraph * gf, int n_past, const std::vector<int32_t> & toks) {
    const int N = (int) toks.size(), n_kv = n_past + N;
    ggml_backend_tensor_set(ggml_graph_get_tensor(gf, "inp_tokens"), toks.data(), 0, N * sizeof(int32_t));
    std::vector<int32_t> pos(N);
    for (int i = 0; i < N; ++i) pos[i] = n_past + i;
    ggml_backend_tensor_set(ggml_graph_get_tensor(gf, "inp_pos"), pos.data(), 0, N * sizeof(int32_t));
    std::vector<float> mf((size_t) n_kv * N);
    for (int i = 0; i < N; ++i)
        for (int j = 0; j < n_kv; ++j) mf[(size_t) i * n_kv + j] = j <= n_past + i ? 0.0f : -INFINITY;
    ggml_backend_tensor_set(ggml_graph_get_tensor(gf, "kq_mask"), mf.data(), 0, mf.size() * sizeof(float));
}

std::vector<int32_t> prompt_tokens() { return { 1, 417, 2093, 58, 3001, 777, 12 }; }

// ------------------------------------------------------------------ compare
struct cmp_state { const char * tag; int n_bad; double worst; bool sync; int first_bad; char first_bad_op[64]; double logits; int n_used; };

double nmse_f32(const float * a, const float * b, size_t n) {       // as tests/test-backend-ops.cpp computes it (a = device, b = cpu)
    double num = 0.0, den = 0.0;
    for (size_t i = 0; i < n; ++i) { const double d = (double) a[i] - (double) b[i]; num += d * d; den += (double) a[i] * (double) a[i]; }
    return den > 0.0 ? num / den : num;
}

void dims(const ggml_tensor * t, char * buf, size_t n) {
    snprintf(buf, n, "[%" PRId64 ",%" PRId64 ",%" PRId64 ",%" PRId64 "]", t->ne[0], t->ne[1], t->ne[2], t->ne[3]);
}

// an i32 node: exact index mismatches; for ARGSORT in free-running mode, the rows whose top-n_used set differs and the CPU's margin there
void on_i32_node(cmp_state * st, int index, ggml_tensor * t1, ggml_tensor * t2) {
    const size_t n = (size_t) ggml_nelements(t1);
    std::vector<int32_t> a(n), b(n);
    ggml_backend_tensor_get(t1, b.data(), 0, n * sizeof(int32_t));                  // t1: CPU
    ggml_backend_tensor_get(t2, a.data(), 0, n * sizeof(int32_t));                  // t2: device
    size_t mism = 0;
    for (size_t i = 0; i < n; ++i) mism += a[i] != b[i];
    char ne[96];
    dims(t1, ne, sizeof(ne));
    printf("inode %s %d %s %s %s mismatches %zu\n", st->tag, index, ggml_op_desc(t1), t1->name, ne, mism);
    if (t1->op == GGML_OP_ARGSORT && !st->sync && mism) {
        const ggml_tensor * p1 = t1->src[0], * p2 = t2->src[0];                      // the router probabilities, contiguous [n_expert, N]
        const int64_t ne0 = t1->ne[0], rows = (int64_t) n / ne0;
        std::vector<float> pc((size_t) ggml_nelements(p1)), pd(pc.size());
        ggml_backend_tensor_get(p1, pc.data(), 0, pc.size() * sizeof(float));
        ggml_backend_tensor_get(p2, pd.data(), 0, pd.size() * sizeof(float));
        double sq = 0.0;
        for (size_t i = 0; i < pc.size(); ++i) sq += ((double) pd[i] - pc[i]) * ((double) pd[i] - pc[i]);
        const double rms = sqrt(sq / (double) pc.size());
        const int k = std::min<int64_t>(st->n_used, ne0);
        for (int64_t r = 0; r < rows; ++r) {
            std::vector<int32_t> sa(a.begin() + r * ne0, a.begin() + r * ne0 + k), sb(b.begin() + r * ne0, b.begin() + r * ne0 + k);
            std::sort(sa.begin(), sa.end());
            std::sort(sb.begin(), sb.end());
            if (sa == sb) continue;
            const float * pr = pc.data() + r * ne0;
            const double margin = k < ne0 ? (double) pr[b[r * ne0 + k - 1]] - (double) pr[b[r * ne0 + k]] : 0.0;
            printf("topk %s %d %" PRId64 " margin %.6e rms %.6e\n", st->tag, index, r, margin, rms);
        }
    }
    if (st->sync) ggml_backend_tensor_set(t2, b.data(), 0, n * sizeof(int32_t));
}

bool on_node(int index, ggml_tensor * t1, ggml_tensor * t2, void * ud) {
    cmp_state * st = (cmp_state *) ud;
    if (!ggml_is_contiguous(t1)) return true;                                       // views / f16 cache writes: compared through their consumers
    if (t1->type == GGML_TYPE_I32) { on_i32_node(st, index, t1, t2); return true; }
    if (t1->type != GGML_TYPE_F32) return true;
    const size_t n = (size_t) ggml_nelements(t1);
    std::vector<float> a(n), b(n);
    ggml_backend_tensor_get(t1, b.data(), 0, n * sizeof(float));                    // t1: CPU
    ggml_backend_tensor_get(t2, a.data(), 0, n * sizeof(float));                    // t2: device
    const double e = nmse_f32(a.data(), b.data(), n);
    if (e > st->worst) st->worst = e;
    if (e > 1e-9) { if (st->n_bad == 0) { st->first_bad = index; snprintf(st->first_bad_op, sizeof(st->first_bad_op), "%s", ggml_op_desc(t1)); } st->n_bad++; }
    if (strcmp(t1->name, "result_output") == 0) st->logits = e;
    if (st->sync) ggml_backend_tensor_set(t2, b.data(), 0, n * sizeof(float));
    char ne[96];
    dims(t1, ne, sizeof(ne));
    printf("node %s %d %s %s %s nmse %.3e\n", st->tag, index, ggml_op_desc(t1), t1->name, ne, e);
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
        set_inputs(gf, n_past, toks);
        cmp_state st{ phase == 0 ? "prompt" : "decode", 0, 0.0, sync, -1, "", -1.0, m.hp.n_used };
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
        set_inputs(gf, n_past, toks);
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
