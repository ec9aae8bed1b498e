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
// usage: moe-graph PRESET compare DEVICE [sync] | PRESET run DEVICE STEPS LOGITS_OUT [FORCE_TOKENS]  (decoder_harness.h), one sequence
// with a 7-token prompt, STEPS + 7 <= n_ctx = 64.  In free-running compare mode each ARGSORT row whose top-n_used set differs from the
// CPU's also prints "topk PHASE INDEX ROW margin D rms R" (D: the CPU's gap between its n_used-th and (n_used+1)-th probability; R: the
// RMS deviation of the device's probabilities from the CPU's over the whole router node).

#include "decoder_harness.h"

#include <algorithm>
#include <cmath>

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
    weight_fill w;
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
    w.run(20240611u);
}

void free_model(model & m) {
    ggml_backend_buffer_free(m.buf_w);
    ggml_backend_buffer_free(m.buf_kv);
    ggml_free(m.ctx_w);
    ggml_free(m.ctx_kv);
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

// a differing ARGSORT in free-running mode: the rows whose top-n_used set differs and the CPU's margin there (a: device, b: CPU)
void report_topk(int n_used, const char * tag, int index, ggml_tensor * t1, ggml_tensor * t2, const std::vector<int32_t> & b,
                 const std::vector<int32_t> & a) {
    if (t1->op != GGML_OP_ARGSORT) return;
    const ggml_tensor * p1 = t1->src[0], * p2 = t2->src[0];                          // the router probabilities, contiguous [n_expert, N]
    const int64_t ne0 = t1->ne[0], rows = (int64_t) b.size() / ne0;
    std::vector<float> pc((size_t) ggml_nelements(p1)), pd(pc.size());
    ggml_backend_tensor_get(p1, pc.data(), 0, pc.size() * sizeof(float));
    ggml_backend_tensor_get(p2, pd.data(), 0, pd.size() * sizeof(float));
    double sq = 0.0;
    for (size_t i = 0; i < pc.size(); ++i) sq += ((double) pd[i] - pc[i]) * ((double) pd[i] - pc[i]);
    const double rms = sqrt(sq / (double) pc.size());
    const int k = std::min<int64_t>(n_used, ne0);
    for (int64_t r = 0; r < rows; ++r) {
        std::vector<int32_t> sa(a.begin() + r * ne0, a.begin() + r * ne0 + k), sb(b.begin() + r * ne0, b.begin() + r * ne0 + k);
        std::sort(sa.begin(), sa.end());
        std::sort(sb.begin(), sb.end());
        if (sa == sb) continue;
        const float * pr = pc.data() + r * ne0;
        const double margin = k < ne0 ? (double) pr[b[r * ne0 + k - 1]] - (double) pr[b[r * ne0 + k]] : 0.0;
        printf("topk %s %d %" PRId64 " margin %.6e rms %.6e\n", tag, index, r, margin, rms);
    }
}

} // namespace

int main(int argc, char ** argv) {
    model m;
    return decoder_main(argc, argv, [&m](const std::string & name) {
        m.hp = preset(name);
        decoder d;
        d.n_vocab = m.hp.n_vocab;
        d.n_ctx = m.hp.n_ctx;
        d.prompt = { 1, 417, 2093, 58, 3001, 777, 12 };
        d.build_model = [&m](ggml_backend_buffer_type_t bt) { build_model(m, bt); };
        d.free_model = [&m] { free_model(m); };
        d.build_graph = [&m](ggml_context * ctx, int n_past, int n_t) { return build_graph(m, ctx, n_past, n_t); };
        d.set_inputs = set_inputs;
        d.on_i32_mismatch = [&m](const char * tag, int index, ggml_tensor * t1, ggml_tensor * t2, const std::vector<int32_t> & b,
                                 const std::vector<int32_t> & a) { report_topk(m.hp.n_used, tag, index, t1, t2, b, a); };
        return d;
    });
}
