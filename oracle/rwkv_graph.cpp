// oracle/rwkv_graph.cpp — TEST INFRASTRUCTURE ONLY.
//
// A synthetic RWKV-6 decoder built in memory on the reference's public API (ggml.h, ggml-alloc.h, ggml-backend.h), in the form of llama.cpp's
// RWKV-6 graph, over n_seqs sequences of n_t tokens each (tokens sequence-major, x [n_embd, n_t n_seqs]):
//   time mix   xa = LN(x);  x_prev = CONCAT(att_shift, first n_t - 1 tokens of xa, 1);  CPY(last token of xa -> att_shift);  sx = x_prev - xa
//              m  = MUL_MAT(w2 [32, n_embd, 1, 5], CONT(PERMUTE(TANH(MUL_MAT(w1, xa + sx * lerp_x)))))   the data-dependent lerp: 5 views
//              xw, xk, xv, xr, xg = xa + sx * (m_* + lerp_*)
//              r, k, v = MUL_MAT(Wr / Wk / Wv, x*) viewed [S, H, T];  g = SILU(MUL_MAT(Wg, xg))
//              w  = EXP(NEG(EXP(time_decay + MUL_MAT(dw2, TANH(MUL_MAT(dw1, xw))))))
//              wkv = RWKV_WKV6(k, v, r, tf, w, state);  CPY(state part -> wkv_states)
//              y  = (NORM(y viewed [S, H, T], 64e-5) viewed [n_embd, T] * ln_x + ln_x_b) * g;  x += MUL_MAT(Wo, y)
//   channel mix xf = LN(x);  token shift as above with ffn_shift;  xk, xr = xf + sx * lerp_k / lerp_r
//              x += SIGMOID(MUL_MAT(Cr, xr)) * MUL_MAT(Cv, SQR(RELU(MUL_MAT(Ck, xk))))
// The states (token shifts and WKV states) live in a buffer of the evaluating device; a batch reads them through GET_ROWS(state_copy) *
// state_mask (0 on the prompt, 1 afterwards).  The decay pre-activations are spread over the range trained RWKV-6 models use.  Weights come
// from fixed seeds (one per tensor, filled in parallel) and are quantized with ggml_quantize_chunk: Q4_K embeddings and r / k / v / g / output
// projections, Q8_0 channel-mix receptance, Q6_K channel-mix value and lm_head; the low-rank lerp / decay matrices stay f32.  4 layers,
// vocabulary 4096, head size 64.
//
// Presets:
//   rwkv6   RWKV-6 1.6B widths: n_embd 2048, 32 heads of 64, n_ff 7168; LayerNorms; two sequences decode side by side
//   qrwkv   RWKV6-Qwen2 ("QRWKV6") form: RMS_NORM, k scaled by (1 - w), GATED_LINEAR_ATTN(k, v, r, w, scale 64^-0.5) without ln_x, and a
//           SwiGLU FFN (n_ff 5632) in place of the channel mix; one sequence
// ggml-cpu's WKV6 / GLA return before an internal barrier on threads ith >= H, so the CPU runs with 8 threads <= 32 heads.
//
// usage: rwkv-graph PRESET compare DEVICE [sync] | PRESET run DEVICE STEPS LOGITS_OUT [FORCE_TOKENS]  (decoder_harness.h), n_seqs
// sequences with 4-token prompts.

#include "decoder_harness.h"

#include <cmath>

namespace {

const int GRAPH_SIZE = 8192;

struct hparams {
    int n_embd = 2048, head_size = 64, n_ff = 7168, n_layer = 4, n_vocab = 4096, n_seqs = 2, lora_mix = 32, lora_decay = 64;
    bool qrwkv = false;
    float eps = 1e-5f;
    int n_head() const { return n_embd / head_size; }
};

struct layer {
    ggml_tensor * ln1, * ln1_b, * ln2, * ln2_b;
    ggml_tensor * lerp_x, * lerp[5], * w1, * w2, * dw1, * dw2, * time_decay, * tf;
    ggml_tensor * wr, * wk, * wv, * wg, * wo, * ln_x, * ln_x_b;
    ggml_tensor * c_lerp_k, * c_lerp_r, * ck, * cv, * cr;                  // channel mix (rwkv6) / SwiGLU gate, down, up (qrwkv)
    ggml_tensor * att_shift, * ffn_shift, * wkv_states;                    // f32 [n_embd n_seqs], [n_embd n_seqs], [S S H n_seqs]
};

struct model {
    hparams hp;
    ggml_context * ctx_w = nullptr, * ctx_s = nullptr;
    ggml_backend_buffer_t buf_w = nullptr, buf_s = nullptr;
    ggml_tensor * tok_embd, * ln0, * ln0_b, * out_norm, * out_norm_b, * lm_head;
    std::vector<layer> layers;
};

hparams preset(const std::string & name) {
    hparams hp;
    if (name == "qrwkv") {
        hp.qrwkv = true; hp.n_seqs = 1; hp.n_ff = 5632;
    } else if (name != "rwkv6") {
        fprintf(stderr, "unknown preset %s (rwkv6 | qrwkv)\n", name.c_str());
        exit(2);
    }
    return hp;
}

enum fill_kind { FILL_NORMAL, FILL_UNIT, FILL_DECAY };

float fill_special(int kind, int64_t, int64_t, std::mt19937 & rng) {
    if (kind == FILL_UNIT) return std::uniform_real_distribution<float>(0.0f, 1.0f)(rng);
    return std::uniform_real_distribution<float>(-6.0f, 0.5f)(rng);                    // exp(-exp(.)) from ~0.998 down to ~0.19 per token
}

// create the tensors of the model in ctx_w / ctx_s, allocate them in buffers of `bt`, fill the weights from fixed seeds
void build_model(model & m, ggml_backend_buffer_type_t bt) {
    const hparams & hp = m.hp;
    const size_t n_t = 8 + 40 * (size_t) hp.n_layer;
    ggml_init_params ip = { ggml_tensor_overhead() * n_t, nullptr, true };
    m.ctx_w = ggml_init(ip);
    m.ctx_s = ggml_init(ip);
    ggml_context * c = m.ctx_w;
    weight_fill w;
    const int64_t E = hp.n_embd, F = hp.n_ff, S = hp.head_size, H = hp.n_head();
    const float se = 1.0f / sqrtf((float) E), sf = 1.0f / sqrtf((float) F);
    auto vec = [&](float scale, float offset) { return w(ggml_new_tensor_1d(c, GGML_TYPE_F32, E), scale, offset); };
    m.tok_embd = w(ggml_new_tensor_2d(c, GGML_TYPE_Q4_K, E, hp.n_vocab), 1.0f, 0.0f);
    m.ln0 = vec(0.05f, 1.0f); m.ln0_b = vec(0.05f, 0.0f);
    m.out_norm = vec(0.05f, 1.0f); m.out_norm_b = vec(0.05f, 0.0f);
    m.lm_head = w(ggml_new_tensor_2d(c, GGML_TYPE_Q6_K, E, hp.n_vocab), se, 0.0f);
    m.layers.resize(hp.n_layer);
    for (layer & l : m.layers) {
        l.ln1 = vec(0.05f, 1.0f); l.ln1_b = vec(0.05f, 0.0f); l.ln2 = vec(0.05f, 1.0f); l.ln2_b = vec(0.05f, 0.0f);
        l.lerp_x = w(ggml_new_tensor_1d(c, GGML_TYPE_F32, E), 0.0f, 0.0f, FILL_UNIT);
        for (ggml_tensor *& t : l.lerp) t = w(ggml_new_tensor_1d(c, GGML_TYPE_F32, E), 0.0f, 0.0f, FILL_UNIT);
        l.w1 = w(ggml_new_tensor_2d(c, GGML_TYPE_F32, E, 5 * hp.lora_mix), 0.5f * se, 0.0f);
        l.w2 = w(ggml_new_tensor_3d(c, GGML_TYPE_F32, hp.lora_mix, E, 5), 0.1f, 0.0f);
        l.dw1 = w(ggml_new_tensor_2d(c, GGML_TYPE_F32, E, hp.lora_decay), 0.5f * se, 0.0f);
        l.dw2 = w(ggml_new_tensor_2d(c, GGML_TYPE_F32, hp.lora_decay, E), 0.1f, 0.0f);
        l.time_decay = w(ggml_new_tensor_1d(c, GGML_TYPE_F32, E), 0.0f, 0.0f, FILL_DECAY);
        l.tf = w(ggml_new_tensor_2d(c, GGML_TYPE_F32, S, H), 0.5f, 0.0f);
        l.wr = w(ggml_new_tensor_2d(c, GGML_TYPE_Q4_K, E, E), se, 0.0f);
        l.wk = w(ggml_new_tensor_2d(c, GGML_TYPE_Q4_K, E, E), se, 0.0f);
        l.wv = w(ggml_new_tensor_2d(c, GGML_TYPE_Q4_K, E, E), se, 0.0f);
        l.wg = w(ggml_new_tensor_2d(c, GGML_TYPE_Q4_K, E, E), se, 0.0f);
        l.wo = w(ggml_new_tensor_2d(c, GGML_TYPE_Q4_K, E, E), se, 0.0f);
        l.ln_x = vec(0.05f, 1.0f); l.ln_x_b = vec(0.05f, 0.0f);
        l.c_lerp_k = w(ggml_new_tensor_1d(c, GGML_TYPE_F32, E), 0.0f, 0.0f, FILL_UNIT);
        l.c_lerp_r = w(ggml_new_tensor_1d(c, GGML_TYPE_F32, E), 0.0f, 0.0f, FILL_UNIT);
        l.ck = w(ggml_new_tensor_2d(c, GGML_TYPE_Q4_K, E, F), se, 0.0f);
        l.cv = w(ggml_new_tensor_2d(c, GGML_TYPE_Q6_K, F, E), sf, 0.0f);
        l.cr = w(ggml_new_tensor_2d(c, hp.qrwkv ? GGML_TYPE_Q4_K : GGML_TYPE_Q8_0, E, hp.qrwkv ? F : E), se, 0.0f);
        l.att_shift = ggml_new_tensor_1d(m.ctx_s, GGML_TYPE_F32, E * hp.n_seqs);
        l.ffn_shift = ggml_new_tensor_1d(m.ctx_s, GGML_TYPE_F32, E * hp.n_seqs);
        l.wkv_states = ggml_new_tensor_1d(m.ctx_s, GGML_TYPE_F32, S * S * H * hp.n_seqs);
    }
    m.buf_w = ggml_backend_alloc_ctx_tensors_from_buft(m.ctx_w, bt);
    m.buf_s = ggml_backend_alloc_ctx_tensors_from_buft(m.ctx_s, bt);
    if (!m.buf_w || !m.buf_s) { fprintf(stderr, "model allocation failed\n"); exit(4); }
    ggml_backend_buffer_set_usage(m.buf_w, GGML_BACKEND_BUFFER_USAGE_WEIGHTS);
    ggml_backend_buffer_clear(m.buf_s, 0);

    w.run(20241005u, fill_special);
}

void free_model(model & m) {
    ggml_backend_buffer_free(m.buf_w);
    ggml_backend_buffer_free(m.buf_s);
    ggml_free(m.ctx_w);
    ggml_free(m.ctx_s);
}

// the states of one cache for this batch: rows state_copy of s viewed as [n_state, n_seqs], cleared by state_mask on a fresh sequence
ggml_tensor * copy_mask_state(ggml_context * ctx, ggml_tensor * s, ggml_tensor * state_copy, ggml_tensor * state_mask, int64_t n_state, int n_seqs) {
    ggml_tensor * states = ggml_get_rows(ctx, ggml_reshape_2d(ctx, s, n_state, n_seqs), state_copy);
    return ggml_mul(ctx, states, state_mask);
}

ggml_tensor * layer_norm(ggml_context * ctx, const hparams & hp, ggml_tensor * x, ggml_tensor * w, ggml_tensor * b) {
    if (hp.qrwkv) return ggml_mul(ctx, ggml_rms_norm(ctx, x, hp.eps), w);
    return ggml_add(ctx, ggml_mul(ctx, ggml_norm(ctx, x, hp.eps), w), b);
}

// x_prev - x for x [n_embd, n_t n_seqs]: each sequence's previous token (the cached one for its first token); the last token of each
// sequence goes back to the cache
ggml_tensor * token_shift_delta(ggml_cgraph * gf, ggml_context * ctx, const hparams & hp, ggml_tensor * x, ggml_tensor * cache,
                                ggml_tensor * state_copy, ggml_tensor * state_mask, int n_t) {
    const int64_t E = hp.n_embd, n_seqs = hp.n_seqs;
    ggml_tensor * shift = ggml_reshape_3d(ctx, copy_mask_state(ctx, cache, state_copy, state_mask, E, hp.n_seqs), E, 1, n_seqs);
    ggml_tensor * x3 = ggml_reshape_3d(ctx, x, E, n_t, n_seqs);
    ggml_tensor * prev = ggml_concat(ctx, shift, ggml_view_3d(ctx, x3, E, n_t - 1, n_seqs, x3->nb[1], x3->nb[2], 0), 1);
    ggml_build_forward_expand(gf, ggml_cpy(ctx, ggml_view_3d(ctx, x3, E, 1, n_seqs, x3->nb[1], x3->nb[2], (n_t - 1) * x3->nb[1]),
                                           ggml_view_1d(ctx, cache, E * n_seqs, 0)));
    return ggml_sub(ctx, ggml_reshape_2d(ctx, prev, E, (int64_t) n_t * n_seqs), x);
}

ggml_tensor * time_mix(ggml_cgraph * gf, ggml_context * ctx, const hparams & hp, const layer & l, ggml_tensor * xa, ggml_tensor * state_copy,
                       ggml_tensor * state_mask, int il, int n_t) {
    const int64_t E = hp.n_embd, S = hp.head_size, H = hp.n_head(), n_seqs = hp.n_seqs, T = (int64_t) n_t * n_seqs;
    const std::string sfx = "-" + std::to_string(il);
    ggml_tensor * sx = token_shift_delta(gf, ctx, hp, xa, l.att_shift, state_copy, state_mask, n_t);

    ggml_tensor * xxx = ggml_add(ctx, ggml_mul(ctx, sx, l.lerp_x), xa);
    xxx = ggml_reshape_4d(ctx, ggml_tanh(ctx, ggml_mul_mat(ctx, l.w1, xxx)), hp.lora_mix, 1, 5, T);
    xxx = ggml_cont(ctx, ggml_permute(ctx, xxx, 0, 1, 3, 2));                                  // [32, 1, T, 5]
    xxx = ggml_mul_mat(ctx, ggml_reshape_4d(ctx, l.w2, hp.lora_mix, E, 1, 5), xxx);            // [n_embd, 1, T, 5]
    ggml_tensor * xm[5];
    for (int i = 0; i < 5; ++i) {
        ggml_tensor * mi = ggml_view_2d(ctx, xxx, E, T, xxx->nb[1], (size_t) i * E * T * sizeof(float));
        xm[i] = ggml_add(ctx, ggml_mul(ctx, ggml_add(ctx, mi, l.lerp[i]), sx), xa);            // xw, xk, xv, xr, xg
    }
    ggml_tensor * r = ggml_reshape_3d(ctx, ggml_mul_mat(ctx, l.wr, xm[3]), S, H, T);
    ggml_tensor * k = ggml_reshape_3d(ctx, ggml_mul_mat(ctx, l.wk, xm[1]), S, H, T);
    ggml_tensor * v = ggml_reshape_3d(ctx, ggml_mul_mat(ctx, l.wv, xm[2]), S, H, T);
    ggml_tensor * g = ggml_silu(ctx, ggml_mul_mat(ctx, l.wg, xm[4]));
    ggml_tensor * w = ggml_mul_mat(ctx, l.dw2, ggml_tanh(ctx, ggml_mul_mat(ctx, l.dw1, xm[0])));
    w = ggml_exp(ctx, ggml_neg(ctx, ggml_exp(ctx, ggml_add(ctx, w, l.time_decay))));
    w = ggml_reshape_3d(ctx, w, S, H, T);

    ggml_tensor * state = copy_mask_state(ctx, l.wkv_states, state_copy, state_mask, S * S * H, hp.n_seqs);
    ggml_tensor * wkv;
    if (hp.qrwkv) {
        k = ggml_sub(ctx, k, ggml_mul(ctx, k, w));
        wkv = ggml_gated_linear_attn(ctx, k, v, r, w, state, powf((float) S, -0.5f));
    } else {
        wkv = ggml_rwkv_wkv6(ctx, k, v, r, l.tf, w, state);
    }
    ggml_set_name(wkv, ("wkv" + sfx).c_str());
    ggml_build_forward_expand(gf, ggml_cpy(ctx, ggml_view_1d(ctx, wkv, S * S * H * n_seqs, E * T * sizeof(float)),
                                           ggml_view_1d(ctx, l.wkv_states, S * S * H * n_seqs, 0)));
    ggml_tensor * y = ggml_view_1d(ctx, wkv, E * T, 0);
    if (!hp.qrwkv) {                                                                             // per-head group norm, then ln_x
        y = ggml_norm(ctx, ggml_reshape_3d(ctx, y, S, H, T), 64e-5f);
        y = ggml_add(ctx, ggml_mul(ctx, ggml_reshape_2d(ctx, y, E, T), l.ln_x), l.ln_x_b);
    } else {
        y = ggml_reshape_2d(ctx, y, E, T);
    }
    return ggml_mul_mat(ctx, l.wo, ggml_mul(ctx, y, g));
}

ggml_tensor * channel_mix(ggml_cgraph * gf, ggml_context * ctx, const hparams & hp, const layer & l, ggml_tensor * xf, ggml_tensor * state_copy,
                          ggml_tensor * state_mask, int n_t) {
    if (hp.qrwkv)                                                                                // SwiGLU: down(silu(gate x) * up x)
        return ggml_mul_mat(ctx, l.cv, ggml_mul(ctx, ggml_silu(ctx, ggml_mul_mat(ctx, l.ck, xf)), ggml_mul_mat(ctx, l.cr, xf)));
    ggml_tensor * sx = token_shift_delta(gf, ctx, hp, xf, l.ffn_shift, state_copy, state_mask, n_t);
    ggml_tensor * xk = ggml_add(ctx, ggml_mul(ctx, sx, l.c_lerp_k), xf);
    ggml_tensor * xr = ggml_add(ctx, ggml_mul(ctx, sx, l.c_lerp_r), xf);
    ggml_tensor * r = ggml_sigmoid(ctx, ggml_mul_mat(ctx, l.cr, xr));
    ggml_tensor * k = ggml_sqr(ctx, ggml_relu(ctx, ggml_mul_mat(ctx, l.ck, xk)));
    return ggml_mul(ctx, r, ggml_mul_mat(ctx, l.cv, k));
}

// the token graph for n_t tokens of each sequence; inputs "inp_tokens" (sequence-major), "state_copy", "state_mask"; output "result_output"
ggml_cgraph * build_graph(const model & m, ggml_context * ctx, int n_t) {
    const hparams & hp = m.hp;
    const int N = n_t * hp.n_seqs;
    ggml_cgraph * gf = ggml_new_graph_custom(ctx, GRAPH_SIZE, false);
    ggml_tensor * tok = ggml_new_tensor_1d(ctx, GGML_TYPE_I32, N);
    ggml_set_name(tok, "inp_tokens"); ggml_set_input(tok);
    ggml_tensor * state_copy = ggml_new_tensor_1d(ctx, GGML_TYPE_I32, hp.n_seqs);
    ggml_set_name(state_copy, "state_copy"); ggml_set_input(state_copy);
    ggml_tensor * state_mask = ggml_new_tensor_2d(ctx, GGML_TYPE_F32, 1, hp.n_seqs);
    ggml_set_name(state_mask, "state_mask"); ggml_set_input(state_mask);

    ggml_tensor * x = layer_norm(ctx, hp, ggml_get_rows(ctx, m.tok_embd, tok), m.ln0, m.ln0_b);    // [n_embd, N]
    for (int il = 0; il < hp.n_layer; ++il) {
        const layer & l = m.layers[il];
        x = ggml_add(ctx, time_mix(gf, ctx, hp, l, layer_norm(ctx, hp, x, l.ln1, l.ln1_b), state_copy, state_mask, il, n_t), x);
        x = ggml_add(ctx, channel_mix(gf, ctx, hp, l, layer_norm(ctx, hp, x, l.ln2, l.ln2_b), state_copy, state_mask, n_t), x);
    }
    ggml_tensor * cur = ggml_mul_mat(ctx, m.lm_head, layer_norm(ctx, hp, x, m.out_norm, m.out_norm_b));
    ggml_set_name(cur, "result_output"); ggml_set_output(cur);
    ggml_build_forward_expand(gf, cur);
    return gf;
}

// the first batch (n_past 0) starts every sequence from a cleared state
void set_inputs(const hparams & hp, ggml_cgraph * gf, int n_past, const std::vector<int32_t> & toks) {
    ggml_backend_tensor_set(ggml_graph_get_tensor(gf, "inp_tokens"), toks.data(), 0, toks.size() * sizeof(int32_t));
    std::vector<int32_t> copy(hp.n_seqs);
    std::vector<float> mask(hp.n_seqs, n_past == 0 ? 0.0f : 1.0f);
    for (int s = 0; s < hp.n_seqs; ++s) copy[s] = s;
    ggml_backend_tensor_set(ggml_graph_get_tensor(gf, "state_copy"), copy.data(), 0, copy.size() * sizeof(int32_t));
    ggml_backend_tensor_set(ggml_graph_get_tensor(gf, "state_mask"), mask.data(), 0, mask.size() * sizeof(float));
}


} // namespace

int main(int argc, char ** argv) {
    model m;
    return decoder_main(argc, argv, [&m](const std::string & name) {
        m.hp = preset(name);
        // 4-token prompts: the projections take the whole batch as one [n_embd, n_t n_seqs] matrix, so 4 tokens keep every quantized
        // mat-mul at n <= 8, on the device's mat-vec path whose integer dot products match ggml-cpu's exactly (a wider batch takes the
        // fp16-operand GEMM, which agrees only to its own tolerance and would hide the recurrence's deviations behind it)
        const std::vector<int32_t> p[2] = { { 1, 417, 2093, 58 }, { 1, 96, 3333, 1024 } };
        decoder d;
        d.n_seqs = m.hp.n_seqs;
        d.n_vocab = m.hp.n_vocab;
        d.graph_size = GRAPH_SIZE;
        for (int s = 0; s < m.hp.n_seqs; ++s) d.prompt.insert(d.prompt.end(), p[s % 2].begin(), p[s % 2].end());
        d.build_model = [&m](ggml_backend_buffer_type_t bt) { build_model(m, bt); };
        d.free_model = [&m] { free_model(m); };
        d.build_graph = [&m](ggml_context * ctx, int, int n_t) { return build_graph(m, ctx, n_t); };
        d.set_inputs = [&m](ggml_cgraph * gf, int n_past, const std::vector<int32_t> & toks) { set_inputs(m.hp, gf, n_past, toks); };
        return d;
    });
}
