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
// usage: rwkv-graph PRESET compare DEVICE [sync]
//          ggml_backend_compare_graph_backend of ggml-cpu against DEVICE over the prompt and one decode step.  Prints
//          "node PHASE INDEX OP NAME [ne] nmse E" per contiguous f32 node, then per phase
//          "summary PHASE sync|free nodes_over_1e-9 N worst W first_over INDEX OP logits L".
//          With "sync" the device copy of each node result is replaced by the CPU's after the comparison.
//        rwkv-graph PRESET run DEVICE STEPS LOGITS_OUT [FORCE_TOKENS]
//          ggml_backend_sched over [DEVICE, CPU], the prompt, then STEPS - 1 decode steps; writes per step the logits of each sequence's
//          last token (STEPS x n_seqs rows of n_vocab f32) and prints "n_splits S", "cpu_nodes C", "tokens t0 t1 ..." (step-major, one per
//          sequence and step) and "decode_ms_per_step M".  FORCE_TOKENS: i32 tokens in the same order, fed instead of the greedy ones.
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
#include <thread>
#include <vector>

namespace {

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

// create the tensors of the model in ctx_w / ctx_s, allocate them in buffers of `bt`, fill the weights from fixed seeds
void build_model(model & m, ggml_backend_buffer_type_t bt) {
    const hparams & hp = m.hp;
    const size_t n_t = 8 + 40 * (size_t) hp.n_layer;
    ggml_init_params ip = { ggml_tensor_overhead() * n_t, nullptr, true };
    m.ctx_w = ggml_init(ip);
    m.ctx_s = ggml_init(ip);
    ggml_context * c = m.ctx_w;
    struct fill_job { ggml_tensor * t; float scale, offset; fill_kind kind; };
    std::vector<fill_job> jobs;
    auto w = [&](ggml_tensor * t, float scale, float offset, fill_kind kind = FILL_NORMAL) { jobs.push_back({ t, scale, offset, kind }); return t; };
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

    // tensor j is drawn from its own generator (seed 20241005 + j), so the parallel fill is deterministic
    std::vector<std::vector<uint8_t>> bytes(jobs.size());
    auto fill = [&](size_t j) {
        const ggml_tensor * t = jobs[j].t;
        std::mt19937 rng(20241005u + (unsigned) j);
        std::normal_distribution<float> nd(0.0f, 1.0f);
        std::uniform_real_distribution<float> unit(0.0f, 1.0f), decay(-6.0f, 0.5f);
        const int64_t n = ggml_nelements(t), k = t->ne[0];
        std::vector<float> x((size_t) n);
        for (int64_t i = 0; i < n; ++i) {
            switch (jobs[j].kind) {
                case FILL_UNIT: x[(size_t) i] = unit(rng); break;
                case FILL_DECAY: x[(size_t) i] = decay(rng); break;                    // exp(-exp(.)) from ~0.998 down to ~0.19 per token
                default: x[(size_t) i] = jobs[j].offset + jobs[j].scale * nd(rng); break;
            }
        }
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
    ggml_cgraph * gf = ggml_new_graph_custom(ctx, 8192, false);
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

void set_inputs(const hparams & hp, ggml_cgraph * gf, bool first, const std::vector<int32_t> & toks) {
    ggml_backend_tensor_set(ggml_graph_get_tensor(gf, "inp_tokens"), toks.data(), 0, toks.size() * sizeof(int32_t));
    std::vector<int32_t> copy(hp.n_seqs);
    std::vector<float> mask(hp.n_seqs, first ? 0.0f : 1.0f);
    for (int s = 0; s < hp.n_seqs; ++s) copy[s] = s;
    ggml_backend_tensor_set(ggml_graph_get_tensor(gf, "state_copy"), copy.data(), 0, copy.size() * sizeof(int32_t));
    ggml_backend_tensor_set(ggml_graph_get_tensor(gf, "state_mask"), mask.data(), 0, mask.size() * sizeof(float));
}

// the prompts, sequence-major: n_seqs x 4 tokens.  The projections take the whole batch as one [n_embd, n_t n_seqs] matrix, so 4 tokens
// keep every quantized mat-mul at n <= 8, on the device's mat-vec path whose integer dot products match ggml-cpu's exactly (a wider batch
// takes the fp16-operand GEMM, which agrees only to its own tolerance and would hide the recurrence's deviations behind it)
std::vector<int32_t> prompt_tokens(const hparams & hp) {
    const std::vector<int32_t> p[2] = { { 1, 417, 2093, 58 }, { 1, 96, 3333, 1024 } };
    std::vector<int32_t> out;
    for (int s = 0; s < hp.n_seqs; ++s) out.insert(out.end(), p[s % 2].begin(), p[s % 2].end());
    return out;
}
const int PROMPT_LEN = 4;

// ------------------------------------------------------------------ compare
struct cmp_state { const char * tag; int n_bad; double worst; bool sync; int first_bad; char first_bad_op[64]; double logits; };

double nmse_f32(const float * a, const float * b, size_t n) {       // as tests/test-backend-ops.cpp computes it (a = device, b = cpu)
    double num = 0.0, den = 0.0;
    for (size_t i = 0; i < n; ++i) { const double d = (double) a[i] - (double) b[i]; num += d * d; den += (double) a[i] * (double) a[i]; }
    return den > 0.0 ? num / den : num;
}

bool on_node(int index, ggml_tensor * t1, ggml_tensor * t2, void * ud) {
    cmp_state * st = (cmp_state *) ud;
    if (!ggml_is_contiguous(t1) || t1->type != GGML_TYPE_F32) return true;     // views: compared through their consumers
    const size_t n = (size_t) ggml_nelements(t1);
    std::vector<float> a(n), b(n);
    ggml_backend_tensor_get(t1, b.data(), 0, n * sizeof(float));                    // t1: CPU
    ggml_backend_tensor_get(t2, a.data(), 0, n * sizeof(float));                    // t2: device
    const double e = nmse_f32(a.data(), b.data(), n);
    if (e > st->worst) st->worst = e;
    if (e > 1e-9) { if (st->n_bad == 0) { st->first_bad = index; snprintf(st->first_bad_op, sizeof(st->first_bad_op), "%s", ggml_op_desc(t1)); } st->n_bad++; }
    if (strcmp(t1->name, "result_output") == 0) st->logits = e;
    if (st->sync) ggml_backend_tensor_set(t2, b.data(), 0, n * sizeof(float));
    printf("node %s %d %s %s [%" PRId64 ",%" PRId64 ",%" PRId64 ",%" PRId64 "] nmse %.3e\n", st->tag, index, ggml_op_desc(t1), t1->name,
           t1->ne[0], t1->ne[1], t1->ne[2], t1->ne[3], e);
    return true;
}

int run_compare(model & m, ggml_backend_t cpu, ggml_backend_t dev, bool sync) {
    const hparams & hp = m.hp;
    ggml_gallocr_t allocr = ggml_gallocr_new(ggml_backend_get_default_buffer_type(cpu));
    int rc = 0;
    for (int phase = 0; phase < 2 && rc == 0; ++phase) {
        const int n_t = phase == 0 ? PROMPT_LEN : 1;
        std::vector<int32_t> toks = prompt_tokens(hp);
        if (phase == 1) { toks.clear(); for (int s = 0; s < hp.n_seqs; ++s) toks.push_back(99 + 11 * s); }
        ggml_init_params ip = { ggml_tensor_overhead() * 8192 + ggml_graph_overhead_custom(8192, false), nullptr, true };
        ggml_context * ctx = ggml_init(ip);
        ggml_cgraph * gf = build_graph(m, ctx, n_t);
        ggml_gallocr_alloc_graph(allocr, gf);
        set_inputs(hp, gf, phase == 0, toks);
        cmp_state st{ phase == 0 ? "prompt" : "decode", 0, 0.0, sync, -1, "", -1.0 };
        // the CPU evaluation also advances the CPU-side state caches that the decode phase copies over
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
    ggml_backend_t backends[2] = { dev, cpu };
    const int n_be = dev == cpu ? 1 : 2;
    ggml_backend_sched_t sched = ggml_backend_sched_new(backends, nullptr, n_be, 8192, false);
    FILE * out = fopen(out_path, "wb");
    if (!out) { fprintf(stderr, "cannot open %s\n", out_path); return 6; }
    std::vector<float> logits(hp.n_vocab);
    std::vector<int32_t> generated;
    int max_splits = 0, max_cpu_nodes = 0;
    double decode_s = 0.0;
    int n_decode = 0;
    std::vector<int32_t> toks = prompt_tokens(hp);
    for (int step = 0; step < steps; ++step) {
        const int n_t = step == 0 ? PROMPT_LEN : 1;
        ggml_init_params ip = { ggml_tensor_overhead() * 8192 + ggml_graph_overhead_custom(8192, false), nullptr, true };
        ggml_context * ctx = ggml_init(ip);
        ggml_cgraph * gf = build_graph(m, ctx, n_t);
        ggml_backend_sched_reset(sched);
        if (!ggml_backend_sched_alloc_graph(sched, gf)) { fprintf(stderr, "sched alloc failed\n"); return 7; }
        set_inputs(hp, gf, step == 0, toks);
        const auto t0 = std::chrono::steady_clock::now();
        if (ggml_backend_sched_graph_compute(sched, gf) != GGML_STATUS_SUCCESS) { fprintf(stderr, "compute failed\n"); return 8; }
        ggml_tensor * res = ggml_graph_get_tensor(gf, "result_output");
        std::vector<int32_t> next(hp.n_seqs);
        for (int s = 0; s < hp.n_seqs; ++s) {
            const size_t row = (size_t) s * n_t + n_t - 1;                         // each sequence's last token
            ggml_backend_tensor_get(res, logits.data(), row * hp.n_vocab * sizeof(float), hp.n_vocab * sizeof(float));
            fwrite(logits.data(), sizeof(float), logits.size(), out);
            int32_t best = 0;
            for (int i = 1; i < hp.n_vocab; ++i) if (logits[i] > logits[best]) best = i;
            const size_t k = (size_t) step * hp.n_seqs + s;
            next[s] = k < force.size() ? force[k] : best;
        }
        const double dt = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
        if (step >= 2) { decode_s += dt; ++n_decode; }                       // step 0: prompt; step 1: first decode (warm-up)
        int cpu_nodes = 0;
        for (int i = 0; i < ggml_graph_n_nodes(gf); ++i)
            if (n_be == 2 && ggml_backend_sched_get_tensor_backend(sched, ggml_graph_node(gf, i)) == cpu) ++cpu_nodes;
        if (ggml_backend_sched_get_n_splits(sched) > max_splits) max_splits = ggml_backend_sched_get_n_splits(sched);
        if (cpu_nodes > max_cpu_nodes) max_cpu_nodes = cpu_nodes;
        generated.insert(generated.end(), next.begin(), next.end());
        toks = next;
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
    ggml_backend_cpu_set_n_threads(cpu, 8);                 // <= the head count: see the note on WKV6 / GLA above
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
    ggml_backend_buffer_free(m.buf_s);
    ggml_free(m.ctx_w);
    ggml_free(m.ctx_s);
    if (dev != cpu) ggml_backend_free(dev);
    ggml_backend_free(cpu);
    return rc;
}
