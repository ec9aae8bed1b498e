// oracle/mamba_graph.cpp — TEST INFRASTRUCTURE ONLY.
//
// A synthetic Mamba-1 decoder built in memory on the reference's public API (ggml.h, ggml-alloc.h, ggml-backend.h).  Each layer is
// llama.cpp's llm_build_mamba form, over n_seqs sequences of n_t tokens each:
//   cur   = RMS_NORM(inp) * norm
//   xz    = MUL_MAT(ssm_in, cur)                                   x, z = the two d_inner halves (views)
//   conv  = GET_ROWS(conv_states, state_copy) * state_mask         -> [d_conv - 1, d_inner, n_seqs]
//   cx    = CONCAT(conv, TRANSPOSE(x), 0);  CPY(last d_conv - 1 columns of cx -> conv_states)
//   x     = SILU(ADD(SSM_CONV(cx, conv1d), conv1d_b))
//   x_db  = MUL_MAT(ssm_x, x)                                      dt, B, C = views of x_db (falcon: RMS_NORM each)
//   dt    = ADD(MUL_MAT(ssm_dt, dt), ssm_dt_b)
//   ssm   = GET_ROWS(ssm_states, state_copy) * state_mask          -> [d_state, d_inner, n_seqs]
//   y_ssm = SSM_SCAN(ssm, x, dt, A, B, C);  CPY(state part of y_ssm -> ssm_states)
//   y     = (y + x * D) * SILU(CONT(z));   out = MUL_MAT(ssm_out, y) + inp
// A = -(i0 + 1) (the S4D-real initialisation); the dt bias is the inverse softplus of values log-uniform in [1e-3, 1e-1], so the
// recurrence decays as a trained model's does.  The conv and ssm state caches live in a buffer of the evaluating device (like the KV
// cache of the other programs); state_mask is 0 on the prompt and 1 afterwards.  Other weights come from fixed seeds (one per tensor,
// filled in parallel) and are quantized with ggml_quantize_chunk.  Q4_K token embeddings, a Q6_K lm_head, 4 layers, vocabulary 4096.
//
// Presets:
//   mamba   Mamba-130m widths: n_embd 768, d_inner 1536, d_state 16, d_conv 4, dt_rank 48; ssm_in / ssm_out Q4_K, ssm_x Q8_0, ssm_dt f32
//           (K = 48 fits no block format: the float mat-mul on a strided src1); two sequences decode side by side, 7-token prompts
//   falcon  FalconMamba form: n_embd 1024, d_inner 2048, d_state 16, d_conv 4, dt_rank 64, RMS_NORM on the dt / B / C views, ssm_x and
//           ssm_dt Q8_0; one sequence
//
// usage: mamba-graph PRESET compare DEVICE [sync] | PRESET run DEVICE STEPS LOGITS_OUT [FORCE_TOKENS]  (decoder_harness.h), n_seqs
// sequences with 7-token prompts.

#include "decoder_harness.h"

#include <cmath>

namespace {

struct hparams {
    int n_embd = 768, d_inner = 1536, d_state = 16, d_conv = 4, dt_rank = 48, n_layer = 4, n_vocab = 4096, n_seqs = 2;
    bool falcon = false;
    ggml_type ssm_dt_type = GGML_TYPE_F32;
    float eps = 1e-5f;
};

struct layer {
    ggml_tensor * norm, * ssm_in, * conv1d, * conv1d_b, * ssm_x, * ssm_dt, * ssm_dt_b, * ssm_a, * ssm_d, * ssm_out;
    ggml_tensor * conv_states, * ssm_states;                   // f32 [(d_conv - 1) * d_inner * n_seqs], [d_state * d_inner * n_seqs]
};

struct model {
    hparams hp;
    ggml_context * ctx_w = nullptr, * ctx_s = nullptr;
    ggml_backend_buffer_t buf_w = nullptr, buf_s = nullptr;
    ggml_tensor * tok_embd, * out_norm, * lm_head;
    std::vector<layer> layers;
};

hparams preset(const std::string & name) {
    hparams hp;
    if (name == "falcon") {
        hp.n_embd = 1024; hp.d_inner = 2048; hp.dt_rank = 64; hp.n_seqs = 1; hp.falcon = true; hp.ssm_dt_type = GGML_TYPE_Q8_0;
    } else if (name != "mamba") {
        fprintf(stderr, "unknown preset %s (mamba | falcon)\n", name.c_str());
        exit(2);
    }
    return hp;
}

enum fill_kind { FILL_NORMAL, FILL_A, FILL_DT_BIAS };

float fill_special(int kind, int64_t i, int64_t k, std::mt19937 & rng) {
    if (kind == FILL_A) return -(float) (i % k + 1);                                                    // A[i0, i1] = -(i0 + 1)
    const double dt = exp(std::uniform_real_distribution<double>(log(1e-3), log(1e-1))(rng));          // softplus^-1(dt) = dt + log(-expm1(-dt))
    return (float) (dt + log(-expm1(-dt)));
}

// create the tensors of the model in ctx_w / ctx_s, allocate them in buffers of `bt`, fill the weights from fixed seeds
void build_model(model & m, ggml_backend_buffer_type_t bt) {
    const hparams & hp = m.hp;
    const size_t n_t = 4 + 12 * (size_t) hp.n_layer;
    ggml_init_params ip = { ggml_tensor_overhead() * n_t, nullptr, true };
    m.ctx_w = ggml_init(ip);
    m.ctx_s = ggml_init(ip);
    ggml_context * c = m.ctx_w;
    weight_fill w;
    const float se = 1.0f / sqrtf((float) hp.n_embd), si = 1.0f / sqrtf((float) hp.d_inner);
    m.tok_embd = w(ggml_new_tensor_2d(c, GGML_TYPE_Q4_K, hp.n_embd, hp.n_vocab), 1.0f, 0.0f);
    m.out_norm = w(ggml_new_tensor_1d(c, GGML_TYPE_F32, hp.n_embd), 0.05f, 1.0f);
    m.lm_head = w(ggml_new_tensor_2d(c, GGML_TYPE_Q6_K, hp.n_embd, hp.n_vocab), se, 0.0f);
    m.layers.resize(hp.n_layer);
    for (layer & l : m.layers) {
        l.norm = w(ggml_new_tensor_1d(c, GGML_TYPE_F32, hp.n_embd), 0.05f, 1.0f);
        l.ssm_in = w(ggml_new_tensor_2d(c, GGML_TYPE_Q4_K, hp.n_embd, 2 * hp.d_inner), se, 0.0f);
        l.conv1d = w(ggml_new_tensor_2d(c, GGML_TYPE_F32, hp.d_conv, hp.d_inner), 1.0f / sqrtf((float) hp.d_conv), 0.0f);
        l.conv1d_b = w(ggml_new_tensor_1d(c, GGML_TYPE_F32, hp.d_inner), 0.1f, 0.0f);
        l.ssm_x = w(ggml_new_tensor_2d(c, GGML_TYPE_Q8_0, hp.d_inner, hp.dt_rank + 2 * hp.d_state), si, 0.0f);
        l.ssm_dt = w(ggml_new_tensor_2d(c, hp.ssm_dt_type, hp.dt_rank, hp.d_inner), 0.5f / sqrtf((float) hp.dt_rank), 0.0f);
        l.ssm_dt_b = w(ggml_new_tensor_1d(c, GGML_TYPE_F32, hp.d_inner), 0.0f, 0.0f, FILL_DT_BIAS);
        l.ssm_a = w(ggml_new_tensor_2d(c, GGML_TYPE_F32, hp.d_state, hp.d_inner), 0.0f, 0.0f, FILL_A);
        l.ssm_d = w(ggml_new_tensor_1d(c, GGML_TYPE_F32, hp.d_inner), 0.1f, 1.0f);
        l.ssm_out = w(ggml_new_tensor_2d(c, GGML_TYPE_Q4_K, hp.d_inner, hp.n_embd), si, 0.0f);
        l.conv_states = ggml_new_tensor_1d(m.ctx_s, GGML_TYPE_F32, (int64_t) (hp.d_conv - 1) * hp.d_inner * hp.n_seqs);
        l.ssm_states = ggml_new_tensor_1d(m.ctx_s, GGML_TYPE_F32, (int64_t) hp.d_state * hp.d_inner * hp.n_seqs);
    }
    m.buf_w = ggml_backend_alloc_ctx_tensors_from_buft(m.ctx_w, bt);
    m.buf_s = ggml_backend_alloc_ctx_tensors_from_buft(m.ctx_s, bt);
    if (!m.buf_w || !m.buf_s) { fprintf(stderr, "model allocation failed\n"); exit(4); }
    ggml_backend_buffer_set_usage(m.buf_w, GGML_BACKEND_BUFFER_USAGE_WEIGHTS);
    ggml_backend_buffer_clear(m.buf_s, 0);

    w.run(20240917u, fill_special);
}

void free_model(model & m) {
    ggml_backend_buffer_free(m.buf_w);
    ggml_backend_buffer_free(m.buf_s);
    ggml_free(m.ctx_w);
    ggml_free(m.ctx_s);
}

// the states of one cache for this batch: rows state_copy of s viewed as [n_state, n_seqs], cleared by state_mask on a fresh sequence
// (llama.cpp's llm_build_copy_mask_state with every cell in use)
ggml_tensor * copy_mask_state(ggml_context * ctx, ggml_tensor * s, ggml_tensor * state_copy, ggml_tensor * state_mask, int64_t n_state, int n_seqs) {
    ggml_tensor * states = ggml_get_rows(ctx, ggml_reshape_2d(ctx, s, n_state, n_seqs), state_copy);
    return ggml_mul(ctx, states, state_mask);
}

// the Mamba block of layer l on cur [n_embd, n_t, n_seqs] (llama.cpp's llm_build_mamba)
ggml_tensor * mamba_block(ggml_cgraph * gf, const hparams & hp, const layer & l, ggml_context * ctx, ggml_tensor * cur, ggml_tensor * state_copy,
                          ggml_tensor * state_mask, int il, int n_t) {
    const int64_t d_conv = hp.d_conv, d_inner = hp.d_inner, d_state = hp.d_state, dt_rank = hp.dt_rank, n_seqs = hp.n_seqs;
    const std::string sfx = "-" + std::to_string(il);
    ggml_tensor * conv = copy_mask_state(ctx, l.conv_states, state_copy, state_mask, (d_conv - 1) * d_inner, hp.n_seqs);
    conv = ggml_reshape_3d(ctx, conv, d_conv - 1, d_inner, n_seqs);
    ggml_tensor * ssm = copy_mask_state(ctx, l.ssm_states, state_copy, state_mask, d_state * d_inner, hp.n_seqs);
    ssm = ggml_reshape_3d(ctx, ssm, d_state, d_inner, n_seqs);

    ggml_tensor * xz = ggml_mul_mat(ctx, l.ssm_in, cur);                                            // [2 d_inner, n_t, n_seqs]
    ggml_tensor * x = ggml_view_3d(ctx, xz, d_inner, xz->ne[1], xz->ne[2], xz->nb[1], xz->nb[2], 0);
    ggml_tensor * z = ggml_view_3d(ctx, xz, d_inner, xz->ne[1], xz->ne[2], xz->nb[1], xz->nb[2], d_inner * ggml_element_size(xz));

    ggml_tensor * conv_x = ggml_concat(ctx, conv, ggml_transpose(ctx, x), 0);                       // [d_conv - 1 + n_t, d_inner, n_seqs]
    ggml_set_name(conv_x, ("conv_x" + sfx).c_str());
    ggml_tensor * last_conv = ggml_view_3d(ctx, conv_x, d_conv - 1, d_inner, n_seqs, conv_x->nb[1], conv_x->nb[2], n_t * conv_x->nb[0]);
    ggml_build_forward_expand(gf, ggml_cpy(ctx, last_conv, ggml_view_1d(ctx, l.conv_states, (d_conv - 1) * d_inner * n_seqs, 0)));
    x = ggml_ssm_conv(ctx, conv_x, l.conv1d);
    ggml_set_name(x, ("ssm_conv" + sfx).c_str());
    x = ggml_silu(ctx, ggml_add(ctx, x, l.conv1d_b));

    ggml_tensor * x_db = ggml_mul_mat(ctx, l.ssm_x, x);                                             // [dt_rank + 2 d_state, n_t, n_seqs]
    ggml_tensor * dt = ggml_view_3d(ctx, x_db, dt_rank, n_t, n_seqs, x_db->nb[1], x_db->nb[2], 0);
    ggml_tensor * B = ggml_view_3d(ctx, x_db, d_state, n_t, n_seqs, x_db->nb[1], x_db->nb[2], ggml_element_size(x_db) * dt_rank);
    ggml_tensor * C = ggml_view_3d(ctx, x_db, d_state, n_t, n_seqs, x_db->nb[1], x_db->nb[2], ggml_element_size(x_db) * (dt_rank + d_state));
    if (hp.falcon) {
        dt = ggml_rms_norm(ctx, dt, hp.eps);
        B = ggml_rms_norm(ctx, B, hp.eps);
        C = ggml_rms_norm(ctx, C, hp.eps);
    }
    dt = ggml_add(ctx, ggml_mul_mat(ctx, l.ssm_dt, dt), l.ssm_dt_b);                                 // [d_inner, n_t, n_seqs]

    ggml_tensor * y_ssm = ggml_ssm_scan(ctx, ssm, x, dt, l.ssm_a, B, C);
    ggml_set_name(y_ssm, ("ssm_scan" + sfx).c_str());
    ggml_build_forward_expand(gf, ggml_cpy(ctx, ggml_view_1d(ctx, y_ssm, d_state * d_inner * n_seqs, x->nb[3]),
                                           ggml_view_1d(ctx, l.ssm_states, d_state * d_inner * n_seqs, 0)));
    ggml_tensor * y = ggml_view_3d(ctx, y_ssm, d_inner, n_t, n_seqs, x->nb[1], x->nb[2], 0);
    y = ggml_add(ctx, y, ggml_mul(ctx, x, l.ssm_d));
    y = ggml_mul(ctx, y, ggml_silu(ctx, ggml_cont(ctx, z)));
    return ggml_mul_mat(ctx, l.ssm_out, y);                                                          // [n_embd, n_t, n_seqs]
}

// the token graph for n_t tokens of each sequence; inputs "inp_tokens" (sequence-major), "state_copy", "state_mask"; output "result_output"
ggml_cgraph * build_graph(const model & m, ggml_context * ctx, int n_t) {
    const hparams & hp = m.hp;
    const int N = n_t * hp.n_seqs;
    ggml_cgraph * gf = ggml_new_graph_custom(ctx, 4096, false);
    ggml_tensor * tok = ggml_new_tensor_1d(ctx, GGML_TYPE_I32, N);
    ggml_set_name(tok, "inp_tokens"); ggml_set_input(tok);
    ggml_tensor * state_copy = ggml_new_tensor_1d(ctx, GGML_TYPE_I32, hp.n_seqs);
    ggml_set_name(state_copy, "state_copy"); ggml_set_input(state_copy);
    ggml_tensor * state_mask = ggml_new_tensor_2d(ctx, GGML_TYPE_F32, 1, hp.n_seqs);
    ggml_set_name(state_mask, "state_mask"); ggml_set_input(state_mask);

    ggml_tensor * inpL = ggml_get_rows(ctx, m.tok_embd, tok);                                       // [n_embd, N]
    for (int il = 0; il < hp.n_layer; ++il) {
        const layer & l = m.layers[il];
        ggml_tensor * cur = ggml_mul(ctx, ggml_rms_norm(ctx, inpL, hp.eps), l.norm);
        cur = ggml_reshape_3d(ctx, cur, hp.n_embd, n_t, hp.n_seqs);
        cur = mamba_block(gf, hp, l, ctx, cur, state_copy, state_mask, il, n_t);
        inpL = ggml_add(ctx, ggml_reshape_2d(ctx, cur, hp.n_embd, N), inpL);
    }
    ggml_tensor * cur = ggml_mul(ctx, ggml_rms_norm(ctx, inpL, hp.eps), m.out_norm);
    cur = ggml_mul_mat(ctx, m.lm_head, cur);
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
        const std::vector<int32_t> p[2] = { { 1, 417, 2093, 58, 3001, 777, 12 }, { 1, 96, 3333, 1024, 7, 2500, 640 } };
        decoder d;
        d.n_seqs = m.hp.n_seqs;
        d.n_vocab = m.hp.n_vocab;
        for (int s = 0; s < m.hp.n_seqs; ++s) d.prompt.insert(d.prompt.end(), p[s % 2].begin(), p[s % 2].end());
        d.build_model = [&m](ggml_backend_buffer_type_t bt) { build_model(m, bt); };
        d.free_model = [&m] { free_model(m); };
        d.build_graph = [&m](ggml_context * ctx, int, int n_t) { return build_graph(m, ctx, n_t); };
        d.set_inputs = [&m](ggml_cgraph * gf, int n_past, const std::vector<int32_t> & toks) { set_inputs(m.hp, gf, n_past, toks); };
        return d;
    });
}
