// oracle/whisper_graph.cpp — TEST INFRASTRUCTURE ONLY.
//
// A synthetic Whisper-style encoder-decoder built in memory on the reference's public API (ggml.h, ggml-alloc.h, ggml-backend.h), in
// whisper.cpp's form, over one sequence:
//   encoder (the prompt phase, n_past == 0), on a log-mel input [3000 frames, n_mels] that set_inputs fills from a seed:
//     cur = GELU(conv_1d_ph(conv1, mel, stride 1) + conv1_b);  cur = GELU(conv_1d_ph(conv2, cur, stride 2) + conv2_b)    [1500, n_state]
//           (each conv_1d is IM2COL (f16 columns) + MUL_MAT(columns, kernel): f16 x f16)
//     cur = CONT(TRANSPOSE(cur)) + positional embedding                                                                   [n_state, 1500]
//     n_audio_layer x pre-LN blocks: x += Wo attn(LN(x)); x += fc2 GELU(fc1 LN(x))          (LN: NORM * w + b; linears with biases)
//     enc = LN_post(x); then every decoder layer's cross-attention K = Wk enc, V = Wv enc + b written into f16 device caches
//   decoder (every phase), on the tokens at positions n_past ..:
//     x = GET_ROWS(token embedding) + VIEW(positional embedding);  n_text_layer x [x += self-attn(LN(x)) over the f16 KV cache (causal
//     mask); x += cross-attn(LN(x)) over the cached K / V of the 1500 audio frames; x += MLP(LN(x))];  logits = token embedding . LN(x)
// Weights come from fixed seeds (one per tensor, filled in parallel) and are stored f16 or quantized with ggml_quantize_chunk.
// Vocabulary 4096, text context 64, a 4-token prompt.
//
// Presets (both decode one sequence with 3000 mel frames, an audio context of 1500):
//   tiny   80 mels, 384 wide, 6 heads, 4 + 4 layers, f16 conv kernels, Q8_0 linears and token embedding; attention as
//          MUL_MAT(K, Q) -> SOFT_MAX_EXT -> MUL_MAT(V^T, KQ).  conv1 (K = 240) takes the plain f16 x f16 kernel, conv2 (K = 1152) the
//          tensor cores
//   large  128 mels, 1280 wide, 20 heads, 2 + 2 layers, f16 conv kernels, linears and token embedding; attention through FLASH_ATTN_EXT
//          (encoder K / V copied to f16).  Both convs (K = 384, 3840) take the tensor cores
//
// usage: whisper-graph PRESET compare DEVICE [sync] | PRESET run DEVICE STEPS LOGITS_OUT [FORCE_TOKENS]  (decoder_harness.h).  Each graph
// built also prints "graph PHASE nodes N im2col I" (I: its IM2COL nodes; their f16 results are compared through their consumers).

#include "decoder_harness.h"

#include <cmath>

namespace {

struct hparams {
    int n_mels = 80, n_frames = 3000, n_state = 384, n_head = 6, n_audio_layer = 4, n_text_layer = 4, n_vocab = 4096, n_text_ctx = 64;
    ggml_type wtype = GGML_TYPE_Q8_0;                          // linears and token embedding
    bool flash_attn = false;
    float eps = 1e-5f;
    int n_audio_ctx() const { return n_frames / 2; }
    int head_dim() const { return n_state / n_head; }
};

struct linear { ggml_tensor * w, * b; };                      // b may be null
struct norm { ggml_tensor * w, * b; };

struct enc_layer { norm ln0, ln1; linear q, k, v, o, fc1, fc2; };
struct dec_layer {
    norm ln0, ln1, ln2; linear q, k, v, o, cq, ck, cv, co, fc1, fc2;
    ggml_tensor * k_cache, * v_cache;                          // self attention: f16 [n_state * n_text_ctx]
    ggml_tensor * ck_cache, * cv_cache;                        // cross attention: f16 [n_state * n_audio_ctx]
};

struct model {
    hparams hp;
    ggml_context * ctx_w = nullptr, * ctx_s = nullptr;
    ggml_backend_buffer_t buf_w = nullptr, buf_s = nullptr;
    ggml_tensor * conv1_w, * conv1_b, * conv2_w, * conv2_b, * enc_pos, * tok_embd, * dec_pos;
    norm ln_post, ln_dec;
    std::vector<enc_layer> enc;
    std::vector<dec_layer> dec;
};

hparams preset(const std::string & name) {
    hparams hp;
    if (name == "large") {
        hp.n_mels = 128; hp.n_state = 1280; hp.n_head = 20; hp.n_audio_layer = 2; hp.n_text_layer = 2; hp.wtype = GGML_TYPE_F16; hp.flash_attn = true;
    } else if (name != "tiny") {
        fprintf(stderr, "unknown preset %s (tiny | large)\n", name.c_str());
        exit(2);
    }
    return hp;
}

void build_model(model & m, ggml_backend_buffer_type_t bt) {
    const hparams & hp = m.hp;
    const int64_t ns = hp.n_state, nff = 4 * ns;
    const size_t n_t = 16 + 20 * (size_t) hp.n_audio_layer + 40 * (size_t) hp.n_text_layer;
    ggml_init_params ip = { ggml_tensor_overhead() * n_t, nullptr, true };
    m.ctx_w = ggml_init(ip);
    m.ctx_s = ggml_init(ip);
    ggml_context * c = m.ctx_w;
    weight_fill w;
    const float se = 1.0f / sqrtf((float) ns);
    auto lin = [&](int64_t in, int64_t out, bool bias, float scale) {
        linear l;
        l.w = w(ggml_new_tensor_2d(c, hp.wtype, in, out), scale, 0.0f);
        l.b = bias ? w(ggml_new_tensor_1d(c, GGML_TYPE_F32, out), 0.05f, 0.0f) : nullptr;
        return l;
    };
    auto ln = [&]() { norm n; n.w = w(ggml_new_tensor_1d(c, GGML_TYPE_F32, ns), 0.05f, 1.0f); n.b = w(ggml_new_tensor_1d(c, GGML_TYPE_F32, ns), 0.05f, 0.0f); return n; };
    m.conv1_w = w(ggml_new_tensor_3d(c, GGML_TYPE_F16, 3, hp.n_mels, ns), 1.0f / sqrtf(3.0f * hp.n_mels), 0.0f);
    m.conv1_b = w(ggml_new_tensor_2d(c, GGML_TYPE_F32, 1, ns), 0.05f, 0.0f);
    m.conv2_w = w(ggml_new_tensor_3d(c, GGML_TYPE_F16, 3, ns, ns), 1.0f / sqrtf(3.0f * ns), 0.0f);
    m.conv2_b = w(ggml_new_tensor_2d(c, GGML_TYPE_F32, 1, ns), 0.05f, 0.0f);
    m.enc_pos = w(ggml_new_tensor_2d(c, GGML_TYPE_F32, ns, hp.n_audio_ctx()), 0.2f, 0.0f);
    m.tok_embd = w(ggml_new_tensor_2d(c, hp.wtype, ns, hp.n_vocab), 1.0f, 0.0f);
    m.dec_pos = w(ggml_new_tensor_2d(c, GGML_TYPE_F32, ns, hp.n_text_ctx), 0.2f, 0.0f);
    m.ln_post = ln();
    m.ln_dec = ln();
    m.enc.resize(hp.n_audio_layer);
    for (enc_layer & l : m.enc) {
        l.ln0 = ln(); l.ln1 = ln();
        l.q = lin(ns, ns, true, se); l.k = lin(ns, ns, false, se); l.v = lin(ns, ns, true, se); l.o = lin(ns, ns, true, se);
        l.fc1 = lin(ns, nff, true, se); l.fc2 = lin(nff, ns, true, 1.0f / sqrtf((float) nff));
    }
    m.dec.resize(hp.n_text_layer);
    for (dec_layer & l : m.dec) {
        l.ln0 = ln(); l.ln1 = ln(); l.ln2 = ln();
        l.q = lin(ns, ns, true, se); l.k = lin(ns, ns, false, se); l.v = lin(ns, ns, true, se); l.o = lin(ns, ns, true, se);
        l.cq = lin(ns, ns, true, se); l.ck = lin(ns, ns, false, se); l.cv = lin(ns, ns, true, se); l.co = lin(ns, ns, true, se);
        l.fc1 = lin(ns, nff, true, se); l.fc2 = lin(nff, ns, true, 1.0f / sqrtf((float) nff));
        l.k_cache = ggml_new_tensor_1d(m.ctx_s, GGML_TYPE_F16, ns * hp.n_text_ctx);
        l.v_cache = ggml_new_tensor_1d(m.ctx_s, GGML_TYPE_F16, ns * hp.n_text_ctx);
        l.ck_cache = ggml_new_tensor_1d(m.ctx_s, GGML_TYPE_F16, ns * hp.n_audio_ctx());
        l.cv_cache = ggml_new_tensor_1d(m.ctx_s, GGML_TYPE_F16, ns * hp.n_audio_ctx());
    }
    m.buf_w = ggml_backend_alloc_ctx_tensors_from_buft(m.ctx_w, bt);
    m.buf_s = ggml_backend_alloc_ctx_tensors_from_buft(m.ctx_s, bt);
    if (!m.buf_w || !m.buf_s) { fprintf(stderr, "model allocation failed\n"); exit(4); }
    ggml_backend_buffer_set_usage(m.buf_w, GGML_BACKEND_BUFFER_USAGE_WEIGHTS);
    ggml_backend_buffer_clear(m.buf_s, 0);
    w.run(20241016u);
}

void free_model(model & m) {
    ggml_backend_buffer_free(m.buf_w);
    ggml_backend_buffer_free(m.buf_s);
    ggml_free(m.ctx_w);
    ggml_free(m.ctx_s);
}

ggml_tensor * apply(ggml_context * ctx, const linear & l, ggml_tensor * x) {
    ggml_tensor * y = ggml_mul_mat(ctx, l.w, x);
    return l.b ? ggml_add(ctx, y, l.b) : y;
}
ggml_tensor * layer_norm(ggml_context * ctx, const norm & n, ggml_tensor * x, float eps) {
    return ggml_add(ctx, ggml_mul(ctx, ggml_norm(ctx, x, eps), n.w), n.b);
}

// attention of q [hd, n_q, H] (permuted) over K and V; non-flash: K [hd, n_kv, H], V transposed [n_kv, hd, H]; flash: K, V [hd, n_kv, H] f16.
// Returns [n_state, n_q].
ggml_tensor * attention(ggml_context * ctx, const hparams & hp, ggml_tensor * q, ggml_tensor * K, ggml_tensor * V, ggml_tensor * mask, int n_q) {
    const float scale = 1.0f / sqrtf((float) hp.head_dim());
    if (hp.flash_attn) return ggml_reshape_2d(ctx, ggml_flash_attn_ext(ctx, q, K, V, mask, scale, 0.0f, 0.0f), hp.n_state, n_q);
    ggml_tensor * kq = ggml_soft_max_ext(ctx, ggml_mul_mat(ctx, K, q), mask, scale, 0.0f);            // [n_kv, n_q, H]
    return ggml_cont_2d(ctx, ggml_permute(ctx, ggml_mul_mat(ctx, V, kq), 0, 2, 1, 3), hp.n_state, n_q);
}

ggml_tensor * heads(ggml_context * ctx, const hparams & hp, ggml_tensor * x, int n) {           // [n_state, n] -> [hd, n, H]
    return ggml_permute(ctx, ggml_reshape_3d(ctx, x, hp.head_dim(), hp.n_head, n), 0, 2, 1, 3);
}

// the encoder on "inp_mel"; writes the cross-attention caches of every decoder layer
void encoder(ggml_cgraph * gf, const model & m, ggml_context * ctx) {
    const hparams & hp = m.hp;
    const int T = hp.n_audio_ctx(), ns = hp.n_state;
    const size_t es = ggml_type_size(GGML_TYPE_F16);
    ggml_tensor * mel = ggml_new_tensor_2d(ctx, GGML_TYPE_F32, hp.n_frames, hp.n_mels);
    ggml_set_name(mel, "inp_mel"); ggml_set_input(mel);
    ggml_tensor * cur = ggml_gelu(ctx, ggml_add(ctx, ggml_conv_1d_ph(ctx, m.conv1_w, mel, 1, 1), m.conv1_b));       // [3000, n_state]
    cur = ggml_gelu(ctx, ggml_add(ctx, ggml_conv_1d_ph(ctx, m.conv2_w, cur, 2, 1), m.conv2_b));                      // [1500, n_state]
    ggml_set_name(cur, "conv2_gelu");
    cur = ggml_add(ctx, ggml_cont(ctx, ggml_transpose(ctx, cur)), m.enc_pos);                                         // [n_state, 1500]
    for (const enc_layer & l : m.enc) {
        ggml_tensor * h = layer_norm(ctx, l.ln0, cur, hp.eps);
        ggml_tensor * q = heads(ctx, hp, apply(ctx, l.q, h), T);
        ggml_tensor * k = heads(ctx, hp, apply(ctx, l.k, h), T);
        ggml_tensor * v = apply(ctx, l.v, h);
        ggml_tensor * a;
        if (hp.flash_attn) {
            // K and V copied into f16 tensors of their own, as whisper.cpp does (ggml_cast's CPY names itself as its destination, which
            // ggml_backend_graph_copy, the compare mode's copy, cannot duplicate)
            auto f16 = [&](ggml_tensor * t) { return ggml_cpy(ctx, t, ggml_new_tensor_3d(ctx, GGML_TYPE_F16, hp.head_dim(), T, hp.n_head)); };
            a = attention(ctx, hp, q, f16(k), f16(heads(ctx, hp, v, T)), nullptr, T);
        } else {
            ggml_tensor * vt = ggml_cont(ctx, ggml_permute(ctx, ggml_reshape_3d(ctx, v, hp.head_dim(), hp.n_head, T), 1, 2, 0, 3));    // [T, hd, H]
            a = attention(ctx, hp, q, k, vt, nullptr, T);
        }
        cur = ggml_add(ctx, apply(ctx, l.o, a), cur);
        h = layer_norm(ctx, l.ln1, cur, hp.eps);
        cur = ggml_add(ctx, apply(ctx, l.fc2, ggml_gelu(ctx, apply(ctx, l.fc1, h))), cur);
    }
    ggml_tensor * enc = layer_norm(ctx, m.ln_post, cur, hp.eps);
    ggml_set_name(enc, "enc_out");
    for (const dec_layer & l : m.dec) {
        ggml_tensor * k = apply(ctx, l.ck, enc), * v = apply(ctx, l.cv, enc);                                         // [n_state, 1500]
        ggml_build_forward_expand(gf, ggml_cpy(ctx, k, ggml_view_1d(ctx, l.ck_cache, (int64_t) ns * T, 0)));
        if (hp.flash_attn) ggml_build_forward_expand(gf, ggml_cpy(ctx, v, ggml_view_1d(ctx, l.cv_cache, (int64_t) ns * T, 0)));
        else ggml_build_forward_expand(gf, ggml_cpy(ctx, ggml_transpose(ctx, v), ggml_view_2d(ctx, l.cv_cache, T, ns, es * T, 0)));
    }
}

// the graph of N tokens at positions n_past ..; inputs "inp_tokens", "kq_mask" (and "inp_mel" when n_past == 0); output "result_output"
ggml_cgraph * build_graph(const model & m, ggml_context * ctx, int n_past, int N) {
    const hparams & hp = m.hp;
    const int n_kv = n_past + N, hd = hp.head_dim(), ns = hp.n_state, T = hp.n_audio_ctx(), H = hp.n_head;
    const size_t es = ggml_type_size(GGML_TYPE_F16);
    ggml_cgraph * gf = ggml_new_graph_custom(ctx, 4096, false);
    if (n_past == 0) encoder(gf, m, ctx);
    ggml_tensor * tok = ggml_new_tensor_1d(ctx, GGML_TYPE_I32, N);
    ggml_set_name(tok, "inp_tokens"); ggml_set_input(tok);
    ggml_tensor * mask = hp.flash_attn ? ggml_new_tensor_2d(ctx, GGML_TYPE_F16, n_kv, GGML_PAD(N, GGML_KQ_MASK_PAD))
                                       : ggml_new_tensor_2d(ctx, GGML_TYPE_F32, n_kv, N);
    ggml_set_name(mask, "kq_mask"); ggml_set_input(mask);

    ggml_tensor * x = ggml_add(ctx, ggml_get_rows(ctx, m.tok_embd, tok), ggml_view_2d(ctx, m.dec_pos, ns, N, m.dec_pos->nb[1], m.dec_pos->nb[1] * n_past));
    for (const dec_layer & l : m.dec) {
        // self attention: K rows, V rows (flash) or V transposed (columns at n_past) into the cache
        ggml_tensor * h = layer_norm(ctx, l.ln0, x, hp.eps);
        ggml_tensor * q = heads(ctx, hp, apply(ctx, l.q, h), N);
        ggml_tensor * k = apply(ctx, l.k, h), * v = apply(ctx, l.v, h);
        ggml_build_forward_expand(gf, ggml_cpy(ctx, k, ggml_view_1d(ctx, l.k_cache, (int64_t) N * ns, es * ns * n_past)));
        if (hp.flash_attn) ggml_build_forward_expand(gf, ggml_cpy(ctx, v, ggml_view_1d(ctx, l.v_cache, (int64_t) N * ns, es * ns * n_past)));
        else ggml_build_forward_expand(gf, ggml_cpy(ctx, ggml_transpose(ctx, v), ggml_view_2d(ctx, l.v_cache, N, ns, es * hp.n_text_ctx, es * n_past)));
        ggml_tensor * K = ggml_view_3d(ctx, l.k_cache, hd, n_kv, H, es * ns, es * hd, 0);
        ggml_tensor * V = hp.flash_attn ? ggml_view_3d(ctx, l.v_cache, hd, n_kv, H, es * ns, es * hd, 0)
                                        : ggml_view_3d(ctx, l.v_cache, n_kv, hd, H, es * hp.n_text_ctx, es * hp.n_text_ctx * hd, 0);
        x = ggml_add(ctx, apply(ctx, l.o, attention(ctx, hp, q, K, V, mask, N)), x);
        // cross attention over the cached K / V of the audio frames
        h = layer_norm(ctx, l.ln1, x, hp.eps);
        q = heads(ctx, hp, apply(ctx, l.cq, h), N);
        K = ggml_view_3d(ctx, l.ck_cache, hd, T, H, es * ns, es * hd, 0);
        V = hp.flash_attn ? ggml_view_3d(ctx, l.cv_cache, hd, T, H, es * ns, es * hd, 0) : ggml_view_3d(ctx, l.cv_cache, T, hd, H, es * T, es * T * hd, 0);
        x = ggml_add(ctx, apply(ctx, l.co, attention(ctx, hp, q, K, V, nullptr, N)), x);
        // MLP
        h = layer_norm(ctx, l.ln2, x, hp.eps);
        x = ggml_add(ctx, apply(ctx, l.fc2, ggml_gelu(ctx, apply(ctx, l.fc1, h))), x);
    }
    ggml_tensor * cur = ggml_mul_mat(ctx, m.tok_embd, layer_norm(ctx, m.ln_dec, x, hp.eps));
    ggml_set_name(cur, "result_output"); ggml_set_output(cur);
    ggml_build_forward_expand(gf, cur);
    int n_im2col = 0;
    for (int i = 0; i < ggml_graph_n_nodes(gf); ++i) n_im2col += ggml_graph_node(gf, i)->op == GGML_OP_IM2COL;
    printf("graph %s nodes %d im2col %d\n", n_past == 0 ? "prompt" : "decode", ggml_graph_n_nodes(gf), n_im2col);
    return gf;
}

void set_inputs(const hparams & hp, ggml_cgraph * gf, int n_past, const std::vector<int32_t> & toks) {
    const int N = (int) toks.size(), n_kv = n_past + N;
    ggml_backend_tensor_set(ggml_graph_get_tensor(gf, "inp_tokens"), toks.data(), 0, N * sizeof(int32_t));
    if (n_past == 0) {                                          // a log-mel spectrogram's range: smooth along time, around 0
        std::mt19937 rng(5489u);
        std::normal_distribution<float> nd(0.0f, 1.0f);
        std::vector<float> mel((size_t) hp.n_frames * hp.n_mels);
        for (int b = 0; b < hp.n_mels; ++b) {
            float prev = 0.0f;
            for (int t = 0; t < hp.n_frames; ++t) { prev = 0.8f * prev + 0.35f * nd(rng); mel[(size_t) b * hp.n_frames + t] = prev; }
        }
        ggml_tensor * t = ggml_graph_get_tensor(gf, "inp_mel");
        ggml_backend_tensor_set(t, mel.data(), 0, ggml_nbytes(t));
    }
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

} // namespace

int main(int argc, char ** argv) {
    model m;
    return decoder_main(argc, argv, [&m](const std::string & name) {
        m.hp = preset(name);
        decoder d;
        d.n_vocab = m.hp.n_vocab;
        d.n_ctx = m.hp.n_text_ctx;
        d.prompt = { 1, 417, 2093, 58 };
        d.build_model = [&m](ggml_backend_buffer_type_t bt) { build_model(m, bt); };
        d.free_model = [&m] { free_model(m); };
        d.build_graph = [&m](ggml_context * ctx, int n_past, int n_t) { return build_graph(m, ctx, n_past, n_t); };
        d.set_inputs = [&m](ggml_cgraph * gf, int n_past, const std::vector<int32_t> & toks) { set_inputs(m.hp, gf, n_past, toks); };
        return d;
    });
}
