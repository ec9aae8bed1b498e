// oracle/sam_graph.cpp — TEST INFRASTRUCTURE ONLY.
//
// A synthetic Segment Anything (SAM) built in memory on the reference's public API (ggml.h, ggml-alloc.h, ggml-backend.h), written from the
// network's structure with weights from fixed seeds.  Every op is a core ggml op (the positional encodings use ggml_sin / ggml_cos), so the
// whole graph can run on one device.
//
// Image encoder (presets vit_b, small): ViT with windowed and global attention.
//   patch embedding ggml_conv_2d 16 x 16 stride 16 (IM2COL + f16 x f16 MUL_MAT) + bias, + absolute position embedding;
//   per layer: x + attn(LN(x)), then x + MLP(LN(x)) (GELU); attention with a fused f16 qkv linear, in 14 x 14 windows (WIN_PART before,
//   WIN_UNPART after; the token grid is padded to a multiple of 14) except in the global layers; the decomposed relative-position bias:
//   GET_REL_POS of the f16 tables along width and height, their MUL_MATs with the queries, ADD_REL_POS into the scaled logits, then SOFT_MAX;
//   neck: 1 x 1 conv -> layer-norm-2d -> 3 x 3 conv -> layer-norm-2d: the image embedding "embd" [T, T, 256].
// Prompt encoder + mask decoder (preset decoder), on a seeded [256, 64, 64] embedding ("embd_in", channels first) and one foreground point:
//   random-Fourier positional encodings (MUL_MAT by a gaussian [2, 128], SCALE by 2 pi, SIN, COS, CONCAT) of the point and of the 64 x 64
//   grid; the sparse tokens (point + label embedding, padding point); the dense no-mask embedding added to the image tokens; a two-way
//   transformer of 2 layers (self-attention, token -> image and image -> token cross-attention with the internal dim halved, MLP 2048 with
//   ReLU, 8 heads), the final token -> image attention; the upscaling CONV_TRANSPOSE_2D 256 -> 64 (k 2, s 2), layer-norm-2d, GELU,
//   CONV_TRANSPOSE_2D 64 -> 32, GELU; the four hypernetwork MLPs and the IoU head.  Outputs "masks" [256 256, 4] and "iou" [4].
//
// Presets:
//   vit_b    1024 x 1024 image, 64 x 64 tokens, 768 wide, 12 heads, 12 layers, global attention at 2 / 5 / 8 / 11, window 14 (64 -> 70: 25
//            windows), MLP 3072: the embedding [64, 64, 256]
//   small    the same structure, 512 x 512 image (32 x 32 tokens, padded to 42: 9 windows), 256 wide, 4 heads, 4 layers, globals at 1 and 3
//   decoder  the prompt encoder and mask decoder above
//
// usage: sam-graph PRESET compare DEVICE [sync]
//          ggml_backend_compare_graph_backend of ggml-cpu against DEVICE with decoder_harness.h's node comparison: "node image INDEX OP NAME
//          [ne] nmse E" per contiguous f32 node, then "summary image sync|free nodes_over_1e-9 N worst W first_over INDEX OP logits -1".
//          With "sync" the device copy of each node result is replaced by the CPU's after the comparison (identical inputs per node).
//        sam-graph PRESET run DEVICE REPS OUT
//          ggml_backend_sched over [DEVICE, CPU] (DEVICE = CPU: the CPU alone), weights in DEVICE's buffer: one warm-up pass, then REPS
//          passes.  Writes the outputs of the last pass (embd; or masks, then iou; f32) to OUT and prints "n_splits S", "cpu_nodes C",
//          "passes_identical 0|1" and "ms_per_pass M" (host clock around compute and the read-back of the outputs).
// Each graph built also prints "ops win_part A win_unpart B get_rel_pos C add_rel_pos D conv_transpose_2d E sin F cos G" (node counts).
// Exit codes: 2 usage or unknown preset, 3 unknown device, 4 model allocation, 5 graph copy, 6 file, 7 scheduler allocation, 8 compute.

#include "decoder_harness.h"

#include <cmath>

namespace {

constexpr int GRAPH_SIZE = 8192;

struct enc_layer {
    bool global;
    ggml_tensor * ln1_g, * ln1_b, * qkv_w, * qkv_b, * proj_w, * proj_b, * rel_h, * rel_w;
    ggml_tensor * ln2_g, * ln2_b, * mlp1_w, * mlp1_b, * mlp2_w, * mlp2_b;
};

struct attn_w { ggml_tensor * q_w, * q_b, * k_w, * k_b, * v_w, * v_b, * o_w, * o_b; };
struct norm_w { ggml_tensor * g, * b; };
struct mlp3_w { ggml_tensor * w[3], * b[3]; };

struct model {
    std::string preset;
    bool decoder = false;
    // encoder
    int img = 0, n_embd = 0, n_head = 0, n_layer = 0, window = 14, n_out = 256;
    ggml_tensor * patch_w = nullptr, * patch_b = nullptr, * pos = nullptr, * neck0 = nullptr, * neck1 = nullptr;
    norm_w neck_ln0{}, neck_ln1{};
    std::vector<enc_layer> layers;
    // decoder
    ggml_tensor * pe_gauss = nullptr, * point_embd = nullptr, * not_a_point = nullptr, * no_mask = nullptr, * iou_token = nullptr, * mask_tokens = nullptr;
    struct dec_layer { attn_w self, t2i, i2t; norm_w n1, n2, n3, n4; ggml_tensor * mlp1_w, * mlp1_b, * mlp2_w, * mlp2_b; };
    std::vector<dec_layer> dec;
    attn_w final_t2i{};
    norm_w final_norm{}, up_ln{};
    ggml_tensor * up1_w = nullptr, * up1_b = nullptr, * up2_w = nullptr, * up2_b = nullptr;
    mlp3_w hyper[4]{}, iou_head{};
    ggml_context * ctx = nullptr;
    ggml_backend_buffer_t buf = nullptr;
    int tokens() const { return img / 16; }
};

void setup(model & m, const std::string & preset) {
    m.preset = preset;
    if (preset == "vit_b")      { m.img = 1024; m.n_embd = 768; m.n_head = 12; m.n_layer = 12; }
    else if (preset == "small") { m.img = 512;  m.n_embd = 256; m.n_head = 4;  m.n_layer = 4; }
    else if (preset == "decoder") m.decoder = true;
    else { fprintf(stderr, "unknown preset %s (vit_b | small | decoder)\n", preset.c_str()); exit(2); }
}

bool is_global(const model & m, int il) {
    if (m.preset == "vit_b") return il == 2 || il == 5 || il == 8 || il == 11;
    return il == 1 || il == 3;
}

void build_model(model & m, ggml_backend_buffer_type_t bt) {
    ggml_init_params ip = { ggml_tensor_overhead() * 1024, nullptr, true };
    m.ctx = ggml_init(ip);
    ggml_context * c = m.ctx;
    weight_fill w;
    auto f32 = [&](int64_t n0, int64_t n1 = 1, int64_t n2 = 1, int64_t n3 = 1) { return ggml_new_tensor_4d(c, GGML_TYPE_F32, n0, n1, n2, n3); };
    auto f16 = [&](int64_t n0, int64_t n1 = 1, int64_t n2 = 1, int64_t n3 = 1) { return ggml_new_tensor_4d(c, GGML_TYPE_F16, n0, n1, n2, n3); };
    auto norm = [&](int64_t n) { norm_w r; r.g = w(f32(n), 0.1f, 1.0f); r.b = w(f32(n), 0.1f, 0.0f); return r; };
    auto attn = [&](int64_t e, int64_t in) {
        attn_w a;
        a.q_w = w(f32(e, in), 1.0f / sqrtf((float) e), 0.0f); a.q_b = w(f32(in), 0.02f, 0.0f);
        a.k_w = w(f32(e, in), 1.0f / sqrtf((float) e), 0.0f); a.k_b = w(f32(in), 0.02f, 0.0f);
        a.v_w = w(f32(e, in), 1.0f / sqrtf((float) e), 0.0f); a.v_b = w(f32(in), 0.02f, 0.0f);
        a.o_w = w(f32(in, e), 1.0f / sqrtf((float) in), 0.0f); a.o_b = w(f32(e), 0.02f, 0.0f);
        return a;
    };
    auto mlp3 = [&](int64_t in, int64_t hid, int64_t out) {
        mlp3_w r;
        const int64_t d[4] = { in, hid, hid, out };
        for (int i = 0; i < 3; ++i) { r.w[i] = w(f32(d[i], d[i + 1]), 1.0f / sqrtf((float) d[i]), 0.0f); r.b[i] = w(f32(d[i + 1]), 0.02f, 0.0f); }
        return r;
    };
    if (!m.decoder) {
        const int64_t E = m.n_embd, T = m.tokens(), hd = E / m.n_head;
        m.patch_w = w(f16(16, 16, 3, E), 1.0f / sqrtf(768.0f), 0.0f);
        m.patch_b = w(f32(1, 1, E), 0.02f, 0.0f);
        m.pos = w(f32(E, T, T), 0.1f, 0.0f);
        for (int il = 0; il < m.n_layer; ++il) {
            enc_layer l;
            l.global = is_global(m, il);
            const int64_t span = l.global ? T : m.window;
            norm_w n1 = norm(E), n2 = norm(E);
            l.ln1_g = n1.g; l.ln1_b = n1.b; l.ln2_g = n2.g; l.ln2_b = n2.b;
            l.qkv_w = w(f16(E, 3 * E), 1.0f / sqrtf((float) E), 0.0f); l.qkv_b = w(f32(3 * E), 0.02f, 0.0f);
            l.proj_w = w(f16(E, E), 1.0f / sqrtf((float) E), 0.0f);     l.proj_b = w(f32(E), 0.02f, 0.0f);
            l.rel_h = w(f16(hd, 2 * span - 1), 0.1f, 0.0f);              l.rel_w = w(f16(hd, 2 * span - 1), 0.1f, 0.0f);
            l.mlp1_w = w(f16(E, 4 * E), 1.0f / sqrtf((float) E), 0.0f);  l.mlp1_b = w(f32(4 * E), 0.02f, 0.0f);
            l.mlp2_w = w(f16(4 * E, E), 1.0f / sqrtf((float) (4 * E)), 0.0f); l.mlp2_b = w(f32(E), 0.02f, 0.0f);
            m.layers.push_back(l);
        }
        m.neck0 = w(f16(1, 1, E, m.n_out), 1.0f / sqrtf((float) E), 0.0f);
        m.neck_ln0 = norm(m.n_out);
        m.neck1 = w(f16(3, 3, m.n_out, m.n_out), 1.0f / sqrtf(9.0f * m.n_out), 0.0f);
        m.neck_ln1 = norm(m.n_out);
    } else {
        const int64_t E = 256;
        m.pe_gauss = w(f32(2, E / 2), 1.0f, 0.0f);
        m.point_embd = w(f32(E), 0.1f, 0.0f);
        m.not_a_point = w(f32(E), 0.1f, 0.0f);
        m.no_mask = w(f32(E), 0.1f, 0.0f);
        m.iou_token = w(f32(E), 0.1f, 0.0f);
        m.mask_tokens = w(f32(E, 4), 0.1f, 0.0f);
        for (int il = 0; il < 2; ++il) {
            model::dec_layer l;
            l.self = attn(E, E); l.t2i = attn(E, E / 2); l.i2t = attn(E, E / 2);
            l.n1 = norm(E); l.n2 = norm(E); l.n3 = norm(E); l.n4 = norm(E);
            l.mlp1_w = w(f32(E, 2048), 1.0f / sqrtf((float) E), 0.0f); l.mlp1_b = w(f32(2048), 0.02f, 0.0f);
            l.mlp2_w = w(f32(2048, E), 1.0f / sqrtf(2048.0f), 0.0f);   l.mlp2_b = w(f32(E), 0.02f, 0.0f);
            m.dec.push_back(l);
        }
        m.final_t2i = attn(E, E / 2);
        m.final_norm = norm(E);
        m.up1_w = w(f16(2, 2, 64, E), 1.0f / sqrtf((float) E), 0.0f); m.up1_b = w(f32(1, 1, 64), 0.02f, 0.0f);
        m.up_ln = norm(64);
        m.up2_w = w(f16(2, 2, 32, 64), 1.0f / sqrtf(64.0f), 0.0f);   m.up2_b = w(f32(1, 1, 32), 0.02f, 0.0f);
        for (mlp3_w & h : m.hyper) h = mlp3(E, E, 32);
        m.iou_head = mlp3(E, 256, 4);
    }
    m.buf = ggml_backend_alloc_ctx_tensors_from_buft(m.ctx, bt);
    if (!m.buf) { fprintf(stderr, "model allocation failed\n"); exit(4); }
    ggml_backend_buffer_set_usage(m.buf, GGML_BACKEND_BUFFER_USAGE_WEIGHTS);
    w.run(20241203u);
}

void free_model(model & m) {
    ggml_backend_buffer_free(m.buf);
    ggml_free(m.ctx);
}

// ------------------------------------------------------------------ image encoder
ggml_tensor * layer_norm(ggml_context * ctx, ggml_tensor * x, ggml_tensor * g, ggml_tensor * b, float eps) {
    return ggml_add(ctx, ggml_mul(ctx, ggml_norm(ctx, x, eps), g), b);
}

// [W, H, C] (channels last) -> normalised over C -> [W, H, C]
ggml_tensor * layer_norm_2d(ggml_context * ctx, ggml_tensor * x, const norm_w & n) {
    x = ggml_cont(ctx, ggml_permute(ctx, x, 1, 2, 0, 3));                 // [C, W, H]
    x = layer_norm(ctx, x, n.g, n.b, 1e-6f);
    return ggml_cont(ctx, ggml_permute(ctx, x, 2, 0, 1, 3));               // [W, H, C]
}

// x [E, S, S, B] (B windows of S x S tokens, or one image) -> attention over each window's S S tokens
ggml_tensor * encoder_attention(ggml_context * ctx, const model & m, const enc_layer & l, ggml_tensor * x) {
    const int64_t E = m.n_embd, nh = m.n_head, hd = E / nh, S = x->ne[1], B = x->ne[3], N = S * S;
    ggml_tensor * qkv = ggml_add(ctx, ggml_mul_mat(ctx, l.qkv_w, x), l.qkv_b);       // [3E, S, S, B]
    auto part = [&](int i) {                                                            // [hd, nh, N, B] of q (0), k (1) or v (2)
        return ggml_view_4d(ctx, qkv, hd, nh, N, B, hd * sizeof(float), 3 * E * sizeof(float), 3 * E * N * sizeof(float), i * E * sizeof(float));
    };
    ggml_tensor * Q = ggml_reshape_3d(ctx, ggml_cont(ctx, ggml_permute(ctx, part(0), 0, 2, 1, 3)), hd, N, nh * B);   // [hd, N, nh B]
    ggml_tensor * K = ggml_reshape_3d(ctx, ggml_cont(ctx, ggml_permute(ctx, part(1), 0, 2, 1, 3)), hd, N, nh * B);
    ggml_tensor * V = ggml_reshape_3d(ctx, ggml_cont(ctx, ggml_permute(ctx, part(2), 1, 2, 0, 3)), N, hd, nh * B);   // [N, hd, nh B]
    ggml_tensor * kq = ggml_scale(ctx, ggml_mul_mat(ctx, K, Q), 1.0f / sqrtf((float) hd));                          // [N keys, N queries, nh B]
    // the decomposed relative-position bias: ph[q, kh] = q . Rh[qh, kh], pw[q, kw] = q . Rw[qw, kw]
    ggml_tensor * rh = ggml_get_rel_pos(ctx, l.rel_h, (int) S, (int) S);                 // [hd, S keys, S queries] f16
    ggml_tensor * rw = ggml_get_rel_pos(ctx, l.rel_w, (int) S, (int) S);
    ggml_tensor * q4 = ggml_reshape_4d(ctx, Q, hd, S, S, nh * B);                       // [hd, qw, qh, nh B]
    ggml_tensor * ph = ggml_mul_mat(ctx, rh, q4);                                        // [kh, qw, qh, nh B]
    ggml_tensor * pw = ggml_mul_mat(ctx, rw, ggml_cont(ctx, ggml_permute(ctx, q4, 0, 2, 1, 3)));   // [kw, qh, qw, nh B]
    pw = ggml_cont(ctx, ggml_permute(ctx, pw, 0, 2, 1, 3));                              // [kw, qw, qh, nh B]
    kq = ggml_add_rel_pos_inplace(ctx, kq, pw, ph);
    ggml_tensor * p = ggml_soft_max(ctx, kq);
    ggml_tensor * o = ggml_mul_mat(ctx, V, p);                                           // [hd, N, nh B]
    o = ggml_cont(ctx, ggml_permute(ctx, ggml_reshape_4d(ctx, o, hd, N, nh, B), 0, 2, 1, 3));   // [hd, nh, N, B]
    o = ggml_reshape_4d(ctx, o, E, S, S, B);
    return ggml_add(ctx, ggml_mul_mat(ctx, l.proj_w, o), l.proj_b);
}

ggml_tensor * build_encoder(const model & m, ggml_context * ctx) {
    const int64_t T = m.tokens();
    ggml_tensor * inp = ggml_new_tensor_4d(ctx, GGML_TYPE_F32, m.img, m.img, 3, 1);
    ggml_set_name(inp, "image"); ggml_set_input(inp);
    ggml_tensor * x = ggml_conv_2d(ctx, m.patch_w, inp, 16, 16, 0, 0, 1, 1);           // [T, T, E, 1]
    x = ggml_add(ctx, x, m.patch_b);
    x = ggml_cont(ctx, ggml_permute(ctx, x, 1, 2, 0, 3));                              // [E, T, T, 1]
    x = ggml_add(ctx, x, m.pos);
    for (const enc_layer & l : m.layers) {
        ggml_tensor * sc = x;
        ggml_tensor * h = layer_norm(ctx, x, l.ln1_g, l.ln1_b, 1e-6f);
        if (!l.global) h = ggml_win_part(ctx, h, m.window);                              // [E, 14, 14, windows]
        h = encoder_attention(ctx, m, l, h);
        if (!l.global) h = ggml_win_unpart(ctx, h, (int) T, (int) T, m.window);
        x = ggml_add(ctx, sc, h);
        h = layer_norm(ctx, x, l.ln2_g, l.ln2_b, 1e-6f);
        h = ggml_add(ctx, ggml_mul_mat(ctx, l.mlp1_w, h), l.mlp1_b);
        h = ggml_add(ctx, ggml_mul_mat(ctx, l.mlp2_w, ggml_gelu(ctx, h)), l.mlp2_b);
        x = ggml_add(ctx, x, h);
    }
    x = ggml_cont(ctx, ggml_permute(ctx, x, 2, 0, 1, 3));                              // [T, T, E]
    x = layer_norm_2d(ctx, ggml_conv_2d_sk_p0(ctx, m.neck0, x), m.neck_ln0);
    x = layer_norm_2d(ctx, ggml_conv_2d_s1_ph(ctx, m.neck1, x), m.neck_ln1);           // [T, T, 256]
    ggml_set_name(x, "embd"); ggml_set_output(x);
    return x;
}

// ------------------------------------------------------------------ prompt encoder + mask decoder
// coords [2, n], already mapped to [-1, 1] (2 c - 1 of the normalised position) -> [256, n]: sin and cos of 2 pi G^T coords
ggml_tensor * fourier_pe(ggml_context * ctx, const model & m, ggml_tensor * coords) {
    ggml_tensor * p = ggml_scale(ctx, ggml_mul_mat(ctx, m.pe_gauss, coords), 2.0f * (float) M_PI);   // [128, n]
    return ggml_concat(ctx, ggml_sin(ctx, p), ggml_cos(ctx, p), 0);
}

// q [E, Nq], k [E, Nk], v [E, Nk] -> [E, Nq]; 8 heads of the attention's internal width
ggml_tensor * attention(ggml_context * ctx, const attn_w & a, ggml_tensor * q, ggml_tensor * k, ggml_tensor * v) {
    const int64_t I = a.q_w->ne[1], nh = 8, hd = I / nh, Nq = q->ne[1], Nk = k->ne[1];
    ggml_tensor * Q = ggml_add(ctx, ggml_mul_mat(ctx, a.q_w, q), a.q_b);
    ggml_tensor * K = ggml_add(ctx, ggml_mul_mat(ctx, a.k_w, k), a.k_b);
    ggml_tensor * V = ggml_add(ctx, ggml_mul_mat(ctx, a.v_w, v), a.v_b);
    Q = ggml_cont(ctx, ggml_permute(ctx, ggml_reshape_3d(ctx, Q, hd, nh, Nq), 0, 2, 1, 3));     // [hd, Nq, nh]
    K = ggml_cont(ctx, ggml_permute(ctx, ggml_reshape_3d(ctx, K, hd, nh, Nk), 0, 2, 1, 3));     // [hd, Nk, nh]
    V = ggml_cont(ctx, ggml_permute(ctx, ggml_reshape_3d(ctx, V, hd, nh, Nk), 1, 2, 0, 3));     // [Nk, hd, nh]
    ggml_tensor * p = ggml_soft_max_ext(ctx, ggml_mul_mat(ctx, K, Q), nullptr, 1.0f / sqrtf((float) hd), 0.0f);   // [Nk, Nq, nh]
    ggml_tensor * o = ggml_cont(ctx, ggml_permute(ctx, ggml_mul_mat(ctx, V, p), 0, 2, 1, 3));    // [hd, nh, Nq]
    return ggml_add(ctx, ggml_mul_mat(ctx, a.o_w, ggml_reshape_2d(ctx, o, I, Nq)), a.o_b);
}

ggml_tensor * mlp3(ggml_context * ctx, const mlp3_w & w, ggml_tensor * x) {
    for (int i = 0; i < 3; ++i) {
        x = ggml_add(ctx, ggml_mul_mat(ctx, w.w[i], x), w.b[i]);
        if (i < 2) x = ggml_relu(ctx, x);
    }
    return x;
}

void build_decoder(const model & m, ggml_context * ctx, ggml_tensor ** masks, ggml_tensor ** iou) {
    const int64_t E = 256, T = 64;
    // the image embedding, channels first: [E, T, T] flattened to [E, T T] (an input consumed through a view would make the scheduler
    // place that view on the CPU)
    ggml_tensor * embd = ggml_new_tensor_2d(ctx, GGML_TYPE_F32, E, T * T);
    ggml_set_name(embd, "embd_in"); ggml_set_input(embd);
    ggml_tensor * point = ggml_new_tensor_2d(ctx, GGML_TYPE_F32, 2, 2);                 // the point and the padding point, in [-1, 1]
    ggml_set_name(point, "point"); ggml_set_input(point);
    ggml_tensor * grid = ggml_new_tensor_2d(ctx, GGML_TYPE_F32, 2, T * T);              // the cell centres of the 64 x 64 grid
    ggml_set_name(grid, "grid"); ggml_set_input(grid);
    // sparse prompt: the point's PE + the foreground label embedding; the padding point is not_a_point
    ggml_tensor * pe = fourier_pe(ctx, m, point);                                       // [E, 2]
    ggml_tensor * sparse = ggml_concat(ctx, ggml_add(ctx, ggml_view_1d(ctx, pe, E, 0), m.point_embd), ggml_reshape_2d(ctx, m.not_a_point, E, 1), 1);
    ggml_tensor * tokens = ggml_concat(ctx, ggml_concat(ctx, ggml_reshape_2d(ctx, m.iou_token, E, 1), m.mask_tokens, 1), sparse, 1);   // [E, 7]
    ggml_tensor * image_pe = fourier_pe(ctx, m, grid);                                  // [E, T T]
    ggml_tensor * keys = ggml_add(ctx, embd, m.no_mask);                                // [E, T T]
    ggml_tensor * queries = tokens;
    for (size_t il = 0; il < m.dec.size(); ++il) {
        const model::dec_layer & l = m.dec[il];
        if (il == 0) queries = attention(ctx, l.self, queries, queries, queries);
        else {
            ggml_tensor * q = ggml_add(ctx, queries, tokens);
            queries = ggml_add(ctx, queries, attention(ctx, l.self, q, q, queries));
        }
        queries = layer_norm(ctx, queries, l.n1.g, l.n1.b, 1e-5f);
        ggml_tensor * q = ggml_add(ctx, queries, tokens), * k = ggml_add(ctx, keys, image_pe);
        queries = layer_norm(ctx, ggml_add(ctx, queries, attention(ctx, l.t2i, q, k, keys)), l.n2.g, l.n2.b, 1e-5f);
        ggml_tensor * h = ggml_relu(ctx, ggml_add(ctx, ggml_mul_mat(ctx, l.mlp1_w, queries), l.mlp1_b));
        queries = layer_norm(ctx, ggml_add(ctx, queries, ggml_add(ctx, ggml_mul_mat(ctx, l.mlp2_w, h), l.mlp2_b)), l.n3.g, l.n3.b, 1e-5f);
        q = ggml_add(ctx, queries, tokens); k = ggml_add(ctx, keys, image_pe);
        keys = layer_norm(ctx, ggml_add(ctx, keys, attention(ctx, l.i2t, k, q, queries)), l.n4.g, l.n4.b, 1e-5f);
    }
    {
        ggml_tensor * q = ggml_add(ctx, queries, tokens), * k = ggml_add(ctx, keys, image_pe);
        queries = layer_norm(ctx, ggml_add(ctx, queries, attention(ctx, m.final_t2i, q, k, keys)), m.final_norm.g, m.final_norm.b, 1e-5f);
    }
    // upscaling: [E, T T] -> [T, T, E] -> [2T, 2T, 64] -> [4T, 4T, 32]
    ggml_tensor * src = ggml_cont(ctx, ggml_permute(ctx, ggml_reshape_3d(ctx, keys, E, T, T), 2, 0, 1, 3));
    ggml_tensor * up = ggml_add(ctx, ggml_conv_transpose_2d_p0(ctx, m.up1_w, src, 2), m.up1_b);
    up = ggml_gelu(ctx, layer_norm_2d(ctx, up, m.up_ln));
    up = ggml_gelu(ctx, ggml_add(ctx, ggml_conv_transpose_2d_p0(ctx, m.up2_w, up, 2), m.up2_b));                  // [4T, 4T, 32]
    ggml_tensor * hyper = nullptr;
    for (int i = 0; i < 4; ++i) {
        ggml_tensor * t = mlp3(ctx, m.hyper[i], ggml_view_2d(ctx, queries, E, 1, queries->nb[1], (1 + i) * queries->nb[1]));   // [32, 1]
        hyper = hyper ? ggml_concat(ctx, hyper, t, 1) : t;
    }
    ggml_tensor * upc = ggml_reshape_2d(ctx, ggml_cont(ctx, ggml_permute(ctx, up, 1, 2, 0, 3)), 32, 16 * T * T);   // [32, 4T 4T]
    *masks = ggml_mul_mat(ctx, upc, hyper);                                              // [4T 4T, 4]
    ggml_set_name(*masks, "masks"); ggml_set_output(*masks);
    *iou = mlp3(ctx, m.iou_head, ggml_view_2d(ctx, queries, E, 1, queries->nb[1], 0));  // [4, 1]
    ggml_set_name(*iou, "iou"); ggml_set_output(*iou);
}

// the graph and its outputs (embd; or masks, iou)
ggml_cgraph * build_graph(const model & m, ggml_context * ctx, std::vector<ggml_tensor *> & outs) {
    ggml_cgraph * gf = ggml_new_graph_custom(ctx, GRAPH_SIZE, false);
    outs.clear();
    if (m.decoder) {
        ggml_tensor * masks, * iou;
        build_decoder(m, ctx, &masks, &iou);
        outs = { masks, iou };
    } else {
        outs = { build_encoder(m, ctx) };
    }
    for (ggml_tensor * t : outs) ggml_build_forward_expand(gf, t);
    const ggml_op ops[7] = { GGML_OP_WIN_PART, GGML_OP_WIN_UNPART, GGML_OP_GET_REL_POS, GGML_OP_ADD_REL_POS, GGML_OP_CONV_TRANSPOSE_2D, GGML_OP_SIN, GGML_OP_COS };
    int n[7] = { 0, 0, 0, 0, 0, 0, 0 };
    for (int i = 0; i < ggml_graph_n_nodes(gf); ++i)
        for (int k = 0; k < 7; ++k) n[k] += ggml_graph_node(gf, i)->op == ops[k];
    printf("ops win_part %d win_unpart %d get_rel_pos %d add_rel_pos %d conv_transpose_2d %d sin %d cos %d\n", n[0], n[1], n[2], n[3], n[4], n[5], n[6]);
    return gf;
}

void set_inputs(const model & m, ggml_cgraph * gf) {
    std::mt19937 rng(5489u);
    std::uniform_real_distribution<float> ud(0.0f, 1.0f);
    if (!m.decoder) {
        ggml_tensor * t = ggml_graph_get_tensor(gf, "image");                            // an image's range, smooth along rows
        std::vector<float> img((size_t) ggml_nelements(t));
        float prev = 0.5f;
        for (float & v : img) { prev = 0.7f * prev + 0.3f * ud(rng); v = prev; }
        ggml_backend_tensor_set(t, img.data(), 0, ggml_nbytes(t));
        return;
    }
    ggml_tensor * e = ggml_graph_get_tensor(gf, "embd_in");
    std::normal_distribution<float> nd(0.0f, 1.0f);
    std::vector<float> x((size_t) ggml_nelements(e));
    for (float & v : x) v = nd(rng);
    ggml_backend_tensor_set(e, x.data(), 0, ggml_nbytes(e));
    // coordinates as the PE takes them, 2 c - 1 of the position normalised to [0, 1]: the point (320.5, 616.5) of a 1024 x 1024 image, the
    // padding point, and the centres of the 64 x 64 grid cells
    const float pt[4] = { 2.0f * 320.5f / 1024.0f - 1.0f, 2.0f * 616.5f / 1024.0f - 1.0f, -1.0f, -1.0f };
    ggml_backend_tensor_set(ggml_graph_get_tensor(gf, "point"), pt, 0, sizeof(pt));
    std::vector<float> grid(2 * 64 * 64);
    for (int y = 0; y < 64; ++y)
        for (int xx = 0; xx < 64; ++xx) { grid[2 * (y * 64 + xx)] = 2.0f * (xx + 0.5f) / 64.0f - 1.0f; grid[2 * (y * 64 + xx) + 1] = 2.0f * (y + 0.5f) / 64.0f - 1.0f; }
    ggml_backend_tensor_set(ggml_graph_get_tensor(gf, "grid"), grid.data(), 0, grid.size() * sizeof(float));
}

ggml_context * graph_ctx() {
    ggml_init_params ip = { ggml_tensor_overhead() * GRAPH_SIZE + ggml_graph_overhead_custom(GRAPH_SIZE, false), nullptr, true };
    return ggml_init(ip);
}

int run_compare(const model & m, ggml_backend_t cpu, ggml_backend_t dev, bool sync) {
    ggml_context * ctx = graph_ctx();
    std::vector<ggml_tensor *> outs;
    ggml_cgraph * gf = build_graph(m, ctx, outs);
    ggml_gallocr_t allocr = ggml_gallocr_new(ggml_backend_get_default_buffer_type(cpu));
    ggml_gallocr_alloc_graph(allocr, gf);
    set_inputs(m, gf);
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
    ggml_backend_sched_t sched = ggml_backend_sched_new(backends, nullptr, n_be, GRAPH_SIZE, false);
    ggml_context * ctx = graph_ctx();
    std::vector<ggml_tensor *> outs;
    ggml_cgraph * gf = build_graph(m, ctx, outs);
    if (!ggml_backend_sched_alloc_graph(sched, gf)) { fprintf(stderr, "sched alloc failed\n"); return 7; }
    size_t n_out = 0;
    for (ggml_tensor * t : outs) n_out += (size_t) ggml_nelements(t);
    std::vector<float> out(n_out), first;
    bool identical = true;
    double total_s = 0.0;
    for (int pass = 0; pass <= reps; ++pass) {                 // pass 0: warm-up
        set_inputs(m, gf);
        const auto t0 = std::chrono::steady_clock::now();
        if (ggml_backend_sched_graph_compute(sched, gf) != GGML_STATUS_SUCCESS) { fprintf(stderr, "compute failed\n"); return 8; }
        size_t o = 0;
        for (ggml_tensor * t : outs) { ggml_backend_tensor_get(t, out.data() + o, 0, ggml_nbytes(t)); o += (size_t) ggml_nelements(t); }
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

} // namespace

int main(int argc, char ** argv) {
    if (argc < 4) {
        fprintf(stderr, "usage: %s PRESET compare DEVICE [sync]\n       %s PRESET run DEVICE REPS OUT\n", argv[0], argv[0]);
        return 2;
    }
    model m;
    setup(m, argv[1]);
    const std::string mode = argv[2];
    ggml_backend_load_all();
    ggml_backend_t cpu = ggml_backend_init_by_type(GGML_BACKEND_DEVICE_TYPE_CPU, nullptr);
    ggml_backend_cpu_set_n_threads(cpu, 8);
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
