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
// usage: mamba-graph PRESET compare DEVICE [sync]
//          ggml_backend_compare_graph_backend of ggml-cpu against DEVICE over the prompt and one decode step.  Prints
//          "node PHASE INDEX OP NAME [ne] nmse E" per contiguous f32 node, then per phase
//          "summary PHASE sync|free nodes_over_1e-9 N worst W first_over INDEX OP logits L".
//          With "sync" the device copy of each node result is replaced by the CPU's after the comparison.
//        mamba-graph PRESET run DEVICE STEPS LOGITS_OUT [FORCE_TOKENS]
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

// create the tensors of the model in ctx_w / ctx_s, allocate them in buffers of `bt`, fill the weights from fixed seeds
void build_model(model & m, ggml_backend_buffer_type_t bt) {
    const hparams & hp = m.hp;
    const size_t n_t = 4 + 12 * (size_t) hp.n_layer;
    ggml_init_params ip = { ggml_tensor_overhead() * n_t, nullptr, true };
    m.ctx_w = ggml_init(ip);
    m.ctx_s = ggml_init(ip);
    ggml_context * c = m.ctx_w;
    struct fill_job { ggml_tensor * t; float scale, offset; fill_kind kind; };
    std::vector<fill_job> jobs;
    auto w = [&](ggml_tensor * t, float scale, float offset, fill_kind kind = FILL_NORMAL) { jobs.push_back({ t, scale, offset, kind }); return t; };
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

    // tensor j is drawn from its own generator (seed 20240917 + j), so the parallel fill is deterministic
    std::vector<std::vector<uint8_t>> bytes(jobs.size());
    auto fill = [&](size_t j) {
        const ggml_tensor * t = jobs[j].t;
        std::mt19937 rng(20240917u + (unsigned) j);
        std::normal_distribution<float> nd(0.0f, 1.0f);
        std::uniform_real_distribution<double> ud(log(1e-3), log(1e-1));
        const int64_t n = ggml_nelements(t), k = t->ne[0];
        std::vector<float> x((size_t) n);
        for (int64_t i = 0; i < n; ++i) {
            switch (jobs[j].kind) {
                case FILL_A: x[(size_t) i] = -(float) (i % k + 1); break;                              // A[i0, i1] = -(i0 + 1)
                case FILL_DT_BIAS: {
                    const double dt = exp(ud(rng));                                                     // softplus^-1(dt) = dt + log(-expm1(-dt))
                    x[(size_t) i] = (float) (dt + log(-expm1(-dt)));
                } break;
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

void set_inputs(const hparams & hp, ggml_cgraph * gf, bool first, const std::vector<int32_t> & toks) {
    ggml_backend_tensor_set(ggml_graph_get_tensor(gf, "inp_tokens"), toks.data(), 0, toks.size() * sizeof(int32_t));
    std::vector<int32_t> copy(hp.n_seqs);
    std::vector<float> mask(hp.n_seqs, first ? 0.0f : 1.0f);
    for (int s = 0; s < hp.n_seqs; ++s) copy[s] = s;
    ggml_backend_tensor_set(ggml_graph_get_tensor(gf, "state_copy"), copy.data(), 0, copy.size() * sizeof(int32_t));
    ggml_backend_tensor_set(ggml_graph_get_tensor(gf, "state_mask"), mask.data(), 0, mask.size() * sizeof(float));
}

// the prompts, sequence-major: n_seqs x 7 tokens
std::vector<int32_t> prompt_tokens(const hparams & hp) {
    const std::vector<int32_t> p[2] = { { 1, 417, 2093, 58, 3001, 777, 12 }, { 1, 96, 3333, 1024, 7, 2500, 640 } };
    std::vector<int32_t> out;
    for (int s = 0; s < hp.n_seqs; ++s) out.insert(out.end(), p[s % 2].begin(), p[s % 2].end());
    return out;
}
const int PROMPT_LEN = 7;

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
        ggml_init_params ip = { ggml_tensor_overhead() * 4096 + ggml_graph_overhead_custom(4096, false), nullptr, true };
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
    ggml_backend_sched_t sched = ggml_backend_sched_new(backends, nullptr, n_be, 4096, false);
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
        ggml_init_params ip = { ggml_tensor_overhead() * 4096 + ggml_graph_overhead_custom(4096, false), nullptr, true };
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
    ggml_backend_buffer_free(m.buf_s);
    ggml_free(m.ctx_w);
    ggml_free(m.ctx_s);
    if (dev != cpu) ggml_backend_free(dev);
    ggml_backend_free(cpu);
    return rc;
}
