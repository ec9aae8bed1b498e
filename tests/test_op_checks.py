"""CPU-only: the acceptance rules of ggml_b200/csrc/b200_op_checks.h compiled for the HOST (tests/hostemu/op_checks_emu.cpp).  The
ggml_b200_op_* launchers return what these checks return, and the plug-in's supports_op asks the same checks, so this pins both without a
device:
  * every case the GPU suites assert through the C ABI (test_gpu_rope.py, test_gpu_moe.py, test_gpu_mamba.py) gives the same status code;
  * the sources the plug-in declines in those suites are refused by the check (rows longer than 1024, unpacked SSM_CONV rows, ...);
  * the nodes of the llama (norm, neox), MoE (moe, moe60) and Mamba (mamba, falcon) decoder presets of oracle/*_graph.cpp are accepted,
    for a prompt and for a decode step;
  * nodes that the plug-in used to accept but its launcher refused are now refused by the check: FLASH_ATTN_EXT whose V or mask does not
    match K, and SUM_ROWS with more rows than one grid holds."""
import ctypes as C
import subprocess
from pathlib import Path

import pytest
import torch

import ggml_b200 as g

ROOT = Path(__file__).resolve().parents[1]
EMU = ROOT / "tests" / "hostemu"
OK, EUNSUPPORTED, EINVAL = 0, -1, -2
F32, F16, Q8_0, Q4_K, I32 = 0, 1, 8, 12, 26
TYPE_SIZE = {F32: (1, 4), F16: (1, 2), I32: (1, 4), Q8_0: (32, 34), Q4_K: (256, 144)}     # (block elements, block bytes)


@pytest.fixture(scope="module")
def L():
    out = EMU / "_build"
    out.mkdir(exist_ok=True)
    so = out / "libop_checks_emu.so"
    srcs = [EMU / "op_checks_emu.cpp", ROOT / "ggml_b200" / "csrc" / "b200_op_checks.h", ROOT / "include" / "ggml-b200.h"]
    if not so.exists() or so.stat().st_mtime < max(p.stat().st_mtime for p in srcs):
        cmd = ["g++", "-std=c++17", "-O1", "-fPIC", "-shared", "-Wall", "-Werror", "-o", str(so), str(EMU / "op_checks_emu.cpp")]
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-3000:]
    return C.CDLL(str(so))


def call(fn, *args):
    """a check with the launcher's arguments: TensorDesc / RopeParams by reference, None for a null pointer, ints as int32_t"""
    return fn(*[C.byref(a) if isinstance(a, (g.TensorDesc, g.RopeParams)) else a for a in args])


def z(*shape, dt=torch.float32):
    return torch.zeros(shape, dtype=dt)


D = g.strided_desc


def T(type_, ne, nb=None):
    """a ggml tensor descriptor: ne in ggml order, nb in bytes (packed when None)"""
    d = g.TensorDesc()
    d.data, d.type = 4096, type_
    blk, bs = TYPE_SIZE[type_]
    ne = list(ne) + [1] * (4 - len(ne))
    if nb is None:
        nb = [bs, bs * ne[0] // blk]
        for i in range(2, 4):
            nb.append(nb[-1] * ne[i - 1])
    for i in range(4):
        d.ne[i], d.nb[i] = ne[i], nb[i]
    return d


# ------------------------------------------------------------------ the GPU suites' C ABI cases
def test_rope_cases_of_the_gpu_suite(L):
    x, pos = D(z(1, 2, 4, 64)), D(z(2, dt=torch.int32))
    assert call(L.emu_rope, x, pos, None, x, g.rope_params(64)) == OK
    bad = [g.rope_params(63), g.rope_params(66), g.rope_params(64, 5), g.rope_params(64, g.ROPE_VISION), g.rope_params(64, g.ROPE_MROPE)]
    for p in bad:
        assert call(L.emu_rope, x, pos, None, x, p) == EUNSUPPORTED
    assert call(L.emu_rope, x, pos, None, x, g.rope_params(64, g.ROPE_MROPE, sections=(16, 8, 8, 0))) == EUNSUPPORTED     # four positions per token
    assert call(L.emu_rope, x, pos, D(z(31)), x, g.rope_params(64)) == EUNSUPPORTED                                     # freq factors: >= n_dims/2
    assert call(L.emu_rope, x, pos, D(z(32)), x, g.rope_params(64)) == OK
    assert call(L.emu_rope, None, pos, None, x, g.rope_params(64)) == EUNSUPPORTED
    wide = D(z(1, 2, 1, 2050))
    assert call(L.emu_rope, wide, pos, None, wide, g.rope_params(1026)) == EUNSUPPORTED                                 # > 1024 rotated dims
    assert call(L.emu_rope, wide, pos, None, wide, g.rope_params(1024)) == OK


def test_argsort_and_sum_rows_cases_of_the_gpu_suite(L):
    x, ids = z(3, 16), z(3, 16, dt=torch.int32)
    d = g.tensor_desc(ids)
    assert call(L.emu_argsort, g.tensor_desc(x), d, 0) == OK
    assert call(L.emu_argsort, g.tensor_desc(x), d, 2) == EINVAL                                        # order neither 0 nor 1
    assert call(L.emu_argsort, g.tensor_desc(x), d, -1) == EINVAL
    assert call(L.emu_argsort, g.tensor_desc(x.half()), d, 0) == EUNSUPPORTED                           # src not f32
    assert call(L.emu_argsort, g.tensor_desc(x), g.tensor_desc(x), 0) == EUNSUPPORTED                   # dst not i32
    s = g.tensor_desc(x); s.nb[0] = 8; s.ne[0] = 8
    assert call(L.emu_argsort, s, g.tensor_desc(ids[:, :8].contiguous()), 0) == EUNSUPPORTED            # nb0 != 4
    assert call(L.emu_argsort, g.tensor_desc(x), g.tensor_desc(ids[:2].contiguous()), 0) == EUNSUPPORTED  # dst shape
    nc = g.tensor_desc(ids); nc.ne[0] = 8                                                               # dst rows of 8 with a stride of 16
    assert call(L.emu_argsort, g.tensor_desc(x[:, :8].contiguous()), nc, 0) == EUNSUPPORTED             # non-contiguous dst
    assert call(L.emu_argsort, g.tensor_desc(z(1, 1025)), g.tensor_desc(z(1, 1025, dt=torch.int32)), 0) == EUNSUPPORTED   # ne0 > 1024
    assert call(L.emu_argsort, g.tensor_desc(z(2, 1024)), g.tensor_desc(z(2, 1024, dt=torch.int32)), 1) == OK

    y = g.tensor_desc(z(3, 1))
    assert call(L.emu_sum_rows, g.tensor_desc(x), y) == OK
    assert call(L.emu_sum_rows, g.tensor_desc(x.half()), y) == EUNSUPPORTED                             # wrong type
    assert call(L.emu_sum_rows, g.tensor_desc(x), g.tensor_desc(ids[:, :1].contiguous())) == EUNSUPPORTED
    s = g.tensor_desc(x); s.nb[0] = 8; s.ne[0] = 8
    assert call(L.emu_sum_rows, s, y) == EUNSUPPORTED                                                   # nb0 != 4
    assert call(L.emu_sum_rows, g.tensor_desc(x), g.tensor_desc(z(2, 1))) == EUNSUPPORTED               # dst shape


def test_concat_ssm_conv_and_ssm_scan_cases_of_the_gpu_suite(L):
    a, b, d = z(2, 3, 4), z(2, 3, 5), z(2, 3, 9)
    assert call(L.emu_concat, D(a), D(b), D(d), 0) == OK
    assert call(L.emu_concat, D(a), D(b), D(d), 4) == EINVAL and call(L.emu_concat, D(a), D(b), D(d), -1) == EINVAL     # bad dim
    assert call(L.emu_concat, D(a.half()), D(b.half()), D(d.half()), 0) == EUNSUPPORTED                 # f16 (the plug-in declines it too)
    assert call(L.emu_concat, D(a), D(b.int()), D(d), 0) == EUNSUPPORTED                                # mixed types
    assert call(L.emu_concat, D(z(2, 4, 3).transpose(1, 2)), D(b), D(d), 0) == EUNSUPPORTED            # src0 nb0 != 4
    assert call(L.emu_concat, D(a), D(b), D(z(2, 3, 8)), 0) == EUNSUPPORTED                             # dst extent along dim
    assert call(L.emu_concat, D(a), D(z(2, 4, 5)), D(d), 0) == EUNSUPPORTED                             # shapes differ outside dim
    assert call(L.emu_concat, D(a), D(z(2, 3, 5).transpose(1, 2).contiguous().transpose(1, 2)), D(d), 0) == OK   # src1 may be any view

    sx, c, y = z(2, 16, 3 + 5), z(16, 4), z(2, 5, 16)
    assert call(L.emu_ssm_conv, D(sx), D(c), D(y)) == OK
    assert call(L.emu_ssm_conv, D(sx.half()), D(c), D(y)) == EUNSUPPORTED                               # type
    assert call(L.emu_ssm_conv, D(z(2, 16, 16)[:, :, :8]), D(c), D(y)) == EUNSUPPORTED                  # sx rows not packed (the plug-in declines it too)
    assert call(L.emu_ssm_conv, D(sx), D(z(16, 8)[:, :4]), D(y)) == EUNSUPPORTED                        # c rows not packed
    assert call(L.emu_ssm_conv, D(sx), D(z(15, 4)), D(y)) == EUNSUPPORTED                               # d_inner mismatch
    assert call(L.emu_ssm_conv, D(sx), D(c), D(z(2, 4, 16))) == EUNSUPPORTED                            # n_t mismatch
    assert call(L.emu_ssm_conv, D(sx), D(c), D(z(2, 16, 5).transpose(1, 2))) == EUNSUPPORTED           # dst nb0 != 4
    assert call(L.emu_ssm_conv, D(z(1, 2, 16, 8)[0:1].expand(2, 2, 16, 8)), D(c), D(y)) == EUNSUPPORTED   # sx not 3-D

    ns, nt, di, ds = 2, 3, 8, 4
    s, x, dt, A, B = z(ns, di, ds), z(ns, nt, di), z(ns, nt, di), z(di, ds), z(ns, nt, ds)
    out = z(x.numel() + s.numel())

    def scan(*t, d=out):
        return call(L.emu_ssm_scan, *[D(v) for v in t], D(d))
    assert scan(s, x, dt, A, B, B) == OK
    assert scan(s.half(), x, dt, A, B, B) == EUNSUPPORTED                                               # type
    assert scan(z(ns, ds, di).transpose(1, 2), x, dt, A, B, B) == EUNSUPPORTED                          # s not contiguous
    assert scan(s, z(ns, di, nt).transpose(1, 2), dt, A, B, B) == EUNSUPPORTED                          # x not contiguous
    assert scan(s, x, z(ns, nt, di + 1), A, B, B) == EUNSUPPORTED                                       # dt shape
    assert scan(s, x, dt, z(di, ds + 1), B, B) == EUNSUPPORTED                                          # A shape
    assert scan(s, x, dt, A, z(ns, nt, ds + 1), z(ns, nt, ds + 1)) == EUNSUPPORTED                      # B shape
    assert scan(s, x, dt, A, z(ns, ds, nt).transpose(1, 2), B) == EUNSUPPORTED                          # B nb0 != 4
    assert scan(s, x, dt, A, B, B, d=z(x.numel() + s.numel() - 1)) == EUNSUPPORTED                      # dst size
    xdb = z(ns, nt, 3 + 2 * ds)
    assert scan(s, x, dt, A, xdb[:, :, 3:3 + ds], xdb[:, :, 3 + ds:]) == OK                             # strided B / C views
    big = (T(F32, (1, 1, 65536)), T(F32, (1, 1, 65536)), T(F32, (1, 1, 65536)), T(F32, (1, 1)), T(F32, (1, 1, 65536)), T(F32, (1, 1, 65536)))
    assert call(L.emu_ssm_scan, *big, T(F32, (2 * 65536,))) == EUNSUPPORTED                             # n_s beyond the grid's y (declined by the plug-in)


# ------------------------------------------------------------------ nodes the plug-in accepted but the launcher refused
def test_flash_attn_ext_v_and_mask_must_match_k(L):
    q, k, mask, dst = T(F32, (64, 7, 16)), T(F16, (64, 32, 4)), T(F16, (32, 64)), T(F32, (64, 16, 7))
    assert call(L.emu_flash_attn_ext, q, k, k, mask, dst) == OK
    assert call(L.emu_flash_attn_ext, q, k, T(F16, (64, 31, 4)), mask, dst) == EUNSUPPORTED            # V has another n_kv than K
    assert call(L.emu_flash_attn_ext, q, k, T(F16, (64, 32, 3)), mask, dst) == EUNSUPPORTED            # V heads do not broadcast
    assert call(L.emu_flash_attn_ext, q, k, k, T(F16, (31, 64)), dst) == EUNSUPPORTED                  # mask shorter than n_kv
    assert call(L.emu_flash_attn_ext, q, k, T(F16, (64, 32, 0)), mask, dst) == EUNSUPPORTED            # no V heads: refused, not divided by


def test_sum_rows_beyond_one_grid(L):
    rows = 4 * 0x7fffffff + 1
    assert call(L.emu_sum_rows, T(F32, (1, rows)), T(F32, (1, rows))) == EUNSUPPORTED
    assert call(L.emu_sum_rows, T(F32, (1, rows - 1)), T(F32, (1, rows - 1))) == OK


# ------------------------------------------------------------------ the decoder presets' nodes
@pytest.mark.parametrize("preset", ["norm", "neox"])
@pytest.mark.parametrize("N,n_past", [(7, 0), (1, 7)], ids=["prompt", "decode"])
def test_llama_preset_nodes_are_accepted(L, preset, N, n_past):
    n_embd, n_head, n_head_kv, hd, n_vocab, n_ctx = 1024, 16, 4, 64, 4096, 64
    ngqa, n_kv = n_head_kv * hd, n_past + N
    neox = preset == "neox"
    x = T(F32, (n_embd, N))
    assert call(L.emu_get_rows, T(Q4_K, (n_embd, n_vocab)), T(I32, (N,)), x) == OK
    assert call(L.emu_norm, x, x) == OK
    assert call(L.emu_norm_affine, x, x, C.c_void_p(64), x, C.c_void_p(64), x) == OK
    assert call(L.emu_bin_bcast, 1, x, T(F32, (n_embd,)), x) == OK
    assert call(L.emu_bin_bcast, 0, x, x, x) == OK
    p = g.rope_params(32 if neox else 64, g.ROPE_NEOX if neox else g.ROPE_NORM, n_ctx_orig=512, freq_scale=0.25 if neox else 1.0,
                      ext_factor=0.5 if neox else 0.0)
    ff = T(F32, (16,)) if neox else None
    for heads in (n_head, n_head_kv):
        r = T(F32, (hd, heads, N))
        assert call(L.emu_rope, r, T(I32, (N,)), ff, r, p) == OK
    k_src, k_dst = T(F32, (hd, n_head_kv, N)), T(F16, (N * ngqa,), (2, 2 * N * ngqa, 2 * N * ngqa, 2 * N * ngqa))
    assert call(L.emu_cpy, k_src, k_dst) == OK
    assert call(L.emu_cpy2, k_src, k_dst, k_src, k_dst) == OK
    Q = T(F32, (hd, N, n_head), (4, 4 * hd * n_head, 4 * hd, 4 * hd * n_head * N))                       # permute(q, 0, 2, 1, 3)
    K = T(F16, (hd, n_kv, n_head_kv), (2, 2 * ngqa, 2 * hd, 2 * ngqa * n_ctx))
    if neox:
        mask = T(F16, (n_kv, 64))
        assert call(L.emu_flash_attn_ext, Q, K, K, mask, T(F32, (hd, n_head, N))) == OK
    else:
        vt = T(F16, (N, ngqa), (2, 2 * n_ctx, 2 * n_ctx * ngqa, 2 * n_ctx * ngqa))
        assert call(L.emu_cpy, T(F32, (N, ngqa), (4 * ngqa, 4, 4 * ngqa * N, 4 * ngqa * N)), vt) == OK   # CPY(transpose(v), view of the V cache)
        kq = T(F32, (n_kv, N, n_head))
        assert call(L.emu_mul_mat_f, K, Q, kq) == OK
        V = T(F16, (n_kv, hd, n_head_kv), (2, 2 * n_ctx, 2 * n_ctx * hd, 2 * n_ctx * hd * n_head_kv))
        kqv = T(F32, (hd, N, n_head))
        assert call(L.emu_mul_mat_f, V, kq, kqv) == OK
        assert call(L.emu_cpy, T(F32, (hd, n_head, N), (4, 4 * hd * N, 4 * hd, 4 * hd * N * n_head)), x) == OK   # CONT of the permuted kqv


@pytest.mark.parametrize("n_expert,n_used", [(8, 2), (60, 4)], ids=["moe", "moe60"])
@pytest.mark.parametrize("N", [7, 1], ids=["prompt", "decode"])
def test_moe_preset_nodes_are_accepted(L, n_expert, n_used, N):
    n_embd = 1024
    probs = T(F32, (n_expert, N))
    assert call(L.emu_argsort, probs, T(I32, (n_expert, N)), 1) == OK
    selected = T(I32, (n_used, N), (4, 4 * n_expert, 4 * n_expert * N, 4 * n_expert * N))             # the first n_used columns of ARGSORT
    weights = T(F32, (1, n_used, N))
    assert call(L.emu_get_rows, T(F32, (1, n_expert, N)), selected, weights) == OK
    w2, sums = T(F32, (n_used, N)), T(F32, (1, N))
    assert call(L.emu_sum_rows, w2, sums) == OK
    assert call(L.emu_bin_bcast, 3, w2, sums, w2) == OK
    expert = T(F32, (n_embd, N), (4, 4 * n_embd * n_used, 4 * n_embd * n_used * N, 4 * n_embd * n_used * N))   # view of experts[:, i, :]
    assert call(L.emu_bin_bcast, 0, expert, expert, T(F32, (n_embd, N))) == OK


@pytest.mark.parametrize("d_inner,dt_rank,n_s", [(1536, 48, 2), (2048, 64, 1)], ids=["mamba", "falcon"])
@pytest.mark.parametrize("n_t", [7, 1], ids=["prompt", "decode"])
def test_mamba_preset_nodes_are_accepted(L, d_inner, dt_rank, n_s, n_t):
    d_state, d_conv = 16, 4
    conv = T(F32, (d_conv - 1, d_inner, n_s))
    xz_nb1 = 4 * 2 * d_inner
    xt = T(F32, (n_t, d_inner, n_s), (xz_nb1, 4, xz_nb1 * n_t, xz_nb1 * n_t * n_s))                    # transpose(view of xz)
    conv_x = T(F32, (d_conv - 1 + n_t, d_inner, n_s))
    assert call(L.emu_concat, conv, xt, conv_x, 0) == OK
    cx_nb1 = 4 * (d_conv - 1 + n_t)
    last = T(F32, (d_conv - 1, d_inner, n_s), (4, cx_nb1, cx_nb1 * d_inner, cx_nb1 * d_inner * n_s))
    assert call(L.emu_cpy, last, T(F32, ((d_conv - 1) * d_inner * n_s,))) == OK
    x = T(F32, (d_inner, n_t, n_s))
    assert call(L.emu_ssm_conv, conv_x, T(F32, (d_conv, d_inner)), x) == OK
    db_nb1 = 4 * (dt_rank + 2 * d_state)
    B = T(F32, (d_state, n_t, n_s), (4, db_nb1, db_nb1 * n_t, db_nb1 * n_t * n_s))                     # views of x_db
    s = T(F32, (d_state, d_inner, n_s))
    y = T(F32, (d_inner * n_t * n_s + d_state * d_inner * n_s,))
    assert call(L.emu_ssm_scan, s, x, x, T(F32, (d_state, d_inner)), B, B, y) == OK
