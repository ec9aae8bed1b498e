"""GPU: GGML_OP_IM2COL and f16 x f16 GGML_OP_MUL_MAT on the device (ops.cu im2col_kernel and mul_mat_f_kernel, the tensor-core GEMM of
mmq_tc2.cu with both operands by TMA, behind ggml_b200_op_im2col / ggml_b200_mul_mat_f16_f16 and the plug-in), and Whisper-style
encoder-decoder graphs whose convolutional front end uses them (oracle/whisper_graph.cpp).

  (a) the reference's own test-backend-ops runs every IM2COL case and every f16 x f16 MUL_MAT case on B2000 against ggml-cpu: all executed
      and passed, none declined;
  (b) one-node graphs (oracle/conv_probe.cpp) on B2000 and on ggml-cpu: IM2COL bit-identical over the host test's grid and at Whisper-large's
      conv1 shape; f16 x f16 on the plain kernel and on the tensor cores within NMSE 1e-10 (the fp16 products are exact, only the order of
      the f32 sums differs), ggml_conv_1d end to end too; the workspace query shows which shapes take the tensor cores; what the C ABI
      declines the plug-in declines;
  (c) the C ABI: invalid arguments give error codes; a captured CUDA graph of IM2COL -> f16 x f16 GEMM, replayed on new inputs, equals eager
      launches bit for bit;
  (d) the `tiny` and `large` presets: every f32 node matches ggml-cpu on identical inputs to NMSE 1e-9 (two IM2COL nodes in the prompt
      graph, both conv mat-muls among the nodes; tiny's Q8_0 encoder linears over 1500 frames, on the existing quantized tensor-core GEMM
      with fp16 activations, and large's FLASH_ATTN_EXT nodes over the 1500 frames, on the existing attention kernel, to the reference's
      5e-4), free-running
      logits stay close, the whole graph is one split with no CPU node, teacher-forced logits track ggml-cpu, and fusions / CUDA-graph
      replay change no logit bit."""
import subprocess

import numpy as np
import pytest

from oracle import conv as V
from oracle import decoder
from oracle import oracle as O

pytestmark = pytest.mark.gpu
PRESETS = ("tiny", "large")
EXE = O.REF_DIR / "whisper-graph"


@pytest.fixture(scope="module")
def plugin():
    return decoder.plugin("test-backend-ops", "whisper-graph", "libggml_conv_probe.so")


# ------------------------------------------------------------------ (a) the reference's test-backend-ops
def test_reference_test_backend_ops_im2col(plugin):
    decoder.check_test_backend_ops(plugin, "IM2COL", 86)


def test_reference_test_backend_ops_mul_mat_f16_f16(plugin):
    env = O.ref_env()
    env["GGML_BACKEND_PATH"] = str(plugin)
    p = subprocess.run([str(O.REF_DIR / "test-backend-ops"), "test", "-o", "MUL_MAT", "-b", "B2000"], env=env, capture_output=True, text=True, timeout=1800)
    out = p.stdout + p.stderr
    tail = "\n".join(out.splitlines()[-25:])
    assert p.returncode == 0 and "FAIL" not in out, tail
    lines = [l for l in out.splitlines() if l.strip().startswith("MUL_MAT(") and "type_a=f16,type_b=f16" in l]
    assert len(lines) >= 24, (len(lines), tail)
    bad = [l for l in lines if "OK" not in l]
    assert not bad, "\n".join(bad[:10])
    print(f"test-backend-ops MUL_MAT f16 x f16 on B2000: {len(lines)} cases executed and OK")


# ------------------------------------------------------------------ (b) probe parity, device vs ggml-cpu
def test_im2col_device_is_bit_identical_to_cpu(plugin):
    cases = V.im2col_grid() + [
        V.Im2colCase((3, 128, 1280, 1), (3000, 128, 1, 1), 1, 0, 1, 0, 1, 0, False, V.F16, V.F16, 0, seed=900),    # Whisper-large conv1
        V.Im2colCase((3, 128, 1280, 1), (3000, 128, 1, 1), 1, 0, 1, 0, 1, 0, False, V.F32, V.F32, 0, seed=901),
    ]
    for case in cases:
        view = case.view_of_input()
        got, want = V.im2col("B2000", case, view), V.im2col("CPU", case, view)
        u = np.uint16 if case.dst_type == V.F16 else np.uint32
        assert np.array_equal(got.view(u), want.view(u)), (str(case), int((got.view(u) != want.view(u)).sum()))
    print(f"IM2COL B2000 vs ggml-cpu: {len(cases)} cases (1-D / 2-D, f32 / f16 columns, strided inputs, Whisper-large conv1) bit-identical")


# (M, N, K, b_view): the Whisper conv shapes (M: output frames, N: output channels, K: 3 x input channels) and small strided ones
MM_SHAPES = [(3000, 384, 240, 0), (1500, 384, 1152, 0), (3000, 1280, 384, 0), (1500, 1280, 3840, 0), (1500, 512, 1536, 1),
             (300, 64, 192, 0), (64, 16, 256, 2), (100, 9, 64, 1), (37, 5, 128, 0)]


def test_mul_mat_f16_f16_device_matches_cpu_on_both_routes(plugin):
    import ggml_b200 as g
    worst = {True: 0.0, False: 0.0}
    for i, (M, N, K, bv) in enumerate(MM_SHAPES):
        ops = V.f16_operands(M, N, K, bv, seed=i)
        got, want = V.mul_mat_f16("B2000", M, N, K, bv, ops), V.mul_mat_f16("CPU", M, N, K, bv, ops)
        # the plug-in takes the tensor cores exactly where the C ABI's workspace query accepts the shape and b's rows are 16-byte aligned
        # (views 0 and 1; view 2 pads them to K + 3 elements)
        tc = bv != 2 and g.mul_mat_f16_f16_workspace_size(M, N, K) > 0
        assert tc == (N >= 9 and K % 64 == 0 and bv != 2), (M, N, K, bv)
        e = O.nmse(got, want)
        assert np.isfinite(got).all() and e <= 1e-10, (M, N, K, bv, tc, e)
        assert O.nmse(got, V.mul_mat_f16_reference(*ops, bv)) <= 1e-10
        worst[tc] = max(worst[tc], e)
    assert g.mul_mat_f16_f16_workspace_size(1500, 384, 1152) > 0 and g.mul_mat_f16_f16_workspace_size(3000, 384, 240) == 0
    print(f"f16 x f16 MUL_MAT B2000 vs ggml-cpu: worst NMSE tensor cores {worst[True]:.2e}, plain kernel {worst[False]:.2e}")


def test_conv_1d_device_matches_cpu(plugin):
    worst = 0.0
    for i, (KW, IC, OC, L, s, p, d) in enumerate([(3, 80, 384, 3000, 1, 1, 1), (3, 384, 384, 3000, 2, 1, 1), (3, 128, 256, 600, 1, 1, 1),
                                                  (5, 16, 32, 97, 2, 2, 2)]):
        got, want = V.conv_1d("B2000", KW, IC, OC, L, s, p, d, seed=i), V.conv_1d("CPU", KW, IC, OC, L, s, p, d, seed=i)
        e = O.nmse(got, want)
        assert e <= 1e-10, (KW, IC, OC, L, s, p, d, e)
        worst = max(worst, e)
    print(f"ggml_conv_1d (IM2COL + f16 x f16 MUL_MAT) B2000 vs ggml-cpu: worst NMSE {worst:.2e}")


def test_what_the_abi_declines_the_plugin_declines(plugin):
    f32_kernel_f16_cols = V.Im2colCase((3, 4, 6, 1), (17, 4, 1, 1), 1, 0, 1, 0, 1, 0, False, V.F16, V.F32)
    assert V.im2col("B2000", f32_kernel_f16_cols, raw=True) == -2                  # ggml-cpu asserts an f16 kernel for f16 columns
    assert V.im2col("B2000", V.Im2colCase((3, 4, 6, 1), (17, 4, 1, 1), 1, 0, 1, 0, 1, 0, False, V.F16, V.F16), raw=True) == 0


# ------------------------------------------------------------------ (c) the C ABI
def test_c_abi_error_codes():
    import ctypes as C
    import torch
    import ggml_b200 as g
    L = g.lib()
    L.ggml_b200_op_im2col.argtypes = [C.POINTER(g.TensorDesc)] * 3 + [C.POINTER(g.Im2colParams), C.c_void_p]
    D = g.strided_desc
    z = lambda *shape, dt=torch.float32: torch.zeros(shape, dtype=dt, device="cuda")

    def im2col(k, x, d, p):
        return L.ggml_b200_op_im2col(C.byref(D(k)), C.byref(D(x)), C.byref(D(d)), C.byref(p), None)
    P = lambda s0=1, p0=1, d0=1, two=0: g.Im2colParams(s0, 0, p0, 0, d0, 0, two)
    k, x, y = z(6, 4, 3, dt=torch.float16), z(2, 4, 17), z(2, 17, 12, dt=torch.float16)
    assert im2col(k, x, y, P()) == 0
    assert im2col(k, x, y, P(two=3)) == -2 and im2col(k, x, y, P(s0=0)) == -2 and im2col(k, x, y, P(d0=0)) == -2
    assert im2col(k.float(), x, y, P()) == -1                                       # f16 columns need an f16 kernel
    assert im2col(k, x.half(), y, P()) == -1                                        # f32 input only
    assert im2col(k, z(2, 17, 4).transpose(1, 2), y, P()) == -1                    # input nb0 != 4
    assert im2col(k, x, z(2, 12, 17, dt=torch.float16).transpose(1, 2), P()) == -1  # columns not packed
    assert im2col(k, x, z(2, 16, 12, dt=torch.float16), P()) == -1                  # OW
    assert im2col(k, z(2, 4, 20)[:, :, :17], y, P()) == 0                           # any input strides beyond nb0

    w, xx = z(1500, 1152, dt=torch.float16), z(384, 1152, dt=torch.float16)
    need = g.mul_mat_f16_f16_workspace_size(1500, 384, 1152)
    assert need > 0 and g.mul_mat_f16_f16_workspace_size(1500, 8, 1152) == 0 and g.mul_mat_f16_f16_workspace_size(1500, 384, 1000) == 0
    L.ggml_b200_mul_mat_f16_f16.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_int64, C.c_int64, C.c_int64,
                                            C.c_void_p, C.c_size_t, C.c_uint32, C.c_void_p]
    out, ws = z(384, 1500), torch.empty(need, dtype=torch.uint8, device="cuda")

    def mm(M, N, K, nb01=2 * 1152, nb11=2 * 1152, wsz=need):
        return L.ggml_b200_mul_mat_f16_f16(w.data_ptr(), nb01, xx.data_ptr(), nb11, out.data_ptr(), M, N, K, ws.data_ptr(), wsz, 0, None)
    assert mm(1500, 384, 1152) == 0
    assert mm(1500, 384, 1152, wsz=need - 1) == -3                                  # workspace too small
    assert mm(1500, 8, 1152) == -1 and mm(1500, 384, 1000, nb01=2000, nb11=2000) == -1   # N < 9, K % 64
    assert mm(1500, 384, 1152, nb11=2 * 1152 + 8) == -1                             # row stride not a multiple of 16 bytes
    assert mm(0, 384, 1152) == 0
    torch.cuda.synchronize()


def test_c_abi_cuda_graph_replay_matches_eager():
    import torch
    import ggml_b200 as g
    torch.cuda.set_device(0)
    IC, OC, L_ = 384, 384, 3000
    kernel = torch.zeros((OC, IC, 3), dtype=torch.float16, device="cuda")
    x = torch.zeros((1, IC, L_), device="cuda")

    def conv():
        cols = g.op_im2col(kernel, x, 2, 1, 1)                               # [1, 1500, 3 IC] f16
        y = g.mul_mat_f16_f16(cols[0], kernel.reshape(OC, 3 * IC))           # [OC, 1500]: the tensor cores
        return cols, y
    conv()                                                                   # workspace and per-device set-up outside the capture
    torch.cuda.synchronize()
    stream = torch.cuda.Stream()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=stream):
        captured = conv()
    rng = np.random.default_rng(31)
    for _ in range(3):
        kernel.copy_(torch.from_numpy((rng.standard_normal((OC, IC, 3)) / np.sqrt(3 * IC)).astype(np.float16)))
        x.copy_(torch.from_numpy(rng.standard_normal((1, IC, L_)).astype(np.float32)))
        graph.replay()
        torch.cuda.synchronize()
        eager = conv()
        torch.cuda.synchronize()
        assert torch.equal(captured[0].view(torch.int16), eager[0].view(torch.int16))
        assert torch.equal(captured[1].view(torch.int32), eager[1].view(torch.int32))
        ref = torch.nn.functional.conv1d(x.double(), kernel.double(), stride=2, padding=1)[0]
        assert O.nmse(eager[1].cpu().numpy(), ref.float().cpu().numpy()) < 1e-5


# ------------------------------------------------------------------ (d) the Whisper presets
def compare_raw(preset: str, sync: bool):
    """compare mode on B2000: (summary per phase, node lines, {phase: IM2COL nodes in its graph})"""
    out = decoder._run(EXE, [preset, "compare", "B2000"] + (["sync"] if sync else []))
    summary, nodes, im2col = {}, [], {}
    for l in out.splitlines():
        f = l.split()
        if f and f[0] == "summary":
            summary[f[1]] = dict(n_over=int(f[4]), worst=float(f[6]), logits=float(f[11]))
        elif f and f[0] == "node":
            nodes.append(f)
        elif f and f[0] == "graph":
            im2col[f[1]] = int(f[5])
    return summary, nodes, im2col


@pytest.mark.parametrize("preset", PRESETS)
def test_whisper_graph_every_node_matches_cpu_on_identical_inputs(plugin, preset):
    summary, nodes, im2col = compare_raw(preset, sync=True)
    assert set(summary) == {"prompt", "decode"}, summary
    assert im2col == {"prompt": 2, "decode": 0}, im2col
    n_state = {"tiny": 384, "large": 1280}[preset]
    conv, q8_gemm, fattn, worst = [], 0.0, 0.0, 0.0
    for n in nodes:
        ne = [int(v) for v in n[-3].strip("[]").split(",")]         # the name before it may contain spaces
        e = float(n[-1])
        if n[3] == "MUL_MAT" and ne[1] == n_state and ne[0] in (3000, 1500):
            conv.append(e)                                        # the conv mat-muls (f16 x f16): [frames, channels]
        if preset == "tiny" and n[1] == "prompt" and n[3] == "MUL_MAT" and ne[:2] == [n_state, 1500]:
            # tiny's Q8_0 encoder linears over 1500 frames run on the quantized tensor-core GEMM, whose activations are fp16 where ggml-cpu's
            # are Q8_0 blocks: that route's documented NMSE (~1e-7 .. 1e-5) against the reference's MUL_MAT gate of 5e-4
            assert e <= 5e-4, n
            q8_gemm = max(q8_gemm, e)
            continue
        if n[3] == "FLASH_ATTN_EXT":
            # over the 1500 audio frames with f16 K / V: ggml-cpu accumulates an f16 V in f16, the existing device kernel in f32 (ops.cu);
            # the reference's gate for the op is 5e-4
            assert e <= 5e-4, n
            fattn = max(fattn, e)
            continue
        assert e <= 1e-9, n
        worst = max(worst, e)
    assert len(conv) == 2, conv
    print(f"whisper graph [{preset}], identical inputs per node: conv mat-muls NMSE {conv[0]:.2e}, {conv[1]:.2e}; worst other node "
          f"{worst:.2e} over {len(nodes)} f32 nodes" + (f"; Q8_0 encoder linears (quantized GEMM) worst {q8_gemm:.2e}" if q8_gemm else "") +
          (f"; FLASH_ATTN_EXT worst {fattn:.2e}" if fattn else ""))


@pytest.mark.parametrize("preset", PRESETS)
def test_whisper_graph_free_running_logits(plugin, preset):
    summary, _, _ = compare_raw(preset, sync=False)
    assert set(summary) == {"prompt", "decode"}, summary
    for phase, s in summary.items():
        assert 0.0 <= s["logits"] <= 5e-3, (phase, s)
    print(f"whisper graph [{preset}], free-running: " + ", ".join(f"{ph}: logits NMSE {s['logits']:.2e}" for ph, s in summary.items()))


@pytest.fixture(scope="module")
def cpu_runs(plugin, tmp_path_factory):
    d = tmp_path_factory.mktemp("whisper_cpu")
    return {p: decoder.run(EXE, p, "CPU", d / f"{p}.logits") for p in PRESETS}


@pytest.mark.parametrize("preset", PRESETS)
def test_whisper_graph_runs_in_one_split_on_the_device(plugin, preset, tmp_path, cpu_runs):
    kv, _ = decoder.run(EXE, preset, "B2000", tmp_path / "l.bin")
    assert int(kv["n_splits"][0]) == 1 and int(kv["cpu_nodes"][0]) == 0, kv
    print(f"whisper graph [{preset}]: one split, no CPU node, decode {kv['decode_ms_per_step'][0]} ms per step on B2000, "
          f"{cpu_runs[preset][0]['decode_ms_per_step'][0]} ms on ggml-cpu")


@pytest.mark.parametrize("preset", PRESETS)
def test_whisper_graph_logits_track_cpu_step_by_step(preset, cpu_runs, tmp_path):
    ties, worst, n_same, ctoks = decoder.check_tracks_cpu(EXE, preset, cpu_runs[preset], tmp_path)
    print(f"whisper graph [{preset}]: {decoder.N_STEPS} teacher-forced steps, worst logits NMSE {worst:.2e}, "
          f"same greedy token at {n_same}/{len(ctoks)}, near-ties {ties[:5]}")


@pytest.mark.parametrize("preset", PRESETS)
def test_whisper_graph_fusions_and_graph_replay_are_bit_exact(plugin, preset, tmp_path):
    decoder.check_fusions_and_graphs_bit_exact(EXE, preset, tmp_path)
