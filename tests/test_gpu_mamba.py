"""GPU: GGML_OP_CONCAT, GGML_OP_SSM_CONV and GGML_OP_SSM_SCAN on the device (ops.cu concat_kernel / ssm_conv_kernel / ssm_scan_kernel behind
ggml_b200_op_concat / _ssm_conv / _ssm_scan and the plug-in), and Mamba decoder graphs that use them (oracle/mamba_graph.cpp).

  (a) the reference's own test-backend-ops runs every CONCAT, SSM_CONV and SSM_SCAN case on B2000 against ggml-cpu: all executed, none declined;
  (b) one-node graphs (oracle/ssm_probe.cpp) on B2000 and on ggml-cpu over the host test's grid: CONCAT and SSM_CONV bit-identical, SSM_SCAN
      y and states within NMSE 1e-10 (the device expf / log1pf against glibc's); what the C ABI declines the plug-in declines;
  (c) the C ABI: invalid arguments give error codes; a captured CUDA graph of the three ops, replayed on new inputs, matches eager launches;
  (d) the `mamba` (Mamba-130m widths, two sequences) and `falcon` (FalconMamba form) presets: every node matches ggml-cpu on identical inputs,
      free-running logits stay close, the whole graph is one split with no CPU node, teacher-forced logits track ggml-cpu, and fusions /
      CUDA-graph replay change no logit bit (a replayed decode graph reads the states the previous replay wrote)."""
import re
import subprocess

import numpy as np
import pytest

from oracle import oracle as O
from oracle import ssm as S

pytestmark = pytest.mark.gpu
PRESETS = {"mamba": 2, "falcon": 1}          # preset -> sequences decoded side by side
N_STEPS = 24
N_VOCAB = 4096
N_LAYER = 4


@pytest.fixture(scope="module")
def plugin():
    import ggml_b200
    if not ggml_b200.BACKEND_SO.exists():
        pytest.fail(f"{ggml_b200.BACKEND_SO} missing: run __graft_entry__.build() where the ggml headers are available")
    for f in ("test-backend-ops", "mamba-graph", "libggml_ssm_probe.so"):
        if not (O.REF_DIR / f).exists():
            pytest.fail(f"oracle/_ref/{f} missing (oracle/Makefile and oracle/mamba.mk in the build container)")
    ref = O.Ref()
    assert ref.load_backend(ggml_b200.BACKEND_SO)
    return ggml_b200.BACKEND_SO


# ------------------------------------------------------------------ (a) the reference's test-backend-ops
@pytest.mark.parametrize("op,n_min", [("CONCAT", 32), ("SSM_CONV", 3), ("SSM_SCAN", 1)])
def test_reference_test_backend_ops(plugin, op, n_min):
    env = O.ref_env()
    env["GGML_BACKEND_PATH"] = str(plugin)
    p = subprocess.run([str(O.REF_DIR / "test-backend-ops"), "test", "-o", op, "-b", "B2000"], env=env, capture_output=True, text=True, timeout=900)
    out = p.stdout + p.stderr
    tail = "\n".join(out.splitlines()[-25:])
    assert p.returncode == 0 and "FAIL" not in out, tail
    cases = [l for l in out.splitlines() if l.strip().startswith(op + "(")]
    declined = [l for l in cases if "not supported" in l]
    assert not declined, "\n".join(declined[:10])
    ok = [l for l in cases if "OK" in l]
    assert len(ok) == len(cases) and len(ok) >= n_min, (len(ok), len(cases), tail)
    m = re.search(r"(\d+)/(\d+) tests passed", out)
    assert m and m.group(1) == m.group(2), tail


# ------------------------------------------------------------------ (b) probe parity, device vs ggml-cpu
def test_concat_device_is_bit_identical_to_cpu(plugin):
    cases = S.concat_grid()
    for case in cases:
        got, want = S.concat("B2000", case), S.concat("CPU", case)
        assert got.dtype == want.dtype and np.array_equal(got.view(np.uint32), want.view(np.uint32)), str(case)
    print(f"CONCAT B2000 vs ggml-cpu: {len(cases)} cases (f32 / i32, dims 0-3, strided and transposed operands) bit-identical")


def test_ssm_conv_device_is_bit_identical_to_cpu(plugin):
    cases = S.conv_grid()
    for case in cases:
        views = case.views()
        got, want = S.ssm_conv("B2000", case, views), S.ssm_conv("CPU", case, views)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (str(case), int(S.ulps_apart(got, want).max()))
    print(f"SSM_CONV B2000 vs ggml-cpu: {len(cases)} cases bit-identical")


def test_ssm_scan_device_matches_cpu(plugin):
    worst_nmse, worst_ulp, n_equal, n_total = 0.0, 0, 0, 0
    for case in S.scan_grid():
        views = case.views()
        (y, st), (wy, wst) = S.ssm_scan("B2000", case, views), S.ssm_scan("CPU", case, views)
        for name, g, w in (("y", y, wy), ("states", st, wst)):
            assert np.isfinite(g).all(), (str(case), name)
            e = O.nmse(g, w)
            assert e <= 1e-10, (str(case), name, e)
            worst_nmse = max(worst_nmse, e)
            worst_ulp = max(worst_ulp, int(S.ulps_apart(g, w).max()))
            n_equal += int((g.view(np.uint32) == w.view(np.uint32)).sum())
            n_total += g.size
    print(f"SSM_SCAN B2000 vs ggml-cpu: worst NMSE {worst_nmse:.2e}, worst distance {worst_ulp} ulp, {n_equal}/{n_total} values bit-identical")


def test_what_the_abi_declines_the_plugin_declines(plugin):
    assert S.concat("B2000", S.ConcatCase(S.F16, (4, 3, 2, 1), (5, 3, 2, 1), 0), raw=True) == -2            # f16: ggml-cpu does not run it
    assert S.ssm_conv("B2000", S.ConvCase(4, 16, 3, 2, view_sx=1), raw=True) == -2                         # sx rows not packed
    assert S.ssm_conv("B2000", S.ConvCase(4, 16, 3, 2, view_c=1), raw=True) == -2                          # c rows not packed
    big = S.ScanCase(1, 1, 1, 65536)                                                                       # n_s beyond the grid's y
    assert S.ssm_scan("B2000", big, raw=True) == -2
    assert S.ssm_scan("CPU", big, raw=True) == 0
    assert S.ssm_scan("B2000", S.ScanCase(1, 1, 1, 65535), raw=True) == 0


# ------------------------------------------------------------------ (c) the C ABI
def test_c_abi_error_codes():
    import ctypes as C
    import torch
    import ggml_b200 as g
    L = g.lib()
    L.ggml_b200_op_concat.argtypes = [C.POINTER(g.TensorDesc)] * 3 + [C.c_int32, C.c_void_p]
    L.ggml_b200_op_ssm_conv.argtypes = [C.POINTER(g.TensorDesc)] * 3 + [C.c_void_p]
    L.ggml_b200_op_ssm_scan.argtypes = [C.POINTER(g.TensorDesc)] * 7 + [C.c_void_p]
    D = g.strided_desc
    z = lambda *shape, dt=torch.float32: torch.zeros(shape, dtype=dt, device="cuda")

    def concat(a, b, d, dim):
        return L.ggml_b200_op_concat(C.byref(a), C.byref(b), C.byref(d), dim, None)
    a, b, d = z(2, 3, 4), z(2, 3, 5), z(2, 3, 9)
    assert concat(D(a), D(b), D(d), 0) == 0
    assert concat(D(a), D(b), D(d), 4) == -2 and concat(D(a), D(b), D(d), -1) == -2                     # bad dim
    assert concat(D(a.half()), D(b.half()), D(d.half()), 0) == -1                                        # f16
    assert concat(D(a), D(b.int()), D(d), 0) == -1                                                       # mixed types
    assert concat(D(z(2, 4, 3).transpose(1, 2)), D(b), D(d), 0) == -1                                  # src0 nb0 != 4
    assert concat(D(a), D(b), D(z(2, 3, 8)), 0) == -1                                                    # dst extent along dim
    assert concat(D(a), D(z(2, 4, 5)), D(d), 0) == -1                                                    # shapes differ outside dim
    assert concat(D(a), D(z(2, 3, 5).transpose(1, 2).contiguous().transpose(1, 2)), D(d), 0) == 0       # src1 may be any view

    def conv(sx, c, d):
        return L.ggml_b200_op_ssm_conv(C.byref(sx), C.byref(c), C.byref(d), None)
    sx, c, y = z(2, 16, 3 + 5), z(16, 4), z(2, 5, 16)
    assert conv(D(sx), D(c), D(y)) == 0
    assert conv(D(sx.half()), D(c), D(y)) == -1                                                          # type
    assert conv(D(z(2, 16, 16)[:, :, :8]), D(c), D(y)) == -1                                             # sx rows not packed
    assert conv(D(sx), D(z(16, 8)[:, :4]), D(y)) == -1                                                   # c rows not packed
    assert conv(D(sx), D(z(15, 4)), D(y)) == -1                                                          # d_inner mismatch
    assert conv(D(sx), D(c), D(z(2, 4, 16))) == -1                                                       # n_t mismatch
    assert conv(D(sx), D(c), D(z(2, 16, 5).transpose(1, 2))) == -1                                      # dst nb0 != 4
    assert conv(D(z(1, 2, 16, 8)[0:1].expand(2, 2, 16, 8)), D(c), D(y)) == -1                           # sx not 3-D

    ns, nt, di, ds = 2, 3, 8, 4
    s, x, dt, A, B = z(ns, di, ds), z(ns, nt, di), z(ns, nt, di), z(di, ds), z(ns, nt, ds)
    out = z(x.numel() + s.numel())

    def scan(*t, d=out):
        return L.ggml_b200_op_ssm_scan(*[C.byref(D(v)) for v in t], C.byref(D(d)), None)
    assert scan(s, x, dt, A, B, B) == 0
    assert scan(s.half(), x, dt, A, B, B) == -1                                                          # type
    assert scan(z(ns, ds, di).transpose(1, 2), x, dt, A, B, B) == -1                                     # s not contiguous
    assert scan(s, z(ns, di, nt).transpose(1, 2), dt, A, B, B) == -1                                     # x not contiguous
    assert scan(s, x, z(ns, nt, di + 1), A, B, B) == -1                                                  # dt shape
    assert scan(s, x, dt, z(di, ds + 1), B, B) == -1                                                     # A shape
    assert scan(s, x, dt, A, z(ns, nt, ds + 1), z(ns, nt, ds + 1)) == -1                                 # B shape
    assert scan(s, x, dt, A, z(ns, ds, nt).transpose(1, 2), B) == -1                                     # B nb0 != 4
    assert scan(s, x, dt, A, B, B, d=z(x.numel() + s.numel() - 1)) == -1                                 # dst size
    xdb = z(ns, nt, 3 + 2 * ds)
    assert scan(s, x, dt, A, xdb[:, :, 3:3 + ds], xdb[:, :, 3 + ds:]) == 0                              # strided B / C views
    torch.cuda.synchronize()


def test_c_abi_cuda_graph_replay_matches_eager():
    import torch
    import ggml_b200 as g
    torch.cuda.set_device(0)
    ns, nt, di, ds, dc = 2, 5, 64, 16, 4
    conv_state, xs = torch.zeros((ns, di, dc - 1), device="cuda"), torch.zeros((ns, nt, di), device="cuda")
    w = torch.zeros((di, dc), device="cuda")
    s0, dt, A = torch.zeros((ns, di, ds), device="cuda"), torch.zeros((ns, nt, di), device="cuda"), torch.zeros((di, ds), device="cuda")
    xdb = torch.zeros((ns, nt, 7 + 2 * ds), device="cuda")

    def layer():
        cx = g.op_concat(conv_state, xs.transpose(1, 2), 0)                 # [ns, di, dc - 1 + nt]: the Mamba layer's conv_x
        u = g.op_ssm_conv(cx, w)                                            # [ns, nt, di]
        y, s_new = g.op_ssm_scan(s0, u, dt, A, xdb[:, :, 7:7 + ds], xdb[:, :, 7 + ds:])
        return cx, u, y, s_new
    layer()                                                                 # lazy per-device set-up outside the capture
    torch.cuda.synchronize()
    stream = torch.cuda.Stream()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=stream):
        captured = layer()
    rng = np.random.default_rng(21)
    for _ in range(3):
        for t in (conv_state, xs, w, s0, xdb):
            t.copy_(torch.from_numpy(rng.standard_normal(tuple(t.shape)).astype(np.float32)))
        dt.copy_(torch.from_numpy(rng.normal(-3.0, 2.0, tuple(dt.shape)).astype(np.float32)))
        A.copy_(-torch.arange(1, ds + 1, dtype=torch.float32, device="cuda").expand(di, ds))
        graph.replay()
        torch.cuda.synchronize()
        eager = layer()
        torch.cuda.synchronize()
        for c, e in zip(captured, eager):
            assert torch.equal(c.view(torch.int32), e.view(torch.int32))
        assert torch.equal(captured[0][:, :, dc - 1:], xs.transpose(1, 2))


# ------------------------------------------------------------------ (d) the Mamba presets
def _run(args, env_extra=None):
    import ggml_b200
    env = O.ref_env()
    env["GGML_BACKEND_PATH"] = str(ggml_b200.BACKEND_SO)
    env.update(env_extra or {})
    p = subprocess.run([str(O.REF_DIR / "mamba-graph"), *args], env=env, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, (p.stdout + p.stderr)[-3000:]
    return p.stdout


def compare(preset, sync):
    out = _run([preset, "compare", "B2000"] + (["sync"] if sync else []))
    summary = {}
    for l in out.splitlines():
        f = l.split()
        if f and f[0] == "summary":
            summary[f[1]] = dict(n_over=int(f[4]), worst=float(f[6]), first=int(f[8]), op=f[9], logits=float(f[11]))
    nodes = [l.split() for l in out.splitlines() if l.startswith("node ")]
    return summary, nodes


def run(preset, dev, path, force=None, env_extra=None):
    out = _run([preset, "run", dev, str(N_STEPS), str(path)] + ([str(force)] if force else []), env_extra)
    kv = {l.split()[0]: l.split()[1:] for l in out.splitlines() if l.strip()}
    logits = np.fromfile(path, dtype=np.float32).reshape(-1, N_VOCAB)
    assert logits.shape[0] == N_STEPS * PRESETS[preset]
    return kv, logits


@pytest.mark.parametrize("preset", list(PRESETS))
def test_mamba_graph_every_node_matches_cpu_on_identical_inputs(plugin, preset):
    summary, nodes = compare(preset, sync=True)
    assert set(summary) == {"prompt", "decode"}, summary
    for n in nodes:
        assert float(n[-1]) <= 1e-9, n
    for phase in ("prompt", "decode"):
        ops = [n[3] for n in nodes if n[1] == phase]
        for op in ("SSM_SCAN", "SSM_CONV", "CONCAT"):
            assert ops.count(op) == N_LAYER, (phase, op, ops.count(op))
    print(f"mamba graph [{preset}], identical inputs per node: worst NMSE prompt {summary['prompt']['worst']:.2e}, "
          f"decode {summary['decode']['worst']:.2e} over {len(nodes)} f32 nodes")


@pytest.mark.parametrize("preset", list(PRESETS))
def test_mamba_graph_free_running_logits(plugin, preset):
    summary, _ = compare(preset, sync=False)
    assert set(summary) == {"prompt", "decode"}, summary
    for phase, s in summary.items():
        assert 0.0 <= s["logits"] <= 5e-3, (phase, s)
    print(f"mamba graph [{preset}], free-running: " + ", ".join(f"{ph}: logits NMSE {s['logits']:.2e}" for ph, s in summary.items()))


@pytest.fixture(scope="module")
def cpu_runs(plugin, tmp_path_factory):
    d = tmp_path_factory.mktemp("mamba_cpu")
    return {p: run(p, "CPU", d / f"{p}.logits") for p in PRESETS}


@pytest.mark.parametrize("preset", list(PRESETS))
def test_mamba_graph_runs_in_one_split_on_the_device(plugin, preset, tmp_path):
    kv, _ = run(preset, "B2000", tmp_path / "l.bin")
    assert int(kv["n_splits"][0]) == 1 and int(kv["cpu_nodes"][0]) == 0, kv
    print(f"mamba graph [{preset}]: one split, no CPU node, decode {kv['decode_ms_per_step'][0]} ms per step")


@pytest.mark.parametrize("preset", list(PRESETS))
def test_mamba_graph_logits_track_cpu_step_by_step(preset, cpu_runs, tmp_path):
    ckv, cpu_logits = cpu_runs[preset]
    ctoks = [int(t) for t in ckv["tokens"]]
    assert ctoks == [int(v) for v in cpu_logits.argmax(1)]
    force = tmp_path / "force.bin"
    np.array(ctoks, dtype=np.int32).tofile(force)
    _, gpu_logits = run(preset, "B2000", tmp_path / "forced.bin", force=force)
    ties, worst, n_same = [], 0.0, 0
    for i in range(cpu_logits.shape[0]):
        c, g_ = cpu_logits[i].astype(np.float64), gpu_logits[i].astype(np.float64)
        nm = O.nmse(gpu_logits[i], cpu_logits[i])
        worst = max(worst, nm)
        assert nm <= 5e-3, (preset, i, nm)
        rms = float(np.sqrt(np.mean((g_ - c) ** 2)))
        top2 = np.sort(c)[-2:]
        margin = float(top2[1] - top2[0])
        if int(g_.argmax()) != int(c.argmax()):
            ties.append((i, margin, rms))
            assert margin <= 6 * rms, f"{preset}: row {i}: argmax differs although the CPU margin {margin:.3e} exceeds 6 x the RMS deviation {rms:.3e}"
        else:
            n_same += 1
    assert n_same >= cpu_logits.shape[0] // 2, (n_same, ties)
    print(f"mamba graph [{preset}]: {N_STEPS} teacher-forced steps x {PRESETS[preset]} sequences, worst logits NMSE {worst:.2e}, "
          f"same greedy token at {n_same}/{cpu_logits.shape[0]}, near-ties {ties[:5]}")


@pytest.mark.parametrize("preset", list(PRESETS))
def test_mamba_graph_fusions_and_graph_replay_are_bit_exact(plugin, preset, tmp_path):
    force = tmp_path / "force.bin"
    np.arange(100, 100 + N_STEPS * PRESETS[preset], dtype=np.int32).tofile(force)
    outs = {}
    for name, env in (("default", {}), ("nofusion", {"GGML_B200_DISABLE_FUSION": "1"}), ("nographs", {"GGML_B200_DISABLE_GRAPHS": "1"})):
        _, outs[name] = run(preset, "B2000", tmp_path / f"{name}.bin", force=force, env_extra=env)
    for name in ("nofusion", "nographs"):
        assert np.array_equal(outs["default"].view(np.uint32), outs[name].view(np.uint32)), (preset, name)
