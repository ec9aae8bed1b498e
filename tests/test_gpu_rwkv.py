"""GPU: GGML_OP_RWKV_WKV6 and GGML_OP_GATED_LINEAR_ATTN on the device (ops.cu wkv_kernel behind ggml_b200_op_rwkv_wkv6 /
_gated_linear_attn and the plug-in), GGML_OP_SQR / GGML_OP_SQRT through the unary kernel, and RWKV-6 decoder graphs that use them
(oracle/rwkv_graph.cpp).

  (a) the reference's own test-backend-ops runs every RWKV_WKV6, GATED_LINEAR_ATTN, SQR and SQRT case on B2000 against ggml-cpu: all
      executed, none declined;
  (b) one-node graphs (oracle/wkv_probe.cpp) on B2000 and on ggml-cpu over the host test's grid: bit-identical where S is a multiple of 16
      (ggml-cpu's fused vector path in every column on every build), NMSE <= 1e-12 for S 8 / 24; SQR and SQRT bit-identical; what the C ABI
      declines the plug-in declines;
  (c) the C ABI: invalid arguments give error codes; a captured CUDA graph of both ops, replayed on new inputs, matches eager launches;
  (d) the `rwkv6` (RWKV-6 1.6B widths, two sequences) and `qrwkv` (RWKV6-Qwen2 form) presets: every node matches ggml-cpu on identical
      inputs, free-running logits stay close, the whole graph is one split with no CPU node, teacher-forced logits track ggml-cpu, and
      fusions / CUDA-graph replay change no logit bit (a replayed decode graph reads the states the previous replay wrote)."""
import numpy as np
import pytest

from oracle import decoder
from oracle import oracle as O
from oracle import wkv as W

pytestmark = pytest.mark.gpu
PRESETS = {"rwkv6": 2, "qrwkv": 1}           # preset -> sequences decoded side by side
N_LAYER = 4
EXE = O.REF_DIR / "rwkv-graph"


@pytest.fixture(scope="module")
def plugin():
    return decoder.plugin("test-backend-ops", "rwkv-graph", "libggml_wkv_probe.so")


# ------------------------------------------------------------------ (a) the reference's test-backend-ops
@pytest.mark.parametrize("op,n_min", [("RWKV_WKV6", 4), ("GATED_LINEAR_ATTN", 4), ("SQR", 1), ("SQRT", 1)])
def test_reference_test_backend_ops(plugin, op, n_min):
    decoder.check_test_backend_ops(plugin, op, n_min)


# ------------------------------------------------------------------ (b) probe parity, device vs ggml-cpu
@pytest.mark.parametrize("gla", [False, True], ids=["wkv6", "gla"])
def test_wkv_device_is_bit_identical_to_cpu(plugin, gla):
    cases = W.grid(gla)
    for case in cases:
        srcs = case.sources()
        (y, st), (wy, wst) = W.wkv("B2000", case, srcs), W.wkv("CPU", case, srcs)
        for name, g, w in (("y", y, wy), ("states", st, wst)):
            assert np.isfinite(w).all(), (str(case), name)
            assert np.array_equal(g.view(np.uint32), w.view(np.uint32)), (str(case), name, O.nmse(g, w))
    print(f"{'GATED_LINEAR_ATTN' if gla else 'RWKV_WKV6'} B2000 vs ggml-cpu: {len(cases)} cases (S 16 / 64 / 128) bit-identical")


@pytest.mark.parametrize("gla", [False, True], ids=["wkv6", "gla"])
def test_wkv_device_tail_head_sizes(plugin, gla):
    worst = 0.0
    for case in W.tail_grid(gla):
        srcs = case.sources()
        (y, st), (wy, wst) = W.wkv("B2000", case, srcs), W.wkv("CPU", case, srcs)
        for name, g, w in (("y", y, wy), ("states", st, wst)):
            e = O.nmse(g, w)
            assert e <= 1e-12, (str(case), name, e)
            worst = max(worst, e)
    print(f"{'GATED_LINEAR_ATTN' if gla else 'RWKV_WKV6'} B2000 vs ggml-cpu, S 8 / 24: worst NMSE {worst:.2e}")


def test_sqr_sqrt_device_is_bit_identical_to_cpu(plugin):
    rng = np.random.default_rng(5)
    x = np.concatenate([rng.standard_normal(4096) * 10.0, rng.uniform(0, 1e-30, 64), [0.0, -0.0, np.inf, 1e30, 3e38, 1e-45]]).astype(np.float32)
    for op in (0, 1):
        xs = np.abs(x) if op == 1 else x
        got, want = W.sqr_sqrt("B2000", op, xs), W.sqr_sqrt("CPU", op, xs)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), ("SQR", "SQRT")[op]


def test_what_the_abi_declines_the_plugin_declines(plugin):
    assert W.wkv("B2000", W.WkvCase(257, 1, 1, 1), raw=True) == -2                       # head size above 256
    assert W.wkv("B2000", W.WkvCase(256, 1, 2, 1), raw=True) == 0
    assert W.wkv("B2000", W.WkvCase(16, 2, 2, 2, gla=True), raw=True, T=5) == -2          # T % n_seqs != 0
    assert W.wkv("B2000", W.WkvCase(16, 2, 2, 2), raw=True, T=5) == -2
    big = W.WkvCase(1, 1, 1, 65536)                                                       # more sequences than one grid holds
    assert W.wkv("B2000", big, raw=True) == -2
    assert W.wkv("CPU", big, raw=True) == 0
    assert W.wkv("B2000", W.WkvCase(1, 1, 1, 65535), raw=True) == 0


# ------------------------------------------------------------------ (c) the C ABI
def test_c_abi_error_codes():
    import ctypes as C
    import torch
    import ggml_b200 as g
    L = g.lib()
    L.ggml_b200_op_rwkv_wkv6.argtypes = [C.POINTER(g.TensorDesc)] * 7 + [C.c_void_p]
    L.ggml_b200_op_gated_linear_attn.argtypes = [C.POINTER(g.TensorDesc)] * 6 + [C.c_float, C.c_void_p]
    D = g.strided_desc
    z = lambda *shape, dt=torch.float32: torch.zeros(shape, dtype=dt, device="cuda")
    S, H, T, ns = 16, 2, 6, 2
    k, tf, s, out = z(T, H, S), z(H, S), z(ns, S * S * H), z(T + S * ns, S * H)

    def wkv6(k_=k, v=k, r=k, tf_=tf, td=k, s_=s, d=out):
        return L.ggml_b200_op_rwkv_wkv6(*[C.byref(D(t)) for t in (k_, v, r, tf_, td, s_, d)], None)

    def gla(k_=k, v=k, q=k, g_=k, s_=s, d=out):
        return L.ggml_b200_op_gated_linear_attn(*[C.byref(D(t)) for t in (k_, v, q, g_, s_, d)], 0.125, None)
    assert wkv6() == 0 and gla() == 0
    for f in (wkv6, gla):
        assert f(v=k.half()) == -1                                                        # type
        assert f(k_=z(T, H, 2 * S)[:, :, :S]) == -1                                       # k not packed
        assert f(v=z(T, H, S + 1)) == -1                                                  # v shape
        assert f(s_=z(ns, S * S * H + 1)) == -1                                           # state size
        assert f(d=z(T + S * ns - 1, S * H)) == -1                                        # dst size
    for T_, code in ((5, -2), (0, 0)):                                                    # T % n_seqs; T = 0: nothing to do
        t_ = z(T_, H, S)
        assert wkv6(k_=t_, v=t_, r=t_, td=t_, d=z(T_ + S * ns, S * H)) == code
        assert gla(k_=t_, v=t_, q=t_, g_=t_, d=z(T_ + S * ns, S * H)) == code
    assert wkv6(tf_=z(H, S + 1)) == -1                                                    # tf size
    assert wkv6(tf_=z(H, 2 * S)[:, :S]) == -1                                             # tf not packed
    torch.cuda.synchronize()


def _np_wkv(k, v, a, b, tf, s0, gla, scale):
    """a float64 model of the recurrence (the parity to the last bit is the probe's job): y [T, H, S], s [n_seqs, H, S, S]"""
    T, H, S = k.shape
    ns = s0.shape[0]
    st, y = s0.astype(np.float64).copy(), np.zeros((T, H, S))
    for t in range(T):
        q = t // (T // ns)
        kv = k[t][:, :, None].astype(np.float64) * v[t][:, None, :]                     # [H, i, j]
        if gla:
            st[q] = st[q] * b[t][:, :, None] + kv
            y[t] = np.einsum("hij,hi->hj", st[q], a[t] * scale)
        else:
            y[t] = np.einsum("hij,hi->hj", kv * tf[:, :, None] + st[q], a[t])
            st[q] = st[q] * b[t][:, :, None] + kv
    return y, st


def test_c_abi_cuda_graph_replay_matches_eager():
    import torch
    import ggml_b200 as g
    torch.cuda.set_device(0)
    S, H, ns, nt = 64, 32, 2, 3
    T = ns * nt
    k, v, r, td = (torch.zeros((T, H, S), device="cuda") for _ in range(4))
    tf, s0 = torch.zeros((H, S), device="cuda"), torch.zeros((ns, H, S, S), device="cuda")

    def step():
        y6, s6 = g.op_rwkv_wkv6(k, v, r, tf, td, s0)
        yg, sg = g.op_gated_linear_attn(k, v, r, td, s0, S ** -0.5)
        return y6, s6, yg, sg
    step()                                                                  # lazy per-device set-up outside the capture
    torch.cuda.synchronize()
    stream = torch.cuda.Stream()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=stream):
        captured = step()
    rng = np.random.default_rng(31)
    for _ in range(3):
        for t in (k, v, r, tf, s0):
            t.copy_(torch.from_numpy(rng.standard_normal(tuple(t.shape)).astype(np.float32)))
        td.copy_(torch.from_numpy(np.exp(-np.exp(rng.uniform(-8, 2, tuple(td.shape)))).astype(np.float32)))
        graph.replay()
        torch.cuda.synchronize()
        eager = step()
        torch.cuda.synchronize()
        for c, e in zip(captured, eager):
            assert torch.equal(c.view(torch.int32), e.view(torch.int32))
    host = [t.cpu().numpy() for t in (k, v, r, td, tf, s0)]
    for gla, (y, st) in ((False, eager[:2]), (True, eager[2:])):
        wy, wst = _np_wkv(host[0], host[1], host[2], host[3], host[4], host[5], gla, S ** -0.5)
        assert O.nmse(y.cpu().numpy(), wy) < 1e-10 and O.nmse(st.cpu().numpy(), wst) < 1e-10, gla


# ------------------------------------------------------------------ (d) the RWKV-6 presets
@pytest.mark.parametrize("preset", list(PRESETS))
def test_rwkv_graph_every_node_matches_cpu_on_identical_inputs(plugin, preset):
    summary, lines = decoder.compare(EXE, preset, sync=True)
    nodes = lines["node"]
    assert set(summary) == {"prompt", "decode"}, summary
    for n in nodes:
        assert float(n[-1]) <= 1e-9, n
    wkv_op = "GATED_LINEAR_ATTN" if preset == "qrwkv" else "RWKV_WKV6"
    for phase in ("prompt", "decode"):
        ops = [n[3] for n in nodes if n[1] == phase]
        assert ops.count(wkv_op) == N_LAYER, (phase, ops.count(wkv_op))
        if preset == "rwkv6":
            assert ops.count("SQR") == N_LAYER, (phase, ops.count("SQR"))
    print(f"rwkv graph [{preset}], identical inputs per node: worst NMSE prompt {summary['prompt']['worst']:.2e}, "
          f"decode {summary['decode']['worst']:.2e} over {len(nodes)} f32 nodes")


@pytest.mark.parametrize("preset", list(PRESETS))
def test_rwkv_graph_free_running_logits(plugin, preset):
    summary, _ = decoder.compare(EXE, preset, sync=False)
    assert set(summary) == {"prompt", "decode"}, summary
    for phase, s in summary.items():
        assert 0.0 <= s["logits"] <= 5e-3, (phase, s)
    print(f"rwkv graph [{preset}], free-running: " + ", ".join(f"{ph}: logits NMSE {s['logits']:.2e}" for ph, s in summary.items()))


@pytest.fixture(scope="module")
def cpu_runs(plugin, tmp_path_factory):
    d = tmp_path_factory.mktemp("rwkv_cpu")
    return {p: decoder.run(EXE, p, "CPU", d / f"{p}.logits", n) for p, n in PRESETS.items()}


@pytest.mark.parametrize("preset", list(PRESETS))
def test_rwkv_graph_runs_in_one_split_on_the_device(plugin, preset, tmp_path):
    kv, _ = decoder.run(EXE, preset, "B2000", tmp_path / "l.bin", PRESETS[preset])
    assert int(kv["n_splits"][0]) == 1 and int(kv["cpu_nodes"][0]) == 0, kv
    print(f"rwkv graph [{preset}]: one split, no CPU node, decode {kv['decode_ms_per_step'][0]} ms per step")


@pytest.mark.parametrize("preset", list(PRESETS))
def test_rwkv_graph_logits_track_cpu_step_by_step(preset, cpu_runs, tmp_path):
    ties, worst, n_same, ctoks = decoder.check_tracks_cpu(EXE, preset, cpu_runs[preset], tmp_path, PRESETS[preset])
    print(f"rwkv graph [{preset}]: {decoder.N_STEPS} teacher-forced steps x {PRESETS[preset]} sequences, worst logits NMSE {worst:.2e}, "
          f"same greedy token at {n_same}/{len(ctoks)}, near-ties {ties[:5]}")


@pytest.mark.parametrize("preset", list(PRESETS))
def test_rwkv_graph_fusions_and_graph_replay_are_bit_exact(plugin, preset, tmp_path):
    decoder.check_fusions_and_graphs_bit_exact(EXE, preset, tmp_path, PRESETS[preset])
