"""GPU: GGML_OP_ARGSORT and GGML_OP_SUM_ROWS on the device (ops.cu argsort_kernel / sum_rows_kernel behind ggml_b200_op_argsort /
ggml_b200_op_sum_rows and the plug-in), and mixture-of-experts decoder graphs that use them (oracle/moe_graph.cpp).

  (a) the reference's own test-backend-ops runs every ARGSORT and SUM_ROWS case on B2000 against ggml-cpu: all executed, none declined;
  (b) one-node graphs (oracle/moe_probe.cpp) on B2000 and on ggml-cpu: ARGSORT index-identical on tie-free rows and value-identical
      with ties in ascending index elsewhere, over the host test's grid plus strided and multi-dimensional sources; SUM_ROWS within one
      f32 ulp and bit-identical where the f64 sum is exact; rows longer than 1024 and rows that are not evenly spaced are declined;
  (c) the C ABI: NaN-laden rows still give permutations, invalid arguments give error codes, a captured CUDA graph sorts the values
      set before each replay;
  (d) the `moe` (8 experts, top-2, normalised weights) and `moe60` (60 experts, top-4, shared expert) presets: every node matches
      ggml-cpu on identical inputs, free-running logits stay close and any differing top-k set is a near-tie, the whole graph is one
      split with no CPU node, teacher-forced logits track ggml-cpu, and fusions / CUDA-graph replay change no logit bit."""
import re
import subprocess

import numpy as np
import pytest

from oracle import moe as M
from oracle import oracle as O

pytestmark = pytest.mark.gpu
PRESETS = ["moe", "moe60"]
N_STEPS = 24
N_VOCAB = 4096
N_LAYER = 4
MARGIN_RMS_MULTIPLE = 10          # a differing top-k set must be a near-tie: CPU margin <= this x the router probabilities' RMS deviation


@pytest.fixture(scope="module")
def plugin():
    import ggml_b200
    if not ggml_b200.BACKEND_SO.exists():
        pytest.fail(f"{ggml_b200.BACKEND_SO} missing: run __graft_entry__.build() where the ggml headers are available")
    for f in ("test-backend-ops", "moe-graph", "libggml_moe_probe.so"):
        if not (O.REF_DIR / f).exists():
            pytest.fail(f"oracle/_ref/{f} missing (oracle/Makefile and oracle/moe.mk in the build container)")
    ref = O.Ref()
    assert ref.load_backend(ggml_b200.BACKEND_SO)
    return ggml_b200.BACKEND_SO


# ------------------------------------------------------------------ (a) the reference's test-backend-ops
@pytest.mark.parametrize("op,n_min", [("ARGSORT", 6), ("SUM_ROWS", 1)])
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
@pytest.mark.parametrize("order", [M.ASC, M.DESC], ids=["asc", "desc"])
def test_argsort_device_matches_cpu_over_the_grid(plugin, order):
    cases = M.argsort_grid(strided=True)
    for case in cases:
        parent = case.parent()
        rows = case.rows(parent)
        got = M.argsort("B2000", case, order, parent)
        want = M.argsort("CPU", case, order, parent)
        for r in range(rows.shape[0]):
            try:
                M.check_sorted_row(rows[r], got[r], order, want[r])
            except AssertionError as e:
                raise AssertionError(f"{case} order {order} row {r}: {e}") from None
    print(f"ARGSORT B2000 vs ggml-cpu: {len(cases)} cases, order {order}")


def test_argsort_declines_what_it_does_not_run(plugin):
    assert M.argsort("B2000", M.Case((1024, 2, 1, 1)), M.DESC).shape == (2, 1024)
    assert M.argsort("B2000", M.Case((1025, 2, 1, 1)), M.DESC, raw=True) == -2
    assert M.argsort("B2000", M.Case((16, 3, 2, 1), view=2), M.ASC, raw=True) == -2     # rows not evenly spaced: ggml-cpu reads i * nb01
    assert M.argsort("CPU", M.Case((1025, 2, 1, 1)), M.DESC, raw=True) == 0


def _ulps_apart(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    def ordered(x):
        i = x.view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7FFFFFFF), i)
    return np.abs(ordered(a) - ordered(b))


def test_sum_rows_device_matches_cpu(plugin):
    worst, n_exact = 0, 0
    for i, n in enumerate([1, 2, 3, 31, 32, 33, 100, 1000, 4096, 10007, 100000]):
        for view in (0, 1, 2):
            case = M.Case((n, 3, 2, 1), "tiefree", view=view, seed=i)
            rng = np.random.default_rng(i * 3 + view)
            parent = rng.standard_normal(case.parent().shape).astype(np.float32) * np.float32(10.0 ** rng.integers(-3, 4))
            got, want = M.sum_rows("B2000", case, parent), M.sum_rows("CPU", case, parent)
            d = _ulps_apart(got, want)
            assert d.max() <= 1, (str(case), int(d.max()))
            worst = max(worst, int(d.max()))
            # exact rows: multiples of 1/256 below 2^20 -- every f64 partial sum is exact, so the result must be bit-identical
            parent = (rng.integers(-(1 << 28), 1 << 28, parent.shape) / 256.0).astype(np.float32)
            got, want = M.sum_rows("B2000", case, parent), M.sum_rows("CPU", case, parent)
            assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), str(case)
            n_exact += got.size
    print(f"SUM_ROWS B2000 vs ggml-cpu: worst {worst} ulp on random rows, {n_exact} exact-sum rows bit-identical")


# ------------------------------------------------------------------ (c) the C ABI
def test_argsort_c_abi_nan_rows_are_permutations():
    import torch
    import ggml_b200 as g
    rng = np.random.default_rng(3)
    for n in (5, 60, 256, 1000):
        x = rng.standard_normal((4, n)).astype(np.float32)
        x[0, :] = np.nan
        x[1, ::3] = np.nan
        x[2, ::2] = -np.inf
        x.view(np.uint32)[3, ::5] = 0xFFFFFFFF                     # negative NaN, full payload
        for desc in (False, True):
            got = g.op_argsort(torch.from_numpy(x).cuda(), descending=desc).cpu().numpy()
            for r in range(4):
                M.check_sorted_row(x[r], got[r], M.DESC if desc else M.ASC)


def test_argsort_and_sum_rows_c_abi_error_codes():
    import ctypes as C
    import torch
    import ggml_b200 as g
    L = g.lib()
    L.ggml_b200_op_argsort.argtypes = [C.POINTER(g.TensorDesc), C.POINTER(g.TensorDesc), C.c_int32, C.c_void_p]
    L.ggml_b200_op_sum_rows.argtypes = [C.POINTER(g.TensorDesc), C.POINTER(g.TensorDesc), C.c_void_p]
    x = torch.zeros((3, 16), dtype=torch.float32, device="cuda")
    ids = torch.zeros((3, 16), dtype=torch.int32, device="cuda")

    def argsort(s, d, order=0):
        return L.ggml_b200_op_argsort(C.byref(s), C.byref(d), order, None)

    d = g.tensor_desc(ids)
    assert argsort(g.tensor_desc(x), d) == 0
    assert argsort(g.tensor_desc(x), d, 2) == -2                                                        # order neither 0 nor 1
    assert argsort(g.tensor_desc(x), d, -1) == -2
    assert argsort(g.tensor_desc(x.half()), d) == -1                                                    # src not f32
    assert argsort(g.tensor_desc(x), g.tensor_desc(x)) == -1                                            # dst not i32
    s = g.tensor_desc(x); s.nb[0] = 8; s.ne[0] = 8
    dd = g.tensor_desc(ids[:, :8].contiguous())
    assert argsort(s, dd) == -1                                                                         # nb0 != 4
    assert argsort(g.tensor_desc(x), g.tensor_desc(ids[:2].contiguous())) == -1                         # dst shape
    nc = g.tensor_desc(ids); nc.ne[0] = 8                                                               # dst rows of 8 with a stride of 16
    assert argsort(g.tensor_desc(x[:, :8].contiguous()), nc) == -1                                      # non-contiguous dst
    big = torch.zeros((1, 1025), dtype=torch.float32, device="cuda")
    assert argsort(g.tensor_desc(big), g.tensor_desc(torch.zeros((1, 1025), dtype=torch.int32, device="cuda"))) == -1   # ne0 > 1024
    with pytest.raises(g.B200Error):
        g.op_argsort(big)

    def sum_rows(s, d):
        return L.ggml_b200_op_sum_rows(C.byref(s), C.byref(d), None)

    y = torch.zeros((3, 1), dtype=torch.float32, device="cuda")
    assert sum_rows(g.tensor_desc(x), g.tensor_desc(y)) == 0
    assert sum_rows(g.tensor_desc(x.half()), g.tensor_desc(y)) == -1                                    # wrong type
    assert sum_rows(g.tensor_desc(x), g.tensor_desc(ids[:, :1].contiguous())) == -1
    s = g.tensor_desc(x); s.nb[0] = 8; s.ne[0] = 8
    assert sum_rows(s, g.tensor_desc(y)) == -1                                                          # nb0 != 4
    assert sum_rows(g.tensor_desc(x), g.tensor_desc(torch.zeros((2, 1), dtype=torch.float32, device="cuda"))) == -1   # dst shape
    torch.cuda.synchronize()


def test_argsort_c_abi_sorts_the_values_set_before_each_replay():
    import torch
    import ggml_b200 as g
    torch.cuda.set_device(0)
    x = torch.zeros((7, 60), dtype=torch.float32, device="cuda")
    g.op_argsort(x, descending=True)                                  # lazy per-device set-up outside the capture
    torch.cuda.synchronize()
    stream = torch.cuda.Stream()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=stream):
        y = g.op_argsort(x, descending=True)
        s = g.op_sum_rows(x)
    rng = np.random.default_rng(11)
    for _ in range(3):
        v = rng.standard_normal((7, 60)).astype(np.float32)
        x.copy_(torch.from_numpy(v))
        graph.replay()
        torch.cuda.synchronize()
        assert np.array_equal(y.cpu().numpy(), np.argsort(-v, axis=1, kind="stable").astype(np.int32))
        assert np.allclose(s.cpu().numpy()[:, 0], v.astype(np.float64).sum(1), rtol=1e-6, atol=1e-6)


# ------------------------------------------------------------------ (d) the mixture-of-experts presets
def _run(args, env_extra=None):
    import ggml_b200
    env = O.ref_env()
    env["GGML_BACKEND_PATH"] = str(ggml_b200.BACKEND_SO)
    env.update(env_extra or {})
    p = subprocess.run([str(O.REF_DIR / "moe-graph"), *args], env=env, capture_output=True, text=True, timeout=900)
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
    inodes = [l.split() for l in out.splitlines() if l.startswith("inode ")]
    topk = [l.split() for l in out.splitlines() if l.startswith("topk ")]
    return summary, nodes, inodes, topk


def run(preset, dev, path, force=None, env_extra=None):
    out = _run([preset, "run", dev, str(N_STEPS), str(path)] + ([str(force)] if force else []), env_extra)
    kv = {l.split()[0]: l.split()[1:] for l in out.splitlines() if l.strip()}
    logits = np.fromfile(path, dtype=np.float32).reshape(-1, N_VOCAB)
    assert logits.shape[0] == N_STEPS
    return kv, logits


@pytest.mark.parametrize("preset", PRESETS)
def test_moe_graph_every_node_matches_cpu_on_identical_inputs(plugin, preset):
    summary, nodes, inodes, _ = compare(preset, sync=True)
    assert set(summary) == {"prompt", "decode"}, summary
    for n in nodes:
        assert float(n[-1]) <= 1e-9, n
    sorts = [n for n in inodes if n[3] == "ARGSORT"]
    assert len(sorts) == 2 * N_LAYER, inodes                          # one router per layer, two phases
    for n in sorts:
        assert int(n[-1]) == 0, n
    ops = {n[3] for n in nodes}
    assert {"MUL_MAT_ID", "GET_ROWS", "SOFT_MAX"} <= ops, ops
    assert ("SUM_ROWS" in ops) == (preset == "moe"), ops
    print(f"moe graph [{preset}], identical inputs per node: worst NMSE prompt {summary['prompt']['worst']:.2e}, "
          f"decode {summary['decode']['worst']:.2e} over {len(nodes)} f32 nodes; {len(sorts)} ARGSORT nodes index-identical")


@pytest.mark.parametrize("preset", PRESETS)
def test_moe_graph_free_running_logits_and_top_k(plugin, preset):
    summary, _, inodes, topk = compare(preset, sync=False)
    assert set(summary) == {"prompt", "decode"}, summary
    for phase, s in summary.items():
        assert 0.0 <= s["logits"] <= 5e-3, (phase, s)
    for t in topk:                                                    # topk PHASE INDEX ROW margin D rms R
        margin, rms = float(t[5]), float(t[7])
        assert margin <= MARGIN_RMS_MULTIPLE * rms, f"{preset}: top-k set differs at {t[:4]} although the CPU margin {margin:.3e} exceeds " \
                                                    f"{MARGIN_RMS_MULTIPLE} x the router RMS deviation {rms:.3e}"
    print(f"moe graph [{preset}], free-running: " + ", ".join(f"{ph}: logits NMSE {s['logits']:.2e}" for ph, s in summary.items()) +
          f"; {len(topk)} router rows with a different top-k set: {[(t[1], t[2], t[3], t[5], t[7]) for t in topk[:5]]}")


@pytest.fixture(scope="module")
def cpu_runs(plugin, tmp_path_factory):
    d = tmp_path_factory.mktemp("moe_cpu")
    return {p: run(p, "CPU", d / f"{p}.logits") for p in PRESETS}


@pytest.mark.parametrize("preset", PRESETS)
def test_moe_graph_runs_in_one_split_on_the_device(plugin, preset, tmp_path):
    kv, _ = run(preset, "B2000", tmp_path / "l.bin")
    assert int(kv["n_splits"][0]) == 1 and int(kv["cpu_nodes"][0]) == 0, kv
    print(f"moe graph [{preset}]: one split, no CPU node, decode {kv['decode_ms_per_step'][0]} ms per step")


@pytest.mark.parametrize("preset", PRESETS)
def test_moe_graph_logits_track_cpu_step_by_step(preset, cpu_runs, tmp_path):
    ckv, cpu_logits = cpu_runs[preset]
    ctoks = [int(t) for t in ckv["tokens"]]
    assert ctoks == [int(v) for v in cpu_logits.argmax(1)]
    force = tmp_path / "force.bin"
    np.array(ctoks, dtype=np.int32).tofile(force)
    _, gpu_logits = run(preset, "B2000", tmp_path / "forced.bin", force=force)
    ties, worst, n_same = [], 0.0, 0
    for i in range(N_STEPS):
        c, g_ = cpu_logits[i].astype(np.float64), gpu_logits[i].astype(np.float64)
        nm = O.nmse(gpu_logits[i], cpu_logits[i])
        worst = max(worst, nm)
        assert nm <= 5e-3, (preset, i, nm)
        rms = float(np.sqrt(np.mean((g_ - c) ** 2)))
        top2 = np.sort(c)[-2:]
        margin = float(top2[1] - top2[0])
        if int(g_.argmax()) != int(c.argmax()):
            ties.append((i, margin, rms))
            assert margin <= 6 * rms, f"{preset}: step {i}: argmax differs although the CPU margin {margin:.3e} exceeds 6 x the RMS deviation {rms:.3e}"
        else:
            n_same += 1
    assert n_same >= N_STEPS // 2, (n_same, ties)
    print(f"moe graph [{preset}]: {N_STEPS} teacher-forced steps, worst logits NMSE {worst:.2e}, same greedy token at {n_same}/{N_STEPS}, "
          f"near-ties {ties[:5]}")


@pytest.mark.parametrize("preset", PRESETS)
def test_moe_graph_fusions_and_graph_replay_are_bit_exact(plugin, preset, tmp_path):
    force = tmp_path / "force.bin"
    np.arange(100, 100 + N_STEPS, dtype=np.int32).tofile(force)
    outs = {}
    for name, env in (("default", {}), ("nofusion", {"GGML_B200_DISABLE_FUSION": "1"}), ("nographs", {"GGML_B200_DISABLE_GRAPHS": "1"})):
        _, outs[name] = run(preset, "B2000", tmp_path / f"{name}.bin", force=force, env_extra=env)
    for name in ("nofusion", "nographs"):
        assert np.array_equal(outs["default"].view(np.uint32), outs[name].view(np.uint32)), (preset, name)
