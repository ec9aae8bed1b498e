"""GPU: a llama-architecture decoder graph (oracle/llama_graph.cpp: Q4_K / Q6_K weights, RMS_NORM, grouped-query attention, ROPE, f16 KV
cache written by CPY into views, SwiGLU FFN, residual ADDs) on the B2000 backend, in two presets: `norm` (RoPE mode 0, attention as
MUL_MAT + SOFT_MAX_EXT) and `neox` (RoPE mode 2 over 32 of 64 dims with freq factors and YaRN, attention through FLASH_ATTN_EXT).

  (a) every node evaluated on identical inputs matches ggml-cpu to NMSE <= 1e-9 (ggml_backend_compare_graph_backend, synced), except
      FLASH_ATTN_EXT (<= 1e-6): ggml-cpu accumulates an f16 V cache in f16, the device kernel in f32;
  (b) free-running, the logits stay within 5e-3 NMSE of ggml-cpu and the first node above 1e-9 is a MUL_MAT (norm): the int8
      re-quantization of the activations in front of each quantized mat-mul (DESIGN.md §3) turns a last-bit difference into a one-code
      jump; with flash attention (neox) it is the first FLASH_ATTN_EXT, for the reason of (a);
  (c) under ggml_backend_sched over [B2000, CPU] the whole graph is one split with no node on the CPU;
  (d) teacher-forced along ggml-cpu's greedy trajectory the logits track the CPU's step by step, and every differing greedy token is a
      near-tie inside the measured noise;
  (e) the graph-level fusions and CUDA-graph replay change no logit bit."""
import subprocess

import numpy as np
import pytest

from oracle import oracle as O

pytestmark = pytest.mark.gpu
PRESETS = ["norm", "neox"]
N_STEPS = 24
N_VOCAB = 4096


@pytest.fixture(scope="module")
def exe():
    import ggml_b200
    e = O.REF_DIR / "llama-graph"
    if not e.exists():
        pytest.fail("oracle/_ref/llama-graph missing (make -C oracle -f llama.mk llama in the build container)")
    if not ggml_b200.BACKEND_SO.exists():
        pytest.fail(f"{ggml_b200.BACKEND_SO} missing")
    return e


def _run(exe, args, env_extra=None):
    import ggml_b200
    env = O.ref_env()
    env["GGML_BACKEND_PATH"] = str(ggml_b200.BACKEND_SO)
    env.update(env_extra or {})
    p = subprocess.run([str(exe), *args], env=env, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, (p.stdout + p.stderr)[-3000:]
    return p.stdout


def compare(exe, preset, sync):
    out = _run(exe, [preset, "compare", "B2000"] + (["sync"] if sync else []))
    summary = {}
    for l in out.splitlines():
        f = l.split()
        if f and f[0] == "summary":
            summary[f[1]] = dict(n_over=int(f[4]), worst=float(f[6]), first=int(f[8]), op=f[9], logits=float(f[11]))
    nodes = [l.split() for l in out.splitlines() if l.startswith("node ")]
    return summary, nodes


def run(exe, preset, dev, path, force=None, env_extra=None):
    out = _run(exe, [preset, "run", dev, str(N_STEPS), str(path)] + ([str(force)] if force else []), env_extra)
    kv = {l.split()[0]: l.split()[1:] for l in out.splitlines() if l.strip()}
    logits = np.fromfile(path, dtype=np.float32).reshape(-1, N_VOCAB)
    assert logits.shape[0] == N_STEPS
    return kv, logits


@pytest.mark.parametrize("preset", PRESETS)
def test_llama_graph_every_node_matches_cpu_on_identical_inputs(exe, preset):
    summary, nodes = compare(exe, preset, sync=True)
    assert set(summary) == {"prompt", "decode"}, summary
    # node line: node PHASE INDEX OP NAME [ne] nmse E.  FLASH_ATTN_EXT (neox preset) is the one op not held to 1e-9: ggml-cpu accumulates
    # V in f16 for an f16 cache where the device kernel accumulates in f32 (ops.cu flash_attn_ext_kernel); it is held to 1e-6
    for n in nodes:
        e = float(n[-1])
        assert e <= (1e-6 if n[3] == "FLASH_ATTN_EXT" else 1e-9), n
    assert sum(1 for n in nodes if n[3] == "FLASH_ATTN_EXT") == (2 * 4 if preset == "neox" else 0)            # 4 layers, two phases
    ropes = [n for n in nodes if n[3] == "ROPE"]
    assert len(ropes) == 2 * 2 * 4, len(ropes)                       # Q and K of 4 layers, two phases
    print(f"llama graph [{preset}], identical inputs per node: worst NMSE prompt {summary['prompt']['worst']:.2e}, "
          f"decode {summary['decode']['worst']:.2e} over {len(nodes)} compared nodes; worst ROPE {max(float(n[-1]) for n in ropes):.2e}")


@pytest.mark.parametrize("preset", PRESETS)
def test_llama_graph_free_running_deviation_starts_at_a_mul_mat(exe, preset):
    summary, _ = compare(exe, preset, sync=False)
    assert set(summary) == {"prompt", "decode"}, summary
    for phase, s in summary.items():
        assert 0.0 <= s["logits"] <= 5e-3, (phase, s)
        if s["n_over"]:
            # neox: the first node over 1e-9 is the first FLASH_ATTN_EXT (the f16 V accumulator of ggml-cpu, see the synced test)
            assert s["op"] == ("FLASH_ATTN_EXT" if preset == "neox" else "MUL_MAT"), (phase, s)
    print(f"llama graph [{preset}], free-running: " + ", ".join(
        f"{ph}: {s['n_over']} nodes over 1e-9, logits NMSE {s['logits']:.2e}, first at node {s['first']} ({s['op']})" for ph, s in summary.items()))


@pytest.fixture(scope="module")
def cpu_runs(exe, tmp_path_factory):
    d = tmp_path_factory.mktemp("llama_cpu")
    return {p: run(exe, p, "CPU", d / f"{p}.logits") for p in PRESETS}


@pytest.mark.parametrize("preset", PRESETS)
def test_llama_graph_runs_in_one_split_on_the_device(exe, preset, tmp_path):
    kv, _ = run(exe, preset, "B2000", tmp_path / "l.bin")
    assert int(kv["n_splits"][0]) == 1 and int(kv["cpu_nodes"][0]) == 0, kv


@pytest.mark.parametrize("preset", PRESETS)
def test_llama_graph_logits_track_cpu_step_by_step(exe, preset, cpu_runs, tmp_path):
    ckv, cpu_logits = cpu_runs[preset]
    ctoks = [int(t) for t in ckv["tokens"]]
    assert ctoks == [int(v) for v in cpu_logits.argmax(1)]
    force = tmp_path / "force.bin"
    np.array(ctoks, dtype=np.int32).tofile(force)
    _, gpu_logits = run(exe, preset, "B2000", tmp_path / "forced.bin", force=force)
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
    gkv, _ = run(exe, preset, "B2000", tmp_path / "free.bin")
    gtoks = [int(t) for t in gkv["tokens"]]
    first_tie = ties[0][0] if ties else N_STEPS
    assert gtoks[:first_tie] == ctoks[:first_tie], f"\ncpu: {ctoks}\ngpu: {gtoks}\nties: {ties}"
    assert n_same >= N_STEPS // 2, (n_same, ties)
    print(f"llama graph [{preset}]: {N_STEPS} teacher-forced steps, worst logits NMSE {worst:.2e}, same greedy token at {n_same}/{N_STEPS}, "
          f"near-ties {ties[:5]}, free-running prefix identical for {first_tie} tokens")


@pytest.mark.parametrize("preset", PRESETS)
def test_llama_graph_fusions_and_graph_replay_are_bit_exact(exe, preset, tmp_path):
    force = tmp_path / "force.bin"
    np.arange(100, 100 + N_STEPS, dtype=np.int32).tofile(force)
    outs = {}
    for name, env in (("default", {}), ("nofusion", {"GGML_B200_DISABLE_FUSION": "1"}), ("nographs", {"GGML_B200_DISABLE_GRAPHS": "1"})):
        _, outs[name] = run(exe, preset, "B2000", tmp_path / f"{name}.bin", force=force, env_extra=env)
    for name in ("nofusion", "nographs"):
        assert np.array_equal(outs["default"].view(np.uint32), outs[name].view(np.uint32)), (preset, name)
