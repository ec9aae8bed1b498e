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
import pytest

from oracle import decoder
from oracle import oracle as O

pytestmark = pytest.mark.gpu
PRESETS = ["norm", "neox"]


@pytest.fixture(scope="module")
def exe():
    decoder.require("llama-graph")
    return O.REF_DIR / "llama-graph"


@pytest.mark.parametrize("preset", PRESETS)
def test_llama_graph_every_node_matches_cpu_on_identical_inputs(exe, preset):
    summary, lines = decoder.compare(exe, preset, sync=True)
    nodes = lines["node"]
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
    summary, _ = decoder.compare(exe, preset, sync=False)
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
    return {p: decoder.run(exe, p, "CPU", d / f"{p}.logits") for p in PRESETS}


@pytest.mark.parametrize("preset", PRESETS)
def test_llama_graph_runs_in_one_split_on_the_device(exe, preset, tmp_path):
    kv, _ = decoder.run(exe, preset, "B2000", tmp_path / "l.bin")
    assert int(kv["n_splits"][0]) == 1 and int(kv["cpu_nodes"][0]) == 0, kv


@pytest.mark.parametrize("preset", PRESETS)
def test_llama_graph_logits_track_cpu_step_by_step(exe, preset, cpu_runs, tmp_path):
    ties, worst, n_same, ctoks = decoder.check_tracks_cpu(exe, preset, cpu_runs[preset], tmp_path)
    gkv, _ = decoder.run(exe, preset, "B2000", tmp_path / "free.bin")
    gtoks = [int(t) for t in gkv["tokens"]]
    first_tie = ties[0][0] if ties else decoder.N_STEPS
    assert gtoks[:first_tie] == ctoks[:first_tie], f"\ncpu: {ctoks}\ngpu: {gtoks}\nties: {ties}"
    print(f"llama graph [{preset}]: {decoder.N_STEPS} teacher-forced steps, worst logits NMSE {worst:.2e}, "
          f"same greedy token at {n_same}/{decoder.N_STEPS}, near-ties {ties[:5]}, free-running prefix identical for {first_tie} tokens")


@pytest.mark.parametrize("preset", PRESETS)
def test_llama_graph_fusions_and_graph_replay_are_bit_exact(exe, preset, tmp_path):
    decoder.check_fusions_and_graphs_bit_exact(exe, preset, tmp_path)
