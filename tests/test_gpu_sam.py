"""GPU: GGML_OP_WIN_PART, GGML_OP_WIN_UNPART, GGML_OP_GET_REL_POS, GGML_OP_ADD_REL_POS, GGML_OP_CONV_TRANSPOSE_2D, GGML_OP_SIN and GGML_OP_COS on
the device (ops.cu win_part_kernel, win_unpart_kernel, get_rel_pos_kernel, add_rel_pos_kernel, ct2d_kernel and unary_kernel behind
ggml_b200_op_* and the plug-in), and Segment-Anything-style graphs that use them (oracle/sam_graph.cpp).

  (a) the reference's own test-backend-ops runs every SIN and COS case on B2000 against ggml-cpu (one each): executed and passed, none
      declined.  It has no cases for the other five ops;
  (b) one-node graphs (oracle/sam_probe.cpp) on B2000 against ggml-cpu: WIN_PART, WIN_UNPART, GET_REL_POS and ADD_REL_POS bit-identical over
      the host test's grid and at the ViT-B shapes; CONV_TRANSPOSE_2D within NMSE 1e-10 of ggml-cpu and of an f64 reference on the
      fp16-rounded operands, at the grid and at the mask decoder's two shapes; SIN / COS within 2 ulp of the f64 value; layouts ggml-cpu reads
      differently are declined;
  (c) the C ABI: invalid arguments give error codes; a captured CUDA graph of WIN_PART -> GET_REL_POS -> ADD_REL_POS -> WIN_UNPART ->
      CONV_TRANSPOSE_2D, replayed on new inputs, equals eager launches bit for bit;
  (d) the `small`, `vit_b` and `decoder` presets node by node: the op counts; on identical inputs the four exact ops' f32 nodes equal
      ggml-cpu (NMSE 0), CONV_TRANSPOSE_2D / SIN / COS nodes are within their probe gates, every other f32 node within NMSE 1e-9 unless
      named in SYNC_EXCEPTIONS with its reason; free-running, the embedding, the masks and the IoU scores stay within OUTPUT_NMSE;
  (e) `run`: one split, no CPU node, passes bitwise identical, and the same outputs without fusions or without CUDA graphs."""
import ctypes as C

import numpy as np
import pytest

from oracle import decoder
from oracle import oracle as O
from oracle import pool as P
from oracle import sam as S

pytestmark = pytest.mark.gpu
PRESETS = ("small", "vit_b", "decoder")
EXE = O.REF_DIR / "sam-graph"
CONV_NMSE = 1e-10
SIN_COS_ULP = 2.0
# free-running NMSE bound of each preset's outputs against ggml-cpu: about 10 x the worst measured (small embd 1.7e-7, vit_b embd 3.0e-7,
# decoder masks 5.7e-9 and iou 6.5e-14; DESIGN.md §8), far under the reference's MUL_MAT gate of 5e-4
OUTPUT_NMSE = {"small": 2e-6, "vit_b": 3e-6, "decoder": 6e-8}
# sync mode: f32 nodes other than the new ops that may exceed 1e-9, with the reason
SYNC_EXCEPTIONS = {}
EXACT_OPS = ("WIN_PART", "WIN_UNPART", "ADD_REL_POS")            # GET_REL_POS is f16: compared through its MUL_MAT consumers
OP_COUNTS = {"small": dict(win_part=2, win_unpart=2, get_rel_pos=8, add_rel_pos=4, conv_transpose_2d=0, sin=0, cos=0),
             "vit_b": dict(win_part=8, win_unpart=8, get_rel_pos=24, add_rel_pos=12, conv_transpose_2d=0, sin=0, cos=0),
             "decoder": dict(win_part=0, win_unpart=0, get_rel_pos=0, add_rel_pos=0, conv_transpose_2d=2, sin=2, cos=2)}


@pytest.fixture(scope="module")
def plugin():
    return decoder.plugin("test-backend-ops", "sam-graph", "libggml_sam_probe.so")


# ------------------------------------------------------------------ (a) the reference's test-backend-ops
@pytest.mark.parametrize("op", ["SIN", "COS"])
def test_reference_test_backend_ops(plugin, op):
    decoder.check_test_backend_ops(plugin, op, 1)


# ------------------------------------------------------------------ (b) probe parity, device vs ggml-cpu
VIT_B_WINDOWS = [S.WinPartCase(P.Source(P.F32, (768, 64, 64, 1), seed=300), 14)]
VIT_B_UNPARTS = [S.WinUnpartCase(P.Source(P.F32, (768, 14, 14, 25), seed=301), 64, 64, 14)]
VIT_B_RELPOS = [S.RelPosCase(P.Source(P.F16, (64, 127), seed=302), 64), S.RelPosCase(P.Source(P.F16, (64, 27), seed=303), 14)]
# the global layer's [4096, 4096, 12] logits and the windowed layers' [196, 196, 12 x 25]
VIT_B_ADDS = [S.AddRelPosCase(64, 64, 64, 12, inplace=True, seed=40), S.AddRelPosCase(14, 14, 14, 300, inplace=True, seed=41)]
# the mask decoder's two output-upscaling conv-transposes
DECODER_CONVS = [S.ConvT2dCase(256, 64, 2, 2, 64, 64, 2, seed=50), S.ConvT2dCase(64, 32, 2, 2, 128, 128, 2, seed=51)]


def test_win_part_unpart_get_rel_pos_device_are_bit_identical_to_cpu(plugin):
    n = 0
    for fn, cases in ((S.win_part, S.win_part_grid() + VIT_B_WINDOWS), (S.win_unpart, S.win_unpart_grid() + VIT_B_UNPARTS),
                      (S.get_rel_pos, S.rel_pos_grid() + VIT_B_RELPOS)):
        for case in cases:
            parent = case.src.parent()
            got, want = fn("B2000", case, parent), fn("CPU", case, parent)
            assert np.array_equal(got, want), str(case)
            n += 1
    print(f"WIN_PART / WIN_UNPART / GET_REL_POS B2000 vs ggml-cpu: {n} cases bit-identical")


def test_add_rel_pos_device_is_bit_identical_to_cpu(plugin):
    cases = S.add_rel_pos_grid() + VIT_B_ADDS
    for case in cases:
        a, pw, ph = case.parents()
        got, want = S.add_rel_pos("B2000", case, (a, pw, ph)), S.add_rel_pos("CPU", case, (a, pw, ph))
        nan = np.isnan(want)
        assert np.array_equal(nan, np.isnan(got)) and np.array_equal(got.view(np.uint32)[~nan], want.view(np.uint32)[~nan]), str(case)
    print(f"ADD_REL_POS B2000 vs ggml-cpu: {len(cases)} cases bit-identical (a NaN of a's equals any NaN)")


def finite_nmse(got, want):
    assert np.array_equal(np.isnan(got), np.isnan(want)) and np.array_equal(np.isinf(got), np.isinf(want))
    f = np.isfinite(want)
    return O.nmse(got[f].astype(np.float64), want[f].astype(np.float64))


def test_conv_transpose_2d_device_is_within_the_gate(plugin):
    worst = 0.0
    for case in S.conv_transpose_grid() + DECODER_CONVS:
        k, x = case.parents()
        got, want = S.conv_transpose_2d("B2000", case, (k, x)), S.conv_transpose_2d("CPU", case, (k, x))
        e_cpu, e_ref = finite_nmse(got, want), finite_nmse(got[0], S.conv_transpose_2d_reference(case, k, x))
        assert e_cpu <= CONV_NMSE and e_ref <= CONV_NMSE, (str(case), e_cpu, e_ref)
        worst = max(worst, e_cpu, e_ref)
    print(f"CONV_TRANSPOSE_2D B2000: worst NMSE {worst:.2e} against ggml-cpu and the f64 reference")


def test_sin_cos_device_are_within_two_ulp(plugin):
    for case in S.sin_cos_grid() + [S.SinCosCase(P.Source(P.F32, (128, 4096), seed=7), S.SIN), S.SinCosCase(P.Source(P.F32, (128, 4096), seed=8), S.COS)]:
        x = S.sin_cos_parent(case)
        got, want = S.sin_cos("B2000", case, x), S.sin_cos("CPU", case, x)
        ref64 = (np.sin if case.op == S.SIN else np.cos)(x.astype(np.float64))
        fin = np.isfinite(ref64)
        assert np.array_equal(np.isnan(got), ~fin) and np.array_equal(np.isnan(want), ~fin)
        ulp = S.ulp_error(got[fin], ref64[fin]).max()
        assert ulp <= SIN_COS_ULP, (str(case), ulp)
        print(f"{case}: worst {ulp:.2f} ulp of the f64 value, {int((got[fin] != want[fin]).sum())} of {int(fin.sum())} differ from glibc")


def test_what_ggml_cpu_reads_differently_is_declined(plugin):
    # ggml-cpu indexes WIN_PART's src and GET_REL_POS's rows as packed, whatever the view says
    assert S.win_part("B2000", S.WinPartCase(P.Source(P.F32, (6, 9, 7, 1), parent_ne=(8, 9, 7, 1)), 4), raw=True) == -2
    assert S.get_rel_pos("B2000", S.RelPosCase(P.Source(P.F16, (6, 9), parent_ne=(8, 9)), 5), raw=True) == -2
    # ADD_REL_POS of a src0 with ne3 > 1: ggml-cpu adds to its first slice only
    assert S.add_rel_pos("B2000", S.AddRelPosCase(2, 2, 2, 3, n3=2), raw=True) == -2
    # CONV_TRANSPOSE_2D: a batch (ggml-cpu computes the first image only), kernel rows not packed
    assert S.conv_transpose_2d("B2000", S.ConvT2dCase(4, 5, 2, 2, 6, 5, 2, n=2), raw=True) == -2
    assert S.conv_transpose_2d("B2000", S.ConvT2dCase(4, 5, 2, 2, 6, 5, 2, k_parent_ne=(3, 2, 5, 4)), raw=True) == -2


# ------------------------------------------------------------------ (c) the C ABI
def test_c_abi_error_codes():
    import torch
    import ggml_b200 as g
    L = g.lib()
    D = g.strided_desc
    z = lambda *shape, dt=torch.float32: torch.zeros(shape, dtype=dt, device="cuda")
    wp = lambda s, d, npx, npy, w: L.ggml_b200_op_win_part(C.byref(D(s)), C.byref(D(d)), npx, npy, w, None)
    x = z(20, 20, 16)
    assert wp(x, z(9, 7, 7, 16), 3, 3, 7) == 0 and wp(x, z(9, 7, 7, 16), 2, 3, 7) == -2 and wp(x, z(8, 7, 7, 16), 3, 3, 7) == -2
    assert wp(x.half(), z(9, 7, 7, 16).half(), 3, 3, 7) == -1 and wp(z(20, 20, 32)[..., :16], z(9, 7, 7, 16), 3, 3, 7) == -1
    wu = lambda s, d, w: L.ggml_b200_op_win_unpart(C.byref(D(s)), C.byref(D(d)), w, None)
    assert wu(z(9, 7, 7, 16), x, 7) == 0 and wu(z(8, 7, 7, 16), x, 7) == -2 and wu(z(9, 7, 7, 16), x, 0) == -2
    gr = lambda s, d: L.ggml_b200_op_get_rel_pos(C.byref(D(s)), C.byref(D(d)), None)
    h = lambda *shape: z(*shape, dt=torch.float16)
    assert gr(h(13, 8), h(7, 7, 8)) == 0 and gr(h(12, 8), h(7, 7, 8)) == -2 and gr(z(13, 8, dt=torch.bfloat16), h(7, 7, 8)) == -1
    ar = lambda a, w, hh, d: L.ggml_b200_op_add_rel_pos(C.byref(D(a)), C.byref(D(w)), C.byref(D(hh)), C.byref(D(d)), None)
    a, p = z(2, 49, 49), z(2, 7, 7, 7)
    assert ar(a, p, p, a) == 0 and ar(a, p, z(2, 7, 7, 6), a) == -2 and ar(z(2, 2, 49, 49), p, p, z(2, 2, 49, 49)) == -1
    ct = lambda k, xx, d, s: L.ggml_b200_op_conv_transpose_2d(C.byref(D(k)), C.byref(D(xx)), C.byref(D(d)), s, None)
    k = h(16, 4, 2, 2)
    assert ct(k, z(16, 5, 6), z(4, 10, 12), 2) == 0 and ct(k, z(16, 5, 6), z(4, 10, 12), 0) == -2 and ct(k, z(16, 5, 6), z(4, 10, 11), 2) == -2
    assert ct(k.float(), z(16, 5, 6), z(4, 10, 12), 2) == -1 and ct(k, z(2, 16, 5, 6), z(2, 4, 10, 12), 2) == -1
    torch.cuda.synchronize()


def test_c_abi_cuda_graph_replay_matches_eager():
    import torch
    import ggml_b200 as g
    torch.cuda.set_device(0)
    x = torch.zeros((20, 20, 16), device="cuda")                      # [H0, W0, C]
    table = torch.zeros((13, 49), dtype=torch.float16, device="cuda")   # a rel-pos table [2w - 1, C'] for w = 7
    logits = torch.zeros((9, 49, 49), device="cuda")                  # [P = 9 windows, 7 x 7 queries, 7 x 7 keys]
    kernel = torch.zeros((16, 4, 2, 2), dtype=torch.float16, device="cuda")

    def chain():
        win = g.op_win_part(x, 7)                                       # [9, 7, 7, 16]
        rel = g.op_get_rel_pos(table)                                   # [7, 7, 49]
        pw = win[..., :7].contiguous() + rel[..., :7].float()           # torch ops in between, as the encoder's MUL_MATs would be
        ph = win[..., 7:14].contiguous()
        att = g.op_add_rel_pos(logits.clone(), pw, ph)
        back = g.op_win_unpart(win, 20, 20, 7)                          # [20, 20, 16]
        up = g.op_conv_transpose_2d(kernel, back.permute(2, 0, 1).contiguous(), 2)   # [4, 40, 40]
        return win, rel, att, back, up
    chain()
    torch.cuda.synchronize()
    stream = torch.cuda.Stream()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=stream):
        captured = chain()
    rng = np.random.default_rng(61)
    for _ in range(3):
        x.copy_(torch.from_numpy(rng.standard_normal(x.shape).astype(np.float32)))
        table.copy_(torch.from_numpy(rng.standard_normal(table.shape).astype(np.float16)))
        logits.copy_(torch.from_numpy(rng.standard_normal(logits.shape).astype(np.float32)))
        kernel.copy_(torch.from_numpy((rng.standard_normal(kernel.shape) / 4).astype(np.float16)))
        graph.replay()
        torch.cuda.synchronize()
        eager = chain()
        torch.cuda.synchronize()
        for a, b in zip(captured, eager):
            assert torch.equal(a.view(torch.int16 if a.dtype == torch.float16 else torch.int32), b.view(torch.int16 if b.dtype == torch.float16 else torch.int32))
        # torch restatements: padding + windows; the inverse; the transposed conv of the fp16-rounded input
        pad = torch.nn.functional.pad(x, (0, 0, 0, 1, 0, 1))
        assert torch.equal(eager[0], pad.reshape(3, 7, 3, 7, 16).permute(0, 2, 1, 3, 4).reshape(9, 7, 7, 16))
        assert torch.equal(eager[3], x)
        want = torch.nn.functional.conv_transpose2d(x.permute(2, 0, 1)[None].half().double(), kernel.double(), stride=2)[0]
        assert ((eager[4].double() - want) ** 2).sum() / (want ** 2).sum() < 1e-10


# ------------------------------------------------------------------ (d) the presets
def compare_raw(preset: str, sync: bool):
    """compare mode on B2000: (summary, node lines, op counts)"""
    out = decoder._run(EXE, [preset, "compare", "B2000"] + (["sync"] if sync else []))
    summary, nodes, ops = None, [], None
    for l in out.splitlines():
        f = l.split()
        if f and f[0] == "summary":
            summary = dict(n_over=int(f[4]), worst=float(f[6]))
        elif f and f[0] == "node":
            nodes.append(f)
        elif f and f[0] == "ops":
            ops = {f[i]: int(f[i + 1]) for i in range(1, len(f), 2)}
    return summary, nodes, ops


@pytest.mark.parametrize("preset", PRESETS)
def test_sam_graph_every_node_matches_cpu_on_identical_inputs(plugin, preset):
    summary, nodes, ops = compare_raw(preset, sync=True)
    assert ops == OP_COUNTS[preset], ops
    seen, worst, over = {}, {}, []
    for n in nodes:
        op, e = n[3], float(n[-1])
        seen[op] = seen.get(op, 0) + 1
        worst[op] = max(worst.get(op, 0.0), e)
        if op in EXACT_OPS:
            assert e == 0.0, n
        elif op == "CONV_TRANSPOSE_2D":
            assert e <= CONV_NMSE, n
        elif op in ("SIN", "COS"):
            assert e <= 1e-12, n                                    # 2 ulp is a relative error of 2.4e-7: an NMSE below 6e-14
        elif e > 1e-9:
            over.append(n)
    print(f"sam graph [{preset}], identical inputs per node: " + ", ".join(f"{op} x{seen[op]} worst {worst[op]:.2e}" for op in sorted(seen)))
    unexplained = [n for n in over if n[3] not in SYNC_EXCEPTIONS.get(preset, {})]
    assert not unexplained, unexplained[:10]
    assert seen.get("WIN_PART", 0) == ops["win_part"] and seen.get("ADD_REL_POS", 0) == ops["add_rel_pos"]
    assert seen.get("CONV_TRANSPOSE_2D", 0) == ops["conv_transpose_2d"] and seen.get("SIN", 0) == ops["sin"]


OUTPUTS = {"small": ("embd",), "vit_b": ("embd",), "decoder": ("masks", "iou")}


@pytest.mark.parametrize("preset", PRESETS)
def test_sam_graph_free_running_outputs(plugin, preset):
    _, nodes, _ = compare_raw(preset, sync=False)
    outs = {n[4]: float(n[-1]) for n in nodes if n[4] in OUTPUTS[preset]}
    assert set(outs) == set(OUTPUTS[preset]), outs
    print(f"sam graph [{preset}], free-running: " + ", ".join(f"{k} NMSE {v:.2e}" for k, v in sorted(outs.items())))
    for name, e in outs.items():
        assert 0.0 <= e <= OUTPUT_NMSE[preset], (preset, name, e)


# ------------------------------------------------------------------ (e) run mode
def run(preset: str, dev: str, path, env_extra=None):
    out = decoder._run(EXE, [preset, "run", dev, "3", str(path)], env_extra)
    kv = {l.split()[0]: l.split()[1:] for l in out.splitlines() if l.strip() and not l.startswith("ops")}
    return kv, np.fromfile(path, dtype=np.float32)


@pytest.mark.parametrize("preset", PRESETS)
def test_sam_graph_runs_in_one_split_and_repeats_bit_for_bit(plugin, preset, tmp_path):
    kv, outs = run(preset, "B2000", tmp_path / "default.bin")
    assert int(kv["n_splits"][0]) == 1 and int(kv["cpu_nodes"][0]) == 0 and kv["passes_identical"] == ["1"], kv
    assert np.isfinite(outs).all()
    for name, env in (("nofusion", {"GGML_B200_DISABLE_FUSION": "1"}), ("nographs", {"GGML_B200_DISABLE_GRAPHS": "1"})):
        _, other = run(preset, "B2000", tmp_path / f"{name}.bin", env)
        assert np.array_equal(outs.view(np.uint32), other.view(np.uint32)), (preset, name)
    print(f"sam graph [{preset}]: one split, no CPU node, {kv['ms_per_pass'][0]} ms per pass on B2000")
