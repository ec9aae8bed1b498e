"""GPU: GGML_OP_POOL_2D, GGML_OP_UPSCALE, GGML_OP_LEAKY_RELU and GGML_OP_REPEAT on the device (ops.cu pool2d_kernel, upscale_kernel,
leaky_relu_kernel, repeat_kernel behind ggml_b200_op_pool_2d / _upscale / _leaky_relu / _repeat and the plug-in), and YOLO-style
convolutional graphs that use them with ggml_conv_2d (oracle/yolo_graph.cpp, and the reference's own examples/yolo program).

  (a) the reference's own test-backend-ops runs every POOL_2D, REPEAT, UPSCALE and LEAKY_RELU case on B2000 against ggml-cpu: all executed
      and passed, none declined;
  (b) one-node graphs (oracle/pool_probe.cpp) on B2000 and on ggml-cpu are bit-identical over the host test's grid and at the YOLO shapes
      (a NaN equals any NaN: see tests/test_hostemu_pool.py); the plain f16 x f16 kernel matches ggml-cpu at the three conv shapes whose
      K (27, 144, 288) is not a multiple of 64; layouts ggml-cpu reads differently are declined;
  (c) the C ABI: invalid arguments give error codes; a captured CUDA graph of REPEAT -> POOL_2D -> UPSCALE -> LEAKY_RELU, replayed on new
      inputs, equals eager launches bit for bit;
  (d) the `tiny` and `batch2` presets: the graph's op counts; on identical inputs every POOL_2D, UPSCALE, LEAKY_RELU and REPEAT node equals
      ggml-cpu exactly and every other f32 node is within NMSE 1e-9; free-running, both heads stay within HEAD_NMSE;
  (e) `run`: one split, no CPU node, passes bitwise identical, and the same heads without fusions or without CUDA graphs;
  (f) the reference's examples/yolo program, unmodified, compiled against the plug-in: it runs on the device end to end and prints the
      layer shapes the CPU build prints."""
import ctypes as C
import subprocess

import numpy as np
import pytest

from oracle import conv as V
from oracle import decoder
from oracle import oracle as O
from oracle import pool as P

pytestmark = pytest.mark.gpu
PRESETS = ("tiny", "batch2")
EXE = O.REF_DIR / "yolo-graph"
# free-running NMSE bound of both heads against ggml-cpu: about 15 x the worst measured (1.4e-7, DESIGN.md §8), far under the reference's
# MUL_MAT gate of 5e-4
HEAD_NMSE = 2e-6


@pytest.fixture(scope="module")
def plugin():
    return decoder.plugin("test-backend-ops", "yolo-graph", "libggml_pool_probe.so", "yolov3-tiny", "yolov3-tiny-b200", "yolo/data/coco.names")


def nan_equal(got, want):
    """bit for bit, except that a NaN equals any NaN (which NaN an IEEE operation returns is the hardware's choice)"""
    u = np.uint32 if got.itemsize == 4 else np.uint16
    nan = np.isnan(got) if got.dtype.kind == "f" else np.zeros(got.shape, bool)
    wnan = np.isnan(want) if want.dtype.kind == "f" else np.zeros(want.shape, bool)
    return np.array_equal(nan, wnan) and np.array_equal(got.view(u)[~nan], want.view(u)[~nan])


# ------------------------------------------------------------------ (a) the reference's test-backend-ops
@pytest.mark.parametrize("op,n_min", [("POOL_2D", 128), ("REPEAT", 14), ("UPSCALE", 3), ("LEAKY_RELU", 1)])
def test_reference_test_backend_ops(plugin, op, n_min):
    decoder.check_test_backend_ops(plugin, op, n_min)


# ------------------------------------------------------------------ (b) probe parity, device vs ggml-cpu
YOLO_POOLS = [P.PoolCase(P.Source(P.F32, (416, 416, 16, 1), seed=200), P.POOL_MAX, 2, 2, 2, 2),
              P.PoolCase(P.Source(P.F32, (13, 13, 512, 1), seed=201), P.POOL_MAX, 2, 2, 1, 1, 0.5, 0.5),
              P.PoolCase(P.Source(P.F32, (20, 20, 256, 2), seed=202), P.POOL_MAX, 2, 2, 2, 2)]
YOLO_UPSCALES = [P.UpscaleCase(P.Source(P.F32, (13, 13, 128, 1), seed=210), (26, 26, 128, 1)),
                 P.UpscaleCase(P.Source(P.F32, (10, 10, 128, 2), seed=211), (20, 20, 128, 2))]
YOLO_REPEATS = [P.RepeatCase(P.Source(P.F32, (1, 1, 16, 1), seed=220), (416, 416, 16, 1)),
                P.RepeatCase(P.Source(P.F32, (1, 1, 255, 1), seed=221), (26, 26, 255, 2))]
YOLO_LEAKIES = [P.LeakyCase(P.Source(P.F32, (416, 416, 16, 1), seed=230), 0.1, inplace=True)]


def test_pool_2d_device_is_bit_identical_to_cpu(plugin):
    cases = P.pool_grid() + YOLO_POOLS
    for case in cases:
        parent = case.src.parent()
        got, want = P.pool_2d("B2000", case, parent), P.pool_2d("CPU", case, parent)
        assert nan_equal(got, want), str(case)
    print(f"POOL_2D B2000 vs ggml-cpu: {len(cases)} cases bit-identical")


def test_upscale_leaky_relu_repeat_device_are_bit_identical_to_cpu(plugin):
    n = 0
    for fn, cases in ((P.upscale, P.upscale_grid() + YOLO_UPSCALES), (P.leaky_relu, P.leaky_grid() + YOLO_LEAKIES),
                      (P.repeat, P.repeat_grid() + YOLO_REPEATS)):
        for case in cases:
            parent = case.src.parent()
            got, want = fn("B2000", case, parent.copy()), fn("CPU", case, parent.copy())
            assert nan_equal(got, want), str(case)
            n += 1
    print(f"UPSCALE / LEAKY_RELU / REPEAT B2000 vs ggml-cpu: {n} cases bit-identical")


def test_plain_f16_kernel_at_the_odd_k_conv_shapes(plugin):
    """the three YOLO convs whose K is not a multiple of 64 run on the plain f16 x f16 kernel; K = 27 rows are 54 bytes"""
    import ggml_b200 as g
    for i, (M, N, K) in enumerate([(4096, 16, 27), (2048, 32, 144), (1024, 64, 288), (333, 16, 27)]):
        assert g.mul_mat_f16_f16_workspace_size(M, N, K) == 0
        ops = V.f16_operands(M, N, K, 0, seed=40 + i)
        got, want = V.mul_mat_f16("B2000", M, N, K, 0, ops), V.mul_mat_f16("CPU", M, N, K, 0, ops)
        assert np.isfinite(got).all() and O.nmse(got, want) <= 1e-10, (M, N, K, O.nmse(got, want))
        assert O.nmse(got, V.mul_mat_f16_reference(*ops, 0)) <= 1e-10


def test_what_ggml_cpu_reads_differently_is_declined(plugin):
    # planes not evenly spaced (nb3 != ne2 nb2): ggml-cpu steps through the planes by nb2
    uneven = P.PoolCase(P.Source(P.F32, (9, 7, 3, 2), parent_ne=(9, 7, 4, 2)), P.POOL_MAX, 2, 2, 2, 2)
    assert P.pool_2d("B2000", uneven, raw=True) == -2
    assert P.pool_2d("B2000", P.PoolCase(P.Source(P.F32, (9, 7, 3, 2), parent_ne=(11, 8, 3, 2)), P.POOL_MAX, 2, 2, 2, 2), raw=True) == 0
    # LEAKY_RELU rows not evenly spaced: ggml-cpu walks the rows at i nb1
    uneven_rows = P.LeakyCase(P.Source(P.F32, (10, 5, 4, 1), parent_ne=(10, 6, 4, 1)), 0.1)
    assert P.leaky_relu("B2000", uneven_rows, raw=True) == -2


# ------------------------------------------------------------------ (c) the C ABI
def test_c_abi_error_codes():
    import torch
    import ggml_b200 as g
    L = g.lib()
    D = g.strided_desc
    z = lambda *shape, dt=torch.float32: torch.zeros(shape, dtype=dt, device="cuda")
    x, y = z(1, 16, 13, 13), z(1, 16, 6, 6)
    pool = lambda s, d, *p: L.ggml_b200_op_pool_2d(C.byref(D(s)), C.byref(D(d)), C.byref(g.PoolParams(*p)), None)
    assert pool(x, y, 0, 2, 2, 2, 2, 0, 0) == 0 and pool(x, y, 1, 2, 2, 2, 2, 0, 0) == 0
    assert pool(x, y, 2, 2, 2, 2, 2, 0, 0) == -2                                     # POOL_COUNT
    assert pool(x, y, 0, 0, 2, 2, 2, 0, 0) == -2 and pool(x, y, 0, 2, 2, 2, 0, 0, 0) == -2
    assert pool(x, z(1, 8, 6, 6), 0, 2, 2, 2, 2, 0, 0) == -2                          # C differs
    assert pool(x.half(), y, 0, 2, 2, 2, 2, 0, 0) == -1                               # f16 input
    assert pool(x, z(1, 16, 6, 12)[..., :6], 0, 2, 2, 2, 2, 0, 0) == -1               # dst not packed
    up = lambda s, d: L.ggml_b200_op_upscale(C.byref(D(s)), C.byref(D(d)), None)
    assert up(z(1, 128, 13, 13), z(1, 128, 26, 26)) == 0 and up(z(1, 128, 13, 13).transpose(2, 3), z(1, 128, 26, 26)) == 0
    assert up(z(1, 128, 13, 13), z(1, 128, 26, 12)) == -2 and up(z(1, 128, 13, 13).half(), z(1, 128, 26, 26).half()) == -1
    lr = lambda s, d: L.ggml_b200_op_leaky_relu(C.byref(D(s)), C.byref(D(d)), 0.1, None)
    a = z(3, 4, 5, 10)
    assert lr(a, a) == 0 and lr(a, z(3, 4, 5, 9)) == -2 and lr(a.transpose(2, 3), z(3, 4, 10, 5)) == -1
    rp = lambda s, d: L.ggml_b200_op_repeat(C.byref(D(s)), C.byref(D(d)), None)
    assert rp(z(1, 16, 1, 1), z(2, 16, 13, 13)) == 0 and rp(z(1, 16, 1, 1, dt=torch.bfloat16), z(2, 16, 13, 13, dt=torch.bfloat16)) == 0
    assert rp(z(1, 16, 1, 1), z(2, 24, 13, 13)) == -2                                 # not a whole repeat
    assert rp(z(1, 16, 1, 1), z(2, 16, 13, 13, dt=torch.float16)) == -1               # types differ
    assert rp(z(1, 16, 1, 3).transpose(2, 3), z(2, 16, 3, 13)) == -1                  # src nb0 != 4
    torch.cuda.synchronize()


def test_c_abi_cuda_graph_replay_matches_eager():
    import torch
    import ggml_b200 as g
    torch.cuda.set_device(0)
    C_, H = 64, 52
    mean = torch.zeros((1, C_, 1, 1), device="cuda")
    x = torch.zeros((2, C_, H, H), device="cuda")

    def chain():
        r = g.op_repeat(mean, (2, C_, H, H))
        s = r.add_(x)                                                          # a torch op in between, as the batch norm's SUB would be
        p = g.op_pool_2d(s, g.POOL_MAX, 2, 2, 2, 2)
        u = g.op_upscale(p, (2, C_, H, H))
        return r, p, u, g.op_leaky_relu(u, 0.1, inplace=True)
    chain()
    torch.cuda.synchronize()
    stream = torch.cuda.Stream()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=stream):
        captured = chain()
    rng = np.random.default_rng(41)
    for _ in range(3):
        mean.copy_(torch.from_numpy(rng.standard_normal((1, C_, 1, 1)).astype(np.float32)))
        x.copy_(torch.from_numpy(rng.standard_normal((2, C_, H, H)).astype(np.float32)))
        graph.replay()
        torch.cuda.synchronize()
        eager = chain()
        torch.cuda.synchronize()
        for a, b in zip(captured, eager):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32))
        want = torch.nn.functional.leaky_relu(torch.nn.functional.interpolate(torch.nn.functional.max_pool2d(mean + x, 2), scale_factor=2), 0.1)
        assert torch.equal(eager[3], want)


# ------------------------------------------------------------------ (d) the YOLO presets
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


NEW_OPS = ("POOL_2D", "UPSCALE", "LEAKY_RELU", "REPEAT")


@pytest.mark.parametrize("preset", PRESETS)
def test_yolo_graph_every_node_matches_cpu_on_identical_inputs(plugin, preset):
    summary, nodes, ops = compare_raw(preset, sync=True)
    assert ops == dict(im2col=13, pool_2d=6, upscale=1, leaky_relu=11, repeat=46, concat=1), ops
    seen, worst = {op: 0 for op in NEW_OPS}, 0.0
    for n in nodes:
        e = float(n[-1])
        if n[3] in NEW_OPS:
            assert e == 0.0, n
            seen[n[3]] += 1
            continue
        assert e <= 1e-9, n
        worst = max(worst, e)
    assert seen == dict(POOL_2D=6, UPSCALE=1, LEAKY_RELU=11, REPEAT=46), seen
    heads = {n[4]: n[-3] for n in nodes if n[4] in ("layer_15", "layer_22")}
    size, batch = {"tiny": (416, 1), "batch2": (320, 2)}[preset]
    assert heads == {"layer_15": f"[{size // 32},{size // 32},255,{batch}]", "layer_22": f"[{size // 16},{size // 16},255,{batch}]"}, heads
    print(f"yolo graph [{preset}], identical inputs per node: {sum(seen.values())} POOL_2D / UPSCALE / LEAKY_RELU / REPEAT nodes exact, "
          f"worst other node NMSE {worst:.2e} over {len(nodes)} f32 nodes")


@pytest.mark.parametrize("preset", PRESETS)
def test_yolo_graph_free_running_heads(plugin, preset):
    _, nodes, _ = compare_raw(preset, sync=False)
    heads = {n[4]: float(n[-1]) for n in nodes if n[4] in ("layer_15", "layer_22")}
    assert set(heads) == {"layer_15", "layer_22"}, heads
    for name, e in heads.items():
        assert 0.0 <= e <= HEAD_NMSE, (preset, name, e)
    print(f"yolo graph [{preset}], free-running: " + ", ".join(f"{k} NMSE {v:.2e}" for k, v in sorted(heads.items())))


# ------------------------------------------------------------------ (e) run mode
def run(preset: str, dev: str, path, env_extra=None):
    out = decoder._run(EXE, [preset, "run", dev, "3", str(path)], env_extra)
    kv = {l.split()[0]: l.split()[1:] for l in out.splitlines() if l.strip() and not l.startswith("ops")}
    return kv, np.fromfile(path, dtype=np.float32)


@pytest.mark.parametrize("preset", PRESETS)
def test_yolo_graph_runs_in_one_split_and_repeats_bit_for_bit(plugin, preset, tmp_path):
    kv, heads = run(preset, "B2000", tmp_path / "default.bin")
    assert int(kv["n_splits"][0]) == 1 and int(kv["cpu_nodes"][0]) == 0 and kv["passes_identical"] == ["1"], kv
    assert np.isfinite(heads).all()
    for name, env in (("nofusion", {"GGML_B200_DISABLE_FUSION": "1"}), ("nographs", {"GGML_B200_DISABLE_GRAPHS": "1"})):
        _, other = run(preset, "B2000", tmp_path / f"{name}.bin", env)
        assert np.array_equal(heads.view(np.uint32), other.view(np.uint32)), (preset, name)
    print(f"yolo graph [{preset}]: one split, no CPU node, {kv['ms_per_pass'][0]} ms per pass on B2000")


# ------------------------------------------------------------------ (f) the reference's examples/yolo program, unmodified
def write_ppm(path, w, h, seed):
    rng = np.random.default_rng(seed)
    img = (rng.random((h, w, 3)) * 255).astype(np.uint8)
    with open(path, "wb") as f:
        f.write(f"P6\n{w} {h}\n255\n".encode() + img.tobytes())


def test_unmodified_yolov3_tiny_runs_on_the_device(plugin, tmp_path):
    subprocess.run([str(EXE), "tiny", "write-gguf", str(tmp_path / "yolov3-tiny.gguf")], env=O.ref_env(), check=True, timeout=600)
    (tmp_path / "data").symlink_to(O.REF_DIR / "yolo" / "data")
    write_ppm(tmp_path / "input.ppm", 500, 375, seed=7)
    shapes = {}
    for name in ("yolov3-tiny", "yolov3-tiny-b200"):
        p = subprocess.run([str(O.REF_DIR / name), "-m", "yolov3-tiny.gguf", "-i", "input.ppm", "-o", f"{name}.jpg"], cwd=tmp_path, env=O.ref_env(),
                           capture_output=True, text=True, timeout=600)
        out = p.stdout + p.stderr
        assert p.returncode == 0, (name, out[-3000:])
        assert "graph_compute() failed" not in out and "GGML_ASSERT" not in out and "abort" not in out.lower(), (name, out[-3000:])
        assert (tmp_path / f"{name}.jpg").stat().st_size > 0, name
        shapes[name] = [l for l in p.stdout.splitlines() if l.startswith("Layer ") and "output shape" in l]
        if name.endswith("b200"):
            assert "using CUDA backend" in p.stderr, p.stderr[-2000:]
    assert len(shapes["yolov3-tiny"]) == 21 and shapes["yolov3-tiny-b200"] == shapes["yolov3-tiny"], shapes
    print(f"examples/yolo yolov3-tiny, unmodified, on B2000: exit 0, {len(shapes['yolov3-tiny'])} layer shapes as on ggml-cpu")
