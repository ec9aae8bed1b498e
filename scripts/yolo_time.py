"""Time the ops around the convs of YOLOv3-tiny on cuda:0, the whole synthetic network on the device against ggml-cpu, and the share of a
device pass the three convs on the plain f16 x f16 kernel take.

1. POOL_2D, UPSCALE, LEAKY_RELU and REPEAT alone, at the `tiny` preset's shapes (416 x 416 input): CUDA events around replays of a captured
   CUDA graph of the op.  Per shape it prints the time per call and the bytes the op must move (src read once, dst written once) over
   that time, against the H100 SXM's 3.35 TB/s HBM3 data-sheet figure.
2. `yolo-graph tiny run` three times each, alternating the device and ggml-cpu (8 threads): ms per pass (host clock around compute and the
   read-back of both heads).
3. The mat-muls of the three convs whose K (27, 144, 288) is not a multiple of 64, on the plain one-warp-per-output kernel
   (ggml_b200_op_mul_mat_f, f16 columns x f16 kernel), timed alone, and their sum as a share of the device's ms per pass from 2.
The card's name and power limit are read in the same run and printed first.

usage: python scripts/yolo_time.py [--iters N]"""
import argparse
import ctypes as C
import os
import subprocess
import sys
import tempfile
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import ggml_b200 as g  # noqa: E402

PEAK_GBS = 3350.0
SIZE = 416
# the tiny preset's six max pools: (input channels, input size, stride, float padding)
POOLS = [(16, 416, 2, 0.0), (32, 208, 2, 0.0), (64, 104, 2, 0.0), (128, 52, 2, 0.0), (256, 26, 2, 0.0), (512, 13, 1, 0.5)]
# the three convs on the plain kernel: (name, M = output pixels, N = output channels, K = k k in)
PLAIN = [("conv0", 416 * 416, 16, 27), ("conv1", 208 * 208, 32, 144), ("conv2", 104 * 104, 64, 288)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or "unknown (nvidia-smi gave no answer)"


def time_op(fn, iters):
    """us per call of `fn`, launched from a captured CUDA graph of `per_graph` calls (the Python wrapper's host cost is not timed)"""
    fn()
    torch.cuda.synchronize()
    per_graph = max(1, min(100, iters))
    graph, stream = torch.cuda.CUDAGraph(), torch.cuda.Stream()
    with torch.cuda.graph(graph, stream=stream):
        for _ in range(per_graph):
            fn()
    reps = max(3, iters // per_graph)
    for _ in range(2):
        graph.replay()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        graph.replay()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / (reps * per_graph)


def report(name, us, nbytes):
    gbs = nbytes / us / 1e3
    print(f"{name:44s}: {us:8.2f} us per call, {nbytes / 1e6:7.2f} MB -> {gbs:7.1f} GB/s ({100 * gbs / PEAK_GBS:5.1f}% of {PEAK_GBS:.0f})")


def kernels(iters):
    gen = torch.Generator(device="cuda").manual_seed(0)
    for c, n, s, p in POOLS:
        x = torch.randn((1, c, n, n), device="cuda", generator=gen)
        y = g.op_pool_2d(x, g.POOL_MAX, 2, 2, s, s, p, p)
        report(f"POOL_2D max k2 s{s} p{p} {n}x{n}x{c}", time_op(lambda: g.op_pool_2d(x, g.POOL_MAX, 2, 2, s, s, p, p), iters), 4 * (x.numel() + y.numel()))
    x = torch.randn((1, 128, 13, 13), device="cuda", generator=gen)
    report("UPSCALE x2 13x13x128", time_op(lambda: g.op_upscale(x, (1, 128, 26, 26)), iters), 4 * (x.numel() + 4 * x.numel()))
    x = torch.randn((1, 16, SIZE, SIZE), device="cuda", generator=gen)
    report(f"LEAKY_RELU in place {SIZE}x{SIZE}x16", time_op(lambda: g.op_leaky_relu(x, 0.1, inplace=True), iters), 8 * x.numel())
    v = torch.randn((1, 16, 1, 1), device="cuda", generator=gen)
    report(f"REPEAT [1,1,16,1] -> [{SIZE},{SIZE},16,1]", time_op(lambda: g.op_repeat(v, (1, 16, SIZE, SIZE)), iters), 4 * 16 * SIZE * SIZE)


def plain_kernel(iters):
    """us of the three plain-kernel conv mat-muls: ggml_b200_op_mul_mat_f, src0 the f16 columns [K, M], src1 the f16 kernel [K, N]"""
    L = g.lib()
    gen = torch.Generator(device="cuda").manual_seed(1)
    total = 0.0
    for name, M, N, K in PLAIN:
        cols = torch.randn((M, K), device="cuda", generator=gen).half()
        w = (torch.randn((N, K), device="cuda", generator=gen) / K ** 0.5).half()
        y = torch.empty((N, M), dtype=torch.float32, device="cuda")
        a, b, d = g.strided_desc(cols), g.strided_desc(w), g.tensor_desc(y)
        us = time_op(lambda: g.check(L.ggml_b200_op_mul_mat_f(C.byref(a), C.byref(b), C.byref(d), g._stream()), "ggml_b200_op_mul_mat_f"),
                     max(5, iters // 20))
        total += us
        print(f"plain f16 x f16 {name} M {M:6d} N {N:3d} K {K:3d}: {us:9.2f} us ({2.0 * M * N * K / us / 1e6:6.2f} TFLOP/s)")
    return total


def graphs():
    from oracle import oracle as O
    env = O.ref_env()
    env["GGML_BACKEND_PATH"] = str(g.BACKEND_SO)
    ms = {"B2000": [], "CPU": []}
    with tempfile.TemporaryDirectory() as d:
        for rep in range(3):
            for dev in ("B2000", "CPU"):
                p = subprocess.run([str(O.REF_DIR / "yolo-graph"), "tiny", "run", dev, "10" if dev == "B2000" else "3", os.path.join(d, "h.bin")],
                                   env=env, capture_output=True, text=True, timeout=900)
                kv = {l.split()[0]: l.split()[1:] for l in p.stdout.splitlines() if l.strip()}
                v = kv.get("ms_per_pass", ["failed: " + p.stderr[-200:]])[0]
                print(f"yolo-graph tiny run {rep} {dev:5s}: {v} ms per pass (n_splits {kv.get('n_splits', ['?'])[0]}, "
                      f"cpu_nodes {kv.get('cpu_nodes', ['?'])[0]})")
                try:
                    ms[dev].append(float(v))
                except ValueError:
                    pass
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=1000)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs cuda:0"
    print("card:", card())
    kernels(a.iters)
    ms = graphs()
    plain_us = plain_kernel(a.iters)
    if ms["B2000"]:
        best = min(ms["B2000"])
        print(f"the three plain-kernel conv mat-muls: {plain_us / 1e3:.3f} ms, {100 * plain_us / 1e3 / best:.1f}% of the fastest device pass "
              f"({best:.3f} ms)")


if __name__ == "__main__":
    main()
