"""Time the convolutional front end of Whisper on cuda:0: IM2COL (f16 columns) + the f16 x f16 MUL_MAT of ggml_conv_1d, at the four conv
shapes of the tiny and large models over 3000 mel frames, on both mat-mul routes: the tensor-core GEMM (ggml_b200_mul_mat_f16_f16, both
operands by TMA) and the plain one-warp-per-output kernel (ggml_b200_op_mul_mat_f).  CUDA events around replays of a captured CUDA graph.

Per shape and route it prints the time of IM2COL alone, of the mat-mul alone and of the pair, and the mat-mul's rate, 2 M N K FLOP over its
time, against the H100 SXM's 989 TFLOP/s dense fp16 data-sheet figure (a 700 W card; the card's name and power limit are read in the same
run and printed first).  A route the shape is not eligible for is printed as such.

--graph runs `whisper-graph PRESET run` three times per preset, alternating device and CPU, and prints each decode_ms_per_step.

usage: python scripts/conv_time.py [--graph] [--iters N]"""
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

PEAK_TFLOPS = 989.0
# (name, input channels, output channels, stride): conv_1d_ph over 3000 frames, kernel width 3, padding 1
SHAPES = [("tiny conv1", 80, 384, 1), ("tiny conv2", 384, 384, 2), ("large conv1", 128, 1280, 1), ("large conv2", 1280, 1280, 2)]
FRAMES = 3000


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or "unknown (nvidia-smi gave no answer)"


def time_op(fn, iters):
    """us per call of `fn`, launched from a captured CUDA graph of up to 20 calls (the Python wrapper's host cost is not timed)"""
    fn()
    torch.cuda.synchronize()
    per_graph = max(1, min(20, iters))
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


def plain_mul_mat(cols, w, y):
    """ggml_b200_op_mul_mat_f on f16 cols [M, K] x f16 w [N, K] -> y f32 [N, M]"""
    L = g.lib()
    L.ggml_b200_op_mul_mat_f.argtypes = [C.POINTER(g.TensorDesc)] * 3 + [C.c_void_p]
    a, b, d = g.strided_desc(cols), g.strided_desc(w), g.tensor_desc(y)
    g.check(L.ggml_b200_op_mul_mat_f(C.byref(a), C.byref(b), C.byref(d), g._stream()), "ggml_b200_op_mul_mat_f")


def kernels(iters):
    gen = torch.Generator(device="cuda").manual_seed(0)
    for name, ic, oc, s in SHAPES:
        x = torch.randn((1, ic, FRAMES), device="cuda", generator=gen)
        kernel = (torch.randn((oc, ic, 3), device="cuda", generator=gen) / (3 * ic) ** 0.5).half()
        w = kernel.reshape(oc, 3 * ic)
        cols = g.op_im2col(kernel, x, s, 1, 1)[0]                          # [OL, 3 IC] f16
        M, K, N = cols.shape[0], cols.shape[1], oc
        y = torch.empty((N, M), dtype=torch.float32, device="cuda")
        flop = 2.0 * M * N * K
        t_i2c = time_op(lambda: g.op_im2col(kernel, x, s, 1, 1), iters)
        ys = {}
        for route in ("tensor cores", "plain kernel"):
            if route == "tensor cores":
                if g.mul_mat_f16_f16_workspace_size(M, N, K) == 0:
                    print(f"{name:12s} M {M:5d} N {N:5d} K {K:5d}  {route:13s}: not eligible (K % 64 != 0)")
                    continue
                mm = lambda: g.mul_mat_f16_f16(cols, w, out=y)
            else:
                mm = lambda: plain_mul_mat(cols, w, y)
            t_mm = time_op(mm, iters if route == "tensor cores" else max(5, iters // 20))
            t_pair = time_op(lambda: (g.op_im2col(kernel, x, s, 1, 1), mm()), iters if route == "tensor cores" else max(5, iters // 20))
            ys[route] = y.clone()
            tf = flop / t_mm / 1e6
            print(f"{name:12s} M {M:5d} N {N:5d} K {K:5d}  {route:13s}: IM2COL {t_i2c:8.2f} us, MUL_MAT {t_mm:9.2f} us "
                  f"({tf:6.1f} TFLOP/s, {100 * tf / PEAK_TFLOPS:5.1f}% of {PEAK_TFLOPS:.0f}), pair {t_pair:9.2f} us")
        if len(ys) == 2:
            a, b = ys["tensor cores"].double(), ys["plain kernel"].double()
            print(f"{name:12s} the two routes' results: NMSE {float(((a - b) ** 2).sum() / (b ** 2).sum()):.2e}")


def graphs():
    from oracle import oracle as O
    env = O.ref_env()
    env["GGML_BACKEND_PATH"] = str(g.BACKEND_SO)
    with tempfile.TemporaryDirectory() as d:
        for preset in ("tiny", "large"):
            for rep in range(3):
                for dev in ("B2000", "CPU"):
                    p = subprocess.run([str(O.REF_DIR / "whisper-graph"), preset, "run", dev, "24", os.path.join(d, "l.bin")], env=env,
                                       capture_output=True, text=True, timeout=900)
                    kv = {l.split()[0]: l.split()[1:] for l in p.stdout.splitlines() if l.strip()}
                    ms = kv.get("decode_ms_per_step", ["failed: " + p.stderr[-200:]])[0]
                    print(f"whisper-graph {preset:5s} run {rep} {dev:5s}: decode {ms} ms per step")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--graph", action="store_true")
    ap.add_argument("--iters", type=int, default=400)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs cuda:0"
    print("card:", card())
    kernels(a.iters)
    if a.graph:
        graphs()


if __name__ == "__main__":
    main()
