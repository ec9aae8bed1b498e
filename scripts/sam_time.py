"""Time the ops of a Segment-Anything-style encoder and decoder on cuda:0, the synthetic SAM presets on the device against ggml-cpu, and the
share of a `vit_b` pass spent in the plain float mat-mul kernel.

1. WIN_PART, WIN_UNPART, GET_REL_POS, ADD_REL_POS and CONV_TRANSPOSE_2D alone, at the ViT-B encoder's and the mask decoder's shapes: CUDA
   events around replays of a captured CUDA graph of the op.  The data ops are given against the H100 SXM's 3.35 TB/s HBM3 data-sheet figure
   (src read once, dst written once), CONV_TRANSPOSE_2D against its 67 TFLOP/s FP32 figure (2 Cin flops per tap).
2. `sam-graph PRESET run` for small, vit_b and decoder, alternating the device and ggml-cpu (8 threads): ms per pass (host clock around
   compute and the read-back of the outputs).
3. Every MUL_MAT of the `vit_b` graph runs on the plain kernel (ggml_b200_op_mul_mat_f: f16 linears on 3-D / 4-D activations, f32 attention
   products, the f16 rel-pos tables by the queries).  Each distinct shape is timed alone with the graph's operand layout; their sum, times
   the count per pass, is given as a share of the fastest device pass from 2.
The card's name and power limit are read in the same run and printed first.

usage: python scripts/sam_time.py [--iters N]"""
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
PEAK_TFLOPS = 67.0


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
    print(f"{name:52s}: {us:9.2f} us per call, {nbytes / 1e6:8.2f} MB -> {gbs:7.1f} GB/s ({100 * gbs / PEAK_GBS:5.1f}% of {PEAK_GBS:.0f})")


def kernels(iters):
    gen = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn((64, 64, 768), device="cuda", generator=gen)
    win = g.op_win_part(x, 14)
    report("WIN_PART [768, 64, 64] w 14 -> 25 windows", time_op(lambda: g.op_win_part(x, 14), iters), 4 * (x.numel() + win.numel()))
    report("WIN_UNPART 25 windows -> [768, 64, 64]", time_op(lambda: g.op_win_unpart(win, 64, 64, 14), iters), 4 * (x.numel() + x.numel()))
    for w in (64, 14):
        t = torch.randn((2 * w - 1, 64), device="cuda", generator=gen).half()
        report(f"GET_REL_POS [64, {2 * w - 1}] -> [64, {w}, {w}]", time_op(lambda: g.op_get_rel_pos(t), iters), 2 * (t.numel() + 64 * w * w))
    for name, L, P in (("global [4096, 4096, 12]", 64, 12), ("windowed [196, 196, 300]", 14, 300)):
        a = torch.randn((P, L * L, L * L), device="cuda", generator=gen)
        pw = torch.randn((P, L, L, L), device="cuda", generator=gen)
        ph = torch.randn((P, L, L, L), device="cuda", generator=gen)
        report(f"ADD_REL_POS in place {name}", time_op(lambda: g.op_add_rel_pos(a, pw, ph, inplace=True), max(20, iters // 20)),
               4 * (2 * a.numel() + pw.numel() + ph.numel()))
        del a
    for cin, cout, n in ((256, 64, 64), (64, 32, 128)):
        k = (torch.randn((cin, cout, 2, 2), device="cuda", generator=gen) / cin ** 0.5).half()
        xi = torch.randn((cin, n, n), device="cuda", generator=gen)
        us = time_op(lambda: g.op_conv_transpose_2d(k, xi, 2), iters)
        flop = 2.0 * cin * cout * 4 * n * n
        nbytes = 4 * (xi.numel() + cout * 4 * n * n) + 2 * k.numel()
        print(f"CONV_TRANSPOSE_2D {cin}->{cout} k2 s2 on {n}x{n}{'':17s}: {us:9.2f} us per call, {flop / 1e9:6.3f} GFLOP -> "
              f"{flop / us / 1e6:6.2f} TFLOP/s ({100 * flop / us / 1e6 / PEAK_TFLOPS:5.1f}% of {PEAK_TFLOPS:.0f}); "
              f"{nbytes / us / 1e3:7.1f} GB/s ({100 * nbytes / us / 1e3 / PEAK_GBS:4.1f}% of HBM)")


def graphs():
    from oracle import oracle as O
    env = O.ref_env()
    env["GGML_BACKEND_PATH"] = str(g.BACKEND_SO)
    ms = {}
    with tempfile.TemporaryDirectory() as d:
        for preset in ("small", "vit_b", "decoder"):
            for rep in range(2):
                for dev in ("B2000", "CPU"):
                    reps = "10" if dev == "B2000" else ("1" if preset == "vit_b" else "3")
                    p = subprocess.run([str(O.REF_DIR / "sam-graph"), preset, "run", dev, reps, os.path.join(d, "o.bin")],
                                       env=env, capture_output=True, text=True, timeout=1800)
                    kv = {l.split()[0]: l.split()[1:] for l in p.stdout.splitlines() if l.strip()}
                    v = kv.get("ms_per_pass", ["failed: " + p.stderr[-200:]])[0]
                    print(f"sam-graph {preset:7s} run {rep} {dev:5s}: {v} ms per pass (n_splits {kv.get('n_splits', ['?'])[0]}, "
                          f"cpu_nodes {kv.get('cpu_nodes', ['?'])[0]})")
                    try:
                        ms.setdefault((preset, dev), []).append(float(v))
                    except ValueError:
                        pass
    return ms


# the vit_b graph's MUL_MATs (ggml order ne of src0, its type, ne of src1; every src1 f32 and contiguous) and their count per pass
WIN, GLB = 8, 4
VIT_B_MATMULS = [
    ("qkv (window)", (768, 2304), torch.float16, (768, 14, 14, 25), WIN), ("qkv (global)", (768, 2304), torch.float16, (768, 64, 64, 1), GLB),
    ("kq (window)", (64, 196, 300), torch.float32, (64, 196, 300), WIN), ("kq (global)", (64, 4096, 12), torch.float32, (64, 4096, 12), GLB),
    ("rel h/w (window)", (64, 14, 14), torch.float16, (64, 14, 14, 300), 2 * WIN),
    ("rel h/w (global)", (64, 64, 64), torch.float16, (64, 64, 64, 12), 2 * GLB),
    ("kqv (window)", (196, 64, 300), torch.float32, (196, 196, 300), WIN), ("kqv (global)", (4096, 64, 12), torch.float32, (4096, 4096, 12), GLB),
    ("proj (window)", (768, 768), torch.float16, (768, 14, 14, 25), WIN), ("proj (global)", (768, 768), torch.float16, (768, 64, 64, 1), GLB),
    ("mlp1", (768, 3072), torch.float16, (768, 64, 64, 1), WIN + GLB), ("mlp2", (3072, 768), torch.float16, (3072, 64, 64, 1), WIN + GLB),
]


def plain_kernel(iters):
    L = g.lib()
    gen = torch.Generator(device="cuda").manual_seed(1)
    total_us, total_flop = 0.0, 0.0
    for name, ne_a, ta, ne_b, count in VIT_B_MATMULS:
        ne_a = tuple(ne_a) + (1,) * (4 - len(ne_a))
        ne_b = tuple(ne_b) + (1,) * (4 - len(ne_b))
        a = (torch.randn(ne_a[::-1], device="cuda", generator=gen) / ne_a[0] ** 0.5).to(ta)
        b = torch.randn(ne_b[::-1], device="cuda", generator=gen)
        ne_d = (ne_a[1], ne_b[1], ne_b[2], ne_b[3])
        d = torch.empty(ne_d[::-1], device="cuda")
        da, db, dd = g.strided_desc(a), g.strided_desc(b), g.tensor_desc(d)
        us = time_op(lambda: g.check(L.ggml_b200_op_mul_mat_f(C.byref(da), C.byref(db), C.byref(dd), g._stream()), "ggml_b200_op_mul_mat_f"),
                     max(3, iters // 200))
        flop = 2.0 * ne_a[0] * d.numel()
        total_us += us * count
        total_flop += flop * count
        print(f"plain mul_mat_f {name:18s} x{count:2d}: {us:10.1f} us each, {flop / 1e9:7.2f} GFLOP -> {flop / us / 1e6:6.2f} TFLOP/s")
    print(f"plain mul_mat_f per vit_b pass: {total_us / 1e3:.2f} ms for {total_flop / 1e9:.0f} GFLOP")
    return total_us


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=1000)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs cuda:0"
    print("card:", card())
    kernels(a.iters)
    ms = graphs()
    plain_us = plain_kernel(a.iters)
    if ms.get(("vit_b", "B2000")):
        best = min(ms[("vit_b", "B2000")])
        print(f"vit_b: the plain-kernel mat-muls take {plain_us / 1e3:.2f} ms, {100 * plain_us / 1e3 / best:.1f}% of the fastest device pass "
              f"({best:.2f} ms)")


if __name__ == "__main__":
    main()
