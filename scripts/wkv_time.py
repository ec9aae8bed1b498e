"""Time RWKV_WKV6 and GATED_LINEAR_ATTN alone on cuda:0 (CUDA events) and, with --graph, the rwkv-graph decode step on the device against
ggml-cpu with 8 threads.

Kernel shapes: 32 heads of 64 (RWKV-6 1.6B), one token per sequence for 1 and 2 sequences (decode), and a 512-token prompt of one sequence.
Per shape it prints the time per call and the state traffic over that time: the S x S x H state of every sequence is read once and
written once per call (2 x 4 S^2 H n_seqs bytes); the r / k / v / decay rows are not counted.  The card's name and power limit are read in
the same run and printed first.

--graph runs `rwkv-graph PRESET run` three times per preset, alternating device and CPU, and prints each decode_ms_per_step.

usage: python scripts/wkv_time.py [--graph] [--iters N]"""
import argparse
import os
import subprocess
import sys
import tempfile
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import ggml_b200 as g  # noqa: E402


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


def kernels(iters):
    S, H = 64, 32
    gen = torch.Generator(device="cuda").manual_seed(0)
    for name, ns, nt in (("decode, 1 sequence", 1, 1), ("decode, 2 sequences", 2, 1), ("prompt, 512 tokens", 1, 512)):
        T = ns * nt
        k, v, r = (torch.randn((T, H, S), device="cuda", generator=gen) for _ in range(3))
        w = torch.exp(-torch.exp(torch.rand((T, H, S), device="cuda", generator=gen) * 10 - 8))
        tf, s = torch.randn((H, S), device="cuda", generator=gen), torch.randn((ns, H, S, S), device="cuda", generator=gen)
        state_bytes = 2 * 4 * S * S * H * ns
        for op, fn in (("RWKV_WKV6", lambda: g.op_rwkv_wkv6(k, v, r, tf, w, s)),
                       ("GATED_LINEAR_ATTN", lambda: g.op_gated_linear_attn(k, v, r, w, s, S ** -0.5))):
            us = time_op(fn, iters if nt == 1 else max(20, iters // 20))
            print(f"{op:18s} {name:22s} H {H} S {S}: {us:8.2f} us per call, state {state_bytes / 1e6:.2f} MB -> {state_bytes / us / 1e3:7.1f} GB/s")


def graphs():
    from oracle import oracle as O
    env = O.ref_env()
    env["GGML_BACKEND_PATH"] = str(g.BACKEND_SO)
    with tempfile.TemporaryDirectory() as d:
        for preset in ("rwkv6", "qrwkv"):
            for rep in range(3):
                for dev in ("B2000", "CPU"):
                    p = subprocess.run([str(O.REF_DIR / "rwkv-graph"), preset, "run", dev, "24", os.path.join(d, "l.bin")], env=env,
                                       capture_output=True, text=True, timeout=900)
                    kv = {l.split()[0]: l.split()[1:] for l in p.stdout.splitlines() if l.strip()}
                    ms = kv.get("decode_ms_per_step", ["failed: " + p.stderr[-200:]])[0]
                    print(f"rwkv-graph {preset:6s} run {rep} {dev:5s}: decode {ms} ms per step")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--graph", action="store_true")
    ap.add_argument("--iters", type=int, default=2000)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs cuda:0"
    print("card:", card())
    kernels(a.iters)
    if a.graph:
        graphs()


if __name__ == "__main__":
    main()
