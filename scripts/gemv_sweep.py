"""Developer sweep (not the bench contract): device-time of the mat-vec kernels over shapes.  A retuning edits a planner's constant
and times the build with this script; each line records the GGML_B200_* variables set (GGML_B200_SB_ACT_REGS=0: the shared-memory
consume path).
Usage: python scripts/gemv_sweep.py [--types q4_K,q8_0] [--n 1]"""
import argparse
import json
import os
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import ggml_b200 as g  # noqa: E402

NAMES = {v: k for k, v in g.TYPE_NAMES.items()}


IND = False


def time_mm(t, M, N, K, flags, reps=400):
    rb = g.row_size(t, K)
    nbuf = max(2, int(np.ceil(300e6 / (rb * M))))           # rotate > 2x L2 worth of weights
    gen = torch.Generator(device="cuda").manual_seed(1)
    Ws = []
    for i in range(nbuf):
        w = torch.randint(0, 256, (M * rb,), dtype=torch.uint8, device="cuda", generator=gen)
        # sane fp16 scales: clear exponent top bits of every block's d so values stay finite
        Ws.append(w)
    X = torch.rand(N * K, device="cuda") * 2 - 1
    Y = torch.empty((1, 1, N, M), device="cuda")
    Ys = [torch.empty((1, 1, N, M), device="cuda") for _ in range(nbuf)] if IND else [Y] * nbuf
    if IND and (flags & g.MM_GEMV) and not (flags & g.MM_GEMV_V1):
        flags = flags | g.MM_SRC0_STATIC | g.MM_SRC1_STATIC
    elif (flags & g.MM_GEMV) and not (flags & g.MM_GEMV_V1) and not os.environ.get("SWEEP_NO_SRC0_STATIC"):
        flags = flags | g.MM_SRC0_STATIC          # weights are graph leaves (what the backend passes)
    for i in range(nbuf):
        g.mul_mat(t, Ws[i], X, M, N, K, flags=flags, out=Ys[i])
    torch.cuda.synchronize()
    # python/ctypes launch overhead (~10 us) exceeds the kernel time: replay a CUDA graph of one sweep instead
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for i in range(nbuf):
            g.mul_mat(t, Ws[i], X, M, N, K, flags=flags, out=Ys[i])
    for _ in range(3):
        graph.replay()
    torch.cuda.synchronize()
    sweeps = max(3, reps // nbuf)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for _ in range(sweeps):
        graph.replay()
    ev1.record()
    torch.cuda.synchronize()
    us = ev0.elapsed_time(ev1) * 1000 / (sweeps * nbuf)
    return us, rb * M


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--types", default="q4_0,q8_0,q4_K,q5_K,q6_K")
    ap.add_argument("--n", default="1")
    ap.add_argument("--shapes", default="4096x4096,11008x4096,4096x11008,32000x4096")
    ap.add_argument("--generic", action="store_true")
    ap.add_argument("--v1", action="store_true")
    ap.add_argument("--independent", action="store_true", help="flag launches SRC0_STATIC|SRC1_STATIC and give each its own output")
    ap.add_argument("--both", action="store_true", help="time dependent and independent launches")
    ap.add_argument("--dp4a", action="store_true", help="force the dp4a task-dot kernel (mmvq_sb.cu) also for n >= 2")
    ap.add_argument("--mma", action="store_true", help="force the mma.sync kernel (mmvq_mma.cu) also for n = 1")
    a = ap.parse_args()
    global IND
    IND = a.independent
    if a.both:
        for IND in (False, True):
            run(a)
        return
    run(a)


def run(a):
    env = {k: v for k, v in os.environ.items() if k.startswith("GGML_B200_")}
    for tn in a.types.split(","):
        t = NAMES[tn]
        for sh in a.shapes.split(","):
            M, K = (int(v) for v in sh.split("x"))
            K = K // 256 * 256
            for n in (int(v) for v in a.n.split(",")):
                base = g.MM_GEMV | (g.MM_GEMV_DP4A if a.dp4a else 0) | (g.MM_GEMV_MMA if a.mma else 0)
                for flags in ([base] + ([g.MM_GEMV | g.MM_GEMV_V1] if a.v1 else []) + ([g.MM_GENERIC] if a.generic else [])):
                    if flags != g.MM_GENERIC and g.mul_mat_plan(t, M, n, K, flags) != g.MM_GEMV:
                        continue
                    us, wb = time_mm(t, M, n, K, flags)
                    kname = ("dp4a" if a.dp4a else "mma" if (a.mma or n > 1) else "gemv") + ("_ind" if IND else "")
                    print(json.dumps({"type": tn, "M": M, "K": K, "N": n, "kernel": {base: kname, g.MM_GEMV | g.MM_GEMV_V1: "gemv_v1"}.get(flags, "generic"),
                                      "us": round(us, 2), "GBps": round(wb / us / 1e3, 1), "env": env}), flush=True)


if __name__ == "__main__":
    main()
