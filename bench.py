#!/usr/bin/env python
"""bench.py — GGML_OP_MUL_MAT over block-quantized weights on H100 (DESIGN.md §4 and §8).

Headline workload (BASELINE.json configs[1]): Q4_K 4096 -> 11008 mat-vec, n_batch = 1 (Llama-7B FFN shape).
  sweep           NBUF = 13 distinct weight matrices (13 x 25.4 MB = 330 MB > 6 x the 50 MB L2), one mat-vec each: every mat-vec
                  streams its weights from HBM
  step            SWEEPS_PER_STEP = 512 sweeps (6656 mat-vecs, ~60 ms on an H100 at 400 W) so that --steps 20 times >= 0.5 s and the clock
                  sampler sees the load; launched as CUDA-graph replays of 8 sweeps
  value           GB/s of quantized weight bytes processed, whole job (all ranks), inputs resident in HBM, CUDA events, max over ranks
  parity          AFTER the timed region a row sample of every timed output is compared with the CPU oracle (NMSE <= 1e-10 for the
                  integer mat-vec paths, <= 2e-5 against the f64 product for the fp16 tensor-core path); the run FAILS above it
  e2e             the same metric through the reference-facing plug-in with HOST buffers: the reference's own graph / backend API
                  (ggml_backend_tensor_set_async -> graph_compute -> tensor_get_async per output -> synchronize) driving
                  libggml-b200.so, exactly the calls the reference arm is timed through; N > 1: through the C ABI with the NVLink
                  exchange and the host copies inside the timed region
  roofline        algorithmic bytes (weights + x + y) / mean device time per launch vs the measured HBM peak
  extra           every other BASELINE configuration, each with its own parity and roofline: configs[0] Q4_0 4096^2 n=1; the dependent
                  chain; configs[2] Q8_0 4096^2 x 512 on the wgmma GEMM (TFLOP/s vs the measured sustained bf16 peak); Q4_K / Q8_0
                  4096 -> 32000 at n = 1 and 512; configs[3] gpt-2 117M Q4_0 tok/s through the unmodified examples/gpt-2 program;
                  configs[4] Q4_K 8192 x 28672 row-sharded (strong scaling) over the N GPUs with the fused NVLink gather
  cpu_baseline    the unmodified reference's ggml-cpu backend (oracle/_ref) on this box's host cores, same shape
  --impl reference  the reference arm: ggml-cpu via its own public API, same metric/config
N > 1: weak scaling — every rank owns one row-shard (M rows) of an (N*M) x K matrix; the mat-vec kernel itself stores its rows into every
peer's gathered y over NVLink (the path's only exchange step, SURVEY.md §8e).
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import math
import os
import re
import statistics
import subprocess
import sys
import threading
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent
sys.path.insert(0, str(ROOT))

WL = {"type": "q4_K", "type_id": 12, "K": 4096, "M": 11008, "N": 1}
METRIC = "mul_mat_q4_K_4096x11008_n1_weight_throughput"
UNIT = "GB/s"
NBUF = 13                # distinct weight matrices per sweep: 13 x 25.4 MB = 330 MB > 6 x the 50 MB L2 (and > the host's last-level cache)
SWEEPS_PER_STEP = 512    # one step = 512 sweeps = 6656 mat-vecs (~62 ms on one H100 at a 400 W power limit)
SWEEPS_PER_GRAPH = 8
CONFIG = {"workload": f"q4_K {WL['K']}x{WL['M']} mat-vec n_batch=1 (BASELINE.json configs[1])", "mat_vecs_per_step": NBUF * SWEEPS_PER_STEP,
          "l2_policy": f"inputs larger than L2: {NBUF} distinct weight matrices (330 MB) visited round-robin"}
DTYPE = "int8 x int4 (q4_K weights x q8_K activations, dp4a), f32 accumulate"

BLOCK = {2: (32, 18), 8: (32, 34), 12: (256, 144), 13: (256, 176), 14: (256, 210)}     # ggml_type -> (weights per block, bytes per block)
TNAME = {2: "q4_0", 8: "q8_0", 12: "q4_K", 13: "q5_K", 14: "q6_K"}


def row_bytes(t, K):
    qk, ts = BLOCK[t]
    return K // qk * ts


def weight_bytes(K, M, t=12):
    return row_bytes(t, K) * M


def algorithmic_bytes(K, M, N, t=12):
    return weight_bytes(K, M, t) + K * N * 4 + M * N * 4


def measured_peaks():
    p = ROOT / "MEASURED_PEAKS.json"
    if p.exists():
        try:
            d = json.loads(p.read_text())
            return {"hbm": float(d["hbm_gbs"]), "tc": float(d.get("bf16_tflops_sustained", d.get("bf16_tflops", 1400.0))), "tc_burst": float(d.get("bf16_tflops", 1590.0)),
                    "src": "measured (MEASURED_PEAKS.json: hbm_gbs, bf16_tflops_sustained)"}
        except Exception:
            pass
    return {"hbm": 6650.0, "tc": 1400.0, "tc_burst": 1590.0, "src": "fallback (B200_PROFILING.md: 6.65 TB/s, 1.4 / 1.59 PFLOP/s bf16)"}


class ClockSampler:
    """nvidia-smi clocks / throttle reasons DURING the timed region."""

    Q = "clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap"

    def __init__(self, index: int):
        self.index = index
        self.rows = []
        self.proc = None

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.index), f"--query-gpu={self.Q}", "--format=csv,noheader,nounits", "-lms", "50"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.thread = threading.Thread(target=self._read, daemon=True)
            self.thread.start()
            time.sleep(0.25)            # nvidia-smi needs a moment before its first sample
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append((time.perf_counter(), line.strip()))

    def mark(self):
        return time.perf_counter()

    def stop(self, t0=None, t1=None):
        if not self.proc:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"], "samples": 0}
        time.sleep(0.1)
        self.proc.terminate()
        try:
            self.proc.wait(timeout=2)
        except Exception:
            self.proc.kill()
        sm, mx, pw, reasons = [], [], [], set()
        for ts, r in self.rows:
            if t0 is not None and not (t0 <= ts <= t1 + 0.06):
                continue
            f = [x.strip() for x in r.split(",")]
            if len(f) < 7:
                continue
            try:
                sm.append(float(f[0])); mx.append(float(f[1])); pw.append(float(f[2]))
            except ValueError:
                continue
            for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), f[3:7]):
                if v.lower().startswith("active"):
                    reasons.add(name)
        return {"sm_mhz": statistics.median(sm) if sm else None, "sm_max_mhz": max(mx) if mx else None, "power_w_max": max(pw) if pw else None,
                "reasons": sorted(reasons), "samples": len(sm)}


def make_weights(torch, t, nbuf, K, M, seed):
    """nbuf distinct packed matrices of ggml type t: arbitrary code bytes, finite small fp16 scales per block."""
    qk, ts = BLOCK[t]
    nb = M * (K // qk)
    gen = torch.Generator(device="cuda").manual_seed(seed)
    out = []
    for _ in range(nbuf):
        w = torch.randint(0, 256, (nb, ts), dtype=torch.uint8, device="cuda", generator=gen)
        if t in (12, 13):          # d, dmin
            d = (torch.rand((nb, 2), device="cuda", generator=gen) * 2e-3 + 1e-4).to(torch.float16).view(torch.uint8)
            w[:, 0:4] = d.reshape(-1, 4)
        elif t == 14:              # d at byte 208
            d = (torch.rand((nb, 1), device="cuda", generator=gen) * 2e-3 + 1e-4).to(torch.float16).view(torch.uint8)
            w[:, 208:210] = d.reshape(-1, 2)
        else:                      # Q4_0 / Q8_0: d at byte 0
            d = ((torch.rand((nb, 1), device="cuda", generator=gen) - 0.5) * 4e-2).to(torch.float16).view(torch.uint8)
            w[:, 0:2] = d.reshape(-1, 2)
        out.append(w.reshape(-1))
    return out


_oracle = None


def oracle():
    global _oracle
    if _oracle is None:
        from oracle import oracle as O           # the checker: never the thing measured
        _oracle = (O, O.Oracle())
    return _oracle


def parity_rows(t, Wdev, Xhost, Ydev_NM, M, N, K, nrows=48, seed=1, f64=False):
    """NMSE of a row sample of a device result Y[N, M] against the CPU oracle on the same packed rows."""
    O, orc = oracle()
    rb = row_bytes(t, K)
    rows = np.sort(np.random.default_rng(seed).choice(M, min(M, nrows), replace=False))
    Wv = Wdev.view(M, rb)
    import torch
    idx = torch.from_numpy(rows).cuda()
    Wsub = Wv.index_select(0, idx).cpu().numpy().reshape(-1)
    got = Ydev_NM.reshape(N, M).index_select(1, idx).cpu().numpy()
    want = orc.mul_mat(t, Wsub, Xhost, len(rows), N, K, f64=f64)
    assert np.isfinite(got).all(), "non-finite output"
    return float(O.nmse(got, want))


# ---------------------------------------------------------------------------------------------------------------- CPU legs (children)
def cpu_baseline(sample_s=12.0):
    """The reference's ggml-cpu MUL_MAT on the host cores (oracle/_ref), bounded sample of the same workload."""
    from oracle import oracle as O
    ref = O.Ref()
    K, M, N, t = WL["K"], WL["M"], WL["N"], WL["type_id"]
    rng = np.random.default_rng(1234)
    W = O.random_blocks(t, M * K // 256, rng)
    X = np.random.default_rng(5678).uniform(-1, 1, K * N).astype(np.float32)
    best = None
    hw = ref.hw_threads()
    nw = NBUF                                   # same sweep as the GPU arm: 13 distinct matrices (330 MB), larger than the host's LLC
    for threads in sorted({hw, max(1, hw // 2), max(1, hw // 4)}, reverse=True):
        _, s = ref.mul_mat_sweep(t, W, X, M, N, K, nw, threads=threads, iters=2, warmup=1)          # probe
        iters = max(1, int(sample_s / 3 / max(s * nw, 1e-6)))
        _, s = ref.mul_mat_sweep(t, W, X, M, N, K, nw, threads=threads, iters=iters, warmup=1)
        if best is None or s < best[0]:
            best = (s, threads, iters * nw)
    s, threads, n = best
    return {"value": weight_bytes(K, M) / s / 1e9, "unit": UNIT, "cores": threads, "kind": "reference",
            "sample": f"{n} MUL_MAT nodes (q4_K {K}x{M}, n=1; {nw} distinct weight tensors per graph = 330 MB sweep, persistent threadpool), "
                      f"ggml-cpu {'native' if ref.native else 'x86-64-v3'} build, {s * 1e6:.1f} us per mat-vec",
            "us_per_matvec": s * 1e6}


def plugin_e2e_child():
    """e2e through the plug-in: the reference's graph/backend API (oracle/_ref: ggml-base + registry, unmodified) loads libggml-b200.so
    and runs the 13-matrix sweep with host buffers; returns seconds per mat-vec for the synchronous and the asynchronous public calls,
    and the NMSE of the device result against the CPU oracle."""
    from oracle import oracle as O
    import ggml_b200 as g
    ref = O.Ref()
    assert ref.load_backend(g.BACKEND_SO), "libggml-b200.so did not load as a ggml backend"
    devs = ref.devices()
    dev = [d for d in devs if d.startswith("B200")][0]
    K, M, N, t = WL["K"], WL["M"], WL["N"], WL["type_id"]
    W = O.random_blocks(t, M * K // 256, np.random.default_rng(1234))
    X = np.random.default_rng(5678).uniform(-1, 1, K * N).astype(np.float32)
    out = {"device": dev}
    for name, mode in (("sync", 1), ("async", 2)):
        Y, _ = ref.mul_mat_sweep(t, W, X, M, N, K, NBUF, dev=dev, iters=20, warmup=5, e2e=mode)
        iters = 1500
        Y, s = ref.mul_mat_sweep(t, W, X, M, N, K, NBUF, dev=dev, iters=iters, warmup=20, e2e=mode)
        rows = np.random.default_rng(3).choice(M, 64, replace=False)
        rb = ref.row_size(t, K)
        Wsub = np.concatenate([W[r * rb:(r + 1) * rb] for r in rows])
        want = O.Oracle().mul_mat(t, Wsub, X, len(rows), N, K)
        out[name] = {"s_per_matvec": s, "iters": iters, "parity_nmse": float(O.nmse(Y[:, rows], want))}
    Y, s = ref.mul_mat_sweep(t, W, X, M, N, K, NBUF, dev=dev, iters=2000, warmup=20, e2e=0)
    out["resident"] = {"s_per_matvec": s}
    print(json.dumps(out), flush=True)


def gpt2_child():
    """configs[3]: the reference's examples/gpt-2 (main-backend.cpp, unmodified, -DGGML_USE_CUDA, linked against libggml-b200.so) on a
    synthetic GPT-2 117M quantized to Q4_0 by the reference's own gpt-2-quantize; ms per generated token, and ggml-cpu beside it."""
    from oracle import oracle as O
    tmp = Path("/tmp/ggml_b200_gpt2_v2")
    tmp.mkdir(exist_ok=True)
    f16, q40 = tmp / "gpt2_f16.bin", tmp / "gpt2_q4_0.bin"
    if not q40.exists():
        subprocess.run([sys.executable, str(ROOT / "scripts" / "make_gpt2_synth.py"), str(f16)], check=True, capture_output=True)
        subprocess.run([str(O.REF_DIR / "gpt-2-quantize"), str(f16), str(q40), "2"], check=True, env=O.ref_env(), capture_output=True)
        f16.unlink(missing_ok=True)

    def run(exe, n, extra=()):
        cmd = [str(O.REF_DIR / exe), "-m", str(q40), "-s", "1234", "-n", str(n), "-t", str(min(16, os.cpu_count() or 8)), "--ignore-eos", "--top_k", "1", "-p", "a b c", *extra]
        p = subprocess.run(cmd, env=O.ref_env(), capture_output=True, text=True, timeout=150)
        o = p.stdout + p.stderr
        m = re.search(r"predict time =\s*([\d.]+) ms /\s*([\d.]+) ms per token", o)
        toks = re.findall(r"<(\d+)>", "".join(l for l in p.stdout.splitlines() if l.startswith("a b c")))
        return (float(m.group(2)) if m else None), toks, p.returncode
    gms, gtok, grc = run("gpt-2-backend-b200", 128, ("-ngl", "12"))
    cms, ctok, crc = run("gpt-2-backend", 32)
    same = 0
    for a, b in zip(gtok, ctok):
        if a != b:
            break
        same += 1
    print(json.dumps({"b200_ms_per_token": gms, "b200_tok_s": (1e3 / gms if gms else None), "b200_rc": grc, "cpu_ms_per_token": cms, "cpu_tok_s": (1e3 / cms if cms else None),
                      "cpu_threads": min(16, os.cpu_count() or 8), "greedy_prefix_identical": same, "tokens_compared": min(len(gtok), len(ctok)),
                      "program": "oracle/_ref/gpt-2-backend-b200 = examples/gpt-2/main-backend.cpp unmodified, -ngl 12, CUDA-graph replay; 128 generated tokens",
                      "model": "GPT-2 117M, synthetic N(0, 0.02^2) weights, Q4_0 via the reference's gpt-2-quantize"}), flush=True)


def run_child(flag, timeout):
    try:
        r = subprocess.run([sys.executable, str(ROOT / "bench.py"), flag], capture_output=True, text=True, timeout=timeout)
        return json.loads(r.stdout.strip().splitlines()[-1])
    except Exception as e:
        return {"failed": f"{type(e).__name__}: {e}"[:300]}


def run_reference_arm(args):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    K, M, N = WL["K"], WL["M"], WL["N"]
    from oracle import oracle as O
    ref = O.Ref()
    t = WL["type_id"]
    rng = np.random.default_rng(1234)
    W = O.random_blocks(t, M * K // 256, rng)
    X = np.random.default_rng(5678).uniform(-1, 1, K * N).astype(np.float32)
    # the reference's threadpool is used with the thread count that serves it best on this box (all hardware threads, or one per
    # physical core: oversubscribing the SMT siblings of a 2-socket host slows ggml-cpu's spin barriers down by several x)
    hw = ref.hw_threads()
    best_s, threads = None, hw
    nbuf = NBUF
    for th in sorted({hw, max(1, hw // 2), max(1, hw // 4)}, reverse=True):
        _, sp = ref.mul_mat_sweep(t, W, X, M, N, K, nbuf, threads=th, iters=3, warmup=1)
        if best_s is None or sp < best_s:
            best_s, threads = sp, th
    # One step of this arm is a BOUNDED SAMPLE of the GPU arm's step: the same sweep of NBUF mat-vecs over NBUF distinct weight tensors
    # (330 MB > the host's last-level cache), `sweeps` of them per step, sized so that steps + warmup end within ~100 s on this box
    # (the GPU arm's 512 sweeps per step would take minutes per step here).  The metric is a rate, so the sample size does not bias it.
    steps = args.steps
    budget = 100.0
    sweeps = int(max(1, min(SWEEPS_PER_STEP, budget / ((steps + args.warmup) * best_s * nbuf))))
    iters = steps * sweeps
    _, s = ref.mul_mat_sweep(t, W, X, M, N, K, nbuf, threads=threads, iters=iters, warmup=args.warmup * sweeps, e2e=2)
    val = weight_bytes(K, M) / s / 1e9
    line = {"impl": "reference", "metric": METRIC, "value": val, "unit": UNIT, "n_gpus": args.gpus, "steps": steps, "warmup": args.warmup,
            "ms_per_step": s * nbuf * sweeps * 1e3, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": DTYPE,
            "data": "synthetic", "config": dict(CONFIG),
            "sample": f"{sweeps} sweeps of {nbuf} mat-vecs per step (bounded sample of the {SWEEPS_PER_STEP}-sweep step)",
            "cpu_baseline": {"value": val, "unit": UNIT, "cores": threads, "kind": "reference",
                             "sample": f"{iters * nbuf} mat-vecs ({nbuf} distinct weight tensors per graph) through ggml_backend_tensor_set_async / graph_compute_async / "
                                       f"tensor_get_async / synchronize on ggml-cpu ({'native' if ref.native else 'x86-64-v3'} build), host copies included"},
            "e2e": {"value": val, "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
    print(json.dumps(line), flush=True)


# ---------------------------------------------------------------------------------------------------------------- GPU arm helpers
class Timer:
    def __init__(self, torch, dist=None):
        self.torch = torch
        self.dist = dist            # multi-rank: every rank must replay the same number of times (the graphs contain an exchange)

    def time_graph(self, fn_capture, min_seconds=0.2, warmup=3, max_replays=20000):
        """capture fn_capture() in a CUDA graph, replay it until >= min_seconds of device time; returns (seconds per replay, replays)"""
        torch = self.torch
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            fn_capture()
        for _ in range(warmup):
            g.replay()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); g.replay(); e1.record(); torch.cuda.synchronize()
        one = max(e0.elapsed_time(e1) * 1e-3, 1e-6)
        if self.dist is not None:
            tt = torch.tensor([one], device="cuda")
            self.dist.all_reduce(tt, op=self.dist.ReduceOp.MAX)
            one = float(tt.item())
        reps = int(min(max_replays, max(5, math.ceil(min_seconds / one))))
        e0.record()
        for _ in range(reps):
            g.replay()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1e-3 / reps, reps


def extra_matvec(torch, g, timer, t, M, K, peaks, dependent_too=True, nbuf=None, seed=7):
    """n = 1 mat-vec of another BASELINE shape: independent sweep (+ dependent chain), parity on the timed outputs, HBM roofline"""
    wb = weight_bytes(K, M, t)
    nbuf = nbuf or max(3, math.ceil(300e6 / wb))
    Ws = make_weights(torch, t, nbuf, K, M, seed)
    X = torch.rand(K, device="cuda", generator=torch.Generator(device="cuda").manual_seed(5678)) * 2 - 1
    Ys = [torch.empty((1, 1, 1, M), dtype=torch.float32, device="cuda") for _ in range(nbuf)]
    Yd = torch.empty((1, 1, 1, M), dtype=torch.float32, device="cuda")
    assert g.mul_mat_plan(t, M, 1, K) == g.MM_GEMV
    F_IND, F_DEP = g.MM_SRC0_STATIC | g.MM_SRC1_STATIC, g.MM_SRC0_STATIC

    def ind():
        for i in range(nbuf):
            g.mul_mat(t, Ws[i], X, M, 1, K, out=Ys[i], flags=F_IND)

    def dep():
        for i in range(nbuf):
            g.mul_mat(t, Ws[i], X, M, 1, K, out=Yd, flags=F_DEP)
    ind(); dep(); torch.cuda.synchronize()
    s, reps = timer.time_graph(ind)
    us = s / nbuf * 1e6
    Xh = X.cpu().numpy()
    nm = max(parity_rows(t, Ws[i], Xh, Ys[i], M, 1, K, seed=i) for i in range(nbuf))
    ab = algorithmic_bytes(K, M, 1, t)
    r = {"shape": f"{TNAME[t]} {K}x{M} n=1", "us_per_matvec": us, "GBps": wb / us / 1e3, "distinct_matrices": nbuf, "parity_nmse": nm,
         "roofline": {"bound": "hbm", "achieved": ab / us / 1e3, "peak": peaks["hbm"], "unit": "GB/s", "frac": ab / us / 1e3 / peaks["hbm"]}}
    assert nm <= 1e-10, f"parity failure {r['shape']}: NMSE {nm}"
    if dependent_too:
        s, _ = timer.time_graph(dep)
        usd = s / nbuf * 1e6
        nmd = parity_rows(t, Ws[nbuf - 1], Xh, Yd, M, 1, K, seed=99)
        assert nmd <= 1e-10, f"parity failure {r['shape']} (dependent): NMSE {nmd}"
        r["dependent_chain"] = {"us_per_matvec": usd, "GBps": wb / usd / 1e3, "parity_nmse": nmd,
                                "roofline": {"bound": "hbm", "achieved": ab / usd / 1e3, "peak": peaks["hbm"], "unit": "GB/s", "frac": ab / usd / 1e3 / peaks["hbm"]}}
    return r


def extra_gemm(torch, g, timer, t, M, N, K, peaks, seed=11):
    """batched mat-mul on the tensor-core (wgmma) path: TFLOP/s over distinct weight matrices, parity against the f64 product on sampled rows"""
    wb = weight_bytes(K, M, t)
    nbuf = max(2, math.ceil(260e6 / wb))
    Ws = make_weights(torch, t, nbuf, K, M, seed)
    X = torch.rand(N * K, device="cuda", generator=torch.Generator(device="cuda").manual_seed(5678)) * 2 - 1
    Ys = [torch.empty((1, 1, N, M), dtype=torch.float32, device="cuda") for _ in range(nbuf)]
    assert g.mul_mat_plan(t, M, N, K) == g.MM_GEMM, "batched shape must run on the tensor-core GEMM kernel"
    F = g.MM_SRC0_STATIC | g.MM_SRC1_STATIC

    def sweep():
        for i in range(nbuf):
            g.mul_mat(t, Ws[i], X, M, N, K, out=Ys[i], flags=F)
    sweep(); torch.cuda.synchronize()
    s, reps = timer.time_graph(sweep)
    us = s / nbuf * 1e6
    flops = 2.0 * M * N * K
    Xh = X.cpu().numpy()
    nm = max(parity_rows(t, Ws[i], Xh, Ys[i], M, N, K, nrows=24, seed=i, f64=True) for i in range(nbuf))
    assert nm <= 2e-5, f"parity failure gemm {TNAME[t]} {M}x{N}x{K}: NMSE {nm}"
    tf = flops / us / 1e6
    return {"shape": f"{TNAME[t]} {K}x{M} n_batch={N}", "us_per_mul_mat": us, "TFLOPs": tf, "weight_GBps": wb / us / 1e3, "distinct_matrices": nbuf,
            "includes": "activation f32->f16 conversion + GEMM kernel (everything ggml_b200_mul_mat launches)", "parity_nmse_vs_f64": nm,
            "roofline": {"bound": "tensor", "achieved": tf, "peak": peaks["tc"], "unit": "TFLOP/s", "frac": tf / peaks["tc"], "peak_burst": peaks["tc_burst"]}}


# ---------------------------------------------------------------------------------------------------------------- main
def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-extra", action="store_true", help="headline only (skips the other BASELINE configurations)")
    ap.add_argument("--no-graph", action="store_true", help="plain stream launches instead of CUDA-graph replay")
    ap.add_argument("--sweeps-per-step", type=int, default=SWEEPS_PER_STEP, help="profiling aid (ncu): fewer sweeps per step than the contract's 512")
    ap.add_argument("--exchange", default="fused", choices=["fused", "nccl"],
                    help="N > 1: 'fused' = the mat-vec kernel stores its rows into every peer's y over NVLink and signals flags; "
                         "'nccl' = ncclAllGather of the slices after the kernel (the baseline)")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write the outputs of the last step (y_<i>.npy, float32, one per weight matrix; with --exchange nccl only the last matrix's gathered y) to DIR")
    ap.add_argument("--cpu-baseline-child", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--plugin-e2e-child", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--gpt2-child", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.cpu_baseline_child:
        print(json.dumps(cpu_baseline()), flush=True)
        return
    if args.plugin_e2e_child:
        return plugin_e2e_child()
    if args.gpt2_child:
        return gpt2_child()
    if args.warmup < 3:
        args.warmup = 3
    globals()["SWEEPS_PER_STEP"] = max(SWEEPS_PER_GRAPH, args.sweeps_per_step // SWEEPS_PER_GRAPH * SWEEPS_PER_GRAPH)
    CONFIG["mat_vecs_per_step"] = NBUF * SWEEPS_PER_STEP
    if args.impl == "reference":
        return run_reference_arm(args)

    import torch
    import ggml_b200 as g
    g.lib()                                    # fail loudly if the CUDA library is missing

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dist = None
    if world > 1:
        import torch.distributed as dist_
        dist = dist_
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    peaks = measured_peaks()
    timer = Timer(torch, dist)

    K, M, N, t = WL["K"], WL["M"], WL["N"], WL["type_id"]
    wb = weight_bytes(K, M)
    nbuf = NBUF
    Ws = make_weights(torch, t, nbuf, K, M, seed=1234 + rank)
    X = torch.rand(N * K, device="cuda", generator=torch.Generator(device="cuda").manual_seed(5678)) * 2 - 1
    Xh = X.cpu().numpy()
    Yloc = torch.empty((1, 1, N, M), dtype=torch.float32, device="cuda")
    Yall = torch.empty((world, N * M), dtype=torch.float32, device="cuda") if world > 1 else None
    assert g.mul_mat_plan(t, M, N, K) == g.MM_GEMV, "headline workload must run on the TMA mat-vec kernel"

    fused = world > 1 and args.exchange == "fused"
    use_graph = (world == 1 or fused) and not args.no_graph
    ex = None
    # Like the reference's own perf harness (tests/test-backend-ops.cpp eval_perf, :657-660: the op node repeated in one graph on the same
    # inputs, one output tensor per node) the mat-vecs of a sweep are INDEPENDENT: fixed activation vector, one output buffer per weight
    # matrix, all final before the timed region -> SRC0_STATIC | SRC1_STATIC, consecutive launches may overlap (programmatic dependent
    # launch).  extra.dependent_chain re-times the sweep with every launch waiting for the previous one: the decode-graph case.
    Ys = [torch.empty((1, 1, N, M), dtype=torch.float32, device="cuda") for _ in range(nbuf)]
    F_IND = g.MM_SRC0_STATIC | g.MM_SRC1_STATIC
    F_DEP = g.MM_SRC0_STATIC
    if fused:
        # same independence rules as N = 1: every op of the sweep has its own gathered-y slot on every rank; the peer stores and flag
        # publication of op i overlap the streaming of op i+1; one stream-wait at the end of the sweep
        ex = g.PeerExchange(world * M, rank, world, rank * M, slots=nbuf)
        margs = [g.mul_mat_args(t, Ws[i], X, Yloc, M, N, K, flags=F_IND) for i in range(nbuf)]

    def sweep(dependent=False):
        for i in range(nbuf):
            if fused:
                ex.mul_mat_gather(margs[i], slot=i)                                    # compute + NVLink peer stores + flag publish
                if i == nbuf - 1:
                    ex.wait()                                                          # every rank's slices of the whole sweep have landed
            elif world > 1:
                g.mul_mat(t, Ws[i], X, M, N, K, out=Yloc, flags=F_DEP)
                dist.all_gather_into_tensor(Yall, Yloc.view(-1))
            elif dependent:
                g.mul_mat(t, Ws[i], X, M, N, K, out=Yloc, flags=F_DEP)
            else:
                g.mul_mat(t, Ws[i], X, M, N, K, out=Ys[i], flags=F_IND)

    sweep()                                                          # first-launch setup outside capture
    if world == 1:
        sweep(True)
    torch.cuda.synchronize()
    launches_per_unit = None
    if use_graph:
        c0 = g.launch_count()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            for _ in range(SWEEPS_PER_GRAPH):
                sweep()
        launches_per_unit = g.launch_count() - c0
        units = SWEEPS_PER_STEP // SWEEPS_PER_GRAPH

        def step():
            for _ in range(units):
                graph.replay()
    else:
        def step():
            for _ in range(SWEEPS_PER_STEP):
                sweep()

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    for _ in range(args.warmup):
        step()
    barrier()
    sampler = ClockSampler(local)
    if rank == 0:
        sampler.start()
    c0 = g.launch_count()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    barrier()
    t_w0 = sampler.mark()
    ev0.record()
    for _ in range(args.steps):
        step()
    ev1.record()
    barrier()
    t_w1 = sampler.mark()
    ms = ev0.elapsed_time(ev1)
    launched = (g.launch_count() - c0) if not use_graph else launches_per_unit * (SWEEPS_PER_STEP // SWEEPS_PER_GRAPH) * args.steps
    clocks = sampler.stop(t_w0, t_w1) if rank == 0 else None
    if world > 1:
        tmax = torch.tensor([ms], device="cuda")
        dist.all_reduce(tmax, op=dist.ReduceOp.MAX)
        ms = float(tmax.item())
    n_mv = nbuf * SWEEPS_PER_STEP * args.steps
    value = world * n_mv * wb / (ms * 1e-3) / 1e9
    us_per_launch = ms * 1e3 / n_mv

    if args.dump_outputs and rank == 0:
        # what the timed path returned in its last step: one y per weight matrix (inputs are seeded, so two builds compare output for output)
        out_dir = Path(args.dump_outputs)
        out_dir.mkdir(parents=True, exist_ok=True)
        torch.cuda.synchronize()
        if world > 1 and not fused:
            # the NCCL exchange gathers every mat-vec into the one buffer Yall: only the sweep's last output survives the step
            np.save(out_dir / f"y_{nbuf - 1:02d}.npy", Yall.view(world * N, M).float().cpu().numpy())
        else:
            for i in range(nbuf):
                y = Ys[i].view(N, M) if world == 1 else ex.y_full(i).view(world * N, M)
                np.save(out_dir / f"y_{i:02d}.npy", y.float().cpu().numpy())

    # ---- parity of the TIMED configuration: the outputs the timed launches wrote, sampled rows against the CPU oracle
    parity = {}
    if world == 1:
        parity["timed_outputs_nmse_max"] = max(parity_rows(t, Ws[i], Xh, Ys[i], M, N, K, seed=100 + i) for i in range(nbuf))
    else:
        torch.cuda.synchronize()
        worst = 0.0
        if fused:
            # own rows (as stored into the own gathered y) against the oracle; the rows RECEIVED from every peer bit-identical to what that peer computed
            rows = np.sort(np.random.default_rng(7).choice(M, 32, replace=False))
            idx = torch.from_numpy(rows).cuda()
            for sl in (0, nbuf // 2, nbuf - 1):
                yf = ex.y_full(sl).view(world, M)
                worst = max(worst, parity_rows(t, Ws[sl], Xh, yf[rank].reshape(1, M), M, 1, K, seed=200 + sl))
                mine = yf[rank].index_select(0, idx).contiguous()
                allv = [torch.empty_like(mine) for _ in range(world)]
                dist.all_gather(allv, mine)
                for q in range(world):
                    assert torch.equal(allv[q], yf[q].index_select(0, idx)), f"rank {rank}: slice received from rank {q} differs from what it computed (slot {sl})"
        else:
            worst = parity_rows(t, Ws[nbuf - 1], Xh, Yall[rank].reshape(1, M), M, 1, K, seed=300)
        tw = torch.tensor([worst], device="cuda")
        dist.all_reduce(tw, op=dist.ReduceOp.MAX)
        parity["timed_outputs_nmse_max"] = float(tw.item())
        parity["exchange"] = "every rank: own rows vs oracle; rows received from each peer bit-identical to the peer's own (sampled)" if fused else "nccl all-gather"
    assert parity["timed_outputs_nmse_max"] <= 1e-10, f"parity failure in the timed configuration: {parity}"
    parity["tolerance"] = 1e-10

    # ---- e2e through the C ABI with host buffers (N = 1: reported beside the plug-in e2e; N > 1: THE e2e, exchange included): per step
    # one CUDA-graph replay of {pinned host x -> device, the sweep (with the NVLink gather and its wait when N > 1), results -> pinned host}
    xh = torch.empty(N * K, dtype=torch.float32).pin_memory()
    xh.copy_(X.cpu())
    Xst = torch.empty_like(X)
    if fused:
        yh = torch.empty((nbuf, world * M), dtype=torch.float32).pin_memory()
        eargs = [g.mul_mat_args(t, Ws[i], Xst, Yloc, M, N, K, flags=F_DEP) for i in range(nbuf)]
    else:
        yh = torch.empty((nbuf, N * M), dtype=torch.float32).pin_memory()

    def e2e_body():
        Xst.copy_(xh, non_blocking=True)
        for i in range(nbuf):
            if fused:
                ex.mul_mat_gather(eargs[i], slot=i)
            else:
                g.mul_mat(t, Ws[i], Xst, M, N, K, out=Ys[i], flags=F_DEP)
                if world > 1:
                    dist.all_gather_into_tensor(Yall, Ys[i].view(-1))
        if fused:
            ex.wait()
            for i in range(nbuf):
                yh[i].copy_(ex.y_full(i), non_blocking=True)
        else:
            for i in range(nbuf):
                yh[i].copy_(Ys[i].view(-1), non_blocking=True)
    e2e_graphable = world == 1 or fused
    if e2e_graphable:
        e2e_body(); torch.cuda.synchronize()
        ge = torch.cuda.CUDAGraph()
        with torch.cuda.graph(ge):
            e2e_body()

        def e2e_step():
            ge.replay()
            torch.cuda.current_stream().synchronize()
    else:
        def e2e_step():
            e2e_body()
            torch.cuda.current_stream().synchronize()
    for _ in range(5):
        e2e_step()
    barrier()
    e2e_steps = 400
    t0 = time.perf_counter()
    for _ in range(e2e_steps):
        e2e_step()
    e2e_s = time.perf_counter() - t0
    if world > 1:
        tt = torch.tensor([e2e_s], device="cuda")
        dist.all_reduce(tt, op=dist.ReduceOp.MAX)
        e2e_s = float(tt.item())
    shim_e2e = {"value": world * e2e_steps * nbuf * wb / e2e_s / 1e9, "unit": UNIT, "us_per_sweep": e2e_s / e2e_steps * 1e6,
                "h2d_bytes_per_sweep": K * N * 4, "d2h_bytes_per_sweep": int(yh.numel() * 4),
                "api": "C ABI (ggml_b200_mul_mat" + ("_gather + gather_wait" if fused else "") + "), one CUDA-graph replay per sweep: pinned host x -> device, 13 mat-vecs"
                       + (", NVLink exchange" if world > 1 else "") + ", 13 results -> pinned host, stream synchronise"}
    # the host copy must hold what the kernels computed
    e2e_nm = parity_rows(t, Ws[nbuf - 1], Xh, (yh[nbuf - 1].view(world, M)[rank] if fused else yh[nbuf - 1]).cuda().reshape(1, M), M, 1, K, seed=400) if (world == 1 or fused) else None
    if e2e_nm is not None:
        assert e2e_nm <= 1e-10, f"e2e parity failure: {e2e_nm}"
        shim_e2e["parity_nmse"] = e2e_nm

    # ---- extra: the other BASELINE configurations (rank 0 of a single-GPU run; configs[4] on every N)
    extra = {}
    if not args.no_extra:
        # configs[4]: Q4_K 8192 x 28672 row-sharded over the N GPUs (strong scaling: the matrix is fixed, every rank owns 28672 / N rows)
        try:
            Ms, Ks = 28672, 8192
            Mr = Ms // world
            nb4 = max(3, math.ceil(300e6 / weight_bytes(Ks, Mr)))
            W4 = make_weights(torch, 12, nb4, Ks, Mr, seed=4321 + rank)
            X4 = torch.rand(Ks, device="cuda", generator=torch.Generator(device="cuda").manual_seed(5678)) * 2 - 1
            Y4 = torch.empty((1, 1, 1, Mr), dtype=torch.float32, device="cuda")
            Y4s = [torch.empty((1, 1, 1, Mr), dtype=torch.float32, device="cuda") for _ in range(nb4)]
            ex4 = g.PeerExchange(Ms, rank, world, rank * Mr, slots=nb4) if world > 1 else None
            a4 = [g.mul_mat_args(12, W4[i], X4, Y4, Mr, 1, Ks, flags=F_IND) for i in range(nb4)] if world > 1 else None

            def sweep4():
                for i in range(nb4):
                    if world > 1:
                        ex4.mul_mat_gather(a4[i], slot=i)
                        if i == nb4 - 1:
                            ex4.wait()
                    else:
                        g.mul_mat(12, W4[i], X4, Mr, 1, Ks, out=Y4s[i], flags=F_IND)
            sweep4(); barrier()
            s4, _ = timer.time_graph(sweep4, min_seconds=0.15)
            if world > 1:
                tt = torch.tensor([s4], device="cuda")
                dist.all_reduce(tt, op=dist.ReduceOp.MAX)
                s4 = float(tt.item())
            us4 = s4 / nb4 * 1e6
            X4h = X4.cpu().numpy()
            if world > 1:
                nm4 = parity_rows(12, W4[nb4 - 1], X4h, ex4.y_full(nb4 - 1).view(world, Mr)[rank].reshape(1, Mr), Mr, 1, Ks, seed=5)
                tw = torch.tensor([nm4], device="cuda"); dist.all_reduce(tw, op=dist.ReduceOp.MAX); nm4 = float(tw.item())
            else:
                nm4 = max(parity_rows(12, W4[i], X4h, Y4s[i], Mr, 1, Ks, seed=5 + i) for i in range(nb4))
            assert nm4 <= 1e-10, f"parity failure configs[4]: {nm4}"
            ab4 = algorithmic_bytes(Ks, Ms, 1)
            extra["row_shard_strong_q4_K_8192x28672"] = {
                "shape": f"q4_K {Ks}x{Ms} n=1 row-sharded x{world} ({Mr} rows per GPU), fused NVLink gather of the {Ms * 4} B output" if world > 1 else f"q4_K {Ks}x{Ms} n=1 on one GPU",
                "scaling": "strong", "us_per_matvec": us4, "GBps_whole_matrix": weight_bytes(Ks, Ms) / us4 / 1e3, "parity_nmse": nm4,
                "roofline": {"bound": "hbm", "achieved": ab4 / us4 / 1e3, "peak": peaks["hbm"] * world, "unit": "GB/s", "frac": ab4 / us4 / 1e3 / (peaks["hbm"] * world),
                             "note": "peak = N x the measured single-GPU HBM copy bandwidth"}}
            if ex4 is not None:
                dist.barrier(); ex4.close()
            del W4
        except AssertionError:
            raise
        except Exception as e:                       # an optional configuration must never cost the headline line
            extra["row_shard_strong_q4_K_8192x28672"] = {"failed": f"{type(e).__name__}: {e}"[:300]}
    if world == 1 and not args.no_extra:
        # the dependent chain of the headline shape (what a decode graph gives the kernel: every launch waits for its predecessor)
        def dep():
            sweep(True)
        sd, _ = timer.time_graph(dep, min_seconds=0.3)
        usd = sd / nbuf * 1e6
        nmd = parity_rows(t, Ws[nbuf - 1], Xh, Yloc, M, N, K, seed=500)
        assert nmd <= 1e-10, f"parity failure (dependent chain): {nmd}"
        ab = algorithmic_bytes(K, M, N)
        extra["dependent_chain_q4_K_4096x11008"] = {
            "note": "every launch waits for the previous kernel (x treated as its output, shared y): the decode-graph case", "us_per_matvec": usd, "GBps": wb / usd / 1e3,
            "parity_nmse": nmd, "roofline": {"bound": "hbm", "achieved": ab / usd / 1e3, "peak": peaks["hbm"], "unit": "GB/s", "frac": ab / usd / 1e3 / peaks["hbm"]}}
        jobs = [("q4_0_4096x4096_n1", lambda: extra_matvec(torch, g, timer, 2, 4096, 4096, peaks)),
                ("q8_0_4096x4096_n512_tcgen05", lambda: extra_gemm(torch, g, timer, 8, 4096, 512, 4096, peaks)),
                ("q4_K_4096x4096_n512_tcgen05", lambda: extra_gemm(torch, g, timer, 12, 4096, 512, 4096, peaks)),
                ("q6_K_4096x4096_n512_tcgen05", lambda: extra_gemm(torch, g, timer, 14, 4096, 512, 4096, peaks)),
                ("q4_K_4096x32000_n1", lambda: extra_matvec(torch, g, timer, 12, 32000, 4096, peaks, dependent_too=False)),
                ("q8_0_4096x32000_n1", lambda: extra_matvec(torch, g, timer, 8, 32000, 4096, peaks, dependent_too=False)),
                ("q4_K_4096x32000_n512_tcgen05", lambda: extra_gemm(torch, g, timer, 12, 32000, 512, 4096, peaks)),
                ("q8_0_4096x32000_n512_tcgen05", lambda: extra_gemm(torch, g, timer, 8, 32000, 512, 4096, peaks)),
                ("q4_K_4096x11008_n8", lambda: extra_small_batch(torch, g, timer, 12, 11008, 8, 4096, peaks)),
                # the reference harness' own perf shape (tests/test-backend-ops.cpp:4340-4346: m = 4096, k = 14336) at n = 8, and n = 2
                ("q4_K_14336x4096_n8", lambda: extra_small_batch(torch, g, timer, 12, 4096, 8, 14336, peaks)),
                ("q8_0_14336x4096_n8", lambda: extra_small_batch(torch, g, timer, 8, 4096, 8, 14336, peaks)),
                ("q6_K_14336x4096_n8", lambda: extra_small_batch(torch, g, timer, 14, 4096, 8, 14336, peaks)),
                ("q4_K_14336x4096_n2", lambda: extra_small_batch(torch, g, timer, 12, 4096, 2, 14336, peaks))]
        for name, job in jobs:
            try:
                extra[name] = job()
            except AssertionError:
                raise                                 # a parity failure fails the run
            except Exception as e:
                extra[name] = {"failed": f"{type(e).__name__}: {e}"[:300]}
            torch.cuda.empty_cache()

    if rank != 0:
        if world > 1:
            dist.barrier()
            if ex is not None:
                ex.close()
            dist.destroy_process_group()
        return
    if world > 1:
        dist.barrier()

    achieved = algorithmic_bytes(K, M, N) / (us_per_launch * 1e-6) / 1e9
    traffic = None
    for name in ("r02_gemv_q4k_traffic.json", "r01_gemv_q4k_traffic.json"):
        tp = ROOT / "profiles" / name
        if tp.exists():
            try:
                traffic = json.loads(tp.read_text()).get("dram_bytes_per_launch")
                break
            except Exception:
                traffic = None
    line = {
        "metric": METRIC, "value": value, "unit": UNIT, "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
        "ms_per_step": ms / args.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": DTYPE, "data": "synthetic", "config": dict(CONFIG),
        "launch": {"mode": f"CUDA-graph replay ({SWEEPS_PER_GRAPH} sweeps per graph)" if use_graph else "plain stream launches",
                   "independence": "mat-vecs of a sweep are independent ops (fixed x, one y per weight matrix) as in the reference's eval_perf; consecutive launches may "
                                   "overlap via programmatic dependent launch; extra.dependent_chain_* is the serialised case",
                   "parallelism": (f"row-shard x{world}, exchange fused into the mat-vec kernel (NVLink peer stores + flags)" if fused else
                                   f"row-shard x{world} + NCCL all-gather of output slices") if world > 1 else "single GPU",
                   "timed_seconds": ms * 1e-3},
        "parity": parity,
        "gpu_launches": int(launched),
        "clocks": clocks,
        "roofline": {"bound": "hbm", "achieved": achieved, "peak": peaks["hbm"], "unit": "GB/s", "frac": achieved / peaks["hbm"], "traffic": traffic,
                     "kernel": "mmvq_sb_kernel<Q4_K>", "us_per_launch": us_per_launch,
                     "algorithmic_bytes_per_launch": algorithmic_bytes(K, M, N), "peak_source": peaks["src"]},
    }
    if world == 1:
        pe = run_child("--plugin-e2e-child", 240)
        if "async" in pe:
            a, s_ = pe["async"], pe["sync"]
            assert a["parity_nmse"] <= 1e-10 and s_["parity_nmse"] <= 1e-10, f"plug-in e2e parity failure: {pe}"
            line["e2e"] = {"value": wb / a["s_per_matvec"] / 1e9, "unit": UNIT, "h2d_bytes_per_step": K * N * 4 * SWEEPS_PER_STEP, "d2h_bytes_per_step": M * N * 4 * nbuf * SWEEPS_PER_STEP,
                           "us_per_matvec": a["s_per_matvec"] * 1e6, "parity_nmse": a["parity_nmse"],
                           "api": f"ggml plug-in ({pe['device']}): the reference's ggml_backend_tensor_set_async(x) -> ggml_backend_graph_compute_async(13 MUL_MAT nodes) -> "
                                  "13 x ggml_backend_tensor_get_async -> ggml_backend_synchronize per sweep, driving libggml-b200.so; the reference arm is timed through the same calls",
                           "sync_calls": {"value": wb / s_["s_per_matvec"] / 1e9, "us_per_matvec": s_["s_per_matvec"] * 1e6,
                                          "api": "ggml_backend_tensor_set / graph_compute / 13 x tensor_get (every call synchronises)"},
                           "resident_through_plugin": {"value": wb / pe["resident"]["s_per_matvec"] / 1e9, "note": "graph_compute only (cached CUDA graph replay), host clock"},
                           "c_abi": shim_e2e}
        else:
            line["e2e"] = dict(shim_e2e, h2d_bytes_per_step=K * N * 4 * SWEEPS_PER_STEP, d2h_bytes_per_step=M * N * 4 * nbuf * SWEEPS_PER_STEP, plugin_failed=pe.get("failed"))
    else:
        line["e2e"] = dict(shim_e2e, h2d_bytes_per_step=K * N * 4 * SWEEPS_PER_STEP, d2h_bytes_per_step=int(yh.numel() * 4) * SWEEPS_PER_STEP)
    if world == 1 and not args.no_extra:
        extra["gpt2_117M_q4_0_decode"] = run_child("--gpt2-child", 420)
    line["extra"] = extra
    if world == 1 and not args.no_cpu_baseline:
        # the baseline is a report, never a reason to lose the GPU line: run the reference in a child with a deadline
        cb = run_child("--cpu-baseline-child", 150)
        line["cpu_baseline"] = cb if "value" in cb else {"value": None, "unit": UNIT, "cores": None, "kind": "reference", "sample": "failed: " + cb.get("failed", "?")}
    print(json.dumps(line), flush=True)
    if world > 1:
        if ex is not None:
            ex.close()
        dist.destroy_process_group()


def extra_small_batch(torch, g, timer, t, M, n, K, peaks, seed=13):
    """2 <= n <= 8 on the bandwidth path (mmvq_mma.cu: int8 mma.sync consume phase; dependent launches, weights streaming from HBM)"""
    wb = weight_bytes(K, M, t)
    nbuf = max(3, math.ceil(300e6 / wb))
    Ws = make_weights(torch, t, nbuf, K, M, seed)
    X = torch.rand(n * K, device="cuda", generator=torch.Generator(device="cuda").manual_seed(5678)) * 2 - 1
    Ys = [torch.empty((1, 1, n, M), dtype=torch.float32, device="cuda") for _ in range(nbuf)]
    assert g.mul_mat_plan(t, M, n, K) == g.MM_GEMV

    def sweep():
        for i in range(nbuf):
            g.mul_mat(t, Ws[i], X, M, n, K, out=Ys[i], flags=g.MM_SRC0_STATIC)
    sweep(); torch.cuda.synchronize()
    s, _ = timer.time_graph(sweep)
    us = s / nbuf * 1e6
    nm = max(parity_rows(t, Ws[i], X.cpu().numpy(), Ys[i], M, n, K, nrows=32, seed=i) for i in range(nbuf))
    assert nm <= 1e-10, f"parity failure small batch: {nm}"
    ab = algorithmic_bytes(K, M, n, t)
    return {"shape": f"{TNAME[t]} {K}x{M} n={n}", "us_per_mul_mat": us, "GBps": wb / us / 1e3, "parity_nmse": nm, "launches_per_mul_mat": 2,
            "kernels": "mma_quantize_kernel (activations -> int8 records, once per launch) + mmvq_mma_kernel",
            "roofline": {"bound": "hbm", "achieved": ab / us / 1e3, "peak": peaks["hbm"], "unit": "GB/s", "frac": ab / us / 1e3 / peaks["hbm"]}}


if __name__ == "__main__":
    main()
