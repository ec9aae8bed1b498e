"""TEST INFRASTRUCTURE ONLY: the checks the decoder-graph tests share (tests/test_gpu_{llama_graph,moe,mamba,rwkv}.py), over the programs
of oracle/decoders.mk and their command line (oracle/decoder_harness.h)."""
from __future__ import annotations

import re
import subprocess
from pathlib import Path

import numpy as np
import pytest

from oracle import oracle as O

N_STEPS = 24
N_VOCAB = 4096


def require(*ref_files: str) -> Path:
    """fails the test where the plug-in or one of `ref_files` (programs in oracle/_ref) is missing; returns the plug-in's path"""
    import ggml_b200
    if not ggml_b200.BACKEND_SO.exists():
        pytest.fail(f"{ggml_b200.BACKEND_SO} missing: run __graft_entry__.build() where the ggml headers are available")
    for f in ref_files:
        if not (O.REF_DIR / f).exists():
            pytest.fail(f"oracle/_ref/{f} missing (oracle/Makefile and oracle/decoders.mk in the build container)")
    return ggml_b200.BACKEND_SO


def plugin(*ref_files: str) -> Path:
    """require(*ref_files), then the plug-in loaded into the reference"""
    so = require(*ref_files)
    assert O.Ref().load_backend(so)
    return so


def check_test_backend_ops(plugin: Path, op: str, n_min: int) -> None:
    """the reference's own test-backend-ops on B2000 against ggml-cpu: every `op` case (at least n_min) executed and passed, none declined"""
    env = O.ref_env()
    env["GGML_BACKEND_PATH"] = str(plugin)
    p = subprocess.run([str(O.REF_DIR / "test-backend-ops"), "test", "-o", op, "-b", "B2000"], env=env, capture_output=True, text=True, timeout=900)
    out = p.stdout + p.stderr
    tail = "\n".join(out.splitlines()[-25:])
    assert p.returncode == 0 and "FAIL" not in out, tail
    cases = [l for l in out.splitlines() if l.strip().startswith(op + "(")]
    declined = [l for l in cases if "not supported" in l]
    assert not declined, "\n".join(declined[:10])
    ok = [l for l in cases if "OK" in l]
    assert len(ok) == len(cases) and len(ok) >= n_min, (len(ok), len(cases), tail)
    m = re.search(r"(\d+)/(\d+) tests passed", out)
    assert m and m.group(1) == m.group(2), tail


def _run(exe: Path, args: list[str], env_extra: dict | None = None) -> str:
    import ggml_b200
    env = O.ref_env()
    env["GGML_BACKEND_PATH"] = str(ggml_b200.BACKEND_SO)
    env.update(env_extra or {})
    p = subprocess.run([str(exe), *args], env=env, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, (p.stdout + p.stderr)[-3000:]
    return p.stdout


def compare(exe: Path, preset: str, sync: bool):
    """compare mode on B2000: ({phase: summary}, {"node" | "inode" | "topk": [the lines of that kind, split into fields]})"""
    out = _run(exe, [preset, "compare", "B2000"] + (["sync"] if sync else []))
    summary, lines = {}, {"node": [], "inode": [], "topk": []}
    for l in out.splitlines():
        f = l.split()
        if f and f[0] == "summary":
            summary[f[1]] = dict(n_over=int(f[4]), worst=float(f[6]), first=int(f[8]), op=f[9], logits=float(f[11]))
        elif f and f[0] in lines:
            lines[f[0]].append(f)
    return summary, lines


def run(exe: Path, preset: str, dev: str, path: Path, n_seqs: int = 1, force: Path | None = None, env_extra: dict | None = None):
    """run mode for N_STEPS steps: ({first word: the other words} of each output line, logits [N_STEPS x n_seqs, N_VOCAB])"""
    out = _run(exe, [preset, "run", dev, str(N_STEPS), str(path)] + ([str(force)] if force else []), env_extra)
    kv = {l.split()[0]: l.split()[1:] for l in out.splitlines() if l.strip()}
    logits = np.fromfile(path, dtype=np.float32).reshape(-1, N_VOCAB)
    assert logits.shape[0] == N_STEPS * n_seqs
    return kv, logits


def check_tracks_cpu(exe: Path, preset: str, cpu_run, tmp_path: Path, n_seqs: int = 1):
    """B2000 teacher-forced along ggml-cpu's greedy tokens (`cpu_run`: run() on the CPU): every logits row within NMSE 5e-3 of the CPU's,
    a differing argmax only where the CPU's top-2 margin is <= 6 x the RMS deviation, the same argmax in at least half the rows.
    Returns (ties: [(row, margin, rms)], worst NMSE, rows with the same argmax, the CPU's tokens)."""
    ckv, cpu_logits = cpu_run
    ctoks = [int(t) for t in ckv["tokens"]]
    assert ctoks == [int(v) for v in cpu_logits.argmax(1)]
    force = tmp_path / "force.bin"
    np.array(ctoks, dtype=np.int32).tofile(force)
    _, gpu_logits = run(exe, preset, "B2000", tmp_path / "forced.bin", n_seqs, force=force)
    ties, worst, n_same = [], 0.0, 0
    for i in range(cpu_logits.shape[0]):
        c, g_ = cpu_logits[i].astype(np.float64), gpu_logits[i].astype(np.float64)
        nm = O.nmse(gpu_logits[i], cpu_logits[i])
        worst = max(worst, nm)
        assert nm <= 5e-3, (preset, i, nm)
        rms = float(np.sqrt(np.mean((g_ - c) ** 2)))
        top2 = np.sort(c)[-2:]
        margin = float(top2[1] - top2[0])
        if int(g_.argmax()) != int(c.argmax()):
            ties.append((i, margin, rms))
            assert margin <= 6 * rms, f"{preset}: row {i}: argmax differs although the CPU margin {margin:.3e} exceeds 6 x the RMS deviation {rms:.3e}"
        else:
            n_same += 1
    assert n_same >= cpu_logits.shape[0] // 2, (n_same, ties)
    return ties, worst, n_same, ctoks


def check_fusions_and_graphs_bit_exact(exe: Path, preset: str, tmp_path: Path, n_seqs: int = 1) -> None:
    """the same forced tokens with GGML_B200_DISABLE_FUSION and with GGML_B200_DISABLE_GRAPHS give the default run's logits bit for bit"""
    force = tmp_path / "force.bin"
    np.arange(100, 100 + N_STEPS * n_seqs, dtype=np.int32).tofile(force)
    outs = {}
    for name, env in (("default", {}), ("nofusion", {"GGML_B200_DISABLE_FUSION": "1"}), ("nographs", {"GGML_B200_DISABLE_GRAPHS": "1"})):
        _, outs[name] = run(exe, preset, "B2000", tmp_path / f"{name}.bin", n_seqs, force=force, env_extra=env)
    for name in ("nofusion", "nographs"):
        assert np.array_equal(outs["default"].view(np.uint32), outs[name].view(np.uint32)), (preset, name)
