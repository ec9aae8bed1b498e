"""Which kernel a mul_mat takes, and the workspace it asks for.

Route pin: ggml_b200_mul_mat_plan (the family code, and the error text on errors), ggml_b200_mul_mat_workspace_size,
ggml_b200_mul_mat_gather_supported, ggml_b200_mul_mat_id_workspace_size and ggml_b200_mul_mat_f16_workspace_size over a fixed grid,
compared with a fixture under tests/golden/.  Planning reads no memory (the pointers are aligned dummies), but it depends on the machine:
without a CUDA driver no GEMM shape is eligible (no tensor-map encoder), and grid and split-K sizes follow the SM count.  So each
fixture records the environment it was made in, and the test uses the one that matches, or skips.  Planning also reads two
environment variables (PLANNING_ENV), so the test skips when either is set.  Regenerate a fixture for the machine at hand with

    python tests/test_mul_mat_routes.py --regen [--lib path/to/libggml-b200-kernels.so]

Workspace agreement (GPU): a launch given exactly the queried workspace succeeds; given one byte less it returns GGML_B200_EWORKSPACE
before it launches anything.
"""
from __future__ import annotations

import argparse
import ctypes as C
import gzip
import json
import os
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

import ggml_b200 as g  # noqa: E402

GOLDEN = ROOT / "tests" / "golden"
EWORKSPACE = -3

TYPES = [t for t in sorted(g.TYPE_NAMES) if t not in (g.F32, g.F16)] + [g.F32]     # the 21 weight types, then an unsupported one
MK = [(16, 256), (64, 320), (4096, 4096), (11008, 4096), (4096, 14336), (1024, 81920)]
NS = [1, 2, 4, 5, 8, 9, 512]
FLAGS = [g.MM_AUTO, g.MM_GENERIC, g.MM_GEMV, g.MM_GEMM, g.MM_GEMV | g.MM_GEMV_V1, g.MM_GEMV_MMA, g.MM_GEMV_DP4A,
         g.MM_SRC0_STATIC | g.MM_SRC1_STATIC]
SRC1 = [256, 260]                                                                 # 16-byte aligned, only 4-byte aligned
# MUL_MAT_ID: (type, M, K, n_expert, n_used, nb1cols, n_tok)
MOE = [(g.Q4_K, 1408, 2048, 64, 6, 1, 1), (g.Q4_K, 1408, 2048, 64, 6, 6, 512), (g.Q8_0, 14336, 4096, 8, 2, 1, 32),
       (g.Q6_K, 4096, 14336, 8, 2, 2, 512), (g.IQ2_XXS, 2048, 4096, 32, 4, 1, 128), (g.Q4_0, 256, 320, 4, 2, 1, 7)]
# dense fp16 weights: (M, N, K)
F16 = [(4096, 512, 4096), (4096, 9, 4096), (4096, 8, 4096), (11008, 64, 4096), (100, 16, 320), (4096, 1, 4096)]
# the variables a plan depends on besides the call's arguments
PLANNING_ENV = ("GGML_B200_FORCE_GENERIC", "GGML_B200_MMID_GROUPED")


def load(path: Path) -> C.CDLL:
    L = C.CDLL(str(path))
    L.ggml_b200_last_error.restype = C.c_char_p
    L.ggml_b200_mul_mat_plan.argtypes = [C.POINTER(g.MulMatArgs)]
    L.ggml_b200_mul_mat.argtypes = [C.POINTER(g.MulMatArgs), C.c_void_p]
    L.ggml_b200_mul_mat_id.argtypes = [C.POINTER(g.MulMatIdArgs), C.c_void_p]
    L.ggml_b200_mul_mat_workspace_size.restype = C.c_size_t
    L.ggml_b200_mul_mat_workspace_size.argtypes = [C.POINTER(g.MulMatArgs)]
    L.ggml_b200_mul_mat_gather_supported.argtypes = [C.POINTER(g.MulMatArgs)]
    L.ggml_b200_mul_mat_id_workspace_size.restype = C.c_size_t
    L.ggml_b200_mul_mat_id_workspace_size.argtypes = [C.POINTER(g.MulMatIdArgs)]
    L.ggml_b200_mul_mat_f16_workspace_size.restype = C.c_size_t
    L.ggml_b200_mul_mat_f16_workspace_size.argtypes = [C.c_int64, C.c_int64, C.c_int64]
    L.ggml_b200_mul_mat_f16.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_int64, C.c_int64, C.c_int64,
                                        C.c_void_p, C.c_size_t, C.c_uint32, C.c_void_p]
    L.ggml_b200_launch_count.restype = C.c_uint64
    L.ggml_b200_row_size.restype = C.c_size_t
    L.ggml_b200_row_size.argtypes = [C.c_int32, C.c_int64]
    return L


def environment(L: C.CDLL) -> dict:
    try:
        C.CDLL("libcuda.so.1")
        driver = True
    except OSError:
        driver = False
    device = "none"
    if L.ggml_b200_device_count() > 0:
        import torch
        device = torch.cuda.get_device_name(0)
    return {"driver": driver, "sm_count": int(L.ggml_b200_sm_count()), "device": device}


def qk(t) -> int:
    return 32 if t in (g.Q4_0, g.Q8_0, g.Q4_1, g.Q5_0, g.Q5_1, g.IQ4_NL) else 256


def mm_args(L, t, M, N, K, flags, src1):
    a = g.MulMatArgs()
    a.type, a.flags, a.K, a.M, a.N = t, flags, K, M, N
    a.ne02 = a.ne03 = a.ne12 = a.ne13 = 1
    rb = int(L.ggml_b200_row_size(t, K))
    a.nb01, a.nb02, a.nb03, a.nb11, a.nb12, a.nb13 = rb, rb * M, rb * M, K * 4, K * 4 * N, K * 4 * N
    a.src0, a.src1, a.dst = 256, src1, 256
    return a


def mmid_args(L, t, M, K, n_expert, n_used, nb1cols, n_tok):
    a = g.MulMatIdArgs()
    a.type, a.K, a.M, a.n_expert, a.n_used, a.nb1cols, a.n_tok = t, K, M, n_expert, n_used, nb1cols, n_tok
    rb = int(L.ggml_b200_row_size(t, K))
    a.nb01, a.nb02, a.nb11, a.nb12, a.ids_nb1 = rb, rb * M, K * 4, K * 4 * nb1cols, n_used * 4
    a.src0 = a.src1 = a.ids = a.dst = 256
    return a


def grid():
    for t in TYPES:
        for M, K in MK:
            for N in NS:
                for flags in FLAGS:
                    for src1 in SRC1:
                        yield t, M, K, N, flags, src1


def record(L) -> dict:
    """The planner's answers over the grid: one [plan, workspace, gather_supported, error] row per case, the error message as an index
    into a table (-1: none set)."""
    errors: list[str] = []
    rows = []
    for t, M, K, N, flags, src1 in grid():
        a = mm_args(L, t, M, N, K, flags, src1)
        L.ggml_b200_mul_mat_plan(None)               # sets a known message: a plan that sets none (a forced family refused) leaves it
        primed = L.ggml_b200_last_error().decode()
        plan = int(L.ggml_b200_mul_mat_plan(C.byref(a)))
        err = -1
        text = L.ggml_b200_last_error().decode()
        if plan < 0 and text != primed:
            if text not in errors:
                errors.append(text)
            err = errors.index(text)
        rows.append([plan, int(L.ggml_b200_mul_mat_workspace_size(C.byref(a))), int(L.ggml_b200_mul_mat_gather_supported(C.byref(a))), err])
    return {"grid": {"types": TYPES, "mk": MK, "n": NS, "flags": FLAGS, "src1": SRC1, "moe": MOE, "f16": F16},
            "mul_mat": rows, "errors": errors,
            "mul_mat_id": [int(L.ggml_b200_mul_mat_id_workspace_size(C.byref(mmid_args(L, *s)))) for s in MOE],
            "mul_mat_f16": [int(L.ggml_b200_mul_mat_f16_workspace_size(M, N, K)) for M, N, K in F16]}


def fixture_name(env: dict) -> str:
    if env["device"] == "none":
        return "mul_mat_routes_nodevice.json.gz"
    return "mul_mat_routes_" + ("h100" if "H100" in env["device"] else "".join(c for c in env["device"].lower() if c.isalnum())) + ".json.gz"


def regen(lib: Path, out: Path) -> Path:
    L = load(lib)
    env = environment(L)
    path = out / fixture_name(env)
    data = {"environment": env, **record(L)}
    path.write_bytes(gzip.compress(json.dumps(data, separators=(",", ":")).encode(), mtime=0))
    return path


@pytest.mark.parametrize("fixture", [pytest.param("mul_mat_routes_nodevice.json.gz", id="nodevice"),
                                     pytest.param("mul_mat_routes_h100.json.gz", id="h100", marks=pytest.mark.gpu)])
def test_route_pin(fixture):
    if any(k in os.environ for k in PLANNING_ENV):
        pytest.skip(f"one of {PLANNING_ENV} is set: planning reads them")
    L = load(g.KERNELS_SO)
    env = environment(L)
    want = json.loads(gzip.decompress((GOLDEN / fixture).read_bytes()))
    if want["environment"] != env:
        pytest.skip(f"{fixture} was made in {want['environment']}, this machine is {env}")
    got = record(L)
    assert json.loads(json.dumps(got["grid"])) == want["grid"], "the fixture was made over another grid: regenerate it"
    bad = []
    for case, r, w in zip(grid(), got["mul_mat"], want["mul_mat"]):
        rt = got["errors"][r[3]] if r[3] >= 0 else None
        wt = want["errors"][w[3]] if w[3] >= 0 else None
        if r[:3] != w[:3] or rt != wt:
            bad.append((case, (r[:3], rt), (w[:3], wt)))
    assert not bad, f"{len(bad)} of {len(got['mul_mat'])} cases differ (type, M, K, N, flags, src1), got, want; first: {bad[:5]}"
    assert got["mul_mat_id"] == want["mul_mat_id"]
    assert got["mul_mat_f16"] == want["mul_mat_f16"]


# ----------------------------------------------------------------------------------------------------------- workspace agreement
# (type, M, N, K, flags, the route it takes)
AGREE_MM = [
    (g.IQ2_XXS, 4096, 1, 4096, g.MM_AUTO, "generic"),
    (g.Q4_K, 4096, 2, 4096, g.MM_GENERIC, "generic (forced)"),
    (g.Q4_K, 4096, 1, 4096, g.MM_GEMV | g.MM_GEMV_V1, "first-generation TMA"),
    (g.Q4_K, 4096, 1, 4096, g.MM_AUTO, "superblock"),
    (g.Q8_0, 4096, 3, 4096, g.MM_GEMV | g.MM_GEMV_DP4A, "superblock, 3 columns"),
    (g.Q4_K, 4096, 7, 16384, g.MM_GEMV | g.MM_GEMV_DP4A, "superblock in column groups"),
    (g.Q4_K, 4096, 4, 4096, g.MM_AUTO, "mma"),
    (g.Q6_K, 4096, 1, 14336, g.MM_AUTO, "mma, n = 1 long rows"),
    (g.Q5_0, 4096, 8, 4096, g.MM_AUTO, "mma"),
    (g.Q4_K, 4096, 512, 4096, g.MM_AUTO, "wgmma"),
    (g.Q8_0, 11008, 64, 4096, g.MM_AUTO, "wgmma, split-K"),
    (g.Q6_K, 4096, 9, 14336, g.MM_AUTO, "wgmma"),
    (g.Q4_K, 4096, 5, 4096, g.MM_GEMM, "wgmma (forced)"),
    (g.IQ2_XXS, 4096, 512, 4096, g.MM_AUTO, "dense"),
    (g.TQ2_0, 1024, 16, 2048, g.MM_AUTO, "dense"),
]
AGREE_F16 = [(4096, 512, 4096), (11008, 9, 4096)]
# (type, M, K, n_expert, n_used, nb1cols, n_tok): grouped when GGML_B200_MMID_GROUPED=1 and there are >= 32 pairs, else per pair
AGREE_MMID = [(g.Q4_K, 1024, 2048, 8, 2, 1, 64), (g.Q8_0, 512, 4096, 8, 2, 2, 128), (g.Q4_K, 1024, 2048, 8, 2, 1, 4)]


def agreement() -> list[str]:
    """Runs every AGREE_* case on cuda:0; returns the failures."""
    import numpy as np
    import torch
    from oracle import oracle as O
    L = load(g.KERNELS_SO)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    rng = np.random.default_rng(0)
    fails = []

    def check(what, ws, call):
        """call(workspace_ptr, workspace_size) -> rc"""
        buf = torch.empty(max(ws, 1), dtype=torch.uint8, device="cuda")
        ptr = buf.data_ptr() if ws else None
        if ws:
            n0 = int(L.ggml_b200_launch_count())
            rc = call(ptr, ws - 1)
            if rc != EWORKSPACE or int(L.ggml_b200_launch_count()) != n0:
                fails.append(f"{what}: workspace {ws} - 1 gave rc {rc} after {int(L.ggml_b200_launch_count()) - n0} launches")
        rc = call(ptr, ws)
        torch.cuda.synchronize()
        if rc != 0:
            fails.append(f"{what}: workspace {ws} gave rc {rc}: {L.ggml_b200_last_error().decode()}")

    for t, M, N, K, flags, route in AGREE_MM:
        W = torch.from_numpy(O.random_blocks(t, M * K // qk(t), rng)).cuda()
        X = torch.randn(N, K, device="cuda")
        Y = torch.empty(N, M, device="cuda")
        a = mm_args(L, t, M, N, K, flags, X.data_ptr())
        a.src0, a.dst = W.data_ptr(), Y.data_ptr()
        ws = int(L.ggml_b200_mul_mat_workspace_size(C.byref(a)))

        def mm(ptr, size, a=a):
            a.workspace, a.workspace_size = ptr, size
            return L.ggml_b200_mul_mat(C.byref(a), st)
        check(f"{g.TYPE_NAMES[t]} M={M} N={N} K={K} flags={flags} ({route})", ws, mm)
    for M, N, K in AGREE_F16:
        W = torch.randn(M, K, device="cuda").half()
        X = torch.randn(N, K, device="cuda")
        Y = torch.empty(N, M, device="cuda")
        check(f"f16 M={M} N={N} K={K}", int(L.ggml_b200_mul_mat_f16_workspace_size(M, N, K)),
              lambda ptr, size: L.ggml_b200_mul_mat_f16(W.data_ptr(), K * 2, X.data_ptr(), K * 4, Y.data_ptr(), M, N, K, ptr, size, 0, st))
    for t, M, K, n_expert, n_used, nb1cols, n_tok in AGREE_MMID:
        W = torch.from_numpy(O.random_blocks(t, n_expert * M * K // qk(t), rng)).cuda()
        X = torch.randn(n_tok, nb1cols, K, device="cuda")
        ids = torch.from_numpy(rng.integers(0, n_expert, size=(n_tok, n_used)).astype(np.int32)).cuda()
        Y = torch.empty(n_tok, n_used, M, device="cuda")
        a = mmid_args(L, t, M, K, n_expert, n_used, nb1cols, n_tok)
        a.src0, a.src1, a.ids, a.dst = W.data_ptr(), X.data_ptr(), ids.data_ptr(), Y.data_ptr()

        def mmid(ptr, size, a=a):
            a.workspace, a.workspace_size = ptr, size
            return L.ggml_b200_mul_mat_id(C.byref(a), st)
        check(f"mul_mat_id {g.TYPE_NAMES[t]} M={M} K={K} experts={n_expert}x{n_used} tokens={n_tok}",
              int(L.ggml_b200_mul_mat_id_workspace_size(C.byref(a))), mmid)
    return fails


@pytest.mark.gpu
def test_workspace_agreement():
    # its own process: the grouped MUL_MAT_ID path is opt-in through a variable the library reads once
    env = dict(os.environ, GGML_B200_MMID_GROUPED="1")
    r = subprocess.run([sys.executable, __file__, "--agreement"], env=env, cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--regen", action="store_true", help="write the route-pin fixture of this machine")
    ap.add_argument("--lib", type=Path, default=g.KERNELS_SO, help="library to record (default: the in-tree build)")
    ap.add_argument("--out", type=Path, default=GOLDEN, help="directory of the fixture")
    ap.add_argument("--agreement", action="store_true", help="run the workspace-agreement cases on cuda:0")
    args = ap.parse_args()
    if args.regen:
        print(regen(args.lib, args.out))
    if args.agreement:
        fails = agreement()
        print("\n".join(fails) or f"workspace agreement: {len(AGREE_MM) + len(AGREE_F16) + len(AGREE_MMID)} cases OK")
        sys.exit(1 if fails else 0)


if __name__ == "__main__":
    main()
