"""CPU-only: the C ABI and the product/test-infrastructure separation.

* every function declared in include/ggml-b200.h is exported by libggml-b200-kernels.so, every entry point declared in
  include/ggml-b200-backend.h and the include/ggml-cuda.h facade by libggml-b200.so (symbols only: no compute without a GPU);
* argument validation of the shim works without a device (error codes, never a CPU fallback);
* the product (ggml_b200/, the two shared libraries) neither imports nor links anything under oracle/;
* the product reads exactly the environment variables INTEGRATION.md lists."""
import ctypes as C
import re
import subprocess
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]


def declared(header):
    txt = (ROOT / "include" / header).read_text()
    return sorted(set(re.findall(r"GGML_B200_API\s+[^;(]*?\b(ggml_[a-z0-9_]+)\s*\(", txt)))


def exported(so):
    out = subprocess.run(["nm", "-D", "--defined-only", str(so)], capture_output=True, text=True, check=True).stdout
    return {l.split()[-1] for l in out.splitlines() if " T " in l}


def test_kernel_shim_exports_every_declared_symbol():
    import ggml_b200
    assert ggml_b200.KERNELS_SO.exists(), "run __graft_entry__.build()"
    want = declared("ggml-b200.h")
    assert len(want) >= 20
    missing = [s for s in want if s not in exported(ggml_b200.KERNELS_SO)]
    assert not missing, missing


def test_backend_plugin_exports_entry_points():
    import ggml_b200
    assert ggml_b200.BACKEND_SO.exists(), "run __graft_entry__.build() where the ggml headers are available"
    have = exported(ggml_b200.BACKEND_SO)
    want = declared("ggml-b200-backend.h") + [
        # include/ggml-cuda.h:23-45 (reference): the ABI bound by programs compiled with -DGGML_USE_CUDA
        "ggml_backend_cuda_init", "ggml_backend_is_cuda", "ggml_backend_cuda_buffer_type", "ggml_backend_cuda_split_buffer_type",
        "ggml_backend_cuda_host_buffer_type", "ggml_backend_cuda_get_device_count", "ggml_backend_cuda_get_device_description",
        "ggml_backend_cuda_get_device_memory", "ggml_backend_cuda_register_host_buffer", "ggml_backend_cuda_unregister_host_buffer",
        "ggml_backend_cuda_reg"]
    missing = [s for s in want if s not in have]
    assert not missing, missing


def test_plugin_without_a_device_reports_nothing_instead_of_aborting():
    """No supported GPU visible (this suite runs without a GPU; skipped where one exists): the plug-in must load, score 0 so that ggml's loader passes it
    over (src/ggml-backend-reg.cpp:220-263), enumerate no device and hand out no backend / buffer type -- in a child process, because the
    reference's own answer to misuse is GGML_ABORT."""
    import ggml_b200
    ref = ROOT / "oracle" / "_ref"
    if not (ref / "libggml-base.so").exists():
        pytest.skip("needs ggml-base (oracle/_ref) to resolve the plug-in's ggml symbols")
    code = f"""
import ctypes as C
C.CDLL(r"{ref / 'libggml-base.so'}", mode=C.RTLD_GLOBAL)
try:
    C.CDLL(r"{ref / 'libggml-cpu.so'}", mode=C.RTLD_GLOBAL)
except OSError:
    pass
B = C.CDLL(r"{ggml_b200.BACKEND_SO}")
for f in ("ggml_backend_b200_host_buffer_type", "ggml_backend_b200_init", "ggml_backend_b200_buffer_type", "ggml_backend_b200_split_buffer_type", "ggml_backend_init"):
    getattr(B, f).restype = C.c_void_p
B.ggml_backend_b200_split_buffer_type.argtypes = [C.c_int, C.c_void_p]
n = B.ggml_backend_b200_get_device_count()
if n > 0:
    print("HAS_GPU")
else:
    assert B.ggml_backend_score() == 0
    assert B.ggml_backend_init() is not None                      # the registry entry itself exists, with zero devices
    assert B.ggml_backend_b200_host_buffer_type() is None
    assert B.ggml_backend_b200_buffer_type(0) is None
    assert B.ggml_backend_b200_split_buffer_type(0, None) is None
    assert B.ggml_backend_b200_init(0) is None
    print("OK")
"""
    p = subprocess.run([__import__("sys").executable, "-c", code], capture_output=True, text=True, timeout=120)
    assert p.returncode == 0, p.stdout + p.stderr
    if "HAS_GPU" in p.stdout:
        pytest.skip("a supported GPU is visible")
    assert "OK" in p.stdout


def test_shim_validates_arguments_without_a_device():
    import ggml_b200 as g
    L = g.lib()
    assert L.ggml_b200_row_size(g.Q4_K, 4096) == 2304 and L.ggml_b200_row_size(g.Q6_K, 256) == 210
    assert L.ggml_b200_row_size(g.Q4_1, 64) == 40 and L.ggml_b200_row_size(g.Q5_0, 64) == 44 and L.ggml_b200_row_size(g.Q5_1, 64) == 48
    assert L.ggml_b200_row_size(g.Q2_K, 512) == 168 and L.ggml_b200_row_size(g.Q3_K, 512) == 220
    assert L.ggml_b200_row_size(g.Q4_0, 4096) == 2304 and L.ggml_b200_row_size(g.Q8_0, 4096) == 4352 and L.ggml_b200_row_size(g.Q5_K, 256) == 176
    a = g.MulMatArgs()
    a.type, a.K, a.M, a.N = 30, 4096, 16, 1                 # BF16 weights: not implemented -> explicit error, not a fallback
    a.ne02 = a.ne03 = a.ne12 = a.ne13 = 1
    assert L.ggml_b200_mul_mat_plan(C.byref(a)) == -1
    a.type, a.K = g.Q4_K, 100                               # K not a multiple of the block size
    assert L.ggml_b200_mul_mat_plan(C.byref(a)) == -2
    assert b"multiple of the block size" in L.ggml_b200_last_error()
    assert g.mul_mat_plan(g.Q4_K, 11008, 1, 4096) == g.MM_GEMV
    assert g.mul_mat_plan(g.Q4_0, 16, 1, 32) == g.MM_GENERIC
    assert L.ggml_b200_dequantize(g.Q4_0, None, None, 0, 33, None) == -2
    assert L.ggml_b200_dequantize(99, None, None, 0, 32, None) == -1


def test_product_does_not_touch_the_oracle():
    import ggml_b200
    for py in (ROOT / "ggml_b200").rglob("*.py"):
        src = py.read_text()
        assert not re.search(r"^\s*(from|import)\s+oracle\b", src, re.M), f"{py} imports the oracle"
        assert "liboracle" not in src and "_ref" not in src.replace("ggml_b200", ""), f"{py} references test infrastructure"
    for src in list((ROOT / "ggml_b200" / "csrc").rglob("*.cu")) + list((ROOT / "ggml_b200" / "csrc").rglob("*.cuh")) + list((ROOT / "ggml_b200" / "csrc").rglob("*.cpp")):
        assert "oracle/" not in src.read_text() and "quants_oracle" not in src.read_text(), f"{src} references the oracle"
    for so in (ggml_b200.KERNELS_SO, ggml_b200.BACKEND_SO):
        if so.exists():
            needed = subprocess.run(["readelf", "-d", str(so)], capture_output=True, text=True).stdout
            assert "oracle" not in needed and "probe" not in needed, needed


# The plug-in's reference arms (no fusion, no CUDA graphs, the graph-update limit, the host-time profile), the generic-kernel arm, the
# shared-memory consume arm of the n = 1 mat-vec and the opt-in grouped MUL_MAT_ID.  Everything else is planned from a call's arguments.
PRODUCT_ENV = {"GGML_B200_DISABLE_FUSION", "GGML_B200_DISABLE_GRAPHS", "GGML_B200_GRAPH_MAX_UPDATES", "GGML_B200_PROFILE",
               "GGML_B200_FORCE_GENERIC", "GGML_B200_SB_ACT_REGS", "GGML_B200_MMID_GROUPED"}


def test_product_reads_only_the_documented_environment():
    csrc = ROOT / "ggml_b200" / "csrc"
    read = set()
    for src in csrc.rglob("*"):
        if src.suffix in (".cu", ".cuh", ".h", ".cpp"):
            read |= set(re.findall(r'getenv\(\s*"(GGML_B200_[A-Z0-9_]+)"', src.read_text()))
    assert read == PRODUCT_ENV, (sorted(read - PRODUCT_ENV), sorted(PRODUCT_ENV - read))
    doc = next(par for par in (ROOT / "INTEGRATION.md").read_text().split("\n\n") if par.startswith("Environment variables"))
    assert set(re.findall(r"`(GGML_B200_[A-Z0-9_]+)`", doc)) == PRODUCT_ENV


def test_missing_library_fails_loudly(tmp_path, monkeypatch):
    import ggml_b200
    monkeypatch.setattr(ggml_b200, "_lib", None)
    monkeypatch.setattr(ggml_b200, "KERNELS_SO", tmp_path / "nope.so")
    with pytest.raises(ggml_b200.B200Error):
        ggml_b200.lib()
