"""Build the in-tree native libraries of ggml_b200 with nvcc for sm_90a (H100).

  libggml-b200-kernels.so  the extern "C" kernel-launch shim (include/ggml-b200.h, layer 1); depends only on
                           the CUDA runtime (linked statically) — always buildable, cross-compiles without a GPU.
  libggml-b200.so          the ggml backend plug-in (layer 2).  It implements the reference's own SPI
                           (src/ggml-backend-impl.h) and is therefore compiled against the reference's headers,
                           exactly as a src/ggml-b200/ directory inside the ggml tree would be.
Where the ggml tree itself is absent, build_all(staged=DIR) takes the build inputs derived from it from DIR: DIR/ggml-src
(a copy of its include/ and src/ headers) and DIR/iq_grids.h (the extracted i-quant codebooks).
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from pathlib import Path

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
ROOT = PKG.parent
REF = Path(os.environ.get("GGML_REFERENCE_DIR", "/root/reference"))

KERNEL_SRCS = ["api.cu", "mmvq.cu", "mmvq_sb.cu", "mmvq_mma.cu", "dequant.cu", "mmid.cu", "mmq_tc2.cu", "ops.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC,-fvisibility=hidden", "--threads", "8"]

KERNELS_SO = PKG / "libggml-b200-kernels.so"
BACKEND_SO = PKG / "libggml-b200.so"


def _newer(target: Path, deps) -> bool:
    if not target.exists():
        return False
    t = target.stat().st_mtime
    return all(Path(d).stat().st_mtime <= t for d in deps if Path(d).exists())


def _nvcc() -> str:
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (Path(c).exists() or c == "nvcc"):
            return c
    raise RuntimeError("nvcc not found")


def generate_iq_grids(staged: Path | None = None) -> Path:
    """csrc/generated/iq_grids.h: the i-quant codebooks (file-format data) extracted from the reference's src/ggml-common.h; git-ignored.
    Regenerated whenever the reference tree is present, else copied from staged/iq_grids.h."""
    out = CSRC / "generated" / "iq_grids.h"
    common = REF / "src" / "ggml-common.h"
    script = ROOT / "scripts" / "extract_iq_grids.py"
    staged = Path(staged or ROOT) / "iq_grids.h"
    if common.exists():
        if not out.exists() or out.stat().st_mtime < max(common.stat().st_mtime, script.stat().st_mtime):
            out.parent.mkdir(exist_ok=True)
            subprocess.run([sys.executable, str(script), str(common), str(out)], check=True)
    elif staged.exists():
        if not out.exists() or out.read_bytes() != staged.read_bytes():
            out.parent.mkdir(exist_ok=True)
            shutil.copyfile(staged, out)
    elif not out.exists():
        raise RuntimeError(f"{out} is missing and neither {common} nor {staged} is available to generate it from")
    return out


def build_kernels(force: bool = False, verbose: bool = False, staged: Path | None = None) -> Path:
    generate_iq_grids(staged)
    srcs = [CSRC / s for s in KERNEL_SRCS if (CSRC / s).exists()]
    deps = srcs + list(CSRC.glob("*.cuh")) + list(CSRC.glob("*.h")) + list((CSRC / "generated").glob("*.h")) + [ROOT / "include" / "ggml-b200.h"]
    if not force and _newer(KERNELS_SO, deps):
        return KERNELS_SO
    objs = []
    procs = []
    (PKG / "build").mkdir(exist_ok=True)
    for s in srcs:
        o = PKG / "build" / (s.stem + ".o")
        objs.append(o)
        if not force and _newer(o, deps):
            continue
        cmd = [_nvcc()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", str(s), "-o", str(o)]
        procs.append((cmd, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for cmd, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError("nvcc failed: " + " ".join(cmd) + "\n" + out)
        if verbose:
            sys.stderr.write(out)
    cmd = [_nvcc(), "-shared", "-o", str(KERNELS_SO)] + [str(o) for o in objs] + ["-gencode", "arch=compute_90a,code=sm_90a"]
    subprocess.run(cmd, check=True)
    return KERNELS_SO


def build_backend(force: bool = False, staged: Path | None = None) -> Path | None:
    src = CSRC / "backend" / "ggml-b200.cpp"
    if not src.exists():
        return None
    cands = [REF] + ([Path(staged) / "ggml-src"] if staged else [])
    ggml = next((d for d in cands if (d / "src" / "ggml-backend-impl.h").exists()), None)
    if ggml is None:
        raise RuntimeError(f"the ggml headers are not available to build {BACKEND_SO} (looked in {', '.join(map(str, cands))})")
    deps = [src, ROOT / "include" / "ggml-b200.h", ROOT / "include" / "ggml-b200-backend.h", CSRC / "b200_op_checks.h", KERNELS_SO]
    if not force and _newer(BACKEND_SO, deps):
        return BACKEND_SO
    cmd = [_nvcc(), "-O2", "-std=c++17", "-Xcompiler", "-fPIC,-fvisibility=hidden", "-shared",
           "-DGGML_BACKEND_DL", "-DGGML_BACKEND_SHARED", "-DGGML_BACKEND_BUILD", "-DGGML_SHARED",
           f"-I{ggml}/include", f"-I{ggml}/src", f"-I{ROOT}/include", f"-I{CSRC}",
           "-o", str(BACKEND_SO), str(src),
           f"-L{PKG}", "-lggml-b200-kernels", "-Xlinker", "-rpath,$ORIGIN"]
    subprocess.run(cmd, check=True)
    return BACKEND_SO


def build_all(force: bool = False, verbose: bool = False, staged: Path | None = None):
    k = build_kernels(force=force, verbose=verbose, staged=staged)
    b = build_backend(force=force, staged=staged)
    return k, b


if __name__ == "__main__":
    print(build_all(force="--force" in sys.argv, verbose="-v" in sys.argv))
