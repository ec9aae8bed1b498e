"""Builds and loads the host-compiled kernel libraries of tests/hostemu, and holds the helpers their tests share.

load("pool_emu") compiles tests/hostemu/pool_emu.cpp into _build/libpool_emu.so with the one flag set below and returns it through
ctypes.  The library is rebuilt when it, its depfile or its recorded command is missing, when the command changed, or when any file the
compiler named in the depfile (the source, the shim, every product header it reaches) is newer than it: editing a header can never leave a
test running against the old code."""
import ctypes as C
import re
import subprocess
from pathlib import Path

import numpy as np

import ggml_b200 as g
from oracle.pool import BF16, F16, F32, I16, I32

HERE = Path(__file__).resolve().parent
BUILD = HERE / "_build"
# -fno-strict-aliasing: the decoders read words through pointer casts as the device code does (b200_tc_dequant.cuh), which -O2 would
# otherwise assume never alias
FLAGS = ["-std=c++17", "-O2", "-fPIC", "-shared", "-pthread", "-mf16c", "-mavx", "-ffp-contract=off", "-fno-strict-aliasing",
         "-Wall", "-Werror", "-Wno-unknown-pragmas", f"-I{HERE / 'shim'}"]

OK, EUNSUPPORTED, EINVAL = 0, -1, -2              # GGML_B200_OK, GGML_B200_EUNSUPPORTED, GGML_B200_EINVAL
I64 = 27
# type -> (elements per block, bytes per block) of the types the tests describe
BLOCK = {F32: (1, 4), F16: (1, 2), BF16: (1, 2), I16: (1, 2), I32: (1, 4), I64: (1, 8), g.Q8_0: (32, 34), g.Q4_K: (256, 144)}


def depfile_inputs(dep: Path) -> list[Path]:
    """the prerequisites of the make rule -MMD wrote (a backslash-escaped space belongs to its path)"""
    rule = dep.read_text().replace("\\\n", " ").split(":", 1)[1]
    return [Path(p.replace("\\ ", " ")) for p in re.split(r"(?<!\\)\s+", rule.strip()) if p]


def build(src: Path, out: Path = BUILD) -> Path:
    """src compiled into out/lib<stem>.so unless that library is up to date; a failed compile fails the caller with g++'s stderr"""
    out.mkdir(parents=True, exist_ok=True)
    so, dep, rec = out / f"lib{src.stem}.so", out / f"{src.stem}.d", out / f"{src.stem}.cmd"
    cmd = ["g++", *FLAGS, "-MMD", "-MF", str(dep), "-o", str(so), str(src)]
    if so.exists() and dep.exists() and rec.exists() and rec.read_text() == " ".join(cmd):
        built = so.stat().st_mtime_ns
        if all(p.exists() and p.stat().st_mtime_ns <= built for p in depfile_inputs(dep)):
            return so
    rec.unlink(missing_ok=True)                   # until this compile succeeds, the library is not up to date
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    rec.write_text(" ".join(cmd))
    return so


def load(name: str) -> C.CDLL:
    """tests/hostemu/<name>.cpp, built if needed; each call returns a new ctypes object, so the signatures one test module sets do not
    reach another"""
    return C.CDLL(str(build(HERE / f"{name}.cpp")))


def desc(type_, ne, nb=None, data=4096) -> g.TensorDesc:
    """a ggml tensor descriptor: ne in ggml order, nb in bytes (packed when None)"""
    d = g.TensorDesc()
    d.data, d.type = data, type_
    ne = tuple(ne) + (1,) * (4 - len(ne))
    if nb is None:
        blk, bs = BLOCK[type_]
        nb = [bs, bs * ne[0] // blk]
        for i in range(2, 4):
            nb.append(nb[-1] * ne[i - 1])
    for i in range(4):
        d.ne[i], d.nb[i] = ne[i], nb[i]
    return d


def view_desc(src, parent: np.ndarray) -> g.TensorDesc:
    """the descriptor through which a node reads an oracle.pool.Source of the host array parent"""
    ne, nb = src.view()
    return desc(src.type, ne, nb, parent.ctypes.data + src.offs)


def bits(a: np.ndarray) -> np.ndarray:
    """the raw words of a 4- or 2-byte array"""
    return np.ascontiguousarray(a).view(np.uint32 if a.itemsize == 4 else np.uint16)
