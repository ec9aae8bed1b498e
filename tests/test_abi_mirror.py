"""The ctypes mirror of include/ggml-b200.h in ggml_b200/__init__.py, checked against the header with the host C compiler: no built
kernel library and no GPU.

Signatures: every GGML_B200_API prototype (prototypes may span lines) is compiled into a stub library, which ggml_b200.lib() loads; each
of its functions must come out declared with the restype and argtypes its C types map to, and ggml_b200.SIGNATURES must name no function
the header does not declare.  Layouts and constants: a C probe of the header prints the size of each ABI struct and the offset and size
of each of its mirror's fields, and the type ids, GGML_B200_MM_* flags and GGML_B200_UNARY_* codes; they must equal the mirror's."""
from __future__ import annotations

import ctypes as C
import re
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

import ggml_b200 as g  # noqa: E402

HEADER = ROOT / "include" / "ggml-b200.h"
STRUCTS = {"ggml_b200_mul_mat_args": g.MulMatArgs, "ggml_b200_mul_mat_id_args": g.MulMatIdArgs, "ggml_b200_gather": g.Gather,
           "ggml_b200_epilogue": g.Epilogue, "ggml_b200_tensor": g.TensorDesc, "ggml_b200_rope_params": g.RopeParams,
           "ggml_b200_im2col_params": g.Im2colParams, "ggml_b200_pool_params": g.PoolParams}
SCALARS = {"int": C.c_int, "int32_t": C.c_int32, "uint32_t": C.c_uint32, "int64_t": C.c_int64, "uint64_t": C.c_uint64,
           "size_t": C.c_size_t, "float": C.c_float}


def header_code() -> str:
    """the header without comments and preprocessor lines"""
    text = re.sub(r"/\*.*?\*/|//[^\n]*", " ", HEADER.read_text(), flags=re.S)
    return re.sub(r"^\s*#.*$", "", text, flags=re.M)


def prototypes() -> dict[str, tuple[str, list[str]]]:
    """name -> (return type, parameter declarations) of every GGML_B200_API function"""
    out = {}
    for decl, params in re.findall(r"GGML_B200_API\s+([^;()]+?)\s*\(([^)]*)\)\s*;", header_code()):
        ret, name = re.fullmatch(r"(.*?)\s*\b(\w+)", decl).groups()
        params = " ".join(params.split())
        out[name] = (ret, [] if params == "void" else [p.strip() for p in params.split(",")])
    return out


def ctype(c_type: str):
    """the ctypes type a C type is mirrored as"""
    words = re.findall(r"\w+|\*", c_type)
    stars = words.count("*")
    (base,) = [w for w in words if w not in ("const", "*")]
    if stars == 0:
        return None if base == "void" else SCALARS[base]
    if stars > 1:
        return C.POINTER(C.c_void_p)
    if base in STRUCTS:
        return C.POINTER(STRUCTS[base])
    return C.c_char_p if base == "char" else C.c_void_p


def param_type(param: str) -> str:
    """the C type of a parameter declaration (its name removed)"""
    return re.fullmatch(r"(.*?)\s*\b\w+", param).group(1)


def compile_c(tmp: Path, name: str, lines: list[str], shared: bool) -> Path:
    src, out = tmp / f"{name}.c", tmp / (f"lib{name}.so" if shared else name)
    src.write_text("\n".join(lines) + "\n")
    cmd = ["gcc", "-std=c11", "-Wall", "-Werror", f"-I{HEADER.parent}", *(["-shared", "-fPIC"] if shared else []), "-o", str(out), str(src)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return out


def test_every_header_function_is_declared(tmp_path, monkeypatch):
    protos = prototypes()
    stub = [f'#include "{HEADER.name}"']
    stub += [f"{ret} {name}({', '.join(params) or 'void'}) {{ {'return 0; ' if ret != 'void' else ''}}}"
             for name, (ret, params) in protos.items()]
    monkeypatch.setattr(g, "_lib", None)
    monkeypatch.setattr(g, "KERNELS_SO", compile_c(tmp_path, "stub", stub, shared=True))
    L = g.lib()
    undeclared, wrong = [], []
    for name, (ret, params) in protos.items():
        fn = getattr(L, name)
        want = [ctype(ret)] + [ctype(param_type(p)) for p in params]
        if fn.argtypes is None:
            undeclared.append(name)
        elif [fn.restype, *fn.argtypes] != want:
            wrong.append((name, [getattr(t, "__name__", t) for t in (fn.restype, *fn.argtypes)], [getattr(t, "__name__", t) for t in want]))
    assert not undeclared, f"{len(undeclared)} of the header's {len(protos)} functions are left without argtypes: {undeclared}"
    assert not wrong, f"signatures that differ from the header (name, declared, header): {wrong}"
    assert sorted(set(g.SIGNATURES) - set(protos)) == [], "signatures of functions the header does not declare"


@pytest.fixture(scope="module")
def probe(tmp_path_factory) -> dict[str, tuple[int, ...]]:
    """what the C compiler makes of the header: 'struct' -> (sizeof,), 'struct.field' -> (offsetof, sizeof), 'ENUMERATOR' -> (value,)"""
    lines = ["#include <stddef.h>", "#include <stdio.h>", f'#include "{HEADER.name}"', "int main(void) {"]
    for cname, mirror in STRUCTS.items():
        lines.append(f'    printf("{cname} %zu\\n", sizeof({cname}));')
        for field, *_ in mirror._fields_:
            lines.append(f'    printf("{cname}.{field} %zu %zu\\n", offsetof({cname}, {field}), sizeof((({cname} *) 0)->{field}));')
    for e in enumerators():
        lines.append(f'    printf("{e} %lld\\n", (long long) {e});')
    lines += ["    return 0;", "}"]
    exe = compile_c(tmp_path_factory.mktemp("probe"), "probe", lines, shared=False)
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout
    return {key: tuple(int(v) for v in values) for key, *values in (line.split() for line in out.splitlines())}


def enumerators() -> list[str]:
    return re.findall(r"\b(GGML_B200_(?:TYPE|MM|UNARY)_\w+)\s*=", header_code())


def test_struct_layouts_match_the_header(probe):
    assert sorted(re.findall(r"typedef\s+struct\s+(\w+)", header_code())) == sorted(STRUCTS), "a struct of the header without a mirror"
    bad = []
    for cname, mirror in STRUCTS.items():
        if probe[cname] != (C.sizeof(mirror),):
            bad.append((cname, "sizeof", probe[cname], C.sizeof(mirror)))
        for field, *_ in mirror._fields_:
            f = getattr(mirror, field)
            if probe[f"{cname}.{field}"] != (f.offset, f.size):
                bad.append((cname, field, probe[f"{cname}.{field}"], (f.offset, f.size)))
    assert not bad, f"(struct, field, header's offset and size, mirror's): {bad}"


def test_constants_match_the_header(probe):
    # GGML_B200_TYPE_Q4_K -> Q4_K, GGML_B200_MM_FORCE_GEMV -> MM_GEMV, GGML_B200_UNARY_SIN -> UNARY_SIN
    header = {e.removeprefix("GGML_B200_").removeprefix("TYPE_").replace("MM_FORCE_", "MM_"): probe[e][0] for e in enumerators()}
    missing = [n for n in header if not n.startswith("UNARY_") and not hasattr(g, n)]
    assert not missing, f"type ids and flags of the header the module does not mirror: {missing}"
    unknown = [n for n in dir(g) if n.startswith(("MM_", "UNARY_")) and n not in header]
    assert not unknown, f"module constants the header does not define: {unknown}"
    differ = {n: (getattr(g, n), v) for n, v in header.items() if hasattr(g, n) and getattr(g, n) != v}
    assert not differ, f"(module, header) values: {differ}"
    assert {header[name.upper()]: name for name in g.TYPE_NAMES.values()} == g.TYPE_NAMES
