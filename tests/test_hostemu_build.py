"""CPU-only: how tests/hostemu/emu.py builds the host-compiled libraries.
  * a library is rebuilt when any header it reaches changes, however deeply that header is included, and only then;
  * every public check_<op> of ggml_b200/csrc/b200_op_checks.h is exported as emu_check_<op> by op_checks_emu.cpp."""
import os
import re
from pathlib import Path

from hostemu import emu

ROOT = Path(__file__).resolve().parents[1]


def test_a_nested_header_change_rebuilds_the_library(tmp_path):
    (tmp_path / "inner.h").write_text("#pragma once\ninline int inner() { return 7; }\n")
    (tmp_path / "outer.h").write_text('#pragma once\n#include "inner.h"\n')
    src = tmp_path / "nested.cpp"
    src.write_text('#include "outer.h"\nextern "C" int nested() { return inner(); }\n')
    out = tmp_path / "_build"
    so = emu.build(src, out)
    past = so.stat().st_mtime_ns - 100_000_000_000                 # every input 200 s old, the library 100 s old
    for p in tmp_path.iterdir():
        if p.is_file():
            os.utime(p, ns=(past - 100_000_000_000,) * 2)
    os.utime(so, ns=(past, past))

    assert emu.build(src, out) == so and so.stat().st_mtime_ns == past       # nothing changed: not rebuilt
    os.utime(tmp_path / "inner.h", ns=(past + 50_000_000_000,) * 2)
    emu.build(src, out)
    assert so.stat().st_mtime_ns > past                                      # the header two includes down is newer: rebuilt


def test_every_check_is_exported():
    header = (ROOT / "ggml_b200" / "csrc" / "b200_op_checks.h").read_text()
    ops = set(re.findall(r"\bop_check check_(\w+)\(", header)) - {"wkv_common"}
    assert len(ops) >= 34
    checks = emu.load("op_checks_emu")
    assert [op for op in sorted(ops) if not hasattr(checks, f"emu_check_{op}")] == []
