"""TEST INFRASTRUCTURE ONLY: GGML_OP_OUT_PROD, GGML_OP_CROSS_ENTROPY_LOSS, GGML_OP_CROSS_ENTROPY_LOSS_BACK, GGML_OP_OPT_STEP_ADAMW,
GGML_OP_ARGMAX, GGML_OP_COUNT_EQUAL, GGML_OP_SUM, GGML_OP_REPEAT_BACK and STEP through oracle/_ref/libggml_train_probe.so
(oracle/train_probe.cpp), on a named ggml device ("CPU": ggml-cpu; "B2000": the plug-in, once loaded with oracle.Ref().load_backend).

Arrays are numpy, ggml dims reversed (the last numpy axis is ggml's dim 0).  Sources that are views (OUT_PROD's src1, SUM's and
REPEAT_BACK's src) are oracle/pool.py's `Source`; `parent` is then the parent's data."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import oracle as O
from .pool import Source, _result

_lib = None


def _probe_lib():
    global _lib
    if _lib is None:
        O.Ref()                                            # loads the reference libraries (and the shared backend registry) globally
        so = O.REF_DIR / "libggml_train_probe.so"
        if not so.exists():
            raise RuntimeError(f"{so} missing (make -C oracle -f train.mk train where the reference tree exists)")
        L = C.CDLL(str(so))
        vp, i64 = C.c_void_p, C.c_int64
        for name, args in (("probe_out_prod", [C.c_char_p] + [vp] * 5), ("probe_cross_entropy_loss", [C.c_char_p] + [vp] * 4),
                           ("probe_cross_entropy_loss_back", [C.c_char_p] + [vp] * 5), ("probe_opt_step_adamw", [C.c_char_p] + [vp] * 9),
                           ("probe_argmax", [C.c_char_p, i64, i64, vp, vp]), ("probe_count_equal", [C.c_char_p] + [vp] * 4),
                           ("probe_sum", [C.c_char_p] + [vp] * 3), ("probe_repeat_back", [C.c_char_p] + [vp] * 4),
                           ("probe_step", [C.c_char_p] + [vp] * 3)):
            fn = getattr(L, name)
            fn.restype, fn.argtypes = C.c_int, args
        _lib = L
    return _lib


def _ne(a: np.ndarray) -> np.ndarray:
    return np.array(list(a.shape[::-1]) + [1] * (4 - a.ndim), dtype=np.int64)


def out_prod(dev: str, sa: Source, sb: Source, a: np.ndarray, b: np.ndarray, raw: bool = False):
    """OUT_PROD of two sources (parents a, b): f32 [ne3, ne2, ne1, ne0]"""
    na, _ = sa.view()
    nbv, _ = sb.view()
    out = np.zeros((nbv[3], nbv[2], nbv[0], na[0]), dtype=np.float32)
    spa, spb = sa.spec(), sb.spec()
    rc = _probe_lib().probe_out_prod(dev.encode(), spa.ctypes.data, spb.ctypes.data, a.ctypes.data, b.ctypes.data, out.ctypes.data)
    return _result(rc, raw, f"probe_out_prod({dev})", out)


def cross_entropy_loss(dev: str, x: np.ndarray, l: np.ndarray, raw: bool = False):
    out = np.zeros(1, dtype=np.float32)
    ne = _ne(x)
    rc = _probe_lib().probe_cross_entropy_loss(dev.encode(), ne.ctypes.data, x.ctypes.data, l.ctypes.data, out.ctypes.data)
    return _result(rc, raw, f"probe_cross_entropy_loss({dev})", out[0])


def cross_entropy_loss_back(dev: str, grad: float, x: np.ndarray, l: np.ndarray, raw: bool = False):
    out = np.zeros_like(x)
    ne, g = _ne(x), np.array([grad], dtype=np.float32)
    rc = _probe_lib().probe_cross_entropy_loss_back(dev.encode(), ne.ctypes.data, g.ctypes.data, x.ctypes.data, l.ctypes.data, out.ctypes.data)
    return _result(rc, raw, f"probe_cross_entropy_loss_back({dev})", out)


def opt_step_adamw(dev: str, w, g, m, v, params, raw: bool = False):
    """one AdamW step: (w, m, v) after it"""
    ow, om, ov = np.zeros_like(w), np.zeros_like(m), np.zeros_like(v)
    ne, p = _ne(w), np.ascontiguousarray(params, dtype=np.float32)
    rc = _probe_lib().probe_opt_step_adamw(dev.encode(), ne.ctypes.data, w.ctypes.data, g.ctypes.data, m.ctypes.data, v.ctypes.data, p.ctypes.data,
                                           ow.ctypes.data, om.ctypes.data, ov.ctypes.data)
    return _result(rc, raw, f"probe_opt_step_adamw({dev})", (ow, om, ov))


def argmax(dev: str, x: np.ndarray, raw: bool = False):
    """x f32 [ne1, ne0] -> i32 [ne1]"""
    out = np.zeros(x.shape[0], dtype=np.int32)
    rc = _probe_lib().probe_argmax(dev.encode(), x.shape[1], x.shape[0], x.ctypes.data, out.ctypes.data)
    return _result(rc, raw, f"probe_argmax({dev})", out)


def count_equal(dev: str, a: np.ndarray, b: np.ndarray, raw: bool = False):
    out = np.zeros(1, dtype=np.int64)
    ne = _ne(a)
    rc = _probe_lib().probe_count_equal(dev.encode(), ne.ctypes.data, a.ctypes.data, b.ctypes.data, out.ctypes.data)
    return _result(rc, raw, f"probe_count_equal({dev})", int(out[0]))


def sum_(dev: str, src: Source, parent: np.ndarray, raw: bool = False):
    out = np.zeros(1, dtype=np.float32)
    spec = src.spec()
    rc = _probe_lib().probe_sum(dev.encode(), spec.ctypes.data, parent.ctypes.data, out.ctypes.data)
    return _result(rc, raw, f"probe_sum({dev})", out[0])


def repeat_back(dev: str, src: Source, ne_dst, parent: np.ndarray, raw: bool = False):
    """REPEAT_BACK of a source into extents ne_dst (ggml order): f32, ggml dims reversed"""
    ne = np.array(list(ne_dst) + [1] * (4 - len(ne_dst)), dtype=np.int64)
    out = np.zeros(ne[::-1], dtype=np.float32)
    spec = src.spec()
    rc = _probe_lib().probe_repeat_back(dev.encode(), spec.ctypes.data, ne.ctypes.data, parent.ctypes.data, out.ctypes.data)
    return _result(rc, raw, f"probe_repeat_back({dev})", out)


def step(dev: str, x: np.ndarray, raw: bool = False):
    out = np.zeros_like(x)
    ne = _ne(x)
    rc = _probe_lib().probe_step(dev.encode(), ne.ctypes.data, x.ctypes.data, out.ctypes.data)
    return _result(rc, raw, f"probe_step({dev})", out)
