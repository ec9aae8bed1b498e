"""TEST INFRASTRUCTURE ONLY: what the ctypes fronts of the one-node op probes (oracle/{attn,conv,core,moe,pool,rope,sam,ssm,train,wkv}.py over
oracle/_ref/libggml_<family>_probe.so) share: loading a family's library with its signatures, and turning a probe's code into a result."""
from __future__ import annotations

import ctypes as C

from . import oracle as O

_libs = {}


def probe_lib(family: str, make_hint: str, signatures: dict) -> C.CDLL:
    """oracle/_ref/libggml_<family>_probe.so, loaded once, every symbol of `signatures` ({name: argtypes}) returning a C int.  make_hint:
    the command that builds the library, for the error raised when it is missing"""
    L = _libs.get(family)
    if L is None:
        O.Ref()                                            # loads the reference libraries (and the shared backend registry) globally
        so = O.REF_DIR / f"libggml_{family}_probe.so"
        if not so.exists():
            raise RuntimeError(f"{so} missing ({make_hint} where the reference tree exists)")
        L = C.CDLL(str(so))
        for name, args in signatures.items():
            fn = getattr(L, name)
            fn.restype, fn.argtypes = C.c_int, args
        _libs[family] = L
    return L


def result(rc: int, raw: bool, what: str, value):
    """the probe's code when raw, else value (raising when the probe failed)"""
    if raw:
        return rc
    if rc != 0:
        raise RuntimeError(f"{what} returned {rc}")
    return value


def ptrs(arrays) -> C.Array:
    """the data pointers of numpy arrays, as the `const void * const *` a probe takes"""
    return (C.c_void_p * len(arrays))(*[a.ctypes.data for a in arrays])
