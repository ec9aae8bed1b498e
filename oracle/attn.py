"""TEST INFRASTRUCTURE ONLY: GGML_OP_FLASH_ATTN_EXT, GGML_OP_SOFT_MAX and GGML_OP_CPY (f32 into a KV cache) cases, their f64 references, and
the reference's ops through oracle/_ref/libggml_attn_probe.so (oracle/attn_probe.cpp).

`FaCase` is one attention node laid out as a llama graph lays it out: K and V are views of [D n_head_kv, n_ctx] caches of any type (nb1 =
a whole cache row, nb2 = one head), Q optionally permuted from [D, n_head, n_q, ne3].  `SoftMaxCase` is one ggml_soft_max_ext node, `CpyCase`
one ggml_cpy of an f32 source (any row layout) into a view of a cache at an offset.  `*_reference` compute the ops in f64 on exactly the
values the node reads (K / V through the bit-exact `Oracle.dequantize`).  `flash_attn_ext(dev, case)` etc. evaluate on a named ggml device
("CPU": ggml-cpu; "B2000": the plug-in, once loaded with oracle.Ref().load_backend)."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

from . import oracle as O
from .pool import F16, F32, Source
from .probe import probe_lib, result

KQ_MASK_PAD = 64                          # GGML_KQ_MASK_PAD: the rows of an attention mask are padded to a multiple of it
BLOCK_TYPES_32 = (O.Q4_0, O.Q4_1, O.Q5_0, O.Q5_1, O.Q8_0, O.IQ4_NL)
BLOCK_TYPES_256 = (O.Q2_K, O.Q3_K, O.Q4_K, O.Q5_K, O.Q6_K, O.IQ4_XS, O.IQ2_XXS, O.IQ2_XS, O.IQ2_S, O.IQ3_XXS, O.IQ3_S, O.IQ1_S, O.IQ1_M,
                   O.TQ1_0, O.TQ2_0)
_orc = None


def orc() -> O.Oracle:
    global _orc
    if _orc is None:
        _orc = O.Oracle()
    return _orc


def pad(n, m):
    return -(-n // m) * m


def row_bytes(t, n):
    return n * 4 if t == F32 else n * 2 if t == F16 else orc().row_size(t, n)


def alibi_slopes(n_head: int, max_bias: float) -> np.ndarray:
    """ggml's ALiBi slope of each head (f64): m0^(h + 1) for the first n_head_log2 heads, then m1^(2 (h - n_head_log2) + 1), n_head_log2 the
    largest power of two <= n_head; all 1 when max_bias is 0"""
    if max_bias <= 0.0:
        return np.ones(n_head)
    nl2 = 1 << int(np.floor(np.log2(n_head)))
    m0, m1 = 2.0 ** (-max_bias / nl2), 2.0 ** (-(max_bias / 2.0) / nl2)
    h = np.arange(n_head)
    return np.where(h < nl2, m0 ** (h + 1.0), m1 ** (2.0 * (h - nl2) + 1.0))


def _softmax_rows(s):
    s = s - s.max(axis=-1, keepdims=True)
    p = np.exp(s)
    return p / p.sum(axis=-1, keepdims=True)


# ------------------------------------------------------------------ FLASH_ATTN_EXT
@dataclass
class FaCase:
    D: int
    n_kv: int
    n_q: int
    n_head: int
    n_head_kv: int
    kt: int
    vt: int
    ne3: int = 1                   # Q's batches; K and V have one, broadcast over them
    mask: str = "none"             # "none", "causal" (-inf after the query's position) or "finite" (-|i - j|, and -inf at some j)
    max_bias: float = 0.0
    softcap: float = 0.0
    permute_q: bool = False
    extra_ctx: int = 3             # cache rows past n_kv, never read
    seed: int = 0

    def __post_init__(self):
        assert self.max_bias == 0.0 or self.mask != "none", "ALiBi needs a mask"

    @property
    def n_ctx(self):
        return self.n_kv + self.extra_ctx

    def q_source(self) -> Source:
        ne = (self.D, self.n_head, self.n_q, self.ne3) if self.permute_q else (self.D, self.n_q, self.n_head, self.ne3)
        return Source(F32, ne)

    def kv_source(self, t) -> Source:
        """a [D, n_kv, n_head_kv] view of the [D n_head_kv, n_ctx] cache"""
        nb1 = row_bytes(t, self.D * self.n_head_kv)
        return Source(t, (self.D, self.n_kv, self.n_head_kv, 1), parent_ne=(self.D * self.n_head_kv, self.n_ctx, 1, 1),
                      nb=(nb1, row_bytes(t, self.D), nb1 * self.n_ctx))

    def __str__(self):
        t = O.TYPE_NAMES
        return (f"fa D={self.D} kv={self.n_kv} q={self.n_q} h={self.n_head}:{self.n_head_kv} {t[self.kt]}/{t[self.vt]} ne3={self.ne3} "
                f"mask={self.mask}{f' alibi={self.max_bias:g}' if self.max_bias else ''}{f' softcap={self.softcap:g}' if self.softcap else ''}"
                f"{' permuted-q' if self.permute_q else ''}")


@dataclass
class FaData:
    q_parent: np.ndarray           # f32, the parent Q's view reads (numpy order of q_source().ne)
    k_cache: np.ndarray            # uint8, the whole K cache
    v_cache: np.ndarray
    mask: np.ndarray | None        # f16 [pad(n_q, KQ_MASK_PAD), n_kv]
    scale: float
    q: np.ndarray                  # f64 [ne3, n_head, n_q, D]: what the node reads as Q
    k: np.ndarray                  # f64 [n_head_kv, n_kv, D]: the K / V values the view reads, dequantized
    v: np.ndarray


def _cache(t, case: FaCase, rng):
    """(cache bytes, its values f64 [n_head_kv, n_kv, D] as the view reads them)"""
    n = case.n_ctx * case.D * case.n_head_kv
    if t in (F32, F16):
        x = rng.standard_normal(n).astype(np.float32 if t == F32 else np.float16)
        raw, vals = x.view(np.uint8), x.astype(np.float64)
    else:
        raw = O.random_blocks(t, n // orc().blck_size(t), rng)
        vals = orc().dequantize(t, raw, n).astype(np.float64)
    return raw, vals.reshape(case.n_ctx, case.n_head_kv, case.D)[: case.n_kv].transpose(1, 0, 2)


def _scores(q, k):
    """q . k of every (batch, head, query, kv position), f64 [ne3, n_head, n_q, n_kv]: head h reads K head h / (n_head / n_head_kv)"""
    b, h, n, D = q.shape
    hk = k.shape[0]
    return (q.reshape(b, hk, h // hk, n, D) @ k.transpose(0, 2, 1)[None, :, None]).reshape(b, h, n, -1)


def fa_data(case: FaCase) -> FaData:
    rng = np.random.default_rng(7000 + case.seed)
    k_raw, k = _cache(case.kt, case, rng)
    v_raw, v = _cache(case.vt, case, rng)
    qp = rng.standard_normal(case.q_source().ne[::-1]).astype(np.float32)
    q = (qp.transpose(0, 2, 1, 3) if case.permute_q else qp).astype(np.float64)
    # scale: scores of standard deviation 2 (60 under a softcap of 30: most of them saturate tanh), whatever the K format's magnitude
    s = _scores(q, k)
    scale = float(np.float32((60.0 if case.softcap else 2.0) / max(float(np.std(s)), 1e-30)))
    mask = None
    if case.mask != "none":
        rows = pad(case.n_q, KQ_MASK_PAD)
        pos = np.maximum(case.n_kv - case.n_q + np.arange(rows), 0)[:, None]      # query i sits at position pos[i]; row 0's pos >= 0
        j = np.arange(case.n_kv)[None, :]
        if case.mask == "causal":
            m = np.where(j > pos, -np.inf, 0.0)
        else:
            m = -np.abs(pos - j).astype(np.float64)
            m = np.where((j % 7 == 3) & (j != np.minimum(pos, case.n_kv - 1)), -np.inf, m)
        m[case.n_q:] = 0.0                                                      # the padding rows are never read
        mask = m.astype(np.float16)
    return FaData(qp, k_raw, v_raw, mask, scale, q, k, v)


def flash_attn_reference(case: FaCase, d: FaData) -> np.ndarray:
    """f64 FLASH_ATTN_EXT: per (batch, head, query) softmax(softcap tanh(scale q.k / softcap) (or scale q.k) + slope mask) . V over the
    head's K / V (head h reads K head h / (n_head / n_head_kv), every batch the one K), returned in ggml's [D, n_head, n_q, ne3] as numpy
    [ne3, n_q, n_head, D]"""
    s = _scores(d.q, d.k) * d.scale
    if case.softcap:
        s = case.softcap * np.tanh(s / case.softcap)
    if d.mask is not None:
        m = d.mask[: case.n_q, : case.n_kv].astype(np.float64)
        with np.errstate(invalid="ignore"):
            s = s + alibi_slopes(case.n_head, case.max_bias)[None, :, None, None] * m[None, None]
    p = _softmax_rows(s)
    b, h, n, _ = p.shape
    hk = d.v.shape[0]
    out = (p.reshape(b, hk, h // hk, n, -1) @ d.v[None, :, None]).reshape(b, h, n, -1)
    return out.transpose(0, 2, 1, 3)


# ------------------------------------------------------------------ SOFT_MAX
@dataclass
class SoftMaxCase:
    ne: tuple                      # ggml order (ne0, ne1, ne2, ne3)
    mask_type: int | None = None   # None, F16 or F32
    mask_rows: int = 0             # >= ne1 (0: ne1)
    scale: float = 1.0
    max_bias: float = 0.0
    seed: int = 0

    def __str__(self):
        m = "" if self.mask_type is None else f" mask={'f16' if self.mask_type == F16 else 'f32'}x{self.mask_rows or self.ne[1]}"
        return f"soft_max ne={self.ne}{m} scale={self.scale:g}{f' alibi={self.max_bias:g}' if self.max_bias else ''}"


def soft_max_data(case: SoftMaxCase):
    """(x f32 [ne3, ne2, ne1, ne0], mask [rows, ne0] or None): scores of standard deviation 3; a finite mask of -|i - j| / 4 with -inf at
    every fifth element (never element 0, so no row is wholly masked)"""
    rng = np.random.default_rng(8000 + case.seed)
    x = (rng.standard_normal(case.ne[::-1]) * 3.0).astype(np.float32)
    if case.mask_type is None:
        return x, None
    rows = case.mask_rows or case.ne[1]
    i, j = np.arange(rows)[:, None], np.arange(case.ne[0])[None, :]
    m = np.where(j % 5 == 2, -np.inf, -np.abs(i - j) / 4.0)
    return x, m.astype(np.float16 if case.mask_type == F16 else np.float32)


def soft_max_reference(case: SoftMaxCase, x, mask) -> np.ndarray:
    """f64 SOFT_MAX: softmax(x scale + slope(i2) mask[i1]) along ne0, row i1 of every matrix reading mask row i1 (ggml's (i1 % ne01) ne00)"""
    s = x.astype(np.float64) * case.scale
    if mask is not None:
        slopes = alibi_slopes(case.ne[2], case.max_bias)
        s = s + slopes[None, :, None, None] * mask[: case.ne[1]].astype(np.float64)[None, None]
    return _softmax_rows(s)


# ------------------------------------------------------------------ CPY into a cache
@dataclass
class CpyCase:
    src: Source                    # f32
    dst_type: int
    dst_ne: tuple                  # the cache view's ne (ggml order), packed rows; as many elements as src
    cache_rows: int                # the cache parent: [dst_ne[0], cache_rows]
    row_offset: int                # the view starts at this cache row
    values: str = "normal"         # "normal", "golden" (tests/golden/act_q8.npz x), "ties" (half-integers, amax 127), "zeros", "signs"

    def dst_source(self) -> Source:
        rb = row_bytes(self.dst_type, self.dst_ne[0])
        ne = tuple(self.dst_ne) + (1,) * (4 - len(self.dst_ne))
        return Source(self.dst_type, ne, parent_ne=(ne[0], self.cache_rows, 1, 1), nb=(rb, rb * ne[1], rb * ne[1] * ne[2]),
                      offs=rb * self.row_offset)

    def __str__(self):
        return (f"cpy f32 {self.src.ne}/{self.src.parent_ne} -> {O.TYPE_NAMES[self.dst_type]} {self.dst_ne} at row {self.row_offset} "
                f"of {self.cache_rows} ({self.values})")


def cpy_parent(case: CpyCase, golden_x=None) -> np.ndarray:
    """the f32 source parent's values (numpy order of src.parent_ne)"""
    rng = np.random.default_rng(9000 + case.src.seed)
    n = int(np.prod(case.src.parent_ne))
    if case.values == "golden":
        x = np.resize(golden_x, n).astype(np.float32)
    elif case.values == "ties":                     # blocks of 32 whose amax is exactly 127: id = 1, so every half-integer is a tie
        x = (rng.integers(-127, 127, n) + 0.5).astype(np.float32)
        x[::32] = np.where(rng.integers(0, 2, n)[::32] == 0, 127.0, -127.0)
    elif case.values == "zeros":                    # whole blocks of +-0, beside ordinary ones
        x = rng.standard_normal(n).astype(np.float32)
        x[: n // 2] = np.where(np.arange(n // 2) % 2 == 0, 0.0, -0.0)
    elif case.values == "signs":                    # the largest magnitude negative, positive, or both (+amax and -amax in one block)
        x = rng.uniform(-1, 1, n).astype(np.float32)
        b = x.reshape(-1, 32)
        b[0::3, 5] = -2.0
        b[1::3, 9] = 2.0
        b[2::3, 1], b[2::3, 30] = 2.0, -2.0
    else:
        x = rng.standard_normal(n).astype(np.float32)
    return x.reshape(case.src.parent_ne[::-1])


def src_logical(case: CpyCase, parent: np.ndarray) -> np.ndarray:
    """the f32 values the source view reads, in ggml's logical order, flat"""
    ne, nb = case.src.view()
    st = np.lib.stride_tricks.as_strided(parent.reshape(-1)[case.src.offs // 4:], shape=ne[::-1], strides=nb[::-1])
    return np.ascontiguousarray(st).reshape(-1)


def cpy_expected(case: CpyCase, parent: np.ndarray, cache_in: np.ndarray) -> np.ndarray:
    """the cache bytes after the copy: the view's bytes are the logical source quantized as ggml-cpu's CPY does on x86 (Q8_0: the AVX
    quantize_row_q8_0, id = 127 / amax rounded half to even; Q4_0: quantize_row_q4_0_ref; f16: round to nearest even), the rest untouched"""
    x = src_logical(case, parent)
    if case.dst_type == O.Q8_0:
        q = orc().quantize(O.Q8_0, x, simd_q8_0=True)
    elif case.dst_type == O.Q4_0:
        q = orc().quantize(O.Q4_0, x)
    elif case.dst_type == F16:
        q = x.astype(np.float16).view(np.uint8)
    else:
        q = x.view(np.uint8)
    out = cache_in.copy()
    offs = case.dst_source().offs
    out[offs: offs + q.size] = q
    return out


def cache_in(case: CpyCase) -> np.ndarray:
    """the cache's bytes before the copy: random (for f16 / f32 caches: no NaN patterns matter, the bytes are compared raw)"""
    rb = row_bytes(case.dst_type, case.dst_ne[0])
    return np.random.default_rng(9500 + case.src.seed).integers(0, 256, rb * case.cache_rows, dtype=np.uint8)


def cpy_grid():
    """Q8_0 on act_q8.npz's activations, on half-integer ties, on all-zero blocks and on +-amax sign cases; Q4_0 and f16 likewise.  f32
    sources packed, with padded rows, and with permuted rows ([D, n_head, n_tok] read from [D, n_tok, n_head]); destinations: views of
    caches at a row offset"""
    out = []
    for i, (t, values) in enumerate([(O.Q8_0, "golden"), (O.Q8_0, "ties"), (O.Q8_0, "zeros"), (O.Q8_0, "signs"), (O.Q4_0, "ties"),
                                     (O.Q4_0, "signs"), (F16, "normal")]):
        out.append(CpyCase(Source(F32, (256, 12), seed=i), t, (256, 12), 20, 5, values))
        out.append(CpyCase(Source(F32, (128, 6, 1, 1), parent_ne=(160, 7, 1, 1), seed=10 + i), t, (128, 6), 9, 2, values))
        out.append(CpyCase(Source(F32, (64, 4, 3, 1), parent_ne=(64, 3, 4, 1), nb=(64 * 3 * 4, 64 * 4, 64 * 12 * 4), seed=20 + i), t,
                           (256, 3), 8, 4, values))
    return out


# ------------------------------------------------------------------ the probe
SIGNATURES = {
    "probe_flash_attn_ext": [C.c_char_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int64] + [C.c_float] * 3 + [C.c_void_p] * 5,
    "probe_soft_max": [C.c_char_p, C.c_void_p, C.c_int, C.c_int64, C.c_float, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p],
    "probe_cpy": [C.c_char_p] + [C.c_void_p] * 5,
}


def _lib():
    return probe_lib("attn", "make -C oracle -f attn.mk attn", SIGNATURES)


def flash_attn_ext(dev: str, case: FaCase, data: FaData | None = None, raw: bool = False):
    """FLASH_ATTN_EXT of `case` on `dev`: f32 [ne3, n_q, n_head, D]"""
    d = fa_data(case) if data is None else data
    specs = [case.q_source().spec(), case.kv_source(case.kt).spec(), case.kv_source(case.vt).spec()]   # held: read through raw pointers
    out = np.zeros((case.ne3, case.n_q, case.n_head, case.D), dtype=np.float32)
    rows = 0 if d.mask is None else d.mask.shape[0]
    rc = _lib().probe_flash_attn_ext(dev.encode(), specs[0].ctypes.data, int(case.permute_q), specs[1].ctypes.data, specs[2].ctypes.data, rows,
                                     d.scale, case.max_bias, case.softcap, d.q_parent.ctypes.data, d.k_cache.ctypes.data,
                                     d.v_cache.ctypes.data, None if d.mask is None else d.mask.ctypes.data, out.ctypes.data)
    return result(rc, raw, f"probe_flash_attn_ext({dev}, {case})", out)


def soft_max(dev: str, case: SoftMaxCase, data=None, raw: bool = False):
    """SOFT_MAX of `case` on `dev`: f32 [ne3, ne2, ne1, ne0]"""
    x, mask = soft_max_data(case) if data is None else data
    ne = np.array(case.ne, dtype=np.int64)
    out = np.zeros(case.ne[::-1], dtype=np.float32)
    mt = -1 if mask is None else case.mask_type
    rows = 0 if mask is None else mask.shape[0]
    rc = _lib().probe_soft_max(dev.encode(), ne.ctypes.data, mt, rows, case.scale, case.max_bias, x.ctypes.data,
                               None if mask is None else mask.ctypes.data, out.ctypes.data)
    return result(rc, raw, f"probe_soft_max({dev}, {case})", out)


def cpy(dev: str, case: CpyCase, parent: np.ndarray, cache: np.ndarray, raw: bool = False):
    """ggml_cpy of `case` on `dev`: the whole cache's bytes afterwards (uint8)"""
    ss, sd = case.src.spec(), case.dst_source().spec()
    out = np.zeros_like(cache)
    rc = _lib().probe_cpy(dev.encode(), ss.ctypes.data, sd.ctypes.data, parent.ctypes.data, cache.ctypes.data, out.ctypes.data)
    return result(rc, raw, f"probe_cpy({dev}, {case})", out)
