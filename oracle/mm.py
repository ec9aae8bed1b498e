"""oracle/mm.py — f64 reference of MUL_MAT / MUL_MAT_ID over block-quantized weights, with a per-element error bound.

TEST INFRASTRUCTURE ONLY (tests/test_oracle_mm.py pins it to ggml-cpu, tests/test_gpu_mul_mat_elements.py pins the kernels to it).

Two reference forms, one per kind of route:

* integer-dot routes (generic, first-generation TMA, superblock, int8 mma, per-pair MUL_MAT_ID, the fused epilogue's y): the
  activations are quantized to the weight type's vec_dot_type exactly as ggml-cpu quantizes them (Q8_0 with the SIMD rounding, Q8_1,
  Q8_K), and decoded as x̂ = d·q.  Then r[n, m] = Σ_k ŵ[m, k] x̂[n, k] in f64, ŵ the oracle's dequantization.  Q4_1 / Q5_1 pair with Q8_1,
  and both ggml-cpu and the device multiply the block minimum by the record's stored fp16 s (not by d·Σq): r does the same.
* fp16-operand routes (wgmma, dense, mul_mat_f16, mul_mat_f16_f16, grouped MUL_MAT_ID): r = Σ_k ŵ x with x unquantized.

Bound.  a[n, m] = Σ_k |ŵ| |x̂| (|x| on the fp16 routes).  Every kernel and ggml-cpu form y as a sum of partial products, each the
integer (or fp16 x fp16, exact in f32) dot of at most one 32-element sub-block times its scales, rounded in f32.  Per sub-block term:
  - scales only (Q4_0, Q5_0, Q8_0, IQ4_NL, Q3_K, Q6_K, IQ4_XS, the grid i-quants, TQ1_0 / TQ2_0): d_w·d_x, the product with the
    integer sum, and the int → f32 conversion of a sum that may exceed 2^24: 3 roundings, each relative to the term, |term| <= Σ|ŵ x̂|
    over the sub-block; 2 more for the K-quants' sub-scale products: c = 5;
  - a scale and a minimum (Q4_1, Q5_1, Q4_K, Q5_K, Q2_K): the scale part and the minimum part are rounded separately (4 roundings), and
    each part is relative to its own magnitude, which can exceed the magnitude Σ|ŵ x̂| of the difference they form.  That factor has no
    bound: a sub-block whose codes all sit where d·q ≈ m makes it as large as one likes.  The bound takes 4, an EMPIRICAL factor (for
    ŵ = d q - m with uniform codes q in 0..15 the average of (d q + m) / |d q - m| is at most 3.75), so c = 16.  It holds on the blocks
    the tests draw (uniformly random codes, scales and minima) and on ggml-cpu (tests/test_oracle_mm.py); it is not a worst case.
Summing K/32 such terms in any order adds at most K/32 - 1 roundings of partial sums each <= a; a final horizontal sum / epilogue adds
at most 4 more.  With u = 2^-24:
    |y - r| <= c_t (K/32 + 4) u a.
The fp16 routes add the operand roundings: x is prescaled by 2^-e (e = exponent(max|x_n|) - 13, the device's row_to_f16) and rounded
to fp16 (2^-11 relative, or 2^(e-25) absolute in the subnormal range), and ŵ reaches the tensor cores as fp16 after c16_t roundings
(1 for a plain conversion, 2 for a scale product, 6 with a minimum: scale, minimum, fused multiply-add and their cancellation):
    |y - r| <= c_t (K/32 + 4) u a + (1 + c16_t) 2^-11 a + 2^(e-25) Σ_k |ŵ[m, k]| + 2^-25 (qmax_t + 2) Σ_k |x[n, k]|.
The last term is for weights whose fp16 form is subnormal: a row of one 256-block with a tiny scale is wholly subnormal in fp16, each
weight off by up to 2^-25 per rounding (the scale's, times the largest code qmax_t a decoder multiplies it by, the minimum's and the
result's), far more than 2^-11 of its magnitude.

Cost: only the weight dequantization and activation quantization run in the C oracle on the host; r and a are f64 torch products on
whichever device the weights live on.

Block gate: nmse_blocks() gives the NMSE per 256-row x 64-column block and per column, which catches an error spread over a region
whose elements each stay under the bound.
"""
from __future__ import annotations

import numpy as np

from oracle import oracle as O

U = 2.0 ** -24
MIN_TYPES = (O.Q4_1, O.Q5_1, O.Q4_K, O.Q5_K, O.Q2_K)
# per-format constants of the bound (module docstring)
C_INT = {t: (16.0 if t in MIN_TYPES else 5.0) for t in O.TYPE_NAMES if t not in (O.F32, O.F16, O.Q8_1, O.Q8_K)}
C_INT[O.F16] = 2.0                                     # fp16 weights: products exact in f32, only the accumulation rounds
DENSE_TYPES = O.IQ_TYPES                               # dequantized to fp16 once by the conversion kernel in front of the GEMM
FP16_OPERAND = {t: (1.0 if t in DENSE_TYPES else 6.0 if t in MIN_TYPES else 2.0) for t in C_INT}
FP16_OPERAND[O.F16] = 0.0
# largest code magnitude a decoder multiplies by an fp16 scale that may be subnormal (absolute error 2^-25 per rounding); 0 where the weight
# reaches fp16 by one conversion of ŵ (the dense formats) or already is fp16
QMAX = {O.Q4_0: 8, O.Q4_1: 15, O.Q5_0: 16, O.Q5_1: 31, O.Q8_0: 128, O.IQ4_NL: 127, O.Q2_K: 3, O.Q3_K: 4, O.Q4_K: 15, O.Q5_K: 31,
        O.Q6_K: 32, O.IQ4_XS: 127}
QBLOCK = {O.Q8_0: (34, 32), O.Q8_1: (36, 32), O.Q8_K: (292, 256)}


def _torch():
    import torch
    return torch


def act_quant(orc: O.Oracle, t: int, X: np.ndarray):
    """x̂ [N, K] f64 as ggml-cpu multiplies it for weight type t, and (Q8_1 pairings only) the stored-s correction per 32-block:
    s[n, b] - d[n, b] Σq[n, b], else None"""
    X = np.ascontiguousarray(X, dtype=np.float32)
    N, K = X.shape
    vt = orc.vec_dot_type(t)
    size, qk = QBLOCK[vt]
    xh = np.empty((N, K), dtype=np.float64)
    corr = np.zeros((N, K // 32), dtype=np.float64) if vt == O.Q8_1 else None
    for n in range(N):
        b = orc.quantize(vt, X[n], simd_q8_0=(vt == O.Q8_0)).reshape(-1, size)
        if vt == O.Q8_K:
            d = b[:, :4].copy().view(np.float32).astype(np.float64)
            q = b[:, 4:260].view(np.int8).astype(np.float64)
        else:
            d = b[:, :2].copy().view(np.float16).astype(np.float64)
            q = b[:, (4 if vt == O.Q8_1 else 2):].view(np.int8).astype(np.float64)
            if vt == O.Q8_1:
                s = b[:, 2:4].copy().view(np.float16).astype(np.float64)[:, 0]
                corr[n] = s - d[:, 0] * q.sum(1)
        xh[n] = (d * q).reshape(-1)
    return xh, corr


def weight_mins(t: int, W: np.ndarray, M: int, K: int) -> np.ndarray:
    """the fp16 block minimum m of Q4_1 / Q5_1 rows, [M, K / 32] f64"""
    size = {O.Q4_1: 20, O.Q5_1: 24}[t]
    return np.ascontiguousarray(W, dtype=np.uint8).reshape(M * K // 32, size)[:, 2:4].copy().view(np.float16).astype(np.float64).reshape(M, K // 32)


def dequant(orc: O.Oracle, t: int, W: np.ndarray, M: int, K: int) -> np.ndarray:
    """ŵ [M, K] f32 (exact values of the f32 dequantization); t == F16: W holds fp16 values"""
    if t == O.F16:
        return np.asarray(W, dtype=np.float16).reshape(M, K).astype(np.float32)
    return orc.dequantize(t, W, M * K).reshape(M, K)


def row_exponent(X: np.ndarray) -> np.ndarray:
    """the device's prescale exponent e per activation row (mmq_tc2.cu row_to_f16): exponent(max|x|) - 13, 0 for a zero row, |e| <= 100"""
    amax = np.abs(np.asarray(X, dtype=np.float32)).max(axis=1)
    e = np.zeros(len(amax), dtype=np.int64)
    ok = (amax > 0) & (amax <= 3.0e38)
    bits = amax.view(np.uint32).astype(np.int64)
    e[ok] = np.clip(((bits[ok] >> 23) & 0xFF) - 127 - 13, -100, 100)
    return e


class Reference:
    """r and the bound of one [M, K] weight against activation rows, computed on `device` in f64 (callers split very large M into row blocks).

    t: the weight type (F16 for fp16 weights); route: "int" or "f16"; W: packed rows (uint8) or, for F16, fp16 values [M, K]."""

    def __init__(self, orc: O.Oracle, t: int, W: np.ndarray, M: int, K: int, device="cpu", w_hat: np.ndarray | None = None):
        torch = _torch()
        self.orc, self.t, self.M, self.K, self.device = orc, t, M, K, device
        wh = dequant(orc, t, W, M, K) if w_hat is None else w_hat
        self.w = torch.from_numpy(np.ascontiguousarray(wh)).to(device=device, dtype=torch.float64)
        self.wabs = self.w.abs()
        self.wsum = self.wabs.sum(1)                                          # Σ_k |ŵ[m, k]|
        self.mins = torch.from_numpy(weight_mins(t, W, M, K)).to(device) if t in (O.Q4_1, O.Q5_1) else None

    def __call__(self, X: np.ndarray, route: str, rows=None):
        """(r, bound) [N, M] f64 torch tensors on `device`; rows: an index subset of the weight rows (then [N, len(rows)])"""
        torch = _torch()
        X = np.ascontiguousarray(X, dtype=np.float32).reshape(-1, self.K)
        w, wabs, wsum = self.w, self.wabs, self.wsum
        mins = self.mins
        if rows is not None:
            idx = torch.as_tensor(rows, device=self.device)
            w, wabs, wsum = w[idx], wabs[idx], wsum[idx]
            mins = mins[idx] if mins is not None else None
        if route == "int":
            xh, corr = act_quant(self.orc, self.t, X)
        else:
            xh, corr = X.astype(np.float64), None
        x = torch.from_numpy(xh).to(self.device)
        r = x @ w.T
        a = x.abs() @ wabs.T
        if corr is not None:                                                  # m s - m d Σq: part of the minimum's term, rounded with it
            c = torch.from_numpy(corr).to(self.device)
            r += c @ mins.T
            a += c.abs() @ mins.abs().T
        bound = C_INT[self.t] * (self.K / 32 + 4) * U * a
        if route == "f16":
            e = torch.from_numpy(row_exponent(X).astype(np.float64)).to(self.device)
            bound += (1.0 + FP16_OPERAND[self.t]) * 2.0 ** -11 * a + torch.outer(torch.exp2(e - 25), wsum)
            if self.t != O.F16:                                               # fp16 weights in (or decoded through) the subnormal range
                bound += torch.outer(x.abs().sum(1), torch.full_like(wsum, 2.0 ** -25 * (QMAX.get(self.t, 0) + 2)))
        return r, bound


def ratio(y, r, bound):
    """|y - r| / bound elementwise (torch f64); 0 where both are 0, inf where y differs from an exact 0 (or is not finite)"""
    torch = _torch()
    d = (y.to(torch.float64) - r).abs()
    out = torch.where(bound > 0, d / torch.where(bound > 0, bound, torch.ones_like(bound)), torch.where(d == 0, torch.zeros_like(d), torch.full_like(d, float("inf"))))
    return torch.where(torch.isfinite(y.to(torch.float64)), out, torch.full_like(out, float("inf")))


def nmse_blocks(y, r, rows: int = 256, cols: int = 64, min_elems: int = 1024):
    """worst NMSE over the [N, M] result's 256-row (M) x 64-column (N) blocks and over its columns (one activation row n: M outputs),
    judging only blocks and columns of at least min_elems elements; NMSE = Σ(y - r)^2 / Σ r^2 (Σ(y - r)^2 where r is all zero)"""
    torch = _torch()
    y = y.to(torch.float64)
    N, M = r.shape
    d2, r2 = (y - r) ** 2, r ** 2

    def worst(num, den, count):
        ok = count >= min_elems
        if not bool(ok.any()):
            return 0.0
        v = torch.where(den > 0, num / torch.where(den > 0, den, torch.ones_like(den)), num)
        return float(v[ok].max())

    nb, mb = -(-N // cols), -(-M // rows)
    pad = (0, mb * rows - M, 0, nb * cols - N)
    bd = torch.nn.functional.pad(d2, pad).reshape(nb, cols, mb, rows).sum((1, 3))
    br = torch.nn.functional.pad(r2, pad).reshape(nb, cols, mb, rows).sum((1, 3))
    cnt = torch.nn.functional.pad(torch.ones_like(r), pad).reshape(nb, cols, mb, rows).sum((1, 3))
    col = worst(d2.sum(1), r2.sum(1), torch.full((N,), float(M), dtype=torch.float64, device=r.device))
    return worst(bd, br, cnt), col
