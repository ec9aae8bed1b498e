"""oracle/seq.py — f64 references of the sequence ops (ROPE, SSM_CONV, SSM_SCAN, RWKV_WKV6, GATED_LINEAR_ATTN), each with a per-element bound
on |computed − reference| for a computation in f32 that rounds as the device kernels and ggml-cpu do.

TEST INFRASTRUCTURE ONLY (tests/test_oracle_seq.py pins it to ggml-cpu, tests/test_gpu_seq_elements.py pins the kernels to it).  No device code.

Notation: u = 2^-24 (one rounding of an f32 result, relative); ulp32(v) the spacing of f32 at |v|; γ_n = n u / (1 − n u).  Every rounding
also gets an absolute 2^-149 (the subnormal spacing), so that a result that underflows keeps a non-zero bound.  The bounds are first order:
products of two error terms (relative size below 2^-40 here) are left out.

SSM_CONV.  y = Σ_{k<d_conv} s_k c_k, one rounded product and one rounded add per term, ascending k from 0: |y − r| ≤ γ_{d_conv} Σ|s_k c_k|.

SSM_SCAN.  Per token and element, with dt_sp = softplus(dt) (dt itself above ggml-cpu's cut-off at 20):
  state' = state · exp(dt_sp A) + B (x dt_sp),   y = Σ_i state'_i C_i (ascending i from 0).
  The reference runs this recurrence in f64 over the same f32 inputs.  Alongside it a running bound δ on each state element and e_y on each
  y, in f64, token by token:
  - softplus: expf returns E within L_exp ulp, log1pf within L_log1p ulp; an error ε in E moves log1p(E) by ε / (1 + E), so
      e_sp = L_exp 2u E / (1 + E) + L_log1p 2u dt_sp   (0 above the cut-off, where dt_sp = dt exactly);
  - a = dt_sp A: e_a = u|a| + |A| e_sp;  dA = exp(a): e_dA = dA (L_exp 2u + e_a);
  - p1 = state dA: e_p1 = dA δ + |state| e_dA + u|p1|  (the carried error δ goes through dA, the exponent's through |state dA A| e_sp);
  - x_dt = x dt_sp: e_xdt = |x| e_sp + u|x_dt|;  p2 = B x_dt: e_p2 = |B| e_xdt + u|p2|;
  - state' = p1 + p2: δ' = e_p1 + e_p2 + u|state'|;
  - y: e_y = Σ_i (|C_i| δ'_i + u|state'_i C_i|) + u Σ_i |partial sum_i|.
  L_exp and L_log1p are each library's documented or measured maximum: the CUDA C Programming Guide gives expf 2 ulp and log1pf 1 ulp; for
  glibc the bound takes 2 ulp for both (its expf and log1pf are each within 1 ulp on x86-64, and tests/test_oracle_seq.py measures the
  glibc in use on every dt the cases draw), so L_exp = L_log1p = 2 covers both libraries.

RWKV_WKV6 / GATED_LINEAR_ATTN.  Per token, head, row i and column j (b200_wkv.cuh spells the roundings):
  WKV6: kv = v_j k_i;  y_j = Σ_i fma(fma(kv, tf_i, p), r_i, ·);  state' = fma(p, td_i, kv)
  GLA:  kv = v_j k_i;  temp = fma(p, g_i, kv);  y_j = Σ_i fma(temp, q_i scale, ·);  state' = temp
  kv and q_i scale are rounded on their own (u each); each FMA rounds once (u of its result).  ggml-cpu computes the tail columns of a head
  size that is not a multiple of its vector width unfused, which rounds each product too: the bound counts those product roundings as well,
  so it holds for both forms.  The state error δ is carried from token to token through |td| (|g|), so the bound follows the state's growth
  (about 1 / (1 − w) over a long prompt with decays w near 1):
  WKV6: e_in = |tf| u|kv| + δ + u|kv tf| + u|kv tf + p|;  e_y = Σ_i (|r_i| e_in + u|(kv tf + p) r_i|) + u Σ_i |partial_i|;
        δ' = |td| δ + u|kv| + u|p td| + u|state'|
  GLA:  δ' = |g| δ + u|kv| + u|p g| + u|temp|;  e_y = Σ_i (|qs_i| δ' + |temp| u|qs_i| + u|temp qs_i|) + u Σ_i |partial_i|.

ROPE.  The angle is part of ggml's semantics, so it is rebuilt exactly in numpy float32 first: the sequential theta *= theta_scale chain
from the f32 position (ggml_rope_cache_init; MROPE / VISION advance four streams together and pick one per section), the division by the
freq factor, freq_scale times it, and with ext_factor != 0 the YaRN ramp and mix, every operation one f32 rounding, with the per-op constants
of ggml_b200.rope_params.  cos and sin of that f32 angle are then taken in f64, times mscale, and the rotation is done in f64.
  cs = fl(cosf(t) mscale): |cs − cos(t) mscale| ≤ mscale L_trig ulp32(cos t) + u|cs|  (sn alike), with L_trig = 2: the CUDA C
  Programming Guide gives 2 ulp for sinf / cosf over the full range; glibc's are within 1 ulp.
  y0 = fl(fl(x0 cs) − fl(x1 sn)): |y0 − r0| ≤ |x0| e_cs + |x1| e_sn + u(|x0 cs| + |x1 sn|) + u|r0|  (y1 alike).
  f16 results add half an f16 ulp of |r| + that bound for the store.  The f16 inputs are exact in f32, so the reference reads the same
  values and there is no input rounding to add (the K-shift reads and writes an f16 cache).  Elements beyond n_dims are copied: bound 0.

angle_drift() measures how far ggml's f32 angle chain lies from the exact pos · base^(−2j/n_dims): that is a property of ggml's definition,
not of any kernel, and it is printed, not gated.
"""
from __future__ import annotations

import numpy as np

U = 2.0 ** -24
TINY = 2.0 ** -149
L_EXP, L_LOG1P, L_TRIG = 2.0, 2.0, 2.0          # libm ulp figures used by the bounds (module docstring)
ROPE_NORM, ROPE_NEOX, ROPE_MROPE, ROPE_VISION = 0, 2, 8, 24
f32 = np.float32


def gamma(n: int) -> float:
    return n * U / (1 - n * U)


def ulp32(v) -> np.ndarray:
    return np.spacing(np.abs(np.asarray(v, dtype=np.float64)).astype(np.float32)).astype(np.float64)


def ratio(y, r, bound) -> np.ndarray:
    """|y − r| / bound per element (0 where both sides are exactly equal, inf where the bound is 0 and they differ, inf for a non-finite y)"""
    y = np.asarray(y, dtype=np.float64)
    d = np.abs(y - r)
    with np.errstate(divide="ignore", invalid="ignore"):
        q = np.where(d == 0, 0.0, d / bound)
    return np.where(np.isfinite(y), q, np.inf)


# ------------------------------------------------------------------ SSM_CONV
def ssm_conv(sx: np.ndarray, c: np.ndarray):
    """sx f32 [n_s, d_inner, d_conv − 1 + n_t], c f32 [d_inner, d_conv] -> (r, bound) f64 [n_s, n_t, d_inner]"""
    n_s, d_inner, ncs = sx.shape
    dc = c.shape[1]
    n_t = ncs - dc + 1
    r = np.zeros((n_s, n_t, d_inner))
    a = np.zeros_like(r)
    for k in range(dc):
        term = sx[:, :, k:k + n_t].astype(np.float64).transpose(0, 2, 1) * c[:, k].astype(np.float64)
        r += term
        a += np.abs(term)
    return r, gamma(dc) * a + 2 * dc * TINY


# ------------------------------------------------------------------ SSM_SCAN
def softplus(dt: np.ndarray):
    """(dt_sp, e_sp) in f64 of f32 dt, with ggml-cpu's cut-off at 20"""
    dt = dt.astype(np.float64)
    E = np.exp(np.minimum(dt, 20.0))
    sp = np.where(dt <= 20.0, np.log1p(E), dt)
    e = np.where(dt <= 20.0, L_EXP * 2 * U * E / (1 + E) + L_LOG1P * 2 * U * sp + 2 * TINY, 0.0)
    return sp, e


def ssm_scan(s0, x, dt, A, B, C):
    """s0 [n_s, d_inner, d_state], x / dt [n_s, n_t, d_inner], A [d_inner, d_state], B / C [n_s, n_t, d_state] (f32, contiguous copies)
    -> (y, y bound [n_s, n_t, d_inner], final state, state bound [n_s, d_inner, d_state]), all f64"""
    n_s, n_t, d_inner = x.shape
    st = s0.astype(np.float64)
    dl = np.zeros_like(st)
    A64 = A.astype(np.float64)[None]
    y = np.zeros((n_s, n_t, d_inner))
    ey = np.zeros_like(y)
    for t in range(n_t):
        sp, e_sp = softplus(dt[:, t, :])
        sp3, esp3 = sp[:, :, None], e_sp[:, :, None]
        a = sp3 * A64
        e_a = U * np.abs(a) + np.abs(A64) * esp3 + TINY
        dA = np.exp(a)
        e_dA = dA * (L_EXP * 2 * U + e_a) + L_EXP * TINY
        p1 = st * dA
        e_p1 = dA * dl + np.abs(st) * e_dA + U * np.abs(p1) + TINY
        xv = x[:, t, :].astype(np.float64)
        xdt = (xv * sp)[:, :, None]
        e_xdt = (np.abs(xv) * e_sp)[:, :, None] + U * np.abs(xdt) + TINY
        b = B[:, t, :].astype(np.float64)[:, None, :]
        p2 = b * xdt
        e_p2 = np.abs(b) * e_xdt + U * np.abs(p2) + TINY
        st = p1 + p2
        dl = e_p1 + e_p2 + U * np.abs(st) + TINY
        cc = C[:, t, :].astype(np.float64)[:, None, :]
        term = st * cc
        y[:, t, :] = term.sum(-1)
        ey[:, t, :] = (np.abs(cc) * dl + U * np.abs(term) + TINY).sum(-1) + U * np.abs(np.cumsum(term, -1)).sum(-1)
    return y, ey, st, dl


# ------------------------------------------------------------------ RWKV_WKV6 / GATED_LINEAR_ATTN
def wkv(k, v, a, b, tf, s0, gla: bool, scale: float = 1.0):
    """k, v, a (r / q), b (td / g) f32 [T, H, S], tf f32 [H, S] (WKV6) or None, s0 f32 [n_seqs, H, S, S] -> (y, y bound [T, H, S], final
    states, their bound [n_seqs, H, S, S]), f64; sequence q owns tokens [q T / n_seqs, (q + 1) T / n_seqs)"""
    T, H, S = k.shape
    ns = s0.shape[0]
    nt = T // ns
    y, ey = np.zeros((T, H, S)), np.zeros((T, H, S))
    st_all, dl_all = np.zeros((ns, H, S, S)), np.zeros((ns, H, S, S))
    tf64 = tf.astype(np.float64)[:, :, None] if tf is not None else None
    for q in range(ns):
        st = s0[q].astype(np.float64)
        dl = np.zeros_like(st)
        for t in range(q * nt, (q + 1) * nt):
            kv = k[t].astype(np.float64)[:, :, None] * v[t].astype(np.float64)[:, None, :]          # [H, i, j]
            e_kv = U * np.abs(kv) + TINY
            bb = b[t].astype(np.float64)[:, :, None]
            pb = st * bb
            if gla:
                qs = (a[t].astype(np.float64) * f32(scale))[:, :, None]                               # q scale, the f32 scale
                e_qs = U * np.abs(qs) + TINY
                temp = pb + kv
                dl = np.abs(bb) * dl + e_kv + U * np.abs(pb) + U * np.abs(temp) + 2 * TINY
                term = temp * qs
                e_term = np.abs(qs) * dl + np.abs(temp) * e_qs + U * np.abs(term) + TINY
                st = temp
            else:
                kt = kv * tf64
                inner = kt + st
                e_in = np.abs(tf64) * e_kv + dl + U * np.abs(kt) + U * np.abs(inner) + 2 * TINY
                rr = a[t].astype(np.float64)[:, :, None]
                term = inner * rr
                e_term = np.abs(rr) * e_in + U * np.abs(term) + TINY
                st = pb + kv
                dl = np.abs(bb) * dl + e_kv + U * np.abs(pb) + U * np.abs(st) + 2 * TINY
            y[t] = term.sum(1)
            ey[t] = e_term.sum(1) + U * np.abs(np.cumsum(term, 1)).sum(1) + S * TINY
        st_all[q], dl_all[q] = st, dl
    return y, ey, st_all, dl_all


# ------------------------------------------------------------------ ROPE
def rope_angles(pos: np.ndarray, n_pos: int, p, ff=None) -> np.ndarray:
    """f32 angles [n_pos, n_cache] of ggml's definition (module docstring) for params p (ggml_b200.RopeParams or alike) and positions pos
    (i32, [n_pos] or [4 n_pos] for MROPE / VISION)"""
    mode, nd = int(p.mode), int(p.n_dims)
    ncache = nd if mode == ROPE_VISION else nd // 2
    ts = f32(p.theta_scale)
    th = np.zeros((n_pos, ncache), dtype=np.float32)
    if not mode & ROPE_MROPE:
        t = pos[:n_pos].astype(np.float32)
        for j in range(ncache):
            th[:, j] = t
            t = (t * ts).astype(np.float32)
    else:
        s = [int(p.sections[i]) for i in range(4)]
        s0, sw = s[0], s[0] + s[1]
        se = sw + s[2]
        sect = se + s[3]
        P = [pos[i * n_pos:(i + 1) * n_pos].astype(np.float32) for i in range(4)]
        cur = [q.copy() for q in P]
        sector = 0
        for j in range(ncache):
            if mode == ROPE_VISION:
                for k, start in enumerate((0, s0, sw, se)):
                    if sector == start:
                        cur[k] = P[k].copy()
            which = 1 if s0 <= sector < sw else 2 if sw <= sector < se else 3 if sector >= se else 0
            th[:, j] = cur[which]
            cur = [(c * ts).astype(np.float32) for c in cur]
            sector += 1
            if sector == sect:
                sector = 0
    ffv = np.ones(ncache, dtype=np.float32) if ff is None else np.asarray(ff, dtype=np.float32)[:ncache]
    extrap = (th / ffv[None, :]).astype(np.float32)
    interp = (f32(p.freq_scale) * extrap).astype(np.float32)
    if float(p.ext_factor) != 0.0:
        c0, c1 = f32(p.corr_dims[0]), f32(p.corr_dims[1])
        span = f32(c1 - c0)
        yv = ((np.arange(ncache, dtype=np.float32) - c0).astype(np.float32) / max(f32(0.001), span)).astype(np.float32)
        ramp = (f32(1) - np.minimum(f32(1), np.maximum(f32(0), yv))).astype(np.float32)
        mix = (ramp * f32(p.ext_factor)).astype(np.float32)
        return ((interp * (f32(1) - mix)).astype(np.float32) + (extrap * mix).astype(np.float32)).astype(np.float32)
    return interp


def rope(x: np.ndarray, pos: np.ndarray, p, ff=None):
    """x f32 / f16 [ne3, n_pos, n_head, ne0] -> (r, bound) f64 of x's shape; p: ggml_b200.rope_params(...)"""
    ne3, n_pos, n_head, ne0 = x.shape
    mode, nd = int(p.mode), int(p.n_dims)
    th = rope_angles(pos, n_pos, p, ff).astype(np.float64)                                             # [n_pos, n_cache]
    ms = float(f32(p.mscale))
    cs, sn = np.cos(th) * ms, np.sin(th) * ms
    e_cs = ms * L_TRIG * ulp32(np.cos(th)) + U * np.abs(cs) + 2 * TINY
    e_sn = ms * L_TRIG * ulp32(np.sin(th)) + U * np.abs(sn) + 2 * TINY
    xd = x.astype(np.float64)
    r, bound = xd.copy(), np.zeros_like(xd)
    if mode == ROPE_VISION:
        i0, i1 = np.arange(nd), np.arange(nd) + nd
    elif mode == ROPE_NORM:
        i0, i1 = np.arange(0, nd, 2), np.arange(1, nd, 2)
    else:
        i0, i1 = np.arange(nd // 2), np.arange(nd // 2) + nd // 2
    if len(i0):
        c, s = cs[None, :, None, :], sn[None, :, None, :]
        ec, es = e_cs[None, :, None, :], e_sn[None, :, None, :]
        x0, x1 = xd[..., i0], xd[..., i1]
        r0, r1 = x0 * c - x1 * s, x0 * s + x1 * c
        base = np.abs(x0) * ec + np.abs(x1) * es + U * (np.abs(x0 * c) + np.abs(x1 * s)) + 3 * TINY
        b0 = base + U * np.abs(r0)
        b1 = np.abs(x0) * es + np.abs(x1) * ec + U * (np.abs(x0 * s) + np.abs(x1 * c)) + 3 * TINY + U * np.abs(r1)
        if x.dtype == np.float16:
            b0 = b0 + 0.5 * np.spacing((np.abs(r0) + b0).astype(np.float16)).astype(np.float64)
            b1 = b1 + 0.5 * np.spacing((np.abs(r1) + b1).astype(np.float16)).astype(np.float64)
        r[..., i0], r[..., i1] = r0, r1
        bound[..., i0], bound[..., i1] = b0, b1
    return r, bound


def angle_drift(positions, n_dims: int = 128, freq_base: float = 10000.0) -> dict:
    """{pos: max over pairs j of |ggml's f32 angle − pos · base^(−2j/n_dims)|, in radians} for NORM / NEOX without scaling"""
    import ggml_b200 as g
    p = g.rope_params(n_dims, ROPE_NEOX, freq_base=freq_base)
    out = {}
    for q in positions:
        th = rope_angles(np.array([q], dtype=np.int32), 1, p)[0].astype(np.float64)
        exact = q * freq_base ** (-2.0 * np.arange(n_dims // 2) / n_dims)
        out[int(q)] = float(np.max(np.abs(th - exact)))
    return out


# ------------------------------------------------------------------ the probes' cases as the arrays the references take
def conv_arrays(case):
    """(sx [n_s, d_inner, d_conv − 1 + n_t], c [d_inner, d_conv]) of an oracle.ssm.ConvCase, contiguous f32"""
    from . import ssm as S
    sx, c = (S.read(v) for v in case.views())
    return sx.reshape(sx.shape[-3:]), c.reshape(c.shape[-2:])


def scan_arrays(case, views=None):
    """(s0, x, dt, A, B, C) of an oracle.ssm.ScanCase in the shapes ssm_scan() takes, contiguous f32"""
    from . import ssm as S
    v = views or case.views()
    s0, x, dt, A, B, C = (S.read(w) for w in v)
    return s0[0], x[0], dt[0], A[0, 0], B[0], C[0]


def wkv_args(case, srcs):
    """wkv()'s arguments for an oracle.wkv.WkvCase and its sources"""
    if case.gla:
        k, v, q, gt, s0 = srcs
        return k, v, q, gt, None, s0, True, case.scale
    k, v, r, tf, td, s0 = srcs
    return k, v, r, td, tf, s0, False, 1.0
