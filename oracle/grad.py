"""TEST INFRASTRUCTURE ONLY: MUL_MAT's gradient as the reference's test-backend-ops checks it, with an exact f64 reference and per-element
rounding bounds, and `mul_mat_grad`, the graph on a named ggml device ("CPU": ggml-cpu; "B2000": the plug-in, once loaded with
oracle.Ref().load_backend) through oracle/_ref/libggml_grad_probe.so (oracle/grad_probe.cpp, built by oracle/grad.mk).

The graph is test_mul_mat's: parents a [k, m, bs0, bs1] and b [k, n, bs0 nr0, bs1 nr1] (ggml order), each created with its extents
permuted by `per` and read through ggml_permute(per); loss L = sum(mul_mat(a, b)); a is a parameter only when bs1 == nr1 == 1.  Its
backward graph is OUT_PROD for dA (then REPEAT_BACK over the nr0 broadcast batches), OUT_PROD of a against the transposed output
gradient for dB, and the PERMUTE views back to the parents.

Reference.  L is bilinear, so with r2 = nr0, r3 = nr1 and q the batch of a that b's batch (i2, i3) reads, (i2 / r2, i3 / r3):
    dA[k, m, j2, j3] = sum over n and the b batches (i2, i3) with q = (j2, j3) of b[k, n, i2, i3]         (P_A = n nr0 nr1 terms)
    dB[k, n, i2, i3] = sum over m of a[k, m, i2 / r2, i3 / r3]                                           (P_B = m terms)
computed in f64 from the f32 inputs (exact: every term is an f32 and P <= 2^29) and mapped back through `per` to each parent's layout.

Bound on ga (the backward graph's gradient).  The output gradient is exactly 1 (SUM's backward repeats the loss gradient 1), so every
product the OUT_PROD kernels form is exact, and each ga element is an f32 sum of the P terms above, in some order and grouping (OUT_PROD's
partial sums, then REPEAT_BACK's).  Any such sum satisfies |ga - g| <= gamma_P sum |terms|, gamma_P = P u / (1 - P u), u = 2^-24.

Bound on gn (test-backend-ops' numerical gradient, gn = fl(fl(fu - fd) / (2 eps)), fu and fd the f32 losses at xu = fl(x0 + eps) and
xd = fl(x0 - eps)).  L is linear in each element, so L(xu) - L(xd) = g (xu - xd) exactly: no truncation term.  Write g_eff =
g (xu - xd) / (2 eps) (computed exactly here) and fu = L(xu) + e_u, fd = L(xd) + e_d.  Then
    gn - g_eff = [(e_u - e_d) + D (d1 + d2 + d1 d2)] / (2 eps),   |d1|, |d2| <= u,  D = fu - fd,  |D| <= |g (xu - xd)| + |e_u - e_d|
(d1 rounds the subtraction, d2 the division; 2 eps = 2 * 0.1f is exact).  fu is the f32 rounding of a sum of the f32 outputs y^ in double
(ggml-cpu's SUM, and the device's), so e_u = [fl32(S_u) - S_u] + [S_u - sum y^_u] + sum (y^_u - y_u): at most u |L(xu)| (1 + ...) for the
final rounding, gamma53_N sum |y^| for the double sum of N outputs, and the dot-product errors.  The outputs the perturbation does not
touch are the same f32 dot products of the same data in both runs, bit for bit, so their errors cancel in e_u - e_d; only the C outputs
that read x remain (C = n nr0 nr1 for an element of a, m for an element of b), each within gamma_K sum_k |a_k b_k| of its exact value in
either run (any summation order of K products).  So
    |gn - g| <= |g_eff - g| + (1 + 3u) [u (|L(xu)| + |L(xd)|) + 2 gamma53_N sum |y| + 2 gamma_K sum over the C outputs of sum_k |a b|] / (2 eps)
                + 2.0001 u |g (xu - xd)| / (2 eps)
with |x| taken as max(|xu|, |xd|) in the C outputs' sums and 1 + 2 gamma_K covering the difference between sum |y^| and sum |y|.

The mean absolute asymmetry test-backend-ops gates at 1e-4, mean |(gn - ga) / (gn + ga)| in float, is `maa`; a g near zero makes its
term unbounded, which is what `maa_terms` lets a test look at."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

from .probe import probe_lib, result

U = 2.0 ** -24
UD = 2.0 ** -53
EPS = np.float32(0.1)                     # test_case::grad_eps()
MAA_MAX = 1e-4                            # test_case::max_maa_err()
GRAD_NMAX = 20000                         # test_mul_mat::grad_nmax()

SIGNATURES = {
    "probe_mul_mat_grad": [C.c_char_p] + [C.c_void_p] * 3 + [C.c_float] + [C.c_void_p] * 3 + [C.c_int64] + [C.c_void_p] * 2
                          + [C.c_int64] + [C.c_void_p] * 2,
}


def gamma(p, u=U):
    return p * u / (1.0 - p * u)


@dataclass(frozen=True)
class GradCase:
    m: int
    n: int
    k: int
    bs: tuple = (1, 1)
    nr: tuple = (1, 1)
    per: tuple = (0, 1, 2, 3)

    def __str__(self):
        return (f"m={self.m},n={self.n},k={self.k},bs=[{self.bs[0]},{self.bs[1]}],nr=[{self.nr[0]},{self.nr[1]}],"
                f"per=[{','.join(map(str, self.per))}]")

    @property
    def a_param(self):
        return self.bs[1] == 1 and self.nr[1] == 1

    def ne_a(self):                       # the logical (un-permuted) extents, ggml order
        return (self.k, self.m, self.bs[0], self.bs[1])

    def ne_b(self):
        return (self.k, self.n, self.bs[0] * self.nr[0], self.bs[1] * self.nr[1])

    def parent_ne(self, ne):
        return tuple(ne[p] for p in self.per)

    def ngrads(self):
        return (int(np.prod(self.ne_a())) if self.a_param else 0) + int(np.prod(self.ne_b()))

    def cfg(self):
        return np.array([self.m, self.n, self.k, *self.bs, *self.nr, *self.per], dtype=np.int64)

    def inputs(self, seed):
        """the parents' data, U(-1, 1) in f32 as test-backend-ops draws it, numpy shapes (ggml dims reversed)"""
        rng = np.random.default_rng(seed)
        a = rng.uniform(-1, 1, self.parent_ne(self.ne_a())[::-1]).astype(np.float32)
        b = rng.uniform(-1, 1, self.parent_ne(self.ne_b())[::-1]).astype(np.float32)
        return a, b


# test-backend-ops' f32 x f32 test_mul_mat cases of make_test_cases_eval() (m = 16, K = 256), without the duplicate
def eval_cases():
    cases = [GradCase(16, i, 256) for i in range(1, 10)]
    for n in (1, 16):
        for bs, nr in (((1, 1), (2, 1)), ((1, 1), (1, 2)), ((3, 1), (1, 1)), ((3, 1), (2, 1)), ((3, 2), (1, 1)), ((3, 2), (2, 1)),
                       ((3, 2), (1, 2)), ((3, 2), (2, 2))):
            cases.append(GradCase(16, n, 256, bs, nr))
    for n in (1, 8, 16):
        for per in ((0, 2, 1, 3), (0, 1, 3, 2), (0, 3, 2, 1)):
            cases.append(GradCase(16, n, 256, (2, 3), (1, 1), per))
    return cases


def _logical(case, parent):
    """a parent's numpy data -> the logical tensor in ggml axis order (axis i = ggml dim i), f64"""
    g = parent.astype(np.float64).transpose(3, 2, 1, 0)
    inv = [0] * 4
    for i, p in enumerate(case.per):
        inv[p] = i
    return np.transpose(g, inv)


def _to_parent(case, logical):
    """a logical gradient in ggml axis order -> the parent's numpy layout"""
    return np.ascontiguousarray(np.transpose(logical, case.per).transpose(3, 2, 1, 0))


@dataclass
class Reference:
    g_a: np.ndarray | None                # exact gradients, parents' numpy layouts
    g_b: np.ndarray
    bound_a: np.ndarray | None            # gamma_P sum |terms|
    bound_b: np.ndarray
    loss: float                           # exact
    A: np.ndarray                         # logical a, b in ggml axis order (f64)
    B: np.ndarray
    absdot: np.ndarray                    # sum_k |a| |b| per output [m, n, i2, i3]
    absy: float                           # sum |y| over the outputs


def _products(x, y):
    """[k, m, i2, i3] x [k, n, i2, i3] -> sum_k x y as [m, n, i2, i3]"""
    return np.matmul(x.transpose(2, 3, 1, 0), y.transpose(2, 3, 0, 1)).transpose(2, 3, 0, 1)


def reference(case, a, b, outputs=True):
    """the exact gradients and their ga bounds; with outputs, also what gn_bound needs (the mat-mul itself, in f64)"""
    A, B = _logical(case, a), _logical(case, b)
    r2, r3 = case.nr
    Ab = np.repeat(np.repeat(A, r2, axis=2), r3, axis=3)                  # a as each b batch reads it
    y = _products(Ab, B) if outputs else np.zeros(1)
    absdot = _products(np.abs(Ab), np.abs(B)) if outputs else None

    def fold(x):                                                           # sum b batches onto the a batch they read
        s = x.shape
        return x.reshape(s[0], s[1], s[2] // r2, r2, s[3] // r3, r3).sum(axis=(3, 5))
    dA = fold(B.sum(axis=1, keepdims=True))[:, 0][:, None].repeat(case.m, axis=1)
    dA_abs = fold(np.abs(B).sum(axis=1, keepdims=True))[:, 0][:, None].repeat(case.m, axis=1)
    dB = Ab.sum(axis=1, keepdims=True).repeat(case.n, axis=1)
    dB_abs = np.abs(Ab).sum(axis=1, keepdims=True).repeat(case.n, axis=1)
    pa, pb = case.n * r2 * r3, case.m
    ga = _to_parent(case, dA) if case.a_param else None
    ba = _to_parent(case, gamma(pa) * dA_abs) if case.a_param else None
    return Reference(ga, _to_parent(case, dB), ba, _to_parent(case, gamma(pb) * dB_abs), float(y.sum()), A, B, absdot, float(np.abs(y).sum()))


def _logical_index(case, which, flat):
    """linear indices into a parent -> its logical ggml indices (k, m|n, i2, i3)"""
    pne = case.parent_ne(case.ne_a() if which == "a" else case.ne_b())
    i3, r = np.divmod(flat, pne[0] * pne[1] * pne[2])
    i2, r = np.divmod(r, pne[0] * pne[1])
    i1, i0 = np.divmod(r, pne[0])
    pidx = np.stack([i0, i1, i2, i3])                                      # parent dim i
    lidx = np.empty_like(pidx)
    for i, p in enumerate(case.per):
        lidx[p] = pidx[i]
    return lidx


def gn_bound(case, ref, which, flat, x0):
    """per-element bound on |gn - g| at the linear parent indices flat (x0: the parent's values there), and g there"""
    g = (ref.g_a if which == "a" else ref.g_b).reshape(-1)[flat]
    x0 = x0.astype(np.float32)
    xu, xd = (x0 + EPS).astype(np.float64), (x0 - EPS).astype(np.float64)
    dx = xu - xd
    x0 = x0.astype(np.float64)
    xmax = np.maximum(np.abs(xu), np.abs(xd))
    k, j, i2, i3 = _logical_index(case, which, flat)
    r2, r3 = case.nr
    if which == "a":                       # the outputs (m = j, every n, the b batches reading a batch (i2, i3))
        ii2 = i2[:, None] * r2 + np.arange(r2)[None, :]
        ii3 = i3[:, None] * r3 + np.arange(r3)[None, :]
        rows = ref.absdot[j[:, None, None, None], np.arange(case.n)[None, :, None, None], ii2[:, None, :, None], ii3[:, None, None, :]]
        other = np.abs(ref.B[k[:, None, None, None], np.arange(case.n)[None, :, None, None], ii2[:, None, :, None], ii3[:, None, None, :]])
    else:                                  # the outputs (every m, n = j, batch (i2, i3))
        rows = ref.absdot[np.arange(case.m)[None, :], j[:, None], i2[:, None], i3[:, None]]
        other = np.abs(ref.A[k[:, None], np.arange(case.m)[None, :], (i2 // r2)[:, None], (i3 // r3)[:, None]])
    extra = (xmax - np.abs(x0)).reshape(-1, *([1] * (other.ndim - 1))) * other
    touched = (rows + extra).reshape(len(flat), -1).sum(axis=1)
    lu, ld = ref.loss + g * (xu - x0), ref.loss + g * (xd - x0)
    n_out = ref.absdot.size
    ge = g * dx / (2.0 * float(EPS))
    err = (U * (np.abs(lu) + np.abs(ld)) * (1 + gamma(case.k)) + 2 * gamma(n_out, UD) * ref.absy * (1 + 2 * gamma(case.k))
           + 2 * gamma(case.k) * touched)
    return np.abs(ge - g) + (1 + 3 * U) * err / (2.0 * float(EPS)) + 2.0001 * U * np.abs(g * dx) / (2.0 * float(EPS)), g


def maa_terms(gn, ga):
    """test-backend-ops' mean_abs_asymm terms: |(gn - ga) / (gn + ga)| in float"""
    gn, ga = np.asarray(gn, np.float32), np.asarray(ga, np.float32)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.abs((gn - ga) / (gn + ga)).astype(np.float64)


def maa(gn, ga):
    """mean_abs_asymm: the terms summed in double over all elements (a 0 / 0 term makes it NaN, which passes the gate as it does there)"""
    return float(maa_terms(gn, ga).sum() / len(gn))


def sample(g, count, seed):
    """count linear indices of a gradient: the smallest |g| first, then a seeded draw of the rest"""
    flat = np.abs(g.reshape(-1))
    small = np.argsort(flat, kind="stable")[: count // 4]
    rest = np.setdiff1d(np.arange(flat.size), small)
    pick = np.random.default_rng(seed).choice(rest, size=min(count - len(small), rest.size), replace=False)
    return np.sort(np.concatenate([small, pick])).astype(np.int64)


def _lib():
    return probe_lib("grad", "make -C oracle -f grad.mk grad", SIGNATURES)


def mul_mat_grad(dev: str, case: GradCase, a: np.ndarray, b: np.ndarray, idx_a=None, idx_b=None, raw: bool = False):
    """MUL_MAT's backward graph for `case` with parents a, b (numpy, as case.inputs gives them): (loss, ga_a, ga_b, gn_a, gn_b).  ga_* are
    the gradients in the parents' layouts (ga_a None when a is not a parameter); gn_* are test-backend-ops' numerical gradients at the
    linear parent indices idx_* (None when not asked)."""
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    ia = np.ascontiguousarray(idx_a if idx_a is not None else [], dtype=np.int64)
    ib = np.ascontiguousarray(idx_b if idx_b is not None else [], dtype=np.int64)
    loss = np.zeros(1, dtype=np.float32)
    ga_a, ga_b = np.full_like(a, np.nan), np.full_like(b, np.nan)
    gn_a, gn_b = np.full(max(len(ia), 1), np.nan, np.float32), np.full(max(len(ib), 1), np.nan, np.float32)
    cfg = case.cfg()
    rc = _lib().probe_mul_mat_grad(dev.encode(), cfg.ctypes.data, a.ctypes.data, b.ctypes.data, float(EPS), loss.ctypes.data, ga_a.ctypes.data,
                                   ga_b.ctypes.data, len(ia), ia.ctypes.data, gn_a.ctypes.data, len(ib), ib.ctypes.data, gn_b.ctypes.data)
    return result(rc, raw, f"probe_mul_mat_grad({dev}, {case})",
                  (float(loss[0]), ga_a if case.a_param else None, ga_b, gn_a[: len(ia)] if idx_a is not None else None,
                   gn_b[: len(ib)] if idx_b is not None else None))
