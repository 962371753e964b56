"""softmax_rgb_blend and soft depth (csrc/blending.cu, sections 2 and 3) against a float64 reference, per element, on
every kernel path.

The reference restates the forward formulas and the backward formulas of the header of blending.cu in float64 numpy,
and next to every value returns a bound beta on how far a correct float32 evaluation of the same steps can lie from
it: a first-order running error bound, propagated step by step with u = 2^-24:

    a +- b      beta_a + beta_b + u |a +- b|
    a * b       |b| beta_a + |a| beta_b + u |a b|
    a / b       (beta_a + |a / b| beta_b) / |b| + u |a / b|
    expf(a)     e^a (beta_a + 2u)                     (CUDA's expf is within 2 ulp)
    n terms     sum beta + (n - 1) u sum |terms|      (a sum or a product, in any order)

The reciprocals 1 / sigma and 1 / gamma are exact in the reference; the kernels' float32 reciprocals (of sigma and
gamma rounded to float32) carry 2u.  Below the normal float32 range the relative terms no longer hold: a product or
quotient that is subnormal adds 2^-150, and an expf or a coverage that is (where expf(-x) overflows, 1 / (1 + inf) is
0) adds its own size, since the float32 result may be 0.  Every element of every output must satisfy

    |got - ref| <= 2 beta + 2^-126

(the factor 2 covers second-order terms, the floor results that are subnormal in float32).  No element is masked and
tied pixels are compared slot by slot.

Discrete decisions are made as the kernels make them.  z_inv is computed in float32 exactly as the kernels compute it
(numpy reproduces it bit for bit), so the argmax (the first slot attaining the float32 maximum) and `m_passed`
(z_max >= 1e-10f) are exact.  `delta_passed` rests on expf, which is not correctly rounded: it is decided in float64,
and within 2 beta of 1e-10f both branches are accepted.  The soft depth masks c_k <= 1 are exact where every coverage
up to slot k is exactly 0, 1/2 or 1 in float32 (empty slots, d = 0, |d / sigma| >= 30); elsewhere they are decided in
float64, and within 2 beta of 1 both branches are accepted.  Where a branch is open the reference returns the
interval between the two values.

Two CPU tests keep the bound honest: the float32 torch chain lies within it on every scene, and defective versions of
that chain fall outside it.
"""
import math

import numpy as np
import pytest
import torch
from scipy.special import expit

from test_blending import softmax_chain
from test_depth_shading import soft_depth_chain

U = 2.0 ** -24
FLOOR = 2.0 ** -126
TINY = 2.0 ** -126  # the smallest normal float32
EPS32 = float(np.float32(1e-10))  # blending.py's eps as the kernels hold it
LN_EPS = -math.log(EPS32)         # delta = exp((eps - m) / gamma) reaches eps at m - eps = 23.03 gamma


# ------------------------------------------------------------------------------------------ error-tracked values
class F:
    """A float64 value and a bound on how far a float32 evaluation of the same steps can lie from it."""

    __slots__ = ("v", "b")

    def __init__(self, v, b=None):
        self.v = np.asarray(v, dtype=np.float64)
        self.b = np.zeros_like(self.v) if b is None else np.asarray(b, dtype=np.float64)

    def __getitem__(self, i):
        return F(self.v[i], np.broadcast_to(self.b, self.v.shape)[i])

    def __add__(self, o):
        o = _f(o)
        v = self.v + o.v
        return F(v, self.b + o.b + U * np.abs(v))

    def __sub__(self, o):
        o = _f(o)
        v = self.v - o.v
        return F(v, self.b + o.b + U * np.abs(v))

    def __mul__(self, o):
        o = _f(o)
        v = self.v * o.v
        return F(v, np.abs(o.v) * self.b + np.abs(self.v) * o.b + rounding(v))

    def __truediv__(self, o):
        o = _f(o)
        v = self.v / o.v
        return F(v, (self.b + np.abs(v) * o.b) / np.abs(o.v) + rounding(v))

    def __neg__(self):
        return F(-self.v, self.b)

    def masked(self, m):
        """Product with an exact 0 / 1 mask (no rounding)."""
        return F(self.v * m, self.b * m)

    def exp(self):
        v = np.exp(self.v)
        return F(v, v * (self.b + 2 * U) + underflow(v))


def rounding(v):
    """The rounding of a float32 product or quotient: u |v|, and 2^-150 where the result is subnormal."""
    return U * np.abs(v) + np.where(np.abs(v) < TINY, 2.0 ** -150, 0.0)


def underflow(v):
    """Where a float32 result of a library function falls below the normal range, it may be subnormal or 0."""
    return np.where(np.abs(v) < TINY, np.abs(v) + 2.0 ** -149, 0.0)


def _f(x):
    return x if isinstance(x, F) else F(x)


def where(c, a, b):
    a, b = _f(a), _f(b)
    return F(np.where(c, a.v, b.v), np.where(c, a.b, b.b))


def fsum(x, axis):
    n = x.v.shape[axis]
    return F(x.v.sum(axis), x.b.sum(axis) + (n - 1) * U * np.abs(x.v).sum(axis))


def excl_prod(x, reverse=False):
    """Exclusive prefix (or suffix) products along axis 1 of (P, K): value and bound of prod over the slots before k
    (after k), sum_i beta_i prod_{j != i} |x_j| + (factors - 1) u |product|."""
    v, b = (x.v[:, ::-1], x.b[:, ::-1]) if reverse else (x.v, x.b)
    P, K = v.shape
    out_v, out_b = np.ones((P, K)), np.zeros((P, K))
    pv, pa, e = np.ones(P), np.ones(P), np.zeros(P)
    for k in range(K):
        out_v[:, k], out_b[:, k] = pv, e + max(k - 1, 0) * U * pa
        e = e * np.abs(v[:, k]) + b[:, k] * pa
        pv, pa = pv * v[:, k], pa * np.abs(v[:, k])
    full = F(pv, e + max(K - 1, 0) * U * pa)
    if reverse:
        out_v, out_b = out_v[:, ::-1], out_b[:, ::-1]
    return F(out_v, out_b), full


def recip(x):
    """1 / x as the kernels hold it: x rounded to float32, then its float32 reciprocal."""
    return F(1.0 / x, 2 * U / abs(x))


def coverage(d, v, inv_sigma):
    """p~ = 1 / (1 + expf(-x)), x = (-d) * (1 / sigma), and 1 - p~, for (P, K) float64 d and a 0 / 1 mask v."""
    y = d * inv_sigma.v
    pt, one_minus = expit(-y), expit(y)
    b = pt * U * (one_minus * (3 * np.abs(y) + 2) + 2) + underflow(pt)  # expf(-x) overflows past x = -88.7
    return F(pt, b), F(one_minus, b + U * one_minus)


# ------------------------------------------------------------------------------------------ z_inv as the kernels do
def is_number(x):
    return not torch.is_tensor(x) and not isinstance(x, np.ndarray)


def z_inv32(zbuf, valid, znear, zfar, img):
    """z_inv (P, K) float32, bit for bit the kernels' (zmap_of / z_inv_of), and d z_inv / d z (P,) with its bound.
    znear / zfar: numbers, or float32 (N,) arrays; img (P,): the image of each pixel."""
    v = valid.astype(np.float32)
    if is_number(znear) and is_number(zfar):
        R = np.float32(zfar - znear)  # the range in double, then float
        inv = np.float32(1.0) / R
        zi = ((np.float32(zfar) - zbuf) * inv) * v
        R = np.full(img.shape, float(R))
    else:
        zf = np.asarray(zfar, np.float32)[img] if not is_number(zfar) else np.full(img.shape, np.float32(zfar))
        zn = np.asarray(znear, np.float32)[img] if not is_number(znear) else np.full(img.shape, np.float32(znear))
        a = (zf - zn).astype(np.float32)
        zi = ((zf[:, None] - zbuf) / a[:, None]) * v
        R = a.astype(np.float64)
    assert zi.dtype == np.float32
    return zi, F(-1.0 / R, 2 * U / np.abs(R))


# ------------------------------------------------------------------------------------------ softmax reference
def _softmax_core(c, d, zi, v, g, sigma, gamma, bg, dzdz, argmax, m_passed, delta_passed):
    """One decision set: c (P, K, 3), d / zi / v (P, K), g (P, 4), bg (3,), dzdz F (P,), argmax / m_passed /
    delta_passed (P,).  Returns {name: F} of the forward pass, the three gradients and dm."""
    P, K = v.shape
    rows = np.arange(P)
    inv_sigma, inv_gamma = recip(sigma), recip(gamma)
    pt, one_minus_pt = coverage(d, v, inv_sigma)
    p = pt.masked(v)
    one_minus_p = F(v * one_minus_pt.v + (1 - v), one_minus_pt.b * v)
    pre, trans = excl_prod(one_minus_p)
    suf, _ = excl_prod(one_minus_p, reverse=True)
    alpha = F(1.0) - trans
    m = np.where(m_passed, zi[rows, argmax], EPS32)
    delta = where(delta_passed, ((F(EPS32) - F(m)) * inv_gamma).exp(), EPS32)
    e = ((F(zi) - F(m[:, None])) * inv_gamma).exp()
    w = p * e
    S = fsum(w, 1)
    A = fsum(w[:, :, None] * F(c), 1)
    D = S + delta
    r = (A + delta[:, None] * F(bg)) / D[:, None]
    # backward
    gc, ga = F(g[:, None, :3]), F(g[:, None, 3])
    inv_D = F(1.0) / D
    grad_colors = (w * inv_D[:, None])[:, :, None] * gc
    q = fsum((F(c) - r[:, None, :]) * gc, 2) * inv_D[:, None]
    dp = q * e + ga * (pre * suf)
    grad_dists = -(((pt.masked(v) * one_minus_pt) * inv_sigma) * dp)
    qw = q * w
    dzi = qw * inv_gamma
    t = fsum(qw, 1)
    t_delta = (delta * fsum((F(bg) - r) * F(g[:, :3]), 1)) * inv_D
    t = where(delta_passed, t + t_delta, t)
    dm = where(m_passed, -(t * inv_gamma), 0.0)
    grad_zbuf = (dzdz[:, None] * dzi).masked(v)
    at = (dzdz * (dzi[rows, argmax] + dm)).masked(v[rows, argmax])
    grad_zbuf.v[rows, argmax], grad_zbuf.b[rows, argmax] = at.v, at.b
    out = F(np.concatenate([r.v, alpha.v[:, None]], 1), np.concatenate([r.b, alpha.b[:, None]], 1))
    return {"out": out, "grad_colors": grad_colors, "grad_dists": grad_dists, "grad_zbuf": grad_zbuf, "dm": dm,
            "delta": delta}


def softmax_decisions(zi, sigma, gamma):
    """argmax (first slot attaining the float32 maximum), m_passed, and delta_passed as (surely, possibly)."""
    zmax = zi.max(1)
    argmax = np.argmax(zi, 1)  # the first occurrence
    m_passed = zmax >= np.float32(EPS32)
    m = np.where(m_passed, zmax, EPS32).astype(np.float64)
    de = ((F(EPS32) - F(m)) * recip(gamma)).exp()
    open_ = np.abs(de.v - EPS32) <= 2 * de.b + FLOOR
    passed = de.v >= EPS32
    return argmax, m_passed, passed & ~open_, passed | open_


def ref_softmax(scene, sigma, gamma, bg, znear, zfar, chunk=16384):
    """{name: (lo, hi, beta)} in the ops' shapes, and the decisions {argmax, m_passed, delta_passed, delta_open,
    argmax_last} per pixel."""
    N, H, W, K = scene["p2f"].shape
    P = N * H * W
    valid = (scene["p2f"] >= 0).reshape(P, K)
    img = np.arange(P) // (H * W)
    zi, dzdz = z_inv32(scene["zbuf"].reshape(P, K), valid, znear, zfar, img)
    c = scene["colors"].reshape(P, K, 3).astype(np.float64)
    d = scene["dists"].reshape(P, K).astype(np.float64)
    g = scene["grad"].reshape(P, 4).astype(np.float64)
    bgv = np.asarray([float(x) for x in bg], np.float64)
    v = valid.astype(np.float64)
    argmax, m_passed, surely, possibly = softmax_decisions(zi, sigma, gamma)
    names = ("out", "grad_colors", "grad_dists", "grad_zbuf")
    parts = {n: [] for n in names}
    for s in range(0, P, chunk):
        sl = slice(s, min(P, s + chunk))
        args = (c[sl], d[sl], zi[sl].astype(np.float64), v[sl], g[sl], sigma, gamma, bgv, dzdz[sl], argmax[sl],
                m_passed[sl])
        a = _softmax_core(*args, surely[sl])
        b = _softmax_core(*args, possibly[sl]) if (surely[sl] != possibly[sl]).any() else a
        for n in names:
            parts[n].append((np.minimum(a[n].v, b[n].v), np.maximum(a[n].v, b[n].v), np.maximum(a[n].b, b[n].b)))
    shapes = {"out": (N, H, W, 4), "grad_colors": (N, H, W, K, 3), "grad_dists": (N, H, W, K),
              "grad_zbuf": (N, H, W, K)}
    ref = {n: tuple(np.concatenate([p[i] for p in parts[n]]).reshape(shapes[n]) for i in range(3)) for n in names}
    last = K - 1 - np.argmax(zi[:, ::-1], 1)
    info = {"argmax": argmax, "m_passed": m_passed, "delta_passed": surely, "delta_open": possibly & ~surely,
            "argmax_last": last, "zi": zi, "valid": valid, "tied_rows": _tied_rows(zi, argmax)}
    return ref, info


def _tied_rows(zi, argmax):
    """Per pixel: the slots attaining the maximum span more than one row of 32."""
    top = zi == zi.max(1, keepdims=True)
    rows = np.arange(zi.shape[1]) // 32
    lo = np.where(top, rows, 99).min(1)
    hi = np.where(top, rows, -1).max(1)
    return hi > lo


# ------------------------------------------------------------------------------------------ soft depth reference
def _depth_core(d, z, zf, v, g, sigma, sure, maybe):
    """d / z / v (P, K), zf / g (P,), sure / maybe (P, K + 1): masks c_k <= 1 that hold surely / may hold.
    Returns {name: (lo, hi, F)}."""
    P, K = v.shape
    inv_sigma = recip(sigma)
    pt, one_minus_pt = coverage(d, v, inv_sigma)
    p = pt.masked(v)
    pv = np.concatenate([p.v, np.ones((P, 1))], 1)
    pb = np.concatenate([p.b, np.zeros((P, 1))], 1)
    n = np.arange(K + 1)
    c = F(pv.cumsum(1), pb.cumsum(1) + n * U * np.abs(pv).cumsum(1))
    possible = sure | maybe
    cl = F(np.minimum(c.v, 1.0), c.b * possible)
    cl_prev = F(np.concatenate([np.zeros((P, 1)), cl.v[:, :-1]], 1),
                np.concatenate([np.zeros((P, 1)), cl.b[:, :-1]], 1))
    wk = cl - cl_prev
    depth = F(np.concatenate([z, zf[:, None]], 1))
    out = fsum(wk * depth, 1)
    grad_zbuf = (F(g[:, None]) * wk)[:, :K]
    gw = F(g[:, None]) * depth
    gw_next = F(np.concatenate([gw.v[:, 1:], np.zeros((P, 1))], 1), np.concatenate([gw.b[:, 1:], np.zeros((P, 1))], 1))
    gct = gw - gw_next
    rev = lambda x: x[:, ::-1].cumsum(1)[:, ::-1]  # noqa: E731  (sum over the slots >= k)
    open_ = maybe & ~sure
    gp_lo = rev(gct.v * sure + np.minimum(gct.v, 0) * open_)
    gp_hi = rev(gct.v * sure + np.maximum(gct.v, 0) * open_)
    cnt = K - n  # terms after the first in the sum over j >= k
    gp = F(np.maximum(np.abs(gp_lo), np.abs(gp_hi)), rev(gct.b * possible) + cnt * U * rev(np.abs(gct.v) * possible))
    chain = ((gp[:, :K].masked(v) * one_minus_pt) * pt) * inv_sigma
    f = v * one_minus_pt.v * pt.v * inv_sigma.v
    lo, hi = -gp_hi[:, :K] * f, -gp_lo[:, :K] * f
    return {"out": (out.v, out.v, out), "grad_zbuf": (grad_zbuf.v, grad_zbuf.v, grad_zbuf),
            "grad_dists": (lo, hi, chain)}


def depth_masks(d, v, sigma, c):
    """(sure, maybe) for c_k <= 1, (P, K + 1), given the float64 prefix sums c (F)."""
    P, K = v.shape
    y = d / sigma
    exact = (v == 0) | (d == 0) | (np.abs(y) >= 30)
    pe = np.where(v == 0, 0.0, np.where(d == 0, 0.5, np.where(y <= -30, 1.0, 0.0)))
    exact = np.concatenate([exact, np.ones((P, 1), bool)], 1)
    pe = np.concatenate([pe, np.ones((P, 1))], 1)
    all_exact = np.logical_and.accumulate(exact, 1)
    open_ = ~all_exact & (np.abs(c.v - 1) <= 2 * c.b + FLOOR)
    sure = np.where(all_exact, pe.cumsum(1) <= 1, (c.v <= 1) & ~open_)
    return sure, sure | open_


def ref_soft_depth(scene, sigma, zfar, chunk=16384):
    """{name: (lo, hi, beta)} in the ops' shapes, and {sure, maybe} masks."""
    N, H, W, K = scene["p2f"].shape
    P = N * H * W
    v = (scene["p2f"] >= 0).reshape(P, K).astype(np.float64)
    d = scene["dists"].reshape(P, K).astype(np.float64)
    z = scene["zbuf"].reshape(P, K).astype(np.float64)
    g = scene["grad"][..., 0].reshape(P).astype(np.float64)
    zf = np.full(P, float(np.float32(float(zfar))))
    pt, _ = coverage(d, v, recip(sigma))
    p = pt.masked(v)
    pv = np.concatenate([p.v, np.ones((P, 1))], 1)
    pb = np.concatenate([p.b, np.zeros((P, 1))], 1)
    c = F(pv.cumsum(1), pb.cumsum(1) + np.arange(K + 1) * U * np.abs(pv).cumsum(1))
    sure, maybe = depth_masks(d, v, sigma, c)
    parts = {n: [] for n in ("out", "grad_zbuf", "grad_dists")}
    for s in range(0, P, chunk):
        sl = slice(s, min(P, s + chunk))
        r = _depth_core(d[sl], z[sl], zf[sl], v[sl], g[sl], sigma, sure[sl], maybe[sl])
        for n, (lo, hi, f) in r.items():
            parts[n].append((lo, hi, f.b))
    shapes = {"out": (N, H, W, 1), "grad_zbuf": (N, H, W, K), "grad_dists": (N, H, W, K)}
    ref = {n: tuple(np.concatenate([p[i] for p in parts[n]]).reshape(shapes[n]) for i in range(3)) for n in parts}
    return ref, {"sure": sure, "maybe": maybe, "c": c.v}


# ------------------------------------------------------------------------------------------ comparison
def assert_within(name, got, ref):
    """|got - [lo, hi]| <= 2 beta + 2^-126 for every element (NaN fails)."""
    lo, hi, beta = ref
    got = np.asarray(got.detach().cpu().numpy() if torch.is_tensor(got) else got, dtype=np.float64)
    assert got.shape == lo.shape, (name, got.shape, lo.shape)
    err = np.maximum(np.maximum(lo - got, got - hi), 0.0)
    tol = 2 * beta + FLOOR
    bad = ~(err <= tol)
    if bad.any():
        ratio = np.where(bad, np.nan_to_num(err / tol, nan=np.inf), 0.0)
        at = np.unravel_index(int(np.argmax(ratio)), got.shape)
        raise AssertionError("%s: %d of %d elements outside 2 beta + 2^-126; worst at %s: got %.9g, want [%.9g, %.9g], "
                             "beta %.3g (%.3g x the bound)" % (name, int(bad.sum()), got.size, at, got[at], lo[at],
                                                               hi[at], beta[at], ratio[at]))


def count_outside(got, ref):
    lo, hi, beta = ref
    got = np.asarray(got.detach().cpu().numpy(), dtype=np.float64)
    err = np.maximum(np.maximum(lo - got, got - hi), 0.0)
    return int((~(err <= 2 * beta + FLOOR)).sum())


# ------------------------------------------------------------------------------------------ scenes
# Every pixel of a scene has a slot layout (trailing empties, interleaved empties, all empty, all valid), a depth
# kind (in range, every covered slot at or beyond zfar, some slots before znear) and a tie kind (none, a tie inside a
# row of 32 slots, a tie of slots k and k + 32, a tie across rows and lanes), cycled so that every combination occurs.
KS = [1, 2, 3, 7, 8, 9, 31, 32, 33, 63, 64, 65, 96, 97, 128, 129, 150]
Z_KINDS = ["numbers", "tensors", "znear_tensor", "zfar_tensor"]
SIGMAS = [1e-4, 1e-2]
GAMMAS = [1e-4, 1e-2, 0.5]
ZN, ZF = 0.7, 43.3  # the numbers: a range that is not a float32 power of two


def z_params(kind, N, seed):
    """znear, zfar of a kind: numbers or float32 (N,) numpy arrays."""
    rng = np.random.default_rng(seed + 1000)
    zn_t = (0.5 + rng.random(N)).astype(np.float32)
    zf_t = (20.0 + 80.0 * rng.random(N)).astype(np.float32)
    return {"numbers": (ZN, ZF), "tensors": (zn_t, zf_t), "znear_tensor": (zn_t, ZF),
            "zfar_tensor": (ZN, zf_t)}[kind]


def _per_image(x, N):
    return np.full(N, np.float32(x)) if is_number(x) else np.asarray(x, np.float32)


def make_scene(N, H, W, K, sigma, znear, zfar, seed=0, ties=True):
    """colors (N,H,W,K,3), p2f (N,H,W,K), zbuf (N,H,W,K) (-1 in empty slots), dists, grad (N,H,W,4): numpy."""
    rng = np.random.default_rng(seed + 7 * K)
    P = N * H * W
    pix = np.arange(P)
    img = pix // (H * W)
    layout, depth_kind, tie_kind = pix % 4, (pix // 4) % 3, (pix // 12) % 4
    ks = np.arange(K)
    valid = np.empty((P, K), bool)
    valid[:] = (ks[None] < rng.integers(0, K + 1, P)[:, None])
    inter = rng.random((P, K)) < 0.6
    valid = np.where((layout == 1)[:, None], inter, valid)
    valid[layout == 2] = False
    valid[layout == 3] = True
    zn, zf = _per_image(znear, N)[img][:, None], _per_image(zfar, N)[img][:, None]
    z = zn + (zf - zn) * (0.02 + 0.96 * rng.random((P, K)))
    beyond = zf + np.where(rng.random((P, K)) < 0.5, 0.0, 5.0 * rng.random((P, K)))  # half of them exactly zfar
    z = np.where((depth_kind == 1)[:, None], beyond, z)
    near = zn * rng.random((P, K))
    z = np.where((depth_kind == 2)[:, None] & (rng.random((P, K)) < 0.3), near, z)
    z = z.astype(np.float32)
    if ties and K > 1:
        for i in np.nonzero((tie_kind > 0) & (depth_kind != 1))[0][:4096]:
            vi = np.nonzero(valid[i])[0]
            if len(vi) < 2:
                continue
            a = vi[rng.integers(len(vi))]
            others = vi[vi != a]
            sel = {1: others // 32 == a // 32, 2: others % 32 == a % 32,
                   3: (others // 32 != a // 32) & (others % 32 != a % 32)}[int(tie_kind[i])]
            cand = others[sel] if sel.any() else others
            z[i, a] = z[i, cand[rng.integers(len(cand))]] = z[i, vi].min()
    z[~valid] = -1.0
    t = rng.normal(0.0, 2.0, (P, K))
    r = rng.random((P, K))
    t = np.where(r < 0.1, -40.0, np.where(r < 0.2, 40.0, np.where(r < 0.25, 120.0, np.where(r < 0.3, 0.0, t))))
    half = ((pix // 48) % 2 == 1)  # the first two valid slots at d = 0: coverage 1/2 + 1/2 = 1 exactly
    for i in np.nonzero(half)[0][:4096]:
        t[i, np.nonzero(valid[i])[0][:2]] = 0.0
    dists = (t * sigma).astype(np.float32)
    colors = ((rng.random((P, K, 3)) * 2 - 1) * 10).astype(np.float32)
    same = (pix // 96) % 2 == 1  # one colour per pixel: c_k - rgb cancels
    colors[same] = colors[same][:, :1]
    p2f = np.where(valid, rng.integers(0, 1000, (P, K)), -1)
    grad = rng.normal(0.0, 1.0, (P, 4)).astype(np.float32)
    return {"colors": colors.reshape(N, H, W, K, 3), "p2f": p2f.reshape(N, H, W, K),
            "zbuf": z.reshape(N, H, W, K), "dists": dists.reshape(N, H, W, K), "grad": grad.reshape(N, H, W, 4)}


def clamp_gammas(scene, znear, zfar):
    """gamma just above and just below m / 23.03 for the median m of the scene's covered pixels: delta passes its
    clamp on one side of the median and not on the other."""
    N, H, W, K = scene["p2f"].shape
    P = N * H * W
    valid = (scene["p2f"] >= 0).reshape(P, K)
    zi, _ = z_inv32(scene["zbuf"].reshape(P, K), valid, znear, zfar, np.arange(P) // (H * W))
    m = zi.max(1).astype(np.float64)
    m = m[valid.any(1) & (m > 1e-3)]
    med = float(np.median(m)) if m.size else 0.5
    return [(med - EPS32) / LN_EPS * 1.002, (med - EPS32) / LN_EPS / 1.002]


def torch_inputs(scene, device="cpu"):
    return [torch.from_numpy(np.ascontiguousarray(scene[k])).to(device)
            for k in ("colors", "p2f", "zbuf", "dists", "grad")]


def z_torch(x, device):
    return x if is_number(x) else torch.from_numpy(np.asarray(x, np.float32)).to(device)


# ------------------------------------------------------------------------------------------ the float32 chains
def chain_softmax(colors, p2f, zbuf, dists, sigma, gamma, bg, znear, zfar, argmax, defect=None):
    """The chain of test_blending.softmax_chain, its maximum taken at `argmax` (N,H,W).  For numbers znear / zfar,
    z_inv is the product with the float32 reciprocal of the range, as torch computes it on CUDA (its CPU kernels
    divide).  `defect` breaks one step of the gradient."""
    valid = p2f >= 0
    prob = torch.sigmoid(-dists / sigma) * valid
    T = torch.prod(1.0 - prob, dim=-1)
    if defect == "prefix":  # d alpha / d p_k = prod_{l <= k} ... prod_{l > k}: the prefix taken one slot too far
        T = T.detach()
        s = (prob * T[..., None]).sum(-1)
        alpha = (1.0 - T) + (s - s.detach())
    else:
        alpha = 1.0 - T
    if is_number(znear) and is_number(zfar):
        z_inv = (zfar - zbuf) * float(np.float32(1.0) / np.float32(zfar - znear)) * valid
    else:
        zf = zfar[:, None, None, None] if torch.is_tensor(zfar) else zfar
        zn = znear[:, None, None, None] if torch.is_tensor(znear) else znear
        z_inv = (zf - zbuf) / (zf - zn) * valid
    z_max = z_inv.gather(-1, argmax[..., None]).clamp(min=1e-10)
    if defect == "detach_zmax":
        z_max = z_max.detach()
    w = prob * torch.exp((z_inv - z_max) / gamma)
    z_delta = z_max.detach() if defect == "drop_delta" else z_max
    delta = torch.exp((1e-10 - z_delta) / gamma).clamp(min=1e-10)
    denom = w.sum(dim=-1)[..., None] + delta
    bg = bg if torch.is_tensor(bg) else torch.tensor(bg, dtype=torch.float32)
    rgb = ((w[..., None] * colors).sum(dim=-2) + delta * bg) / denom
    return torch.cat([rgb, alpha[..., None]], -1)


def chain_soft_depth(p2f, zbuf, dists, sigma, zfar, defect=None):
    """test_depth_shading.soft_depth_chain; `defect` "lt" passes the clamp's gradient only where c_k < 1."""
    N, H, W, K = p2f.shape
    prob = torch.sigmoid(-dists / sigma) * (p2f >= 0)
    depth = torch.cat((zbuf, torch.ones((N, H, W, 1), dtype=zbuf.dtype) * zfar), dim=3)
    c = torch.cat((prob, torch.ones((N, H, W, 1), dtype=zbuf.dtype)), dim=3).cumsum(dim=3)
    c = torch.where(c < 1, c, torch.ones_like(c)) if defect == "lt" else c.clamp(max=1)
    w = c.diff(dim=3, prepend=torch.zeros((N, H, W, 1), dtype=zbuf.dtype))
    return (w * depth).sum(dim=3).unsqueeze(3)


def run_softmax_chain(scene, sigma, gamma, bg, znear, zfar, argmax, defect=None):
    colors, p2f, zbuf, dists, grad = torch_inputs(scene)
    c, z, d = (t.clone().requires_grad_(True) for t in (colors, zbuf, dists))
    out = chain_softmax(c, p2f, z, d, sigma, gamma, bg, z_torch(znear, "cpu"), z_torch(zfar, "cpu"),
                        torch.from_numpy(argmax.reshape(p2f.shape[:3])), defect)
    out.backward(grad)
    return {"out": out.detach(), "grad_colors": c.grad, "grad_dists": d.grad, "grad_zbuf": z.grad}


def run_depth_chain(scene, sigma, zfar, defect=None):
    _, p2f, zbuf, dists, grad = torch_inputs(scene)
    z, d = zbuf.clone().requires_grad_(True), dists.clone().requires_grad_(True)
    out = chain_soft_depth(p2f, z, d, sigma, zfar, defect)
    out.backward(grad[..., :1])
    return {"out": out.detach(), "grad_zbuf": z.grad, "grad_dists": d.grad}


# ------------------------------------------------------------------------------------------ CPU: the reference
CPU_SCENES = [(K, zk) for K in (1, 3, 8, 9, 33, 65, 97) for zk in Z_KINDS]


def _autograd_softmax(scene, sigma, gamma, bg, znear, zfar, argmax, m_passed, delta_passed, dzdz, zi):
    """The header's forward formulas in float64 torch with the same decisions; z_inv has the float32 values and
    derivative dzdz."""
    N, H, W, K = scene["p2f"].shape
    P = N * H * W
    c = torch.tensor(scene["colors"].reshape(P, K, 3), dtype=torch.float64, requires_grad=True)
    d = torch.tensor(scene["dists"].reshape(P, K), dtype=torch.float64, requires_grad=True)
    z = torch.tensor(scene["zbuf"].reshape(P, K), dtype=torch.float64, requires_grad=True)
    v = torch.tensor((scene["p2f"] >= 0).reshape(P, K), dtype=torch.float64)
    prob = torch.sigmoid(-d / sigma) * v
    alpha = 1 - torch.prod(1 - prob, 1)
    zinv = (torch.tensor(zi, dtype=torch.float64) + (z - z.detach()) * torch.tensor(dzdz.v)[:, None]) * v
    rows = torch.arange(P)
    m = torch.where(torch.tensor(m_passed), zinv[rows, torch.tensor(argmax)], torch.full((P,), EPS32,
                                                                                      dtype=torch.float64))
    w = prob * torch.exp((zinv - m[:, None]) / gamma)
    delta = torch.where(torch.tensor(delta_passed), torch.exp((EPS32 - m) / gamma), torch.full_like(m, EPS32))
    bgt = torch.tensor([float(x) for x in bg], dtype=torch.float64)
    D = w.sum(1) + delta
    rgb = ((w[:, :, None] * c).sum(1) + delta[:, None] * bgt) / D[:, None]
    out = torch.cat([rgb, alpha[:, None]], 1)
    out.backward(torch.tensor(scene["grad"].reshape(P, 4), dtype=torch.float64))
    return {"out": out.detach().numpy(), "grad_colors": c.grad.numpy(), "grad_dists": d.grad.numpy(),
            "grad_zbuf": z.grad.numpy()}


@pytest.mark.parametrize("K,zk", CPU_SCENES)
def test_softmax_reference_equals_autograd(K, zk):
    """The gradients written out from the header's backward formulas equal float64 autograd of its forward formulas,
    with the same decisions, to far below the float32 bound."""
    znear, zfar = z_params(zk, 2, K)
    scene = make_scene(2, 6, 8, K, 1e-2, znear, zfar, seed=K)
    N, H, W, _ = scene["p2f"].shape
    P = N * H * W
    valid = (scene["p2f"] >= 0).reshape(P, K)
    zi, dzdz = z_inv32(scene["zbuf"].reshape(P, K), valid, znear, zfar, np.arange(P) // (H * W))
    for gamma in GAMMAS + clamp_gammas(scene, znear, zfar):
        argmax, m_passed, surely, _ = softmax_decisions(zi, 1e-2, gamma)
        bg = (0.2, -3.0, 7.5)
        got = _softmax_core(scene["colors"].reshape(P, K, 3).astype(np.float64),
                            scene["dists"].reshape(P, K).astype(np.float64), zi.astype(np.float64),
                            valid.astype(np.float64), scene["grad"].reshape(P, 4).astype(np.float64), 1e-2, gamma,
                            np.asarray(bg), dzdz, argmax, m_passed, surely)
        want = _autograd_softmax(scene, 1e-2, gamma, bg, znear, zfar, argmax, m_passed, surely, dzdz, zi)
        for name in want:
            err = np.abs(got[name].v - want[name])
            assert (err <= 1e-6 * got[name].b + 1e-300).all(), (name, gamma, float(err.max()))


@pytest.mark.parametrize("K", [1, 3, 8, 9, 33, 64, 97, 150])
def test_soft_depth_reference_equals_autograd(K):
    scene = make_scene(2, 6, 8, K, 1e-2, ZN, ZF, seed=K + 1)
    N, H, W, _ = scene["p2f"].shape
    P = N * H * W
    ref, masks = ref_soft_depth(scene, 1e-2, 20.0)
    mask = torch.tensor(masks["sure"])
    d = torch.tensor(scene["dists"].reshape(P, K), dtype=torch.float64, requires_grad=True)
    z = torch.tensor(scene["zbuf"].reshape(P, K), dtype=torch.float64, requires_grad=True)
    v = torch.tensor((scene["p2f"] >= 0).reshape(P, K), dtype=torch.float64)
    p = torch.cat([torch.sigmoid(-d / 1e-2) * v, torch.ones(P, 1, dtype=torch.float64)], 1)
    c = p.cumsum(1)
    cl = c.detach().clamp(max=1) + torch.where(mask, c - c.detach(), torch.zeros_like(c))
    w = cl.diff(dim=1, prepend=torch.zeros(P, 1, dtype=torch.float64))
    depth = torch.cat([z, torch.full((P, 1), float(np.float32(20.0)), dtype=torch.float64)], 1)
    out = (w * depth).sum(1)
    out.backward(torch.tensor(scene["grad"][..., 0].reshape(P), dtype=torch.float64))
    want = {"out": out.detach().numpy().reshape(N, H, W, 1), "grad_zbuf": z.grad.numpy().reshape(N, H, W, K),
            "grad_dists": d.grad.numpy().reshape(N, H, W, K)}
    for name, x in want.items():
        lo, hi, beta = ref[name]  # autograd takes the open masks as false, one end of the reference's interval
        err = np.maximum(np.maximum(lo - x, x - hi), 0.0)
        assert (err <= 1e-6 * beta + 1e-300).all(), name
        assert name == "grad_dists" or np.array_equal(lo, hi)


def test_reference_closed_form():
    """One pixel, K = 2, gamma = 0.5: the forward pass written out by hand."""
    sigma, gamma, bg = 1.0, 0.5, (0.0, 0.0, 1.0)
    scene = {"colors": np.array([[[[[1.0, 0, 0], [0, 1.0, 0]]]]], np.float32), "p2f": np.array([[[[3, 4]]]]),
             "zbuf": np.array([[[[2.0, 3.0]]]], np.float32), "dists": np.array([[[[0.0, 0.0]]]], np.float32),
             "grad": np.zeros((1, 1, 1, 4), np.float32)}
    ref, info = ref_softmax(scene, sigma, gamma, bg, 1.0, 5.0)
    zi = np.array([0.75, 0.5])  # (5 - z) / 4
    w = 0.5 * np.exp((zi - 0.75) / gamma)  # p = sigmoid(0) = 1/2
    delta = np.exp((EPS32 - 0.75) / gamma)
    want = np.array([w[0], w[1], delta, 0.0]) / (w.sum() + delta)
    want[3] = 1 - 0.5 * 0.5
    np.testing.assert_allclose(ref["out"][0].reshape(4), want, rtol=1e-14)
    assert int(info["argmax"][0]) == 0 and bool(info["m_passed"][0]) and bool(info["delta_passed"][0])


# ------------------------------------------------------------------------------------------ CPU: the bound is honest
@pytest.mark.parametrize("K,zk", CPU_SCENES)
def test_softmax_chain_within_bound(K, zk):
    """The float32 torch chain, its maximum at the reference's argmax, lies within the bound."""
    znear, zfar = z_params(zk, 2, K)
    for sigma in SIGMAS:
        scene = make_scene(2, 8, 8, K, sigma, znear, zfar, seed=K)
        for gamma in GAMMAS + clamp_gammas(scene, znear, zfar):
            bg = (0.3, -2.0, 9.5)
            ref, info = ref_softmax(scene, sigma, gamma, bg, znear, zfar)
            got = run_softmax_chain(scene, sigma, gamma, bg, znear, zfar, info["argmax"])
            for name, x in got.items():
                assert_within("K=%d %s sigma=%g gamma=%g %s" % (K, zk, sigma, gamma, name), x, ref[name])


DEFECTS = ["detach_zmax", "drop_delta", "last_tied", "prefix"]


@pytest.mark.parametrize("defect", DEFECTS)
def test_softmax_defective_chain_fails(defect):
    """Each defect puts elements of the gradient outside the bound on the matrix's scenes."""
    outside = 0
    for K, zk in [(3, "numbers"), (9, "tensors"), (65, "zfar_tensor")]:
        znear, zfar = z_params(zk, 2, K)
        scene = make_scene(2, 8, 8, K, 1e-2, znear, zfar, seed=K)
        for gamma in (1e-2, 0.5):
            ref, info = ref_softmax(scene, 1e-2, gamma, (0.3, -2.0, 9.5), znear, zfar)
            argmax = info["argmax_last"] if defect == "last_tied" else info["argmax"]
            got = run_softmax_chain(scene, 1e-2, gamma, (0.3, -2.0, 9.5), znear, zfar, argmax,
                                    None if defect == "last_tied" else defect)
            outside += sum(count_outside(got[n], ref[n]) for n in got)
    assert outside > 0, "the %s chain passes the bound" % defect


@pytest.mark.parametrize("K", [1, 3, 8, 9, 33, 64, 97, 150])
@pytest.mark.parametrize("sigma", SIGMAS)
def test_soft_depth_chain_within_bound(K, sigma):
    scene = make_scene(2, 8, 8, K, sigma, ZN, ZF, seed=K + 1)
    for zfar in (20.0, 41.25):
        ref, _ = ref_soft_depth(scene, sigma, zfar)
        got = run_depth_chain(scene, sigma, zfar)
        for name, x in got.items():
            assert_within("K=%d sigma=%g %s" % (K, sigma, name), x, ref[name])


def test_soft_depth_defective_chain_fails():
    """The clamp's test c_k <= 1 replaced by c_k < 1: pixels whose coverage reaches 1 exactly lose the gradient of
    their later slots."""
    outside = 0
    for K in (3, 9, 33):
        scene = make_scene(2, 8, 8, K, 1e-2, ZN, ZF, seed=K + 1)
        ref, _ = ref_soft_depth(scene, 1e-2, 20.0)
        got = run_depth_chain(scene, 1e-2, 20.0, defect="lt")
        outside += sum(count_outside(got[n], ref[n]) for n in got)
    assert outside > 0


def test_restated_chains_equal_the_suites_chains():
    """chain_softmax and chain_soft_depth are the chains of test_blending / test_depth_shading: equal forward values
    where the maximum is not tied and z_inv is computed alike (tensors), and equal soft depth."""
    znear, zfar = z_params("tensors", 2, 0)
    scene = make_scene(2, 8, 8, 9, 1e-2, znear, zfar, seed=3, ties=False)
    colors, p2f, zbuf, dists, _ = torch_inputs(scene)
    zn, zf = z_torch(znear, "cpu"), z_torch(zfar, "cpu")
    _, info = ref_softmax(scene, 1e-2, 1e-2, (1.0, 1.0, 1.0), znear, zfar)
    a = chain_softmax(colors, p2f, zbuf, dists, 1e-2, 1e-2, (1.0, 1.0, 1.0), zn, zf,
                      torch.from_numpy(info["argmax"].reshape(p2f.shape[:3])))
    b = softmax_chain(colors, p2f, zbuf, dists, 1e-2, 1e-2, (1.0, 1.0, 1.0), zn, zf)
    assert torch.equal(a, b)
    assert torch.equal(chain_soft_depth(p2f, zbuf, dists, 1e-2, 20.0), soft_depth_chain(p2f, zbuf, dists, 1e-2, 20.0))


def test_scenes_reach_every_edge():
    """The matrix launches softmax NS 1..5 and soft depth NS 1..5 on both sides of each boundary, and its scenes hold
    covered pixels with m_passed false, pixels on both sides of the delta clamp, ties across rows and lanes, ties with
    an empty slot's z_inv = 0, and coverages that reach 1 exactly."""
    assert {-(-K // 32) for K in KS if K > 8} == {1, 2, 3, 4, 5}
    assert {-(-(K + 1) // 32) for K in KS if K > 8} == {1, 2, 3, 4, 5}
    for ns in (3, 4):
        assert sum(1 for K in KS if K > 8 and -(-K // 32) == ns) >= 2
        assert sum(1 for K in KS if K > 8 and -(-(K + 1) // 32) == ns) >= 2
    m_false_covered = delta_sides = tied_rows = empty_tie = 0
    passed, clamped = 0, 0
    for K in (8, 40, 97):
        znear, zfar = z_params("numbers", 2, K)
        scene = make_scene(2, 8, 8, K, 1e-2, znear, zfar, seed=K)
        for gamma in clamp_gammas(scene, znear, zfar):
            _, info = ref_softmax(scene, 1e-2, gamma, (1.0, 1.0, 1.0), znear, zfar)
            covered = info["valid"].any(1)
            m_false_covered += int((covered & ~info["m_passed"]).sum())
            passed += int((info["m_passed"] & info["delta_passed"]).sum())
            clamped += int((info["m_passed"] & ~info["delta_passed"] & ~info["delta_open"]).sum())
            tied_rows += int(info["tied_rows"].sum())
            rows = np.arange(len(covered))  # the maximum 0 at an empty slot, tied by a covered slot at zfar
            empty_tie += int((~info["valid"][rows, info["argmax"]] & ((info["zi"] == 0) & info["valid"]).any(1)).sum())
    assert m_false_covered > 0 and passed > 0 and clamped > 0 and tied_rows > 0 and empty_tie > 0
    scene = make_scene(2, 8, 8, 9, 1e-2, ZN, ZF, seed=10)
    _, masks = ref_soft_depth(scene, 1e-2, 20.0)
    assert (masks["sure"] & (masks["c"] == 1)).any()


# ------------------------------------------------------------------------------------------ GPU
DEV = "cuda:0"


def _softmax_gpu(scene, sigma, gamma, bg, znear, zfar, what, shift=False):
    """The fused ops through _C, compared with the reference element by element."""
    from pytorch3d_b200 import _C
    colors, p2f, zbuf, dists, grad = torch_inputs(scene, DEV)
    if shift:
        colors, p2f, zbuf, dists, grad = (shifted(t) for t in (colors, p2f, zbuf, dists, grad))
    bgd = torch.tensor(bg, dtype=torch.float32, device=DEV) if isinstance(bg, list) else bg
    zn, zf = z_torch(znear, DEV), z_torch(zfar, DEV)
    out = _C.softmax_rgb_blend(colors, p2f, zbuf, dists, sigma, gamma, bgd, zn, zf)
    gc, gd, gz = _C.softmax_rgb_blend_backward(grad, colors, p2f, zbuf, dists, sigma, gamma, bgd, zn, zf)
    ref, info = ref_softmax(scene, sigma, gamma, bg, znear, zfar)
    for name, x in (("out", out), ("grad_colors", gc), ("grad_dists", gd), ("grad_zbuf", gz)):
        assert_within("%s sigma=%g gamma=%g %s" % (what, sigma, gamma, name), x, ref[name])
    return info


def shifted(t):
    """A contiguous copy whose storage starts one element past a 16-byte boundary."""
    flat = torch.empty(t.numel() + 4, dtype=t.dtype, device=t.device)
    base = (16 - flat.data_ptr() % 16) % 16 // t.element_size()
    out = flat[base + 1:base + 1 + t.numel()].view(t.shape)
    out.copy_(t)
    assert out.data_ptr() % 16 != 0 and out.is_contiguous()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("zk", Z_KINDS)
@pytest.mark.parametrize("K", KS)
def test_softmax_matches_fp64(built_lib, K, zk):
    """K from 1 to 150: the register kernel and the warp kernel with NS = 1..5 on both sides of each boundary."""
    znear, zfar = z_params(zk, 2, K)
    for i, sigma in enumerate(SIGMAS):
        scene = make_scene(2, 8, 8, K, sigma, znear, zfar, seed=K)
        for j, gamma in enumerate(GAMMAS + clamp_gammas(scene, znear, zfar)):
            bg = [0.3, -2.0, 9.5] if (i + j) % 2 else (0.3, -2.0, 9.5)  # a list: a device tensor
            _softmax_gpu(scene, sigma, gamma, bg, znear, zfar, "K=%d %s" % (K, zk))


@pytest.mark.gpu
@pytest.mark.parametrize("aligned", [True, False])
def test_softmax_k8_vector_and_scalar_paths(built_lib, aligned):
    """K = 8 from 16-byte aligned storage (the 16-byte loads and stores) and from one float past it (scalar)."""
    znear, zfar = z_params("tensors", 2, 8)
    scene = make_scene(2, 8, 8, 8, 1e-2, znear, zfar, seed=80)
    if aligned:
        assert all(t.data_ptr() % 16 == 0 for t in torch_inputs(scene, DEV))
    for gamma in GAMMAS + clamp_gammas(scene, znear, zfar):
        _softmax_gpu(scene, 1e-2, gamma, [0.3, -2.0, 9.5], znear, zfar, "K=8 aligned=%s" % aligned,
                     shift=not aligned)


@pytest.mark.gpu
@pytest.mark.parametrize("N,S,K", [(2, 768, 1), (1, 200, 40), (1, 200, 97)])
def test_softmax_grid_stride_second_pass(built_lib, N, S, K):
    """More pixels than the capped grid holds (32 CTAs per SM; 256 pixels per CTA for K <= 8, 8 for K > 8)."""
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    assert N * S * S > sms * 32 * (256 if K <= 8 else 8)
    znear, zfar = z_params("tensors", N, K)
    scene = make_scene(N, S, S, K, 1e-2, znear, zfar, seed=K + 3)
    _softmax_gpu(scene, 1e-2, 1e-2, (0.3, -2.0, 9.5), znear, zfar, "grid stride K=%d" % K)


def _depth_gpu(scene, sigma, zfar, what, shift=False):
    from pytorch3d_b200 import _C
    _, p2f, zbuf, dists, grad = torch_inputs(scene, DEV)
    g = grad[..., :1].contiguous()
    if shift:
        p2f, zbuf, dists, g = (shifted(t) for t in (p2f, zbuf, dists, g))
    zf = torch.tensor([zfar], dtype=torch.float32, device=DEV) if isinstance(zfar, list) else zfar
    out = _C.soft_depth_blend(p2f, zbuf, dists, sigma, zf)
    gz, gd = _C.soft_depth_blend_backward(g, p2f, zbuf, dists, sigma, zf)
    ref, _ = ref_soft_depth(scene, sigma, zfar[0] if isinstance(zfar, list) else zfar)
    for name, x in (("out", out), ("grad_zbuf", gz), ("grad_dists", gd)):
        assert_within("%s sigma=%g %s" % (what, sigma, name), x, ref[name])


@pytest.mark.gpu
@pytest.mark.parametrize("K", KS)
def test_soft_depth_matches_fp64(built_lib, K):
    """K from 1 to 150: the register kernel and the warp kernel with NS = ceil((K + 1) / 32) = 1..5."""
    for sigma in SIGMAS:
        scene = make_scene(2, 8, 8, K, sigma, ZN, ZF, seed=K + 1)
        for zfar in (20.0, [41.25]):  # a number, a device tensor
            _depth_gpu(scene, sigma, zfar, "K=%d" % K)


@pytest.mark.gpu
@pytest.mark.parametrize("aligned", [True, False])
def test_soft_depth_k8_vector_and_scalar_paths(built_lib, aligned):
    scene = make_scene(2, 8, 8, 8, 1e-2, ZN, ZF, seed=81)
    if aligned:
        assert all(t.data_ptr() % 16 == 0 for t in torch_inputs(scene, DEV))
    _depth_gpu(scene, 1e-2, 20.0, "K=8 aligned=%s" % aligned, shift=not aligned)


@pytest.mark.gpu
@pytest.mark.parametrize("N,S,K", [(2, 768, 1), (1, 200, 40), (1, 200, 97)])
def test_soft_depth_grid_stride_second_pass(built_lib, N, S, K):
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    assert N * S * S > sms * 32 * (256 if K <= 8 else 8)
    scene = make_scene(N, S, S, K, 1e-2, ZN, ZF, seed=K + 4)
    _depth_gpu(scene, 1e-2, 20.0, "grid stride K=%d" % K)
