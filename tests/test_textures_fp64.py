"""UV texture sampling (csrc/textures.cu, DESIGN.md section 13) against a float64 reference, per element, on every
kernel path.

The reference restates TexturesUV.sample_textures for one map per image in numpy: the UV interpolated from the face's
corner UVs, the y-flipping torch.lerp to grid coordinates, and F.grid_sample's rules as torch's CUDA grid sampler
(ATen/native/cuda/GridSampler.cuh) states them and the kernel header restates them: the unnormalisation, the border
clip, the reflection, the out-of-int-range guard, "nearest" rounding half to even, the four bilinear corners and the
backward's grid gradient with its unnormalise / clip / reflect multipliers.  For every element of texels, grad_maps,
grad_barycentric_coords and grad_face_uvs it returns (lo, hi, beta): beta bounds how far a correct float32 evaluation
of the same steps can lie from the float64 value, propagated with the rules in the header of test_blending_fp64
(u = 2^-24; every scatter is a sum of n terms in any order and carries (n - 1) u sum |terms|).  Every element must
satisfy

    |got - [lo, hi]| <= 2 beta + 2^-126.

No element is masked.

Discrete decisions are taken as a correct float32 kernel takes them, in numpy float32: the UV is the FMA chain
fma(w2,a2, fma(w1,a1, fma(w0,a0, 0))) (numpy has no FMA; `fma32` rounds the exact float64 product-sum to odd and then
to float32, which is exact), the two-branch lerp, the unnormalisation (aligned: (x + 1) * 0.5 * (size - 1);
unaligned: one FMA (x + 1) * size - 1, then * 0.5), the reflection's subtraction, fmod, division and floor, and the
guard.  From those float32 coordinates every corner floor, in-bounds test, clip branch, reflection sign and flip
parity, and "nearest" rounding is exact, so no decision of the kernel path is open and lo == hi everywhere.  The
continuous values (weights, corner sums, the grid gradient, the lerp's (2, -2), the dot product with the corner UVs
and the scatters) are evaluated in float64 from the float32 coordinates.

Semantics pinned where torch's CPU and CUDA samplers part:
  * The flip count of the reflection is converted to int as torch's CUDA sampler converts it; the conversion
    saturates, so past 2^31 flips the parity is odd.  torch's CPU sampler picks other texels there: at UVs near 1e10
    under reflection the two samplers differ.
  * Non-finite coordinates: the forward clips with fmin / fmax, so under border and reflection padding a NaN (and a
    reflected +-inf, which becomes NaN) samples coordinate 0; the backward's `_set_grad` twins compare instead, so the
    same NaN falls to the guard's -100, out of bounds, and the slot gets no gradient at all.  torch's CPU grid_sample
    is no witness for these: with a NaN or infinite grid, "bilinear" returns NaN texels under zeros padding and reads
    outside the map under border (NaN) and reflection (NaN, +-inf) padding (torch 2.11 crashes there); only its
    "nearest" agrees with the CUDA semantics.
  * A coordinate of exactly 2^31 passes the guard (float(INT_MAX - 1) is 2^31) and one of exactly -2^31 too; both are
    out of bounds with all their corners, so the slot samples 0 and gets no gradient.

The float32 torch chain on the CPU interpolates the UV differently, with three products and a sum, so a slot's
coordinate (and a decision) may move by an ulp.  It is compared with the reference taken from its own float32 UVs
(model "cpu", reproduced bit for bit), so such a slot is still compared, on the branch the chain took.  torch 2.11's
CPU sampler contracts the unaligned unnormalisation to the same FMA as the CUDA one (checked against its texels and
map gradients).

CPU tests keep the reference honest: `fma32` equals exact rational arithmetic; the reference equals float64 autograd
through the suite's chain; the float32 chain lies within the bound; float32 restatements with one defect each fall
outside it; and the scenes reach every case the kernels treat specially.
"""
import fractions
import itertools
import types

import numpy as np
import pytest
import torch

from test_blending_fp64 import FLOOR, TINY, U, F, assert_within, count_outside, fsum
from test_textures import chain_sample, packed_face_uvs, texture_scene

assert TINY == FLOOR  # the bound's floor is the smallest normal float32
MODES = ("bilinear", "nearest")
PADDINGS = ("zeros", "border", "reflection")
FIELDS = ("texels", "grad_maps", "grad_bary", "grad_face_uvs")
I31 = 2.0 ** 31
BIG = np.float32(3e38)  # a barycentric that makes the interpolated UV overflow


# ------------------------------------------------------------------------------------------ float32 decisions
def fma32(a, b, c):
    """fmaf(a, b, c) for float32 arrays: the product is exact in float64; the float64 sum is rounded to odd (an inexact
    sum whose last bit is even moves one ulp towards the exact value) so that the final rounding to float32 is the
    correctly rounded fma."""
    a, b, c = (np.asarray(x, np.float32).astype(np.float64) for x in (a, b, c))
    with np.errstate(invalid="ignore", over="ignore"):
        p = a * b
        s = p + c
        bb = s - p
        e = (p - (s - bb)) + (c - bb)  # TwoSum: p + c = s + e exactly
        even = (s.view(np.int64) & 1) == 0
        fix = np.isfinite(s) & (e != 0) & even
        s = np.where(fix, np.nextafter(s, np.where(e > 0, np.inf, -np.inf)), s)
        return s.astype(np.float32)


def interp_uv(w, a, model):
    """(S,) u and v of slots with barycentrics w (S, 3) and corner UVs a (S, 3, 2)."""
    if model == "cuda":
        z = np.zeros(w.shape[0], np.float32)
        return [fma32(w[:, 2], a[:, 2, j], fma32(w[:, 1], a[:, 1, j], fma32(w[:, 0], a[:, 0, j], z))) for j in (0, 1)]
    with np.errstate(invalid="ignore", over="ignore"):
        p = w[:, :, None] * a  # the chain's interpolate_face_attributes: products, then a sum over the corners
        uv = (p[:, 0] + p[:, 1]) + p[:, 2]
    return [uv[:, 0], uv[:, 1]]


def lerp(start, end, w):
    """torch.lerp: start + w (end - start) where |w| < 0.5, else end - (end - start) (1 - w)."""
    T = w.dtype.type
    d = T(end - start)
    with np.errstate(invalid="ignore", over="ignore"):
        return np.where(np.abs(w) < 0.5, T(start) + w * d, T(end) - d * (T(1) - w))


def clip_grad(x, S, defect=None):
    """clip_coordinates_set_grad: the borders count as out of bounds for the gradient (NaN compares false: kept)."""
    T = x.dtype.type
    lo, hi = (x < 0, x > S - 1) if defect == "border_grad" else (x <= 0, x >= S - 1)
    val = np.where(x <= 0, T(0), np.where(x >= S - 1, T(S - 1), x))
    return val, np.where(lo | hi, T(0), T(1))


def reflect(x, twice_low, twice_high, defect=None):
    """reflect_coordinates_set_grad -> (coordinate, d coordinate / d x, odd flips)."""
    T = x.dtype.type
    if twice_low == twice_high:
        return np.zeros_like(x), np.zeros_like(x), np.zeros(x.shape, bool)
    mn, span = T(twice_low / 2), T((twice_high - twice_low) / 2)
    with np.errstate(invalid="ignore", over="ignore"):
        y = x - mn
        neg = y < 0
        mult = np.where(neg & (defect != "reflect_sign"), T(-1), T(1))
        y = np.where(neg, -y, y)
        extra = np.fmod(y, span)
        q = np.floor(y / span)
        # (int) floorf, as torch's CUDA sampler converts it: saturating, NaN -> 0
        # (in float64: 2^31 - 1 is not a float32)
        q = q.astype(np.float64)
        odd = np.where(np.isnan(q), 0, np.minimum(q, I31 - 1)).astype(np.int64) % 2 == 1
        r = np.where(odd, (span - extra) + mn, extra + mn)
    return r, np.where(odd, -mult, mult), odd


def guard(x):
    """safe_downgrade_to_int_range: -100 for non-finite values and values beyond float(INT_MAX - 1), float(INT_MIN)."""
    T = x.dtype.type
    return np.where((x > T(I31)) | (x < T(-I31)) | ~np.isfinite(x), T(-100), x)


def axis_coords(g, S, pad, align, defect=None):
    """One axis of grid_sampler_compute_source_index(_set_grad): (forward coordinate, backward coordinate, multiplier,
    {case: mask})."""
    T = g.dtype.type
    with np.errstate(invalid="ignore", over="ignore"):
        c1 = g + T(1)
        if align:
            c = (c1 * T(0.5)) * T(S if defect == "size" else S - 1)
            mult = T((S - 1) / 2)
        elif T is np.float32:  # torch's CPU sampler contracts it to the same FMA
            c = fma32(c1, T(S), T(-1)) * T(0.5)
            mult = T(S / 2)
        else:  # float64 decisions: a rounding of 2^-53 moves none of them
            c = (c1 * T(S) - T(1)) * T(0.5)
            mult = T(S / 2)
        fwd, bwd, m = c, c, np.full(c.shape, mult, T)
        cases = {"coord": c}
        if pad in ("border", "reflection"):
            r = c
            if pad == "reflection":
                r, gr, odd = reflect(c, 0, 2 * (S - 1), defect) if align else \
                    reflect(c, -1, 2 * S - 1, defect)
                m = m * gr
                lo2 = 0 if align else -1
                span = (S - 1) if align else S
                q = (c - lo2 / 2) / span if span else np.zeros_like(c)
                cases.update(reflected=r, odd=odd & np.isfinite(c), even=~odd & np.isfinite(c),
                             negative=(c < lo2 / 2), flip_boundary=np.isfinite(q) & (q == np.round(q)) & (q != 0))
            fwd = np.fmin(T(S - 1), np.fmax(r, T(0)))
            bwd, gc = clip_grad(r, S, defect)
            m = m * gc
            cases.update(clip_lo=r <= 0, clip_hi=r >= S - 1, clip_in=(r > 0) & (r < S - 1), on_0=r == 0,
                         on_max=r == S - 1)
    return guard(fwd), guard(bwd), m, cases


# ------------------------------------------------------------------------------------------ float32 arithmetic
class R32:
    """Plain float32 values with F's interface: a float32 restatement of the kernel through the reference's code."""

    __slots__ = ("v",)

    def __init__(self, v, b=None):
        self.v = np.asarray(v, np.float32)

    def __getitem__(self, i):
        return R32(self.v[i])

    def __add__(self, o):
        return R32(self.v + _r(o).v)

    def __sub__(self, o):
        return R32(self.v - _r(o).v)

    def __mul__(self, o):
        return R32(self.v * _r(o).v)

    def __neg__(self):
        return R32(-self.v)

    def masked(self, m):
        return R32(np.where(m, self.v, np.float32(0)))


def _r(x):
    return x if isinstance(x, R32) else R32(x)


def _sum(x, axis):
    return R32(x.v.sum(axis, dtype=np.float32)) if isinstance(x, R32) else fsum(x, axis)


def _stack(xs, axis):
    if isinstance(xs[0], R32):
        return R32(np.stack([x.v for x in xs], axis))
    return F(np.stack([x.v for x in xs], axis), np.stack([np.broadcast_to(x.b, x.v.shape) for x in xs], axis))


def _masked(x, m):
    return x.masked(m) if isinstance(x, R32) else F(np.where(m, x.v, 0.0), np.where(m, np.broadcast_to(x.b, x.v.shape),
                                                                                     0.0))


def scatter(keys, terms, size, drop_one=False):
    """sum of terms (flat) per key in [0, size); keys < 0 add nothing.  F: value, beta = sum beta + (n - 1) u sum |t|.
    `drop_one`: the last term of every key with at least two terms is lost (a defect)."""
    keys = keys.reshape(-1)
    ok = keys >= 0
    if drop_one:
        order = np.flatnonzero(ok)
        k = keys[order]
        last = np.zeros(len(keys), bool)
        _, first_rev = np.unique(k[::-1], return_index=True)
        idx = order[len(k) - 1 - first_rev]
        cnt = np.bincount(k, minlength=size)
        last[idx[cnt[keys[idx]] >= 2]] = True
        ok &= ~last
    kk = keys[ok]
    if isinstance(terms, R32):
        out = np.zeros(size, np.float32)
        np.add.at(out, kk, terms.v.reshape(-1)[ok])
        return R32(out)
    v = terms.v.reshape(-1)[ok]
    b = np.broadcast_to(terms.b, terms.v.shape).reshape(-1)[ok]
    n = np.bincount(kk, minlength=size)
    total = np.bincount(kk, v, minlength=size)
    absum = np.bincount(kk, np.abs(v), minlength=size)
    return F(total, np.bincount(kk, b, minlength=size) + np.maximum(n - 1, 0) * U * absum)


# ------------------------------------------------------------------------------------------ the reference
def reference(scene, mode, pad, align, model="cuda", dtype=np.float32, arith="fp64", defect=None):
    """{field: (lo, hi, beta)} (arith "fp64") or {field: float32 array} (arith "f32"), and {name: per-slot info}.

    scene: numpy maps (N, H_in, W_in, C) f32, p2f (N, H, W, K) i64, bary (N, H, W, K, 3) f32, face_uvs (F, 3, 2) f32,
    grad (N, H, W, K, C) f32.  model "cuda" takes the decisions as the kernel's spec, "cpu" as torch's CPU chain; dtype
    is the precision of the decisions (float64 only with "cpu", to compare with float64 autograd)."""
    maps, p2f, bary, fuv, go = (scene[k] for k in ("maps", "p2f", "bary", "face_uvs", "grad"))
    N, Hi, Wi, C = maps.shape
    S = p2f.size
    spi = S // N
    Fn = fuv.shape[0]
    T = dtype
    A = F if arith == "fp64" else R32
    f = p2f.reshape(-1)
    fg = f >= 0
    fi = np.where(fg, f, 0)
    w = np.where(fg[:, None], bary.reshape(S, 3), 0).astype(T)
    a = fuv.astype(T)[fi]
    u, v = interp_uv(w, a, model)
    u, v = np.where(fg, u, T(0)).astype(T), np.where(fg, v, T(0)).astype(T)
    gx, gy = lerp(-1.0, 1.0, u), lerp(1.0, -1.0, v)
    fx, bx, mx, cx = axis_coords(gx, Wi, pad, align, defect)
    fy, by, my, cy = axis_coords(gy, Hi, pad, align, defect)
    n = np.arange(S) // spi
    g = go.reshape(S, C).astype(np.float64)
    mflat = maps.reshape(-1, C).astype(np.float64)
    info = {"u": u, "v": v, "fx": fx, "fy": fy, "bx": bx, "by": by, "cx": cx, "cy": cy, "fg": fg, "grad": g}

    def corners(x, y):
        """the four corners (nw, ne, sw, se): in-bounds masks, flat texel rows, and the float64 differences."""
        x, y = x.astype(np.float64), y.astype(np.float64)
        x0, y0 = np.floor(x), np.floor(y)
        ins, rows = [], []
        for k in range(4):
            xk, yk = x0 + (k & 1), y0 + (k >> 1)
            inb = (xk >= 0) & (xk < Wi) & (yk >= 0) & (yk < Hi)
            ins.append(inb)
            rows.append(np.where(inb, n * Hi * Wi + np.where(inb, yk, 0) * Wi + np.where(inb, xk, 0), -1).astype(
                np.int64))
        d = [A(x0 + 1) - A(x), A(x) - A(x0), A(y0 + 1) - A(y), A(y) - A(y0)]  # dx1, dx0, dy1, dy0
        return ins, rows, d

    def weights(d):
        dx1, dx0, dy1, dy0 = d
        wk = [dx1 * dy1, dx0 * dy1, dx1 * dy0, dx0 * dy0]
        if defect == "swap":
            wk[1], wk[2] = wk[2], wk[1]
        return wk

    def nearest_rows(x, y):
        if defect == "round_away":
            r = lambda t: np.sign(t) * np.floor(np.abs(t.astype(np.float64)) + 0.5)  # noqa: E731
        else:
            r = lambda t: np.rint(t.astype(np.float64))  # noqa: E731  (half to even)
        xr, yr = r(x), r(y)
        inb = (xr >= 0) & (xr < Wi) & (yr >= 0) & (yr < Hi)
        info.setdefault("ties", (np.abs(x.astype(np.float64) % 1 - 0.5) == 0) | (np.abs(y.astype(np.float64) % 1 - 0.5)
                                                                                  == 0))
        return np.where(inb, n * Hi * Wi + np.where(inb, yr, 0) * Wi + np.where(inb, xr, 0), -1).astype(np.int64)

    out = {}
    # forward
    if mode == "nearest":
        row = nearest_rows(fx, fy)
        out["texels"] = A(np.where((row >= 0)[:, None], mflat[np.maximum(row, 0)], 0.0))
    else:
        ins, rows, d = corners(fx, fy)
        wk = weights(d)
        info["in_corners"] = sum(i.astype(int) for i in ins)
        terms = [_masked(wk[k][:, None] * A(mflat[np.maximum(rows[k], 0)]), ins[k][:, None]) for k in range(4)]
        out["texels"] = _sum(_stack(terms, 0), 0)
    # backward
    zero_bary = A(np.zeros((S, 3)))
    if mode == "nearest":
        row = nearest_rows(bx, by)
        keys = np.where((row >= 0)[:, None], row[:, None] * C + np.arange(C), -1)
        out["grad_maps"] = scatter(keys, A(g), N * Hi * Wi * C, drop_one=defect == "drop_texel")
        out["grad_bary"] = zero_bary
        out["grad_face_uvs"] = A(np.zeros(Fn * 6))
    else:
        ins, rows, d = corners(bx, by)
        wk = weights(d)
        dx1, dx0, dy1, dy0 = d
        wxs, wys = [-dy1, dy1, -dy0, dy0], [-dx1, -dx0, dx1, dx0]
        gm_keys, gm_terms, gx_terms, gy_terms = [], [], [], []
        for k in range(4):
            gm_keys.append(np.where(ins[k][:, None], rows[k][:, None] * C + np.arange(C), -1))
            gm_terms.append(_masked(wk[k][:, None] * A(g), ins[k][:, None]))
            val = A(mflat[np.maximum(rows[k], 0)])
            gx_terms.append(_masked((val * wxs[k][:, None]) * A(g), ins[k][:, None]))
            gy_terms.append(_masked((val * wys[k][:, None]) * A(g), ins[k][:, None]))
        keys = np.stack(gm_keys, 0)
        out["grad_maps"] = scatter(keys, _stack(gm_terms, 0), N * Hi * Wi * C, drop_one=defect == "drop_texel")
        gix = _sum(_sum(_stack(gx_terms, 0), 0), 1)
        giy = _sum(_sum(_stack(gy_terms, 0), 0), 1)
        gu = (A(mx.astype(np.float64)) * gix) * A(2.0)
        gv = (A(my.astype(np.float64)) * giy) * A(2.0 if defect == "gv_sign" else -2.0)
        a64 = a.astype(np.float64)
        gb = [A(a64[:, i, 0]) * gu + A(a64[:, i, 1]) * gv for i in range(3)]
        out["grad_bary"] = _masked(_stack(gb, 1), fg[:, None])
        w64 = w.astype(np.float64)
        ft = _stack([A(w64[:, i]) * (gu, gv)[j] for i in range(3) for j in range(2)], 1)
        fkeys = np.where(fg[:, None], fi[:, None] * 6 + np.arange(6), -1)
        if defect == "drop_face":  # the last slot of every face with at least two slots loses its contribution
            _, last_rev = np.unique(f[::-1], return_index=True)
            last = np.zeros(S, bool)
            idx = S - 1 - last_rev
            cnt = np.bincount(fi[fg], minlength=Fn)
            last[idx[(f[idx] >= 0) & (cnt[np.maximum(f[idx], 0)] >= 2)]] = True
            fkeys = np.where(last[:, None], -1, fkeys)
        out["grad_face_uvs"] = scatter(fkeys, ft, Fn * 6)
    shapes = {"texels": p2f.shape + (C,), "grad_maps": maps.shape, "grad_bary": p2f.shape + (3,),
              "grad_face_uvs": fuv.shape}
    if arith != "fp64":
        return {k: x.v.reshape(shapes[k]) for k, x in out.items()}, info
    ref = {}
    for k, x in out.items():
        val = x.v.reshape(shapes[k])
        ref[k] = (val, val, np.broadcast_to(x.b, x.v.shape).reshape(shapes[k]))
    return ref, info


# ------------------------------------------------------------------------------------------ scenes
def special_uvs(Hi, Wi, align, far10=True):
    """(u, v) pairs whose coordinates land on 0, on size - 1 and on flip boundaries, and far UVs (1e3, 1e10 unless
    not `far10`, 2^27)."""
    def ends(n):
        return (0.0, 1.0) if align else (0.5 / n, 1.0 - 0.5 / n)
    u_sp = list(ends(Wi)) + [-1.0, 2.0, 3.0, 1e3, -1e3, 1e10, -1e10, 2.0 ** 27, -2.0 ** 27]
    v_sp = [1.0 - t for t in ends(Hi)] + [-1.0, 2.0, 3.0, 1e3, -1e10, 2.0 ** 27]
    out = [(uu, 0.37) for uu in u_sp] + [(0.61, vv) for vv in v_sp] + [(1e10, 1e3), (-1e3, 2.0), (2.0, -1.0)]
    return [(uu, vv) for uu, vv in out if far10 or max(abs(uu), abs(vv)) < 1e9]


def fp64_scene(N, H, W, K, Hi, Wi, C, align, seed=0, extras=True, nonfinite=True, frac_background=0.3, far10=True):
    """texture_scene as numpy, with (extras) faces whose three corners sit on one special UV, sampled by the first
    slots of every image with barycentrics (1, 0, 0), (0, 1, 0) or (0, 0, 1) (so the UV is exact), (nonfinite)
    slots whose barycentric 3e38 makes the UV +-inf and whose infinite barycentrics make it NaN, and upstream
    gradients with exact zeros and -0.0."""
    s = texture_scene(N, H, W, K, Hi, Wi, C, align, seed=seed, frac_background=frac_background)
    sc = {"maps": s["maps"].numpy(), "p2f": s["pix_to_face"].numpy().copy(), "bary": s["bary"].numpy().copy(),
          "face_uvs": packed_face_uvs(s["verts_uvs"], s["faces_uvs"]).numpy(), "grad": s["grad_texels"].numpy().copy()}
    S = sc["p2f"].size
    spi = S // N
    p2f, bary, grad = sc["p2f"].reshape(-1), sc["bary"].reshape(S, 3), sc["grad"].reshape(S, C)
    extra_faces, slots = [], []  # (face, barycentrics) for the first slots of each image
    if extras:
        for j, (uu, vv) in enumerate(special_uvs(Hi, Wi, align, far10)):
            extra_faces.append(np.full((3, 2), (uu, vv), np.float32))
            slots.append((len(extra_faces) - 1, np.eye(3, dtype=np.float32)[j % 3]))
    if nonfinite:
        extra_faces.append(np.array([[10, -10], [-10, 10], [0.5, 0.5]], np.float32))
        nf = len(extra_faces) - 1
        extra_faces.append(np.array([[10, 0.25], [-10, 0.25], [0.5, 0.5]], np.float32))
        extra_faces.append(np.array([[0.25, 10], [0.25, -10], [0.5, 0.5]], np.float32))
        inf = np.inf
        for fj, b in ((nf, (BIG, 0, 0)), (nf, (0, BIG, 0)), (nf, (inf, inf, 0)), (nf + 1, (inf, inf, 0)),
                      (nf + 2, (inf, inf, 0)), (nf + 1, (BIG, BIG, 0)), (nf, (0, 0, 1))):
            slots.append((fj, np.array(b, np.float32)))
    F0 = sc["face_uvs"].shape[0]
    if extra_faces:
        sc["face_uvs"] = np.concatenate([sc["face_uvs"], np.stack(extra_faces)])
        for n in range(N):
            for i, (fj, b) in enumerate(slots[:spi]):
                p2f[n * spi + i] = F0 + fj
                bary[n * spi + i] = b
    grad[5::7] = 0.0
    grad[3::11, 0] = -0.0
    return sc


def torch_scene(sc, device):
    return {k: torch.from_numpy(np.ascontiguousarray(v)).to(device) for k, v in sc.items()}


def run_chain(sc, mode, pad, align, dtype=torch.float32):
    """chain_sample forward and backward on the CPU: {field: array} with the face-UV gradient taken at face_uvs."""
    t = torch_scene(sc, "cpu")
    maps = t["maps"].to(dtype).requires_grad_(True)
    bary = t["bary"].to(dtype).requires_grad_(True)
    fuv = t["face_uvs"].to(dtype).requires_grad_(True)
    frags = types.SimpleNamespace(pix_to_face=t["p2f"], bary_coords=bary)
    texels = chain_sample(frags, maps, fuv, mode, pad, align)
    texels.backward(t["grad"].to(dtype))
    grads = [x.grad if x.grad is not None else torch.zeros_like(x) for x in (maps, bary, fuv)]
    return dict(zip(FIELDS, [texels.detach().numpy()] + [x.numpy() for x in grads]))


def split_nan(name, got, ref):
    """A NaN of the reference (an infinite barycentric times a zero grid gradient gives the face UVs NaN, as in the
    chain) must be NaN in `got` too; the other elements are returned for the bound."""
    got = np.array(got.detach().cpu().numpy() if torch.is_tensor(got) else got, np.float64)
    lo, hi, beta = ref
    nan = np.isnan(lo)
    assert np.array_equal(np.isnan(got), nan), "%s: NaN where the reference has none, or none where it has" % name
    keep = lambda x: np.where(nan, 0.0, x)  # noqa: E731
    return keep(got), (keep(lo), keep(hi), keep(beta))


def check(name, got, ref):
    assert_within(name, *split_nan(name, got, ref))


def outside(got, ref):
    """count_outside, a NaN where the reference has none (or none where it has one) counting as outside."""
    try:
        g, r = split_nan("", got, ref)
    except AssertionError:
        return 1
    return count_outside(torch.from_numpy(g), r)


def ratio(got, ref):
    got, (lo, hi, beta) = split_nan("", got, ref)
    err = np.maximum(np.maximum(lo - got, got - hi), 0.0)
    return float(np.nan_to_num(err / (2 * beta + FLOOR), nan=np.inf).max()) if got.size else 0.0


# ------------------------------------------------------------------------------------------ CPU: the reference
CPU_CASES = list(itertools.product(MODES, PADDINGS, (True, False)))
CPU_MAPS = ((9, 17), (8, 5), (1, 1), (1, 12), (16, 8), (7, 1))


def test_fma32_is_exact():
    """fma32 equals the correctly rounded a * b + c of exact rational arithmetic on every UV step of the CPU scenes
    (the FMA chain's partial sums, and the unaligned unnormalisation's (x + 1) * size - 1)."""
    def exact(a, b, c):
        x = fractions.Fraction(float(a)) * fractions.Fraction(float(b)) + fractions.Fraction(float(c))
        f = np.float32(float(x))
        cands = [f, np.nextafter(f, np.float32(-np.inf)), np.nextafter(f, np.float32(np.inf))]
        cands = [cd for cd in cands if np.isfinite(cd)]
        best = min(cands, key=lambda cd: (abs(fractions.Fraction(float(cd)) - x),
                                          int(np.float32(cd).view(np.int32)) & 1))
        return best
    triples = []
    for (hi, wi), align in itertools.product(CPU_MAPS[:3], (True, False)):
        sc = fp64_scene(2, 4, 5, 3, hi, wi, 3, align, nonfinite=False)
        f = sc["p2f"].reshape(-1)
        fg = f >= 0
        w = sc["bary"].reshape(-1, 3)[fg]
        a = sc["face_uvs"][f[fg]]
        for j in (0, 1):
            p0 = fma32(w[:, 0], a[:, 0, j], 0.0)
            p1 = fma32(w[:, 1], a[:, 1, j], p0)
            triples += list(zip(w[:, 0], a[:, 0, j], np.zeros_like(p0)))
            triples += list(zip(w[:, 1], a[:, 1, j], p0)) + list(zip(w[:, 2], a[:, 2, j], p1))
        ref, info = reference(sc, "bilinear", "zeros", align)
        g = lerp(-1.0, 1.0, info["u"]) + np.float32(1)
        triples += list(zip(g, np.full_like(g, wi), np.full_like(g, -1.0)))
    rng = np.random.default_rng(0)
    x = (rng.standard_normal((3, 2000)) * np.exp2(rng.integers(-30, 30, (3, 2000)))).astype(np.float32)
    triples += list(zip(*x))
    a, b, c = (np.array(t, np.float32) for t in zip(*triples))
    got = fma32(a, b, c)
    want = np.array([exact(*t) for t in zip(a, b, c)], np.float32)
    assert np.array_equal(got.view(np.int32), want.view(np.int32))
    assert len(triples) > 5000


@pytest.mark.parametrize("C", [1, 2, 3, 4, 5, 8])
@pytest.mark.parametrize("mode,pad,align", CPU_CASES)
def test_reference_equals_float64_autograd(mode, pad, align, C):
    """With its decisions taken in float64 as the CPU chain takes them, the reference's values equal float64 autograd
    through chain_sample (F.grid_sample runs in float64 on the CPU, forward and backward)."""
    for hi, wi in CPU_MAPS:
        sc = fp64_scene(2, 4, 5, 3, hi, wi, C, align, seed=C, extras=False, nonfinite=False)
        ref, _ = reference(sc, mode, pad, align, model="cpu", dtype=np.float64)
        want = run_chain(sc, mode, pad, align, torch.float64)
        for name in FIELDS:
            lo, _, beta = ref[name]
            err = np.abs(lo - want[name])
            scale = np.abs(want[name]).max() + 1e-300
            assert (err <= 1e-6 * beta + 1e-12 * scale).all(), (name, hi, wi, float(err.max()))


def test_reference_closed_form():
    """One slot on a 2 x 2 map, align_corners, border: UV (0.25, 0.75) is grid (-0.5, -0.5), coordinate (0.25, 0.25)."""
    sc = {"maps": np.array([[[[1.0], [2.0]], [[3.0], [5.0]]]], np.float32), "p2f": np.zeros((1, 1, 1, 1), np.int64),
          "bary": np.array([1, 0, 0], np.float32).reshape(1, 1, 1, 1, 3),
          "face_uvs": np.array([[[0.25, 0.75], [0.5, 0.5], [1.0, 0.0]]], np.float32),
          "grad": np.ones((1, 1, 1, 1, 1), np.float32)}
    ref, _ = reference(sc, "bilinear", "border", True)
    w = np.array([0.75 * 0.75, 0.25 * 0.75, 0.75 * 0.25, 0.25 * 0.25])
    assert ref["texels"][0].reshape(()) == w @ [1.0, 2.0, 3.0, 5.0]
    assert np.array_equal(ref["grad_maps"][0].reshape(-1), w)
    gix = -0.75 * 1 + 0.75 * 2 - 0.25 * 3 + 0.25 * 5  # corner values times d w / d ix
    giy = -0.75 * 1 - 0.25 * 2 + 0.75 * 3 + 0.25 * 5
    gu, gv = 0.5 * gix * 2, 0.5 * giy * -2
    want = [0.25 * gu + 0.75 * gv, 0.5 * gu + 0.5 * gv, 1.0 * gu]
    np.testing.assert_allclose(ref["grad_bary"][0].reshape(-1), want, rtol=1e-15)
    np.testing.assert_allclose(ref["grad_face_uvs"][0].reshape(-1), [gu, gv, 0, 0, 0, 0], rtol=1e-15)


# ------------------------------------------------------------------------------------------ CPU: the bound is honest
@pytest.mark.parametrize("mode,pad,align", CPU_CASES)
def test_float32_chain_within_bound(mode, pad, align):
    """The float32 chain on the CPU, far UVs included, against the reference taken from its own float32 UVs.  Its
    sampler cannot take non-finite grids, and under reflection it picks another texel than torch's CUDA sampler from
    coordinates past 2^31 flips, so those UVs are left out there."""
    for C, (hi, wi) in zip((1, 3, 4, 2, 5, 3), CPU_MAPS):
        sc = fp64_scene(2, 4, 5, 3, hi, wi, C, align, seed=11, nonfinite=False, far10=pad != "reflection")
        ref, _ = reference(sc, mode, pad, align, model="cpu")
        got = run_chain(sc, mode, pad, align)
        for name in FIELDS:
            check("chain %s-%s-%s %dx%d %s" % (mode, pad, align, hi, wi, name), got[name], ref[name])


@pytest.mark.parametrize("mode,pad,align", CPU_CASES)
def test_float32_restatement_within_bound(mode, pad, align):
    """The kernel's spec evaluated in float32 (plain numpy float32 through the reference's own steps), non-finite UVs
    included."""
    for C, (hi, wi) in zip((1, 3, 4, 2, 5, 3), CPU_MAPS):
        sc = fp64_scene(2, 4, 5, 3, hi, wi, C, align, seed=12)
        ref, _ = reference(sc, mode, pad, align)
        got, _ = reference(sc, mode, pad, align, arith="f32")
        for name in FIELDS:
            check("f32 %s-%s-%s %dx%d %s" % (mode, pad, align, hi, wi, name), got[name], ref[name])


DEFECTS = {  # defect: the (mode, padding, align) cases it is looked for in
    "round_away": [("nearest", p, a) for p in PADDINGS for a in (True, False)],
    "size": [(m, p, True) for m in MODES for p in PADDINGS],
    "gv_sign": [("bilinear", p, a) for p in PADDINGS for a in (True, False)],
    "reflect_sign": [("bilinear", "reflection", a) for a in (True, False)],
    "border_grad": [("bilinear", "border", a) for a in (True, False)],
    "swap": [("bilinear", p, a) for p in PADDINGS for a in (True, False)],
    "drop_texel": [(m, p, a) for m in MODES for p in PADDINGS for a in (True, False)],
    "drop_face": [("bilinear", p, a) for p in PADDINGS for a in (True, False)],
}


@pytest.mark.parametrize("defect", list(DEFECTS))
def test_defective_restatement_fails(defect):
    """Each defect, in an otherwise correct float32 restatement, puts elements outside the bound."""
    n_out = 0
    for mode, pad, align in DEFECTS[defect]:
        for C, (hi, wi) in ((3, (9, 17)), (1, (16, 8))):
            sc = fp64_scene(2, 4, 5, 3, hi, wi, C, align, seed=13)
            ref, _ = reference(sc, mode, pad, align)
            got, _ = reference(sc, mode, pad, align, arith="f32", defect=defect)
            n_out += sum(outside(got[n], ref[n]) for n in FIELDS)
    assert n_out > 0, "the %s restatement passes the bound" % defect


def test_scenes_reach_every_case():
    """Every clip and reflect branch (on 0, on size - 1, on a flip boundary), 0, 1, 2 and 4 corners in bounds (never
    3), "nearest" ties, texel centres, UVs of 1e3 and 1e10, NaN and +-inf UVs, coordinates of exactly +-2^31 under zeros
    padding, background slots, and exact-zero and -0.0 upstream gradients."""
    seen = {}

    def add(k, m):
        seen[k] = seen.get(k, 0) + int(np.count_nonzero(m))
    for (hi, wi), align in itertools.product(CPU_MAPS, (True, False)):
        sc = fp64_scene(2, 4, 5, 3, hi, wi, 3, align)
        for pad in PADDINGS:
            _, info = reference(sc, "bilinear", pad, align)
            _, ninfo = reference(sc, "nearest", pad, align)
            for c in (info["cx"], info["cy"]):
                for k, m in c.items():
                    if k not in ("coord", "reflected"):
                        add("%s %s" % (pad, k), m)
            for k in range(5):
                add("%d corners" % k, (info["in_corners"] == k) & info["fg"])
            add("ties", ninfo["ties"])
            frac = np.concatenate([info["fx"], info["fy"]]).astype(np.float64) % 1
            add("centres", frac == 0)
            uv = np.abs(np.concatenate([info["u"], info["v"]]))
            add("uv 1e3", uv == np.float32(1e3))
            add("uv 1e10", uv == np.float32(1e10))
            add("uv nan", np.isnan(uv))
            add("uv inf", np.isinf(np.concatenate([info["u"], info["v"]])) & (np.concatenate([info["u"], info["v"]])
                                                                              > 0))
            add("uv -inf", np.isneginf(np.concatenate([info["u"], info["v"]])))
            add("background", ~info["fg"])
            g = info["grad"]
            add("grad 0", (g == 0) & ~np.signbit(g))
            add("grad -0", (g == 0) & np.signbit(g))
            if pad == "zeros" and align and wi == 17:
                add("2^31", info["cx"]["coord"] == np.float32(I31))
                add("-2^31", info["cx"]["coord"] == np.float32(-I31))
    # uv_x = 2^27 on a map 17 wide with align_corners: gx = 2^28, ix = 2^28 * 0.5 * 16 = 2^31 exactly
    g = lerp(-1.0, 1.0, np.array([2.0 ** 27, -2.0 ** 27], np.float32))
    ix = axis_coords(g, 17, "zeros", True)[3]["coord"]
    assert ix.dtype == np.float32 and ix.tolist() == [2.0 ** 31, -2.0 ** 31]
    # past 2^31 flips the count saturates to INT_MAX, odd: 1.1e11 reflects to span - fmod(1.1e11, span)
    r, _, odd = reflect(np.array([1.1e11], np.float32), 0, 22)
    assert odd.tolist() == [True] and r[0] == np.float32(11) - np.fmod(np.float32(1.1e11), np.float32(11))
    want = ["%s %s" % (p, k) for p in ("border", "reflection") for k in ("clip_lo", "clip_hi", "clip_in", "on_0",
                                                                         "on_max")]
    want += ["reflection odd", "reflection even", "reflection negative", "reflection flip_boundary"]
    assert seen["3 corners"] == 0  # a 2 x 2 footprint meets a rectangle in 0, 1, 2 or 4 corners
    want += ["%d corners" % k for k in (0, 1, 2, 4)] + ["ties", "centres", "uv 1e3", "uv 1e10", "uv nan", "uv inf",
                                                    "uv -inf", "2^31", "-2^31", "background", "grad 0", "grad -0"]
    missing = [k for k in want if seen.get(k, 0) == 0]
    assert not missing, missing


# ------------------------------------------------------------------------------------------ GPU
DEV = "cuda:0"
GPU_MAPS = ((1, 1), (1, 12), (7, 1), (9, 17), (5, 8), (16, 8))


class Worst:
    """The worst err / bound per field over a test, recorded with record_property."""

    def __init__(self, record_property):
        self.rp, self.worst = record_property, {}

    def add(self, name, got, ref):
        self.worst[name] = max(self.worst.get(name, 0.0), ratio(got, ref))

    def record(self):
        for k, v in sorted(self.worst.items()):
            self.rp("worst err/bound " + k, v)


def _exact_checks(sc, info, mode, pad, align, got, what):
    texels, gm, gb, gf = got
    zero = lambda x: (x == 0) | np.isnan(x)  # noqa: E731  (NaN where the reference has NaN: checked by check())
    fg = info["fg"]
    if gb is not None:
        gb = gb.reshape(-1, 3)
        assert zero(gb[~fg]).all(), "%s: grad_bary of background slots" % what
        if mode == "nearest" or (align and sc["maps"].shape[1:3] == (1, 1)):
            assert zero(gb).all(), "%s: grad_bary must be exactly 0" % what
    if gf is not None:
        used = np.zeros(sc["face_uvs"].shape[0], bool)
        used[sc["p2f"].reshape(-1)[fg]] = True
        gf = gf.reshape(-1, 6)
        assert zero(gf[~used]).all(), "%s: grad_face_uvs of faces no foreground slot samples" % what
        if mode == "nearest" or (align and sc["maps"].shape[1:3] == (1, 1)):
            assert zero(gf).all(), "%s: grad_face_uvs must be exactly 0" % what
    # a coordinate out of range on every corner: a 0 texel and no gradient
    out_f = (info["fx"] == -100) | (info["fy"] == -100)
    out_b = (info["bx"] == -100) | (info["by"] == -100)
    if texels is not None:
        assert (texels.reshape(out_f.size, -1)[out_f] == 0).all(), "%s: texel of an out-of-range slot" % what
    if gb is not None:
        assert zero(gb[out_b]).all(), "%s: grad_bary of an out-of-range slot" % what


def _gpu_check(sc, mode, pad, align, what, worst=None, needs=(True, True, True), autograd=False):
    """_C forward and backward (and, with `autograd`, sample_textures_uv through autograd) against the reference."""
    from pytorch3d_b200 import _C
    from pytorch3d_b200.interp_face_attrs import interpolate_face_attributes
    t = torch_scene(sc, DEV)
    ref, info = reference(sc, mode, pad, align)
    texels = _C.texture_uv_forward(t["p2f"], t["bary"], t["face_uvs"], t["maps"], mode, pad, align)
    grads = _C.texture_uv_backward(t["grad"], t["p2f"], t["bary"], t["face_uvs"], t["maps"], mode, pad, align,
                                   needs_input_grad=needs)
    got = [texels] + list(grads)
    if autograd:
        from pytorch3d_b200.textures import sample_textures_uv
        leaves = [t[k].clone().requires_grad_(True) for k in ("maps", "bary", "face_uvs")]
        frags = types.SimpleNamespace(pix_to_face=t["p2f"], bary_coords=leaves[1])
        out = sample_textures_uv(frags, leaves[0], leaves[2], sampling_mode=mode, padding_mode=pad,
                                 align_corners=align)
        out.backward(t["grad"])
        assert torch.equal(out, texels)
        got_ag = [out.detach()] + [x.grad for x in leaves]
    got = [None if x is None else x.detach().cpu().numpy() for x in got]
    for name, x in zip(FIELDS, got):
        if x is None:
            continue
        if worst is not None:
            worst.add(name, x, ref[name])
        check("%s %s" % (what, name), x, ref[name])
    if autograd:
        for name, x in zip(FIELDS, got_ag):
            x = x.cpu().numpy()
            if worst is not None:
                worst.add(name, x, ref[name])
            check("%s autograd %s" % (what, name), x, ref[name])
    _exact_checks(sc, info, mode, pad, align, got, what)
    # the reference's float32 UV is interpolate_face_attributes on the device, bit for bit
    uv = interpolate_face_attributes(t["p2f"], t["bary"], t["face_uvs"]).cpu().numpy().reshape(-1, 2)
    for j, name in enumerate("uv"):
        same = (uv[:, j].view(np.int32) == info[name].view(np.int32)) | (np.isnan(uv[:, j]) & np.isnan(info[name]))
        assert same.all(), "%s: %s differs from interpolate_face_attributes at %d slots" % (what, name, (~same).sum())
    return ref, info, got


@pytest.mark.gpu
@pytest.mark.parametrize("C", [1, 2, 3, 4, 5, 8, 11])
@pytest.mark.parametrize("mode", MODES)
def test_every_kernel_instance_matches_fp64(built_lib, record_property, mode, C):
    """texture_uv_{forward,backward}_kernel<MODE, CT> for CT = 1, 2, 3 and 4 (C = 5, 8, 11: a partial last pass and
    several full ones), every padding and alignment, maps of 1 x 1, 1 x W, H x 1, non-square and dyadic sizes, with
    far and non-finite UVs."""
    worst = Worst(record_property)
    for pad, align, (hi, wi) in itertools.product(PADDINGS, (True, False), GPU_MAPS):
        sc = fp64_scene(2, 6, 7, 3, hi, wi, C, align, seed=C + hi)
        _gpu_check(sc, mode, pad, align, "%s-%s-%s C=%d %dx%d" % (mode, pad, align, C, hi, wi), worst)
    worst.record()


@pytest.mark.gpu
@pytest.mark.parametrize("pad", PADDINGS)
def test_far_and_nonfinite_uvs_fused_and_autograd(built_lib, record_property, pad):
    """Far (1e3, 1e10, +-2^31 coordinates) and non-finite UVs through _C and through autograd, every mode and
    alignment.  Pinned: under border and reflection a NaN UV samples coordinate 0 in the forward and gives no gradient
    in the backward."""
    worst = Worst(record_property)
    for mode, align, C in itertools.product(MODES, (True, False), (1, 3)):
        sc = fp64_scene(1, 2, 16, 1, 9, 17, C, align, seed=21, frac_background=0.0)
        _gpu_check(sc, mode, pad, align, "%s-%s-%s C=%d" % (mode, pad, align, C), worst, autograd=True)
    worst.record()
    # the asymmetry, on its own: one slot whose face has a NaN u at the corner it sits on, v = 0.3
    maps = np.random.default_rng(5).random((1, 4, 6, 2)).astype(np.float32)
    sc = {"maps": maps, "p2f": np.zeros((1, 1, 1, 1), np.int64),
          "bary": np.array([1, 0, 0], np.float32).reshape(1, 1, 1, 1, 3),
          "face_uvs": np.array([[[np.nan, 0.3], [0.2, 0.1], [0.9, 0.8]]], np.float32),
          "grad": np.ones((1, 1, 1, 1, 2), np.float32)}
    for mode, align in itertools.product(MODES, (True, False)):
        _, info, (tex, gm, gb, gf) = _gpu_check(sc, mode, pad, align, "NaN u %s-%s-%s" % (mode, pad, align))
        assert np.isnan(info["u"][0]) and info["v"][0] == np.float32(0.3)
        if pad == "zeros":
            assert (tex == 0).all()
        else:  # the forward samples x = 0 (a texel of column 0 under "nearest")
            assert info["fx"][0] == 0 and (tex != 0).all()
        assert info["bx"][0] == -100 and (gm == 0).all() and (gf == 0).all()  # the backward: none at all


def _pattern_scene(keys, mode, C=3, Hi=8, Wi=8, seed=0):
    """One image of len(keys) slots; slot s samples face keys[s] (-1: background), and face j's corners sit around
    the centre of texel j, so that a warp's lanes share texels and faces in the pattern of `keys`."""
    rng = np.random.default_rng(seed)
    keys = np.asarray(keys)
    S = len(keys)
    Fn = max(int(keys.max()) + 1, 1)
    cx = (np.arange(Fn) % Wi + 0.5) / Wi
    cy = 1.0 - ((np.arange(Fn) // Wi) % Hi + 0.5) / Hi
    centre = np.stack([cx, cy], -1)[:, None, :]
    if mode == "nearest":
        fuv = np.broadcast_to(centre, (Fn, 3, 2))
    else:
        fuv = centre + (rng.random((Fn, 3, 2)) - 0.5) * 0.4 / np.array([Wi, Hi])
    bary = rng.random((S, 3)) + 0.05
    bary /= bary.sum(1, keepdims=True)
    grad = rng.normal(0.0, 1.0, (S, C)) * np.exp2(rng.integers(-3, 4, (S, 1)))
    return {"maps": rng.random((1, Hi, Wi, C)).astype(np.float32), "p2f": keys.reshape(1, 1, S, 1).astype(np.int64),
            "bary": bary.reshape(1, 1, S, 1, 3).astype(np.float32),
            "face_uvs": np.ascontiguousarray(fuv, np.float32), "grad": grad.reshape(1, 1, S, 1, C).astype(np.float32)}


WARP_PATTERNS = {
    "all_same": lambda lane, w: np.zeros_like(lane),
    "alternating": lambda lane, w: lane % 2 + 2 * (w % 3),
    "runs_of_3": lambda lane, w: lane // 3,
    "runs_of_5": lambda lane, w: lane // 5 + 7 * (w % 2),
    "lane_31_alone": lambda lane, w: np.where(lane == 31, 1, 0),
    "background_between": lambda lane, w: np.where(lane % 3 == 1, -1, lane // 6),
}


@pytest.mark.gpu
@pytest.mark.parametrize("C", [1, 3, 5])
@pytest.mark.parametrize("mode", MODES)
def test_warp_merge_patterns(built_lib, record_property, mode, C):
    """Lanes of a warp on the same texel and face in fixed patterns (all 32, two alternating keys, runs of 3 and 5,
    lane 31 alone, background lanes between), over 4 warps, and a ragged last warp with one active lane."""
    worst = Worst(record_property)
    for name, fn in WARP_PATTERNS.items():
        for warps, tail in ((4, 0), (4, 1)):
            lane = np.arange(32 * warps + tail) % 32
            keys = fn(lane, np.arange(len(lane)) // 32)
            sc = _pattern_scene(keys, mode, C, seed=len(keys))
            for pad, align in (("border", True), ("zeros", False), ("reflection", False)):
                _gpu_check(sc, mode, pad, align, "%s tail=%d %s-%s-%s" % (name, tail, mode, pad, align), worst)
    worst.record()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_contention_on_one_texel_and_one_face(built_lib, record_property, mode):
    """Every slot of a 200,704-slot scene on face 0, its UVs within one texel: each element within
    (n - 1) u sum |terms| of the float64 sum."""
    worst = Worst(record_property)
    S = 448 * 448
    rng = np.random.default_rng(4)
    Hi, Wi, C = 6, 10, 3
    centre = np.array([(3 + 0.5) / Wi, 1.0 - (2 + 0.5) / Hi])
    fuv = (centre + (rng.random((1, 3, 2)) - 0.5) * 0.5 / np.array([Wi, Hi])).astype(np.float32)
    bary = rng.random((S, 3)) + 0.05
    bary /= bary.sum(1, keepdims=True)
    sc = {"maps": rng.random((1, Hi, Wi, C)).astype(np.float32), "p2f": np.zeros((1, 448, 448, 1), np.int64),
          "bary": bary.reshape(1, 448, 448, 1, 3).astype(np.float32), "face_uvs": fuv,
          "grad": rng.normal(0.0, 1.0, (1, 448, 448, 1, C)).astype(np.float32)}
    for pad, align in (("border", True), ("reflection", False)):
        _, info, got = _gpu_check(sc, mode, pad, align, "contention %s-%s-%s" % (mode, pad, align), worst)
    if mode == "nearest":
        assert np.unique(np.stack([np.rint(info["fx"]), np.rint(info["fy"])]), axis=1).shape[1] == 1  # one texel
    worst.record()


@pytest.mark.gpu
@pytest.mark.parametrize("mode,pad,align,C", [("bilinear", "reflection", False, 3), ("nearest", "border", True, 5)])
def test_grid_stride_second_pass(built_lib, record_property, mode, pad, align, C):
    """More slots than the capped grid holds (32 CTAs of 256 threads per SM), with a ragged tail: the second pass of
    the grid-stride loop, forward and backward."""
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    W = 32 * sms * 256 // 2 + 77
    assert 2 * W > 32 * sms * 256 and (2 * W) % 256 != 0
    worst = Worst(record_property)
    sc = fp64_scene(2, 1, W, 1, 9, 17, C, align, seed=31)
    _gpu_check(sc, mode, pad, align, "grid stride %s-%s-%s C=%d" % (mode, pad, align, C), worst)
    worst.record()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_skipped_outputs_within_bound(built_lib, mode):
    """Every needs_input_grad subset: the outputs that remain are still within the bound, the others None."""
    sc = fp64_scene(2, 6, 7, 3, 9, 17, 3, True, seed=41)
    for needs in itertools.product((True, False), repeat=3):
        for pad in PADDINGS:
            _, _, got = _gpu_check(sc, mode, pad, True, "needs=%s %s-%s" % (needs, mode, pad), needs=needs)
            assert [g is None for g in got[1:]] == [not x for x in needs]
