"""Splatter blending (csrc/splatter_blend.cu, DESIGN.md section 11) against a float64 reference, per element, on every
kernel path.

The reference restates in float64 numpy the forward and backward formulas of the header of splatter_blend.cu: the
occlusion ids, c = floor(xy) - xy + 0.5, the Gaussian weights and norm, the three layer sums, 1 / max(W_l, 1), the
compose over the background, the record E_l (with dW_l through torch.maximum) and the gather into the gradients of the
colours and of the positions.  Next to every value it returns a first-order running error bound beta on how far a
correct float32 evaluation of the same steps can lie from it, propagated with the rules and helpers of
test_blending_fp64 (u = 2^-24; sums of n terms carry (n - 1) u sum |terms| in any order).  The constants:

    1 / (2 sigma^2)   exact in the reference; the kernels' float32 reciprocal of 2 sigma^2 rounded to float32 carries 2u
    norm              1.05f / sum_d expf(-|o_d|^2 inv), computed on the device in float32: tracked step by step, 1.05f
                      carrying u
    expf              within 2 ulp; a result below the normal float32 range may be subnormal or 0

Every element of the image, of grad_colors and of grad_pixel_coords_screen must satisfy

    |got - ref| <= 2 beta + 2^-126.

No element is masked and slots are compared one by one; background slots and the z gradient must be exactly 0.

Discrete decisions are taken as the kernels take them.  |p_k - q_0| and |p_0 - q_k| are one float32 subtraction and an
abs, which numpy float32 reproduces bit for bit, so the argmins (the first slot on ties), the strict minB < minA, the
zero padding and the background depth 1 are exact, and so are the layer buckets that follow from them.  floor is exact.
max(W_l, 1) and the half gradient at W_l == 1 are decided in float64; within 2 beta of 1 the reference returns the
interval spanned by the branches (the forward value is continuous there; the record's dW_l and the position gradients
that go through it are intervals).  The warp-uniform skip of empty sources changes no value.

CPU tests keep the reference honest: its backward equals float64 autograd through the suite's splatter_chain, the
float32 chain lies within the bound on every CPU scene, defective chains fall outside it, and the GPU scenes reach every
case the kernels treat specially.
"""
import contextlib

import numpy as np
import pytest
import torch
import torch.nn.functional as tF

from test_blending_fp64 import FLOOR, TINY, U, F, assert_within, count_outside, fsum, where
from test_splatter_blend import splatter_chain

DIRS = [(d // 3 - 1, d % 3 - 1) for d in range(9)]  # o_d, and the neighbour the occlusion test of direction d reads
SRC = [(d % 3 - 1, d // 3 - 1) for d in range(9)]   # the source of the splat a pixel receives in direction d
TILE_H, TILE_W, CHUNK = 8, 32, 8                     # the kernels' tile and slot chunk


# ------------------------------------------------------------------------------------------ the float64 reference
def shift(x, dh, dw):
    """x[n, h + dh, w + dw] at [n, h, w] and 0 outside the image (the zero padding); x (N, H, W, ...) or an F."""
    if isinstance(x, F):
        return F(shift(x.v, dh, dw), shift(np.broadcast_to(x.b, x.v.shape), dh, dw))
    H, W = x.shape[1:3]
    out = np.zeros_like(x)
    out[:, max(0, -dh):min(H, H - dh), max(0, -dw):min(W, W - dw)] = \
        x[:, max(0, dh):min(H, H + dh), max(0, dw):min(W, W + dw)]
    return out


def stack(terms):
    return F(np.stack([t.v for t in terms]), np.stack([np.broadcast_to(t.b, t.v.shape) for t in terms]))


def occlusion(z):
    """occ (N, H, W, 9) from the depths z (N, H, W, K) as the kernels take it (float32 z: bit for bit), and counts of
    the cases the coverage test asks for."""
    occ = np.empty(z.shape[:3] + (9,), np.int64)
    info = {"occ_neg": 0, "occ_zero": 0, "occ_pos": 0, "tie_in_argmin": 0, "tie_min_a_min_b": 0, "padding": 0}
    for d, (dh, dw) in enumerate(DIRS):
        p = shift(z, dh, dw)
        a, b = np.abs(p - z[..., :1]), np.abs(p[..., :1] - z)
        min_a, min_b = a.min(-1), b.min(-1)
        occ[..., d] = np.where(min_b < min_a, -b.argmin(-1), a.argmin(-1))
        for x, mx in ((a, min_a), (b, min_b)):
            info["tie_in_argmin"] += int(((x == mx[..., None]).sum(-1) > 1).sum())
        info["tie_min_a_min_b"] += int((min_a == min_b).sum())
        inside = shift(np.ones(z.shape[:3], bool), dh, dw)
        info["padding"] += int((~inside).sum())
    info.update(occ_neg=int((occ < 0).sum()), occ_zero=int((occ == 0).sum()), occ_pos=int((occ > 0).sum()))
    return occ, info


def reference(colors, coords, mask, grad, sigma, bg, z_dtype=np.float32):
    """{name: (lo, hi, beta)} of out (N,H,W,4), grad_colors and grad_pixel_coords_screen (N,H,W,K,3), and the info of
    the coverage test.  colors / coords / grad float32 and mask bool numpy arrays, bg 3 numbers; z_dtype float64 takes
    the occlusion decisions in float64 (the autograd comparison)."""
    N, H, W, K = mask.shape
    valid = (~mask).astype(np.float64)
    occ, info = occlusion(np.where(mask, 1.0, coords[..., 2]).astype(z_dtype))
    inv = F(0.5 / sigma ** 2, U / sigma ** 2)
    s = F(0.0)
    for oh, ow in DIRS:
        s = s + (F(-float(oh * oh + ow * ow)) * inv).exp()
    norm = F(1.05, 1.05 * U) / s
    xy = np.where(mask[..., None], 1.0, coords[..., :2].astype(np.float64))
    c = [F(np.floor(xy[..., i])) - F(xy[..., i]) + 0.5 for i in range(2)]
    rgb = [F(colors[..., j].astype(np.float64) * valid) for j in range(3)]
    ks = np.arange(K)

    # the splats each source slot sends in direction d, and the layer sums of the pixels receiving them
    w_d, e_d, buckets = [], [], []
    Sv, Sb, Sa = np.zeros((3, 4, N, H, W)), np.zeros((3, 4, N, H, W)), np.zeros((3, 4, N, H, W))
    count = np.zeros((3, N, H, W))
    info["w_zero"] = info["w_subnormal"] = 0
    for d, (oh, ow) in enumerate(DIRS):
        e0, e1 = c[0] + float(oh), c[1] + float(ow)
        w = (-(e0 * e0 + e1 * e1) * inv).exp()
        w_d.append(w)
        e_d.append((e0, e1))
        info["w_zero"] += int(((w.v < 2.0 ** -150) & (valid > 0)).sum())
        info["w_subnormal"] += int(((w.v >= 2.0 ** -150) & (w.v < TINY) & (valid > 0)).sum())
        sw = (norm * w).masked(valid)
        o = occ[..., d][..., None]
        lay = np.where(o > ks, 0, np.where(o == ks, 1, 2))
        buckets.append(lay)
        dh, dw = SRC[d]
        for j, term in enumerate([sw * rgb[0], sw * rgb[1], sw * rgb[2], sw]):
            t = shift(term, dh, dw)
            for l in range(3):
                m = lay == l
                Sv[l, j] += (t.v * m).sum(-1)
                Sb[l, j] += (t.b * m).sum(-1)
                Sa[l, j] += (np.abs(t.v) * m).sum(-1)
        for l in range(3):
            count[l] += (lay == l).sum(-1)
    S = [[F(Sv[l, j], Sb[l, j] + np.maximum(count[l] - 1, 0) * U * Sa[l, j]) for j in range(4)] for l in range(3)]

    # normalise and compose over the background: o[0] = (bg, 0), o[i + 1] = N_{2 - i} + (1 - N_{2 - i}.a) o[i]
    inv_l, Nl = [], []
    for l in range(3):
        Wl = S[l][3]
        inv_l.append(F(1.0) / F(np.maximum(Wl.v, 1.0), Wl.b))
        Nl.append([S[l][j] * inv_l[l] for j in range(4)])
        info["W%d_below_1" % l] = int(((Wl.v > 0) & (Wl.v < 1 - 2 * Wl.b - FLOOR)).sum())
        info["W%d_above_1" % l] = int((Wl.v > 1 + 2 * Wl.b + FLOOR).sum())
    o = [[F(np.full((N, H, W), float(np.float32(x)))) for x in bg] + [F(np.zeros((N, H, W)))]]
    for i in range(3):
        t = F(1.0) - Nl[2 - i][3]
        o.append([Nl[2 - i][j] + t * o[i][j] for j in range(4)])
    out = stack(o[3])

    # the record: E_l = (dS_l.rgb, dS_l.a + dW_l), l = 0 first (composed last)
    g = [F(grad[..., j].astype(np.float64)) for j in range(4)]
    E, info["W_open"] = [], 0
    for l in range(3):
        ob = o[2 - l]
        ea = -fsum(stack([g[j] * ob[j] for j in range(4)]), 0)
        dNa = g[3] + ea
        dinv = fsum(stack([g[0] * S[l][0], g[1] * S[l][1], g[2] * S[l][2], dNa * S[l][3]]), 0)
        dmax = -(dinv * inv_l[l]) * inv_l[l]
        Wl = S[l][3]
        open_ = np.abs(Wl.v - 1.0) <= 2 * Wl.b + FLOOR
        above = (Wl.v > 1.0) & ~open_
        info["W_open"] += int(open_.sum())
        dW = where(open_, F(0.5 * dmax.v, dmax.b), where(above, dmax, 0.0))
        E.append({"rgb": [g[j] * inv_l[l] for j in range(3)], "aN": dNa * inv_l[l], "dW": dW,
                  "rad": np.where(open_, 0.5 * np.abs(dmax.v), 0.0)})
        t = F(1.0) - Nl[l][3]
        g = [g[j] * t for j in range(4)]

    # the gather: source slot s reads, for each direction d, the record of the pixel its splat landed on
    def select(lay, key, j=None):
        pick = [shift(E[l][key] if j is None else E[l][key][j], -dh, -dw) for l in range(3)]
        if not isinstance(pick[0], F):
            return np.where(lay == 0, pick[0][..., None], np.where(lay == 1, pick[1][..., None], pick[2][..., None]))
        v = [p.v[..., None] for p in pick]
        b = [np.broadcast_to(p.b, p.v.shape)[..., None] for p in pick]
        return F(np.where(lay == 0, v[0], np.where(lay == 1, v[1], v[2])),
                 np.where(lay == 0, b[0], np.where(lay == 1, b[1], b[2])))

    gc_terms, gx_terms = [[], [], []], [[], []]
    rad = [np.zeros((N, H, W, K)), np.zeros((N, H, W, K))]
    info["subnormal_products"] = 0
    for d in range(9):
        dh, dw = SRC[d]
        lay = shift(buckets[d], -dh, -dw)
        Er = [select(lay, "rgb", j) for j in range(3)]
        aN, dW, rd = select(lay, "aN"), select(lay, "dW"), select(lay, "rad")
        w, (e0, e1) = w_d[d], e_d[d]
        swn = norm * w
        dsw = fsum(stack([Er[0] * rgb[0], Er[1] * rgb[1], Er[2] * rgb[2], aN, dW]), 0)
        for j in range(3):
            gc_terms[j].append(Er[j] * swn)
        dsw_w = (dsw * norm) * w
        info["subnormal_products"] += int(((np.abs(dsw_w.v) > 0) & (np.abs(dsw_w.v) < TINY) & (valid > 0)).sum())
        X = dsw_w * inv
        for i, e in enumerate((e0, e1)):
            gx_terms[i].append((X * 2.0) * e)
            rad[i] += np.abs(norm.v * w.v * inv.v * 2.0 * e.v) * rd
    gc = [fsum(stack(t), 0).masked(valid) for t in gc_terms]
    gx = [fsum(stack(t), 0).masked(valid) for t in gx_terms]
    zero = np.zeros((N, H, W, K))
    gcv, gcb = np.stack([x.v for x in gc], -1), np.stack([x.b for x in gc], -1)
    gxv, gxb = np.stack([gx[0].v, gx[1].v, zero], -1), np.stack([gx[0].b, gx[1].b, zero], -1)
    gxr = np.stack([rad[0] * valid, rad[1] * valid, zero], -1)
    ref = {"out": (out.v.transpose(1, 2, 3, 0), out.v.transpose(1, 2, 3, 0), out.b.transpose(1, 2, 3, 0)),
           "grad_colors": (gcv, gcv, gcb), "grad_pixel_coords_screen": (gxv - gxr, gxv + gxr, gxb)}
    info["occ"] = occ
    info["c_zero"] = int(sum(((x.v == 0) & (valid > 0)).sum() for x in c))
    info["c_half"] = int(sum(((x.v == 0.5) & (valid > 0)).sum() for x in c))
    x32 = coords[..., :2]
    rounds = (np.floor(x32) - x32).astype(np.float64) != np.floor(x32.astype(np.float64)) - x32.astype(np.float64)
    info["negative_rounding"] = int((rounds & (x32 < 0) & (valid[..., None] > 0)).sum())
    return ref, info


def warp_sources(mask):
    """(warp-slot-directions whose 32 lanes all have an empty source, those where only some have): a warp is one row of
    a 32 x 8 tile, and lane x's source in direction d is pixel (y, x) + SRC[d], empty outside the image."""
    N, H, W, K = mask.shape
    TY, TX = -(-H // TILE_H), -(-W // TILE_W)
    v = np.zeros((N, TY * TILE_H + 2, TX * TILE_W + 2, K), bool)
    v[:, 1:H + 1, 1:W + 1] = ~mask
    none = some = 0
    for dh, dw in SRC:
        src = v[:, 1 + dh:1 + dh + TY * TILE_H, 1 + dw:1 + dw + TX * TILE_W].reshape(N, TY * TILE_H, TX, TILE_W, K)
        n_valid = src.sum(3)
        none += int((n_valid == 0).sum())
        some += int(((n_valid > 0) & (n_valid < TILE_W)).sum())
    return none, some


# ------------------------------------------------------------------------------------------ scenes
def make_scene(N, H, W, K, sigma, seed=0):
    """colors, coords (N,H,W,K,3) float32, mask (N,H,W,K) bool, grad (N,H,W,4) float32, as numpy arrays.

    Blocks of 4 rows by one tile column take one of four slot layouts (trailing empties, interleaved, all empty, all
    valid), so that whole warps see empty sources; blocks of 2 x 5 pixels take one of four depth kinds (sorted in
    [1, 6], integers with ties across slots and neighbours, some slots at depth 0 (ties with the padding), unsorted);
    every coordinate takes one of five position kinds (anywhere in its pixel, within 12 sigma of the centre, exactly on
    the centre, on an integer, negative)."""
    rng = np.random.default_rng(seed + 1000 * K + 7 * H + W)
    n, h, w = np.meshgrid(np.arange(N), np.arange(H), np.arange(W), indexing="ij")
    layout = ((h // 4 + w // TILE_W + n) % 4)[..., None]
    ks = np.arange(K)
    valid = np.where(layout == 0, ks < rng.integers(0, K + 1, (N, H, W, 1)),
                     np.where(layout == 1, rng.random((N, H, W, K)) < 0.6, layout == 3))
    kind = ((h // 2 + w // 5 + 2 * n) % 4)[..., None]
    z = np.sort(1.0 + 5.0 * rng.random((N, H, W, K)), -1)
    z = np.where(kind == 1, np.round(z), z)
    z = np.where((kind == 2) & (rng.random((N, H, W, K)) < 0.3), 0.0, z)
    z = np.where(kind == 3, 1.0 + 5.0 * rng.random((N, H, W, K)), z)
    centre = np.stack([h, w], -1)[:, :, :, None, :] + 0.5
    pk = rng.integers(0, 5, (N, H, W, K, 2))
    xy = np.where(pk == 0, centre + rng.random((N, H, W, K, 2)) - 0.5,
                  np.where(pk == 1, centre + np.clip(sigma * rng.uniform(-12, 12, (N, H, W, K, 2)), -0.49, 0.49),
                           np.where(pk == 2, centre, np.where(pk == 3, centre + np.where(
                               rng.random((N, H, W, K, 2)) < 0.5, -0.5, 0.5), -2.0 * rng.random((N, H, W, K, 2))))))
    coords = np.concatenate([xy, z[..., None]], -1).astype(np.float32)
    colors = rng.random((N, H, W, K, 3)).astype(np.float32)
    grad = rng.normal(0.0, 1.0, (N, H, W, 4)).astype(np.float32)
    return colors, coords, ~valid, grad


BG = (0.2, 0.4, 0.6)
GPU_KS = [1, 2, 7, 8, 9, 15, 16, 17, 33, 64, 150]   # one stage; full chunks; last chunks of 1 to 7 slots
SHAPES = [(2, 16, 64), (2, 25, 65), (2, 1, 40), (2, 37, 1), (3, 1, 1)]
SIGMAS = [1e-4, 0.25, 0.5, 1.0, 3.0]


def gpu_scenes(K):
    """(N, H, W, K, sigma, background as a tensor) of the GPU matrix at K: every shape, sigma cycled over K."""
    i = GPU_KS.index(K)
    return [(*shape, K, SIGMAS[(i + j) % len(SIGMAS)], (i + j) % 2 == 1) for j, shape in enumerate(SHAPES)]


CPU_SCENES = [(2, 10, 34, 2, 0.25), (2, 10, 34, 9, 0.5), (2, 10, 34, 17, 1e-4), (2, 10, 34, 17, 3.0),
              (1, 9, 33, 16, 1.0)]  # tile crossings in x, in y and at corners; K from one stage to three chunks


# ------------------------------------------------------------------------------------------ the float32 chains
DEFECTS = ["corrected", "last_tie", "le", "replicate", "order", "no_max", "dc_plus", "halo", "chunk"]


def defective_chain(colors, coords, mask, sigma, background, defect=None):
    """test_splatter_blend.splatter_chain with one step broken: "corrected" the corrected direction pairing,
    "last_tie" argmin ties sent to the last slot, "le" <= in the occ decision, "replicate" replicate padding of the
    depths, "order" layers composed 0, 1, 2, "no_max" normalisation by W_l, "dc_plus" d c / d xy = +1, "halo" splats
    from another 32 x 8 tile dropped, "chunk" the occlusion minima restarted at every chunk of 8 slots."""
    N, H, W, K, _ = colors.shape
    m = mask[..., None]
    coords = torch.where(m, torch.ones(()), coords)
    rgba = torch.cat([colors, torch.ones_like(colors[..., :1])], dim=-1)
    rgba = torch.where(m, torch.zeros(()), rgba)
    directions = [(d // 3 - 1, d % 3 - 1) for d in range(9)]

    z = coords[..., 2].permute(0, 3, 1, 2)
    zp = tF.pad(z, [1, 1, 1, 1], mode="replicate" if defect == "replicate" else "constant")
    p = torch.stack([zp[:, :, 1 + dh:1 + dh + H, 1 + dw:1 + dw + W] for dh, dw in directions], dim=2)
    q = z.view(N, K, 1, H, W)
    a, b = torch.abs(p - q[:, 0:1]), torch.abs(p[:, 0:1] - q)
    k0 = CHUNK * ((K - 1) // CHUNK) if defect == "chunk" else 0
    if defect == "last_tie":
        min_a, arg_a = a.flip(1).min(dim=1)
        min_b, arg_b = b.flip(1).min(dim=1)
        arg_a, arg_b = K - 1 - arg_a, K - 1 - arg_b
    else:
        min_a, arg_a = a[:, k0:].min(dim=1)
        min_b, arg_b = b[:, k0:].min(dim=1)
        arg_a, arg_b = arg_a + k0, arg_b + k0
    occ = torch.where(min_b <= min_a if defect == "le" else min_b < min_a, -arg_b, arg_a).permute(0, 2, 3, 1)
    if defect == "corrected":
        occ = occ[..., [(d % 3) * 3 + d // 3 for d in range(9)]]

    offsets = torch.tensor(directions, dtype=torch.long)
    norm = torch.div(1.05, torch.exp(-torch.square(offsets).sum(dim=1) / (2 * sigma ** 2)).sum())
    c = torch.floor(coords[..., :2]) - coords[..., :2] + 0.5
    if defect == "dc_plus":
        c = c.detach() + (coords[..., :2] - coords[..., :2].detach())
    c = c.view(N, H, W, K, 1, 2)
    w = torch.exp(-torch.sum(torch.square(c + offsets), dim=5) / (2 * sigma ** 2))
    sw = (rgba[..., 3:4] * norm * w).unsqueeze(5)
    splats = torch.cat([sw * rgba.unsqueeze(4), sw], dim=5)

    sp = tF.pad(splats, [0, 0, 0, 0, 0, 0, 1, 1, 1, 1])
    splats = torch.stack([sp[:, 1 + dw:1 + dw + H, 1 + dh:1 + dh + W, :, d] for d, (dh, dw) in enumerate(directions)],
                         dim=4)
    if defect == "halo":
        hh, ww = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
        same = torch.stack([((hh + dw) // TILE_H == hh // TILE_H) & ((ww + dh) // TILE_W == ww // TILE_W)
                            for dh, dw in directions], -1)
        splats = splats * same.view(1, H, W, 1, 9, 1)

    k = torch.arange(K).view(1, 1, 1, K, 1)
    o = occ.view(N, H, W, 1, 9)
    layer_mask = torch.stack([o > k, o == k, o < k], dim=5).to(splats.dtype)
    sums = torch.bmm(splats.permute(0, 1, 2, 5, 3, 4).reshape(N * H * W, 5, K * 9),
                     layer_mask.reshape(N * H * W, K * 9, 3)).reshape(N, H, W, 5, 3)
    S, Wt = sums[..., :4, :], sums[..., 4:5, :]
    normed = S * torch.div(1.0, Wt if defect == "no_max" else torch.maximum(Wt, torch.tensor([1.0])))
    out = torch.cat([torch.tensor(background, dtype=torch.float32), torch.tensor([0.0])])
    for layer in ((-3, -2, -1) if defect == "order" else (-1, -2, -3)):
        out = normed[..., layer] + (1.0 - normed[..., 3:4, layer]) * out
    return out


def run_chain(fn, scene):
    colors, coords, mask, grad = (torch.from_numpy(a) for a in scene)
    c, x = colors.clone().requires_grad_(True), coords.clone().requires_grad_(True)
    out = fn(c, x, mask)
    out.backward(grad)
    return {"out": out.detach(), "grad_colors": c.grad, "grad_pixel_coords_screen": x.grad}


@contextlib.contextmanager
def default_dtype(dtype):
    old = torch.get_default_dtype()
    torch.set_default_dtype(dtype)
    try:
        yield
    finally:
        torch.set_default_dtype(old)


# ------------------------------------------------------------------------------------------ CPU: the reference
@pytest.mark.parametrize("args", CPU_SCENES[:2] + [(2, 9, 13, 8, 0.5)])
def test_reference_equals_float64_autograd(args):
    """The backward written out from the header's formulas equals float64 autograd through splatter_chain, on scenes
    whose float32 and float64 occlusion ids agree, to far below the float32 bound.  splatter_chain takes its layer
    masks in float32, so the float64 run goes through defective_chain without a defect, which equals it bit for bit in
    float32 (test_defective_chain_restates_the_suites_chain)."""
    N, H, W, K, sigma = args
    scene = make_scene(N, H, W, K, sigma, seed=5)
    ref, info = reference(*scene, sigma, BG)
    _, info64 = reference(*scene, sigma, BG, z_dtype=np.float64)
    assert np.array_equal(info["occ"], info64["occ"])
    colors, coords, mask, grad = (torch.from_numpy(a) for a in scene)
    with default_dtype(torch.float64):
        c, x = colors.double().requires_grad_(True), coords.double().requires_grad_(True)
        out = defective_chain(c, x, mask, sigma, BG)
        out.backward(grad.double())
    for name, got in (("out", out.detach()), ("grad_colors", c.grad), ("grad_pixel_coords_screen", x.grad)):
        lo, hi, beta = ref[name]
        got = got.numpy()
        err = np.maximum(np.maximum(lo - got, got - hi), 0.0)
        assert (err <= 1e-6 * beta + 1e-300).all(), (args, name, float(err.max()))


def test_reference_closed_form():
    """One pixel, one slot on its centre.  occ_4 = 0 = k puts the splat in layer 1; layers 0 and 2 are empty.  At sigma
    = 1 the splat weighs norm = 1.05 / (1 + 4 e^-1/2 + 4 e^-1) < 1 and the layer is drawn at that alpha over the
    background; at sigma = 1e-4 it weighs 1.05 and is normalised to alpha 1."""
    colors = np.array([0.25, 0.5, 1.0], np.float32).reshape(1, 1, 1, 1, 3)
    coords = np.array([0.5, 0.5, 2.0], np.float32).reshape(1, 1, 1, 1, 3)
    grad = np.zeros((1, 1, 1, 4), np.float32)
    mask = np.zeros((1, 1, 1, 1), bool)
    ref, info = reference(colors, coords, mask, grad, 1.0, BG)
    norm = 1.05 / (1 + 4 * np.exp(-0.5) + 4 * np.exp(-1.0))
    bg = np.array([float(np.float32(x)) for x in BG] + [0.0])
    np.testing.assert_allclose(ref["out"][0].reshape(4), norm * np.array([0.25, 0.5, 1.0, 1.0]) + (1 - norm) * bg,
                               rtol=1e-14)
    assert info["occ"][0, 0, 0, 4] == 0 and info["W1_below_1"] == 1
    ref, info = reference(colors, coords, mask, grad, 1e-4, BG)
    np.testing.assert_allclose(ref["out"][0].reshape(4), [0.25, 0.5, 1.0, 1.0], rtol=1e-14)
    assert info["W1_above_1"] == 1


@pytest.mark.parametrize("args", CPU_SCENES)
def test_float32_chain_within_bound(args):
    """The float32 torch chain of the suite lies within the bound, both sigma extremes included."""
    N, H, W, K, sigma = args
    scene = make_scene(N, H, W, K, sigma, seed=1)
    ref, _ = reference(*scene, sigma, BG)
    got = run_chain(lambda c, x, m: splatter_chain(c, x, m, sigma, BG), scene)
    for name, x in got.items():
        assert_within("%s %s" % (args, name), x, ref[name])


def test_defective_chain_restates_the_suites_chain():
    scene = make_scene(2, 10, 34, 9, 0.5, seed=1)
    a = run_chain(lambda c, x, m: defective_chain(c, x, m, 0.5, BG), scene)
    b = run_chain(lambda c, x, m: splatter_chain(c, x, m, 0.5, BG), scene)
    for name in a:
        assert torch.equal(a[name], b[name]), name


@pytest.mark.parametrize("defect", DEFECTS)
def test_defective_chain_fails(defect):
    """Each defect puts elements outside the bound on at least one CPU scene; "halo" and "chunk" show that the scenes
    see the two bugs the kernels' tiles and chunks are most prone to."""
    outside = 0
    for N, H, W, K, sigma in CPU_SCENES:
        scene = make_scene(N, H, W, K, sigma, seed=1)
        ref, _ = reference(*scene, sigma, BG)
        got = run_chain(lambda c, x, m: defective_chain(c, x, m, sigma, BG, defect), scene)
        outside += sum(count_outside(got[n], ref[n]) for n in got)
    assert outside > 0, "the %s chain passes the bound" % defect


def test_gpu_scenes_reach_every_case():
    """The GPU matrix reaches every case the kernels decide or treat specially."""
    total = {}
    for K in GPU_KS:
        for N, H, W, _, sigma, _ in gpu_scenes(K):
            scene = make_scene(N, H, W, K, sigma)
            _, info = reference(*scene, sigma, BG)
            info["warp_all_empty"], info["warp_some_empty"] = warp_sources(scene[2])
            info["w_zero_sigma_1e-4"] = info["w_zero"] if sigma == 1e-4 else 0
            info["subnormal_products_sigma_1e-4"] = info["subnormal_products"] if sigma == 1e-4 else 0
            info["tile_edge_x"] = N * H * 2 * (W > TILE_W)
            info["tile_edge_y"] = N * W * 2 * (H > TILE_H)
            info["tile_corner"] = N * 4 * (W > TILE_W and H > TILE_H)
            for key, v in info.items():
                if key != "occ":
                    total[key] = total.get(key, 0) + v
    cases = ["occ_neg", "occ_zero", "occ_pos", "tie_in_argmin", "tie_min_a_min_b", "padding", "W0_below_1",
             "W0_above_1", "W1_below_1", "W1_above_1", "W2_below_1", "W2_above_1", "w_zero_sigma_1e-4",
             "subnormal_products_sigma_1e-4", "c_zero", "c_half", "negative_rounding", "tile_edge_x", "tile_edge_y",
             "tile_corner", "warp_all_empty", "warp_some_empty"]
    missing = [k for k in cases if total[k] == 0]
    assert not missing, missing


# ------------------------------------------------------------------------------------------ GPU
DEV = "cuda:0"


def _gpu_matches(scene, sigma, bg_tensor, what, record_property=None):
    """splatter_blend forward and backward through autograd, and _C.splatter_blend_backward, against the reference."""
    from pytorch3d_b200 import _C
    from pytorch3d_b200.blending import BlendParams
    from pytorch3d_b200.splatter_blend import splatter_blend
    colors, coords, mask, grad = (torch.from_numpy(a).to(DEV) for a in scene)
    bg = torch.tensor(BG, dtype=torch.float32, device=DEV) if bg_tensor else BG
    c, x = colors.clone().requires_grad_(True), coords.clone().requires_grad_(True)
    out = splatter_blend(c, x, mask, BlendParams(sigma=sigma, background_color=bg))
    out.backward(grad)
    gc, gx = _C.splatter_blend_backward(grad, colors, coords, mask, sigma, bg)
    ref, _ = reference(*scene, sigma, BG)
    for name, got, key in (("out", out, "out"), ("grad_colors", c.grad, "grad_colors"),
                           ("grad_pixel_coords_screen", x.grad, "grad_pixel_coords_screen"),
                           ("_C grad_colors", gc, "grad_colors"),
                           ("_C grad_pixel_coords_screen", gx, "grad_pixel_coords_screen")):
        if record_property is not None:
            lo, hi, beta = ref[key]
            g = got.detach().cpu().numpy().astype(np.float64)
            ratio = np.maximum(np.maximum(lo - g, g - hi), 0.0) / (2 * beta + FLOOR)
            record_property("%s %s" % (what, name), float(ratio.max()))
        assert_within("%s %s" % (what, name), got, ref[key])
    assert torch.equal(gc, c.grad) and torch.equal(gx, x.grad)
    return ref


@pytest.mark.gpu
@pytest.mark.parametrize("K", GPU_KS)
def test_splatter_matches_fp64(built_lib, record_property, K):
    """Every shape of the matrix at K: tile multiples, partial tiles on both axes, single rows, columns and pixels."""
    for N, H, W, _, sigma, bg_tensor in gpu_scenes(K):
        _gpu_matches(make_scene(N, H, W, K, sigma), sigma, bg_tensor, "K=%d %dx%dx%d sigma=%g" % (K, N, H, W, sigma),
                     record_property)


@pytest.mark.gpu
def test_splatter_matches_fp64_on_rendered_fragments(built_lib, record_property):
    """A torus batch through the fused rasterizer: most deeper layers are empty, the realistic case of the warp skip."""
    from pytorch3d_b200 import _C, synthetic
    m = synthetic.torus_batch(2, 24, 24, seed=2)
    p2f, zbuf = _C.rasterize_meshes_indexed(m.verts_packed().to(DEV), m.faces_packed().to(DEV),
                                            m.mesh_to_faces_packed_first_idx().to(DEV), m.num_faces_per_mesh().to(DEV),
                                            (40, 72), 0.0, 8, False, False, False)[:2]
    mask = (p2f < 0).cpu().numpy()
    N, H, W, K = mask.shape
    assert mask.any() and (~mask).any() and min(warp_sources(mask)) > 0
    rng = np.random.default_rng(3)
    centre = np.stack(np.meshgrid(np.arange(H), np.arange(W), indexing="ij"), -1)[None, :, :, None] + 0.5
    xy = centre + 0.4 * (rng.random((N, H, W, K, 2)) - 0.5)
    coords = np.concatenate([xy, zbuf.cpu().numpy()[..., None]], -1).astype(np.float32)
    colors = rng.random((N, H, W, K, 3)).astype(np.float32)
    grad = rng.normal(0.0, 1.0, (N, H, W, 4)).astype(np.float32)
    _gpu_matches((colors, coords, mask, grad), 0.5, True, "torus", record_property)


@pytest.mark.gpu
def test_splatter_more_than_65535_images(built_lib):
    """65,537 images of 1 x 1: grid.z holds at most 65,535 images per launch."""
    _gpu_matches(make_scene(65537, 1, 1, 2, 0.5), 0.5, False, "N=65537")


@pytest.mark.gpu
def test_splatter_more_than_65535_tile_rows(built_lib):
    """One image of 524,296 x 1: 65,537 tile rows of 8, beyond grid.y's 65,535."""
    _gpu_matches(make_scene(1, 524296, 1, 1, 0.5), 0.5, True, "H=524296")
