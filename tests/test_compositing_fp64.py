"""Point compositing (csrc/compositing.cu) against a float64 reference, on every kernel path.

The reference below restates the four ops from their formulas alone, in float64 torch:

    alpha composite      out_c = sum_k w_k f_c[idx_k],   w_k = cum_k alpha_k,   cum_k = prod_{l<k} (1 - alpha_l)
    weighted sum         out_c = sum_k alpha_k f_c[idx_k]
    normalised sum       out_c = sum_k alpha_k f_c[idx_k] / S,   S = max(sum_k alpha_k, 1e-4)
    fused point render   the alpha composite of alpha = 1 - d * (1 / r^2)

with the reference's semantics: an empty slot (index < 0) may sit anywhere in a pixel's list and is skipped; the
alpha-composite backward is grad_alpha_t = cum_t A_t - sum_{k>t} w_k A_k / (1 - alpha_t + 1e-9) with
A_k = sum_c grad_c f_c[idx_k]; the normalised sum's backward is A_k / S - sum_t alpha_t A_t / S^2 with the clamped S;
the weighted sums read the index as an int.  The fused op forms its alphas in float32 exactly as the renderer's torch
chain does (`1 - dists / (r * r)`); everything after that is float64.  The transmittance is a `cumprod` and the suffix
sums a reversed `cumsum`, so the reference has no division to lose when the float32 product would underflow.

Next to each value the reference returns its magnitude `mag`: the same expression evaluated on absolute values.
Every element of every output must satisfy

    |got - ref| <= (n + 8) * 2^-24 * mag + 1e-35

n = K + C for per-pixel outputs and n = (contributions to that element) + K + C for grad_features: a float32
evaluation of n rounded operations on those terms.  The 1e-35 floor only admits results that are subnormal in
float32.  No element is masked.  The float32 oracle (the reference's CPU ops restated) sums C * K terms into each
grad_alpha, so against it n = C * K + K + C.

In the exact scene every value is a small dyadic rational, so every product and every partial sum is exact in float32
in any order: there the forward pass and grad_features must equal the reference bit for bit.
"""
import numpy as np
import pytest
import torch

import oracle

ULP = 2.0 ** -24
COMP_EPS = 1e-9
NORM_EPS = float(np.float32(1e-4))  # the reference's float threshold

CHANNELS = [1, 3, 4, 5, 8, 9, 17]  # CMAX = 4, 8 and 0 (any C)
WSUM_CHANNELS = [1, 4, 9]
KS = [1, 2, 8, 11, 33, 150]
EMPTIES = ["trailing", "interleaved", "all", "repeat"]
# (regime, K): in the last four the float32 product of the (1 - alpha) underflows
REGIMES = [("uniform", 8), ("zero", 8), ("one_first", 8), ("one_middle", 8), ("one_last", 8), ("recompute", 8),
           ("divide", 8), ("saturated", 10), ("saturated", 20), ("saturated", 40), ("uniform", 150)]
SATURATED = {10: float(np.float32(1 - 6e-6)), 20: 0.995, 40: 0.95}
SCENE = (2, 13, 17)  # N, H, W: small, non-square


def feature_layouts(C):
    return ["contiguous", "point_major", "strided"] + (["point_major_offset"] if C == 4 else [])


def channel_cases(channels):
    return [pytest.param(C, lay, id="C%d-%s" % (C, lay)) for C in channels for lay in feature_layouts(C)]


# ------------------------------------------------------------------------------------------ the float64 reference

def _gather(f, idx):
    """f (C, P), idx (N, K, H, W) -> (N, C, K, H, W); empty slots read point 0 (callers zero their weights)."""
    return f[:, idx.clamp(min=0)].transpose(0, 1)


def _scatter(values, idx, valid, P):
    """Sum of values (N, C, K, H, W) over every valid (n, k, y, x) into (C, P) at idx."""
    C = values.shape[1]
    m = valid.reshape(-1)
    out = values.new_zeros(C, P)
    out.index_add_(1, idx.reshape(-1)[m], values.transpose(0, 1).reshape(C, -1)[:, m])
    return out


def _exclusive_suffix(x):
    """s_k = sum_{t > k} x_t along dim 1 (shifted, so that no term is subtracted back out)."""
    rc = x.flip(1).cumsum(1).flip(1)
    return torch.cat([rc[:, 1:], torch.zeros_like(rc[:, :1])], 1)


def _exclusive_cumprod(x):
    return torch.cumprod(torch.cat([torch.ones_like(x[:, :1]), x[:, :-1]], 1), 1)


def ref_alpha_composite(features, alphas, idx, grad):
    """features (C, P), alphas / idx (N, K, H, W), grad (N, C, H, W) -> {name: (value, mag)} in float64, plus the
    number of contributions to each point."""
    f, a, g = features.double(), alphas.double(), grad.double()
    P = f.shape[1]
    valid = idx >= 0
    a = torch.where(valid, a, torch.zeros_like(a))
    one_minus = torch.where(valid, 1 - a, torch.ones_like(a))
    cum, cum_m = _exclusive_cumprod(one_minus), _exclusive_cumprod(one_minus.abs())
    w, w_m = cum * a, cum_m * a.abs()
    fg = _gather(f, idx)
    out, out_m = (fg * w[:, None]).sum(2), (fg.abs() * w_m[:, None]).sum(2)
    A = (g[:, :, None] * fg).sum(1) * valid
    A_m = (g.abs()[:, :, None] * fg.abs()).sum(1) * valid
    den = 1 - a + COMP_EPS
    ga = torch.where(valid, cum * A - _exclusive_suffix(w * A) / den, torch.zeros_like(a))
    ga_m = torch.where(valid, cum_m * A_m + _exclusive_suffix(w_m * A_m) / den.abs(), torch.zeros_like(a))
    gf = _scatter(g[:, :, None] * w[:, None], idx, valid, P)
    gf_m = _scatter(g.abs()[:, :, None] * w_m[:, None], idx, valid, P)
    count = torch.bincount(idx[valid].reshape(-1), minlength=P)
    return {"out": (out, out_m), "grad_features": (gf, gf_m), "grad_alphas": (ga, ga_m), "count": count}


def ref_weighted_sum(features, alphas, idx, grad, norm):
    """As ref_alpha_composite, for the weighted sum (norm: normalised by the clamped total)."""
    f, a, g = features.double(), alphas.double(), grad.double()
    P = f.shape[1]
    idx = idx.to(torch.int32).long()  # the reference's kernels read the index into an int
    valid = idx >= 0
    a = torch.where(valid, a, torch.zeros_like(a))
    S = a.sum(1, keepdim=True).clamp(min=NORM_EPS) if norm else torch.ones_like(a[:, :1])
    fg = _gather(f, idx)
    out, out_m = (fg * a[:, None]).sum(2) / S, (fg.abs() * a.abs()[:, None]).sum(2) / S
    A = (g[:, :, None] * fg).sum(1) * valid
    A_m = (g.abs()[:, :, None] * fg.abs()).sum(1) * valid
    if norm:
        T, T_m = (a * A).sum(1, keepdim=True), (a.abs() * A_m).sum(1, keepdim=True)
        ga = torch.where(valid, A / S - T / (S * S), torch.zeros_like(a))
        ga_m = torch.where(valid, A_m / S + T_m / (S * S), torch.zeros_like(a))
    else:
        ga, ga_m = A, A_m
    gf = _scatter(g[:, :, None] * (a / S)[:, None], idx, valid, P)
    gf_m = _scatter(g.abs()[:, :, None] * (a.abs() / S)[:, None], idx, valid, P)
    count = torch.bincount(idx[valid].reshape(-1), minlength=P)
    return {"out": (out, out_m), "grad_features": (gf, gf_m), "grad_alphas": (ga, ga_m), "count": count}


def render_inv(radius):
    """1 / r^2 as torch divides a float32 tensor by the scalar r * r: a product with the float32 reciprocal."""
    return np.float32(1.0) / np.float32(radius * radius)


def render_alphas(dists, radius):
    """The renderer's weights, 1 - dists / (r * r), each step rounded to float32."""
    return 1 - dists * torch.tensor(render_inv(radius), device=dists.device)


def ref_render(features, idx, dists, radius, grad):
    """Fused op: idx / dists (N, H, W, K) -> {name: (value, mag)}, with grad_dists in the (N, H, W, K) layout."""
    alphas = render_alphas(dists, radius).permute(0, 3, 1, 2)
    r = ref_alpha_composite(features, alphas, idx.long().permute(0, 3, 1, 2), grad)
    inv = float(render_inv(radius))
    ga, ga_m = r.pop("grad_alphas")
    r["grad_dists"] = (-ga * inv).permute(0, 2, 3, 1), (ga_m * inv).permute(0, 2, 3, 1)
    return r


# ------------------------------------------------------------------------------------------ comparison

def assert_within(name, got, ref, mag, n):
    """|got - ref| <= (n + 8) 2^-24 mag + 1e-35 elementwise (NaN fails)."""
    got = got.double().to(ref.device)
    assert got.shape == ref.shape, (name, got.shape, ref.shape)
    err = (got - ref).abs()
    tol = (n + 8) * ULP * mag + 1e-35
    bad = ~(err <= tol)
    if bool(bad.any()):
        ratio = torch.where(bad, torch.nan_to_num(err / tol, nan=float("inf")), torch.zeros_like(err))
        flat = int(ratio.reshape(-1).argmax())
        at = tuple(int(i) for i in np.unravel_index(flat, tuple(got.shape)))
        n_at = float(n.expand_as(got).reshape(-1)[flat]) if torch.is_tensor(n) else n
        raise AssertionError(
            "%s: %d of %d elements outside (n + 8) 2^-24 mag + 1e-35; worst at %s: got %.9g, want %.9g, mag %.3g, "
            "n %d (%.3g x the bound)" % (name, int(bad.sum()), got.numel(), at, float(got[at]), float(ref[at]),
                                         float(mag[at]), n_at, float(ratio[at])))


def assert_all_within(got, ref, K, C, n_pix=None):
    """got: {name: tensor} for the outputs in ref."""
    n_pix = K + C if n_pix is None else n_pix
    for name, t in got.items():
        value, mag = ref[name]
        n = (ref["count"][None, :] + K + C).double() if name == "grad_features" else n_pix
        assert_within(name, t, value, mag, n)


# ------------------------------------------------------------------------------------------ scenes

def make_scene(K, P, regime="uniform", empties="interleaved", seed=0, shape=SCENE):
    """alphas (N, K, H, W) float32, idx (N, K, H, W) int64, on the CPU."""
    N, H, W = shape
    g = torch.Generator().manual_seed(seed)
    alphas = torch.rand(N, K, H, W, generator=g)
    idx = torch.randint(0, P, (N, K, H, W), generator=g)
    u = torch.rand(N, K, H, W, generator=g)
    if empties == "trailing":  # z-buffer padding: once a slot is empty, so are all later ones
        n_valid = torch.randint(0, K + 1, (N, 1, H, W), generator=g)
        idx[(torch.arange(K).view(1, K, 1, 1) >= n_valid).expand_as(idx)] = -1
    elif empties == "interleaved":
        idx[u < 0.3] = -1
    elif empties == "all":
        idx.fill_(-1)
    elif empties == "repeat":  # the same point in every other slot of a pixel, and a few holes
        idx[:, 1::2] = idx[:, :1].expand_as(idx[:, 1::2])
        idx[u < 0.1] = -1
    else:
        assert empties == "none"
    valid = idx >= 0
    rank = valid.long().cumsum(1) - 1
    count = valid.long().sum(1, keepdim=True)
    j = torch.randint(1, 17, (N, K, H, W), generator=g).double()
    if regime == "zero":
        alphas[u > 0.6] = 0.0
    elif regime.startswith("one_"):
        target = {"one_first": torch.zeros_like(count), "one_middle": count // 2, "one_last": count - 1}[regime]
        alphas[valid & (rank == target)] = 1.0
    elif regime in ("recompute", "divide"):  # two such slots per pixel at most: the product stays a normal float
        sel = valid & (rank % 4 == 1)
        if regime == "divide":  # 1 - alpha in (1e-6, 1e-4]
            j = torch.randint(17, 1678, (N, K, H, W), generator=g).double()
        alphas[sel] = (1 - j * ULP).float()[sel]  # 1 - alpha = j 2^-24, exact in float32
    elif regime == "saturated":
        alphas.fill_(SATURATED[K])
    elif regime == "tiny":  # totals below the 1e-4 floor on every other row
        alphas[:, :, ::2] *= 1e-6
    else:
        assert regime == "uniform"
    return alphas, idx


def make_features(C, P, layout, dev, seed=1):
    """(C, P) float32 features on dev in the given memory layout, and their values on the CPU.  Asserts the
    properties that route each layout through the kernels."""
    vals = torch.rand(C, P, generator=torch.Generator().manual_seed(seed)) * 2 - 1
    if layout == "contiguous":
        f = vals.to(dev)
        assert f.is_contiguous()
    elif layout == "point_major":  # features_packed().permute(1, 0), as the renderer passes them
        f = vals.t().contiguous().to(dev).permute(1, 0)
        assert f.stride() == (1, C) or C == 1  # (C = 1: the same memory as contiguous)
        if C == 4:
            assert f.data_ptr() % 16 == 0  # the 16-byte load / red.global.add.v4.f32 path
    elif layout == "point_major_offset":  # 4 bytes past a 16-byte boundary: the scalar fallback
        buf = torch.zeros(P * C + 1, device=dev)
        buf[1:] = vals.t().reshape(-1).to(dev)
        f = buf[1:].view(P, C).permute(1, 0)
        assert C == 4 and f.stride() == (1, 4) and f.data_ptr() % 16 == 4
    else:
        assert layout == "strided"  # not dense: read through a contiguous copy
        buf = torch.zeros(C, 2 * P, device=dev)
        buf[:, ::2] = vals.to(dev)
        f = buf[:, ::2]
        assert f.stride() == (2 * P, 2)
    assert torch.equal(f.cpu(), vals)
    return f, vals


def place(alphas, idx, layout, dev):
    """alphas / idx as (N, K, H, W) tensors on dev: contiguous, both (N, H, W, K) memory (the renderer's permuted
    rasterizer outputs), or only the alphas so."""
    N, K, H, W = alphas.shape

    def nhwk(t):
        v = t.permute(0, 2, 3, 1).contiguous().to(dev).permute(0, 3, 1, 2)
        assert v.stride() == (H * W * K, 1, W * K, K) or K == 1  # (K = 1: the same memory as contiguous)
        return v

    if layout == "nkhw":
        return alphas.to(dev), idx.to(dev)
    if layout == "nhwk":
        return nhwk(alphas), nhwk(idx)
    assert layout == "alphas_nhwk"
    return nhwk(alphas), idx.to(dev)


def fused_inputs(alphas, idx, radius):
    """The rasterizer's (N, H, W, K) int32 indices and float32 squared distances for a scene, d = (1 - alpha) r^2
    (so alpha is recovered exactly for r = 1 and alpha >= 1/2); empty slots carry d = -1 as the rasterizer writes."""
    i = idx.permute(0, 2, 3, 1).contiguous().int()
    d = ((1 - alphas.double()) * radius * radius).float().permute(0, 2, 3, 1).contiguous()
    d[i < 0] = -1.0
    return i, d


def upstream(N, C, H, W, dev, seed=2):
    return (torch.rand(N, C, H, W, generator=torch.Generator().manual_seed(seed)) * 2 - 1).to(dev)


# ------------------------------------------------------------------------------------------ one call per op

def check_alpha_composite(feats, vals, alphas, idx, layout="nhwk"):
    from pytorch3d_b200 import _C
    dev = feats.device
    (C, P), (N, K, H, W) = vals.shape, alphas.shape
    a, i = place(alphas, idx, layout, dev)
    go = upstream(N, C, H, W, dev)
    out = _C.accum_alphacomposite(feats, a, i)
    gf, ga = _C.accum_alphacomposite_backward(go, feats, a, i)
    point_major = feats.stride() == (1, C) and C > 1
    assert gf.stride() == ((1, C) if point_major else (P, 1)), "grad_features takes the layout of the features"
    ref = ref_alpha_composite(vals.to(dev), alphas.to(dev), idx.to(dev), go)
    assert_all_within({"out": out, "grad_features": gf, "grad_alphas": ga}, ref, K, C)


def check_weighted_sum(feats, vals, alphas, idx, norm, layout="nhwk"):
    from pytorch3d_b200 import _C
    dev = feats.device
    (C, P), (N, K, H, W) = vals.shape, alphas.shape
    a, i = place(alphas, idx, layout, dev)
    go = upstream(N, C, H, W, dev)
    fwd = _C.accum_weightedsumnorm if norm else _C.accum_weightedsum
    bwd = _C.accum_weightedsumnorm_backward if norm else _C.accum_weightedsum_backward
    out = fwd(feats, a, i)
    gf, ga = bwd(go, feats, a, i)
    ref = ref_weighted_sum(vals.to(dev), alphas.to(dev), idx.to(dev), go, norm)
    assert_all_within({"out": out, "grad_features": gf, "grad_alphas": ga}, ref, K, C)


def check_render(feats, vals, alphas, idx, radius):
    from pytorch3d_b200 import _C
    dev = feats.device
    (C, P), (N, K, H, W) = vals.shape, alphas.shape
    ii, dd = (t.to(dev) for t in fused_inputs(alphas, idx, radius))
    # the reference's alpha step is the renderer's torch chain, bit for bit
    assert torch.equal(render_alphas(dd, radius), 1 - dd / (radius * radius))
    go = upstream(N, C, H, W, dev)
    out = _C.points_alpha_render(feats, ii, dd, radius)
    gf, gd = _C.points_alpha_render_backward(go, feats, ii, dd, radius)
    point_major = feats.stride() == (1, C) and C > 1
    assert gf.stride() == ((1, C) if point_major else (P, 1)), "grad_features takes the layout of the features"
    ref = ref_render(vals.to(dev), ii, dd, radius, go)
    assert_all_within({"out": out, "grad_features": gf, "grad_dists": gd}, ref, K, C)


# ------------------------------------------------------------------------------------------ CPU: the reference

ORACLE_SCENES = [("uniform", "interleaved", 8), ("uniform", "trailing", 11), ("uniform", "repeat", 1),
                 ("zero", "interleaved", 8), ("one_middle", "interleaved", 8), ("recompute", "none", 8),
                 ("divide", "none", 8), ("saturated", "none", 10), ("saturated", "none", 20),
                 ("saturated", "none", 40), ("uniform", "interleaved", 150)]


def _oracle_ids(scenes):
    return ["%s-%s-K%d" % s for s in scenes]


@pytest.mark.parametrize("regime,empties,K", ORACLE_SCENES, ids=_oracle_ids(ORACLE_SCENES))
def test_reference_equals_oracle_alpha_composite(regime, empties, K):
    """The float64 reference encodes the reference's semantics: it agrees with the float32 O(K^2) restatement of its
    CPU op, which walks the transmittance front to back and so stays right where the product underflows."""
    C, P = 3, 53
    alphas, idx = make_scene(K, P, regime, empties, seed=K)
    vals = torch.rand(C, P, generator=torch.Generator().manual_seed(3)) * 2 - 1
    go = upstream(SCENE[0], C, SCENE[1], SCENE[2], "cpu")
    ref = ref_alpha_composite(vals, alphas, idx, go)
    out = oracle.alpha_composite(vals.numpy(), alphas.numpy(), idx.numpy(), arith=oracle.ARITH_CPU)
    gf, ga = oracle.alpha_composite_backward(go.numpy(), vals.numpy(), alphas.numpy(), idx.numpy())
    got = {"out": torch.from_numpy(out), "grad_features": torch.from_numpy(gf), "grad_alphas": torch.from_numpy(ga)}
    assert_all_within(got, ref, K, C, n_pix=C * K + K + C)
    if regime == "saturated":  # the scenes that matter: the float32 product underflows, the gradient does not vanish
        assert float(torch.prod(1 - alphas[0, :, 0, 0])) == 0.0
        assert float(ref["grad_features"][0].abs().max()) > 0.1


@pytest.mark.parametrize("norm", [False, True])
@pytest.mark.parametrize("regime,empties,K", ORACLE_SCENES[:5] + [("tiny", "interleaved", 11)],
                         ids=_oracle_ids(ORACLE_SCENES[:5] + [("tiny", "interleaved", 11)]))
def test_reference_equals_oracle_weighted_sum(regime, empties, K, norm):
    C, P = 3, 53
    alphas, idx = make_scene(K, P, regime, empties, seed=K + 1)
    vals = torch.rand(C, P, generator=torch.Generator().manual_seed(4)) * 2 - 1
    go = upstream(SCENE[0], C, SCENE[1], SCENE[2], "cpu")
    ref = ref_weighted_sum(vals, alphas, idx, go, norm)
    out = oracle.weighted_sum(vals.numpy(), alphas.numpy(), idx.numpy(), norm=norm)
    gf, ga = oracle.weighted_sum_backward(go.numpy(), vals.numpy(), alphas.numpy(), idx.numpy(), norm=norm)
    got = {"out": torch.from_numpy(out), "grad_features": torch.from_numpy(gf), "grad_alphas": torch.from_numpy(ga)}
    assert_all_within(got, ref, K, C, n_pix=C * K + K + C)
    if regime == "tiny" and norm:
        assert float((alphas * (idx >= 0)).sum(1)[:, ::2].max()) < NORM_EPS


def test_reference_closed_form():
    """One pixel, three slots with a hole: the formulas written out by hand."""
    f = torch.tensor([[2.0, 3.0, 5.0]])
    a = torch.tensor([0.25, 0.5, 0.75, 0.5]).view(1, 4, 1, 1)
    idx = torch.tensor([0, -1, 1, 2]).view(1, 4, 1, 1)
    go = torch.tensor([2.0]).view(1, 1, 1, 1)
    r = ref_alpha_composite(f, a, idx, go)
    w = [0.25, 0.0, 0.75 * 0.75, 0.75 * 0.25 * 0.5]
    assert float(r["out"][0]) == 0.25 * 2 + w[2] * 3 + w[3] * 5
    assert r["grad_features"][0].tolist() == [[2 * w[0], 2 * w[2], 2 * w[3]]]
    A = [4.0, 0.0, 6.0, 10.0]
    want = [1.0 * A[0] - (w[2] * A[2] + w[3] * A[3]) / (0.75 + COMP_EPS), 0.0,
            0.75 * A[2] - w[3] * A[3] / (0.25 + COMP_EPS), 0.75 * 0.25 * A[3]]
    assert torch.allclose(r["grad_alphas"][0].view(-1), torch.tensor(want, dtype=torch.float64), rtol=1e-15)
    s = ref_weighted_sum(f, a, idx, go, norm=True)
    total = 0.25 + 0.75 + 0.5
    assert float(s["out"][0]) == pytest.approx((0.25 * 2 + 0.75 * 3 + 0.5 * 5) / total, rel=1e-15)


# ------------------------------------------------------------------------------------------ GPU: alpha composite

@pytest.mark.gpu
@pytest.mark.parametrize("C,layout", channel_cases(CHANNELS))
def test_alpha_composite_channel_paths(built_lib, C, layout):
    feats, vals = make_features(C, 97, layout, torch.device("cuda:0"))
    alphas, idx = make_scene(11, 97, seed=C)
    check_alpha_composite(feats, vals, alphas, idx)


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["nkhw", "nhwk", "alphas_nhwk"])
def test_alpha_composite_alpha_layouts(built_lib, layout):
    feats, vals = make_features(4, 97, "point_major", torch.device("cuda:0"))
    alphas, idx = make_scene(11, 97, seed=5)
    check_alpha_composite(feats, vals, alphas, idx, layout)


@pytest.mark.gpu
@pytest.mark.parametrize("empties", EMPTIES)
@pytest.mark.parametrize("K", KS)
def test_alpha_composite_slots(built_lib, K, empties):
    feats, vals = make_features(4, 61, "point_major", torch.device("cuda:0"))
    alphas, idx = make_scene(K, 61, "uniform", empties, seed=K)
    check_alpha_composite(feats, vals, alphas, idx)


@pytest.mark.gpu
@pytest.mark.parametrize("C,layout", [(4, "point_major"), (9, "contiguous")])
@pytest.mark.parametrize("regime,K", REGIMES, ids=["%s-K%d" % r for r in REGIMES])
def test_alpha_composite_regimes(built_lib, regime, K, C, layout):
    feats, vals = make_features(C, 61, layout, torch.device("cuda:0"))
    alphas, idx = make_scene(K, 61, regime, "none" if regime == "saturated" else "interleaved", seed=K + 2)
    check_alpha_composite(feats, vals, alphas, idx)


# ------------------------------------------------------------------------------------------ GPU: weighted sums

@pytest.mark.gpu
@pytest.mark.parametrize("norm", [False, True])
@pytest.mark.parametrize("C,layout", channel_cases(WSUM_CHANNELS))
def test_weighted_sum_channel_paths(built_lib, C, layout, norm):
    feats, vals = make_features(C, 97, layout, torch.device("cuda:0"))
    alphas, idx = make_scene(11, 97, seed=C + 10)
    check_weighted_sum(feats, vals, alphas, idx, norm)


@pytest.mark.gpu
@pytest.mark.parametrize("norm", [False, True])
@pytest.mark.parametrize("layout", ["nkhw", "nhwk", "alphas_nhwk"])
def test_weighted_sum_alpha_layouts(built_lib, layout, norm):
    feats, vals = make_features(4, 97, "point_major", torch.device("cuda:0"))
    alphas, idx = make_scene(11, 97, seed=6)
    check_weighted_sum(feats, vals, alphas, idx, norm, layout)


@pytest.mark.gpu
@pytest.mark.parametrize("norm", [False, True])
@pytest.mark.parametrize("empties", EMPTIES)
@pytest.mark.parametrize("K", KS)
def test_weighted_sum_slots(built_lib, K, empties, norm):
    feats, vals = make_features(4, 61, "contiguous", torch.device("cuda:0"))
    alphas, idx = make_scene(K, 61, "uniform", empties, seed=K + 20)
    check_weighted_sum(feats, vals, alphas, idx, norm)


@pytest.mark.gpu
@pytest.mark.parametrize("norm", [False, True])
@pytest.mark.parametrize("regime", ["zero", "one_middle", "tiny"])
def test_weighted_sum_regimes(built_lib, regime, norm):
    feats, vals = make_features(4, 61, "contiguous", torch.device("cuda:0"))
    alphas, idx = make_scene(11, 61, regime, seed=30)
    if regime == "tiny":
        assert float((alphas * (idx >= 0)).sum(1)[:, ::2].max()) < NORM_EPS
    check_weighted_sum(feats, vals, alphas, idx, norm)


# ------------------------------------------------------------------------------------------ GPU: fused point render

@pytest.mark.gpu
@pytest.mark.parametrize("C,layout", channel_cases(CHANNELS))
def test_render_channel_paths(built_lib, C, layout):
    feats, vals = make_features(C, 97, layout, torch.device("cuda:0"))
    alphas, idx = make_scene(11, 97, seed=C + 40)
    check_render(feats, vals, alphas, idx, radius=0.05)


@pytest.mark.gpu
@pytest.mark.parametrize("empties", EMPTIES)
@pytest.mark.parametrize("K", KS)
def test_render_slots(built_lib, K, empties):
    feats, vals = make_features(4, 61, "point_major", torch.device("cuda:0"))
    alphas, idx = make_scene(K, 61, "uniform", empties, seed=K + 50)
    check_render(feats, vals, alphas, idx, radius=1.0)


@pytest.mark.gpu
@pytest.mark.parametrize("C,layout", [(4, "point_major"), (9, "contiguous")])
@pytest.mark.parametrize("regime,K", REGIMES, ids=["%s-K%d" % r for r in REGIMES])
def test_render_regimes(built_lib, regime, K, C, layout):
    """r = 1, so each scene's alphas reach the kernel unchanged (d = 1 - alpha exactly for alpha >= 1/2)."""
    feats, vals = make_features(C, 61, layout, torch.device("cuda:0"))
    alphas, idx = make_scene(K, 61, regime, "none" if regime == "saturated" else "interleaved", seed=K + 60)
    check_render(feats, vals, alphas, idx, radius=1.0)


# ------------------------------------------------------------------------------------------ GPU: whole-op properties

@pytest.mark.gpu
@pytest.mark.parametrize("op", ["alpha_composite", "weighted_sum", "norm_weighted_sum", "render"])
def test_grid_stride_second_pass(built_lib, op):
    """More pixels than the grid has threads (it is capped at 32 blocks of 256 per SM), so each thread takes a
    second pixel."""
    dev = torch.device("cuda:0")
    threads = torch.cuda.get_device_properties(dev).multi_processor_count * 32 * 256
    H, W = 1024, (threads * 5 // 4 + 1023) // 1024 | 1  # a quarter of the pixels in the second pass
    assert H * W >= threads * 5 // 4
    feats, vals = make_features(4, 4099, "point_major", dev)
    alphas, idx = make_scene(2, 4099, seed=70, shape=(1, H, W))
    if op == "alpha_composite":
        check_alpha_composite(feats, vals, alphas, idx)
    elif op == "render":
        check_render(feats, vals, alphas, idx, radius=0.05)
    else:
        check_weighted_sum(feats, vals, alphas, idx, op == "norm_weighted_sum")


def _dyadic(t, b):
    return bool(torch.equal(t * 2.0 ** b, torch.round(t * 2.0 ** b)))


@pytest.mark.gpu
@pytest.mark.parametrize("C,layout", [(4, "point_major"), (3, "contiguous")])
@pytest.mark.parametrize("op", ["alpha_composite", "weighted_sum", "render"])
def test_exact_scene_under_contention(built_lib, op, C, layout):
    """16384 pixels x 4 slots hit 4 points.  alpha in {1/4, 1/2, 3/4}, integer features and upstream gradients: every
    value is a multiple of 2^-b and every sum of absolute contributions stays below 2^(24-b), so every partial sum is
    exact in float32 whatever order the atomics run in.  The forward pass and grad_features must then be the
    reference's values exactly: a dropped, doubled or misrouted contribution cannot hide in a tolerance."""
    from pytorch3d_b200 import _C
    dev = torch.device("cuda:0")
    N, K, H, W, P = 1, 4, 128, 128, 4
    g = torch.Generator().manual_seed(80)
    alphas = torch.randint(1, 4, (N, K, H, W), generator=g).float() / 4
    idx = torch.randint(0, P, (N, K, H, W), generator=g)
    idx[torch.rand(N, K, H, W, generator=g) < 0.2] = -1
    vals = torch.randint(-3, 4, (C, P), generator=g).float()
    go = torch.randint(-2, 3, (N, C, H, W), generator=g).float().to(dev)
    feats = vals.to(dev) if layout == "contiguous" else vals.t().contiguous().to(dev).permute(1, 0)
    if layout == "point_major":
        assert feats.stride() == (1, 4) and feats.data_ptr() % 16 == 0
    if op == "alpha_composite":
        a, i = place(alphas, idx, "nhwk", dev)
        out = _C.accum_alphacomposite(feats, a, i)
        gf, ga = _C.accum_alphacomposite_backward(go, feats, a, i)
        ref = ref_alpha_composite(vals.to(dev), alphas.to(dev), idx.to(dev), go)
        b = 2 * K  # w_k: a product of at most K factors in {1/4, 1/2, 3/4}
    elif op == "render":
        ii, dd = (t.to(dev) for t in fused_inputs(alphas, idx, 1.0))
        valid = idx >= 0
        assert torch.equal(render_alphas(dd, 1.0).permute(0, 3, 1, 2).cpu()[valid], alphas[valid])  # r = 1: exact
        out = _C.points_alpha_render(feats, ii, dd, 1.0)
        gf, ga = _C.points_alpha_render_backward(go, feats, ii, dd, 1.0)
        ref = ref_render(vals.to(dev), ii, dd, 1.0, go)
        ref["grad_alphas"] = ref.pop("grad_dists")
        b = 2 * K
    else:
        a, i = place(alphas, idx, "nhwk", dev)
        out = _C.accum_weightedsum(feats, a, i)
        gf, ga = _C.accum_weightedsum_backward(go, feats, a, i)
        ref = ref_weighted_sum(vals.to(dev), alphas.to(dev), idx.to(dev), go, norm=False)
        b = 2
    assert int(ref["count"].min()) >= 4096
    for name in ("out", "grad_features"):
        value, mag = ref[name]
        assert _dyadic(value, b) and float(mag.max()) < 2.0 ** (24 - b), name
    assert torch.equal(out.double(), ref["out"][0]), "forward differs from the exact result"
    assert torch.equal(gf.double(), ref["grad_features"][0]), "grad_features differs from the exact result"
    assert_within("grad_alphas", ga, *ref["grad_alphas"], n=K + C)


@pytest.mark.gpu
@pytest.mark.parametrize("op", ["alpha_composite", "weighted_sum", "norm_weighted_sum", "render_points_alpha"])
def test_autograd_wrappers_point_major(built_lib, op):
    """The autograd functions with the renderer's point-major features: gradients in the inputs' layouts, equal to
    the reference's."""
    from pytorch3d_b200 import compositing
    dev = torch.device("cuda:0")
    C, P, K = 4, 61, 33
    alphas, idx = make_scene(K, P, seed=90)
    feats, vals = make_features(C, P, "point_major", dev)
    feats.requires_grad_(True)
    go = upstream(SCENE[0], C, SCENE[1], SCENE[2], dev)
    if op == "render_points_alpha":
        ii, dd = (t.to(dev) for t in fused_inputs(alphas, idx, 0.05))
        x = dd.clone().requires_grad_(True)
        out = compositing.render_points_alpha((ii, None, x), feats, 0.05)
        ref = ref_render(vals.to(dev), ii, dd, 0.05, go)
        second = "grad_dists"
    else:
        a, i = place(alphas, idx, "nhwk", dev)
        x = a.clone().requires_grad_(True)  # clone keeps the permuted strides
        assert x.stride() == a.stride()
        out = getattr(compositing, op)(i, x, feats)
        if op == "alpha_composite":
            ref = ref_alpha_composite(vals.to(dev), alphas.to(dev), idx.to(dev), go)
        else:
            ref = ref_weighted_sum(vals.to(dev), alphas.to(dev), idx.to(dev), go, op == "norm_weighted_sum")
        second = "grad_alphas"
    (out * go).sum().backward()
    assert feats.grad.stride() == feats.stride() == (1, C)
    assert x.grad.stride() == x.stride()
    assert_all_within({"out": out.detach(), "grad_features": feats.grad, second: x.grad}, ref, K, C)
