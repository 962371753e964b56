"""Splatter blending (DESIGN.md section 11): the fused `splatter_blend` against a torch restatement of the reference's
pytorch3d/renderer/splatter_blend.py, `SplatterBlender`, and `install_splatter()`.

The stored outputs of the reference (tests/golden/reference_golden_splatter.npz, tests/golden/make_splatter_golden.py)
pin the restatement below to the reference: its SplatterBlender run on the CPU with an identity camera."""
import sys
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import assert_equals_reference, reference

# ------------------------------------------------------------------------------------------------ scenes
# (N, H, W, K, sigma, kind): kind "centre" = positions within 0.05 px of the pixel centres, "far" = anywhere up to
# +-0.5 px away, "ties" = depths on a coarse grid (exact ties across layers and between neighbours).
SPLATTER_CASES = [(2, 9, 13, 1, 0.5, "centre"), (1, 7, 10, 1, 0.3, "far"), (2, 9, 13, 2, 0.5, "far"),
                  (2, 9, 13, 2, 0.3, "ties"), (2, 9, 13, 4, 0.3, "centre"), (1, 11, 6, 4, 0.5, "ties"),
                  (2, 9, 13, 8, 0.5, "far"), (2, 9, 13, 8, 0.3, "ties")]
BACKGROUND = (0.2, 0.4, 0.6)


def splatter_case(args):
    return "splatter/" + "-".join(str(a) for a in args)


def splatter_scene(N, H, W, K, sigma=0.5, kind="far", seed=0, device="cpu", frac_background=0.3):
    """colors, pixel_coords_screen, background_mask, upstream gradient (N,H,W,4)."""
    g = torch.Generator().manual_seed(seed + 1000 * K + 7 * H + W)
    hh, ww = torch.meshgrid(torch.arange(H) + 0.5, torch.arange(W) + 0.5, indexing="ij")
    xy = torch.stack([hh, ww], -1)[None, :, :, None].expand(N, H, W, K, 2)
    if kind == "centre":
        xy = xy + 0.05 * (2 * torch.rand(N, H, W, K, 2, generator=g) - 1)
    else:
        xy = xy + (torch.rand(N, H, W, K, 2, generator=g) - 0.5)
    z = torch.sort(1.0 + 5.0 * torch.rand(N, H, W, K, generator=g), dim=-1).values
    if kind == "ties":
        z = torch.round(z)  # 1..6: equal depths in neighbouring pixels and within a pixel
    coords = torch.cat([xy, z[..., None]], -1).contiguous()
    colors = torch.rand(N, H, W, K, 3, generator=g)
    mask = torch.rand(N, H, W, K, generator=g) < frac_background
    grad = torch.randn(N, H, W, 4, generator=g)
    return [t.to(device) for t in (colors, coords, mask, grad)]


def quirk_scene(device="cpu"):
    """A depth step between columns 2 and 3: the left half at depths (1, 4), the right half at (4, 7) -- the far
    surface is the second layer of the near one.  Directions d whose occlusion neighbour and splat source differ
    (d = 1, 2, 3, 5, 6, 7) classify splats across the step with the other neighbour's occlusion id, so the image depends
    on the direction pairing."""
    g = torch.Generator().manual_seed(11)
    N, H, W, K = 1, 6, 7, 2
    hh, ww = torch.meshgrid(torch.arange(H) + 0.5, torch.arange(W) + 0.5, indexing="ij")
    xy = torch.stack([hh, ww], -1)[None, :, :, None].expand(N, H, W, K, 2)
    xy = xy + 0.4 * (torch.rand(N, H, W, K, 2, generator=g) - 0.5)
    near = torch.arange(W) < 3
    z0 = torch.where(near, 1.0, 4.0).view(1, 1, W, 1).expand(N, H, W, 1)
    z = torch.cat([z0, z0 + 3.0], -1)
    coords = torch.cat([xy, z[..., None]], -1).contiguous()
    colors = torch.rand(N, H, W, K, 3, generator=g)
    mask = torch.zeros(N, H, W, K, dtype=torch.bool)
    mask[0, 0, 0, 1] = True
    grad = torch.randn(N, H, W, 4, generator=g)
    return [t.to(device) for t in (colors, coords, mask, grad)]


# ------------------------------------------------------------------------------------------------ restatement
def splatter_chain(colors, pixel_coords_screen, background_mask, sigma, background, pairing="reference"):
    """The torch chain of the reference's SplatterBlender.forward after its projection step, in the same operations.

    pairing "reference": the splat of direction d comes from the neighbour at (d%3 - 1, d//3 - 1) while its occlusion
    id was computed against the neighbour at (d//3 - 1, d%3 - 1), as in the reference.  "corrected": the occlusion id of
    the neighbour that sends the splat."""
    N, H, W, K, _ = colors.shape
    dev = colors.device
    m = background_mask[..., None]
    coords = torch.where(m, torch.ones((), device=dev), pixel_coords_screen)  # background: (1, 1, 1)
    rgba = torch.cat([colors, torch.ones_like(colors[..., :1])], dim=-1)
    rgba = torch.where(m, torch.zeros((), device=dev), rgba)  # background: RGBA 0
    directions = [(d // 3 - 1, d % 3 - 1) for d in range(9)]

    # occlusion ids: the 3 x 3 neighbourhood of the depths, zero padded
    z = coords[..., 2].permute(0, 3, 1, 2)  # (N, K, H, W)
    zp = F.pad(z, [1, 1, 1, 1])
    p = torch.stack([zp[:, :, 1 + dh:1 + dh + H, 1 + dw:1 + dw + W] for dh, dw in directions], dim=2)  # (N,K,9,H,W)
    q = z.view(N, K, 1, H, W)
    min_a, arg_a = torch.abs(p - q[:, 0:1]).min(dim=1)
    min_b, arg_b = torch.abs(p[:, 0:1] - q).min(dim=1)
    occ = torch.where(min_b < min_a, -arg_b, arg_a).permute(0, 2, 3, 1)  # (N, H, W, 9)
    if pairing == "corrected":
        occ = occ[..., [(d % 3) * 3 + d // 3 for d in range(9)]]

    # splat colours and weights of each source slot in each direction
    offsets = torch.tensor(directions, dtype=torch.long, device=dev)
    norm = torch.div(1.05, torch.exp(-torch.square(offsets).sum(dim=1) / (2 * sigma ** 2)).sum())
    c = (torch.floor(coords[..., :2]) - coords[..., :2] + 0.5).view(N, H, W, K, 1, 2)
    w = torch.exp(-torch.sum(torch.square(c + offsets), dim=5) / (2 * sigma ** 2))
    sw = (rgba[..., 3:4] * norm * w).unsqueeze(5)  # (N, H, W, K, 9, 1)
    splats = torch.cat([sw * rgba.unsqueeze(4), sw], dim=5)  # (N, H, W, K, 9, 5)

    # the splat pixel (h, w) receives in direction d comes from (h + d%3 - 1, w + d//3 - 1); zero outside the image
    sp = F.pad(splats, [0, 0, 0, 0, 0, 0, 1, 1, 1, 1])
    splats = torch.stack([sp[:, 1 + dw:1 + dw + H, 1 + dh:1 + dh + W, :, d] for d, (dh, dw) in enumerate(directions)],
                         dim=4)

    # per-layer sums: layer 0 where occ > k, 1 where occ == k, 2 where occ < k
    k = torch.arange(K, device=dev).view(1, 1, 1, K, 1)
    o = occ.view(N, H, W, 1, 9)
    layer_mask = torch.stack([o > k, o == k, o < k], dim=5).float()  # (N, H, W, K, 9, 3)
    sums = torch.bmm(splats.permute(0, 1, 2, 5, 3, 4).reshape(N * H * W, 5, K * 9),
                     layer_mask.reshape(N * H * W, K * 9, 3)).reshape(N, H, W, 5, 3)
    S, Wt = sums[..., :4, :], sums[..., 4:5, :]

    # normalise each layer, compose layers 2, 1, 0 over the background
    normed = S * torch.div(1.0, torch.maximum(Wt, torch.tensor([1.0], device=dev)))
    bg = background.to(dev) if torch.is_tensor(background) else torch.tensor(background, dtype=torch.float32,
                                                                             device=dev)
    out = torch.cat([bg, torch.tensor([0.0], device=dev)])
    for layer in (-1, -2, -3):
        out = normed[..., layer] + (1.0 - normed[..., 3:4, layer]) * out
    return out


def with_grads(fn, colors, coords, mask, grad):
    c, x = colors.clone().requires_grad_(True), coords.clone().requires_grad_(True)
    out = fn(c, x, mask)
    out.backward(grad)
    return [out.detach(), c.grad, x.grad]


def chain_fn(sigma, background=BACKGROUND, pairing="reference"):
    return lambda c, x, m: splatter_chain(c, x, m, sigma, background, pairing)


def fused_fn(sigma, background=BACKGROUND):
    from pytorch3d_b200.blending import BlendParams
    from pytorch3d_b200.splatter_blend import splatter_blend
    params = BlendParams(sigma=sigma, background_color=background)
    return lambda c, x, m: splatter_blend(c, x, m, params)


# ------------------------------------------------------------------------------------------------ CPU tests
@pytest.mark.parametrize("args", SPLATTER_CASES)
def test_splatter_chain_equals_reference_cpu(args):
    colors, coords, mask, grad = splatter_scene(*args)
    got = with_grads(chain_fn(args[4]), colors, coords, mask, grad)
    assert_equals_reference(got, splatter_case(args), "torch restatement vs the reference's SplatterBlender (CPU)")


def test_quirk_scene_depends_on_the_direction_pairing_cpu():
    colors, coords, mask, grad = quirk_scene()
    got = with_grads(chain_fn(0.5), colors, coords, mask, grad)
    assert_equals_reference(got, "splatter/quirk", "restatement vs the reference on the pairing scene (CPU)")
    corrected = with_grads(chain_fn(0.5, pairing="corrected"), colors, coords, mask, grad)
    assert not torch.equal(got[0], corrected[0]), "the scene must be sensitive to the direction pairing"
    assert (got[0] - corrected[0]).abs().max() > 1e-3


def test_splatter_argument_errors():
    from pytorch3d_b200 import _C
    from pytorch3d_b200.blending import BlendParams
    from pytorch3d_b200.splatter_blend import splatter_blend
    colors, coords, mask, grad = splatter_scene(1, 3, 4, 2)
    with pytest.raises(RuntimeError, match="CUDA"):
        _C.splatter_blend(colors, coords, mask, 0.5, BACKGROUND)
    with pytest.raises(RuntimeError, match="CUDA"):
        _C.splatter_blend_backward(grad, colors, coords, mask, 0.5, BACKGROUND)
    with pytest.raises(RuntimeError):
        _C.splatter_blend(colors.double(), coords, mask, 0.5, BACKGROUND)
    with pytest.raises(ValueError, match="Only positive standard deviations make sense."):
        splatter_blend(colors, coords, mask, BlendParams(sigma=0.0))
    with pytest.raises(ValueError, match="Only positive standard deviations make sense."):
        splatter_blend(colors, coords, mask, BlendParams(sigma=-0.5))
    with pytest.raises(ValueError, match="background_color"):
        splatter_blend(colors, coords, mask, BlendParams(sigma=0.5, background_color=torch.ones(3, requires_grad=True)))
    with pytest.raises(RuntimeError, match="CUDA"):
        splatter_blend(colors, coords, mask, BlendParams(sigma=0.5))


class _IdentityCamera:
    """Duck-typed camera: positions are already in screen space."""

    def __init__(self):
        self.calls = []

    def transform_points_screen(self, points, image_size, with_xyflip=True):
        self.calls.append((tuple(points.shape), tuple(image_size), with_xyflip))
        return points * 1.0


def _fake_pytorch3d(monkeypatch):
    calls = []

    class RefSplatterBlender(torch.nn.Module):
        def __init__(self, input_shape, device):
            super().__init__()
            calls.append(("init", tuple(input_shape), device))

        def forward(self, colors, pixel_coords_cameras, cameras, background_mask, blend_params):
            calls.append("ref_forward")
            return "ref_splatter"

    for n in ["pytorch3d", "pytorch3d.renderer", "pytorch3d.renderer.splatter_blend", "pytorch3d.renderer.mesh",
              "pytorch3d.renderer.mesh.shader"]:
        m = types.ModuleType(n)
        m.__path__ = []
        monkeypatch.setitem(sys.modules, n, m)
    for n in ("pytorch3d.renderer.splatter_blend", "pytorch3d.renderer.mesh.shader"):
        sys.modules[n].SplatterBlender = RefSplatterBlender
    return RefSplatterBlender, calls


def _stand_in(shape, dtype=torch.float32, is_cuda=True):
    """An object that claims to be a tensor on the GPU (routing looks at device, dtype and shape only)."""
    return types.SimpleNamespace(is_cuda=is_cuda, dtype=dtype, shape=torch.Size(shape), dim=lambda: len(shape))


def test_install_splatter_and_uninstall(monkeypatch, built_lib):
    from pytorch3d_b200 import install as inst
    from pytorch3d_b200 import splatter_blend as ours
    ref_cls, calls = _fake_pytorch3d(monkeypatch)
    patched = inst.install_splatter()
    assert patched == ["pytorch3d.renderer.splatter_blend", "pytorch3d.renderer.mesh.shader"]
    sb, sh = sys.modules["pytorch3d.renderer.splatter_blend"], sys.modules["pytorch3d.renderer.mesh.shader"]
    assert sb.SplatterBlender is not ref_cls and sh.SplatterBlender is not ref_cls
    routed = []
    monkeypatch.setattr(ours, "splatter_blend", lambda c, x, m, p: routed.append("fused") or "b200_splatter")
    cam = _IdentityCamera()
    params = types.SimpleNamespace(sigma=0.5, background_color=(1.0, 1.0, 1.0))
    blender = sh.SplatterBlender((1, 2, 3, 4), "cuda:0")
    # CPU tensors, float64 and a background colour that requires grad keep the original class
    cpu = torch.zeros(1, 2, 3, 4, 3)
    mask = torch.zeros(1, 2, 3, 4, dtype=torch.bool)
    assert blender(cpu, cpu, cam, mask, params) == "ref_splatter"
    assert calls[0] == ("init", (1, 2, 3, 4), "cuda:0")
    cuda64 = _stand_in((1, 2, 3, 4, 3), torch.float64)
    assert blender(cuda64, cuda64, cam, mask, params) == "ref_splatter"
    grad_bg = types.SimpleNamespace(sigma=0.5, background_color=torch.ones(3, requires_grad=True))
    cuda32 = _stand_in((1, 2, 3, 4, 3))
    assert blender(cuda32, cuda32, cam, mask, grad_bg) == "ref_splatter"
    too_deep = _stand_in((1, 2, 3, 151, 3))
    assert blender(too_deep, too_deep, cam, mask, params) == "ref_splatter"
    assert routed == [] and calls.count("ref_forward") == 4 and len([c for c in calls if c[0] == "init"]) == 1
    # CUDA float32 inputs go to the fused op, after the reference's projection
    xyz = torch.zeros(1, 2, 3, 4, 3)
    xyz_cuda = types.SimpleNamespace(is_cuda=True, dtype=torch.float32, shape=xyz.shape, dim=xyz.dim, view=xyz.view)
    assert blender(cuda32, xyz_cuda, cam, mask, params) == "b200_splatter"
    assert routed == ["fused"] and cam.calls[-1] == ((1, 24, 3), (2, 3), False)
    assert isinstance(sb.SplatterBlender((1, 1, 1, 1), "cpu"), torch.nn.Module)
    inst.uninstall()
    assert sb.SplatterBlender is ref_cls and sh.SplatterBlender is ref_cls


def test_install_splatter_leaves_install_blending_alone(monkeypatch, built_lib):
    from pytorch3d_b200 import install as inst
    ref_cls, _ = _fake_pytorch3d(monkeypatch)
    inst.install_splatter()
    try:
        assert ("pytorch3d.renderer.mesh.shader", "softmax_rgb_blend") not in inst._saved_blend
    finally:
        inst.uninstall()
    assert inst._saved_blend == {}


# ------------------------------------------------------------------------------------------------ GPU tests
DEV = "cuda:0"


def _assert_close(got, want, what=""):
    """Forward rtol 1e-5 / atol 1e-6; gradients rtol 1e-4 / atol 1e-5 of the largest magnitude."""
    np.testing.assert_allclose(got[0].cpu().numpy(), want[0].cpu().numpy(), rtol=1e-5, atol=1e-6, err_msg=what)
    for i, name in ((1, "colors"), (2, "pixel_coords_screen")):
        b = want[i].cpu().numpy()
        np.testing.assert_allclose(got[i].cpu().numpy(), b, rtol=1e-4, atol=1e-5 * float(np.abs(b).max()) + 1e-30,
                                   err_msg="%s grad_%s" % (what, name))


def _assert_exact_zeros(got, mask, what=""):
    assert torch.equal(got[2][..., 2], torch.zeros_like(got[2][..., 2])), "%s: the z gradient must be exactly 0" % what
    assert (got[1][mask] == 0).all() and (got[2][mask] == 0).all(), "%s: background slots must get exactly 0" % what


def _tf32_off():
    assert not torch.backends.cuda.matmul.allow_tf32, "the torch chain's bmm must run in full float32"


@pytest.mark.gpu
@pytest.mark.parametrize("args", SPLATTER_CASES + ["quirk"])
def test_fused_matches_reference_records(built_lib, args):
    if args == "quirk":
        colors, coords, mask, grad = quirk_scene(DEV)
        sigma, case = 0.5, "splatter/quirk"
    else:
        colors, coords, mask, grad = splatter_scene(*args, device=DEV)
        sigma, case = args[4], splatter_case(args)
    got = with_grads(fused_fn(sigma), colors, coords, mask, grad)
    for mine, ref, (rtol, name) in zip(got, reference(case), ((1e-5, "out"), (1e-4, "colors"), (1e-4, "coords"))):
        atol = 1e-6 if name == "out" else 1e-5 * max(ref.absmax, 1e-30)
        np.testing.assert_allclose(ref.rows_of(mine), ref.sample, rtol=rtol, atol=atol, err_msg="%s %s" % (case, name))
    _assert_exact_zeros(got, mask, case)


@pytest.mark.gpu
@pytest.mark.parametrize("sigma", [0.5, 0.25])
@pytest.mark.parametrize("K", [1, 2, 8, 13, 40, 150])
def test_fused_matches_torch_chain(built_lib, K, sigma):
    _tf32_off()
    colors, coords, mask, grad = splatter_scene(2, 33, 17, K, sigma, "far", device=DEV)
    got = with_grads(fused_fn(sigma), colors, coords, mask, grad)
    want = with_grads(chain_fn(sigma), colors, coords, mask, grad)
    _assert_close(got, want, "K=%d sigma=%g" % (K, sigma))
    _assert_exact_zeros(got, mask, "K=%d" % K)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(1, 1, 40), (1, 37, 1), (1, 1, 1), (3, 8, 32), (1, 9, 70)])
@pytest.mark.parametrize("K,kind", [(1, "far"), (8, "ties"), (13, "far")])
def test_fused_matches_torch_chain_on_odd_sizes(built_lib, shape, K, kind):
    _tf32_off()
    colors, coords, mask, grad = splatter_scene(*shape, K, 0.5, kind, device=DEV)
    got = with_grads(fused_fn(0.5), colors, coords, mask, grad)
    want = with_grads(chain_fn(0.5), colors, coords, mask, grad)
    _assert_close(got, want, "shape=%s K=%d %s" % (shape, K, kind))
    _assert_exact_zeros(got, mask, "shape=%s" % (shape,))


@pytest.mark.gpu
def test_all_background_gives_the_background(built_lib):
    from pytorch3d_b200 import _C
    colors, coords, _, grad = splatter_scene(2, 9, 13, 4, device=DEV)
    mask = torch.ones(colors.shape[:4], dtype=torch.bool, device=DEV)
    for bg in (BACKGROUND, torch.tensor([0.3, 0.1, 0.9], device=DEV)):
        out = _C.splatter_blend(colors, coords, mask, 0.5, bg)
        bgt = torch.tensor(bg, device=DEV) if not torch.is_tensor(bg) else bg
        want = torch.cat([bgt, torch.zeros(1, device=DEV)]).expand_as(out)
        assert torch.equal(out, want)
        gc, gx = _C.splatter_blend_backward(grad, colors, coords, mask, 0.5, bg)
        assert not gc.any() and not gx.any()


@pytest.mark.gpu
@pytest.mark.parametrize("K", [8, 13])
def test_unaligned_inputs_give_identical_bits(built_lib, K):
    from pytorch3d_b200 import _C
    colors, coords, mask, grad = splatter_scene(2, 9, 13, K, device=DEV)

    def shifted(t):
        flat = torch.empty(t.numel() + 1, dtype=t.dtype, device=t.device)
        out = flat[1:].view(t.shape)
        out.copy_(t)
        return out

    want_f = _C.splatter_blend(colors, coords, mask, 0.5, BACKGROUND)
    want_b = _C.splatter_blend_backward(grad, colors, coords, mask, 0.5, BACKGROUND)
    sc, sx, sm, sg = (shifted(t) for t in (colors, coords, mask, grad))
    assert sg.data_ptr() % 16 != 0
    assert torch.equal(_C.splatter_blend(sc, sx, sm, 0.5, BACKGROUND), want_f)
    for a, b in zip(_C.splatter_blend_backward(sg, sc, sx, sm, 0.5, BACKGROUND), want_b):
        assert torch.equal(a, b)


@pytest.mark.gpu
def test_splatter_errors_on_the_device(built_lib):
    from pytorch3d_b200 import _C
    colors, coords, mask, grad = splatter_scene(1, 3, 4, 2, device=DEV)
    with pytest.raises(RuntimeError, match="Float"):
        _C.splatter_blend(colors.double(), coords, mask, 0.5, BACKGROUND)
    with pytest.raises(RuntimeError, match="Float"):
        _C.splatter_blend(colors, coords.half(), mask, 0.5, BACKGROUND)
    with pytest.raises(RuntimeError, match="Bool"):
        _C.splatter_blend(colors, coords, mask.long(), 0.5, BACKGROUND)
    with pytest.raises(RuntimeError, match=r"\(N, H, W, K"):
        _C.splatter_blend(colors, coords[..., :2], mask, 0.5, BACKGROUND)
    with pytest.raises(RuntimeError, match=r"\(N, H, W, K"):
        _C.splatter_blend(colors[..., :1, :], coords, mask, 0.5, BACKGROUND)
    with pytest.raises(RuntimeError, match="background_mask must have dimensions"):
        _C.splatter_blend(colors, coords, mask[0], 0.5, BACKGROUND)
    with pytest.raises(RuntimeError, match="background_mask must be a CUDA tensor"):
        _C.splatter_blend(colors, coords, mask.cpu(), 0.5, BACKGROUND)
    with pytest.raises(RuntimeError, match="grad_out"):
        _C.splatter_blend_backward(grad[..., :3], colors, coords, mask, 0.5, BACKGROUND)
    with pytest.raises(RuntimeError, match="Only positive"):
        _C.splatter_blend(colors, coords, mask, 0.0, BACKGROUND)
    c151, x151, m151, _ = splatter_scene(1, 2, 2, 151, device=DEV)
    with pytest.raises(RuntimeError, match="Must have faces_per_pixel <= 150"):
        _C.splatter_blend(c151, x151, m151, 0.5, BACKGROUND)


@pytest.mark.gpu
def test_splatter_no_host_sync_and_deterministic(built_lib):
    from pytorch3d_b200.blending import BlendParams
    from pytorch3d_b200.splatter_blend import splatter_blend
    colors, coords, mask, grad = splatter_scene(2, 33, 17, 8, device=DEV)
    bg = torch.tensor(BACKGROUND, device=DEV)

    def run():
        outs = []
        for params in (BlendParams(sigma=0.5, background_color=bg), BlendParams(sigma=0.5, background_color=BACKGROUND)):
            c, x = colors.clone().requires_grad_(True), coords.clone().requires_grad_(True)
            out = splatter_blend(c, x, mask, params)
            out.backward(grad)
            outs += [out.detach(), c.grad, x.grad]
        return outs

    run()  # warm-up outside the checked region
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        first = run()
        second = run()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    for a, b in zip(first, second):
        assert torch.equal(a, b)


class _PerspectiveCamera:
    """Test-local pinhole projection onto the (H, W) pixel grid: x along the rows, y along the columns, no flip."""

    def __init__(self, focal):
        self.focal = focal

    def transform_points_screen(self, points, image_size, with_xyflip=True):
        H, W = image_size
        z = points[..., 2:3]
        u = points[..., 1:2] / z * self.focal * (H / 2.0) + H / 2.0
        v = points[..., 0:1] / z * self.focal * (W / 2.0) + W / 2.0
        return torch.cat([u, v, z], dim=-1)


def _torus_splatter_pipeline(blend):
    """Rasterize a torus batch (fused indexed path, no blur), interpolate camera-space positions and vertex colours with
    detached barycentrics, as SplatterPhongShader does, splat, take a loss and return the vertex gradient."""
    from pytorch3d_b200 import synthetic
    from pytorch3d_b200.interp_face_attrs import interpolate_face_attributes
    from pytorch3d_b200.rasterize_meshes import rasterize_meshes
    m = synthetic.torus_batch(2, 24, 24, seed=1)
    verts = m.verts_packed().to(DEV).requires_grad_(True)
    faces = m.faces_packed().to(DEV)
    mesh = types.SimpleNamespace(verts_packed=lambda: verts, faces_packed=lambda: faces,
                                 mesh_to_faces_packed_first_idx=lambda: m.mesh_to_faces_packed_first_idx().to(DEV),
                                 num_faces_per_mesh=lambda: m.num_faces_per_mesh().to(DEV))
    H, W = 48, 80
    p2f, zbuf, bary, dists = rasterize_meshes(mesh, (H, W), blur_radius=0.0, faces_per_pixel=4)
    bary = bary.detach()
    # camera-space positions: the synthetic tori lie in NDC at depths > 0; a pinhole camera of focal 2 looks at them
    cam_verts = torch.cat([verts[:, :2] * verts[:, 2:3] / 2.0, verts[:, 2:3]], dim=-1)
    vcol = torch.rand(verts.shape, generator=torch.Generator().manual_seed(4)).to(DEV)
    pos = interpolate_face_attributes(p2f, bary, cam_verts[faces])
    colors = interpolate_face_attributes(p2f, bary, vcol[faces])
    cam = _PerspectiveCamera(2.0)
    N, K = p2f.shape[0], p2f.shape[3]
    coords = cam.transform_points_screen(pos.view(N, -1, 3), (H, W), with_xyflip=False).reshape(pos.shape)
    img = blend(colors, coords, p2f < 0)
    w = torch.rand(img.shape, generator=torch.Generator().manual_seed(6)).to(DEV)
    (img * w).sum().backward()
    return img.detach(), verts.grad


@pytest.mark.gpu
def test_end_to_end_vertex_gradient_matches_torch_chain(built_lib):
    _tf32_off()
    img, g = _torus_splatter_pipeline(fused_fn(0.5))
    img_ref, g_ref = _torus_splatter_pipeline(chain_fn(0.5))
    np.testing.assert_allclose(img.cpu().numpy(), img_ref.cpu().numpy(), rtol=1e-5, atol=1e-6)
    assert float(g_ref.abs().max()) > 0
    np.testing.assert_allclose(g.cpu().numpy(), g_ref.cpu().numpy(), rtol=0, atol=1e-3 * float(g_ref.abs().max()))


@pytest.mark.gpu
def test_splatter_blender_equals_functional_op(built_lib):
    from pytorch3d_b200.blending import BlendParams
    from pytorch3d_b200.splatter_blend import SplatterBlender, splatter_blend
    colors, coords, mask, grad = splatter_scene(2, 9, 13, 8, device=DEV)
    params = BlendParams(sigma=0.5, background_color=BACKGROUND)
    blender = SplatterBlender((1, 1, 1, 1), DEV)  # any input_shape: nothing depends on it
    assert blender.to(DEV) is blender
    cam = _IdentityCamera()
    got = with_grads(lambda c, x, m: blender(c, x, cam, m, params), colors, coords, mask, grad)
    want = with_grads(lambda c, x, m: splatter_blend(c, x, m, params), colors, coords, mask, grad)
    assert cam.calls == [((2, 9 * 13 * 8, 3), (9, 13), False)]
    for a, b in zip(got, want):
        assert torch.equal(a, b)
