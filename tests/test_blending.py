"""Mesh blending (SURVEY.md 8f-5): `sigmoid_alpha_blend` bit-identical to the reference's CUDA kernels, the fused
`softmax_rgb_blend` against the torch chain of the reference's pytorch3d/renderer/blending.py, `hard_rgb_blend`, and
`install_blending()`.

The stored outputs of the reference (tests/golden/reference_golden_blend*.npz, tests/golden/make_blend_golden.py) pin
the CPU restatements below to the reference: its C++ CPU sigmoid op and its torch blending functions run on the CPU,
and its CUDA sigmoid kernels on an H100."""
import sys
import types

import numpy as np
import pytest
import torch

from helpers import assert_equals_reference, reference

# ------------------------------------------------------------------------------------------------ scenes
# (N, H, W, K, sigma, kind): kind "tail" = empty slots after the valid ones (the rasterizer's layout), "interleaved" =
# empty slots anywhere, "saturated" = dists << 0 (probabilities of exactly 1) mixed with dists >> 0.
SIGMOID_CASES = [(2, 17, 33, 1, 1e-4, "tail"), (2, 17, 33, 2, 1e-2, "interleaved"), (1, 9, 13, 8, 1e-4, "tail"),
                 (2, 17, 33, 8, 1e-2, "interleaved"), (1, 17, 33, 16, 1e-4, "interleaved"),
                 (1, 5, 7, 100, 1e-2, "tail"), (1, 17, 33, 8, 1e-4, "saturated")]
# the rasterizer's own blur Fragments: torus batch, 48 x 80 image, blur 1e-4, K = 8
TORUS_SIGMOID = ("torus", 1e-4)


def sigmoid_case(args):
    return "blend_sigmoid/" + "-".join(str(a) for a in args)


def _pix_to_face(g, N, H, W, K, kind, frac_empty=0.3):
    p2f = torch.randint(0, 1000, (N, H, W, K), generator=g)
    if kind == "interleaved":
        p2f[torch.rand(N, H, W, K, generator=g) < 0.35] = -1
    else:
        n_valid = (torch.rand(N, H, W, 1, generator=g) * (K + 1) * (1 + frac_empty)).long().clamp(max=K)
        p2f[torch.arange(K).view(1, 1, 1, K) >= n_valid] = -1
    return p2f


def sigmoid_scene(N, H, W, K, sigma, kind, seed=0):
    g = torch.Generator().manual_seed(seed + K)
    p2f = _pix_to_face(g, N, H, W, K, kind)
    dists = torch.randn(N, H, W, K, generator=g) * (8 * sigma)
    if kind == "saturated":
        dists = torch.where(torch.rand(N, H, W, K, generator=g) < 0.5, -0.5 - dists.abs(), 0.5 + dists.abs())
    grad_alphas = torch.randn(N, H, W, generator=g)
    return dists, p2f, grad_alphas


def torus_fragments(dev):
    """Blur Fragments of the rasterizer (fused indexed path): 2 tori, 48 x 80, blur 1e-4, K = 8."""
    from pytorch3d_b200 import _C, synthetic
    m = synthetic.torus_batch(2, 24, 24, seed=0)
    return _C.rasterize_meshes_indexed(m.verts_packed().to(dev), m.faces_packed().to(dev),
                                       m.mesh_to_faces_packed_first_idx().to(dev), m.num_faces_per_mesh().to(dev),
                                       (48, 80), 1e-4, 8, False, False, False)[:4]


# (N, H, W, K, sigma, gamma, z): z "scalar" (znear = 1, zfar = 100 as numbers) or "tensor" ((N,) tensors)
SOFTMAX_CASES = [(2, 9, 13, 1, 1e-4, 1e-4, "scalar"), (2, 9, 13, 4, 1e-4, 1e-4, "scalar"),
                 (2, 9, 13, 4, 1e-3, 1e-2, "tensor"), (1, 7, 11, 8, 1e-3, 0.5, "scalar"),
                 (2, 5, 7, 12, 1e-2, 0.5, "tensor")]


def softmax_case(args):
    return "blend_softmax/" + "-".join(str(a) for a in args)


def softmax_scene(N, H, W, K, sigma, z, seed=0, device="cpu"):
    """colors, pix_to_face, zbuf (-1 in empty slots, like the rasterizer), dists, znear, zfar, upstream gradient."""
    g = torch.Generator().manual_seed(seed + 31 * K + N)
    p2f = _pix_to_face(g, N, H, W, K, "tail")
    p2f[:, 0, :2] = -1  # pixels without any face
    colors = torch.rand(N, H, W, K, 3, generator=g)
    zbuf = torch.where(p2f >= 0, 1.0 + 9.0 * torch.rand(N, H, W, K, generator=g), torch.full((), -1.0))
    dists = torch.randn(N, H, W, K, generator=g) * (4 * sigma)
    if z == "tensor":
        znear, zfar = 0.5 + torch.rand(N, generator=g), 20.0 + 80.0 * torch.rand(N, generator=g)
    else:
        znear, zfar = 1.0, 100.0
    grad = torch.randn(N, H, W, 4, generator=g)
    out = [colors, p2f, zbuf, dists, znear, zfar, grad]
    return [t.to(device) if torch.is_tensor(t) else t for t in out]


def reference_8x8_scene(device="cpu", seed=0):
    """The scene of the reference's test_softmax_rgb_blend (tests/test_blending.py): 1 x 8 x 8, K = 2, a block of
    random faces in the middle, random depths, distances of random sign, sigma = 1e-3."""
    g = torch.Generator().manual_seed(seed)
    N, S, K = 1, 8, 2
    p2f = torch.full((N, S, S, K), -1, dtype=torch.int64)
    p2f[:, 2:6, 2:6, :] = torch.randint(0, 100, (N, 4, 4, K), generator=g)
    flip = torch.rand((N, S, S, K), generator=g)
    flip[flip > 0.5] *= -1.0
    zbuf = torch.randn((N, S, S, K), generator=g)
    dists = torch.randn((N, S, S, K), generator=g) * flip
    colors = torch.randn((N, S, S, K, 3), generator=g)
    grad = torch.randn((N, S, S, 4), generator=g)
    return [t.to(device) for t in (colors, p2f, zbuf, dists, grad)]


# ------------------------------------------------------------------------------------------------ restatements
def softmax_chain(colors, pix_to_face, zbuf, dists, sigma, gamma, background, znear=1.0, zfar=100.0):
    """The torch chain of the reference's softmax_rgb_blend, step by step in the same operations."""
    N, H, W, K = pix_to_face.shape
    out = torch.ones((N, H, W, 4), dtype=colors.dtype, device=colors.device)
    bg = background.to(pix_to_face.device) if torch.is_tensor(background) else \
        torch.tensor(background, dtype=torch.float32, device=pix_to_face.device)
    eps = 1e-10
    valid = pix_to_face >= 0
    prob = torch.sigmoid(-dists / sigma) * valid
    transmittance = torch.prod(1.0 - prob, dim=-1)
    if torch.is_tensor(zfar):
        zfar = zfar[:, None, None, None]
    if torch.is_tensor(znear):
        znear = znear[:, None, None, None]
    z_inv = (zfar - zbuf) / (zfar - znear) * valid
    z_max = torch.max(z_inv, dim=-1).values[..., None].clamp(min=eps)
    w = prob * torch.exp((z_inv - z_max) / gamma)
    delta = torch.exp((eps - z_max) / gamma).clamp(min=eps)
    denom = w.sum(dim=-1)[..., None] + delta
    rgb = (w[..., None] * colors).sum(dim=-2)
    out[..., :3] = (rgb + delta * bg) / denom
    out[..., 3] = 1.0 - transmittance
    return out


def hard_chain(colors, pix_to_face, background):
    """The reference's hard_rgb_blend: masked_scatter of the background colour (counts background pixels on the host)."""
    bg = background if torch.is_tensor(background) else \
        torch.tensor(background, dtype=torch.float32, device=pix_to_face.device)
    is_bg = pix_to_face[..., 0] < 0
    rgb = colors[..., 0, :].masked_scatter(is_bg[..., None], bg[None, :].expand(int(is_bg.sum()), -1))
    return torch.cat([rgb, (~is_bg).type_as(rgb)[..., None]], dim=-1)


def sigmoid_numpy(dists, pix_to_face, sigma, grad_alphas):
    """float64 restatement of the sigmoid op: alpha = 1 - prod (1 - p), d alpha / d dist_k = -(1/sigma) p_k (1 - alpha),
    where the backward takes 1 - alpha from the saved float32 output, as the op does."""
    d = dists.numpy().astype(np.float64)
    valid = pix_to_face.numpy().astype(np.int32) >= 0  # the reference reads the index into an int
    p = np.where(valid, 1.0 / (1.0 + np.exp(np.clip(d / sigma, -700, 700))), 0.0)
    trans = np.prod(1.0 - p, axis=-1)
    alphas = 1.0 - trans
    trans_saved = 1.0 - alphas.astype(np.float32).astype(np.float64)
    grad = grad_alphas.numpy().astype(np.float64)[..., None] * (-1.0 / sigma) * p * trans_saved[..., None]
    return alphas, np.where(valid, grad, 0.0)


def frags(pix_to_face, zbuf, dists):
    return types.SimpleNamespace(pix_to_face=pix_to_face, zbuf=zbuf, dists=dists)


def softmax_with_grads(fn, colors, p2f, zbuf, dists, grad):
    c, z, d = (t.clone().requires_grad_(True) for t in (colors, zbuf, dists))
    out = fn(c, p2f, z, d)
    out.backward(grad)
    return [out.detach(), c.grad, d.grad, z.grad]


# ------------------------------------------------------------------------------------------------ CPU tests
@pytest.mark.parametrize("args", SIGMOID_CASES)
def test_sigmoid_numpy_restatement_matches_reference_cpu(args):
    dists, p2f, ga = sigmoid_scene(*args)
    alphas, grad = sigmoid_numpy(dists, p2f, args[4], ga)
    ref_a, ref_g = reference(sigmoid_case(args) + "/cpu")
    np.testing.assert_allclose(ref_a.rows_of(alphas), ref_a.sample, rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(ref_g.rows_of(grad), ref_g.sample, rtol=1e-4, atol=1e-6 * max(ref_g.absmax, 1e-30))


def _softmax_fn_chain(args):
    sigma, gamma = args[4], args[5]

    def fn(c, p2f, z, d, znear, zfar, bg=(0.2, 0.4, 0.6)):
        return softmax_chain(c, p2f, z, d, sigma, gamma, bg, znear, zfar)
    return fn


@pytest.mark.parametrize("args", SOFTMAX_CASES)
def test_softmax_chain_equals_reference_cpu(args):
    colors, p2f, zbuf, dists, znear, zfar, grad = softmax_scene(*args[:5], args[6])
    fn = _softmax_fn_chain(args)
    got = softmax_with_grads(lambda c, p, z, d: fn(c, p, z, d, znear, zfar), colors, p2f, zbuf, dists, grad)
    assert_equals_reference(got, softmax_case(args), "torch restatement vs the reference's softmax_rgb_blend (CPU)")


def test_softmax_chain_equals_reference_cpu_8x8():
    colors, p2f, zbuf, dists, grad = reference_8x8_scene()
    got = softmax_with_grads(lambda c, p, z, d: softmax_chain(c, p, z, d, 1e-3, 1e-4, (1.0, 1.0, 1.0)), colors, p2f,
                             zbuf, dists, grad)
    assert_equals_reference(got, "blend_softmax/reference_8x8", "torch restatement vs the reference (CPU)")


def test_hard_rgb_blend_equals_reference_cpu():
    """pytorch3d_b200.blending.hard_rgb_blend is plain torch: on the CPU it equals the reference's, values and gradient."""
    from pytorch3d_b200 import blending
    colors, p2f, zbuf, dists, _, _, grad = softmax_scene(2, 9, 13, 4, 1e-4, "scalar")
    c = colors.clone().requires_grad_(True)
    out = blending.hard_rgb_blend(c, frags(p2f, zbuf, dists), blending.BlendParams(background_color=(0.2, 0.4, 0.6)))
    out.backward(grad)
    assert_equals_reference([out.detach(), c.grad], "blend_hard/2-9-13-4", "hard_rgb_blend vs the reference (CPU)")


def test_cpu_tensors_and_wrong_dtypes_raise():
    from pytorch3d_b200 import _C, blending
    d, p2f, ga = sigmoid_scene(1, 3, 4, 2, 1e-4, "tail")
    with pytest.raises(RuntimeError, match="CUDA"):
        _C.sigmoid_alpha_blend(d, p2f, 1e-4)
    with pytest.raises(RuntimeError, match="CUDA"):
        _C.sigmoid_alpha_blend_backward(ga, ga, d, p2f, 1e-4)
    with pytest.raises(RuntimeError):
        _C.sigmoid_alpha_blend(d.double(), p2f, 1e-4)
    colors, p2f, zbuf, dists, _, _, _ = softmax_scene(1, 3, 4, 2, 1e-4, "scalar")
    with pytest.raises(RuntimeError, match="CUDA"):
        _C.softmax_rgb_blend(colors, p2f, zbuf, dists, 1e-4, 1e-4, (1.0, 1.0, 1.0))
    with pytest.raises(RuntimeError):
        _C.softmax_rgb_blend(colors.double(), p2f, zbuf, dists, 1e-4, 1e-4, (1.0, 1.0, 1.0))
    with pytest.raises(RuntimeError):
        blending.softmax_rgb_blend(colors, frags(p2f, zbuf, dists), blending.BlendParams())
    with pytest.raises(RuntimeError):
        blending.sigmoid_alpha_blend(colors, frags(p2f, zbuf, dists), blending.BlendParams())


def test_softmax_rejects_grad_through_constants():
    from pytorch3d_b200 import blending
    colors, p2f, zbuf, dists, _, _, _ = softmax_scene(1, 3, 4, 2, 1e-4, "scalar")
    f = frags(p2f, zbuf, dists)
    with pytest.raises(ValueError, match="background_color"):
        blending.softmax_rgb_blend(colors, f, blending.BlendParams(background_color=torch.ones(3, requires_grad=True)))
    with pytest.raises(ValueError, match="znear"):
        blending.softmax_rgb_blend(colors, f, blending.BlendParams(), znear=torch.ones(1, requires_grad=True))
    with pytest.raises(ValueError, match="zfar"):
        blending.softmax_rgb_blend(colors, f, blending.BlendParams(), zfar=torch.ones(1, requires_grad=True))


def test_blend_params_match_the_reference_defaults():
    from pytorch3d_b200.blending import BlendParams
    assert BlendParams() == (1e-4, 1e-4, (1.0, 1.0, 1.0))
    assert BlendParams._fields == ("sigma", "gamma", "background_color")


def _fake_pytorch3d(monkeypatch):
    calls = []
    orig_C = types.SimpleNamespace(sigmoid_alpha_blend=lambda *a, **k: calls.append("ref_sigmoid") or "ref",
                                   sigmoid_alpha_blend_backward=lambda *a, **k: "ref_bwd", knn_points_idx=lambda: "knn")

    def ref_softmax(colors, fragments, blend_params, znear=1.0, zfar=100):
        calls.append("ref_softmax")
        return "ref_softmax"

    def ref_hard(colors, fragments, blend_params):
        calls.append("ref_hard")
        return "ref_hard"

    for n in ["pytorch3d", "pytorch3d.renderer", "pytorch3d.renderer.blending", "pytorch3d.renderer.mesh",
              "pytorch3d.renderer.mesh.shader"]:
        m = types.ModuleType(n)
        m.__path__ = []
        monkeypatch.setitem(sys.modules, n, m)
    for n in ("pytorch3d.renderer.blending", "pytorch3d.renderer.mesh.shader"):
        sys.modules[n].softmax_rgb_blend = ref_softmax
        sys.modules[n].hard_rgb_blend = ref_hard
    sys.modules["pytorch3d.renderer.blending"]._C = orig_C
    return orig_C, ref_softmax, ref_hard, calls


def test_install_blending_and_uninstall(monkeypatch, built_lib):
    from pytorch3d_b200 import install as inst
    orig_C, ref_softmax, ref_hard, calls = _fake_pytorch3d(monkeypatch)
    patched = inst.install_blending()
    assert patched == ["pytorch3d.renderer.blending", "pytorch3d.renderer.mesh.shader"]
    bl, sh = sys.modules["pytorch3d.renderer.blending"], sys.modules["pytorch3d.renderer.mesh.shader"]
    assert bl._C is not orig_C and bl.softmax_rgb_blend is not ref_softmax and sh.hard_rgb_blend is not ref_hard
    # CPU tensors keep the reference's implementations; unrelated _C ops pass through untouched
    cpu = torch.zeros(1, 2, 2, 1, 3)
    assert bl._C.sigmoid_alpha_blend(torch.zeros(1)) == "ref" and bl._C.knn_points_idx() == "knn"
    assert sh.softmax_rgb_blend(cpu, None, None) == "ref_softmax" and bl.hard_rgb_blend(cpu, None, None) == "ref_hard"
    # CUDA inputs go to pytorch3d_b200 (stand-ins that claim to be on the GPU), unless a constant requires grad
    routed = []
    from pytorch3d_b200 import blending
    monkeypatch.setattr(blending, "softmax_rgb_blend", lambda *a: routed.append("softmax") or "b200_softmax")
    monkeypatch.setattr(blending, "hard_rgb_blend", lambda *a: routed.append("hard") or "b200_hard")
    monkeypatch.setattr(inst._b200_C, "sigmoid_alpha_blend", lambda *a: routed.append("sigmoid") or "b200_sigmoid")
    fake_cuda = types.SimpleNamespace(is_cuda=True, dtype=torch.float32)
    fr32 = types.SimpleNamespace(zbuf=fake_cuda, dists=fake_cuda)
    params = types.SimpleNamespace(background_color=(1.0, 1.0, 1.0))
    assert sh.softmax_rgb_blend(fake_cuda, fr32, params) == "b200_softmax"
    assert bl.hard_rgb_blend(fake_cuda, None, params) == "b200_hard"
    assert bl._C.sigmoid_alpha_blend(fake_cuda) == "b200_sigmoid"
    assert sh.softmax_rgb_blend(fake_cuda, fr32, params, torch.ones(1, requires_grad=True)) == "ref_softmax"
    # other dtypes keep the original torch code
    fake_cuda64 = types.SimpleNamespace(is_cuda=True, dtype=torch.float64)
    assert sh.softmax_rgb_blend(fake_cuda64, fr32, params) == "ref_softmax"
    assert bl.hard_rgb_blend(fake_cuda64, None, params) == "ref_hard"
    assert routed == ["softmax", "hard", "sigmoid"]
    inst.uninstall()
    assert bl._C is orig_C and bl.softmax_rgb_blend is ref_softmax and sh.hard_rgb_blend is ref_hard
    assert sh.softmax_rgb_blend is ref_softmax and bl.hard_rgb_blend is ref_hard


# ------------------------------------------------------------------------------------------------ GPU tests
DEV = "cuda:0"


@pytest.mark.gpu
@pytest.mark.parametrize("args", SIGMOID_CASES + [TORUS_SIGMOID])
def test_sigmoid_alpha_blend_bit_identical_to_reference_cuda(built_lib, args):
    from pytorch3d_b200 import _C
    if args[0] == "torus":
        p2f, _, _, dists = torus_fragments(DEV)
        ga = torch.randn(p2f.shape[:3], generator=torch.Generator().manual_seed(5)).to(DEV)
        sigma = args[1]
    else:
        dists, p2f, ga = (t.to(DEV) for t in sigmoid_scene(*args))
        sigma = args[4]
    alphas = _C.sigmoid_alpha_blend(dists, p2f, sigma)
    grad = _C.sigmoid_alpha_blend_backward(ga, alphas, dists, p2f, sigma)
    assert_equals_reference([alphas, grad], sigmoid_case(args) + "/cuda",
                            "sigmoid_alpha_blend must be bit-identical to the reference CUDA kernels")


@pytest.mark.gpu
@pytest.mark.parametrize("z", ["scalar", "tensor"])
def test_softmax_k1_equals_torch_chain(built_lib, z):
    from pytorch3d_b200 import _C
    colors, p2f, zbuf, dists, znear, zfar, _ = softmax_scene(2, 33, 17, 1, 1e-4, z, device=DEV)
    for gamma in (1e-4, 1e-2, 0.5):
        got = _C.softmax_rgb_blend(colors, p2f, zbuf, dists, 1e-4, gamma, (0.2, 0.4, 0.6), znear, zfar)
        want = softmax_chain(colors, p2f, zbuf, dists, 1e-4, gamma, (0.2, 0.4, 0.6), znear, zfar)
        assert torch.equal(got, want), "gamma %g: %d values differ" % (gamma, int((got != want).sum()))


def _assert_softmax_close(got, want, tied_zbuf_ok=None, what=""):
    np.testing.assert_allclose(got[0].cpu().numpy(), want[0].cpu().numpy(), rtol=1e-5, atol=1e-6, err_msg=what)
    for i, name in ((1, "colors"), (2, "dists"), (3, "zbuf")):
        a, b = got[i], want[i]
        if name == "zbuf" and tied_zbuf_ok is not None:  # tied maxima: compare the pixel's sum over the slots
            a = torch.where(tied_zbuf_ok[..., None], a, a.sum(-1, keepdim=True).expand_as(a))
            b = torch.where(tied_zbuf_ok[..., None], b, b.sum(-1, keepdim=True).expand_as(b))
        atol = 1e-5 * float(b.abs().max()) + 1e-30
        np.testing.assert_allclose(a.cpu().numpy(), b.cpu().numpy(), rtol=1e-4, atol=atol,
                                   err_msg="%s grad_%s" % (what, name))


def _no_tie(zbuf, p2f, znear, zfar):
    """Pixels whose maximum inverse depth is attained by one slot only."""
    if torch.is_tensor(zfar):
        zfar, znear = zfar[:, None, None, None], znear[:, None, None, None]
    zi = (zfar - zbuf) / (zfar - znear) * (p2f >= 0)
    return (zi == zi.max(-1, keepdim=True).values).sum(-1) == 1


@pytest.mark.gpu
@pytest.mark.parametrize("gamma", [1e-4, 1e-2, 0.5])
@pytest.mark.parametrize("z", ["scalar", "tensor"])
@pytest.mark.parametrize("K,sigma", [(2, 1e-4), (8, 1e-3), (13, 1e-2), (40, 1e-3), (150, 1e-3)])
def test_softmax_matches_torch_chain(built_lib, gamma, z, K, sigma):
    from pytorch3d_b200 import blending
    colors, p2f, zbuf, dists, znear, zfar, grad = softmax_scene(2, 33, 17, K, sigma, z, device=DEV)
    bg = torch.tensor([0.2, 0.4, 0.6], device=DEV)
    params = blending.BlendParams(sigma=sigma, gamma=gamma, background_color=bg)
    got = softmax_with_grads(lambda c, p, zz, d: blending.softmax_rgb_blend(c, frags(p, zz, d), params, znear, zfar),
                             colors, p2f, zbuf, dists, grad)
    want = softmax_with_grads(lambda c, p, zz, d: softmax_chain(c, p, zz, d, sigma, gamma, bg, znear, zfar),
                              colors, p2f, zbuf, dists, grad)
    _assert_softmax_close(got, want, _no_tie(zbuf, p2f, znear, zfar), "K=%d gamma=%g z=%s" % (K, gamma, z))
    empty = (p2f < 0).all(-1)
    assert empty.any()
    assert torch.equal(got[0][empty][:, :3], bg.expand(int(empty.sum()), 3)), "empty pixels must be exactly bg"
    assert (got[0][empty][:, 3] == 0).all(), "empty pixels must have alpha 0"


@pytest.mark.gpu
def test_softmax_reference_8x8_scene(built_lib):
    from pytorch3d_b200 import blending
    colors, p2f, zbuf, dists, grad = reference_8x8_scene(DEV)
    params = blending.BlendParams(sigma=1e-3)
    got = softmax_with_grads(lambda c, p, z, d: blending.softmax_rgb_blend(c, frags(p, z, d), params), colors, p2f,
                             zbuf, dists, grad)
    want = softmax_with_grads(lambda c, p, z, d: softmax_chain(c, p, z, d, 1e-3, 1e-4, (1.0, 1.0, 1.0)), colors, p2f,
                              zbuf, dists, grad)
    _assert_softmax_close(got, want, _no_tie(zbuf, p2f, 1.0, 100.0), "reference 8x8 scene")


@pytest.mark.gpu
def test_softmax_on_tied_blur_fragments(built_lib):
    """Structured mesh with blur: slots of one pixel share their depth; the gradient of the maximum goes to one of
    them, so grad_zbuf is compared summed over the pixel's slots where the maximum is tied."""
    from pytorch3d_b200 import blending
    p2f, zbuf, _, dists = torus_fragments(DEV)
    colors = torch.rand(p2f.shape + (3,), generator=torch.Generator().manual_seed(2)).to(DEV)
    grad = torch.randn(p2f.shape[:3] + (4,), generator=torch.Generator().manual_seed(3)).to(DEV)
    for gamma in (1e-4, 1e-2):
        params = blending.BlendParams(sigma=1e-4, gamma=gamma)
        got = softmax_with_grads(lambda c, p, z, d: blending.softmax_rgb_blend(c, frags(p, z, d), params), colors,
                                 p2f, zbuf, dists, grad)
        want = softmax_with_grads(lambda c, p, z, d: softmax_chain(c, p, z, d, 1e-4, gamma, (1.0, 1.0, 1.0)), colors,
                                  p2f, zbuf, dists, grad)
        _assert_softmax_close(got, want, _no_tie(zbuf, p2f, 1.0, 100.0), "torus gamma=%g" % gamma)


@pytest.mark.gpu
def test_hard_rgb_blend_bit_identical_to_chain(built_lib):
    from pytorch3d_b200 import blending
    colors, p2f, zbuf, dists, _, _, grad = softmax_scene(2, 33, 17, 4, 1e-4, "scalar", device=DEV)
    for bg in ((0.2, 0.4, 0.6), torch.tensor([0.3, 0.1, 0.9], device=DEV)):
        c1, c2 = colors.clone().requires_grad_(True), colors.clone().requires_grad_(True)
        got = blending.hard_rgb_blend(c1, frags(p2f, zbuf, dists), blending.BlendParams(background_color=bg))
        want = hard_chain(c2, p2f, bg)
        got.backward(grad)
        want.backward(grad)
        assert torch.equal(got, want) and torch.equal(c1.grad, c2.grad)


@pytest.mark.gpu
@pytest.mark.parametrize("K", [8, 40])
def test_softmax_accepts_unaligned_tensors(built_lib, K):
    """Contiguous tensors whose storage starts at an odd float (views into larger buffers) give the same results."""
    from pytorch3d_b200 import _C
    colors, p2f, zbuf, dists, znear, zfar, grad = softmax_scene(2, 9, 13, K, 1e-3, "scalar", device=DEV)

    def shifted(t):
        flat = torch.empty(t.numel() + 1, dtype=t.dtype, device=t.device)
        out = flat[1:].view(t.shape)
        out.copy_(t)
        return out

    args = (1e-3, 1e-2, (0.2, 0.4, 0.6))
    want_f = _C.softmax_rgb_blend(colors, p2f, zbuf, dists, *args)
    want_b = _C.softmax_rgb_blend_backward(grad, colors, p2f, zbuf, dists, *args)
    sc, sp, sz, sd, sg = (shifted(t) for t in (colors, p2f, zbuf, dists, grad))
    assert sg.data_ptr() % 16 != 0
    assert torch.equal(_C.softmax_rgb_blend(sc, sp, sz, sd, *args), want_f)
    for a, b in zip(_C.softmax_rgb_blend_backward(sg, sc, sp, sz, sd, *args), want_b):
        assert torch.equal(a, b)


@pytest.mark.gpu
def test_errors_on_the_device(built_lib):
    from pytorch3d_b200 import _C
    colors, p2f, zbuf, dists, _, _, _ = softmax_scene(1, 3, 4, 2, 1e-4, "scalar", device=DEV)
    with pytest.raises(RuntimeError, match="Float"):
        _C.softmax_rgb_blend(colors.double(), p2f, zbuf, dists, 1e-4, 1e-4, (1.0, 1.0, 1.0))
    with pytest.raises(RuntimeError, match="Float"):
        _C.sigmoid_alpha_blend(dists.double(), p2f, 1e-4)
    with pytest.raises(RuntimeError, match="Long"):
        _C.sigmoid_alpha_blend(dists, p2f.int(), 1e-4)
    with pytest.raises(RuntimeError, match=r"\(N, H, W, K\)"):
        _C.softmax_rgb_blend(colors, p2f, zbuf[..., :1], dists, 1e-4, 1e-4, (1.0, 1.0, 1.0))
    with pytest.raises(RuntimeError, match=r"\(N, H, W, K\)"):
        _C.sigmoid_alpha_blend(dists[..., :1], p2f, 1e-4)


def _torus_pipeline(blend):
    """Rasterize a torus batch with blur through the fused indexed path, interpolate vertex colours, blend, take a
    loss and return the gradient w.r.t. the vertices."""
    from pytorch3d_b200 import blending, synthetic
    from pytorch3d_b200.interp_face_attrs import interpolate_face_attributes
    from pytorch3d_b200.rasterize_meshes import rasterize_meshes
    m = synthetic.torus_batch(2, 24, 24, seed=1)
    verts = m.verts_packed().to(DEV).requires_grad_(True)
    faces = m.faces_packed().to(DEV)
    mesh = types.SimpleNamespace(verts_packed=lambda: verts, faces_packed=lambda: faces,
                                 mesh_to_faces_packed_first_idx=lambda: m.mesh_to_faces_packed_first_idx().to(DEV),
                                 num_faces_per_mesh=lambda: m.num_faces_per_mesh().to(DEV))
    p2f, zbuf, bary, dists = rasterize_meshes(mesh, (64, 96), blur_radius=1e-4, faces_per_pixel=8)
    vcol = torch.rand(verts.shape, generator=torch.Generator().manual_seed(4)).to(DEV)
    colors = interpolate_face_attributes(p2f, bary, vcol[faces])
    params = blending.BlendParams(sigma=1e-4, gamma=1e-2)
    fr = frags(p2f, zbuf, dists)
    img = blend(colors, fr, params)
    sil = blending.sigmoid_alpha_blend(colors, fr, params)
    w = torch.rand(img.shape, generator=torch.Generator().manual_seed(6)).to(DEV)
    loss = (img * w).sum() + (sil[..., 3] * w[..., 3]).sum()
    loss.backward()
    return img.detach(), verts.grad


@pytest.mark.gpu
def test_end_to_end_gradient_matches_torch_chain(built_lib):
    from pytorch3d_b200 import blending
    img, g = _torus_pipeline(blending.softmax_rgb_blend)
    img_ref, g_ref = _torus_pipeline(
        lambda c, f, p: softmax_chain(c, f.pix_to_face, f.zbuf, f.dists, p.sigma, p.gamma, p.background_color))
    np.testing.assert_allclose(img.cpu().numpy(), img_ref.cpu().numpy(), rtol=1e-5, atol=1e-6)
    assert float(g_ref.abs().max()) > 0
    np.testing.assert_allclose(g.cpu().numpy(), g_ref.cpu().numpy(), rtol=0,
                               atol=1e-3 * float(g_ref.abs().max()))


@pytest.mark.gpu
def test_no_host_sync_and_deterministic(built_lib):
    from pytorch3d_b200 import blending
    colors, p2f, zbuf, dists, znear, zfar, grad = softmax_scene(2, 33, 17, 8, 1e-3, "tensor", device=DEV)
    bg = torch.tensor([0.2, 0.4, 0.6], device=DEV)
    params = blending.BlendParams(sigma=1e-3, gamma=1e-2, background_color=bg)
    f = frags(p2f, zbuf, dists)

    def run():
        c, z, d = (t.clone().requires_grad_(True) for t in (colors, zbuf, dists))
        fr = frags(p2f, z, d)
        outs = [blending.softmax_rgb_blend(c, fr, params, znear, zfar), blending.sigmoid_alpha_blend(c, fr, params),
                blending.hard_rgb_blend(c, fr, params),
                blending.hard_rgb_blend(c, fr, blending.BlendParams())]
        sum((o * grad).sum() for o in outs).backward()
        return [o.detach() for o in outs] + [c.grad, z.grad, d.grad]

    run()  # warm-up outside the checked region
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        first = run()
        second = run()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert f is not None
    for a, b in zip(first, second):
        assert torch.equal(a, b)
