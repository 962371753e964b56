"""Depth shading (DESIGN.md section 19): the fused `soft_depth` / `hard_depth` against the torch chains of the
reference's SoftDepthShader / HardDepthShader (pytorch3d/renderer/mesh/shader.py), and `install_depth_shading()`.

The stored outputs of the reference (tests/golden/reference_golden_depth.npz, tests/golden/make_depth_golden.py: its
own shader.py run on the CPU) pin the torch restatements below to the reference.

Tolerances.  HardDepth copies values, so it is bit-identical.  SoftDepth sums K + 1 coverages in a prefix sum; the
kernels add them in ascending k (K <= 8) or in warp scans (K > 8), torch's cumsum in its own order.  Each prefix sum
c_k <= 1 then differs by a few ulps of 1, so each weight w_k = min(c_k, 1) - min(c_{k-1}, 1) does, and the output
sum_k w_k depth_k may differ by

    FWD_ULPS * (K + 1) * 2^-24 * max_k |depth_k|

per pixel.  At K = 1 the sums have two terms and the forward is bit-identical to the chain on CUDA.  Gradients
agree to 1e-5 of their largest magnitude on the pixels where the kernel's and the chain's masks c_k <= 1 agree; where
reordering moves a c_k across 1, the clamp passes the gradient in one and not in the other, so those pixels are
counted, reported and left out.  The kernels' prefix sums are restated exactly by `fused_cumsum`.
"""
import sys
import types

import numpy as np
import pytest
import torch

from helpers import assert_equals_reference, reference

FWD_ULPS = 8

# ------------------------------------------------------------------------------------------------ scenes
# (N, H, W, K, sigma, zfar): zfar "number" (the camera's zfar a Python number), "tensor" (a 1-element tensor) or
# "kwarg" (the forward's zfar= overriding the camera's (1,) tensor)
DEPTH_CASES = [(2, 9, 13, 1, 1e-4, "number"), (2, 9, 13, 1, 1.0, "tensor"), (2, 9, 13, 2, 1e-2, "tensor"),
               (2, 9, 13, 3, 1.0, "kwarg"), (2, 9, 13, 8, 1e-4, "tensor"), (2, 9, 13, 8, 1.0, "number"),
               (2, 9, 13, 9, 1e-2, "kwarg"), (2, 7, 11, 32, 1.0, "tensor"), (2, 7, 11, 33, 1e-4, "number"),
               (2, 5, 7, 150, 1e-2, "kwarg")]
ZFAR = {"number": 37.5, "tensor": 41.25, "kwarg": 55.0}


def depth_case(args):
    return "-".join(str(a) for a in args)


def depth_scene(N, H, W, K, sigma, seed=0):
    """pix_to_face (empty slots after the valid ones, -1), zbuf (-1 in empty slots, like the rasterizer), dists and the
    upstream gradient (N, H, W, 1).  Pixel kinds: background only (the first three of row 0), ordinary, interior
    (p_0 exactly 1, later slots half at p = 0 exactly), coverage crossing 1 after a few slots, and saturated
    (|dists| / sigma of 20, 100 or 200: p tiny, exactly 0 or exactly 1)."""
    g = torch.Generator().manual_seed(seed + 131 * K + N)
    n_valid = (torch.rand(N, H, W, 1, generator=g) * (K + 1)).long().clamp(min=1, max=K)
    p2f = torch.randint(0, 1000, (N, H, W, K), generator=g)
    p2f[torch.arange(K).view(1, 1, 1, K) >= n_valid] = -1
    p2f[:, 0, :3] = -1
    zbuf = torch.where(p2f >= 0, 1.0 + 9.0 * torch.rand(N, H, W, K, generator=g), torch.full((), -1.0))
    t = torch.randn(N, H, W, K, generator=g) * 2.0  # dists / sigma
    kind = torch.randint(0, 4, (N, H, W), generator=g)
    interior = kind == 1
    t[..., 0] = torch.where(interior, -20.0 - 10.0 * torch.rand(N, H, W, generator=g), t[..., 0])
    zero_after = interior[..., None] & (torch.rand(N, H, W, K, generator=g) < 0.5)
    zero_after[..., 0] = False
    t = torch.where(zero_after, 100.0 + 100.0 * torch.rand(N, H, W, K, generator=g), t)
    t = torch.where((kind == 2)[..., None], -2.0 * torch.rand(N, H, W, K, generator=g), t)
    mag = torch.tensor([20.0, 100.0, 200.0])[torch.randint(0, 3, (N, H, W, K), generator=g)]
    sign = torch.where(torch.rand(N, H, W, K, generator=g) < 0.5, -1.0, 1.0)
    t = torch.where((kind == 3)[..., None], sign * mag, t)
    dists = t * sigma
    grad = torch.randn(N, H, W, 1, generator=g)
    return p2f, zbuf, dists, grad


def scene_zfar(kind, device="cpu"):
    """(the camera's zfar, the forward's kwargs, the zfar the shader resolves)."""
    if kind == "number":
        return ZFAR[kind], {}, ZFAR[kind]
    if kind == "tensor":
        z = torch.tensor([ZFAR[kind]], device=device)
        return z, {}, z
    return torch.tensor([100.0], device=device), {"zfar": ZFAR[kind]}, ZFAR[kind]


def frags(pix_to_face, zbuf, dists):
    return types.SimpleNamespace(pix_to_face=pix_to_face, zbuf=zbuf, dists=dists)


# ------------------------------------------------------------------------------------------------ restatements
def soft_depth_chain(pix_to_face, zbuf, dists, sigma, zfar):
    """The torch chain of the reference's SoftDepthShader.forward, step by step in the same operations."""
    N, H, W, K = pix_to_face.shape
    device = zbuf.device
    mask = pix_to_face >= 0
    prob_map = torch.sigmoid(-dists / sigma) * mask
    depth = torch.cat((zbuf, torch.ones((N, H, W, 1), device=device, dtype=zbuf.dtype) * zfar), dim=3)
    probs = torch.cat((prob_map, torch.ones((N, H, W, 1), device=device, dtype=zbuf.dtype)), dim=3)
    probs = probs.cumsum(dim=3)
    probs = probs.clamp(max=1)
    probs = probs.diff(dim=3, prepend=torch.zeros((N, H, W, 1), device=device, dtype=zbuf.dtype))
    return (probs * depth).sum(dim=3).unsqueeze(3)


def hard_depth_chain(pix_to_face, zbuf, zfar):
    """The torch chain of the reference's HardDepthShader.forward."""
    mask = pix_to_face[..., 0:1] < 0
    out = zbuf[..., 0:1].clone()
    out[mask] = zfar
    return out


def coverages(pix_to_face, dists, sigma):
    """p (..., K + 1): the chain's sigmoid coverages and the background's 1."""
    p = torch.sigmoid(-dists / sigma) * (pix_to_face >= 0)
    return torch.cat((p, torch.ones_like(p[..., :1])), dim=-1)


def fused_cumsum(p):
    """The kernels' prefix sums of p (..., K + 1) in float32: one add per slot in ascending order for K <= 8; for K > 8
    Hillis-Steele scans inside rows of 32 slots (lane l adds lane l - o for o = 1, 2, 4, 8, 16), the running total of
    the rows before added to each row."""
    K1 = p.shape[-1]
    if K1 - 1 <= 8:
        c, out = torch.zeros_like(p[..., 0]), []
        for k in range(K1):
            c = c + p[..., k]
            out.append(c)
        return torch.stack(out, -1)
    NS = (K1 + 31) // 32
    x = torch.nn.functional.pad(p, (0, 32 * NS - K1)).reshape(p.shape[:-1] + (NS, 32))
    for o in (1, 2, 4, 8, 16):
        x = torch.cat([x[..., :o], x[..., o:] + x[..., :-o]], -1)
    before, rows = torch.zeros_like(p[..., 0]), []
    for j in range(NS):
        rows.append(x[..., j, :] + before[..., None])
        before = before + x[..., j, 31]
    return torch.cat(rows, -1)[..., :K1]


def soft_with_grads(fn, p2f, zbuf, dists, grad):
    z, d = zbuf.clone().requires_grad_(True), dists.clone().requires_grad_(True)
    out = fn(p2f, z, d)
    out.backward(grad)
    return [out.detach(), z.grad, d.grad]


def hard_with_grads(fn, p2f, zbuf, grad):
    z = zbuf.clone().requires_grad_(True)
    out = fn(p2f, z)
    out.backward(grad)
    return [out.detach(), z.grad]


def forward_bound(zbuf, zfar, K):
    """The per-pixel bound of the module docstring."""
    zf = float(zfar) if not torch.is_tensor(zfar) else float(zfar.reshape(()))
    depth = torch.maximum(zbuf.abs().amax(-1, keepdim=True), torch.full((), abs(zf), device=zbuf.device))
    return FWD_ULPS * (K + 1) * 2.0 ** -24 * depth


# ------------------------------------------------------------------------------------------------ CPU tests
@pytest.mark.parametrize("args", DEPTH_CASES, ids=depth_case)
def test_soft_chain_equals_reference_cpu(args):
    N, H, W, K, sigma, zk = args
    p2f, zbuf, dists, grad = depth_scene(N, H, W, K, sigma)
    zfar = scene_zfar(zk)[2]
    got = soft_with_grads(lambda p, z, d: soft_depth_chain(p, z, d, sigma, zfar), p2f, zbuf, dists, grad)
    assert_equals_reference(got, "depth_soft/" + depth_case(args), "torch restatement vs SoftDepthShader (CPU)")


@pytest.mark.parametrize("args", DEPTH_CASES, ids=depth_case)
def test_hard_chain_equals_reference_cpu(args):
    N, H, W, K, sigma, zk = args
    p2f, zbuf, dists, grad = depth_scene(N, H, W, K, sigma)
    zfar = scene_zfar(zk)[2]
    got = hard_with_grads(lambda p, z: hard_depth_chain(p, z, zfar), p2f, zbuf, grad)
    assert_equals_reference(got, "depth_hard/" + depth_case(args), "torch restatement vs HardDepthShader (CPU)")


def test_scenes_cover_the_edge_cases():
    """Each recorded scene has background-only pixels, p_0 exactly 1, coverage crossing 1 before the last slot and
    saturated or underflowing sigmoids."""
    for N, H, W, K, sigma, _ in DEPTH_CASES:
        p2f, zbuf, dists, _ = depth_scene(N, H, W, K, sigma)
        p = coverages(p2f, dists, sigma)
        c = p.cumsum(-1)
        assert (p2f < 0).all(-1).any()
        assert (p[..., 0] == 1).any()
        assert (p[..., :K] == 0).logical_and(p2f >= 0).any()
        if K > 1:
            assert ((c[..., 1:K] > 1).any(-1) & (c[..., 0] < 1)).any()


def test_fused_cumsum_restates_a_prefix_sum():
    p = torch.rand(3, 151, dtype=torch.float64)
    for K1 in (2, 9, 10, 33, 34, 64, 65, 151):
        np.testing.assert_allclose(fused_cumsum(p[:, :K1]).numpy(), p[:, :K1].cumsum(-1).numpy(), rtol=1e-14)


def test_errors():
    from pytorch3d_b200 import _C, blending
    p2f, zbuf, dists, grad = depth_scene(1, 3, 4, 2, 1e-4)
    with pytest.raises(RuntimeError, match="CUDA"):
        _C.soft_depth_blend(p2f, zbuf, dists, 1e-4, 100.0)
    with pytest.raises(RuntimeError, match="CUDA"):
        _C.soft_depth_blend_backward(grad, p2f, zbuf, dists, 1e-4, 100.0)
    with pytest.raises(RuntimeError, match="CUDA"):
        _C.hard_depth(p2f, zbuf, 100.0)
    with pytest.raises(RuntimeError, match="CUDA"):
        _C.hard_depth_backward(grad, p2f)
    with pytest.raises(ValueError, match="zfar"):
        blending.soft_depth(frags(p2f, zbuf, dists), 1e-4, torch.ones(1, requires_grad=True))
    with pytest.raises(ValueError, match="zfar"):
        blending.hard_depth(frags(p2f, zbuf, dists), torch.ones(1, requires_grad=True))


# ---- install_depth_shading() on stand-in modules
class _Fake:
    """Stands for a CUDA tensor: the routing reads only these attributes."""

    def __init__(self, shape, dtype, device="cpu"):
        self.shape, self.dtype, self.device, self.is_cuda = torch.Size(shape), dtype, torch.device(device), True

    def dim(self):
        return len(self.shape)


def _fake_shader_module(monkeypatch):
    calls = []

    class ShaderBase:
        def __init__(self, cameras=None, blend_params=None):
            self.cameras = cameras
            self.blend_params = blend_params or types.SimpleNamespace(sigma=1e-4)

        def __call__(self, *args, **kwargs):
            return self.forward(*args, **kwargs)

        def _get_cameras(self, **kwargs):
            cameras = kwargs.get("cameras", self.cameras)
            if cameras is None:
                raise ValueError("Cameras must be specified either at initialization or in the forward pass")
            return cameras

    class HardDepthShader(ShaderBase):
        def forward(self, fragments, meshes, **kwargs):
            calls.append("ref_hard")
            return "ref_hard"

    class SoftDepthShader(ShaderBase):
        def forward(self, fragments, meshes, **kwargs):
            calls.append("ref_soft")
            if fragments.dists is None:
                raise ValueError("SoftDepthShader requires Fragments.dists to be present.")
            return "ref_soft"

    for n in ["pytorch3d", "pytorch3d.renderer", "pytorch3d.renderer.mesh", "pytorch3d.renderer.mesh.shader"]:
        m = types.ModuleType(n)
        m.__path__ = []
        monkeypatch.setitem(sys.modules, n, m)
    shader = sys.modules["pytorch3d.renderer.mesh.shader"]
    shader.ShaderBase, shader.HardDepthShader, shader.SoftDepthShader = ShaderBase, HardDepthShader, SoftDepthShader
    return shader, calls


def test_install_depth_shading_routes_and_uninstalls(monkeypatch, built_lib):
    from pytorch3d_b200 import blending
    from pytorch3d_b200 import install as inst
    shader, calls = _fake_shader_module(monkeypatch)
    originals = {c: getattr(shader, c).__dict__["forward"] for c in ("SoftDepthShader", "HardDepthShader")}
    assert inst.install_depth_shading() == ["pytorch3d.renderer.mesh.shader"]
    routed = []
    monkeypatch.setattr(blending, "soft_depth", lambda f, s, z: routed.append(("soft", s, z)) or "b200_soft")
    monkeypatch.setattr(blending, "hard_depth", lambda f, z: routed.append(("hard", z)) or "b200_hard")

    shape = (2, 3, 4, 5)
    p2f, z32 = _Fake(shape, torch.int64), _Fake(shape, torch.float32)
    fr = frags(p2f, z32, z32)
    cam_t = types.SimpleNamespace(zfar=torch.tensor([7.0]))  # a 1-element tensor "on the Fragments' device"
    soft = shader.SoftDepthShader(cameras=types.SimpleNamespace(zfar=3.0))
    hard = shader.HardDepthShader(cameras=cam_t)
    # fused: numbers, 1-element float32 tensors, kwargs overrides, cameras given at call time, no camera zfar
    assert soft(fr, None) == "b200_soft" and routed[-1] == ("soft", 1e-4, 3.0)
    assert hard(fr, None) == "b200_hard" and torch.equal(routed[-1][1], torch.tensor([7.0]))
    assert hard(fr, None, zfar=9) == "b200_hard" and routed[-1] == ("hard", 9)
    assert soft(fr, None, cameras=types.SimpleNamespace()) == "b200_soft" and routed[-1][2] == 100.0
    assert soft(fr, None, zfar=torch.tensor(5.0)) == "b200_soft"
    assert len(routed) == 5 and calls == []
    # everything else goes to the originals
    cpu_p2f = _Fake(shape, torch.int64)
    cpu_p2f.is_cuda = False
    fallbacks = [
        (soft, frags(p2f, z32, None), {}),                                       # no dists: the original raises
        (soft, frags(cpu_p2f, z32, z32), {}),                                    # CPU pix_to_face
        (soft, frags(p2f, _Fake(shape, torch.float64), z32), {}),                # float64 zbuf
        (soft, frags(p2f, z32, _Fake(shape, torch.float16)), {}),                # float16 dists
        (hard, frags(_Fake(shape, torch.int32), z32, z32), {}),                  # int32 pix_to_face
        (hard, frags(p2f, _Fake((2, 3, 4, 4), torch.float32), z32), {}),         # shapes differ
        (hard, frags(_Fake((2, 3, 4, 0), torch.int64), _Fake((2, 3, 4, 0), torch.float32), None), {}),  # K = 0
        (hard, frags(_Fake((1, 2, 2, 151), torch.int64), _Fake((1, 2, 2, 151), torch.float32), None), {}),
        (hard, frags(_Fake((6, 5, 4), torch.int64), _Fake((6, 5, 4), torch.float32), None), {}),  # 3-D
        (hard, frags(p2f, _Fake(shape, torch.float32, "meta"), None), {}),       # zbuf on another device
        (hard, fr, {"zfar": torch.tensor([1.0, 2.0])}),                          # per-image zfar: the original raises
        (hard, fr, {"zfar": torch.tensor([1.0], dtype=torch.float64)}),
        (hard, fr, {"zfar": torch.tensor([1.0], requires_grad=True)}),
        (hard, fr, {"zfar": torch.tensor([[1.0]])}),
        (hard, fr, {"zfar": torch.tensor([1.0], device="meta")}),
        (hard, fr, {"zfar": "far"}),
    ]
    for i, (sh, f, kw) in enumerate(fallbacks):
        n = len(calls)
        if f.dists is None and sh is soft:
            with pytest.raises(ValueError, match="dists"):
                sh(f, None, **kw)
        else:
            assert sh(f, None, **kw) in ("ref_soft", "ref_hard"), "fallback %d was fused" % i
        assert len(calls) == n + 1, "fallback %d" % i
    soft_tensor_sigma = shader.SoftDepthShader(cameras=cam_t, blend_params=types.SimpleNamespace(sigma=torch.ones(())))
    assert soft_tensor_sigma(fr, None) == "ref_soft"
    # no cameras: the reference's error, raised on the fused path as well
    with pytest.raises(ValueError, match="Cameras must be specified"):
        shader.HardDepthShader()(fr, None)
    assert len(routed) == 5
    inst.uninstall()
    for c, f in originals.items():
        assert getattr(shader, c).__dict__["forward"] is f


# ------------------------------------------------------------------------------------------------ GPU tests
DEV = "cuda:0"


def _on(device, *ts):
    return [t.to(device) for t in ts]


def _zfar_on(zfar, device):
    return zfar.to(device) if torch.is_tensor(zfar) else zfar


def _masks_agree(p2f, dists, sigma, chain_c):
    """Pixels where the kernels' masks c_k <= 1 (restated on the CUDA coverages) equal those of `chain_c`."""
    fused = fused_cumsum(coverages(p2f, dists, sigma)) <= 1
    return (fused == (chain_c.to(fused.device) <= 1)).all(-1)


def _assert_grads_close(got, want, agree, what):
    for name, a, b in (("zbuf", got[1], want[1]), ("dists", got[2], want[2])):
        b = b.to(a.device)
        tol = 1e-5 * float(b.abs().max())
        err = (a - b).abs()[agree]
        assert float(err.max()) <= tol, "%s grad_%s: max error %g > %g" % (what, name, float(err.max()), tol)


def _check_soft(p2f, zbuf, dists, grad, sigma, zfar, what):
    """Fused vs the CUDA chain and a float64 restatement: the forward within the bound, gradients to 1e-5 of their
    largest magnitude where the masks agree.  Returns the fused outputs and the agreement mask."""
    from pytorch3d_b200 import blending
    K = p2f.shape[-1]
    got = soft_with_grads(lambda p, z, d: blending.soft_depth(frags(p, z, d), sigma, zfar), p2f, zbuf, dists, grad)
    want = soft_with_grads(lambda p, z, d: soft_depth_chain(p, z, d, sigma, zfar), p2f, zbuf, dists, grad)
    zf64 = zfar.double() if torch.is_tensor(zfar) else zfar
    f64 = soft_depth_chain(p2f, zbuf.double(), dists.double(), sigma, zf64)
    bound = forward_bound(zbuf, zfar, K)
    for ref, name in ((want[0], "CUDA chain"), (f64, "float64")):
        excess = ((got[0].double() - ref).abs() - bound).max()
        assert float(excess) <= 0, "%s: forward beyond the bound against the %s by %g" % (what, name, float(excess))
    agree = _masks_agree(p2f, dists, sigma, coverages(p2f, dists, sigma).cumsum(-1))
    print("%s: masks c_k <= 1 differ from the CUDA chain's on %d of %d pixels" % (
        what, int((~agree).sum()), agree.numel()))
    assert float(agree.float().mean()) > 0.95
    _assert_grads_close(got, want, agree, what + " vs the CUDA chain")
    return got, agree


@pytest.mark.gpu
@pytest.mark.parametrize("args", DEPTH_CASES, ids=depth_case)
def test_soft_depth_matches_chain_and_records(built_lib, args):
    N, H, W, K, sigma, zk = args
    p2f, zbuf, dists, grad = depth_scene(N, H, W, K, sigma)
    zfar = scene_zfar(zk)[2]
    got, _ = _check_soft(*_on(DEV, p2f, zbuf, dists, grad), sigma, _zfar_on(zfar, DEV), depth_case(args))
    # the records: the reference's chain on the CPU, whose masks come from the CPU chain's prefix sums
    rec = reference("depth_soft/" + depth_case(args))
    bound = forward_bound(zbuf, zfar, K).numpy()
    out = got[0].cpu().numpy()
    assert (np.abs(rec[0].rows_of(out).astype(np.float64) - rec[0].sample) <= rec[0].rows_of(bound)).all()
    agree = _masks_agree(*_on(DEV, p2f, dists), sigma, coverages(p2f, dists, sigma).cumsum(-1)).cpu().numpy()
    rows = rec[1].rows_of(np.repeat(agree[..., None], K, -1).astype(np.float32)) > 0
    for i, name in ((1, "zbuf"), (2, "dists")):
        r = rec[i]
        err = np.abs(r.rows_of(got[i].cpu().numpy()).astype(np.float64) - r.sample)[rows]
        assert err.max(initial=0) <= 1e-5 * r.absmax, "grad_%s vs the records: %g" % (name, err.max())


@pytest.mark.gpu
@pytest.mark.parametrize("args", DEPTH_CASES, ids=depth_case)
def test_hard_depth_bit_identical_to_chain_and_records(built_lib, args):
    from pytorch3d_b200 import blending
    N, H, W, K, sigma, zk = args
    p2f, zbuf, dists, grad = _on(DEV, *depth_scene(N, H, W, K, sigma))
    zfar = _zfar_on(scene_zfar(zk)[2], DEV)
    got = hard_with_grads(lambda p, z: blending.hard_depth(frags(p, z, None), zfar), p2f, zbuf, grad)
    want = hard_with_grads(lambda p, z: hard_depth_chain(p, z, zfar), p2f, zbuf, grad)
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
    assert_equals_reference(got, "depth_hard/" + depth_case(args), "hard_depth vs HardDepthShader")


@pytest.mark.gpu
@pytest.mark.parametrize("sigma", [1e-4, 1e-2, 1.0])
def test_soft_depth_k1_bit_identical_to_chain(built_lib, sigma):
    from pytorch3d_b200 import blending
    p2f, zbuf, dists, _ = _on(DEV, *depth_scene(2, 33, 17, 1, sigma, seed=3))
    for zfar in (37.5, torch.tensor([41.25], device=DEV), torch.tensor(12.0, device=DEV)):
        got = blending.soft_depth(frags(p2f, zbuf, dists), sigma, zfar)
        want = soft_depth_chain(p2f, zbuf, dists, sigma, zfar)
        assert got.shape == want.shape == (2, 33, 17, 1) and got.is_contiguous()
        assert torch.equal(got, want), "%d values differ" % int((got != want).sum())


@pytest.mark.gpu
@pytest.mark.parametrize("K", [1, 2, 4, 7, 8, 9, 12, 30, 31, 32, 63, 64, 95, 96, 127, 128, 149, 150])
def test_soft_depth_every_bucket(built_lib, K):
    """K <= 8 (one thread per pixel) and every row count NS = ceil((K + 1) / 32) of the warp kernels."""
    p2f, zbuf, dists, grad = _on(DEV, *depth_scene(2, 17, 23, K, 1e-2, seed=7))
    _check_soft(p2f, zbuf, dists, grad, 1e-2, 20.0, "K=%d" % K)


@pytest.mark.gpu
@pytest.mark.parametrize("K", [3, 8, 40])
def test_unaligned_and_non_contiguous_inputs(built_lib, K):
    from pytorch3d_b200 import _C
    p2f, zbuf, dists, grad = _on(DEV, *depth_scene(2, 9, 13, K, 1e-2))
    want_s = _C.soft_depth_blend(p2f, zbuf, dists, 1e-2, 20.0)
    want_b = _C.soft_depth_blend_backward(grad, p2f, zbuf, dists, 1e-2, 20.0)
    want_h = _C.hard_depth(p2f, zbuf, 20.0)
    want_hb = _C.hard_depth_backward(grad, p2f)

    def shifted(t):
        flat = torch.empty(t.numel() + 1, dtype=t.dtype, device=t.device)
        out = flat[1:].view(t.shape)
        out.copy_(t)
        return out

    def strided(t):
        wide = torch.zeros(t.shape[:-1] + (2 * t.shape[-1],), dtype=t.dtype, device=t.device)
        wide[..., ::2] = t
        return wide[..., ::2]

    for make in (shifted, strided):
        sp, sz, sd, sg = (make(t) for t in (p2f, zbuf, dists, grad))
        assert make is strided or sz.data_ptr() % 16 != 0
        assert make is shifted or not sz.is_contiguous()
        assert torch.equal(_C.soft_depth_blend(sp, sz, sd, 1e-2, 20.0), want_s)
        for a, b in zip(_C.soft_depth_blend_backward(sg, sp, sz, sd, 1e-2, 20.0), want_b):
            assert torch.equal(a, b)
        assert torch.equal(_C.hard_depth(sp, sz, 20.0), want_h)
        assert torch.equal(_C.hard_depth_backward(sg, sp), want_hb)


@pytest.mark.gpu
def test_no_host_sync_with_a_device_zfar(built_lib):
    from pytorch3d_b200 import blending
    p2f, zbuf, dists, grad = _on(DEV, *depth_scene(2, 33, 17, 12, 1e-2))
    zfar = torch.tensor([41.25], device=DEV)

    def run():
        z, d = zbuf.clone().requires_grad_(True), dists.clone().requires_grad_(True)
        f = frags(p2f, z, d)
        (blending.soft_depth(f, 1e-2, zfar) * grad + blending.hard_depth(f, zfar) * grad).sum().backward()
        return z.grad, d.grad

    run()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        run()
    finally:
        torch.cuda.set_sync_debug_mode("default")


@pytest.mark.gpu
@pytest.mark.parametrize("K", [8, 50])
def test_deterministic(built_lib, K):
    from pytorch3d_b200 import blending
    p2f, zbuf, dists, grad = _on(DEV, *depth_scene(2, 33, 17, K, 1e-2))
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        runs = [soft_with_grads(lambda p, z, d: blending.soft_depth(frags(p, z, d), 1e-2, 30.0), p2f, zbuf, dists,
                                grad) + hard_with_grads(lambda p, z: blending.hard_depth(frags(p, z, None), 30.0), p2f,
                                                        zbuf, grad) for _ in range(2)]
    finally:
        torch.use_deterministic_algorithms(prev)
    for a, b in zip(*runs):
        assert torch.equal(a, b)


@pytest.mark.gpu
def test_errors_on_the_device(built_lib):
    from pytorch3d_b200 import _C
    p2f, zbuf, dists, grad = _on(DEV, *depth_scene(1, 3, 4, 2, 1e-4))
    with pytest.raises(RuntimeError, match="Float"):
        _C.soft_depth_blend(p2f, zbuf.double(), dists, 1e-4, 1.0)
    with pytest.raises(RuntimeError, match="Long"):
        _C.hard_depth(p2f.int(), zbuf, 1.0)
    with pytest.raises(RuntimeError, match=r"\(N, H, W, K\)"):
        _C.soft_depth_blend(p2f, zbuf, dists[..., :1], 1e-4, 1.0)
    with pytest.raises(RuntimeError, match="faces_per_pixel"):
        _C.hard_depth(p2f[..., :0], zbuf[..., :0], 1.0)
    big = torch.zeros(1, 1, 1, 151, dtype=torch.int64, device=DEV)
    with pytest.raises(RuntimeError, match="faces_per_pixel"):
        _C.soft_depth_blend(big, big.float(), big.float(), 1e-4, 1.0)
    for bad in (torch.ones(2, device=DEV), torch.ones(1, device=DEV, dtype=torch.float64), torch.ones(1)):
        with pytest.raises(RuntimeError, match="zfar"):
            _C.soft_depth_blend(p2f, zbuf, dists, 1e-4, bad)
    with pytest.raises(RuntimeError, match="grad_out"):
        _C.soft_depth_blend_backward(grad[..., 0], p2f, zbuf, dists, 1e-4, 1.0)
    with pytest.raises(RuntimeError, match="grad_out"):
        _C.hard_depth_backward(grad.double(), p2f)


@pytest.mark.gpu
def test_forward_past_2_31_slots(built_lib):
    """N = 1, 16384 x 16384, K = 9: 2.4e9 slots (39 GB of inputs), so every slot offset needs 64 bits.  Checked at
    sampled pixels against the CUDA chain."""
    from pytorch3d_b200 import _C
    N, S, K, sigma = 1, 16384, 9, 1e-2
    assert N * S * S * K > 2 ** 31
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    g = torch.Generator(device=DEV).manual_seed(11)
    p2f = torch.empty((N, S, S, K), dtype=torch.int64, device=DEV).random_(-300, 1000, generator=g)
    zbuf = torch.empty((N, S, S, K), device=DEV).uniform_(1.0, 10.0, generator=g)
    dists = torch.empty((N, S, S, K), device=DEV).normal_(0.0, 2 * sigma, generator=g)
    out = _C.soft_depth_blend(p2f, zbuf, dists, sigma, 20.0)
    hard = _C.hard_depth(p2f, zbuf, 20.0)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated()
    pix = torch.cat([torch.randint(0, S * S, (4096,), generator=torch.Generator().manual_seed(1)),
                     torch.arange(S * S - 64, S * S)]).to(DEV)
    rows = lambda t: t.reshape(S * S, K)[pix].reshape(1, -1, 1, K)  # noqa: E731
    sp, sz, sd = rows(p2f), rows(zbuf), rows(dists)
    want = soft_depth_chain(sp, sz, sd, sigma, 20.0)
    got = out.reshape(-1)[pix].reshape(want.shape)
    assert ((got - want).abs() <= forward_bound(sz, 20.0, K)).all()
    assert torch.equal(hard.reshape(-1)[pix].reshape(want.shape), hard_depth_chain(sp, sz, 20.0))
    del p2f, zbuf, dists, out, hard
    torch.cuda.empty_cache()
    assert peak < 48e9, "peak %.1f GB" % (peak / 1e9)


# ---- end to end: the rasterizer's blur Fragments, soft depth, an L2 loss
class _Affine:
    """x -> x * scale + shift, with the compose / transform_points protocol of Transform3d."""

    def __init__(self, scale, shift):
        self.scale, self.shift = scale, shift

    def compose(self, other):
        return _Affine(self.scale * other.scale, self.shift * other.scale + other.shift)

    def transform_points(self, points, eps=None):
        return points * self.scale + self.shift


class _OrthoCamera:
    """An orthographic camera 3 units in front of the origin, with a 1-element zfar tensor like FoVPerspectiveCameras."""

    def __init__(self, device):
        self.device = device
        self.zfar = torch.tensor([8.0], device=device)
        self.one = torch.ones(3, device=device)

    def __len__(self):
        return 1

    def is_perspective(self):
        return False

    def get_znear(self):
        return None

    def get_world_to_view_transform(self, **kwargs):
        return _Affine(self.one, torch.tensor([0.0, 0.0, 3.0], device=self.device))

    def get_projection_transform(self, **kwargs):
        return _Affine(torch.tensor([0.9, 0.9, 1.0], device=self.device), 0.0 * self.one)

    def get_ndc_camera_transform(self, **kwargs):
        return _Affine(self.one, 0.0 * self.one)


class _TorusBatch:
    """Two rotated copies of one torus, with the padded / packed accessors MeshRasterizer uses."""

    def __init__(self, verts_padded, faces):
        self._vp, self._faces = verts_padded, faces

    def __len__(self):
        return self._vp.shape[0]

    def verts_padded(self):
        return self._vp

    def update_padded(self, new_verts_padded):
        return _TorusBatch(new_verts_padded, self._faces)

    def verts_packed(self):
        return self._vp.reshape(-1, 3)

    def faces_packed(self):
        off = (torch.arange(len(self), device=self._faces.device) * self._vp.shape[1]).view(-1, 1, 1)
        return (self._faces[None] + off).reshape(-1, 3)

    def mesh_to_faces_packed_first_idx(self):
        return torch.arange(len(self), device=self._faces.device) * self._faces.shape[0]

    def num_faces_per_mesh(self):
        return torch.full((len(self),), self._faces.shape[0], dtype=torch.int64, device=self._faces.device)


def _depth_fit_step(K, soft_depth_fn):
    import pytorch3d_b200 as p3b
    from pytorch3d_b200 import synthetic
    m = synthetic.torus_batch(2, 24, 24, seed=1)
    verts = torch.stack([m.verts_packed()[:m.num_verts_per_mesh()[0]], m.verts_packed()[m.num_verts_per_mesh()[0]:]])
    faces = m.faces_packed()[:m.num_faces_per_mesh()[0]]
    vw = verts.to(DEV).requires_grad_(True)
    cameras = _OrthoCamera(DEV)
    rs = p3b.RasterizationSettings(image_size=(48, 64), blur_radius=2e-4, faces_per_pixel=K)
    fr = p3b.MeshRasterizer(cameras=cameras, raster_settings=rs)(_TorusBatch(vw, faces.to(DEV)))
    depth = soft_depth_fn(fr, 1e-4, cameras.zfar)
    target = 2.5 + torch.rand(depth.shape, generator=torch.Generator().manual_seed(4)).to(DEV)
    ((depth - target) ** 2).mean().backward()
    return depth.detach(), vw.grad, fr


@pytest.mark.gpu
@pytest.mark.parametrize("K", [8, 50])
def test_depth_fitting_step_matches_chain(built_lib, K):
    from pytorch3d_b200 import blending
    depth, g, fr = _depth_fit_step(K, blending.soft_depth)
    depth_ref, g_ref, _ = _depth_fit_step(
        K, lambda f, s, z: soft_depth_chain(f.pix_to_face, f.zbuf, f.dists, s, z))
    assert (fr.pix_to_face[..., 0] >= 0).float().mean() > 0.1 and (fr.pix_to_face[..., 1] >= 0).any()
    assert (depth - depth_ref).abs().max() <= float(forward_bound(fr.zbuf, 8.0, K).max())
    assert float(g_ref.abs().max()) > 0
    np.testing.assert_allclose(g.cpu().numpy(), g_ref.cpu().numpy(), rtol=0, atol=1e-4 * float(g_ref.abs().max()))


@pytest.mark.gpu
def test_install_routes_cuda_fragments(monkeypatch, built_lib):
    """install_depth_shading() on stand-in shader classes that run the torch chains: CUDA Fragments and a camera's
    (1,) zfar go to the fused ops, a per-image (2,) zfar to the original (which raises)."""
    from pytorch3d_b200 import install as inst
    shader, _ = _fake_shader_module(monkeypatch)
    shader.SoftDepthShader.forward = lambda self, f, m, **kw: soft_depth_chain(
        f.pix_to_face, f.zbuf, f.dists, self.blend_params.sigma, kw.get("zfar", self.cameras.zfar))
    shader.HardDepthShader.forward = lambda self, f, m, **kw: hard_depth_chain(
        f.pix_to_face, f.zbuf, kw.get("zfar", self.cameras.zfar))
    inst.install_depth_shading()
    try:
        p2f, zbuf, dists, _ = _on(DEV, *depth_scene(2, 9, 13, 1, 1e-2))
        cam = types.SimpleNamespace(zfar=torch.tensor([30.0], device=DEV))
        fr = frags(p2f, zbuf, dists)
        params = types.SimpleNamespace(sigma=1e-2)
        soft = shader.SoftDepthShader(cameras=cam, blend_params=params)
        hard = shader.HardDepthShader(cameras=cam)
        assert torch.equal(soft(fr, None), soft_depth_chain(p2f, zbuf, dists, 1e-2, cam.zfar))
        assert torch.equal(hard(fr, None), hard_depth_chain(p2f, zbuf, cam.zfar))
        with pytest.raises(RuntimeError):
            soft(fr, None, zfar=torch.tensor([30.0, 40.0], device=DEV))
        with pytest.raises(RuntimeError):
            hard(fr, None, zfar=torch.tensor([30.0, 40.0], device=DEV))
    finally:
        inst.uninstall()
