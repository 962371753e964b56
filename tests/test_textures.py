"""UV texture sampling (DESIGN.md section 13): the fused `sample_textures_uv` / `sample_textures` against a torch
restatement of the reference's TexturesUV.sample_textures (pytorch3d/renderer/mesh/textures.py), and
`install_textures()`.

The stored outputs of the reference (tests/golden/reference_golden_textures.npz, tests/golden/make_texture_golden.py)
pin the restatement below to the reference: its own textures module runs on the CPU."""
import itertools
import sys
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import reference

# ------------------------------------------------------------------------------------------------ scenes
MODES = ("bilinear", "nearest")
PADDINGS = ("zeros", "border", "reflection")
# (map H_in, W_in): non-square, 1 x 1, 1 x W, and sizes whose texel centres and half-texel ties are dyadic
MAP_SIZES = ((9, 17), (8, 5), (1, 1), (1, 12), (16, 9), (5, 8))
CHANNELS = (1, 3, 4)
TEXTURE_CASES = [(mode, pad, align, CHANNELS[i % 3], MAP_SIZES[i % len(MAP_SIZES)])
                 for i, (mode, pad, align) in enumerate(itertools.product(MODES, PADDINGS, (True, False)))]
TEXTURE_CASES += [("nearest", "zeros", True, 3, (1, 1)), ("bilinear", "reflection", False, 4, (1, 12)),
                  ("bilinear", "border", True, 3, (1, 1)), ("nearest", "reflection", True, 1, (1, 12))]
SCENE = (2, 5, 7, 3)  # N, H, W, K: non-square
FIELDS = ("texels", "grad_maps", "grad_verts_uvs", "grad_bary")


def texture_case(args):
    mode, pad, align, C, (hi, wi) = args
    return "textures/%s-%s-%s-C%d-%dx%d" % (mode, pad, "align" if align else "noalign", C, hi, wi)


def special_uvs(H_in, W_in, align):
    """UVs that land exactly on texel centres and on the half-texel ties of "nearest" rounding (exact where the
    denominators are powers of two)."""
    def axis(n, centre):
        if align:
            d = max(n - 1, 1)
            return [(k + (0.0 if centre else 0.5)) / d for k in range(n)]
        return [(k + (0.5 if centre else 1.0)) / n for k in range(n)]
    us = axis(W_in, True) + axis(W_in, False)
    vs = [1.0 - t for t in axis(H_in, True) + axis(H_in, False)]
    n = max(len(us), len(vs))
    return [(us[i % len(us)], vs[(3 * i) % len(vs)]) for i in range(n)]


def texture_scene(N, H, W, K, H_in, W_in, C, align=True, seed=0, device="cpu", frac_background=0.3, Fm=8, Vm=12):
    """A dict: maps (N, H_in, W_in, C), different per image; per-mesh verts_uvs (N, Vm, 2) in [-0.25, 1.25) (outside
    [0, 1] too) with the first vertices on texel centres and nearest-rounding ties; faces_uvs (N, Fm, 3); pix_to_face
    into the packed faces of each image's own mesh with about `frac_background` background slots; barycentrics, with
    some slots exactly on a corner (barycentrics (1, 0, 0)); and an upstream gradient that is nonzero everywhere,
    background slots included."""
    g = torch.Generator().manual_seed(seed + 1000 * K + 31 * H + W + 7 * H_in + W_in + C)
    maps = torch.rand(N, H_in, W_in, C, generator=g)
    verts_uvs = torch.rand(N, Vm, 2, generator=g) * 1.5 - 0.25
    sp = special_uvs(H_in, W_in, align)[:Vm - 2]
    verts_uvs[:, :len(sp)] = torch.tensor(sp, dtype=torch.float32)
    faces_uvs = torch.randint(0, Vm, (N, Fm, 3), generator=g)
    faces_uvs[:, : min(Fm, Vm), 0] = torch.arange(min(Fm, Vm))  # corner 0 of face j is vertex j
    p2f = torch.randint(0, Fm, (N, H, W, K), generator=g) + (torch.arange(N) * Fm).view(N, 1, 1, 1)
    p2f[torch.rand(N, H, W, K, generator=g) < frac_background] = -1
    bary = torch.rand(N, H, W, K, 3, generator=g) + 0.05
    bary = bary / bary.sum(-1, keepdim=True)
    corner = torch.rand(N, H, W, K, generator=g) < 0.25
    bary[corner] = torch.tensor([1.0, 0.0, 0.0])
    s = {"maps": maps, "verts_uvs": verts_uvs, "faces_uvs": faces_uvs, "pix_to_face": p2f, "bary": bary,
         "grad_texels": torch.randn(N, H, W, K, C, generator=g)}
    return {k: v.to(device) for k, v in s.items()}


def case_scene(args, device="cpu"):
    mode, pad, align, C, (hi, wi) = args
    return texture_scene(*SCENE, hi, wi, C, align, device=device)


# ------------------------------------------------------------------------------------------------ restatement
def _interp(pix_to_face, bary, face_attrs):
    """interpolate_face_attributes as the reference runs it: its python path on the CPU, its kernel on CUDA (ours
    equals it bit for bit)."""
    if pix_to_face.is_cuda:
        from pytorch3d_b200.interp_face_attrs import interpolate_face_attributes
        return interpolate_face_attributes(pix_to_face, bary, face_attrs)
    N, H, W, K = pix_to_face.shape
    D = face_attrs.shape[-1]
    mask = pix_to_face < 0
    p2f = pix_to_face.clone()
    p2f[mask] = 0
    idx = p2f.view(N * H * W * K, 1, 1).expand(N * H * W * K, 3, D)
    vals = face_attrs.gather(0, idx).view(N, H, W, K, 3, D)
    out = (bary[..., None] * vals).sum(dim=-2)
    out[mask] = 0
    return out


def packed_face_uvs(verts_uvs, faces_uvs):
    """torch.cat([v[f] for v, f in zip(verts_uvs_list(), faces_uvs_list())]), as the reference forms it."""
    return torch.cat([v[f] for v, f in zip(verts_uvs, faces_uvs)])


def chain_sample(fragments, maps, face_uvs, sampling_mode="bilinear", padding_mode="border", align_corners=True):
    """TexturesUV.sample_textures without maps_ids, in the reference's operations."""
    pixel_uvs = _interp(fragments.pix_to_face, fragments.bary_coords, face_uvs)
    N, H_out, W_out, K = fragments.pix_to_face.shape
    pixel_uvs = pixel_uvs.permute(0, 3, 1, 2, 4).reshape(N * K, H_out, W_out, 2)
    N, H_in, W_in, C = maps.shape
    texture_maps = maps.permute(0, 3, 1, 2)[None, ...].expand(K, -1, -1, -1, -1).transpose(0, 1)
    texture_maps = texture_maps.reshape(N * K, C, H_in, W_in)
    pixel_uvs = torch.lerp(pixel_uvs.new_tensor([-1.0, 1.0]), pixel_uvs.new_tensor([1.0, -1.0]), pixel_uvs)
    texels = F.grid_sample(texture_maps, pixel_uvs, mode=sampling_mode, align_corners=align_corners,
                           padding_mode=padding_mode)
    return texels.reshape(N, K, C, H_out, W_out).permute(0, 3, 4, 1, 2)


def fused_sample(fragments, maps, face_uvs, sampling_mode="bilinear", padding_mode="border", align_corners=True):
    from pytorch3d_b200.textures import sample_textures_uv
    return sample_textures_uv(fragments, maps, face_uvs, sampling_mode=sampling_mode, padding_mode=padding_mode,
                              align_corners=align_corners)


def with_grads(fn, s, mode, pad, align):
    """[(name, tensor)]: the texels, then the gradients of the maps, the vertex UVs and the barycentrics under the
    scene's upstream gradient."""
    maps = s["maps"].clone().requires_grad_(True)
    verts_uvs = s["verts_uvs"].clone().requires_grad_(True)
    bary = s["bary"].clone().requires_grad_(True)
    frags = types.SimpleNamespace(pix_to_face=s["pix_to_face"], bary_coords=bary)
    texels = fn(frags, maps, packed_face_uvs(verts_uvs, s["faces_uvs"]), mode, pad, align)
    (texels * s["grad_texels"]).sum().backward()
    grads = [maps.grad, verts_uvs.grad, bary.grad]
    # a nearest sample gives the grid no gradient: the chain leaves these untouched (None), the fused op returns 0
    grads = [torch.zeros_like(t) if g is None else g for g, t in zip(grads, (maps, verts_uvs, bary))]
    return list(zip(FIELDS, [texels.detach()] + grads))


# ------------------------------------------------------------------------------------------------ CPU tests
@pytest.mark.parametrize("args", TEXTURE_CASES, ids=[texture_case(a)[9:] for a in TEXTURE_CASES])
def test_texture_chain_equals_reference_cpu(args):
    mode, pad, align, _, _ = args
    got = with_grads(chain_sample, case_scene(args), mode, pad, align)
    for name, t in got:
        ref = reference(texture_case(args) + "/" + name)[0]
        err = ref.equals(t)
        assert err is None, "%s %s: torch restatement vs the reference (CPU): %s" % (texture_case(args), name, err)


def test_special_uvs_hit_centres_and_ties():
    """The scene's special UVs land exactly on texel centres and on half-texel ties of a dyadic map."""
    for align, (hi, wi) in ((True, (9, 17)), (False, (16, 8))):
        uv = torch.tensor(special_uvs(hi, wi, align))
        g = torch.lerp(uv.new_tensor([-1.0, 1.0]), uv.new_tensor([1.0, -1.0]), uv)
        if align:
            ix, iy = (g[:, 0] + 1) / 2 * (wi - 1), (g[:, 1] + 1) / 2 * (hi - 1)
        else:
            ix, iy = ((g[:, 0] + 1) * wi - 1) / 2, ((g[:, 1] + 1) * hi - 1) / 2
        frac = torch.cat([ix, iy]) % 1
        assert ((frac == 0) | (frac == 0.5)).all()
        assert (frac == 0.5).any() and (frac == 0).any()


def test_textured_torus_uvs():
    from pytorch3d_b200 import synthetic
    meshes, verts_uvs, faces_uvs, maps = synthetic.textured_torus_batch(2, 6, 8, map_size=(16, 32), seed=3)
    faces = meshes.faces_packed()[:faces_uvs[0].shape[0]]
    assert faces_uvs[0].shape == faces.shape and not torch.equal(faces_uvs[0], faces)
    assert verts_uvs[0].shape == (7 * 9, 2) and maps.shape == (2, 16, 32, 3)
    assert float(verts_uvs[0].min()) == 0.0 and float(verts_uvs[0].max()) == 1.0
    # every face's UV triangle is a half cell of the (ring, side) grid: no face spans the seam
    tri = verts_uvs[0][faces_uvs[0]]
    span = tri.max(dim=1).values - tri.min(dim=1).values
    assert torch.allclose(span, torch.tensor([1 / 6, 1 / 8]).expand_as(span))
    again = synthetic.textured_torus_batch(2, 6, 8, map_size=(16, 32), seed=3)[3]
    assert torch.equal(maps, again) and not torch.equal(maps[0], maps[1])


def test_texture_argument_errors():
    from pytorch3d_b200 import _C
    from pytorch3d_b200.textures import sample_textures_uv
    s = texture_scene(2, 3, 4, 2, 5, 6, 3)
    fuv = packed_face_uvs(s["verts_uvs"], s["faces_uvs"])
    p2f, bary, maps = s["pix_to_face"], s["bary"], s["maps"]
    with pytest.raises(RuntimeError, match="CUDA"):
        _C.texture_uv_forward(p2f, bary, fuv, maps)
    with pytest.raises(RuntimeError, match="sampling_mode must be one of"):
        _C.texture_uv_forward(p2f, bary, fuv, maps, "bicubic")
    with pytest.raises(RuntimeError, match="padding_mode must be one of"):
        _C.texture_uv_forward(p2f, bary, fuv, maps, "bilinear", "wrap")
    with pytest.raises(RuntimeError, match="barycentric_coords must be"):
        _C.texture_uv_forward(p2f, bary[..., :2], fuv, maps)
    with pytest.raises(RuntimeError, match="face_uvs must be"):
        _C.texture_uv_forward(p2f, bary, fuv[..., :1], maps)
    with pytest.raises(RuntimeError, match="maps must be"):
        _C.texture_uv_forward(p2f, bary, fuv, maps[:, :0])
    with pytest.raises(RuntimeError, match="pix_to_face must have dimensions"):
        _C.texture_uv_forward(p2f[0], bary, fuv, maps)
    frags = types.SimpleNamespace(pix_to_face=p2f, bary_coords=bary)
    with pytest.raises(ValueError, match="one map per image"):
        sample_textures_uv(frags, maps[:1], fuv)


class _TexturesUV:
    """A stand-in for PyTorch3D's TexturesUV (routing looks at its maps, modes, maps_ids and emptiness only)."""

    def __init__(self, maps, maps_ids=None, empty=False, sampling_mode="bilinear", padding_mode="border"):
        self._maps, self._maps_ids, self._empty = maps, maps_ids, empty
        self.sampling_mode, self.padding_mode, self.align_corners = sampling_mode, padding_mode, True

    def maps_padded(self):
        return self._maps

    def maps_ids_padded(self):
        return self._maps_ids

    def isempty(self):
        return self._empty


def _fake_textures_module(monkeypatch):
    for n in ["pytorch3d", "pytorch3d.renderer", "pytorch3d.renderer.mesh"]:
        m = types.ModuleType(n)
        m.__path__ = []
        monkeypatch.setitem(sys.modules, n, m)
    mod = types.ModuleType("pytorch3d.renderer.mesh.textures")

    class TexturesUV(_TexturesUV):
        def sample_textures(self, fragments, **kwargs):  # defined on the class itself, as in PyTorch3D
            return "ref"

    mod.TexturesUV = TexturesUV
    monkeypatch.setitem(sys.modules, "pytorch3d.renderer.mesh.textures", mod)
    return TexturesUV


def _stand_in(shape, dtype=torch.float32, is_cuda=True, device=None):
    """An object that claims to be a tensor on the GPU (routing looks at device, dtype and shape only)."""
    device = torch.device(device or ("cuda:0" if is_cuda else "cpu"))
    return types.SimpleNamespace(is_cuda=is_cuda, dtype=dtype, shape=torch.Size(shape), dim=lambda: len(shape),
                                 device=device)


def test_install_textures_and_uninstall(monkeypatch, built_lib):
    from pytorch3d_b200 import install as inst
    from pytorch3d_b200 import textures as ours
    cls = _fake_textures_module(monkeypatch)
    original = cls.__dict__["sample_textures"]
    routed = []
    monkeypatch.setattr(ours, "sample_textures", lambda tex, frags, **kw: routed.append(tex) or "b200")
    assert inst.install_textures() == ["pytorch3d.renderer.mesh.textures"]
    assert cls.__dict__["sample_textures"] is not original
    maps = _stand_in((2, 16, 16, 3))
    frags = types.SimpleNamespace(pix_to_face=_stand_in((2, 4, 5, 3), torch.int64),
                                  bary_coords=_stand_in((2, 4, 5, 3, 3)))
    for mode in ("bilinear", "nearest"):
        for pad in ("zeros", "border", "reflection"):
            assert cls(maps, sampling_mode=mode, padding_mode=pad).sample_textures(frags) == "b200"
    assert len(routed) == 6
    # everything else keeps the original method
    cpu_frags = types.SimpleNamespace(pix_to_face=_stand_in((2, 4, 5, 3), torch.int64, is_cuda=False),
                                      bary_coords=_stand_in((2, 4, 5, 3, 3), is_cuda=False))
    i32_frags = types.SimpleNamespace(pix_to_face=_stand_in((2, 4, 5, 3), torch.int32), bary_coords=frags.bary_coords)
    f64_frags = types.SimpleNamespace(pix_to_face=frags.pix_to_face, bary_coords=_stand_in((2, 4, 5, 3, 3),
                                                                                             torch.float64))
    fallbacks = [
        (cls(maps, maps_ids=_stand_in((2, 10), torch.int64)), frags),  # multi-map
        (cls(maps, empty=True), frags),
        (cls(_stand_in((2, 16, 16, 3), is_cuda=False)), frags),  # CPU maps
        (cls(maps), cpu_frags),
        (cls(_stand_in((2, 16, 16, 3), torch.float64)), frags),
        (cls(maps), f64_frags),
        (cls(maps), i32_frags),
        (cls(maps, sampling_mode="bicubic"), frags),
        (cls(maps, padding_mode="wrap"), frags),
        (cls(_stand_in((1, 16, 16, 3))), frags),  # one map for two images
        (cls(_stand_in((2, 16, 16, 3), device="cuda:1")), frags),  # the reference moves these maps to the Fragments
    ]
    for tex, fr in fallbacks:
        assert tex.sample_textures(fr) == "ref"
    assert len(routed) == 6
    inst.uninstall()
    assert cls.__dict__["sample_textures"] is original
    assert inst._saved_methods == {}


def test_install_textures_leaves_the_other_installs_alone(monkeypatch, built_lib):
    from pytorch3d_b200 import install as inst
    _fake_textures_module(monkeypatch)
    inst.install_textures()
    try:
        assert set(inst._saved_methods) == {("pytorch3d.renderer.mesh.textures", "TexturesUV", "sample_textures")}
        assert inst._saved == {} and inst._saved_blend == {}
    finally:
        inst.uninstall()
    assert inst._saved_methods == {}


def test_sample_textures_forms_face_uvs_like_the_reference(monkeypatch):
    from pytorch3d_b200 import textures as ours
    s = texture_scene(2, 3, 4, 2, 5, 6, 3)
    seen = {}

    def spy(fragments, maps, face_uvs, **kw):
        seen.update(kw, maps=maps, face_uvs=face_uvs)
        return "texels"

    monkeypatch.setattr(ours, "sample_textures_uv", spy)
    tex = types.SimpleNamespace(verts_uvs_list=lambda: list(s["verts_uvs"]), faces_uvs_list=lambda: list(s["faces_uvs"]),
                                maps_padded=lambda: s["maps"], isempty=lambda: False, sampling_mode="nearest",
                                padding_mode="zeros", align_corners=False)
    assert ours.sample_textures(tex, None) == "texels"
    assert torch.equal(seen["face_uvs"], packed_face_uvs(s["verts_uvs"], s["faces_uvs"]))
    assert seen["maps"] is s["maps"]
    assert (seen["sampling_mode"], seen["padding_mode"], seen["align_corners"]) == ("nearest", "zeros", False)


# ------------------------------------------------------------------------------------------------ GPU tests
DEV = "cuda:0"


def _close(a, b, name, what, forward_rtol=1e-5, forward_atol=1e-6):
    a, b = a.detach().cpu().double().numpy(), b.detach().cpu().double().numpy()
    forward = not name.startswith("grad_")
    rtol, atol = (forward_rtol, forward_atol) if forward else (1e-4, 1e-5 * float(np.abs(b).max()) + 1e-30)
    assert a.shape == b.shape, "%s %s: shape %s vs %s" % (what, name, a.shape, b.shape)
    assert np.isfinite(a).all(), "%s %s: not finite" % (what, name)
    ok = np.abs(a - b) <= atol + rtol * np.abs(b)
    assert ok.all(), "%s %s: %d values differ, max abs diff %g" % (what, name, int((~ok).sum()),
                                                                  float(np.abs(a - b).max()))


def _compare(s, mode, pad, align, what):
    """The fused op against the chain on CUDA: "nearest" texels bit for bit, "bilinear" within rtol 1e-5 / atol 1e-6,
    gradients within rtol 1e-4 / atol 1e-5 of the largest magnitude.  Returns the largest texel difference."""
    got = with_grads(fused_sample, s, mode, pad, align)
    want = with_grads(chain_sample, s, mode, pad, align)
    for (name, a), (_, b) in zip(got, want):
        if name == "texels" and mode == "nearest":
            assert torch.equal(a, b), "%s texels: %d differ" % (what, int((a != b).sum()))
        else:
            _close(a, b, name, what)
    return float((got[0][1] - want[0][1]).abs().max())


@pytest.mark.gpu
@pytest.mark.parametrize("args", TEXTURE_CASES, ids=[texture_case(a)[9:] for a in TEXTURE_CASES])
def test_fused_matches_reference_records(built_lib, args):
    mode, pad, align, _, _ = args
    s = case_scene(args, device=DEV)
    got = dict(with_grads(fused_sample, s, mode, pad, align))
    mismatched = []
    for name in FIELDS:
        ref = reference(texture_case(args) + "/" + name)[0]
        mine = ref.rows_of(got[name])
        forward = name == "texels"
        rtol, atol = (1e-5, 1e-6) if forward else (1e-4, 1e-5 * max(ref.absmax, 1e-30))
        if not np.all(np.abs(mine - ref.sample) <= atol + rtol * np.abs(ref.sample)):
            mismatched.append(name)
    if mismatched:
        # "nearest" is discontinuous: the CPU chain interpolates the UVs with separate products and a sum, the GPU
        # with an FMA chain.  A slot whose two UVs differ may round to another texel; there the fused op must equal
        # the CUDA chain instead.
        # Only those slots are excused: the texels of every other slot must equal the records, and the map gradient
        # of every other slot's upstream gradient must equal the (CPU) chain's.
        what = texture_case(args)
        assert mode == "nearest", "%s: %s differ from the records" % (what, mismatched)
        assert set(mismatched) <= {"texels", "grad_maps"}, "%s: %s differ from the records" % (what, mismatched)
        s_cpu = {k: v.cpu() for k, v in s.items()}
        fuv = packed_face_uvs(s_cpu["verts_uvs"], s_cpu["faces_uvs"])
        uv_cpu = _interp(s_cpu["pix_to_face"], s_cpu["bary"], fuv)
        uv_gpu = _interp(s["pix_to_face"], s["bary"], fuv.to(DEV)).cpu()
        excused = (uv_cpu != uv_gpu).any(dim=-1).reshape(-1)  # per slot
        ref = reference(what + "/texels")[0]
        mine = ref.rows_of(got["texels"])
        bad_rows = ref.rows[np.flatnonzero((mine != ref.sample).reshape(len(ref.rows), -1).any(axis=1))]
        assert excused[torch.as_tensor(bad_rows, dtype=torch.int64)].all(), \
            "%s: texels differ from the records at slots whose UVs agree" % what
        if "grad_maps" in mismatched:
            keep = (~excused).view(s["pix_to_face"].shape + (1,)).to(torch.float32)
            masked = dict(s_cpu, grad_texels=s_cpu["grad_texels"] * keep)
            got_m = dict(with_grads(fused_sample, {k: v.to(DEV) for k, v in masked.items()}, mode, pad, align))
            want_m = dict(with_grads(chain_sample, masked, mode, pad, align))
            _close(got_m["grad_maps"], want_m["grad_maps"], "grad_maps", what + " (agreeing slots)")
        _compare(s, mode, pad, align, what)  # the excused slots: against the CUDA chain


@pytest.mark.gpu
@pytest.mark.parametrize("args", TEXTURE_CASES[:12], ids=[texture_case(a)[9:] for a in TEXTURE_CASES[:12]])
@pytest.mark.parametrize("K", [1, 2, 8, 50, 200])
def test_fused_matches_torch_chain(built_lib, K, args):
    mode, pad, align, C, (hi, wi) = args
    s = texture_scene(2, 6, 11, K, hi, wi, C, align, seed=1, device=DEV)
    _compare(s, mode, pad, align, "K=%d %s" % (K, texture_case(args)))


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(1, 1, 1, 1), (1, 1, 40, 2), (1, 37, 1, 3), (3, 8, 32, 8), (1, 2, 2, 1)])
@pytest.mark.parametrize("mode,pad,align", [("bilinear", "zeros", False), ("nearest", "border", True),
                                            ("bilinear", "reflection", True)])
def test_fused_matches_torch_chain_on_odd_sizes(built_lib, shape, mode, pad, align):
    for hi, wi, C in ((1, 1, 3), (7, 1, 2), (13, 10, 7)):
        s = texture_scene(*shape, hi, wi, C, align, seed=3, device=DEV)
        _compare(s, mode, pad, align, "shape=%s map=%dx%dx%d %s-%s" % (shape, hi, wi, C, mode, pad))


@pytest.mark.gpu
def test_bilinear_largest_difference_against_the_chain(built_lib):
    """The largest bilinear texel difference over a large scene of every padding and alignment (DESIGN.md section 13
    reports it): only the contraction of the four-corner sum could differ, and the kernel follows torch's."""
    worst = 0.0
    for pad, align in itertools.product(PADDINGS, (True, False)):
        s = texture_scene(4, 64, 64, 8, 37, 53, 3, align, seed=9, device=DEV)
        frags = types.SimpleNamespace(pix_to_face=s["pix_to_face"], bary_coords=s["bary"])
        fuv = packed_face_uvs(s["verts_uvs"], s["faces_uvs"])
        a = fused_sample(frags, s["maps"], fuv, "bilinear", pad, align)
        b = chain_sample(frags, s["maps"], fuv, "bilinear", pad, align)
        worst = max(worst, float((a - b).abs().max()))
    print("largest bilinear texel difference against the CUDA chain: %g" % worst)
    assert worst <= 1e-6


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("pad", PADDINGS)
@pytest.mark.parametrize("align", [True, False])
def test_background_texel_is_exact(built_lib, mode, pad, align):
    """Every slot a background slot: UV (0, 0), i.e. grid (-1, 1), the bottom-left texel."""
    for hi, wi in ((5, 6), (4, 4), (1, 1)):
        s = texture_scene(2, 4, 5, 3, hi, wi, 3, align, seed=4, device=DEV, frac_background=1.0)
        assert (s["pix_to_face"] < 0).all()
        got = dict(with_grads(fused_sample, s, mode, pad, align))
        want = dict(with_grads(chain_sample, s, mode, pad, align))
        assert torch.equal(got["texels"], want["texels"])
        corner = s["maps"][:, hi - 1, 0]  # (N, C)
        if align or pad != "zeros":
            expect = corner  # grid (-1, 1) is the corner texel's centre, or clips / reflects onto it
        elif mode == "bilinear":
            expect = 0.25 * corner  # (-0.5, H_in - 0.5): one of four corners in bounds, weight 1/4
        else:
            expect = corner if (hi - 1) % 2 == 0 else torch.zeros_like(corner)  # rint(H_in - 0.5), half to even
        assert torch.equal(got["texels"], expect[:, None, None, None, :].expand_as(got["texels"]))
        assert (got["grad_bary"] == 0).all() and (got["grad_verts_uvs"] == 0).all()
        _close(got["grad_maps"], want["grad_maps"], "grad_maps", "background %s %s %s" % (mode, pad, align))


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_unaligned_inputs_give_identical_bits(built_lib, mode):
    from pytorch3d_b200 import _C
    s = texture_scene(2, 9, 13, 8, 11, 7, 3, seed=7, device=DEV)
    fuv = packed_face_uvs(s["verts_uvs"], s["faces_uvs"])

    def shifted(t):
        flat_t = torch.empty(t.numel() + 1, dtype=t.dtype, device=t.device)
        out = flat_t[1:].view(t.shape)
        out.copy_(t)
        return out

    args = [s["pix_to_face"], s["bary"], fuv, s["maps"]]
    want_f = _C.texture_uv_forward(*args, mode, "reflection", False)
    want_b = _C.texture_uv_backward(s["grad_texels"], *args, mode, "reflection", False)
    sargs = [shifted(t) for t in args]
    assert sargs[1].data_ptr() % 16 != 0 and sargs[3].data_ptr() % 16 != 0
    got_f = _C.texture_uv_forward(*sargs, mode, "reflection", False)
    got_b = _C.texture_uv_backward(shifted(s["grad_texels"]), *sargs, mode, "reflection", False)
    assert torch.equal(got_f, want_f)
    assert torch.equal(got_b[1], want_b[1])  # grad_bary: written once per slot
    for a, b, name in ((got_b[0], want_b[0], "grad_maps"), (got_b[2], want_b[2], "grad_face_uvs")):
        _close(a, b, name, "unaligned")


@pytest.mark.gpu
def test_outputs_can_be_skipped(built_lib):
    from pytorch3d_b200 import _C
    s = texture_scene(2, 9, 13, 4, 11, 7, 3, seed=8, device=DEV)
    args = [s["grad_texels"], s["pix_to_face"], s["bary"], packed_face_uvs(s["verts_uvs"], s["faces_uvs"]),
            s["maps"], "bilinear", "border", True]
    full = _C.texture_uv_backward(*args)
    for i in range(3):
        part = _C.texture_uv_backward(*args, needs_input_grad=tuple(j != i for j in range(3)))
        assert part[i] is None
        if i != 1:
            assert torch.equal(part[1], full[1])  # grad_bary: written once per slot
        for j in (0, 2):
            if j != i:
                _close(part[j], full[j], ("grad_maps", "", "grad_face_uvs")[j], "without output %d" % i)


@pytest.mark.gpu
def test_texture_errors_on_the_device(built_lib):
    from pytorch3d_b200 import _C
    s = texture_scene(2, 3, 4, 2, 5, 6, 3, device=DEV)
    fuv = packed_face_uvs(s["verts_uvs"], s["faces_uvs"])
    p2f, bary, maps = s["pix_to_face"], s["bary"], s["maps"]
    with pytest.raises(RuntimeError, match="maps.*Float"):
        _C.texture_uv_forward(p2f, bary, fuv, maps.double())
    with pytest.raises(RuntimeError, match="Long"):
        _C.texture_uv_forward(p2f.int(), bary, fuv, maps)
    with pytest.raises(RuntimeError, match="face_uvs must be a CUDA tensor"):
        _C.texture_uv_forward(p2f, bary, fuv.cpu(), maps)
    with pytest.raises(ValueError, match="one map per image"):
        _C.texture_uv_forward(p2f, bary, fuv, maps[:1])
    with pytest.raises(RuntimeError, match="grad_texels"):
        _C.texture_uv_backward(s["grad_texels"][..., :2], p2f, bary, fuv, maps)


@pytest.mark.gpu
def test_deterministic_mode_raises_like_the_grid_sampler(built_lib):
    """Under torch.use_deterministic_algorithms(True) the backward refuses the two atomically accumulated gradients, as
    the chain's CUDA grid sampler backward does; the barycentric gradient alone is deterministic."""
    s = texture_scene(2, 4, 5, 3, 6, 7, 3, device=DEV)
    frags = types.SimpleNamespace(pix_to_face=s["pix_to_face"], bary_coords=s["bary"].clone().requires_grad_(True))
    fuv = packed_face_uvs(s["verts_uvs"], s["faces_uvs"])
    maps = s["maps"].clone().requires_grad_(True)
    was = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        for fn in (fused_sample, chain_sample):
            with pytest.raises(RuntimeError, match="deterministic"):
                fn(frags, maps, fuv).sum().backward()
        fused_sample(frags, s["maps"], fuv).sum().backward()  # grad_bary only
        assert frags.bary_coords.grad is not None
    finally:
        torch.use_deterministic_algorithms(was)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_texture_no_host_sync_and_deterministic(built_lib, mode):
    s = texture_scene(2, 33, 17, 8, 64, 48, 3, seed=8, device=DEV)

    def run():
        return with_grads(fused_sample, s, mode, "border", True)

    run()  # warm-up outside the checked region
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        first = run()
        second = run()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    for (name, a), (_, b) in zip(first, second):
        if name in ("grad_maps", "grad_verts_uvs"):  # atomics
            _close(a, b, name, "repeat")
        else:
            assert torch.equal(a, b), name


@pytest.mark.gpu
def test_map_with_more_than_2_to_the_31_elements(built_lib):
    """Three 16384 x 16384 RGB maps (2.4e9 floats, 9.7 GB), sampled at and near the last texel of the last image, whose
    flat offsets lie past 2^31 - 1, forward and backward."""
    from pytorch3d_b200 import _C
    N, hi, wi, C = 3, 16384, 16384, 3
    last = ((N - 1) * hi + hi - 1) * wi + wi - 1  # flat texel index of maps[N-1, -1, -1]
    assert last * C > 2 ** 31 - 1  # every channel of the texel sampled below is out of reach of 32-bit offsets
    maps = torch.zeros((N, hi, wi, C), dtype=torch.float32, device=DEV)
    maps[N - 1, -4:, -4:] = torch.rand(4, 4, C, generator=torch.Generator().manual_seed(2)).to(DEV)
    K = 6
    p2f = torch.full((N, 1, 1, K), -1, dtype=torch.int64, device=DEV)
    p2f[N - 1] = torch.arange(K, device=DEV).view(1, 1, K)
    eps = 1.0 / (wi - 1)
    uvs = torch.tensor([[1.0, 0.0], [1.0 - 0.3 * eps, 0.2 * eps], [1.0 - 1.5 * eps, 2.5 * eps], [1.0, 1.0 * eps],
                        [1.0 - 2.0 * eps, 0.0], [1.0 - 0.5 * eps, 0.5 * eps]], device=DEV)
    fuv = uvs[:, None, :].expand(K, 3, 2).contiguous()  # face j: all three corners at uvs[j]
    bary = torch.zeros((N, 1, 1, K, 3), device=DEV)
    bary[..., 0] = 1.0
    grid = torch.lerp(uvs.new_tensor([-1.0, 1.0]), uvs.new_tensor([1.0, -1.0]), uvs).view(1, 1, K, 2)
    for mode in MODES:
        got = _C.texture_uv_forward(p2f, bary, fuv, maps, mode, "border", True)
        want = F.grid_sample(maps[N - 1:].permute(0, 3, 1, 2), grid, mode=mode, padding_mode="border",
                             align_corners=True)  # (1, C, 1, K): a strided view of the maps, no copy
        want = want[0, :, 0].transpose(0, 1)
        assert want.abs().sum() > 0
        if mode == "nearest":
            assert torch.equal(got[N - 1, 0, 0], want)
        else:
            _close(got[N - 1, 0, 0], want, "texels", "bilinear near the last texel")
    g = torch.zeros((N, 1, 1, K, C), device=DEV)
    # slot 0 samples exactly texel (H_in-1, W_in-1), with weight 1 under "bilinear" too
    g[N - 1, 0, 0, 0] = torch.tensor([1.0, 2.0, 3.0], device=DEV)
    for mode in MODES:
        g_maps, _, _ = _C.texture_uv_backward(g, p2f, bary, fuv, maps, mode, "border", True, (True, False, False))
        assert torch.equal(g_maps[N - 1, -1, -1], g[N - 1, 0, 0, 0]), mode
        assert int(g_maps.view(-1).count_nonzero()) == C, mode  # nothing landed anywhere else
        del g_maps


def _textured_pipeline(sample, H=48, W=80):
    """Rasterize a textured torus batch, sample its texture with `sample`, shade with the fused Phong shading, blend
    with the fused softmax blend, take a loss; returns the image and the gradients of the vertices, the vertex UVs
    and the maps."""
    from pytorch3d_b200 import synthetic
    from pytorch3d_b200.blending import BlendParams, softmax_rgb_blend
    from pytorch3d_b200.rasterize_meshes import rasterize_meshes
    from pytorch3d_b200.shading import phong_shading
    m, verts_uvs, faces_uvs, maps = synthetic.textured_torus_batch(2, 24, 24, map_size=(64, 96), seed=1, device=DEV)
    m.requires_grad_(True)
    verts_uvs = [v.clone().requires_grad_(True) for v in verts_uvs]
    maps = maps.clone().requires_grad_(True)
    verts = m.verts_packed()
    p2f, zbuf, bary, dists = rasterize_meshes(m, (H, W), blur_radius=1e-4, faces_per_pixel=4)
    frags = types.SimpleNamespace(pix_to_face=p2f, bary_coords=bary, zbuf=zbuf, dists=dists)
    texels = sample(frags, maps, packed_face_uvs(verts_uvs, faces_uvs))
    lights = types.SimpleNamespace(ambient_color=torch.tensor([[0.3, 0.3, 0.3]], device=DEV),
                                   diffuse_color=torch.tensor([[0.6, 0.5, 0.4]], device=DEV),
                                   specular_color=torch.tensor([[0.3, 0.3, 0.3]], device=DEV),
                                   location=torch.tensor([[0.5, 1.0, -1.0]], device=DEV))
    cameras = types.SimpleNamespace(get_camera_center=lambda: torch.zeros(1, 3, device=DEV))
    materials = types.SimpleNamespace(ambient_color=torch.ones(1, 3, device=DEV),
                                      diffuse_color=torch.ones(1, 3, device=DEV),
                                      specular_color=torch.ones(1, 3, device=DEV),
                                      shininess=torch.tensor([64.0], device=DEV))
    colors = phong_shading(m, frags, lights, cameras, materials, texels)
    img = softmax_rgb_blend(colors, frags, BlendParams(sigma=1e-4, gamma=1e-4))
    w = torch.rand(img.shape, generator=torch.Generator().manual_seed(6)).to(DEV)
    (img * w).sum().backward()
    return img.detach(), verts.grad, verts_uvs[0].grad + verts_uvs[1].grad, maps.grad


@pytest.mark.gpu
def test_end_to_end_textured_phong_softmax_matches_torch_chain(built_lib):
    got = _textured_pipeline(fused_sample)
    want = _textured_pipeline(chain_sample)
    _close(got[0], want[0], "image", "textured torus")
    for name, a, b in zip(("grad_verts", "grad_verts_uvs", "grad_maps"), got[1:], want[1:]):
        assert float(b.abs().max()) > 0, name
        _close(a, b, name, "textured torus")
