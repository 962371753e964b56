"""Phong and flat shading (DESIGN.md section 12): the fused `phong_shading`, `_phong_shading_with_pixels` and
`flat_shading` against a torch restatement of the reference's pytorch3d/renderer/mesh/shading.py and
renderer/lighting.py, `PackedMeshes.verts_normals_packed()`, and `install_shading()`.

The stored outputs of the reference (tests/golden/reference_golden_shading.npz, tests/golden/make_shading_golden.py)
pin the restatement below to the reference: its own shading, lighting and materials modules run on the CPU."""
import sys
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import assert_equals_reference, reference

# ------------------------------------------------------------------------------------------------ scenes
MODES = ("phong", "pixels", "flat")  # phong_shading, _phong_shading_with_pixels, flat_shading
LIGHTS = (("point", 1), ("point", "N"), ("directional", 1), ("directional", "N"), ("ambient", 1), ("ambient", "N"))
SHININESS = (64.0, 10.0, 0.0)
# every light kind and batch in every mode; each mode sees every shininess
SHADING_CASES = [(mode, kind, batch, SHININESS[(i + j) % 3])
                 for j, mode in enumerate(MODES) for i, (kind, batch) in enumerate(LIGHTS)]
SCENE = (2, 6, 9, 3)  # N, H, W, K: non-square
LEAVES = ("texels", "bary", "verts", "verts_normals", "faces_normals", "light_ambient", "light_diffuse",
          "light_specular", "light_where", "material_ambient", "material_diffuse", "material_specular", "shininess",
          "camera_center")


def shading_case(args):
    return "shading/%s-%s-%s-%g" % args


def shading_scene(N, H, W, K, light_batch=1, shininess=64.0, seed=0, device="cpu", frac_background=0.3):
    """A dict of float32 tensors (and int64 pix_to_face / faces): random faces, normals and texels, about 30 %
    background slots, zero-length normals (face 0's corners, face 1's face normal), a point light exactly on the first
    corner of face 2 (hit with barycentrics (1, 0, 0) by the last image's first slot), and upstream gradients."""
    g = torch.Generator().manual_seed(seed + 1000 * K + 7 * H + W)
    V, Fn = 24, 16
    verts = torch.randn(V, 3, generator=g)
    faces = torch.randint(0, V, (Fn, 3), generator=g)
    faces[2] = torch.tensor([20, 21, 22])
    faces[0] = torch.tensor([3, 4, 5])
    verts_normals = torch.randn(V, 3, generator=g)
    verts_normals[faces[0]] = 0.0
    faces_normals = torch.randn(Fn, 3, generator=g)
    faces_normals[1] = 0.0
    p2f = torch.randint(0, Fn, (N, H, W, K), generator=g)
    p2f[torch.rand(N, H, W, K, generator=g) < frac_background] = -1
    bary = torch.rand(N, H, W, K, 3, generator=g) + 0.05
    bary = bary / bary.sum(-1, keepdim=True)
    if H * W * K >= 3:
        flat_p2f = p2f.view(N, -1)
        flat_p2f[0, 0], flat_p2f[0, 1] = 0, 1
        flat_p2f[N - 1, -1] = 2
        bary.view(N, -1, 3)[N - 1, -1] = torch.tensor([1.0, 0.0, 0.0])
    B = 1 if light_batch == 1 else N
    where = torch.randn(B, 3, generator=g) * 2.0
    where[-1] = verts[faces[2, 0]]
    s = {
        "pix_to_face": p2f, "faces": faces, "bary": bary, "texels": torch.rand(N, H, W, K, 3, generator=g),
        "verts": verts, "verts_normals": verts_normals, "faces_normals": faces_normals,
        "light_ambient": 0.5 * torch.rand(B, 3, generator=g), "light_diffuse": torch.rand(B, 3, generator=g),
        "light_specular": torch.rand(B, 3, generator=g), "light_where": where,
        "material_ambient": torch.rand(1, 3, generator=g), "material_diffuse": torch.rand(1, 3, generator=g),
        "material_specular": torch.rand(1, 3, generator=g), "shininess": torch.tensor([float(shininess)]),
        "camera_center": torch.randn(B, 3, generator=g) * 3.0,
        "grad_colors": torch.randn(N, H, W, K, 3, generator=g), "grad_positions": torch.randn(N, H, W, K, 3, generator=g),
    }
    return {k: v.to(device) for k, v in s.items()}


def scene_objects(s, kind, leaves):
    """Duck-typed meshes, fragments, lights, cameras and materials over the tensors of `leaves` (a scene dict)."""
    meshes = types.SimpleNamespace(verts_packed=lambda: leaves["verts"], faces_packed=lambda: s["faces"],
                                   verts_normals_packed=lambda: leaves["verts_normals"],
                                   faces_normals_packed=lambda: leaves["faces_normals"])
    fragments = types.SimpleNamespace(pix_to_face=s["pix_to_face"], bary_coords=leaves["bary"])
    lights = types.SimpleNamespace(ambient_color=leaves["light_ambient"])
    if kind != "ambient":
        lights.diffuse_color, lights.specular_color = leaves["light_diffuse"], leaves["light_specular"]
        setattr(lights, "location" if kind == "point" else "direction", leaves["light_where"])
    cameras = types.SimpleNamespace(get_camera_center=lambda: leaves["camera_center"])
    materials = types.SimpleNamespace(ambient_color=leaves["material_ambient"], diffuse_color=leaves["material_diffuse"],
                                      specular_color=leaves["material_specular"], shininess=leaves["shininess"])
    return meshes, fragments, lights, cameras, materials


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


def _broadcast(*ts):
    sizes = [t.shape[0] for t in ts]
    n = max(sizes)
    if any(s not in (1, n) for s in sizes):
        raise ValueError("Got non-broadcastable sizes %r" % sizes)
    return [t.expand((n,) + tuple(t.shape[1:])) for t in ts]


def _normalize(x):
    return F.normalize(x, p=2, dim=-1, eps=1e-6)


def chain_lighting(points, normals, lights, cameras, materials):
    """_apply_lighting with the light's diffuse() and specular(), in the reference's operations."""
    from pytorch3d_b200.shading import light_kind
    kind = light_kind(lights)
    expand = (-1,) + (1,) * (points.dim() - 2) + (3,)
    if kind == "ambient":
        light_diffuse = torch.zeros(*points.shape[:-1], 3, device=points.device)
        light_specular = torch.zeros(*points.shape[:-1], 3, device=points.device)
    else:
        def direction():  # evaluated once by diffuse() and once by specular(), as in the reference
            return lights.location[:, None, None, None, :] - points if kind == "point" else lights.direction

        nrm, color, d = _broadcast(normals, lights.diffuse_color, direction())
        d = d if d.shape == nrm.shape else d.view(expand)
        color = color if color.shape == nrm.shape else color.view(expand)
        angle = F.relu(torch.sum(_normalize(nrm) * _normalize(d), dim=-1))
        light_diffuse = color * angle[..., None]
        _, color, d, cam, shin = _broadcast(points, lights.specular_color, direction(), cameras.get_camera_center(),
                                            materials.shininess)
        d = d if d.shape == normals.shape else d.view(expand)
        color = color if color.shape == normals.shape else color.view(expand)
        cam = cam if cam.shape == normals.shape else cam.view(expand)
        shin = shin if shin.shape == normals.shape else shin.view(expand[:-1])
        nn, dn = _normalize(normals), _normalize(d)
        cos = torch.sum(nn * dn, dim=-1)
        mask = (cos > 0).to(torch.float32)
        view = _normalize(cam - points)
        reflect = -dn + 2 * (cos[..., None] * nn)
        alpha = F.relu(torch.sum(view * reflect, dim=-1)) * mask
        light_specular = color * torch.pow(alpha, shin)[..., None]
    ambient = materials.ambient_color * lights.ambient_color
    diffuse = materials.diffuse_color * light_diffuse
    specular = materials.specular_color * light_specular
    if ambient.ndim != diffuse.ndim:
        ambient = ambient[:, None, None, None, :]
    return ambient, diffuse, specular


def chain_phong_with_pixels(meshes, fragments, lights, cameras, materials, texels):
    verts, faces = meshes.verts_packed(), meshes.faces_packed()
    normals = meshes.verts_normals_packed()
    coords = _interp(fragments.pix_to_face, fragments.bary_coords, verts[faces])
    pixel_normals = _interp(fragments.pix_to_face, fragments.bary_coords, normals[faces])
    ambient, diffuse, specular = chain_lighting(coords, pixel_normals, lights, cameras, materials)
    return (ambient + diffuse) * texels + specular, coords


def chain_phong(meshes, fragments, lights, cameras, materials, texels):
    return chain_phong_with_pixels(meshes, fragments, lights, cameras, materials, texels)[0]


def chain_flat(meshes, fragments, lights, cameras, materials, texels):
    verts, faces = meshes.verts_packed(), meshes.faces_packed()
    face_normals = meshes.faces_normals_packed()
    face_coords = verts[faces].mean(dim=-2)
    mask = fragments.pix_to_face == -1
    pix_to_face = fragments.pix_to_face.clone()
    pix_to_face[mask] = 0
    N, H, W, K = pix_to_face.shape
    idx = pix_to_face.view(N * H * W * K, 1).expand(N * H * W * K, 3)
    pixel_coords = face_coords.gather(0, idx).view(N, H, W, K, 3)
    pixel_coords[mask] = 0.0
    pixel_normals = face_normals.gather(0, idx).view(N, H, W, K, 3)
    pixel_normals[mask] = 0.0
    ambient, diffuse, specular = chain_lighting(pixel_coords, pixel_normals, lights, cameras, materials)
    return (ambient + diffuse) * texels + specular


CHAIN = {"phong": chain_phong, "pixels": chain_phong_with_pixels, "flat": chain_flat}


def fused(mode):
    from pytorch3d_b200 import shading
    return {"phong": shading.phong_shading, "pixels": shading._phong_shading_with_pixels,
            "flat": shading.flat_shading}[mode]


def with_grads(fn, s, mode, kind, dtype=torch.float32, param_grads=True):
    """[(name, tensor)]: the outputs, then the gradient of every leaf that received one, under the scene's upstream
    gradients (of the colours, and of the positions in "pixels" mode)."""
    params = {"light_ambient", "light_diffuse", "light_specular", "light_where", "material_ambient",
              "material_diffuse", "material_specular", "shininess", "camera_center"}
    leaves = {k: s[k].to(dtype).clone().requires_grad_(param_grads or k not in params) for k in LEAVES}
    objs = scene_objects(s, kind, leaves)
    out = fn(*objs, leaves["texels"])
    outs = list(out) if isinstance(out, tuple) else [out]
    loss = (outs[0] * s["grad_colors"].to(dtype)).sum()
    if len(outs) > 1:
        loss = loss + (outs[1] * s["grad_positions"].to(dtype)).sum()
    loss.backward()
    named = [("colors", outs[0].detach())] + ([("pixel_coords", outs[1].detach())] if len(outs) > 1 else [])
    return named + [("grad_" + k, leaves[k].grad) for k in LEAVES if leaves[k].grad is not None]


# ------------------------------------------------------------------------------------------------ CPU tests
@pytest.mark.parametrize("args", SHADING_CASES, ids=[shading_case(a)[8:] for a in SHADING_CASES])
def test_shading_chain_equals_reference_cpu(args):
    mode, kind, batch, shininess = args
    s = shading_scene(*SCENE, batch, shininess)
    got = with_grads(CHAIN[mode], s, mode, kind)
    for name, t in got:
        assert_equals_reference([t], shading_case(args) + "/" + name, "torch restatement vs the reference (CPU)")


def test_verts_normals_packed_equals_reference_cpu():
    from pytorch3d_b200 import synthetic
    m = synthetic.torus_batch(2, 7, 9, seed=3)
    assert_equals_reference([m.verts_normals_packed()], "shading/torus_verts_normals", "verts_normals_packed")


def test_verts_normals_packed_is_differentiable_and_unit():
    from pytorch3d_b200 import synthetic
    m = synthetic.torus_batch(1, 6, 8, seed=2).requires_grad_(True)
    n = m.verts_normals_packed()
    assert torch.allclose(n.norm(dim=1), torch.ones(n.shape[0]), atol=1e-5)
    n.sum().backward()
    assert m.verts_packed().grad is not None


def test_shading_argument_errors():
    from pytorch3d_b200 import _C
    from pytorch3d_b200.shading import phong_shading
    s = shading_scene(1, 3, 4, 2)
    prm = torch.zeros(1, _C.SHADING_PARAMS)
    fv = s["verts"][s["faces"]]
    with pytest.raises(RuntimeError, match="CUDA"):
        _C.shading_forward(s["pix_to_face"], s["bary"], fv, fv, s["texels"], prm, False, "point")
    with pytest.raises(RuntimeError, match="light must be one of"):
        _C.shading_forward(s["pix_to_face"], s["bary"], fv, fv, s["texels"], prm, False, "spot")
    meshes, fragments, lights, cameras, materials = scene_objects(s, "point", s)
    lights.location = torch.zeros(3, 3)  # batch 3 against an image batch of 1
    with pytest.raises(ValueError, match="Got non-broadcastable sizes"):
        phong_shading(meshes, fragments, lights, cameras, materials, s["texels"])
    meshes, fragments, lights, cameras, materials = scene_objects(s, "directional", s)
    materials.diffuse_color = torch.ones(2, 3)
    with pytest.raises(ValueError, match="non-broadcastable"):
        phong_shading(meshes, fragments, lights, cameras, materials, s["texels"])
    meshes, fragments, lights, cameras, materials = scene_objects(s, "directional", s)
    with pytest.raises(ValueError, match="texels must have shape"):
        phong_shading(meshes, fragments, lights, cameras, materials, s["texels"][..., :2])
    with pytest.raises(RuntimeError, match="CUDA"):
        phong_shading(meshes, fragments, lights, cameras, materials, s["texels"])


class _Lights:
    def __init__(self, **kw):
        self.__dict__.update(kw)


def _fake_pytorch3d(monkeypatch):
    calls = []
    lighting = types.ModuleType("pytorch3d.renderer.lighting")

    class PointLights(_Lights):
        pass

    class DirectionalLights(_Lights):
        pass

    class AmbientLights(_Lights):
        pass

    class Materials(_Lights):
        pass

    lighting.PointLights, lighting.DirectionalLights, lighting.AmbientLights = PointLights, DirectionalLights, AmbientLights
    materials = types.ModuleType("pytorch3d.renderer.materials")
    materials.Materials = Materials
    for n in ["pytorch3d", "pytorch3d.renderer", "pytorch3d.renderer.mesh", "pytorch3d.renderer.mesh.shading",
              "pytorch3d.renderer.mesh.shader"]:
        m = types.ModuleType(n)
        m.__path__ = []
        monkeypatch.setitem(sys.modules, n, m)
    monkeypatch.setitem(sys.modules, "pytorch3d.renderer.lighting", lighting)
    monkeypatch.setitem(sys.modules, "pytorch3d.renderer.materials", materials)
    originals = {}
    for name in ("phong_shading", "_phong_shading_with_pixels", "flat_shading"):
        def ref(meshes, fragments, lights, cameras, materials, texels, _name=name):
            calls.append(_name)
            return "ref_" + _name
        originals[name] = ref
        for n in ("pytorch3d.renderer.mesh.shading", "pytorch3d.renderer.mesh.shader"):
            setattr(sys.modules[n], name, ref)
    return types.SimpleNamespace(PointLights=PointLights, DirectionalLights=DirectionalLights,
                                 AmbientLights=AmbientLights, Materials=Materials), originals, calls


def _stand_in(shape, dtype=torch.float32, is_cuda=True):
    """An object that claims to be a tensor on the GPU (routing looks at device, dtype and shape only)."""
    return types.SimpleNamespace(is_cuda=is_cuda, dtype=dtype, shape=torch.Size(shape), dim=lambda: len(shape))


def test_install_shading_and_uninstall(monkeypatch, built_lib):
    from pytorch3d_b200 import install as inst
    from pytorch3d_b200 import shading as ours
    cls, originals, calls = _fake_pytorch3d(monkeypatch)
    patched = inst.install_shading()
    assert patched == ["pytorch3d.renderer.mesh.shading", "pytorch3d.renderer.mesh.shader"]
    sh = sys.modules["pytorch3d.renderer.mesh.shader"]
    routed = []
    for name in originals:
        monkeypatch.setattr(ours, name, lambda *a, _n=name: routed.append(_n) or "b200_" + _n)
    for modname in patched:
        for name in originals:
            assert getattr(sys.modules[modname], name) is not originals[name]
    c3 = torch.ones(1, 3)
    mats = cls.Materials(ambient_color=c3, diffuse_color=c3, specular_color=c3, shininess=torch.ones(1))
    point = cls.PointLights(ambient_color=c3, diffuse_color=c3, specular_color=c3, location=c3)
    texels = _stand_in((1, 2, 3, 4, 3))
    frags = types.SimpleNamespace(pix_to_face=_stand_in((1, 2, 3, 4), torch.int64), bary_coords=texels)
    assert sh.phong_shading(None, frags, point, None, mats, texels) == "b200_phong_shading"
    assert sh._phong_shading_with_pixels(None, frags, point, None, mats, texels) == "b200__phong_shading_with_pixels"
    amb = cls.AmbientLights(ambient_color=c3)
    dirl = cls.DirectionalLights(ambient_color=c3, diffuse_color=c3, specular_color=c3, direction=c3)
    assert sys.modules["pytorch3d.renderer.mesh.shading"].flat_shading(None, frags, amb, None, mats, texels) \
        == "b200_flat_shading"
    assert sh.flat_shading(None, frags, dirl, None, mats, texels) == "b200_flat_shading"
    assert calls == []
    # everything else keeps the originals
    class MyLights(cls.PointLights):  # a subclass may have its own diffuse / specular
        pass

    mine = MyLights(ambient_color=c3, diffuse_color=c3, specular_color=c3, location=c3)
    assert sh.phong_shading(None, frags, mine, None, mats, texels) == "ref_phong_shading"
    assert sh.phong_shading(None, frags, types.SimpleNamespace(ambient_color=c3), None, mats, texels) \
        == "ref_phong_shading"
    cpu = _stand_in((1, 2, 3, 4, 3), is_cuda=False)
    assert sh.phong_shading(None, frags, point, None, mats, cpu) == "ref_phong_shading"
    f64 = _stand_in((1, 2, 3, 4, 3), torch.float64)
    assert sh.flat_shading(None, frags, point, None, mats, f64) == "ref_flat_shading"
    four = _stand_in((1, 2, 3, 4, 4))
    assert sh.phong_shading(None, frags, point, None, mats, four) == "ref_phong_shading"
    mats4 = cls.Materials(ambient_color=torch.ones(1, 4), diffuse_color=torch.ones(1, 4),
                          specular_color=torch.ones(1, 4), shininess=torch.ones(1))
    assert sh.phong_shading(None, frags, point, None, mats4, texels) == "ref_phong_shading"
    mats2 = cls.Materials(ambient_color=torch.ones(2, 3), diffuse_color=torch.ones(2, 3),
                          specular_color=torch.ones(2, 3), shininess=torch.ones(2))
    assert sh.phong_shading(None, frags, point, None, mats2, texels) == "ref_phong_shading"
    assert sh._phong_shading_with_pixels(None, frags, point, None, cls.Materials, texels) \
        == "ref__phong_shading_with_pixels"
    assert len(calls) == 8 and len(routed) == 4
    inst.uninstall()
    for modname in patched:
        for name in originals:
            assert getattr(sys.modules[modname], name) is originals[name]
    assert inst._saved_blend == {}


def test_install_shading_leaves_the_other_installs_alone(monkeypatch, built_lib):
    from pytorch3d_b200 import install as inst
    _fake_pytorch3d(monkeypatch)
    inst.install_shading()
    try:
        assert set(inst._saved_blend) == {(m, n) for m in inst._SHADING_MODULES for n in inst._SHADING_FUNCTIONS}
        assert inst._saved == {}
    finally:
        inst.uninstall()
    assert inst._saved_blend == {}


# ------------------------------------------------------------------------------------------------ GPU tests
DEV = "cuda:0"


def _tol_check(got, want, what, f64=None, f32=None):
    """Forward rtol 1e-5 / atol 1e-6; gradients rtol 1e-4 / atol 1e-5 of the largest magnitude.  Where `f64` (a float64
    chain) and `f32` (the float32 chain) are given, a field outside those tolerances still passes when its largest
    error against float64 is at most twice the float32 chain's own (shininess >= 64: pow amplifies relative errors)."""
    want_d = dict(want)
    got_names = [n for n, _ in got]
    assert all(n in got_names for n in want_d), "%s: fields %s vs %s" % (what, got_names, list(want_d))
    for name, a in got:
        if name not in want_d:  # an input the chain's graph does not reach: the fused op returns exact zeros for it
            assert not a.any(), "%s %s: the chain gives no gradient, the fused op a nonzero one" % (what, name)
            continue
        a, b = a.detach().cpu().double().numpy(), want_d[name].detach().cpu().double().numpy()
        forward = not name.startswith("grad_")
        rtol, atol = (1e-5, 1e-6) if forward else (1e-4, 1e-5 * float(np.abs(b).max()) + 1e-30)
        assert np.isfinite(a).all(), "%s %s: not finite" % (what, name)
        if np.all(np.abs(a - b) <= atol + rtol * np.abs(b)):
            continue
        assert f64 is not None, "%s %s: max abs diff %g" % (what, name, float(np.abs(a - b).max()))
        ref = dict(f64)[name].detach().cpu().numpy()
        err = float(np.abs(a - ref).max())
        own = float(np.abs(dict(f32)[name].detach().cpu().double().numpy() - ref).max())
        assert err <= 2.0 * own, "%s %s: error %g against float64, the float32 chain's %g" % (what, name, err, own)


def _compare(mode, kind, s, what, param_grads=True):
    got = with_grads(fused(mode), s, mode, kind, param_grads=param_grads)
    want = with_grads(CHAIN[mode], s, mode, kind, param_grads=param_grads)
    f64 = None
    if float(s["shininess"][0]) >= 64:
        f64 = with_grads(CHAIN[mode], {k: v.cpu() for k, v in s.items()}, mode, kind, torch.float64, param_grads)
    _tol_check(got, want, what, f64, want)
    return got, want


@pytest.mark.gpu
@pytest.mark.parametrize("args", SHADING_CASES, ids=[shading_case(a)[8:] for a in SHADING_CASES])
def test_fused_matches_reference_records(built_lib, args):
    mode, kind, batch, shininess = args
    s = shading_scene(*SCENE, batch, shininess, device=DEV)
    got = dict(with_grads(fused(mode), s, mode, kind))
    want = with_grads(CHAIN[mode], {k: v.cpu() for k, v in s.items()}, mode, kind)  # equals the records (CPU test)
    f64 = with_grads(CHAIN[mode], {k: v.cpu() for k, v in s.items()}, mode, kind, torch.float64)
    for name, _ in want:
        ref = reference(shading_case(args) + "/" + name)[0]
        mine = ref.rows_of(got[name])
        forward = not name.startswith("grad_")
        rtol, atol = (1e-5, 1e-6) if forward else (1e-4, 1e-5 * max(ref.absmax, 1e-30))
        if not np.all(np.abs(mine - ref.sample) <= atol + rtol * np.abs(ref.sample)):
            assert shininess >= 64, "%s %s: max abs diff %g" % (args, name, float(np.abs(mine - ref.sample).max()))
            d64 = dict(f64)[name].detach().numpy()
            err = float(np.abs(got[name].detach().cpu().double().numpy() - d64).max())
            own = float(np.abs(dict(want)[name].detach().double().numpy() - d64).max())
            assert err <= 2.0 * own, "%s %s: error %g against float64, the float32 chain's %g" % (args, name, err, own)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("K", [1, 2, 8, 13, 150, 200])
def test_fused_matches_torch_chain(built_lib, K, mode):
    s = shading_scene(2, 11, 7, K, "N", 10.0, seed=1, device=DEV)
    _compare(mode, "point", s, "K=%d %s" % (K, mode))


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("shininess", SHININESS)
@pytest.mark.parametrize("kind,batch", LIGHTS)
def test_fused_matches_torch_chain_every_light(built_lib, kind, batch, shininess, mode):
    s = shading_scene(3, 16, 21, 8, batch, shininess, seed=2, device=DEV)
    _compare(mode, kind, s, "%s-%s s=%g %s" % (kind, batch, shininess, mode))


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(1, 1, 1, 1), (1, 1, 40, 2), (1, 37, 1, 3), (3, 8, 32, 8), (1, 2, 2, 1)])
@pytest.mark.parametrize("mode", MODES)
def test_fused_matches_torch_chain_on_odd_sizes(built_lib, shape, mode):
    s = shading_scene(*shape, 1, 10.0, seed=3, device=DEV)
    _compare(mode, "directional", s, "shape=%s %s" % (shape, mode))


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_without_parameter_gradients_no_grad_params_is_computed(built_lib, monkeypatch, mode):
    from pytorch3d_b200 import _C
    seen = []
    real = _C.shading_backward

    def spy(*args):
        out = real(*args)
        seen.append((tuple(args[-1]), out[4]))
        return out

    monkeypatch.setattr(_C, "shading_backward", spy)
    s = shading_scene(2, 9, 13, 4, "N", 10.0, seed=4, device=DEV)
    got = with_grads(fused(mode), s, mode, "point", param_grads=False)
    want = with_grads(CHAIN[mode], s, mode, "point", param_grads=False)
    _tol_check(got, want, "no parameter grads, %s" % mode)
    assert not any(name.startswith("grad_light") or name == "grad_shininess" for name, _ in got)
    assert seen and seen[-1][0][4] is False and seen[-1][1] is None


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("kind", ["point", "directional", "ambient"])
def test_exact_zeros_and_the_shininess_zero_background(built_lib, kind, mode):
    s = shading_scene(2, 9, 13, 4, 1, 0.0, seed=5, device=DEV)
    got, want = _compare(mode, kind, s, "shininess 0 %s %s" % (kind, mode))
    got, want = dict(got), dict(want)
    bg = s["pix_to_face"] < 0
    # background slots: ambient * texel + ms * ls (pow(0, 0) = 1), bit for bit
    assert torch.equal(got["colors"][bg], want["colors"][bg])
    if kind != "ambient":
        amb = (s["material_ambient"] * s["light_ambient"])[0]
        spec = s["material_specular"][0] * (s["light_specular"][0] * 1.0)
        assert torch.equal(got["colors"][bg], amb * s["texels"][bg] + spec)
    if mode != "flat":
        assert (got["grad_bary"][bg] == 0).all()
    if "pixel_coords" in got:
        assert (got["pixel_coords"][bg] == 0).all()
    for name, t in got.items():
        assert torch.isfinite(t).all(), name


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["point", "ambient"])
def test_positions_equal_interp_face_attrs_bit_for_bit(built_lib, kind):
    from pytorch3d_b200 import _C
    from pytorch3d_b200.shading import _phong_shading_with_pixels
    s = shading_scene(2, 33, 17, 8, 1, 64.0, seed=6, device=DEV)
    _, positions = _phong_shading_with_pixels(*scene_objects(s, kind, s), s["texels"])
    P = s["pix_to_face"].numel()
    want = _C.interp_face_attrs_forward(s["pix_to_face"].view(P), s["bary"].view(P, 3), s["verts"][s["faces"]])
    assert torch.equal(positions.reshape(P, 3), want)


@pytest.mark.gpu
@pytest.mark.parametrize("flat", [False, True])
def test_unaligned_inputs_give_identical_bits(built_lib, flat):
    from pytorch3d_b200 import _C
    s = shading_scene(2, 9, 13, 8, "N", 10.0, seed=7, device=DEV)
    if flat:
        fp, fn = s["verts"][s["faces"]].mean(dim=-2), s["faces_normals"]
    else:
        fp, fn = s["verts"][s["faces"]], s["verts_normals"][s["faces"]]
    prm = torch.rand(2, _C.SHADING_PARAMS, device=DEV)
    prm[:, 21] = 10.0

    def shifted(t):
        flat_t = torch.empty(t.numel() + 1, dtype=t.dtype, device=t.device)
        out = flat_t[1:].view(t.shape)
        out.copy_(t)
        return out

    args = [s["pix_to_face"], s["bary"], fp, fn, s["texels"], prm]
    gc, gp = s["grad_colors"], s["grad_positions"]
    want_f = _C.shading_forward(*args, flat, "point", not flat)
    want_b = _C.shading_backward(gc, None if flat else gp, *args, flat, "point", (True, True, False, False, True))
    sargs = [shifted(t) for t in args]
    assert sargs[1].data_ptr() % 16 != 0
    got_f = _C.shading_forward(*sargs, flat, "point", not flat)
    got_b = _C.shading_backward(shifted(gc), None if flat else shifted(gp), *sargs, flat, "point",
                                (True, True, False, False, True))
    for a, b in zip(list(got_f) + list(got_b), list(want_f) + list(want_b)):
        assert (a is None and b is None) or torch.equal(a, b)


@pytest.mark.gpu
def test_shading_errors_on_the_device(built_lib):
    from pytorch3d_b200 import _C
    s = shading_scene(1, 3, 4, 2, device=DEV)
    fv, fn = s["verts"][s["faces"]], s["verts_normals"][s["faces"]]
    prm = torch.zeros(1, _C.SHADING_PARAMS, device=DEV)
    p2f, bary, tx = s["pix_to_face"], s["bary"], s["texels"]
    with pytest.raises(RuntimeError, match="texels.*Float"):
        _C.shading_forward(p2f, bary, fv, fn, tx.double(), prm, False, "point")
    with pytest.raises(RuntimeError, match="Long"):
        _C.shading_forward(p2f.int(), bary, fv, fn, tx, prm, False, "point")
    with pytest.raises(RuntimeError, match="texels must be"):
        _C.shading_forward(p2f, bary, fv, fn, tx[..., :2], prm, False, "point")
    with pytest.raises(RuntimeError, match="barycentric_coords must be"):
        _C.shading_forward(p2f, bary[:, :1], fv, fn, tx, prm, False, "point")
    with pytest.raises(RuntimeError, match="face_positions must be"):
        _C.shading_forward(p2f, bary, fv[:, :2], fn, tx, prm, False, "point")
    with pytest.raises(RuntimeError, match="face_normals must be"):
        _C.shading_forward(p2f, bary, fv, fn[:, 0], tx, prm, False, "point")
    with pytest.raises(RuntimeError, match="params must be"):
        _C.shading_forward(p2f, bary, fv, fn, tx, prm[:, :21], False, "point")
    with pytest.raises(RuntimeError, match="pix_to_face must be a CUDA tensor"):
        _C.shading_forward(p2f.cpu(), bary, fv, fn, tx, prm, False, "point")
    with pytest.raises(RuntimeError, match="grad_colors"):
        _C.shading_backward(s["grad_colors"][..., :2], None, p2f, bary, fv, fn, tx, prm, False, "point")


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_shading_no_host_sync_and_deterministic(built_lib, mode):
    s = shading_scene(2, 33, 17, 8, "N", 64.0, seed=8, device=DEV)

    def run():
        return with_grads(fused(mode), s, mode, "point")

    run()  # warm-up outside the checked region
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        first = run()
        second = run()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    for (name, a), (_, b) in zip(first, second):
        if name in ("grad_verts", "grad_verts_normals", "grad_faces_normals"):  # atomics in the face scatter
            np.testing.assert_allclose(a.cpu().numpy(), b.cpu().numpy(), rtol=1e-5,
                                       atol=1e-6 * float(b.abs().max()), err_msg=name)
        else:
            assert torch.equal(a, b), name


def _torus_scene():
    from pytorch3d_b200 import synthetic
    m = synthetic.torus_batch(2, 24, 24, seed=1, device=DEV)
    m.requires_grad_(True)
    return m


def _torus_objects(m):
    verts = m.verts_packed()
    lights = types.SimpleNamespace(ambient_color=torch.tensor([[0.3, 0.3, 0.3]], device=DEV),
                                   diffuse_color=torch.tensor([[0.6, 0.5, 0.4]], device=DEV),
                                   specular_color=torch.tensor([[0.3, 0.3, 0.3]], device=DEV),
                                   location=torch.tensor([[0.5, 1.0, -1.0]], device=DEV))
    cameras = types.SimpleNamespace(get_camera_center=lambda: torch.zeros(1, 3, device=DEV))
    materials = types.SimpleNamespace(ambient_color=torch.ones(1, 3, device=DEV),
                                      diffuse_color=torch.ones(1, 3, device=DEV),
                                      specular_color=torch.ones(1, 3, device=DEV),
                                      shininess=torch.tensor([64.0], device=DEV))
    return verts, lights, cameras, materials


def _torus_phong_pipeline(shade):
    """Rasterize a torus batch, shade it with `shade`, blend with the fused softmax blend, take a loss and return the
    image and the vertex gradient."""
    from pytorch3d_b200.blending import BlendParams, softmax_rgb_blend
    from pytorch3d_b200.rasterize_meshes import rasterize_meshes
    m = _torus_scene()
    verts, lights, cameras, materials = _torus_objects(m)
    H, W = 48, 80
    p2f, zbuf, bary, dists = rasterize_meshes(m, (H, W), blur_radius=1e-4, faces_per_pixel=4)
    frags = types.SimpleNamespace(pix_to_face=p2f, bary_coords=bary, zbuf=zbuf, dists=dists)
    texels = torch.rand(p2f.shape + (3,), generator=torch.Generator().manual_seed(4)).to(DEV)
    colors = shade(m, frags, lights, cameras, materials, texels)
    img = softmax_rgb_blend(colors, frags, BlendParams(sigma=1e-4, gamma=1e-4))
    w = torch.rand(img.shape, generator=torch.Generator().manual_seed(6)).to(DEV)
    (img * w).sum().backward()
    return img.detach(), verts.grad


def _torus_splatter_pipeline(shade):
    """_phong_shading_with_pixels, then the fused splatter blend (an identity projection of the camera-space positions
    scaled onto the pixel grid), a loss, and the vertex gradient."""
    from pytorch3d_b200.blending import BlendParams
    from pytorch3d_b200.rasterize_meshes import rasterize_meshes
    from pytorch3d_b200.splatter_blend import splatter_blend
    m = _torus_scene()
    verts, lights, cameras, materials = _torus_objects(m)
    H, W = 48, 80
    p2f, zbuf, bary, dists = rasterize_meshes(m, (H, W), blur_radius=0.0, faces_per_pixel=4)
    frags = types.SimpleNamespace(pix_to_face=p2f, bary_coords=bary.detach())
    texels = torch.rand(p2f.shape + (3,), generator=torch.Generator().manual_seed(4)).to(DEV)
    colors, coords = shade(m, frags, lights, cameras, materials, texels)
    scale = torch.tensor([H / 2.0, W / 2.0, 1.0], device=DEV)
    offset = torch.tensor([H / 2.0, W / 2.0, 0.0], device=DEV)
    screen = coords[..., [1, 0, 2]] * scale + offset
    img = splatter_blend(colors, screen, p2f < 0, BlendParams(sigma=0.5, background_color=(1.0, 1.0, 1.0)))
    w = torch.rand(img.shape, generator=torch.Generator().manual_seed(6)).to(DEV)
    (img * w).sum().backward()
    return img.detach(), verts.grad


@pytest.mark.gpu
def test_end_to_end_phong_softmax_matches_torch_chain(built_lib):
    from pytorch3d_b200.shading import phong_shading
    img, g = _torus_phong_pipeline(phong_shading)
    img_ref, g_ref = _torus_phong_pipeline(chain_phong)
    np.testing.assert_allclose(img.cpu().numpy(), img_ref.cpu().numpy(), rtol=1e-5, atol=1e-6)
    assert float(g_ref.abs().max()) > 0
    np.testing.assert_allclose(g.cpu().numpy(), g_ref.cpu().numpy(), rtol=1e-4, atol=1e-5 * float(g_ref.abs().max()))


@pytest.mark.gpu
def test_end_to_end_phong_splatter_matches_torch_chain(built_lib):
    from pytorch3d_b200.shading import _phong_shading_with_pixels
    img, g = _torus_splatter_pipeline(_phong_shading_with_pixels)
    img_ref, g_ref = _torus_splatter_pipeline(chain_phong_with_pixels)
    np.testing.assert_allclose(img.cpu().numpy(), img_ref.cpu().numpy(), rtol=1e-5, atol=1e-6)
    assert float(g_ref.abs().max()) > 0
    np.testing.assert_allclose(g.cpu().numpy(), g_ref.cpu().numpy(), rtol=1e-4, atol=1e-5 * float(g_ref.abs().max()))
