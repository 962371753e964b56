"""Gouraud shading (DESIGN.md section 16): the fused `gouraud_shading` against a torch restatement of the reference's
pytorch3d/renderer/mesh/shading.py gouraud_shading (per-vertex `_apply_lighting` with the light, material and camera
properties gathered per vertex, `verts_colors * (ambient + diffuse) + specular`, the (F, 3, 3) gather and
interpolate_face_attributes), `PackedMeshes`' vertex accessors, and `install_gouraud()`."""
import sys
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_shading import _stand_in, _tol_check

DEV = "cuda:0"
LIGHTS = (("point", 1), ("point", "N"), ("directional", 1), ("directional", "N"), ("ambient", 1), ("ambient", "N"))
SHININESS = (64.0, 10.0, 0.0)
# every light kind and batch, each shininess, one and three meshes
CASES = [(kind, batch, SHININESS[i % 3], meshes) for i, (kind, batch) in enumerate(LIGHTS) for meshes in (1, 3)]
LEAVES = ("verts", "normals", "colors", "bary", "light_ambient", "light_diffuse", "light_specular", "light_where",
          "material_ambient", "material_diffuse", "material_specular", "shininess", "camera_center")


class _Meshes:
    """Duck-typed packed meshes with vertex colours; `normals` is a leaf so that its gradient can be checked."""

    def __init__(self, s, leaves):
        self._s, self._l = s, leaves
        self.textures = types.SimpleNamespace(verts_features_packed=lambda: leaves["colors"])

    def __len__(self):
        return int(self._s["num"].shape[0])

    def verts_packed(self):
        return self._l["verts"]

    def faces_packed(self):
        return self._s["faces"]

    def verts_normals_packed(self):
        return self._l["normals"]

    def num_verts_per_mesh(self):
        return self._s["num"]

    def mesh_to_verts_packed_first_idx(self):
        return self._s["first"]


def gouraud_scene(sizes, H, W, K, light_batch=1, shininess=64.0, seed=0, device="cpu", frac_background=0.3,
                  material_batch=1):
    """Meshes of `sizes` vertices (a 0 is an empty mesh) with random faces inside each mesh, random normals and
    colours, one isolated vertex with a zero normal per mesh of >= 4 vertices, about 30 % background slots, a point
    light on the first vertex of the last non-empty mesh, and upstream gradients."""
    g = torch.Generator().manual_seed(seed + 1000 * K + 7 * H + W + 31 * len(sizes))
    N = len(sizes)
    V = sum(sizes)
    first = torch.tensor([sum(sizes[:i]) for i in range(N)], dtype=torch.int64)
    faces = []
    for i, n in enumerate(sizes):
        if n >= 3:
            usable = n - 1 if n >= 4 else n  # the last vertex of a mesh of >= 4 is in no face
            faces.append(torch.randint(0, usable, (2 * n, 3), generator=g) + first[i])
    faces = torch.cat(faces) if faces else torch.zeros((0, 3), dtype=torch.int64)
    Fn = faces.shape[0]
    verts = torch.randn(V, 3, generator=g)
    normals = torch.randn(V, 3, generator=g)
    for i, n in enumerate(sizes):
        if n >= 4:
            normals[first[i] + n - 1] = 0.0
    p2f = torch.randint(0, max(Fn, 1), (N, H, W, K), generator=g) if Fn else torch.full((N, H, W, K), -1)
    p2f[torch.rand(N, H, W, K, generator=g) < frac_background] = -1
    bary = torch.rand(N, H, W, K, 3, generator=g) + 0.05
    bary = bary / bary.sum(-1, keepdim=True)
    B = 1 if light_batch == 1 else N
    MB = 1 if material_batch == 1 else N
    where = torch.randn(B, 3, generator=g) * 2.0
    last = max(i for i, n in enumerate(sizes) if n > 0) if V else 0
    if V:
        where[min(last, B - 1)] = verts[first[last]]
    s = {
        "first": first, "num": torch.tensor(sizes, dtype=torch.int64), "faces": faces, "pix_to_face": p2f,
        "bary": bary, "verts": verts, "normals": normals, "colors": torch.rand(V, 3, generator=g),
        "light_ambient": 0.5 * torch.rand(B, 3, generator=g), "light_diffuse": torch.rand(B, 3, generator=g),
        "light_specular": torch.rand(B, 3, generator=g), "light_where": where,
        "material_ambient": torch.rand(MB, 3, generator=g), "material_diffuse": torch.rand(MB, 3, generator=g),
        "material_specular": torch.rand(MB, 3, generator=g), "shininess": torch.full((MB,), float(shininess)),
        "camera_center": torch.randn(B, 3, generator=g) * 3.0,
        "grad_colors": torch.randn(N, H, W, K, 3, generator=g),
    }
    return {k: v.to(device) for k, v in s.items()}


def scene_objects(s, kind, leaves):
    meshes = _Meshes(s, leaves)
    fragments = types.SimpleNamespace(pix_to_face=s["pix_to_face"], bary_coords=leaves["bary"])
    lights = types.SimpleNamespace(ambient_color=leaves["light_ambient"])
    if kind != "ambient":
        lights.diffuse_color, lights.specular_color = leaves["light_diffuse"], leaves["light_specular"]
        setattr(lights, "location" if kind == "point" else "direction", leaves["light_where"])
    cameras = types.SimpleNamespace(get_camera_center=lambda: leaves["camera_center"])
    materials = types.SimpleNamespace(ambient_color=leaves["material_ambient"], diffuse_color=leaves["material_diffuse"],
                                      specular_color=leaves["material_specular"], shininess=leaves["shininess"])
    return meshes, fragments, lights, cameras, materials


# ------------------------------------------------------------------------------------------------ golden scenes
# The scenes of tests/golden/make_gouraud_golden.py: every light kind with one mesh, with three meshes and batch-1
# properties, and with three meshes and batch-3 lights, materials and cameras; shininess 64, 10 and 0.
GOLDEN_CASES = [(kind, batch, SHININESS[(i + j) % 3], meshes) for i, kind in enumerate(("point", "directional", "ambient"))
                for j, (batch, meshes) in enumerate(((1, 1), (1, 3), ("N", 3)))]
GOLDEN_SIZES = {1: [26], 3: [20, 13, 27]}
GOLDEN_LEAVES = ("verts", "colors", "bary", "light_ambient", "light_diffuse", "light_specular", "light_where",
                 "material_ambient", "material_diffuse", "material_specular", "shininess", "R", "T")


def golden_case(args):
    return "gouraud/%s-%s-%g-%d" % args


def golden_scene(kind, batch, shininess, meshes, seed=0):
    """CPU tensors of one golden scene: meshes of GOLDEN_SIZES[meshes] vertices, random faces inside each mesh (its
    last vertex in none, so its normal is zero), 5 x 7 x 3 Fragments whose faces come from the image's own mesh with
    about 30 % background slots, a point light on a vertex, camera rotations R and translations T, and the upstream
    gradient."""
    sizes = GOLDEN_SIZES[meshes]
    g = torch.Generator().manual_seed(seed + 100 * meshes + 10 * SHININESS.index(shininess) + (batch != 1))
    N, H, W, K = meshes, 5, 7, 3
    first = [sum(sizes[:i]) for i in range(N)]
    faces, face_first, face_num = [], [], []
    for i, n in enumerate(sizes):
        face_first.append(sum(int(f.shape[0]) for f in faces))
        faces.append(torch.randint(0, n - 1, (2 * n, 3), generator=g))  # per-mesh indices
        face_num.append(2 * n)
    verts = torch.randn(sum(sizes), 3, generator=g)
    p2f = torch.empty(N, H, W, K, dtype=torch.int64)
    for i in range(N):
        p2f[i] = torch.randint(0, face_num[i], (H, W, K), generator=g) + face_first[i]
    p2f[torch.rand(N, H, W, K, generator=g) < 0.3] = -1
    bary = torch.rand(N, H, W, K, 3, generator=g) + 0.05
    B = 1 if batch == 1 else N
    where = torch.randn(B, 3, generator=g) * 2.0
    where[-1] = verts[first[-1]]  # a point light on a vertex
    q = F.normalize(torch.randn(B, 4, generator=g), dim=-1)
    w, x, y, z = q.unbind(-1)
    R = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
                     2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
                     2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], -1).view(B, 3, 3)
    return {
        "sizes": sizes, "faces": faces, "pix_to_face": p2f, "verts": verts,
        "colors": torch.rand(sum(sizes), 3, generator=g), "bary": bary / bary.sum(-1, keepdim=True),
        "light_ambient": 0.5 * torch.rand(B, 3, generator=g), "light_diffuse": torch.rand(B, 3, generator=g),
        "light_specular": torch.rand(B, 3, generator=g), "light_where": where,
        "material_ambient": torch.rand(B, 3, generator=g), "material_diffuse": torch.rand(B, 3, generator=g),
        "material_specular": torch.rand(B, 3, generator=g), "shininess": torch.full((B,), float(shininess)),
        "R": R, "T": torch.randn(B, 3, generator=g) * 2.0 + torch.tensor([0.0, 0.0, 4.0]),
        "grad_colors": torch.randn(N, H, W, K, 3, generator=g),
    }


def golden_leaves(s, device="cpu", dtype=torch.float32):
    return {k: s[k].to(device=device, dtype=dtype).clone().requires_grad_(True) for k in GOLDEN_LEAVES}


def camera_center(R, T):
    """The camera centre of world-to-view X R + T, formed as cameras.py's get_camera_center() forms it: the rotation
    composed with the translation is a plain Transform3d, whose inverse() inverts the rotation's 4 x 4 matrix with
    torch.inverse and negates the translation; the centre is the last row of I @ Translate^-1 @ Rotate^-1.  So the R
    gradient runs through a matrix inverse, not a transpose."""
    B = R.shape[0]
    rot = torch.cat([torch.cat([R, R.new_zeros(B, 3, 1)], 2), R.new_tensor([[[0.0, 0.0, 0.0, 1.0]]]).expand(B, 1, 4)], 1)
    tra = torch.eye(4, dtype=T.dtype, device=T.device).repeat(B, 1, 1)
    tra = torch.cat([tra[:, :3], torch.cat([T, T.new_ones(B, 1)], 1)[:, None]], 1)
    mask = T.new_ones(1, 4, 4)
    mask[0, 3, :3] = -1.0
    P = torch.eye(4, dtype=T.dtype, device=T.device).expand(B, 4, 4).bmm(tra * mask).bmm(torch.inverse(rot))
    return P[:, 3, :3]


def golden_objects(s, kind, leaves, center=None):
    """PackedMeshes with vertex colours, Fragments, lights, cameras (centre `center`, or camera_center(R, T)) and
    materials over `leaves`, on the leaves' device."""
    from pytorch3d_b200.structures import PackedMeshes
    dev = leaves["verts"].device
    bounds = [sum(s["sizes"][:i]) for i in range(len(s["sizes"]) + 1)]
    m = PackedMeshes([leaves["verts"][a:b] for a, b in zip(bounds[:-1], bounds[1:])], [f.to(dev) for f in s["faces"]])
    m.textures = types.SimpleNamespace(verts_features_packed=lambda: leaves["colors"])
    fragments = types.SimpleNamespace(pix_to_face=s["pix_to_face"].to(dev), bary_coords=leaves["bary"])
    lights = types.SimpleNamespace(ambient_color=leaves["light_ambient"])
    if kind != "ambient":
        lights.diffuse_color, lights.specular_color = leaves["light_diffuse"], leaves["light_specular"]
        setattr(lights, "location" if kind == "point" else "direction", leaves["light_where"])
    cameras = types.SimpleNamespace(
        get_camera_center=lambda: camera_center(leaves["R"], leaves["T"]) if center is None else center)
    materials = types.SimpleNamespace(ambient_color=leaves["material_ambient"], diffuse_color=leaves["material_diffuse"],
                                      specular_color=leaves["material_specular"], shininess=leaves["shininess"])
    return m, fragments, lights, cameras, materials


def golden_grads(fn, s, kind, device="cpu", dtype=torch.float32, center=None):
    """[(name, tensor)]: the colours, then the gradient of <colours, grad_colors> of every leaf that gets one."""
    leaves = golden_leaves(s, device, dtype)
    out = fn(*golden_objects(s, kind, leaves, center))
    (out * s["grad_colors"].to(device=device, dtype=dtype)).sum().backward()
    return [("colors", out.detach())] + [("grad_" + k, leaves[k].grad) for k in GOLDEN_LEAVES
                                         if leaves[k].grad is not None]


# ------------------------------------------------------------------------------------------------ restatement
def _interp(pix_to_face, bary, face_attrs):
    from test_shading import _interp as interp
    return interp(pix_to_face, bary, face_attrs)


def chain_gouraud(meshes, fragments, lights, cameras, materials):
    """The reference's gouraud_shading: with more than one mesh every batched property is gathered per vertex
    (gather_props keeps batch-1 properties), then _apply_lighting on (V, 3), the colour, the gather and the
    interpolation.  The camera centres are formed per mesh and gathered, where the reference forms them per vertex."""
    from pytorch3d_b200.shading import light_kind
    verts, faces = meshes.verts_packed(), meshes.faces_packed()
    colors = meshes.textures.verts_features_packed()
    V = verts.shape[0]
    idx = torch.repeat_interleave(torch.arange(len(meshes), device=verts.device), meshes.num_verts_per_mesh(),
                                  output_size=V)

    def gather(t):  # TensorProperties.gather_props: torch.gather of every property with batch > 1
        if len(meshes) == 1 or t.shape[0] == 1:
            return t
        return t.gather(0, idx.view((-1,) + (1,) * (t.dim() - 1)).expand((V,) + tuple(t.shape[1:])))

    kind = light_kind(lights)
    if kind == "ambient":
        light_diffuse = torch.zeros(V, 3, device=verts.device)
        light_specular = torch.zeros(V, 3, device=verts.device)
    else:
        # lighting.py's diffuse() and specular(), each forming its own light direction and normalising the normals, with
        # batch-1 properties expanded to the points first (convert_to_tensors_and_broadcast): the same graph, so the
        # same gradient summation order
        def expand(t):
            return t.expand((V,) + tuple(t.shape[1:])) if t.shape[0] == 1 else t

        where = gather(lights.location if kind == "point" else lights.direction)

        def direction():
            return where - verts if kind == "point" else where

        normals = meshes.verts_normals_packed()
        color, d = expand(gather(lights.diffuse_color)), expand(direction())
        nn, dn = F.normalize(normals, eps=1e-6, dim=-1), F.normalize(d, eps=1e-6, dim=-1)
        light_diffuse = color * F.relu(torch.sum(nn * dn, dim=-1))[..., None]
        color, d = expand(gather(lights.specular_color)), expand(direction())
        cam, shin = expand(gather(cameras.get_camera_center())), expand(gather(materials.shininess))
        nn, dn = F.normalize(normals, eps=1e-6, dim=-1), F.normalize(d, eps=1e-6, dim=-1)
        cos = torch.sum(nn * dn, dim=-1)
        mask = (cos > 0).to(nn.dtype)
        view = F.normalize(cam - verts, eps=1e-6, dim=-1)
        reflect = -dn + 2 * (cos[..., None] * nn)
        alpha = F.relu(torch.sum(view * reflect, dim=-1)) * mask
        light_specular = color * torch.pow(alpha, shin)[..., None]
    ambient = gather(materials.ambient_color) * gather(lights.ambient_color)
    diffuse = gather(materials.diffuse_color) * light_diffuse
    specular = gather(materials.specular_color) * light_specular
    shaded = colors * (ambient + diffuse) + specular
    return _interp(fragments.pix_to_face, fragments.bary_coords, shaded[faces])


def fused(meshes, fragments, lights, cameras, materials):
    from pytorch3d_b200.shading import gouraud_shading
    return gouraud_shading(meshes, fragments, lights, cameras, materials)


def with_grads(fn, s, kind, dtype=torch.float32, param_grads=True):
    """[(name, tensor)]: the colours, then the gradient of <colours, grad_colors> for every leaf that gets one."""
    names = LEAVES if param_grads else LEAVES[:4]
    leaves = {k: s[k].to(dtype).clone().requires_grad_(k in names) for k in LEAVES}
    out = fn(*scene_objects(s, kind, leaves))
    (out * s["grad_colors"].to(dtype)).sum().backward()
    return [("colors", out.detach())] + [("grad_" + k, leaves[k].grad) for k in names if leaves[k].grad is not None]


# ------------------------------------------------------------------------------------------------ CPU tests
def _recorded(case, field):
    """A whole stored array (the records keep every row of these small ones)."""
    from helpers import reference
    ref = reference(case + "/" + field)[0]
    assert len(ref.rows) == int(np.prod(ref.shape[:ref.lead])), "%s/%s is sampled, not whole" % (case, field)
    return torch.from_numpy(np.ascontiguousarray(ref.sample.reshape(ref.shape)))


@pytest.mark.parametrize("args", GOLDEN_CASES, ids=[golden_case(a)[8:] for a in GOLDEN_CASES])
def test_camera_centre_per_mesh_equals_the_references_per_vertex_one_cpu(args):
    """gouraud_shading forms the camera centre from the cameras gathered per vertex (V world-to-view transforms,
    inverted); the fused op forms it once per camera.  On these scenes the per-vertex centres equal the per-camera ones
    gathered, bit for bit, so forming the centre once per camera changes no bit.  camera_center() restates the
    reference's matrix chain; it agrees with the recorded centres to 1e-6, and the tests below feed the recorded centres
    to the bit-exact comparison and use camera_center() where the R and T gradients are compared with tolerances."""
    case = golden_case(args)
    mesh_c, vert_c = _recorded(case, "camera_center_mesh"), _recorded(case, "camera_center_vertex")
    s = golden_scene(*args)
    if vert_c.shape[0] == 1:
        assert torch.equal(vert_c, mesh_c)
    else:
        idx = torch.repeat_interleave(torch.arange(len(s["sizes"])), torch.tensor(s["sizes"]))
        assert torch.equal(vert_c, mesh_c[idx])
    np.testing.assert_allclose(camera_center(s["R"], s["T"]).numpy(), mesh_c.numpy(), rtol=1e-6, atol=1e-6)


@pytest.mark.parametrize("args", GOLDEN_CASES, ids=[golden_case(a)[8:] for a in GOLDEN_CASES])
def test_gouraud_chain_equals_reference_cpu(args):
    """The torch restatement, fed the recorded camera centres, equals the reference's colours and gradients bit for
    bit, except two gradients that several terms reach: the vertices (through the normals, the light direction and the
    view direction) and a light location or direction.  autograd adds those terms in an order this restatement does not
    reproduce, so they agree to 1e-6 of their largest magnitude (a few ulps).  The camera-centre gradient, summed per
    camera, equals the reference's per-vertex one summed the same way; the R and T gradients, through
    camera_center(), agree within rtol 1e-5."""
    from helpers import assert_equals_reference, reference
    kind = args[0]
    case = golden_case(args)
    s = golden_scene(*args)
    center = _recorded(case, "camera_center_mesh").clone().requires_grad_(True)
    got = golden_grads(chain_gouraud, s, kind, center=center)
    for name, t in got:
        if name in ("grad_R", "grad_T"):  # the centre is given: no gradient reaches R and T here
            continue
        if name in ("grad_verts", "grad_light_where"):
            ref = reference(case + "/" + name)[0]
            np.testing.assert_allclose(ref.rows_of(t), ref.sample, rtol=0, atol=1e-6 * ref.absmax, err_msg=name)
        else:
            assert_equals_reference([t], case + "/" + name, "torch restatement vs the reference (CPU)")
    if kind != "ambient":
        want = _recorded(case, "grad_camera_center_vertex")
        if want.shape[0] != center.shape[0]:
            idx = torch.repeat_interleave(torch.arange(len(s["sizes"])), torch.tensor(s["sizes"]))
            want = torch.zeros_like(center).index_put_((idx,), want, accumulate=True)
        assert torch.equal(center.grad, want)
        rt = dict(golden_grads(chain_gouraud, s, kind))
        for name in ("grad_R", "grad_T"):
            ref = _recorded(case, name)
            np.testing.assert_allclose(rt[name].numpy(), ref.numpy(), rtol=1e-5, atol=1e-6 * float(ref.abs().max()),
                                       err_msg=name)


def test_packed_meshes_vertex_accessors():
    from pytorch3d_b200.structures import PackedMeshes
    verts = [torch.zeros(5, 3), torch.zeros(0, 3), torch.zeros(4, 3)]
    faces = [torch.zeros(2, 3, dtype=torch.int64), torch.zeros(0, 3, dtype=torch.int64),
             torch.zeros(1, 3, dtype=torch.int64)]
    m = PackedMeshes(verts, faces)
    assert m.num_verts_per_mesh().tolist() == [5, 0, 4]
    assert m.mesh_to_verts_packed_first_idx().tolist() == [0, 5, 5]
    assert m.num_verts_per_mesh().dtype == torch.int64 == m.mesh_to_verts_packed_first_idx().dtype


def test_gouraud_argument_errors(built_lib):
    from pytorch3d_b200 import _C
    from pytorch3d_b200.shading import gouraud_shading
    s = gouraud_scene([5, 4], 2, 3, 2)
    meshes, frags, lights, cameras, mats = scene_objects(s, "point", s)
    meshes.textures = types.SimpleNamespace()
    with pytest.raises(ValueError, match="Mesh textures must be an instance of TexturesVertex"):
        gouraud_shading(meshes, frags, lights, cameras, mats)
    meshes.textures = types.SimpleNamespace(verts_features_packed=lambda: torch.rand(9, 1))
    with pytest.raises(ValueError, match=r"\(V, 3\)"):
        gouraud_shading(meshes, frags, lights, cameras, mats)
    params = torch.zeros(2, _C.SHADING_PARAMS)
    args = [s["verts"], s["normals"], s["colors"], s["first"], s["num"], params, s["faces"], s["pix_to_face"], s["bary"],
            "point"]
    with pytest.raises(RuntimeError, match="must be a CUDA tensor"):
        _C.gouraud_forward(*args)
    with pytest.raises(RuntimeError, match="light must be one of"):
        _C.gouraud_forward(*args[:-1], "spot")
    with pytest.raises(RuntimeError, match="normals are required"):
        _C.gouraud_forward(args[0], None, *args[2:])


def _fake_pytorch3d(monkeypatch):
    from test_shading import _Lights
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

    class TexturesVertex:
        def __init__(self, feats):
            self._f = feats

        def verts_features_packed(self):
            return self._f

    lighting.PointLights, lighting.DirectionalLights, lighting.AmbientLights = PointLights, DirectionalLights, AmbientLights
    materials = types.ModuleType("pytorch3d.renderer.materials")
    materials.Materials = Materials
    textures = types.ModuleType("pytorch3d.renderer.mesh.textures")
    textures.TexturesVertex = TexturesVertex
    for n in ["pytorch3d", "pytorch3d.renderer", "pytorch3d.renderer.mesh", "pytorch3d.renderer.mesh.shading",
              "pytorch3d.renderer.mesh.shader"]:
        m = types.ModuleType(n)
        m.__path__ = []
        monkeypatch.setitem(sys.modules, n, m)
    monkeypatch.setitem(sys.modules, "pytorch3d.renderer.lighting", lighting)
    monkeypatch.setitem(sys.modules, "pytorch3d.renderer.materials", materials)
    monkeypatch.setitem(sys.modules, "pytorch3d.renderer.mesh.textures", textures)

    def ref(meshes, fragments, lights, cameras, materials):
        calls.append("gouraud_shading")
        return "ref"

    for n in ("pytorch3d.renderer.mesh.shading", "pytorch3d.renderer.mesh.shader"):
        sys.modules[n].gouraud_shading = ref
    return types.SimpleNamespace(PointLights=PointLights, DirectionalLights=DirectionalLights,
                                 AmbientLights=AmbientLights, Materials=Materials, TexturesVertex=TexturesVertex), ref, calls


class _FakeMeshes:
    def __init__(self, n, verts, textures):
        self._n, self._v, self.textures = n, verts, textures

    def __len__(self):
        return self._n

    def verts_packed(self):
        return self._v


def test_install_gouraud_and_uninstall(monkeypatch, built_lib):
    from pytorch3d_b200 import install as inst
    from pytorch3d_b200 import shading as ours
    cls, original, calls = _fake_pytorch3d(monkeypatch)
    patched = inst.install_gouraud()
    assert patched == ["pytorch3d.renderer.mesh.shading", "pytorch3d.renderer.mesh.shader"]
    routed = []
    monkeypatch.setattr(ours, "gouraud_shading", lambda *a: routed.append(1) or "b200")
    sh = sys.modules["pytorch3d.renderer.mesh.shader"]
    for modname in patched:
        assert sys.modules[modname].gouraud_shading is not original
    c3, c2 = torch.ones(1, 3), torch.ones(2, 3)
    mats = cls.Materials(ambient_color=c3, diffuse_color=c2, specular_color=c2, shininess=torch.ones(2))
    point = cls.PointLights(ambient_color=c3, diffuse_color=c3, specular_color=c3, location=c2)
    verts = _stand_in((10, 3))
    feats = _stand_in((10, 3))
    verts.device = feats.device = "cuda:0"
    bary = _stand_in((2, 2, 3, 4, 3))
    p2f = _stand_in((2, 2, 3, 4), torch.int64)
    bary.device = p2f.device = "cuda:0"
    frags = types.SimpleNamespace(pix_to_face=p2f, bary_coords=bary)
    meshes = _FakeMeshes(2, verts, cls.TexturesVertex(feats))
    cams = types.SimpleNamespace(R=torch.eye(3).expand(2, 3, 3), T=torch.zeros(2, 3))
    assert sh.gouraud_shading(meshes, frags, point, cams, mats) == "b200"
    amb = cls.AmbientLights(ambient_color=c3)
    assert sys.modules["pytorch3d.renderer.mesh.shading"].gouraud_shading(meshes, frags, amb, cams, mats) == "b200"
    dirl = cls.DirectionalLights(ambient_color=c3, diffuse_color=c3, specular_color=c3, direction=c3)
    assert sh.gouraud_shading(meshes, frags, dirl, cams, mats) == "b200"
    assert calls == []
    # everything else keeps the original

    class MyLights(cls.PointLights):
        pass

    mine = MyLights(ambient_color=c3, diffuse_color=c3, specular_color=c3, location=c3)
    assert sh.gouraud_shading(meshes, frags, mine, cams, mats) == "ref"
    one = _stand_in((10, 1))
    one.device = "cuda:0"
    assert sh.gouraud_shading(_FakeMeshes(2, verts, cls.TexturesVertex(one)), frags, point, cams, mats) == "ref"
    other = types.SimpleNamespace(verts_features_packed=lambda: feats)  # not a TexturesVertex
    assert sh.gouraud_shading(_FakeMeshes(2, verts, other), frags, point, cams, mats) == "ref"
    cpu = _stand_in((10, 3), is_cuda=False)
    cpu.device = "cpu"
    assert sh.gouraud_shading(_FakeMeshes(2, cpu, cls.TexturesVertex(feats)), frags, point, cams, mats) == "ref"
    f64 = _stand_in((10, 3), torch.float64)
    f64.device = "cuda:0"
    assert sh.gouraud_shading(_FakeMeshes(2, verts, cls.TexturesVertex(f64)), frags, point, cams, mats) == "ref"
    three = cls.PointLights(ambient_color=c3, diffuse_color=c3, specular_color=c3, location=torch.ones(3, 3))
    assert sh.gouraud_shading(meshes, frags, three, cams, mats) == "ref"
    cams3 = types.SimpleNamespace(R=torch.eye(3).expand(3, 3, 3), T=torch.zeros(3, 3))  # a batch the kernels lack
    assert sh.gouraud_shading(meshes, frags, point, cams3, mats) == "ref"
    assert len(calls) == 7 and len(routed) == 3
    inst.uninstall()
    for modname in patched:
        assert sys.modules[modname].gouraud_shading is original
    assert inst._saved_blend == {}


def test_install_gouraud_leaves_the_other_installs_alone(monkeypatch, built_lib):
    from pytorch3d_b200 import install as inst
    _fake_pytorch3d(monkeypatch)
    inst.install_gouraud()
    try:
        assert set(inst._saved_blend) == {(m, "gouraud_shading") for m in inst._SHADING_MODULES}
        assert inst._saved == {} and inst._saved_methods == {}
    finally:
        inst.uninstall()
    assert inst._saved_blend == {}
    assert "gouraud_shading" not in inst._SHADING_FUNCTIONS  # install_shading() patches what it always did


# ------------------------------------------------------------------------------------------------ GPU tests
@pytest.mark.gpu
@pytest.mark.parametrize("args", GOLDEN_CASES, ids=[golden_case(a)[8:] for a in GOLDEN_CASES])
def test_fused_matches_reference_records(built_lib, args):
    """The fused op, with the camera centre formed from R and T requiring grad, against the reference's records:
    forward rtol 1e-5 / atol 1e-6, gradients rtol 1e-4 / atol 1e-5 of the largest magnitude, and for shininess >= 64
    an error against the float64 chain of at most twice the float32 chain's own."""
    from helpers import reference
    kind, _, shininess, _ = args
    s = golden_scene(*args)
    got = dict(golden_grads(fused, s, kind, device=DEV))
    want = dict(golden_grads(chain_gouraud, s, kind))
    f64 = dict(golden_grads(chain_gouraud, s, kind, dtype=torch.float64))
    assert set(want) <= set(got), "fields %s vs the chain's %s" % (sorted(got), sorted(want))
    for name in got:
        if name not in want:  # the reference's graph does not reach this input: the fused op gives exact zeros
            assert not got[name].any(), name
            continue
        ref = reference(golden_case(args) + "/" + name)[0]
        mine = ref.rows_of(got[name])
        rtol, atol = (1e-5, 1e-6) if name == "colors" else (1e-4, 1e-5 * max(ref.absmax, 1e-30))
        if not np.all(np.abs(mine - ref.sample) <= atol + rtol * np.abs(ref.sample)):
            assert shininess >= 64, "%s %s: max abs diff %g" % (args, name, float(np.abs(mine - ref.sample).max()))
            d64 = f64[name].detach().numpy()
            err = float(np.abs(got[name].detach().cpu().double().numpy() - d64).max())
            own = float(np.abs(want[name].detach().double().numpy() - d64).max())
            assert err <= 2.0 * own, "%s %s: error %g against float64, the float32 chain's %g" % (args, name, err, own)


def _compare(s, kind, what, param_grads=True):
    got = with_grads(fused, s, kind, param_grads=param_grads)
    want = with_grads(chain_gouraud, s, kind, param_grads=param_grads)
    f64 = None
    if float(s["shininess"][0]) >= 64:
        f64 = with_grads(chain_gouraud, {k: v.cpu() for k, v in s.items()}, kind, torch.float64, param_grads)
    _tol_check(got, want, what, f64, want if f64 is not None else None)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,batch,shininess,meshes", CASES)
def test_fused_matches_torch_chain_every_light(built_lib, kind, batch, shininess, meshes):
    sizes = [40] if meshes == 1 else [40, 17, 29]
    s = gouraud_scene(sizes, 6, 9, 3, batch, shininess, seed=1, device=DEV, material_batch=batch)
    _compare(s, kind, "%s-%s-%g-%d" % (kind, batch, shininess, meshes))


@pytest.mark.gpu
@pytest.mark.parametrize("K", [1, 2, 50, 200])
def test_fused_matches_torch_chain_for_K(built_lib, K):
    s = gouraud_scene([30, 12], 5, 4, K, "N", 10.0, seed=2, device=DEV)
    _compare(s, "point", "K=%d" % K)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(1, 1, 1), (1, 1, 5), (3, 1, 2), (17, 33, 3)])
def test_fused_matches_torch_chain_on_odd_sizes(built_lib, shape):
    s = gouraud_scene([9, 7], *shape, 1, 10.0, seed=3, device=DEV)
    _compare(s, "directional", "shape %r" % (shape,))


@pytest.mark.gpu
def test_heterogeneous_meshes_with_an_empty_mesh(built_lib):
    s = gouraud_scene([300, 0, 5, 1000], 8, 8, 4, "N", 10.0, seed=4, device=DEV, material_batch="N")
    _compare(s, "point", "heterogeneous")
    got = dict(with_grads(fused, s, "point"))
    assert not got["grad_light_where"][1].any() and not got["grad_camera_center"][1].any()  # the empty mesh


@pytest.mark.gpu
def test_without_parameter_gradients(built_lib):
    s = gouraud_scene([40, 17], 6, 9, 3, "N", 10.0, seed=5, device=DEV)
    _compare(s, "point", "no param grads", param_grads=False)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["point", "directional", "ambient"])
def test_colors_and_grad_bary_equal_interp_face_attrs_bit_for_bit(built_lib, kind):
    from pytorch3d_b200 import _C
    from pytorch3d_b200.shading import _params
    s = gouraud_scene([50, 31], 7, 5, 4, "N", 10.0, seed=6, device=DEV)
    meshes, frags, lights, cameras, mats = scene_objects(s, kind, s)
    params = _params(2, lights, cameras, mats, kind, DEV, batched_material_colors=True)
    normals = None if kind == "ambient" else s["normals"]
    colors, shaded = _C.gouraud_forward(s["verts"], normals, s["colors"], s["first"], s["num"], params, s["faces"],
                                        s["pix_to_face"], s["bary"], kind)
    face_colors = shaded[s["faces"]].contiguous()
    p2f, bary = s["pix_to_face"].view(-1), s["bary"].view(-1, 3)  # pytorch3d._C takes (P,) and (P, 3)
    assert torch.equal(colors.view(-1, 3), _C.interp_face_attrs_forward(p2f, bary, face_colors))
    g_bary = _C.gouraud_backward(s["grad_colors"], s["verts"], normals, s["colors"], s["first"], s["num"], params,
                                 s["faces"], s["pix_to_face"], s["bary"], kind, shaded,
                                 (False, False, False, True, False))[3]
    want = _C.interp_face_attrs_backward(p2f, bary, face_colors, s["grad_colors"].view(-1, 3))[0]
    assert torch.equal(g_bary, want.view_as(g_bary))
    # verts_shaded against the float32 chain
    want_shaded = chain_gouraud_shaded(s, kind, params)
    np.testing.assert_allclose(shaded.cpu().numpy(), want_shaded.cpu().numpy(), rtol=1e-5, atol=1e-6)


def chain_gouraud_shaded(s, kind, params):
    """verts_shaded of the chain: the interpolation of the chain with one-hot barycentrics at every vertex."""
    V = s["verts"].shape[0]
    _, _, lights, cameras, mats = scene_objects(s, kind, s)
    s2 = dict(s)  # one face (v, v, v) per vertex, hit once with barycentrics (1, 0, 0)
    s2["faces"] = torch.arange(V, device=DEV)[:, None].expand(V, 3).contiguous()
    s2["pix_to_face"] = torch.arange(V, device=DEV).view(1, V, 1, 1)
    meshes2 = _Meshes(s2, s)
    frags2 = types.SimpleNamespace(pix_to_face=s2["pix_to_face"],
                                   bary_coords=torch.tensor([1.0, 0.0, 0.0], device=DEV).expand(1, V, 1, 1, 3))
    return chain_gouraud(meshes2, frags2, lights, cameras, mats).view(V, 3)


@pytest.mark.gpu
def test_unaligned_inputs_give_identical_bits(built_lib):
    s = gouraud_scene([40, 17, 29], 6, 9, 3, "N", 10.0, seed=7, device=DEV)

    def shifted(t):
        buf = torch.empty(t.numel() + 1, dtype=t.dtype, device=t.device)
        out = buf[1:].view(t.shape)
        out.copy_(t)
        return out

    s2 = {k: shifted(v) if v.dtype == torch.float32 and v.dim() > 0 else v for k, v in s.items()}
    a, b = with_grads(fused, s, "point"), with_grads(fused, s2, "point")
    for (name, x), (_, y) in zip(a, b):
        if name in ("colors", "grad_bary"):
            assert torch.equal(x, y), name
        else:
            np.testing.assert_allclose(x.cpu().numpy(), y.cpu().numpy(), rtol=1e-5,
                                       atol=1e-6 * float(y.abs().max()) + 1e-30, err_msg=name)


@pytest.mark.gpu
def test_no_host_sync_and_reproducible(built_lib):
    s = gouraud_scene([400, 130, 270], 33, 17, 8, "N", 64.0, seed=8, device=DEV)

    def run():
        return with_grads(fused, s, "point")

    run()  # warm-up outside the checked region
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        first = run()
        second = run()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    for (name, a), (_, b) in zip(first, second):
        if name in ("colors", "grad_bary"):
            assert torch.equal(a, b), name
        else:  # downstream of the atomically accumulated gradient of the shaded vertex colours
            np.testing.assert_allclose(a.cpu().numpy(), b.cpu().numpy(), rtol=1e-5,
                                       atol=1e-6 * float(b.abs().max()) + 1e-30, err_msg=name)


@pytest.mark.gpu
def test_verts_shaded_is_reproducible(built_lib):
    from pytorch3d_b200 import _C
    from pytorch3d_b200.shading import _params
    s = gouraud_scene([400, 130], 9, 9, 4, "N", 10.0, seed=9, device=DEV)
    _, _, lights, cameras, mats = scene_objects(s, "point", s)
    params = _params(2, lights, cameras, mats, "point", DEV)
    a = _C.gouraud_forward(s["verts"], s["normals"], s["colors"], s["first"], s["num"], params, s["faces"],
                           s["pix_to_face"], s["bary"], "point")
    b = _C.gouraud_forward(s["verts"], s["normals"], s["colors"], s["first"], s["num"], params, s["faces"],
                           s["pix_to_face"], s["bary"], "point")
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


@pytest.mark.gpu
def test_deterministic_mode_raises_for_vertex_gradients(built_lib):
    s = gouraud_scene([40, 17], 6, 9, 3, 1, 10.0, seed=10, device=DEV)
    was = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        with pytest.raises(RuntimeError, match="deterministic"):
            with_grads(fused, s, "point")
        # barycentric-only backward stays allowed
        leaves = {k: s[k].clone().requires_grad_(k == "bary") for k in LEAVES}
        out = fused(*scene_objects(s, "point", leaves))
        (out * s["grad_colors"]).sum().backward()
        assert leaves["bary"].grad is not None
    finally:
        torch.use_deterministic_algorithms(was)


def _torus_gouraud_pipeline(shade):
    """Rasterize a torus batch, shade it per vertex with `shade`, blend with the fused softmax blend, take a loss and
    return the image and the gradients of the vertices, vertex colours and light location."""
    from pytorch3d_b200 import synthetic
    from pytorch3d_b200.blending import BlendParams, softmax_rgb_blend
    from pytorch3d_b200.rasterize_meshes import rasterize_meshes
    m = synthetic.torus_batch(2, 24, 24, seed=1, device=DEV)
    m.requires_grad_(True)
    V = m.verts_packed().shape[0]
    colors = torch.rand(V, 3, generator=torch.Generator().manual_seed(5)).to(DEV).requires_grad_(True)
    m.textures = types.SimpleNamespace(verts_features_packed=lambda: colors)
    location = torch.tensor([[0.5, 1.0, -1.0]], device=DEV, requires_grad=True)
    lights = types.SimpleNamespace(ambient_color=torch.tensor([[0.3, 0.3, 0.3]], device=DEV),
                                   diffuse_color=torch.tensor([[0.6, 0.5, 0.4]], device=DEV),
                                   specular_color=torch.tensor([[0.3, 0.3, 0.3]], device=DEV), location=location)
    cameras = types.SimpleNamespace(get_camera_center=lambda: torch.zeros(1, 3, device=DEV))
    materials = types.SimpleNamespace(ambient_color=torch.ones(1, 3, device=DEV),
                                      diffuse_color=torch.ones(1, 3, device=DEV),
                                      specular_color=torch.ones(1, 3, device=DEV),
                                      shininess=torch.tensor([64.0], device=DEV))
    H, W = 48, 80
    p2f, zbuf, bary, dists = rasterize_meshes(m, (H, W), blur_radius=1e-4, faces_per_pixel=4)
    frags = types.SimpleNamespace(pix_to_face=p2f, bary_coords=bary, zbuf=zbuf, dists=dists)
    img = softmax_rgb_blend(shade(m, frags, lights, cameras, materials), frags, BlendParams(sigma=1e-4, gamma=1e-4))
    w = torch.rand(img.shape, generator=torch.Generator().manual_seed(6)).to(DEV)
    (img * w).sum().backward()
    return img.detach(), m.verts_packed().grad, colors.grad, location.grad


@pytest.mark.gpu
def test_end_to_end_gouraud_softmax_matches_torch_chain(built_lib):
    got = _torus_gouraud_pipeline(fused)
    want = _torus_gouraud_pipeline(chain_gouraud)
    np.testing.assert_allclose(got[0].cpu().numpy(), want[0].cpu().numpy(), rtol=1e-5, atol=1e-6)
    for name, g, r in zip(("verts", "colors", "location"), got[1:], want[1:]):
        assert float(r.abs().max()) > 0, name
        np.testing.assert_allclose(g.cpu().numpy(), r.cpu().numpy(), rtol=1e-4, atol=1e-5 * float(r.abs().max()),
                                   err_msg=name)
