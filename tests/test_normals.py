"""Mesh normals on the GPU (DESIGN.md section 17): `pytorch3d_b200.normals`, `_C.face_areas_normals_forward/_backward`,
`_C.verts_normals_forward/_backward` and `install_normals()`.

The reference records (tests/golden/make_normals_golden.py) come from the reference's own `Meshes` on the CPU
(reference_golden_normals.npz) and from its CUDA face op built for sm_90a (reference_golden_normals_cuda.npz), on the
seeded scenes below.
"""
import math
import sys
import types

import numpy as np
import pytest
import torch

from helpers import assert_equals_reference, reference

DEV = "cuda"

SCENES = ("torus_hetero", "ico_sphere", "isolated", "degenerate", "cancelling", "fan")


def _from_lists(verts_list, faces_list):
    nverts = [int(v.shape[0]) for v in verts_list]
    offs = np.cumsum([0] + nverts[:-1]).tolist()
    return {"verts": torch.cat(verts_list).to(torch.float32).contiguous(),
            "faces": torch.cat([f + o for f, o in zip(faces_list, offs)]).to(torch.int64).contiguous(),
            "faces_list": [f.to(torch.int64) for f in faces_list], "nverts": nverts}


def scene(name):
    """{verts (V,3) f32 packed, faces (F,3) i64 packed, faces_list (per-mesh local faces), nverts}."""
    from pytorch3d_b200 import synthetic
    g = torch.Generator().manual_seed(SCENES.index(name) + 17)
    if name == "torus_hetero":  # a batch of unequal sizes
        m = synthetic.torus_batch_hetero([150, 400, 900], seed=5)
        nv = m.num_verts_per_mesh().tolist()
        nf = m.num_faces_per_mesh().tolist()
        vl = list(torch.split(m.verts_packed(), nv))
        fl = [f - o for f, o in zip(torch.split(m.faces_packed(), nf), m.mesh_to_verts_packed_first_idx().tolist())]
        return _from_lists(vl, fl)
    if name == "ico_sphere":  # closed
        v, f = synthetic.ico_sphere(3)
        return _from_lists([v * 0.7 + torch.tensor([0.1, -0.2, 2.0])], [f])
    if name == "isolated":  # vertices 0 and V-1 are in no face
        v, f = synthetic.torus(8, 6)
        v = torch.cat([torch.tensor([[0.5, 0.5, 0.5]]), v.to(torch.float32), torch.tensor([[-1.0, 2.0, 0.0]])])
        return _from_lists([v], [f + 1])
    if name == "degenerate":  # collinear corners, a repeated index, a zero-length edge
        v = torch.randn(12, 3, generator=g)
        v[2] = 0.25 * v[0] + 0.75 * v[1]  # collinear with 0 and 1
        v[8] = v[7]
        f = torch.tensor([[0, 1, 2], [3, 3, 5], [4, 5, 6], [6, 7, 8], [9, 10, 11], [2, 9, 4], [5, 3, 10], [11, 1, 0]])
        return _from_lists([v], [f])
    if name == "cancelling":
        # a0..a2: two faces of opposite orientation with integer coordinates (exact products), so the sum is exactly 0
        # at each of them; b0..b3: [b0, b2, b3] is [b0, b1, b2] reversed up to 3e-7, so |s| < 1e-6 at b0 and b2
        a = torch.tensor([[0.0, 0.0, 1.0], [1.0, 0.0, 1.0], [0.0, 1.0, 2.0]])
        b = torch.tensor([[2.0, 0.0, 0.0], [3.0, 0.1, 0.3], [2.2, 1.0, 0.1], [3.0, 0.1, 0.3 + 3e-7]])
        v = torch.cat([a, b, torch.randn(3, 3, generator=g)])
        f = torch.tensor([[0, 1, 2], [0, 2, 1], [3, 4, 5], [3, 5, 6], [7, 8, 9], [9, 8, 6]])
        return _from_lists([v], [f])
    if name == "fan":  # vertex 0 is in 3000 faces
        n = 3000
        t = torch.arange(n, dtype=torch.float64) * (2 * math.pi / n)
        ring = torch.stack([torch.cos(t), torch.sin(t), 0.05 * torch.randn(n, generator=g, dtype=torch.float64)], 1)
        v = torch.cat([torch.tensor([[0.0, 0.0, 0.3]], dtype=torch.float64), ring]).to(torch.float32)
        i = torch.arange(1, n + 1)
        f = torch.stack([torch.zeros_like(i), i, i % n + 1], 1)
        return _from_lists([v], [f])
    raise KeyError(name)


def upstream_grads(s):
    g = torch.Generator().manual_seed(int(s["verts"].shape[0]) * 7 + int(s["faces"].shape[0]))
    V, F = int(s["verts"].shape[0]), int(s["faces"].shape[0])
    return {"verts_normals": torch.randn(V, 3, generator=g), "faces_areas": torch.randn(F, generator=g),
            "faces_normals": torch.randn(F, 3, generator=g)}


def chain_verts_normals(verts, faces):
    """The reference's vertex-normal chain (Meshes._compute_vertex_normals), restated by PackedMeshes."""
    from pytorch3d_b200.structures import PackedMeshes
    return PackedMeshes([verts], [faces]).verts_normals_packed()


def _corner_counts(faces, V):
    return np.bincount(faces.reshape(-1).numpy(), minlength=V)


def _close(got, want, rtol, atol, what):
    got, want = got.detach().double().cpu(), want.detach().double().cpu()
    scale = max(float(want.abs().max()) if want.numel() else 0.0, 1e-30)
    err = (got - want).abs()
    bound = atol * scale + rtol * scale
    assert not torch.isnan(got[~torch.isnan(want)]).any(), "%s: NaN where the reference has none" % what
    assert float(err[~torch.isnan(want)].max()) <= bound if err.numel() else True, \
        "%s: max abs error %g > %g" % (what, float(err.max()), bound)


# ---------------------------------------------------------------------------------------------------------- CPU ---

@pytest.mark.parametrize("name", SCENES)
def test_restatement_equals_reference_records_cpu(name):
    """The torch restatement (PackedMeshes.verts_normals_packed) equals the reference's Meshes bit for bit, normals and
    vertex gradients."""
    s = scene(name)
    leaf = s["verts"].clone().requires_grad_(True)
    n = chain_verts_normals(leaf, s["faces"])
    (n * upstream_grads(s)["verts_normals"]).sum().backward()
    assert_equals_reference([n.detach()], "normals/%s/verts_normals" % name, "restatement")
    assert_equals_reference([leaf.grad], "normals/%s/grad_verts_normals" % name, "restatement's gradient")


def test_scenes_cover_the_special_cases():
    iso = scene("isolated")
    counts = _corner_counts(iso["faces"], iso["verts"].shape[0])
    assert counts[0] == 0 and counts[-1] == 0
    deg = scene("degenerate")
    assert [3, 3, 5] in deg["faces"].tolist()
    with torch.no_grad():
        c = scene("cancelling")
        s = torch.zeros_like(c["verts"])
        corners = c["verts"][c["faces"]]
        n = torch.cross(corners[:, 2] - corners[:, 1], corners[:, 0] - corners[:, 1], dim=1)
        for j in range(3):
            s = s.index_add(0, c["faces"][:, j], n)
        norms = s.norm(dim=1)
    assert float(norms[0]) == 0.0 and 0.0 < float(norms[3]) < 1e-6
    fan = scene("fan")
    assert _corner_counts(fan["faces"], fan["verts"].shape[0])[0] == 3000
    assert len(scene("torus_hetero")["nverts"]) == 3


def test_key_bits_and_table_size():
    from pytorch3d_b200 import _C
    assert [_C.normals_key_bits(v) for v in (0, 1, 2, 3, 4, 7, 8, 2 ** 31 - 2)] == [1, 1, 2, 2, 3, 3, 4, 31]
    for V in (1, 5, 1000, 2 ** 20):  # vertex ids and the key V all fit, one bit less would not fit V
        bits = _C.normals_key_bits(V)
        assert V < 2 ** bits and (bits == 1 or V >= 2 ** (bits - 1))
    assert _C.normals_table_size(10, 4) == 11 + 12


def test_argument_errors_cpu():
    from pytorch3d_b200 import _C, normals
    v, f = torch.rand(4, 3), torch.tensor([[0, 1, 2]])
    for fn in (_C.face_areas_normals_forward, _C.verts_normals_forward):
        with pytest.raises(RuntimeError, match="CUDA"):
            fn(v, f)
    with pytest.raises(ValueError, match="Vx3"):
        normals.face_areas_normals(torch.rand(4, 2), f)
    with pytest.raises(ValueError, match="Fx3"):
        normals.face_areas_normals(v, torch.tensor([[0, 1]]))
    with pytest.raises(ValueError, match="int64"):
        normals.face_areas_normals(v, f.int())


def _stand_in(shape, dtype=torch.float32, is_cuda=True, device=None):
    device = torch.device(device or ("cuda:0" if is_cuda else "cpu"))
    return types.SimpleNamespace(is_cuda=is_cuda, dtype=dtype, shape=torch.Size(shape), dim=lambda: len(shape),
                                 device=device)


def _fake_normals_modules(monkeypatch):
    """Stand-ins for pytorch3d.ops.mesh_face_areas_normals (with a `_C`) and pytorch3d.structures.meshes (with a `Meshes`
    whose `_compute_vertex_normals` has the reference's caching)."""
    for n in ["pytorch3d", "pytorch3d.ops", "pytorch3d.structures", "pytorch3d.renderer", "pytorch3d.renderer.mesh"]:
        m = types.ModuleType(n)
        m.__path__ = []
        monkeypatch.setitem(sys.modules, n, m)
    ops = types.ModuleType("pytorch3d.ops.mesh_face_areas_normals")
    ops._C = types.SimpleNamespace(face_areas_normals_forward=lambda *a: "ref-fwd",
                                   face_areas_normals_backward=lambda *a: "ref-bwd", other_op=lambda: "other")
    monkeypatch.setitem(sys.modules, ops.__name__, ops)
    meshes = types.ModuleType("pytorch3d.structures.meshes")

    class Meshes:
        def __init__(self, verts, faces, empty=False):
            self._verts, self._faces, self._empty = verts, faces, empty
            self._verts_normals_packed = None
            self.original_calls = 0

        def isempty(self):
            return self._empty

        def verts_packed(self):
            return self._verts

        def faces_packed(self):
            return self._faces

        def _compute_vertex_normals(self, refresh=False):
            if not (refresh or any(v is None for v in [self._verts_normals_packed])):
                return
            self.original_calls += 1
            self._verts_normals_packed = "ref-normals"

        def verts_normals_packed(self):
            self._compute_vertex_normals()
            return self._verts_normals_packed

        def offset_verts_(self, new_verts):  # what the reference does when normals were cached
            self._verts = new_verts
            if self._verts_normals_packed is not None:
                self._compute_vertex_normals(refresh=True)
            return self

    meshes.Meshes = Meshes
    monkeypatch.setitem(sys.modules, meshes.__name__, meshes)
    return ops, Meshes


def test_install_normals_routing_and_uninstall(monkeypatch, built_lib):
    from pytorch3d_b200 import _C as b200_C
    from pytorch3d_b200 import install as inst
    from pytorch3d_b200 import normals as ours
    ops, Meshes = _fake_normals_modules(monkeypatch)
    original_C, original_method = ops._C, Meshes.__dict__["_compute_vertex_normals"]
    monkeypatch.setattr(b200_C, "face_areas_normals_forward", lambda *a: "b200-fwd")
    monkeypatch.setattr(b200_C, "face_areas_normals_backward", lambda *a: "b200-bwd")
    fused = []
    monkeypatch.setattr(ours, "verts_normals", lambda v, f: fused.append((v, f)) or "b200-normals-%d" % len(fused))
    assert inst.install_normals() == ["pytorch3d.ops.mesh_face_areas_normals", "pytorch3d.structures.meshes"]
    v, f = _stand_in((10, 3)), _stand_in((4, 3), torch.int64)
    g_a, g_n = _stand_in((4,)), _stand_in((4, 3))
    assert ops._C.face_areas_normals_forward(v, f) == "b200-fwd"
    assert ops._C.face_areas_normals_backward(g_a, g_n, v, f) == "b200-bwd"
    assert ops._C.other_op() == "other"
    for vv, ff in ((_stand_in((10, 3), is_cuda=False), _stand_in((4, 3), torch.int64, is_cuda=False)),
                   (_stand_in((10, 3), torch.float64), f), (v, _stand_in((4, 3), torch.int32)),
                   (v, _stand_in((4, 3), torch.int64, device="cuda:1"))):
        assert ops._C.face_areas_normals_forward(vv, ff) == "ref-fwd"
        assert ops._C.face_areas_normals_backward(g_a, g_n, vv, ff) == "ref-bwd"
    # vertex normals: the fused op, cached; refresh recomputes; offset_verts_ recomputes only when cached
    m = Meshes(v, f)
    assert m.verts_normals_packed() == "b200-normals-1" and m.verts_normals_packed() == "b200-normals-1"
    m._compute_vertex_normals(refresh=True)
    assert m._verts_normals_packed == "b200-normals-2"
    v2 = _stand_in((10, 3))
    m.offset_verts_(v2)
    assert m._verts_normals_packed == "b200-normals-3" and fused[-1] == (v2, f)
    fresh = Meshes(v, f)
    fresh.offset_verts_(v2)
    assert fresh._verts_normals_packed is None and len(fused) == 3
    for mm in (Meshes(v, f, empty=True), Meshes(_stand_in((10, 3), is_cuda=False), f),
               Meshes(_stand_in((10, 3), torch.float64), f), Meshes(v, _stand_in((4, 3), torch.int32)),
               Meshes(v, _stand_in((4, 3), torch.int64, device="cuda:1"))):
        assert mm.verts_normals_packed() == "ref-normals" and mm.original_calls == 1
        mm.verts_normals_packed()
        assert mm.original_calls == 1  # cached by the original, not recomputed
    assert len(fused) == 3
    inst.uninstall()
    assert ops._C is original_C and Meshes.__dict__["_compute_vertex_normals"] is original_method
    assert inst._saved_methods == {} and inst._saved_blend == {}


def test_install_normals_leaves_the_other_installs_alone(monkeypatch, built_lib):
    from pytorch3d_b200 import install as inst
    ops, Meshes = _fake_normals_modules(monkeypatch)
    inst.install_normals()
    try:
        assert set(inst._saved_methods) == {("pytorch3d.structures.meshes", "Meshes", "_compute_vertex_normals")}
        assert set(inst._saved_blend) == {("pytorch3d.ops.mesh_face_areas_normals", "_C")}
        assert inst._saved == {}
    finally:
        inst.uninstall()
    assert inst._saved_methods == {} and inst._saved_blend == {}


# ---------------------------------------------------------------------------------------------------------- GPU ---

def _face_op(s, grads=True):
    from pytorch3d_b200 import normals
    leaf = s["verts"].to(DEV).requires_grad_(True)
    a, n = normals.face_areas_normals(leaf, s["faces"].to(DEV))
    if not grads:
        return a.detach(), n.detach(), None
    g = upstream_grads(s)
    ((a * g["faces_areas"].to(DEV)).sum() + (n * g["faces_normals"].to(DEV)).sum()).backward()
    return a.detach(), n.detach(), leaf.grad


def _vn_op(s, fused=True, device=DEV):
    from pytorch3d_b200 import normals
    leaf = s["verts"].to(device).requires_grad_(True)
    faces = s["faces"].to(device)
    n = normals.verts_normals(leaf, faces) if fused else chain_verts_normals(leaf, faces)
    (n * upstream_grads(s)["verts_normals"].to(device)).sum().backward()
    return n.detach(), leaf.grad


@pytest.mark.gpu
@pytest.mark.parametrize("name", SCENES)
def test_face_op_matches_reference_cuda_records(built_lib, name):
    """Forward bit-identical to the reference's CUDA kernel; backward within rtol 1e-5 of its largest magnitude, and
    bit-identical at vertices with a single corner (one term, nothing to reorder)."""
    s = scene(name)
    a, n, grad = _face_op(s)
    assert_equals_reference([a.cpu()], "normals_cuda/%s/faces_areas" % name, "face areas")
    assert_equals_reference([n.cpu()], "normals_cuda/%s/faces_normals" % name, "face normals")
    (rec,) = reference("normals_cuda/%s/grad_faces" % name)
    got = rec.rows_of(grad.cpu())
    scale = max(rec.absmax, 1e-30)
    assert np.abs(got.astype(np.float64) - rec.sample).max() <= 1e-5 * scale
    single = _corner_counts(s["faces"], s["verts"].shape[0])[rec.rows] == 1
    assert np.array_equal(got[single], rec.sample[single])


@pytest.mark.gpu
@pytest.mark.parametrize("name", SCENES)
def test_verts_normals_match_reference_records(built_lib, name):
    """Forward bit-identical to the reference's CPU chain; backward within rtol 1e-4 / atol 1e-5 of the records' and
    the CUDA chain's largest magnitude, with no NaN where the chain has none."""
    s = scene(name)
    n, grad = _vn_op(s)
    assert_equals_reference([n.cpu()], "normals/%s/verts_normals" % name, "vertex normals")
    (rec,) = reference("normals/%s/grad_verts_normals" % name)
    got = rec.rows_of(grad.cpu()).astype(np.float64)
    assert not np.isnan(got).any()
    assert np.abs(got - rec.sample).max() <= 1e-4 * max(rec.absmax, 1e-30) + 1e-5 * max(rec.absmax, 1e-30)
    cn, cgrad = _vn_op(s, fused=False)
    _close(n, cn, 1e-6, 1e-7, "normals vs the CUDA chain")
    _close(grad, cgrad, 1e-4, 1e-5, "gradient vs the CUDA chain")


@pytest.mark.gpu
def test_verts_normals_match_the_shading_records(built_lib):
    from pytorch3d_b200 import normals, synthetic
    m = synthetic.torus_batch(2, 7, 9, seed=3, device=DEV)
    assert_equals_reference([normals.verts_normals_packed(m).cpu()], "shading/torus_verts_normals", "fused normals")


@pytest.mark.gpu
def test_reproducible_deterministic_and_no_host_sync(built_lib):
    from pytorch3d_b200 import normals
    s = scene("torus_hetero")
    verts, faces = s["verts"].to(DEV), s["faces"].to(DEV)
    g = {k: v.to(DEV) for k, v in upstream_grads(s).items()}

    def run():
        leaf = verts.clone().requires_grad_(True)
        n = normals.verts_normals(leaf, faces)
        (n * g["verts_normals"]).sum().backward()
        leaf2 = verts.clone().requires_grad_(True)
        a, fn = normals.face_areas_normals(leaf2, faces)
        ((a * g["faces_areas"]).sum() + (fn * g["faces_normals"]).sum()).backward()
        return n.detach(), leaf.grad, a.detach(), fn.detach(), leaf2.grad

    was = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        first = run()
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            second = run()
        finally:
            torch.cuda.set_sync_debug_mode("default")
    finally:
        torch.use_deterministic_algorithms(was)
    for a, b in zip(first, second):
        assert torch.equal(a, b)


@pytest.mark.gpu
def test_sizes_and_layouts(built_lib):
    from pytorch3d_b200 import normals
    # no faces: unit normals are 0, gradients 0; areas and face normals empty
    v = torch.rand(5, 3, device=DEV, requires_grad=True)
    f = torch.zeros((0, 3), dtype=torch.int64, device=DEV)
    n = normals.verts_normals(v, f)
    n.sum().backward()
    assert torch.equal(n, torch.zeros_like(n)) and torch.equal(v.grad, torch.zeros_like(v))
    a, fn = normals.face_areas_normals(v.detach(), f)
    assert a.shape == (0,) and fn.shape == (0, 3)
    # V = 1: one degenerate face
    v1 = torch.rand(1, 3, device=DEV, requires_grad=True)
    f1 = torch.zeros((1, 3), dtype=torch.int64, device=DEV)
    n1 = normals.verts_normals(v1, f1)
    n1.sum().backward()
    assert torch.equal(n1, torch.zeros_like(n1)) and torch.equal(v1.grad, torch.zeros_like(v1))
    a1, _ = normals.face_areas_normals(v1.detach(), f1)
    assert torch.equal(a1, torch.zeros(1, device=DEV))
    # unaligned and non-contiguous inputs give the contiguous results
    s = scene("ico_sphere")
    V, F = s["verts"].shape[0], s["faces"].shape[0]
    want_n, want_g = _vn_op(s)
    want_a, want_fn, _ = _face_op(s, grads=False)
    vbuf = torch.empty(V * 3 + 1, device=DEV)
    vbuf[1:] = s["verts"].reshape(-1).to(DEV)
    v_unaligned = vbuf[1:].view(V, 3)
    f_strided = torch.empty((F, 6), dtype=torch.int64, device=DEV)
    f_strided[:, ::2] = s["faces"].to(DEV)
    f_nc = f_strided[:, ::2]
    v_nc = s["verts"].to(DEV).t().contiguous().t()
    for vv, ff in ((v_unaligned, s["faces"].to(DEV)), (v_nc, f_nc)):
        leaf = vv.detach().requires_grad_(True)
        got = normals.verts_normals(leaf, ff)
        (got * upstream_grads(s)["verts_normals"].to(DEV)).sum().backward()
        assert torch.equal(got, want_n) and torch.equal(leaf.grad, want_g)
        a, fn = normals.face_areas_normals(vv, ff)
        assert torch.equal(a, want_a) and torch.equal(fn, want_fn)


@pytest.mark.gpu
def test_argument_errors_on_the_device(built_lib):
    from pytorch3d_b200 import _C, _lib
    v = torch.rand(4, 3, device=DEV)
    f = torch.tensor([[0, 1, 2]], device=DEV)
    with pytest.raises(RuntimeError, match="Float"):
        _C.verts_normals_forward(v.double(), f)
    with pytest.raises(RuntimeError, match="Long"):
        _C.face_areas_normals_forward(v, f.int())
    with pytest.raises(RuntimeError, match=r"\(V, 3\)"):
        _C.verts_normals_forward(torch.rand(4, 2, device=DEV), f)
    with pytest.raises(RuntimeError, match="grad_areas"):
        _C.face_areas_normals_backward(torch.rand(2, device=DEV), torch.rand(1, 3, device=DEV), v, f)
    n, table, sums = _C.verts_normals_forward(v, f)
    with pytest.raises(RuntimeError, match="table"):
        _C.verts_normals_backward(torch.rand(4, 3, device=DEV), v, f, table[:-1], sums)
    lib = _lib.load()
    assert lib.b200r_normals_workspace_bytes(4, 1) >= 4 * (9 + 3 * 4) + 4 * (4 + 1 + 3)
    assert lib.b200r_verts_normals_forward(None, 2 ** 31, None, 1, None, 0, None, None, None, None) != 0
    assert "vertices" in _lib.last_error()
    assert lib.b200r_face_areas_normals_forward(None, 4, None, 2 ** 30, None, None, None) != 0
    assert "faces" in _lib.last_error()


@pytest.mark.gpu
def test_64_bit_offsets(built_lib):
    """A vertex array past 2^31 floats (V = 716,000,000, 8.6 GB) with a few faces on its last vertices: forward and
    backward of both ops agree with the same faces on a copy of those vertices alone.  Peak memory stays under 48 GB;
    skipped when the card has less free memory than that."""
    from pytorch3d_b200 import _C
    free, _ = torch.cuda.mem_get_info()
    if free < 48 * 2 ** 30:
        pytest.skip("needs 48 GB of free device memory, %.1f GB free" % (free / 2 ** 30))
    V = 716_000_000
    assert V * 3 > 2 ** 31
    g = torch.Generator().manual_seed(9)
    tail = torch.rand(8, 3, generator=g).to(DEV)
    local = torch.tensor([[0, 1, 2], [2, 1, 3], [4, 5, 6], [7, 6, 5], [3, 3, 4]], device=DEV)
    gn = torch.randn(8, 3, generator=g).to(DEV)
    ga, gfn = torch.randn(5, generator=g).to(DEV), torch.randn(5, 3, generator=g).to(DEV)
    want_n, table, sums = _C.verts_normals_forward(tail, local)
    want_gv = _C.verts_normals_backward(gn, tail, local, table, sums)
    want_a, want_fn = _C.face_areas_normals_forward(tail, local)
    want_gf = _C.face_areas_normals_backward(ga, gfn, tail, local)

    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    verts = torch.zeros((V, 3), device=DEV)
    verts[-8:] = tail
    faces = local + (V - 8)
    n, table, sums = _C.verts_normals_forward(verts, faces)
    assert torch.equal(n[-8:], want_n) and not bool(n[:-8].any())
    del n  # freed between the forward and the backward
    grad_n = torch.zeros((V, 3), device=DEV)
    grad_n[-8:] = gn
    gv = _C.verts_normals_backward(grad_n, verts, faces, table, sums)
    assert torch.equal(gv[-8:], want_gv) and not bool(gv[:-8].any())
    del gv, grad_n, table, sums
    a, fn = _C.face_areas_normals_forward(verts, faces)
    assert torch.equal(a, want_a) and torch.equal(fn, want_fn)
    gf = _C.face_areas_normals_backward(ga, gfn, verts, faces)
    assert torch.equal(gf[-8:], want_gf) and not bool(gf[:-8].any())
    del gf, verts
    peak = torch.cuda.max_memory_allocated()
    torch.cuda.empty_cache()
    assert peak < 48 * 2 ** 30, peak


def _render(mesh_cls, shade, normals_fn):
    """Rasterize a torus batch, shade it (fused Phong or flat) with normals from `normals_fn`, blend with the fused
    softmax blend; returns the image and the vertex gradient."""
    from pytorch3d_b200 import shading, synthetic
    from pytorch3d_b200.blending import BlendParams, softmax_rgb_blend
    from pytorch3d_b200.rasterize_meshes import rasterize_meshes
    m = synthetic.torus_batch(2, 24, 24, seed=1, device=DEV)
    m.requires_grad_(True)
    verts = m.verts_packed()
    mesh = mesh_cls(m, normals_fn)
    p2f, zbuf, bary, dists = rasterize_meshes(m, (48, 80), blur_radius=0.0, faces_per_pixel=4)
    frags = types.SimpleNamespace(pix_to_face=p2f, bary_coords=bary, zbuf=zbuf, dists=dists)
    texels = torch.full(p2f.shape + (3,), 0.8, device=DEV)
    lights = types.SimpleNamespace(ambient_color=torch.tensor([[0.3, 0.3, 0.3]], device=DEV),
                                   diffuse_color=torch.tensor([[0.6, 0.5, 0.4]], device=DEV),
                                   specular_color=torch.tensor([[0.3, 0.3, 0.3]], device=DEV),
                                   location=torch.tensor([[0.5, 1.0, -1.0]], device=DEV))
    cameras = types.SimpleNamespace(get_camera_center=lambda: torch.zeros(1, 3, device=DEV))
    materials = types.SimpleNamespace(ambient_color=torch.ones(1, 3, device=DEV),
                                      diffuse_color=torch.ones(1, 3, device=DEV),
                                      specular_color=torch.ones(1, 3, device=DEV),
                                      shininess=torch.tensor([64.0], device=DEV))
    colors = getattr(shading, shade)(mesh, frags, lights, cameras, materials, texels)
    img = softmax_rgb_blend(colors, frags, BlendParams(sigma=1e-4, gamma=1e-4))
    w = torch.rand(img.shape, generator=torch.Generator().manual_seed(6)).to(DEV)
    (img * w).sum().backward()
    return img.detach(), verts.grad


class _WithNormals:
    def __init__(self, m, normals_fn):
        self._m, self._fn = m, normals_fn

    def __getattr__(self, name):
        return getattr(self._m, name)

    def verts_normals_packed(self):
        return self._fn(self._m)[0]

    def faces_normals_packed(self):
        return self._fn(self._m)[1]


def _fused_normals(m):
    from pytorch3d_b200 import normals
    return normals.verts_normals_packed(m), normals.faces_areas_normals_packed(m)[1]


def reference_face_normals_backward(grad_normals, verts, faces):
    """The reference's FaceAreasNormalsBackwardKernel with grad_areas = 0, restated in float64 torch: its per-corner
    terms, including the cx it uses where cy belongs in one term of corner 1's z gradient, scattered to the vertices.
    This is not autograd's gradient of the normals, so a chain that wants the reference's face-normal gradient uses
    this."""
    p = verts.double()[faces]
    a, b = p[:, 1] - p[:, 0], p[:, 2] - p[:, 0]
    c = torch.cross(a, b, dim=1)
    inv = 1.0 / c.norm(dim=1).clamp_min(1e-6)
    g = grad_normals.double()
    ax, ay, az, bx, by, bz = a[:, 0], a[:, 1], a[:, 2], b[:, 0], b[:, 1], b[:, 2]
    cx, cy, cz = c[:, 0], c[:, 1], c[:, 2]

    def term(t, d, cs):  # d: the partials of (cx, cy, cz), None where structurally 0; cs: the c multiplying t per k
        out = 0.0
        for k in range(3):
            if d[k] is None:
                out = out - cs[k] * t * inv ** 3 * g[:, k]
            else:
                out = out + (d[k] - cs[k] * t * inv ** 2) * inv * g[:, k]
        return out

    C = (cx, cy, cz)
    rows = [
        term((-az + bz) * cy + (-by + ay) * cz, (None, -az + bz, -by + ay), C),
        term((-bz + az) * cx + (-ax + bx) * cz, (-bz + az, None, -ax + bx), C),
        term((-ay + by) * cx + (-bx + ax) * cy, (-ay + by, -bx + ax, None), C),
        term(by * cz - bz * cy, (None, -bz, by), C),
        term(bz * cx - bx * cz, (bz, None, -bx), C),
        term(bx * cy - by * cx, (-by, bx, None), (cx, cx, cz)),
        term(az * cy - ay * cz, (None, az, -ay), C),
        term(ax * cz - az * cx, (-az, None, ax), C),
        term(ay * cx - ax * cy, (ay, -ax, None), C),
    ]
    corner = torch.stack(rows, 1).reshape(-1, 3, 3)
    out = torch.zeros(verts.shape, dtype=torch.float64, device=verts.device)
    out.index_add_(0, faces.reshape(-1), corner.reshape(-1, 3))
    return out.to(verts.dtype)


class _ChainFaceNormals(torch.autograd.Function):
    """Face normals by torch ops, with the reference's backward."""

    @staticmethod
    def forward(ctx, verts, faces):
        corners = verts[faces]
        c = torch.cross(corners[:, 1] - corners[:, 0], corners[:, 2] - corners[:, 0], dim=1)
        ctx.save_for_backward(verts, faces)
        return c / c.norm(dim=1, keepdim=True).clamp_min(1e-6)

    @staticmethod
    def backward(ctx, grad):
        verts, faces = ctx.saved_tensors
        return reference_face_normals_backward(grad, verts, faces), None


def _chain_normals(m):
    return m.verts_normals_packed(), _ChainFaceNormals.apply(m.verts_packed(), m.faces_packed())


def test_reference_face_normals_backward_restatement_cpu():
    """The float64 restatement of the reference's face-normal backward equals autograd's gradient of the normals
    wherever the reference's formula is right (x and y, and z at vertices that are never corner 1), and differs in
    corner 1's z."""
    s = scene("ico_sphere")
    leaf = s["verts"].double().requires_grad_(True)
    p = leaf[s["faces"]]
    c = torch.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0], dim=1)
    n = c / c.norm(dim=1, keepdim=True).clamp_min(1e-6)
    g = upstream_grads(s)["faces_normals"].double()
    (n * g).sum().backward()
    mine = reference_face_normals_backward(g, s["verts"].double(), s["faces"])
    # only vertices whose every corner is corner 0 or 2 are free of the reference's typo
    as1 = torch.zeros(s["verts"].shape[0], dtype=torch.bool)
    as1[s["faces"][:, 1]] = True
    assert torch.allclose(mine[~as1], leaf.grad[~as1], rtol=1e-9, atol=1e-12)
    assert torch.allclose(mine[:, :2], leaf.grad[:, :2], rtol=1e-9, atol=1e-12)
    assert not torch.allclose(mine[as1, 2], leaf.grad[as1, 2], rtol=1e-3)


@pytest.mark.gpu
@pytest.mark.parametrize("shade", ["phong_shading", "flat_shading"])
def test_end_to_end_render_matches_torch_chain(built_lib, shade):
    got = _render(_WithNormals, shade, _fused_normals)
    want = _render(_WithNormals, shade, _chain_normals)
    _close(got[0], want[0], 1e-5, 1e-6, "image")
    assert float(want[1].abs().max()) > 0
    _close(got[1], want[1], 1e-4, 1e-5, "grad_verts")
