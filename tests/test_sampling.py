"""Mesh surface sampling on the GPU (DESIGN.md section 20): `pytorch3d_b200.sampling`, the `_C.sample_points_*` ops,
the `_C._sample_points_from_draws` hook and `install_sampling()`.

The records (tests/golden/make_sampling_golden.py, reference_golden_sampling.npz) come from the reference's own
`sample_points_from_meshes` on the CPU, with the draws that produced them.  `restated` is a float64 torch restatement of
the positions and normals for given draws, written from their definitions; it is checked against the records on the
CPU and is the second yardstick of the fused op's gradients on the GPU.
"""
import math
import sys
import types
import warnings

import numpy as np
import pytest
import torch

import test_normals as tn
import test_regularizers as tr
from helpers import GOLDEN_DIR, reference

DEV = "cuda"
SEED = 20
NUM_SAMPLES = 100
SCENES = ("torus_hetero", "ico_sphere", "empty_middle", "zero_area", "sliver")
TEXTURED = ("torus_hetero", "ico_sphere")
TOL = 1e-5


def scene(name):
    """{verts (V,3) f32 packed, faces (F,3) i64 packed, faces_list, nverts}: two scenes of test_normals, a batch with a
    mesh without faces in the middle, a mesh with zero-area faces mixed in (exactly collinear corners, a repeated
    vertex), the sliver of test_regularizers, and a mesh whose faces all have zero area."""
    if name in ("torus_hetero", "ico_sphere"):
        return tn.scene(name)
    if name == "sliver":
        return tr.scene(name)
    from pytorch3d_b200 import synthetic
    g = torch.Generator().manual_seed(SCENES.index(name) + 301 if name in SCENES else 399)
    if name == "empty_middle":
        v0, f0 = synthetic.ico_sphere(1)
        v2, f2 = synthetic.torus(6, 5)
        return tn._from_lists([v0.float(), torch.randn(4, 3, generator=g), v2.float()],
                              [f0, torch.zeros((0, 3), dtype=torch.int64), f2])
    if name == "zero_area":
        v = torch.randn(12, 3, generator=g)
        v[9], v[10], v[11] = torch.tensor([0.0, 0.0, 0.0]), torch.tensor([1.0, 1.0, 1.0]), torch.tensor([2.0, 2.0, 2.0])
        f = torch.tensor([[0, 1, 2], [9, 10, 11], [3, 4, 5], [6, 6, 7], [1, 3, 8], [10, 11, 9], [2, 5, 7], [4, 4, 4]])
        return tn._from_lists([v], [f])
    if name == "zero_total":
        v = torch.tensor([[0.0, 0.0, 0.0], [1.0, 1.0, 1.0], [2.0, 2.0, 2.0], [0.5, 0.2, 0.1]])
        return tn._from_lists([v], [torch.tensor([[0, 1, 2], [3, 3, 1]])])
    raise KeyError(name)


def textures(s):
    """Per-vertex colours (V, 3), and a TexturesUV's maps (N, 8, 8, 3), verts_uvs and faces_uvs lists."""
    g = torch.Generator().manual_seed(int(s["verts"].shape[0]))
    N = len(s["faces_list"])
    return {"colors": torch.rand(s["verts"].shape[0], 3, generator=g),
            "maps": torch.rand(N, 8, 8, 3, generator=g),
            "verts_uvs": [torch.rand(n, 2, generator=g) for n in s["nverts"]],
            "faces_uvs": [f.clone() for f in s["faces_list"]]}


def upstream(name, shape):
    g = torch.Generator().manual_seed(SCENES.index(name) * 7 + 3)
    return torch.randn(shape + (3,), generator=g), torch.randn(shape + (3,), generator=g)


def record(name, field):
    (rec,) = reference("sampling/%s/%s" % (name, field))
    return torch.from_numpy(rec.sample.reshape(rec.shape))


def sqrt_rn(u):
    """The correctly rounded float32 square root, as torch's CUDA sqrt computes it.  torch's vectorised CPU sqrt is
    off by one ulp for about 1% of float32 inputs, so the CPU records differ from it there."""
    return torch.from_numpy(np.sqrt(u.detach().cpu().numpy())).to(u.device)


def barycentrics(u, v):
    """_rand_barycentric_coords for given (u, v), in the reference's float32 torch ops with sqrt_rn."""
    s = sqrt_rn(u)
    return 1.0 - s, s * (1.0 - v), s * v


# ---------------------------------------------------------------------------------------- float64 restatement ---

def restated(verts, faces, face, w, valid):
    """(samples, normals) in float64 for verts (V,3) (may require grad), the packed draws face (N,S) and the
    barycentrics w (N,S,3) (constants); rows of invalid meshes are zeros."""
    v = verts.double()
    f = faces[face.clamp_min(0)]
    a, b, c = v[f[..., 0]], v[f[..., 1]], v[f[..., 2]]
    w = w.double()
    p = w[..., 0:1] * a + w[..., 1:2] * b + w[..., 2:3] * c
    n = torch.cross(b - a, c - b, dim=-1)
    n = n / n.norm(dim=-1, keepdim=True).clamp_min(sys.float_info.epsilon)
    keep = valid[:, None, None].to(v.device)
    return torch.where(keep, p, torch.zeros_like(p)), torch.where(keep, n, torch.zeros_like(n))


def well_conditioned(verts, faces, face):
    """Samples whose face normal float32 resolves: |a| |b| / |a x b| < 1e3."""
    v = verts.double()
    f = faces[face.clamp_min(0)]
    a, b = v[f[..., 1]] - v[f[..., 0]], v[f[..., 2]] - v[f[..., 1]]
    return a.norm(dim=-1) * b.norm(dim=-1) < 1e3 * torch.cross(a, b, dim=-1).norm(dim=-1)


def valid_of(s):
    return torch.tensor([f.shape[0] > 0 for f in s["faces_list"]])


def _rel(got, want):
    return float((got.double() - want.double()).abs().max()) / max(float(want.double().abs().max()), 1e-30)


def restated_textures(s, tex, face, w, kind):
    """TexturesVertex / TexturesUV (bilinear, border padding, align_corners) sampled at the draws, in torch."""
    fl = s["faces"].to(face.device)
    if kind == "vertex":
        corners = tex["colors"].to(face.device)[fl][face]
        return (w[..., None] * corners).sum(dim=-2)
    offs = torch.tensor(np.cumsum([0] + s["nverts"][:-1]).tolist(), device=face.device)
    uvs = torch.cat(tex["verts_uvs"]).to(face.device)
    fu = torch.cat([f + o for f, o in zip(tex["faces_uvs"], offs.tolist())]).to(face.device)
    pix = (w[..., None] * uvs[fu][face]).sum(dim=-2)  # (N, S, 2)
    grid = (pix * 2.0 - 1.0)[:, :, None, :]  # (N, S, 1, 2)
    maps = torch.flip(tex["maps"].to(face.device).permute(0, 3, 1, 2), [2])
    out = torch.nn.functional.grid_sample(maps, grid, mode="bilinear", padding_mode="border", align_corners=True)
    return out[..., 0].permute(0, 2, 1)


# ------------------------------------------------------------------------------------------------------- CPU ---

@pytest.mark.parametrize("name", SCENES)
def test_restatement_matches_records_cpu(name):
    s = scene(name)
    face, u, v = (record(name, k) for k in ("face", "u", "v"))
    w = torch.stack(barycentrics(u, v), -1)
    valid = valid_of(s)
    leaf = s["verts"].double().requires_grad_(True)
    p, n = restated(leaf, s["faces"], face, w, valid)
    assert _rel(p.detach(), record(name, "samples")) <= 1e-6
    ok = well_conditioned(s["verts"], s["faces"], face) & valid[:, None]
    assert _rel(n.detach()[ok], record(name, "normals")[ok]) <= 1e-5
    gs, gn = upstream(name, tuple(face.shape))
    (g1,) = torch.autograd.grad((p * gs.double()).sum(), leaf, retain_graph=True)
    assert _rel(g1, record(name, "grad_samples")) <= TOL
    if name != "sliver" and name != "zero_area":  # ill-conditioned normals: compared on the GPU against the records
        (g2,) = torch.autograd.grad((p * gs.double()).sum() + (n * gn.double()).sum(), leaf)
        assert _rel(g2, record(name, "grad_normals")) <= TOL


@pytest.mark.parametrize("name", TEXTURED)
def test_texture_restatement_matches_records_cpu(name):
    s = scene(name)
    face, u, v = (record(name, k) for k in ("face", "u", "v"))
    w = torch.stack(barycentrics(u, v), -1)
    tex = textures(s)
    for kind in ("vertex", "uv"):
        assert _rel(restated_textures(s, tex, face, w, kind), record(name, "textures_" + kind)) <= 1e-6, kind


def test_records_cover_the_special_cases_cpu():
    face = record("zero_area", "face")
    s = scene("zero_area")
    p = s["verts"][s["faces"]]
    area = torch.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0], dim=1).norm(dim=1)
    zero = (area == 0).nonzero().flatten()
    assert len(zero) == 4 and not bool(torch.isin(face, zero).any())
    assert torch.equal(record("empty_middle", "samples")[1], torch.zeros(NUM_SAMPLES, 3))
    msg = bytes(np.load(GOLDEN_DIR + "/reference_golden_sampling.npz")["sampling/zero_total/error/0/message"]).decode()
    assert msg == "invalid multinomial distribution (sum of probabilities <= 0)"


class _Batch:
    def __init__(self, n=2, V=10, F=4, dtype=torch.float32, fdtype=torch.int64, is_cuda=True):
        dev = types.SimpleNamespace(type="cuda" if is_cuda else "cpu")
        self._v = types.SimpleNamespace(is_cuda=is_cuda, device=dev, dtype=dtype, shape=(V, 3), dim=lambda: 2)
        self._f = types.SimpleNamespace(is_cuda=is_cuda, device=dev, dtype=fdtype, shape=(F, 3), dim=lambda: 2)
        self._n = n

    def __len__(self):
        return self._n

    def verts_packed(self):
        return self._v

    def faces_packed(self):
        return self._f


def _fake_ops_modules(monkeypatch):
    for n in ["pytorch3d"]:
        m = types.ModuleType(n)
        m.__path__ = []
        monkeypatch.setitem(sys.modules, n, m)
    package = types.ModuleType("pytorch3d.ops")
    package.__path__ = []
    mod = types.ModuleType("pytorch3d.ops.sample_points_from_meshes")

    def sample_points_from_meshes(meshes, num_samples=10000, return_normals=False, return_textures=False):
        return ("ref", num_samples, return_normals, return_textures)

    mod.sample_points_from_meshes = sample_points_from_meshes
    package.sample_points_from_meshes = sample_points_from_meshes  # the package attribute is the function
    monkeypatch.setitem(sys.modules, package.__name__, package)
    monkeypatch.setitem(sys.modules, mod.__name__, mod)
    return package, mod


def test_install_sampling_routing_and_uninstall(monkeypatch, built_lib):
    from pytorch3d_b200 import install as inst
    from pytorch3d_b200 import sampling as ours
    package, mod = _fake_ops_modules(monkeypatch)
    original = mod.sample_points_from_meshes
    calls = []

    def fused(m, num_samples=10000, return_normals=False, return_textures=False):
        calls.append(return_textures)
        if getattr(m, "empty_with_textures", False) and return_textures:
            raise ours.EmptyMeshWithTextures("empty")
        return ("b200", num_samples, return_normals, return_textures)

    monkeypatch.setattr(ours, "sample_points_from_meshes", fused)
    assert inst.install_sampling() == ["pytorch3d.ops", "pytorch3d.ops.sample_points_from_meshes"]
    good = _Batch()
    for owner in (package, mod):
        assert owner.sample_points_from_meshes(good) == ("b200", 10000, False, False)
        assert owner.sample_points_from_meshes(good, 50, return_normals=True) == ("b200", 50, True, False)
        assert owner.sample_points_from_meshes(good, 5, True, True) == ("b200", 5, True, True)
    empty = _Batch()
    empty.empty_with_textures = True
    assert package.sample_points_from_meshes(empty, 7, return_textures=True) == ("ref", 7, False, True)
    assert package.sample_points_from_meshes(empty, 7) == ("b200", 7, False, False)
    for bad, S in ((_Batch(is_cuda=False), 10), (_Batch(dtype=torch.float64), 10), (_Batch(fdtype=torch.int32), 10),
                   (_Batch(n=0), 10), (_Batch(), 0), (_Batch(), 2.5), (_Batch(), True), (_Batch(V=(1 << 31) - 1), 10),
                   (_Batch(n=4), (1 << 40) // 4 + 1)):
        assert package.sample_points_from_meshes(bad, S) == ("ref", S, False, False)
    inst.install_sampling()  # idempotent
    inst.uninstall()
    assert package.sample_points_from_meshes is original and mod.sample_points_from_meshes is original
    assert inst._saved_blend == {}


def test_host_errors_cpu(built_lib):
    from pytorch3d_b200 import PackedMeshes, _C, sampling
    with pytest.raises(ValueError, match="Meshes are empty."):
        sampling.sample_points_from_meshes(PackedMeshes([], []))
    v, f = torch.zeros(3, 3), torch.tensor([[0, 1, 2]])
    first, num = torch.zeros(1, dtype=torch.int64), torch.ones(1, dtype=torch.int64)
    seed = torch.zeros(2, dtype=torch.int64)
    with pytest.raises(RuntimeError, match="must be a CUDA tensor"):
        _C.sample_points_forward(v, f, first, num, 10, False, seed)
    assert _C.sampling_sizes_ok(10, 4, 2, 1 << 39) and not _C.sampling_sizes_ok(10, 4, 2, (1 << 39) + 1)
    assert not _C.sampling_sizes_ok((1 << 31) - 1, 4, 1, 1) and not _C.sampling_sizes_ok(10, 4, 1, 0)


# ----------------------------------------------------------------------------------------------------- GPU ---

def _packed(s, device=DEV):
    from pytorch3d_b200 import PackedMeshes
    return PackedMeshes(list(torch.split(s["verts"].to(device), s["nverts"])), [f.to(device) for f in s["faces_list"]])


def _from_draws(m, face, u, v, normals=True):
    from pytorch3d_b200 import sampling
    return sampling._sample_from_draws(m, face.to(DEV), u.to(DEV), v.to(DEV), return_normals=normals)


@pytest.mark.gpu
@pytest.mark.parametrize("name", SCENES)
def test_given_draws_match_records(built_lib, name):
    from pytorch3d_b200 import _C
    s = scene(name)
    face, u, v = (record(name, k) for k in ("face", "u", "v"))
    m = _packed(s)
    out = _C._sample_points_from_draws(m.verts_packed(), m.faces_packed(), m.mesh_to_faces_packed_first_idx(),
                                       m.num_faces_per_mesh(), True, face.to(DEV), u.to(DEV), v.to(DEV))
    samples, normals, fidx, bary, status = (t.cpu() for t in out)
    valid = valid_of(s)
    # bit-identical to the reference's chain on the device, and to the CPU records wherever the CPU's sqrt(u) is
    # correctly rounded (one ulp of w0, w1, w2 elsewhere)
    chain = _torch_chain(m.verts_packed(), m.faces_packed(), face.to(DEV), u.to(DEV), v.to(DEV)).cpu()
    chain[~valid] = 0
    assert torch.equal(samples, chain), _rel(samples, chain)
    rn = sqrt_rn(u) == u.sqrt()
    assert float(rn.double().mean()) > 0.9
    assert torch.equal(samples[rn], record(name, "samples")[rn]), _rel(samples, record(name, "samples"))
    assert _rel(samples, record(name, "samples")) <= 2.0 ** -21
    assert torch.equal(normals, record(name, "normals")), _rel(normals, record(name, "normals"))
    w = torch.stack(barycentrics(u, v), -1)
    assert torch.equal(bary[valid], w[valid]) and torch.equal(fidx[valid], face[valid])
    assert bool((fidx[~valid] == -1).all()) and not bool(bary[~valid].any())
    gs, gn = upstream(name, tuple(face.shape))
    for field, with_normals in (("grad_samples", False), ("grad_normals", True)):
        m.requires_grad_(True)
        m.verts_packed().grad = None
        out = _from_draws(m, face, u, v, normals=with_normals)
        p, n = out if with_normals else (out, None)
        loss = (p * gs.to(DEV)).sum() + ((n * gn.to(DEV)).sum() if with_normals else 0.0)
        loss.backward()
        grad = m.verts_packed().grad.cpu()
        assert _rel(grad, record(name, field)) <= TOL, (field, _rel(grad, record(name, field)))
        if with_normals and name in ("sliver", "zero_area"):
            continue
        leaf = s["verts"].double().requires_grad_(True)
        p, n = restated(leaf, s["faces"], face, w, valid)
        ((p * gs.double()).sum() + ((n * gn.double()).sum() if with_normals else 0.0)).backward()
        assert _rel(grad, leaf.grad) <= TOL, (field, _rel(grad, leaf.grad))


class _Textured:
    """A PackedMeshes with `textures` and `sample_textures` of a TexturesVertex or TexturesUV, restated."""

    def __init__(self, s, kind):
        self._m, self._s, self._kind, self._tex = _packed(s), s, kind, textures(s)
        self.textures = kind

    def __getattr__(self, name):
        return getattr(self._m, name)

    def __len__(self):
        return len(self._m)

    def sample_textures(self, fragments):
        face = fragments.pix_to_face[:, :, 0, 0]
        w = fragments.bary_coords[:, :, 0, 0, :]
        return restated_textures(self._s, self._tex, face, w, self._kind)[:, :, None, None, :]


@pytest.mark.gpu
@pytest.mark.parametrize("name", TEXTURED)
def test_textures_match_records(built_lib, name):
    from pytorch3d_b200 import sampling
    s = scene(name)
    face, u, v = (record(name, k) for k in ("face", "u", "v"))
    for kind in ("vertex", "uv"):
        m = _Textured(s, kind)
        samples, tex = sampling._sample_from_draws(m, face.to(DEV), u.to(DEV), v.to(DEV), return_textures=True)
        assert tex.shape == (len(s["faces_list"]), NUM_SAMPLES, 3)
        assert _rel(tex.cpu(), record(name, "textures_" + kind)) <= 1e-6, kind


def _weighted_mesh(n=40, seed=0):
    """A fan of n faces whose areas span four decades, with every fifth face of zero area (a repeated vertex)."""
    g = torch.Generator().manual_seed(seed)
    t = torch.linspace(0, 2 * math.pi, n + 1)[:-1]
    r = 10 ** (torch.rand(n, generator=g) * 4 - 2)
    ring = torch.stack([torch.cos(t) * r, torch.sin(t) * r, torch.zeros(n)], 1)
    v = torch.cat([torch.zeros(1, 3), ring])
    i = torch.arange(1, n + 1)
    f = torch.stack([torch.zeros_like(i), i, i % n + 1], 1)
    f[::5, 2] = f[::5, 1]
    return v, f


def _areas(v, f):
    p = v.double()[f]
    return torch.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0], dim=1).norm(dim=1) / 2


@pytest.mark.gpu
def test_distribution_chi_square_and_marginals(built_lib):
    from scipy import stats

    from pytorch3d_b200 import PackedMeshes, _C, sampling
    v, f = _weighted_mesh()
    m = PackedMeshes([v.to(DEV)], [f.to(DEV)])
    S = 2_000_000
    seed = torch.tensor([31, 41], dtype=torch.int64, device=DEV)
    samples, _, fidx, bary, _ = _C.sample_points_forward(m.verts_packed(), m.faces_packed(),
                                                         m.mesh_to_faces_packed_first_idx(), m.num_faces_per_mesh(),
                                                         S, False, seed)
    counts = torch.bincount(fidx.flatten(), minlength=f.shape[0]).cpu().double()
    area = _areas(v, f)
    assert float(counts[area == 0].sum()) == 0
    pos = area > 0
    expected = area[pos] / area[pos].sum() * S
    assert stats.chisquare(counts[pos].numpy(), expected.numpy()).pvalue > 1e-4
    w = bary[0, :200_000].double().cpu()
    assert stats.kstest(w[:, 0].numpy(), lambda t: 1 - (1 - t) ** 2).pvalue > 1e-4
    ok = w[:, 0] < 1
    assert stats.kstest((w[ok, 1] / (1 - w[ok, 0])).numpy(), "uniform").pvalue > 1e-4
    p = m.verts_packed()[m.faces_packed()][fidx[0]]
    lo, hi = p.min(dim=1).values, p.max(dim=1).values
    slack = 1e-6 * (1 + hi.abs())
    assert bool(((samples[0] >= lo - slack) & (samples[0] <= hi + slack)).all())
    zero = torch.zeros_like(bary[..., 0])
    s0 = sampling._sample_from_draws(m, fidx, zero, zero)
    assert torch.equal(s0[0], p[:, 0])  # u = 0: corner 0 exactly


@pytest.mark.gpu
def test_zero_area_faces_never_drawn(built_lib):
    """>= 10^7 samples over 3 chunks of the prefix scan, zero-area faces at the chunk and warp boundaries and every
    seventh face."""
    from pytorch3d_b200 import PackedMeshes, _C
    F = 3 * 4096 + 100
    g = torch.Generator().manual_seed(5)
    v = torch.randn(F + 2, 3, generator=g)
    i = torch.arange(F)
    f = torch.stack([i, i + 1, i + 2], 1)
    zero = (i % 7 == 0) | (i % 4096 == 0) | (i % 4096 == 4095) | (i % 32 == 0) | (i % 512 == 511)
    f[zero, 2] = f[zero, 0]
    m = PackedMeshes([v.to(DEV)], [f.to(DEV)])
    seed = torch.tensor([123, 456], dtype=torch.int64, device=DEV)
    _, _, fidx, _, status = _C.sample_points_forward(m.verts_packed(), m.faces_packed(),
                                                     m.mesh_to_faces_packed_first_idx(), m.num_faces_per_mesh(),
                                                     10_000_000, False, seed)
    counts = torch.bincount(fidx.flatten(), minlength=F).cpu()
    assert int(status.item()) == _C.SAMPLE_HAS_VALID
    assert int(counts[zero].sum()) == 0 and bool((counts[~zero] > 0).all())


@pytest.mark.gpu
def test_reproducible_and_consecutive_calls_differ(built_lib):
    from pytorch3d_b200 import sampling
    s = scene("torus_hetero")
    gs, gn = (t.to(DEV) for t in upstream("torus_hetero", (3, 5000)))

    def run():
        m = _packed(s).requires_grad_(True)
        p, n = sampling.sample_points_from_meshes(m, 5000, return_normals=True)
        ((p * gs).sum() + (n * gn).sum()).backward()
        return p.detach(), n.detach(), m.verts_packed().grad

    torch.use_deterministic_algorithms(True)
    try:
        torch.manual_seed(7)
        a = run()
        b = run()
        torch.manual_seed(7)
        c = run()
    finally:
        torch.use_deterministic_algorithms(False)
    for x, y in zip(a, c):
        assert torch.equal(x, y)
    assert not torch.equal(a[0], b[0])


@pytest.mark.gpu
def test_one_host_sync_forward_none_backward(built_lib):
    from pytorch3d_b200 import sampling
    s = scene("torus_hetero")
    m = _packed(s).requires_grad_(True)
    sampling.sample_points_from_meshes(m, 100, return_normals=True)  # warm up
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("warn")
    try:
        with warnings.catch_warnings(record=True) as fwd:
            warnings.simplefilter("always")
            p, n = sampling.sample_points_from_meshes(m, 1000, return_normals=True)
        with warnings.catch_warnings(record=True) as bwd:
            warnings.simplefilter("always")
            (p.sum() + n.sum()).backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    sync = [w for w in fwd if "synchroniz" in str(w.message)]
    assert len(sync) == 1, [str(w.message) for w in fwd]
    assert not [w for w in bwd if "synchroniz" in str(w.message)]


@pytest.mark.gpu
def test_empty_meshes_and_error_paths(built_lib):
    from pytorch3d_b200 import PackedMeshes, sampling
    s = scene("empty_middle")
    m = _packed(s).requires_grad_(True)
    p, n = sampling.sample_points_from_meshes(m, 300, return_normals=True)
    assert not bool(p[1].any()) and not bool(n[1].any())
    (p.sum() + n.sum()).backward()
    a, b = s["nverts"][0], s["nverts"][0] + s["nverts"][1]
    g = m.verts_packed().grad
    assert not bool(g[a:b].any()) and bool(g[:a].any())
    e = torch.zeros((0, 3), dtype=torch.int64, device=DEV)
    with pytest.raises(ValueError, match="^Meshes are empty.$"):
        sampling.sample_points_from_meshes(PackedMeshes([torch.rand(3, 3, device=DEV)] * 2, [e, e]))
    z = scene("zero_total")
    bad = z["verts"].clone()
    bad[3, 1] = float("nan")  # a vertex in no face still counts
    zm = _packed(dict(z, verts=bad))
    zm.textures = None
    with pytest.raises(ValueError, match="^Meshes contain nan or inf.$"):
        sampling.sample_points_from_meshes(zm, 10, return_textures=True)
    zm = _packed(z)
    zm.textures = None
    with pytest.raises(ValueError, match="^Meshes do not contain textures.$"):
        sampling.sample_points_from_meshes(zm, 10, return_textures=True)
    msg = bytes(np.load(GOLDEN_DIR + "/reference_golden_sampling.npz")["sampling/zero_total/error/0/message"]).decode()
    with pytest.raises(RuntimeError) as err:
        sampling.sample_points_from_meshes(_packed(z), 10)
    assert str(err.value) == msg
    with pytest.raises(sampling.EmptyMeshWithTextures):
        mt = _packed(s)
        mt.textures = "anything"
        sampling.sample_points_from_meshes(mt, 10, return_textures=True)
    torch.cuda.synchronize()  # no device fault


def _torch_chain(verts, faces, face, u, v):
    """The reference's float32 position chain on the device, for given draws."""
    w0, w1, w2 = barycentrics(u, v)
    fv = verts[faces]
    a, b, c = fv[:, 0][face], fv[:, 1][face], fv[:, 2][face]
    return w0[:, :, None] * a + w1[:, :, None] * b + w2[:, :, None] * c


@pytest.mark.gpu
def test_forced_draws_s1_and_layouts(built_lib):
    s = scene("torus_hetero")
    m = _packed(s)
    first, num = m.mesh_to_faces_packed_first_idx(), m.num_faces_per_mesh()
    face = torch.stack([first, first + num - 1, first, first + num - 1], 1)
    one = 1.0 - 2.0 ** -24
    u = torch.tensor([[0.0, 0.0, one, one]], device=DEV).expand(3, 4).contiguous()
    v = torch.tensor([[0.0, one, one, 0.5]], device=DEV).expand(3, 4).contiguous()
    p = _from_draws(m, face, u, v, normals=False)
    assert torch.equal(p, _torch_chain(m.verts_packed(), m.faces_packed(), face, u, v))
    from pytorch3d_b200 import sampling
    torch.manual_seed(3)
    p1 = sampling.sample_points_from_meshes(m, 1)
    assert p1.shape == (3, 1, 3)
    base = m.verts_packed()
    # unaligned (offset by one float) and non-contiguous (a column slice) verts give the contiguous results
    store = torch.empty(base.numel() + 1, device=DEV)
    store[1:] = base.flatten()
    wide = torch.zeros(base.shape[0], 4, device=DEV)
    wide[:, :3] = base
    want = _from_draws(m, face, u, v)
    for verts in (store[1:].view(-1, 3), wide[:, :3]):
        m._verts_packed = verts
        got = _from_draws(m, face, u, v)
        assert all(torch.equal(x, y) for x, y in zip(got, want))
    m._verts_packed = base


@pytest.mark.gpu
def test_more_faces_than_multinomial_takes(built_lib):
    """One mesh of 2^24 + 4096 faces, which torch.multinomial refuses: coarse distribution, every sample in its face."""
    from pytorch3d_b200 import PackedMeshes, _C
    F = (1 << 24) + 4096
    g = torch.Generator(device=DEV).manual_seed(11)
    v = torch.rand(F + 2, 3, device=DEV, generator=g)
    i = torch.arange(F, device=DEV)
    f = torch.stack([i, i + 1, i + 2], 1)
    m = PackedMeshes([v], [f])
    seed = torch.tensor([9, 10], dtype=torch.int64, device=DEV)
    S = 4_000_000
    samples, _, fidx, bary, status = _C.sample_points_forward(v, f, m.mesh_to_faces_packed_first_idx(),
                                                              m.num_faces_per_mesh(), S, False, seed)
    assert int(status.item()) == _C.SAMPLE_HAS_VALID
    area = _areas(v, f)
    bins = 16
    expect = torch.stack([c.sum() for c in area.chunk(bins)]) / area.sum() * S
    got = torch.bincount(fidx.flatten() * bins // F, minlength=bins).double()
    assert bool(((got - expect).abs() < 6 * expect.sqrt()).all()), (got, expect)
    p = v[f[fidx[0]]]
    w = bary[0]
    want = (w[:, 0:1] * p[:, 0] + w[:, 1:2] * p[:, 1]) + w[:, 2:3] * p[:, 2]
    assert torch.equal(samples[0], want)
    lo, hi = p.min(dim=1).values, p.max(dim=1).values
    assert bool(((samples[0] >= lo - 1e-6) & (samples[0] <= hi + 1e-6)).all())


@pytest.mark.gpu
def test_samples_past_2_31_floats(built_lib):
    from pytorch3d_b200 import PackedMeshes, _C
    v, f = _weighted_mesh()
    m = PackedMeshes([v.to(DEV)], [f.to(DEV)])
    S = (1 << 31) // 3 + 4096
    seed = torch.tensor([1, 2], dtype=torch.int64, device=DEV)
    samples, _, fidx, bary, status = _C.sample_points_forward(m.verts_packed(), m.faces_packed(),
                                                              m.mesh_to_faces_packed_first_idx(),
                                                              m.num_faces_per_mesh(), S, False, seed)
    assert samples.numel() > (1 << 31) and int(status.item()) == _C.SAMPLE_HAS_VALID
    tail = slice(S - 100_000, S)
    p = m.verts_packed()[m.faces_packed()][fidx[0, tail]]
    w = bary[0, tail]
    want = (w[:, 0:1] * p[:, 0] + w[:, 1:2] * p[:, 1]) + w[:, 2:3] * p[:, 2]
    assert torch.equal(samples[0, tail], want)
    assert bool((_areas(v, f).to(DEV)[fidx[0, tail]] > 0).all())


@pytest.mark.gpu
def test_tutorial_step_gradient(built_lib):
    """ico_sphere(4) offset by deform_verts, 5000 samples with normals, a torch point loss; the gradient against the
    float64 restatement fed the same draws."""
    from pytorch3d_b200 import PackedMeshes, sampling, synthetic
    v, f = synthetic.ico_sphere(4)
    v, f = v.float().to(DEV), f.to(DEV)
    deform = torch.full(v.shape, 0.0, device=DEV, requires_grad=True)
    g = torch.Generator().manual_seed(4)
    target = torch.randn(5000, 3, generator=g).to(DEV)
    m = PackedMeshes([v + deform], [f])
    torch.manual_seed(0)
    p, n = sampling.sample_points_from_meshes(m, 5000, return_normals=True)
    loss = ((p[0] - target) ** 2).sum() + (n[0] * target).sum()
    loss.backward()
    from pytorch3d_b200 import _C  # the same draws: replay through the hook
    torch.manual_seed(0)
    seed = torch.randint(0, 1 << 32, (2,), dtype=torch.int64, device=DEV)
    _, _, fidx, bary, _ = _C.sample_points_forward(v, f, m.mesh_to_faces_packed_first_idx(), m.num_faces_per_mesh(),
                                                   5000, False, seed)
    leaf = v.double().cpu().requires_grad_(True)
    rp, rn = restated(leaf, f.cpu(), fidx.cpu(), bary.cpu(), torch.tensor([True]))
    assert _rel(p.detach().cpu(), rp.detach()) <= 1e-6
    (((rp[0] - target.cpu().double()) ** 2).sum() + (rn[0] * target.cpu().double()).sum()).backward()
    assert _rel(deform.grad.cpu(), leaf.grad) <= TOL
