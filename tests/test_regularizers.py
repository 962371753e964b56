"""Mesh regularisers on the GPU (DESIGN.md section 18): `pytorch3d_b200.regularizers`, the `_C.mesh_*` ops,
`_C._mesh_edge_table` and `install_regularizers()`.

The records (tests/golden/make_regularizers_golden.py, reference_golden_regularizers.npz) come from the reference's own
`Meshes` and losses on the CPU, on the scenes of tests/test_normals.py and four more below.  `restated` is a float64
torch restatement of the three losses written from their definitions; it is checked against the records on the CPU and
is the second yardstick of the fused ops on the GPU.
"""
import itertools
import sys
import types

import numpy as np
import pytest
import torch

import test_normals as tn
from helpers import reference

DEV = "cuda"
SCENES = tn.SCENES + ("book", "soup", "faceless", "sliver")
# (case name, loss, keyword argument)
CASES = (("edge_t0", "edge", 0.0), ("edge_t005", "edge", 0.05), ("lap_uniform", "laplacian", "uniform"),
         ("lap_cot", "laplacian", "cot"), ("lap_cotcurv", "laplacian", "cotcurv"), ("normal", "normal", None))


def scene(name):
    """{verts (V,3) f32 packed, faces (F,3) i64 packed, faces_list, nverts}: the scenes of test_normals plus a book of
    64 faces on one edge, a triangle soup, a batch with a mesh of vertices and no faces (one of them at the origin),
    and a near-degenerate sliver."""
    if name in tn.SCENES:
        return tn.scene(name)
    g = torch.Generator().manual_seed(SCENES.index(name) + 101)
    if name == "book":  # 64 pages on the spine (0, 1): 64 * 63 / 2 = 2016 pairs
        pages = torch.randn(64, 3, generator=g)
        v = torch.cat([torch.tensor([[0.0, 0.0, -1.0], [0.0, 0.0, 1.0]]), pages])
        f = torch.stack([torch.zeros(64, dtype=torch.int64), torch.ones(64, dtype=torch.int64),
                         torch.arange(2, 66)], 1)
        return tn._from_lists([v], [f])
    if name == "soup":  # no two faces share an edge
        v = torch.randn(30, 3, generator=g)
        return tn._from_lists([v], [torch.arange(30).reshape(10, 3)])
    if name == "faceless":
        from pytorch3d_b200 import synthetic
        v0, f0 = synthetic.ico_sphere(1)
        v2, f2 = synthetic.torus(6, 5)
        lonely = torch.cat([torch.zeros(1, 3), torch.randn(4, 3, generator=g)])
        return tn._from_lists([v0.float(), lonely, v2.float()], [f0, torch.zeros((0, 3), dtype=torch.int64), f2])
    if name == "sliver":  # face 0 is a sliver whose Heron product rounds to <= 0 and is clamped
        v = torch.tensor([[0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [0.5, 1e-7, 0.0], [0.5, -0.8, 0.1], [0.4, 0.9, -0.2]])
        f = torch.tensor([[0, 1, 2], [1, 0, 3], [2, 1, 4], [0, 2, 4]])
        return tn._from_lists([v], [f])
    raise KeyError(name)


# The records are float32 results of the reference.  Where its float32 arithmetic cancels, they carry rounding noise far
# above float32's resolution: the Laplacian of a smooth closed surface (L v is a small difference of large terms), the
# clamped Heron areas of collinear and sliver faces (the product s (s - A) (s - B) (s - C) cancels), and the normal of
# a face with a repeated vertex, d x d, which is the rounding residue of torch.cross.  Those cases are checked to the
# (loss, gradient) tolerances below; every other case to 1e-5.
ILL_CONDITIONED = {
    ("torus_hetero", "lap_uniform"): (1e-5, 1e-4), ("torus_hetero", "lap_cot"): (1e-5, 2e-3),
    ("torus_hetero", "lap_cotcurv"): (1e-5, 2e-3), ("ico_sphere", "lap_uniform"): (1e-5, 1e-4),
    ("ico_sphere", "lap_cot"): (1e-5, 2e-2), ("ico_sphere", "lap_cotcurv"): (1e-5, 2e-3),
    ("degenerate", "lap_cot"): (1e-5, 1e-1), ("degenerate", "lap_cotcurv"): (5e-2, 1e-1),
    ("degenerate", "normal"): (None, None), ("sliver", "lap_cot"): (1e-5, 2e-2),
    ("sliver", "lap_cotcurv"): (5e-3, 2e-3), ("fan", "lap_cot"): (1e-5, 1e-4),
    ("fan", "lap_cotcurv"): (1e-5, 1e-3), ("fan", "normal"): (1e-5, 1e-4),
    ("book", "lap_cotcurv"): (1e-5, 1e-4),
}
TOL = 1e-5


def tolerances(name, case):
    """(loss, gradient) tolerances against the records; None: the float64 restatement is not compared (the reference
    computes rounding noise)."""
    return ILL_CONDITIONED.get((name, case), (TOL, TOL))


def upstream(name, case):
    return torch.randn((), generator=torch.Generator().manual_seed(SCENES.index(name) * 10 + [c[0] for c in CASES]
                                                                    .index(case) + 1))


# ---------------------------------------------------------------------------------------- float64 restatement ---

def mesh_of_verts(nverts):
    return torch.repeat_interleave(torch.arange(len(nverts)), torch.tensor(nverts))


def restated_edges(faces, nverts):
    """(edges (E,2), face_to_edge (F,3), edges per mesh (N,)): the distinct sorted vertex pairs of the face-edges
    (v1, v2), (v2, v0), (v0, v1), in lexicographic order."""
    F = faces.shape[0]
    fe = torch.cat([faces[:, [1, 2]], faces[:, [2, 0]], faces[:, [0, 1]]]).sort(dim=1).values
    edges, inverse = torch.unique(fe, dim=0, return_inverse=True)
    counts = torch.bincount(mesh_of_verts(nverts)[edges[:, 0]], minlength=len(nverts)) if len(edges) else \
        torch.zeros(len(nverts), dtype=torch.int64)
    return edges, inverse.reshape(3, F).t(), counts


def restated(verts, faces, nverts, loss, arg):
    """The loss in float64 for verts (V,3) (any float dtype, may require grad), faces (F,3) and the per-mesh vertex
    counts."""
    v = verts.double()
    N, V = len(nverts), v.shape[0]
    vm = mesh_of_verts(nverts).to(v.device)
    nv = torch.tensor(nverts, dtype=torch.float64, device=v.device)
    edges, f2e, counts = restated_edges(faces.cpu(), nverts)
    edges, f2e, counts = edges.to(v.device), f2e.to(v.device), counts.to(v.device)
    if loss == "edge":
        lengths = (v[edges[:, 0]] - v[edges[:, 1]]).norm(dim=1)
        return ((lengths - arg) ** 2 / counts[vm[edges[:, 0]]].double()).sum() / N
    if loss == "laplacian":
        if arg == "uniform":
            a, b = edges[:, 0], edges[:, 1]
            deg = torch.zeros(V, dtype=torch.float64, device=v.device)
            deg.index_add_(0, a, torch.ones_like(a, dtype=torch.float64))
            deg.index_add_(0, b, torch.ones_like(b, dtype=torch.float64))
            s = torch.zeros_like(v).index_add(0, a, v[b]).index_add(0, b, v[a])
            y = torch.where(deg[:, None] > 0, s / deg.clamp_min(1)[:, None], torch.zeros_like(s)) - v
        else:
            with torch.no_grad():
                p = v.detach()[faces]
                A = (p[:, 1] - p[:, 2]).norm(dim=1)
                B = (p[:, 0] - p[:, 2]).norm(dim=1)
                C = (p[:, 0] - p[:, 1]).norm(dim=1)
                s = (A + B + C) / 2
                area = (s * (s - A) * (s - B) * (s - C)).clamp(min=1e-12).sqrt()
                cot = torch.stack([B * B + C * C - A * A, A * A + C * C - B * B, A * A + B * B - C * C], 1) / area[:, None] / 4
                L = torch.zeros(V, V, dtype=torch.float64, device=v.device)
                for k in range(3):  # the angle at corner k faces the edge of the other two corners
                    L.index_put_((faces[:, (k + 1) % 3], faces[:, (k + 2) % 3]), cot[:, k], accumulate=True)
                L = L + L.t()
                rows = L.sum(1)
                areas = torch.zeros(V, dtype=torch.float64, device=v.device)
                for k in range(3):
                    areas.index_add_(0, faces[:, k], area)
            if arg == "cot":
                w = torch.where(rows > 0, 1 / torch.where(rows > 0, rows, torch.ones_like(rows)), rows)
                y = (L @ v) * w[:, None] - v
            else:
                w = 0.25 * torch.where(areas > 0, 1 / torch.where(areas > 0, areas, torch.ones_like(areas)),
                                       torch.zeros_like(areas))
                y = (L @ v - rows[:, None] * v) * w[:, None]
        return (y.norm(dim=1) / nv[vm]).sum() / N
    # normal consistency: every pair of face-edges on one edge
    F = faces.shape[0]
    fe_edge = f2e.t().reshape(-1).cpu()  # face-edge id j * F + f
    order = torch.argsort(fe_edge, stable=True).tolist()
    a_idx, b_idx = [], []
    for _, group in itertools.groupby(order, key=lambda c: int(fe_edge[c])):
        a_idx_b = list(group)
        for x, y in itertools.combinations(a_idx_b, 2):
            a_idx.append(x)
            b_idx.append(y)
    if not a_idx:
        return v.sum() * 0.0
    ids = torch.arange(3 * F, device=v.device)
    e = fe_edge.to(v.device)[ids]
    v0, v1 = v[edges[e, 0]], v[edges[e, 1]]
    corners = v[faces[ids % F]]
    n = sum(torch.cross(v1 - v0, corners[:, k] - v0, dim=1) for k in range(3))
    a_idx, b_idx = torch.tensor(a_idx, device=v.device), torch.tensor(b_idx, device=v.device)
    terms = 1 - torch.cosine_similarity(n[a_idx], -n[b_idx], dim=1, eps=1e-8)
    pm = vm[edges[e[a_idx], 0]]
    pairs = torch.bincount(pm, minlength=N).double()
    return (terms / pairs[pm]).sum() / N


# ----------------------------------------------------------------------------------------------------- CPU ---

def test_scenes_cover_the_special_cases():
    book = scene("book")
    edges, f2e, _ = restated_edges(book["faces"], book["nverts"])
    assert int(torch.bincount(f2e.reshape(-1)).max()) == 64
    soup = scene("soup")
    assert int(torch.bincount(restated_edges(soup["faces"], soup["nverts"])[1].reshape(-1)).max()) == 1
    fl = scene("faceless")
    assert fl["faces_list"][1].shape[0] == 0 and fl["nverts"][1] == 5
    s = scene("sliver")
    p = s["verts"][s["faces"][0]]
    A, B, C = (p[1] - p[2]).norm(), (p[0] - p[2]).norm(), (p[0] - p[1]).norm()
    h = (A + B + C) / 2
    assert float(h * (h - A) * (h - B) * (h - C)) < 1e-12
    deg = scene("degenerate")
    assert [3, 3, 5] in deg["faces"].tolist()  # a self-loop edge (3, 3)


@pytest.mark.parametrize("name", SCENES)
def test_restatement_matches_reference_records_cpu(name):
    s = scene(name)
    edges, f2e, counts = restated_edges(s["faces"], s["nverts"])
    for got, field in ((edges, "edges"), (f2e, "faces_to_edges"), (counts, "num_edges_per_mesh")):
        (rec,) = reference("regularizers/%s/%s" % (name, field))
        assert rec.equals(got.to(torch.int64)) is None, field
    for case, loss, arg in CASES:
        tol_loss, tol_grad = tolerances(name, case)
        if tol_loss is None:
            continue
        leaf = s["verts"].double().requires_grad_(True)
        out = restated(leaf, s["faces"], s["nverts"], loss, arg)
        (out * upstream(name, case)).backward()
        (rec,) = reference("regularizers/%s/%s/loss" % (name, case))
        want = float(rec.sample.reshape(-1)[0])
        assert abs(float(out.detach()) - want) <= tol_loss * max(abs(want), 1e-30), (case, float(out.detach()), want)
        (rec,) = reference("regularizers/%s/%s/grad" % (name, case))
        got = rec.rows_of(leaf.grad.float()).astype(np.float64)
        assert np.abs(got - rec.sample).max() <= tol_grad * max(rec.absmax, 1e-30), case


def test_empty_batches_and_bad_methods_cpu():
    from pytorch3d_b200 import PackedMeshes, regularizers
    none = PackedMeshes([], [])
    faceless = PackedMeshes([torch.rand(4, 3)], [torch.zeros((0, 3), dtype=torch.int64)])
    for m in (none, faceless):
        for out in (regularizers.mesh_edge_loss(m), regularizers.mesh_laplacian_smoothing(m),
                    regularizers.mesh_laplacian_smoothing(m, method="bogus"), regularizers.mesh_normal_consistency(m)):
            assert out.shape == (1,) and out.requires_grad and float(out) == 0.0
    one = PackedMeshes([torch.rand(3, 3)], [torch.tensor([[0, 1, 2]])])
    with pytest.raises(ValueError, match=r"Method should be one of \{uniform, cot, cotcurv\}"):
        regularizers.mesh_laplacian_smoothing(one, method="bogus")


def _stand_in_mesh(n=2, V=10, F=4, is_cuda=True, dtype=torch.float32, fdtype=torch.int64):
    dev = torch.device("cuda:0" if is_cuda else "cpu")
    verts = types.SimpleNamespace(is_cuda=is_cuda, dtype=dtype, shape=torch.Size((V, 3)), dim=lambda: 2, device=dev)
    faces = types.SimpleNamespace(is_cuda=is_cuda, dtype=fdtype, shape=torch.Size((F, 3)), dim=lambda: 2, device=dev)
    return types.SimpleNamespace(verts_packed=lambda: verts, faces_packed=lambda: faces)


class _Batch:
    def __init__(self, n=2, **kw):
        self._m = _stand_in_mesh(n=n, **kw)
        self._n = n

    def __len__(self):
        return self._n

    def verts_packed(self):
        return self._m.verts_packed()

    def faces_packed(self):
        return self._m.faces_packed()


def _fake_loss_modules(monkeypatch):
    for n in ["pytorch3d"]:
        m = types.ModuleType(n)
        m.__path__ = []
        monkeypatch.setitem(sys.modules, n, m)
    package = types.ModuleType("pytorch3d.loss")
    package.__path__ = []
    monkeypatch.setitem(sys.modules, "pytorch3d.loss", package)
    modules = {}
    for name, sig in (("mesh_edge_loss", "target_length"), ("mesh_laplacian_smoothing", "method"),
                      ("mesh_normal_consistency", None)):
        mod = types.ModuleType("pytorch3d.loss." + name)
        if sig == "target_length":
            def f(meshes, target_length=0.0):
                return ("ref-edge", target_length)
        elif sig == "method":
            def f(meshes, method="uniform"):
                if method not in ("uniform", "cot", "cotcurv"):
                    raise ValueError("Method should be one of {uniform, cot, cotcurv}")
                return ("ref-lap", method)
        else:
            def f(meshes):
                return ("ref-nc",)
        setattr(mod, name, f)
        setattr(package, name, f)
        monkeypatch.setitem(sys.modules, mod.__name__, mod)
        modules[name] = mod
    return package, modules


def test_install_regularizers_routing_and_uninstall(monkeypatch, built_lib):
    from pytorch3d_b200 import install as inst
    from pytorch3d_b200 import regularizers as ours
    package, modules = _fake_loss_modules(monkeypatch)
    originals = {n: (package.__dict__[n], m.__dict__[n]) for n, m in modules.items()}
    monkeypatch.setattr(ours, "mesh_edge_loss", lambda m, t=0.0: ("b200-edge", t))
    monkeypatch.setattr(ours, "mesh_laplacian_smoothing", lambda m, method="uniform": ("b200-lap", method))
    monkeypatch.setattr(ours, "mesh_normal_consistency", lambda m: ("b200-nc",))
    patched = inst.install_regularizers()
    assert patched == ["pytorch3d.loss", "pytorch3d.loss.mesh_edge_loss", "pytorch3d.loss.mesh_laplacian_smoothing",
                       "pytorch3d.loss.mesh_normal_consistency"]
    good = _Batch()
    for owner in (package, modules["mesh_edge_loss"]):
        assert owner.mesh_edge_loss(good) == ("b200-edge", 0.0)
        assert owner.mesh_edge_loss(good, target_length=0.5) == ("b200-edge", 0.5)
    for owner in (package, modules["mesh_laplacian_smoothing"]):
        assert owner.mesh_laplacian_smoothing(good) == ("b200-lap", "uniform")
        assert owner.mesh_laplacian_smoothing(good, method="cotcurv") == ("b200-lap", "cotcurv")
        with pytest.raises(ValueError, match="Method should be one of"):
            owner.mesh_laplacian_smoothing(good, method="bogus")  # the original raises
    for owner in (package, modules["mesh_normal_consistency"]):
        assert owner.mesh_normal_consistency(good) == ("b200-nc",)
    for bad in (_Batch(is_cuda=False), _Batch(dtype=torch.float64), _Batch(fdtype=torch.int32), _Batch(n=0),
                _Batch(F=(1 << 31) // 6 + 1), _Batch(V=(1 << 31) - 1)):
        assert package.mesh_edge_loss(bad) == ("ref-edge", 0.0)
        assert package.mesh_laplacian_smoothing(bad, "cot") == ("ref-lap", "cot")
        assert package.mesh_normal_consistency(bad) == ("ref-nc",)
    inst.install_regularizers()  # idempotent
    inst.uninstall()
    for n, m in modules.items():
        assert package.__dict__[n] is originals[n][0] and m.__dict__[n] is originals[n][1]
    assert inst._saved_blend == {}


# ----------------------------------------------------------------------------------------------------- GPU ---

def _packed(s, device=DEV):
    from pytorch3d_b200 import PackedMeshes
    verts = list(torch.split(s["verts"].to(device), s["nverts"]))
    return PackedMeshes(verts, [f.to(device) for f in s["faces_list"]])


def _fused(m, loss, arg):
    from pytorch3d_b200 import regularizers as r
    if loss == "edge":
        return r.mesh_edge_loss(m, target_length=arg)
    if loss == "laplacian":
        return r.mesh_laplacian_smoothing(m, method=arg)
    return r.mesh_normal_consistency(m)


def _run(s, loss, arg, g, verts=None):
    m = _packed(s)
    if verts is not None:
        m._verts_packed = verts
    m.requires_grad_(True)
    out = _fused(m, loss, arg)
    (out * g.to(DEV)).backward()
    return out.detach(), m.verts_packed().grad


@pytest.mark.gpu
@pytest.mark.parametrize("name", SCENES)
def test_edge_table_matches_reference_records(built_lib, name):
    from pytorch3d_b200 import _C
    s = scene(name)
    m = _packed(s)
    edges, f2e, counts = _C._mesh_edge_table(m.faces_packed(), m.verts_packed().shape[0],
                                             m.mesh_to_verts_packed_first_idx(), m.num_verts_per_mesh())
    for got, field in ((edges, "edges"), (f2e, "faces_to_edges"), (counts, "num_edges_per_mesh")):
        (rec,) = reference("regularizers/%s/%s" % (name, field))
        assert rec.equals(got.cpu()) is None, field


@pytest.mark.gpu
@pytest.mark.parametrize("name", SCENES)
@pytest.mark.parametrize("case", [c[0] for c in CASES])
def test_losses_match_reference_records_and_restatement(built_lib, name, case):
    _, loss, arg = next(c for c in CASES if c[0] == case)
    s = scene(name)
    g = upstream(name, case)
    out, grad = _run(s, loss, arg, g)
    assert out.shape == () and out.dtype == torch.float32
    tol_loss, tol_grad = tolerances(name, case)
    if tol_loss is None:  # the fused op rounds d x d as the reference does, so it follows the records
        tol_loss, tol_grad = TOL, TOL
    (rec,) = reference("regularizers/%s/%s/loss" % (name, case))
    want = float(rec.sample.reshape(-1)[0])
    assert abs(float(out) - want) <= tol_loss * max(abs(want), 1e-30), (float(out), want)
    (rec,) = reference("regularizers/%s/%s/grad" % (name, case))
    got = rec.rows_of(grad.cpu()).astype(np.float64)
    assert np.array_equal(np.isnan(got), np.isnan(rec.sample)), "NaN only where the records have NaN"
    ok = ~np.isnan(rec.sample)
    err = np.abs(got[ok] - rec.sample[ok]).max(initial=0.0) / max(rec.absmax, 1e-30)
    assert err <= tol_grad, err
    if tolerances(name, case)[0] is None:
        return
    leaf = s["verts"].double().requires_grad_(True)
    r = restated(leaf, s["faces"], s["nverts"], loss, arg)
    (r * g).backward()
    r = float(r.detach())
    assert abs(float(out) - r) <= tol_loss * max(abs(r), 1e-30), (float(out), r)
    full = leaf.grad
    err = float((grad.cpu().double() - full).abs().max()) / max(float(full.abs().max()), 1e-30)
    assert err <= tol_grad, err


@pytest.mark.gpu
def test_exact_zero_gradients(built_lib):
    """A vertex whose edges all have zero length gets an exactly zero edge-loss gradient; a Laplacian row with
    |y| = 0 (an isolated vertex at the origin) gets an exactly zero gradient."""
    from pytorch3d_b200 import PackedMeshes, regularizers
    v = torch.tensor([[0.3, 0.2, 0.1], [0.3, 0.2, 0.1], [1.0, 0.0, 0.0], [2.0, 1.0, 0.5], [0.0, 0.0, 0.0]],
                     device=DEV)
    f = torch.tensor([[0, 0, 1], [2, 3, 2]], device=DEV)  # only zero-length edges at 0 and 1, self-loops
    for t in (0.0, 0.05):
        m = PackedMeshes([v.clone()], [f]).requires_grad_(True)
        regularizers.mesh_edge_loss(m, target_length=t).backward()
        gv = m.verts_packed().grad
        assert torch.equal(gv[:2], torch.zeros_like(gv[:2])) and bool(gv[2:4].ne(0).any())
    for method in ("uniform", "cot", "cotcurv"):
        m = PackedMeshes([v.clone()], [f]).requires_grad_(True)
        regularizers.mesh_laplacian_smoothing(m, method=method).backward()
        assert torch.equal(m.verts_packed().grad[4], torch.zeros(3, device=DEV))


@pytest.mark.gpu
def test_soup_divergence_is_a_connected_zero(built_lib):
    """The reference returns a detached tensor([0.]) when no edge has two faces; the fused op returns a 0-dim zero
    connected to the verts, with a zero gradient."""
    s = scene("soup")
    out, grad = _run(s, "normal", None, torch.tensor(1.0))
    assert out.shape == () and float(out) == 0.0
    assert torch.equal(grad, torch.zeros_like(grad))


@pytest.mark.gpu
def test_deterministic_and_no_host_sync(built_lib):
    s = scene("torus_hetero")
    m = _packed(s)
    verts = m.verts_packed()
    g = torch.tensor(0.7, device=DEV)

    def run():
        outs = []
        for _, loss, arg in CASES:
            m._verts_packed = verts.detach().clone().requires_grad_(True)
            out = _fused(m, loss, arg)
            (out * g).backward()
            outs += [out.detach(), m._verts_packed.grad]
        return outs

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
def test_unaligned_and_non_contiguous_verts(built_lib):
    s = scene("ico_sphere")
    V = s["verts"].shape[0]
    buf = torch.empty(3 * V + 1, device=DEV)
    buf[1:] = s["verts"].reshape(-1).to(DEV)
    layouts = (buf[1:].view(V, 3), s["verts"].to(DEV).t().contiguous().t())
    for case, loss, arg in CASES:
        g = upstream("ico_sphere", case)
        want = _run(s, loss, arg, g)
        for vv in layouts:
            leaf = vv.detach().requires_grad_(True)
            out = _fused(_with_verts(s, leaf), loss, arg)
            (out * g.to(DEV)).backward()
            assert torch.equal(out.detach(), want[0]) and torch.equal(leaf.grad, want[1]), case


def _with_verts(s, verts):
    m = _packed(s)
    m._verts_packed = verts
    return m


@pytest.mark.gpu
def test_argument_errors(built_lib):
    from pytorch3d_b200 import _C, _lib
    v = torch.rand(4, 3, device=DEV)
    f = torch.tensor([[0, 1, 2]], device=DEV)
    first, num = torch.zeros(1, dtype=torch.int64, device=DEV), torch.full((1,), 4, dtype=torch.int64, device=DEV)
    with pytest.raises(RuntimeError, match="Float"):
        _C.mesh_edge_loss_forward(v.double(), f, first, num, 0.0)
    with pytest.raises(RuntimeError, match="Long"):
        _C.mesh_normal_consistency_forward(v, f.int(), first, num)
    with pytest.raises(RuntimeError, match="mesh_num_verts"):
        _C.mesh_laplacian_smoothing_forward(v, f, first, num[:0], "cot")
    with pytest.raises(ValueError, match="Method should be one of"):
        _C.mesh_laplacian_smoothing_forward(v, f, first, num, "bogus")
    loss, ws = _C.mesh_edge_loss_forward(v, f, first, num, 0.0)
    with pytest.raises(RuntimeError, match="workspace"):
        _C.mesh_edge_loss_backward(torch.ones((), device=DEV), v, f, first, num, 0.0, ws[:-1])
    lib = _lib.load()
    assert lib.b200r_mesh_edge_loss_forward(None, 2 ** 31, None, 1, None, None, 1, 0.0, None, 0, None, None) != 0
    assert "vertices" in _lib.last_error()
    assert lib.b200r_mesh_normal_consistency_forward(None, 4, None, 2 ** 31 // 6 + 1, None, None, 1, None, 0, None,
                                                     None) != 0
    assert "faces" in _lib.last_error()
    assert lib.b200r_mesh_laplacian_smoothing_forward(None, 4, None, 1, None, None, 1, 7, None, 0, None, None) != 0


@pytest.mark.gpu
def test_64_bit_offsets(built_lib):
    """A verts array past 2^31 floats (V = 716,000,000) with faces on its last vertices: every loss and gradient
    equals that of the same faces on a copy of those vertices alone.  Skipped below 48 GB of free device memory."""
    free, _ = torch.cuda.mem_get_info()
    if free < 48 * 2 ** 30:
        pytest.skip("needs 48 GB of free device memory, %.1f GB free" % (free / 2 ** 30))
    V = 716_000_000
    gen = torch.Generator().manual_seed(9)
    tail = torch.rand(8, 3, generator=gen).to(DEV)
    # well-conditioned faces: the Laplacian's weight 1 / V differs from 1 / 8, so rounding differs, and a clamped
    # face's cancelling cotangents would turn that into noise
    local = torch.tensor([[0, 1, 2], [2, 1, 3], [4, 5, 6], [7, 6, 5], [3, 4, 2], [1, 0, 5]], device=DEV)

    def one(verts, faces, nverts, loss, arg):
        from pytorch3d_b200 import PackedMeshes
        m = PackedMeshes([verts], [faces])
        m._verts_packed = verts.requires_grad_(True)
        out = _fused(m, loss, arg)
        out.backward()
        return out.detach(), verts.grad[-8:].clone()

    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    for _, loss, arg in CASES:
        want = one(tail.clone(), local, [8], loss, arg)
        verts = torch.zeros((V, 3), device=DEV)
        verts[-8:] = tail
        got = one(verts, local + (V - 8), [V], loss, arg)
        del verts
        # the vertex weight 1 / V differs: compare the unweighted Laplacian through the ratio of the weights
        scale = 8.0 / V if loss == "laplacian" else 1.0
        assert torch.allclose(got[0], want[0] * scale, rtol=1e-5, atol=0), loss
        err = float((got[1] - want[1] * scale).abs().max()) / float((want[1] * scale).abs().max())
        assert err <= 1e-5, (loss, arg, err)
        torch.cuda.empty_cache()
    assert torch.cuda.max_memory_allocated() < 48 * 2 ** 30


@pytest.mark.gpu
def test_tutorial_fitting_step_matches_float64_losses(built_lib):
    """One step of the reference tutorials' fitting loop: an ico_sphere(3) offset by deform_verts, rendered by the
    fused rasterizer and sigmoid_alpha_blend; silhouette MSE + edge + 0.01 normal + laplacian.  The gradient to
    deform_verts equals that of the same step with the float64 restated losses to 1e-4 of its largest magnitude."""
    from pytorch3d_b200 import PackedMeshes, synthetic
    from pytorch3d_b200.blending import BlendParams, sigmoid_alpha_blend
    from pytorch3d_b200.rasterize_meshes import rasterize_meshes
    v0, f0 = synthetic.ico_sphere(3)
    src = (v0.float() * 0.6 + torch.tensor([0.0, 0.0, 2.0])).to(DEV)
    faces = f0.to(DEV)
    target = (torch.rand(1, 64, 64, generator=torch.Generator().manual_seed(4)) > 0.5).float().to(DEV)
    deform0 = 0.01 * torch.randn(src.shape, generator=torch.Generator().manual_seed(5)).to(DEV)

    def step(fused):
        deform = deform0.clone().requires_grad_(True)
        verts = src + deform
        m = PackedMeshes([verts], [faces])
        m._verts_packed = verts
        p2f, zbuf, bary, dists = rasterize_meshes(m, 64, blur_radius=1e-4, faces_per_pixel=8)
        frags = types.SimpleNamespace(pix_to_face=p2f, bary_coords=bary, zbuf=zbuf, dists=dists)
        colors = torch.ones(p2f.shape + (3,), device=DEV)
        sil = sigmoid_alpha_blend(colors, frags, BlendParams(sigma=1e-4))[..., 3]
        loss = ((sil - target) ** 2).mean()
        if fused:
            loss = loss + _fused(m, "edge", 0.0) + 0.01 * _fused(m, "normal", None) + _fused(m, "laplacian", "uniform")
        else:
            nv = [verts.shape[0]]
            loss = loss + (restated(verts, faces, nv, "edge", 0.0) + 0.01 * restated(verts, faces, nv, "normal", None)
                           + restated(verts, faces, nv, "laplacian", "uniform")).float()
        loss.backward()
        return deform.grad

    got, want = step(True), step(False)
    assert float(want.abs().max()) > 0
    assert float((got - want).abs().max()) <= 1e-4 * float(want.abs().max())
