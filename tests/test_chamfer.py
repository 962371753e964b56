"""Chamfer distance (pytorch3d_b200.chamfer, DESIGN.md section 21): the fused search against the reference's own CUDA
kernel recompiled for sm_90a (oracle/_ref/ref_knn_cuda.so), bit for bit; the losses and gradients against the
records of the reference's CPU chamfer_distance (tests/golden/make_chamfer_golden.py) and a float64 restatement of
pytorch3d/loss/chamfer.py; determinism, host synchronisations, errors and `install_chamfer()`.

`restated` is written from the reference's formulas: the distance of each point to the neighbour it is given, with
the backward of the reference's KNearestNeighborBackwardKernel (norm 1 sends -g at equal coordinates), the masks,
weights, F.cosine_similarity(eps=1e-6) term and reductions of chamfer.py, evaluated by torch's float64 autograd, so
the tie rules of max(1) and torch.maximum are torch's own.
"""
import itertools
import os
import sys
import types
import warnings

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import GOLDEN_DIR

DEV = "cuda"
TOL = 1e-5


# ---- scenes and options (shared with tests/golden/make_chamfer_golden.py) -----------------------------------------

def chamfer_scenes():
    g = torch.Generator().manual_seed(21)
    s = {}
    xn = torch.randn(2, 37, 3, generator=g)
    xn[0, 3] = 0.0          # a zero normal
    xn[1, 5] *= 1e-7        # a normal below eps
    s["uniform"] = dict(x=torch.randn(2, 37, 3, generator=g), y=torch.randn(2, 29, 3, generator=g), xn=xn,
                        yn=torch.randn(2, 29, 3, generator=g), xl=None, yl=None,
                        w=torch.tensor([0.5, 2.0]))
    s["ragged"] = dict(x=torch.randn(3, 20, 3, generator=g), y=torch.randn(3, 17, 3, generator=g),
                       xn=torch.randn(3, 20, 3, generator=g), yn=torch.randn(3, 17, 3, generator=g),
                       xl=torch.tensor([20, 0, 11]), yl=torch.tensor([17, 9, 0]), w=torch.tensor([1.0, 0.0, 3.0]))
    # integer coordinates: many exact ties in distance, and coordinates equal to their neighbour's (norm 1 signs)
    s["grid"] = dict(x=torch.randint(0, 3, (2, 24, 3), generator=g).float(),
                     y=torch.randint(0, 3, (2, 20, 3), generator=g).float(),
                     xn=torch.randint(-1, 2, (2, 24, 3), generator=g).float(),
                     yn=torch.randint(-1, 2, (2, 20, 3), generator=g).float(), xl=torch.tensor([24, 13]), yl=None,
                     w=torch.tensor([1.0, 1.0]))
    return s


def _options():
    out = {}
    pairs = [("mean", "mean"), ("mean", "sum"), ("mean", None), ("sum", "mean"), ("sum", "sum"), ("sum", None),
             ("max", "mean"), ("max", "sum"), ("max", None), (None, None)]
    for (pr, br), single, normals, weights in itertools.product(pairs, (False, True), (False, True),
                                                                (None, "w")):
        if pr == "max" and normals:
            continue
        out["%s_%s_n2_s%d_nrm%d_%s" % (pr, br, single, normals, weights)] = dict(
            point_reduction=pr, batch_reduction=br, norm=2, single_directional=single, normals=normals,
            weights=weights, abs_cosine=True)
    for pr, br in pairs:
        out["%s_%s_n1" % (pr, br)] = dict(point_reduction=pr, batch_reduction=br, norm=1, single_directional=False,
                                          normals=pr != "max", weights="w", abs_cosine=True)
    for pr, br in (("mean", "mean"), ("sum", None), (None, None)):
        out["%s_%s_cos" % (pr, br)] = dict(point_reduction=pr, batch_reduction=br, norm=2, single_directional=False,
                                           normals=True, weights=None, abs_cosine=False)
    for pr, br in (("mean", "mean"), ("max", None), (None, None)):
        out["%s_%s_w0" % (pr, br)] = dict(point_reduction=pr, batch_reduction=br, norm=2, single_directional=False,
                                          normals=False, weights="w0", abs_cosine=True)
    out["wneg"] = dict(point_reduction="mean", batch_reduction="mean", norm=2, single_directional=False,
                       normals=False, weights="wneg", abs_cosine=True)
    return out


OPTIONS = _options()


def upstream(shape, k):
    g = torch.Generator().manual_seed(1000 + 17 * k + sum(shape))
    return 0.5 + torch.rand(shape, generator=g, dtype=torch.float64)


def _weights(scene, kind):
    if kind is None:
        return None
    w = scene["w"]
    if kind == "w0":
        return torch.zeros_like(w)
    if kind == "wneg":
        return -w
    return w


def _outputs(loss, loss_normals):
    """The output tensors in a fixed order, named as the records."""
    out = {}
    for name, v in (("loss", loss), ("loss_normals", loss_normals)):
        if isinstance(v, tuple):
            out[name], out[name + "_y"] = v
        elif v is not None:
            out[name] = v
    return out


def run_with_grads(cd, scene, opts, device="cpu", dtype=torch.float32):
    """cd(x, y, ...) on the scene with the options; returns its outputs and the gradients of sum(out * upstream)."""
    t = {k: (v.to(device=device, dtype=dtype) if v is not None and v.is_floating_point() else
             (v.to(device) if v is not None else None)) for k, v in scene.items()}
    x, y = t["x"].clone().requires_grad_(), t["y"].clone().requires_grad_()
    xn = t["xn"].clone().requires_grad_() if opts["normals"] else None
    yn = t["yn"].clone().requires_grad_() if opts["normals"] else None
    w = _weights(scene, opts["weights"])
    w = w.to(device=device, dtype=dtype) if w is not None else None
    loss, ln = cd(x, y, x_lengths=t["xl"], y_lengths=t["yl"], x_normals=xn, y_normals=yn, weights=w,
                  batch_reduction=opts["batch_reduction"], point_reduction=opts["point_reduction"], norm=opts["norm"],
                  single_directional=opts["single_directional"], abs_cosine=opts["abs_cosine"])
    outs = _outputs(loss, ln)
    total = sum((o.double() * upstream(tuple(o.shape), k).to(device)).sum() for k, o in enumerate(outs.values()))
    leaves = {"grad_x": x, "grad_y": y, "grad_x_normals": xn, "grad_y_normals": yn}
    leaves = {k: v for k, v in leaves.items() if v is not None}
    grads = torch.autograd.grad(total, list(leaves.values()), allow_unused=True)
    res = {k: v.detach().double().cpu().numpy() for k, v in outs.items()}
    for (k, leaf), gr in zip(leaves.items(), grads):
        res[k] = (gr if gr is not None else torch.zeros_like(leaf)).detach().double().cpu().numpy()
    return res


# ---- float64 restatement ------------------------------------------------------------------------------------------

class _PairDist(torch.autograd.Function):
    """dist(a, b) with the reference's knn backward: 2 g (a - b) for norm 2, g sign where sign = 1 if a > b else -1."""

    @staticmethod
    def forward(ctx, a, b, norm):
        ctx.save_for_backward(a, b)
        ctx.norm = norm
        d = a - b
        return (d * d).sum(-1) if norm == 2 else d.abs().sum(-1)

    @staticmethod
    def backward(ctx, g):
        a, b = ctx.saved_tensors
        diff = 2.0 * g[..., None] * (a - b) if ctx.norm == 2 else g[..., None] * torch.where(a > b, 1.0, -1.0)
        return diff, -diff, None


def restated(scene, opts, idx_x, idx_y):
    """chamfer.py in float64 at the given neighbour indices (N, P1) and (N, P2) -> run_with_grads' dict."""
    def cd(x, y, x_lengths, y_lengths, x_normals, y_normals, weights, batch_reduction, point_reduction, norm,
           single_directional, abs_cosine):
        N, P1, P2 = x.shape[0], x.shape[1], y.shape[1]
        xl = x_lengths if x_lengths is not None else torch.full((N,), P1)
        yl = y_lengths if y_lengths is not None else torch.full((N,), P2)

        def one(a, b, la, lb, na, nb, idx):
            P = a.shape[1]
            gi = idx.clamp(0, b.shape[1] - 1)[..., None].expand(-1, -1, 3)
            valid = torch.arange(P)[None] < la[:, None]
            has_t = (lb > 0)[:, None]
            dist = _PairDist.apply(a, b.gather(1, gi), norm)
            dist = torch.where(valid & has_t, dist, torch.zeros_like(dist))
            if weights is not None:
                dist = dist * weights.view(N, 1)
            cn = None
            if na is not None:
                nbg = torch.where(has_t[..., None], nb.gather(1, gi), torch.zeros_like(na))
                cos = F.cosine_similarity(na, nbg, dim=2, eps=1e-6)
                cn = 1 - (torch.abs(cos) if abs_cosine else cos)
                cn = torch.where(valid, cn, torch.zeros_like(cn))
                if weights is not None:
                    cn = cn * weights.view(N, 1)
            if point_reduction == "max":
                dist = dist.max(1).values
            elif point_reduction is not None:
                lc = la.clamp(min=1)
                dist = dist.sum(1)
                cn = cn.sum(1) if cn is not None else None
                if point_reduction == "mean":
                    dist = dist / lc
                    cn = cn / lc if cn is not None else None
            return dist, cn

        cx, cnx = one(x, y, xl, yl, x_normals, y_normals, idx_x)
        if single_directional:
            loss, ln = cx, cnx
        else:
            cy, cny = one(y, x, yl, xl, y_normals, x_normals, idx_y)
            if point_reduction == "max":
                loss, ln = torch.maximum(cx, cy), None
            elif point_reduction is not None:
                loss, ln = cx + cy, (cnx + cny if cnx is not None else None)
            else:
                loss, ln = (cx, cy), ((cnx, cny) if cnx is not None else None)
        if batch_reduction is not None:
            loss = loss.sum()
            ln = ln.sum() if ln is not None else None
            if batch_reduction == "mean":
                div = max(N, 1) if weights is None else weights.sum()
                loss = loss / div
                ln = ln / div if ln is not None else None
        return loss, ln

    return run_with_grads(cd, scene, opts, dtype=torch.float64)


def cpu_reference_nn(a, b, la, lb):
    """knn_cpu.cpp's neighbours: float32 diff * diff summed without FMA, the first minimum (tie rule: lowest index)."""
    a, b = a.numpy(), b.numpy()
    N, P = a.shape[0], a.shape[1]
    idx = np.zeros((N, P), dtype=np.int64)
    for n in range(N):
        lq = P if la is None else int(la[n])
        lt = b.shape[1] if lb is None else int(lb[n])
        if lt <= 0:
            continue
        for p in range(lq):
            dd = a[n, p][None] - b[n, :lt]
            d = (dd[:, 0] * dd[:, 0] + dd[:, 1] * dd[:, 1]) + dd[:, 2] * dd[:, 2]
            idx[n, p] = int(np.argmin(d))
    return torch.from_numpy(idx)


def _rel_err(got, want):
    scale = max(float(np.abs(want).max()) if want.size else 0.0, 1e-30)
    return float(np.abs(got - want).max()) / scale if want.size else 0.0


_records = None


def _record(sname, oname):
    """The fields of record chamfer/<scene>/<option>/0 of reference_golden_chamfer.npz."""
    global _records
    if _records is None:
        _records = {}
        data = np.load(os.path.join(GOLDEN_DIR, "reference_golden_chamfer.npz"))
        for key in data.files:
            name, _, field = key.rsplit("/", 2)
            _records.setdefault(name, {})[field] = data[key]
    return _records["chamfer/%s/%s" % (sname, oname)]


def _rec_dict(rec):
    return dict(rec)


# ---- CPU tests ----------------------------------------------------------------------------------------------------

def _norm2_opts(oname):
    return OPTIONS[oname]["norm"] == 2


@pytest.mark.parametrize("sname", sorted(chamfer_scenes()))
def test_restatement_matches_records_cpu(sname):
    scene = chamfer_scenes()[sname]
    ix = cpu_reference_nn(scene["x"], scene["y"], scene["xl"], scene["yl"])
    iy = cpu_reference_nn(scene["y"], scene["x"], scene["yl"], scene["xl"])
    checked = 0
    for oname, opts in OPTIONS.items():
        rec = _rec_dict(_record(sname, oname))
        if "error" in rec or opts["weights"] in ("w0", "wneg") or opts["norm"] != 2:
            continue  # the zero-weight result and the errors are checked on their own; norm 1 below
        mine = restated(scene, opts, ix, iy)
        for k, v in mine.items():
            assert k in rec, (oname, k)
            assert _rel_err(v, rec[k]) < TOL, (sname, oname, k, _rel_err(v, rec[k]))
        checked += 1
    assert checked > 40


def test_records_cover_errors_and_zero_weights_cpu():
    rec = _rec_dict(_record("uniform", "wneg"))
    assert bytes(rec["error"]).decode() == "weights cannot be negative."
    z = _rec_dict(_record("uniform", "mean_mean_w0"))
    assert z["loss"].shape == () and z["loss"] == 0.0
    z = _rec_dict(_record("uniform", "None_None_w0"))
    assert z["loss"].shape == (2, 2) and z["loss_normals"].shape == (2, 2)


def _cos_grad_as_kernel(a, b, g, eps=1e-6):
    """The kernel's cosine backward (chamfer.cu: cosine_backward), in float64."""
    sa, sb = np.linalg.norm(a), np.linalg.norm(b)
    ma, mb = max(sa, eps), max(sb, eps)
    gu = g * b / mb
    gm = -np.sum(gu * (a / ma) / ma)
    k = 0.0 if sa == 0 else gm / sa
    return gu / ma + a * k


def test_cosine_term_matches_torch_cpu():
    g = torch.Generator().manual_seed(3)
    cases = [torch.randn(2, 3, generator=g, dtype=torch.float64) for _ in range(20)]
    cases += [torch.stack([torch.zeros(3, dtype=torch.float64), torch.randn(3, generator=g, dtype=torch.float64)]),
              torch.stack([1e-7 * torch.randn(3, generator=g, dtype=torch.float64),
                           torch.randn(3, generator=g, dtype=torch.float64)]),
              torch.stack([3e-7 * torch.ones(3, dtype=torch.float64), 2e-7 * torch.ones(3, dtype=torch.float64)])]
    for ab in cases:
        a, b = ab[0].clone().requires_grad_(), ab[1].clone().requires_grad_()
        cos = F.cosine_similarity(a[None], b[None], dim=1, eps=1e-6)[0]
        na, nb = max(float(a.detach().norm()), 1e-6), max(float(b.detach().norm()), 1e-6)
        assert abs(float(cos) - float((a / na * b / nb).sum())) <= 1e-15
        ga, gb = torch.autograd.grad(cos * 0.7, (a, b))
        np.testing.assert_allclose(_cos_grad_as_kernel(ab[0].numpy(), ab[1].numpy(), 0.7), ga.numpy(), rtol=1e-9,
                                   atol=1e-12 * max(1.0, float(ga.abs().max())))
        np.testing.assert_allclose(_cos_grad_as_kernel(ab[1].numpy(), ab[0].numpy(), 0.7), gb.numpy(), rtol=1e-9,
                                   atol=1e-12 * max(1.0, float(gb.abs().max())))


def test_host_errors_cpu():
    from pytorch3d_b200.chamfer import chamfer_distance as cd
    x, y = torch.zeros(2, 4, 3), torch.zeros(2, 5, 3)
    cases = [
        (dict(batch_reduction="x"), 'batch_reduction must be one of ["mean", "sum"] or None'),
        (dict(point_reduction="x"), 'point_reduction must be one of ["mean", "sum", "max"] or None'),
        (dict(point_reduction=None), "Batch reduction must be None if point_reduction is None"),
        (dict(norm=3), "Support for 1 or 2 norm."),
        (dict(point_reduction="max", x_normals=x), 'Normals must be None if point_reduction is "max"'),
        (dict(x_lengths=torch.zeros(3, dtype=torch.int64)), "Expected lengths to be of shape (N,)"),
        (dict(x_normals=torch.zeros(2, 4)), "Expected normals to be of shape (N, P, 3"),
        (dict(weights=torch.ones(3)), "weights must be of shape (N,)."),
    ]
    for kw, msg in cases:
        with pytest.raises(ValueError) as e:
            cd(x, y, **kw)
        assert str(e.value) == msg, (kw, str(e.value))
    with pytest.raises(ValueError, match="Expected points to be of shape"):
        cd(torch.zeros(2, 3), y)
    with pytest.raises(ValueError, match="y does not have the correct shape."):
        cd(x, torch.zeros(3, 5, 3))
    with pytest.raises(ValueError, match="should be either Pointclouds"):
        cd(x, [1, 2])
    # a data check the reference makes earlier wins over a later host-decided error
    with pytest.raises(ValueError, match="A length value was too long"):
        cd(x, torch.zeros(3, 5, 3), x_lengths=torch.tensor([5, 1]))


def _fake_loss_modules(monkeypatch):
    m = types.ModuleType("pytorch3d")
    m.__path__ = []
    monkeypatch.setitem(sys.modules, "pytorch3d", m)
    package = types.ModuleType("pytorch3d.loss")
    package.__path__ = []
    mod = types.ModuleType("pytorch3d.loss.chamfer")

    def chamfer_distance(x, y, x_lengths=None, y_lengths=None, x_normals=None, y_normals=None, weights=None,
                         batch_reduction="mean", point_reduction="mean", norm=2, single_directional=False,
                         abs_cosine=True):
        return ("ref", point_reduction, norm)

    mod.chamfer_distance = chamfer_distance
    package.chamfer_distance = chamfer_distance
    monkeypatch.setitem(sys.modules, package.__name__, package)
    monkeypatch.setitem(sys.modules, mod.__name__, mod)
    return package, mod, chamfer_distance


def test_install_chamfer_routing_and_uninstall_cpu(monkeypatch):
    from pytorch3d_b200 import install as inst
    package, mod, original = _fake_loss_modules(monkeypatch)
    calls = []
    from pytorch3d_b200 import chamfer as ours
    monkeypatch.setattr(ours, "chamfer_distance", lambda *a: calls.append(a) or ("b200",))
    assert inst.install_chamfer() == ["pytorch3d.loss", "pytorch3d.loss.chamfer"]
    x = torch.zeros(2, 4, 3)
    for owner in (package, mod):
        assert owner.chamfer_distance(x, x)[0] == "ref"                    # CPU
        assert owner.chamfer_distance(x.double(), x.double())[0] == "ref"  # float64
        assert owner.chamfer_distance(torch.zeros(2, 4, 2), torch.zeros(2, 4, 2))[0] == "ref"  # D != 3
    assert not inst._chamfer_fused(x, x, None, None, None, None, None, 2, "mean")
    if torch.cuda.is_available():
        xc = x.cuda()
        assert package.chamfer_distance(xc, xc) == ("b200",)
        w = torch.ones(2, device="cuda", requires_grad=True)
        assert package.chamfer_distance(xc, xc, weights=w)[0] == "ref"
        assert package.chamfer_distance(xc, x)[0] == "ref"  # mixed devices
    inst.install_chamfer()  # idempotent
    inst.uninstall()
    assert package.chamfer_distance is original and mod.chamfer_distance is original
    assert not any(k[1] == "chamfer_distance" for k in inst._saved_blend)


# ---- GPU tests ----------------------------------------------------------------------------------------------------

def _ref_cuda():
    from oracle import build_ref_knn
    mod = build_ref_knn.load(cuda=True)
    if mod is None:
        pytest.skip("oracle/_ref/ref_knn_cuda.so not built (the reference sources were absent at build time)")
    return mod


def _same_bits(a, b):
    a, b = a.detach().cpu(), b.detach().cpu()
    nan = torch.isnan(a) & torch.isnan(b)
    return bool(((a.view(torch.int32) == b.view(torch.int32)) | nan).all())


def _search_cases():
    g = torch.Generator().manual_seed(5)
    cases = {}
    cases["uniform"] = (torch.rand(2, 1000, 3, generator=g), torch.rand(2, 777, 3, generator=g), None, None)
    cases["grid_ties"] = (torch.randint(0, 4, (2, 600, 3), generator=g).float(),
                          torch.randint(0, 4, (2, 650, 3), generator=g).float(), None, None)
    base = torch.rand(1, 300, 3, generator=g)
    cases["duplicates"] = (torch.rand(1, 500, 3, generator=g), torch.cat([base, base, base[:, :50]], 1), None, None)
    cases["ragged"] = (torch.randn(4, 300, 3, generator=g), torch.randn(4, 280, 3, generator=g),
                       torch.tensor([300, 0, 17, 250]), torch.tensor([0, 280, 5, 1]))
    for p1, p2 in ((1, 31), (31, 33), (33, 1), (4097, 33), (1, 4097)):
        cases["sizes_%d_%d" % (p1, p2)] = (torch.randn(2, p1, 3, generator=g), torch.randn(2, p2, 3, generator=g),
                                           None, None)
    x, y = torch.randn(2, 200, 3, generator=g), torch.randn(2, 300, 3, generator=g)
    y[0, 0, 1] = float("nan")   # NaN at target 0: every query of cloud 0 keeps (NaN, 0)
    y[1, 0, 2] = float("inf")   # inf at target 0
    y[1, 7, 0] = float("nan")
    y[1, 9, 1] = float("inf")
    x[1, 3, 0] = float("inf")   # a query at infinity: every distance inf or NaN
    x[0, 4, 2] = float("nan")
    cases["nan_inf"] = (x, y, None, None)
    cases["split_merge"] = (torch.randn(1, 5000, 3, generator=g), torch.randn(1, 6000, 3, generator=g), None, None)
    cases["unsplit"] = (torch.randn(8, 20000, 3, generator=g), torch.randn(8, 3000, 3, generator=g), None, None)
    return cases


@pytest.mark.gpu
@pytest.mark.parametrize("norm", [1, 2])
@pytest.mark.parametrize("case", sorted(_search_cases()))
def test_search_bit_identical_to_reference_kernel(built_lib, case, norm):
    from pytorch3d_b200 import _C
    ref = _ref_cuda()
    x, y, xl, yl = _search_cases()[case]
    x, y = x.to(DEV), y.to(DEV)
    N = x.shape[0]
    xl = (xl if xl is not None else torch.full((N,), x.shape[1])).to(DEV)
    yl = (yl if yl is not None else torch.full((N,), y.shape[1])).to(DEV)
    dx, ix, dy, iy = _C._chamfer_nn(x, y, xl, yl, norm)
    rix, rdx = ref.knn_points_idx(x, y, xl, yl, norm, 1, -1)
    riy, rdy = ref.knn_points_idx(y, x, yl, xl, norm, 1, -1)
    assert _same_bits(dx, rdx[..., 0]) and torch.equal(ix, rix[..., 0]), case
    assert _same_bits(dy, rdy[..., 0]) and torch.equal(iy, riy[..., 0]), case


def _fused():
    from pytorch3d_b200.chamfer import chamfer_distance
    return chamfer_distance


@pytest.mark.gpu
@pytest.mark.parametrize("sname", sorted(chamfer_scenes()))
def test_losses_and_gradients(built_lib, sname):
    from pytorch3d_b200 import _C
    scene = chamfer_scenes()[sname]
    dev_scene = {k: (v.to(DEV) if v is not None else None) for k, v in scene.items()}
    _, ix, _, iy = _C._chamfer_nn(dev_scene["x"], dev_scene["y"], dev_scene["xl"], dev_scene["yl"], 2)
    _, ix1, _, iy1 = _C._chamfer_nn(dev_scene["x"], dev_scene["y"], dev_scene["xl"], dev_scene["yl"], 1)
    for oname, opts in OPTIONS.items():
        rec = _rec_dict(_record(sname, oname))
        if "error" in rec:
            with pytest.raises(ValueError) as e:
                run_with_grads(_fused(), scene, opts, device=DEV)
            assert str(e.value) == bytes(rec["error"]).decode()
            continue
        got = run_with_grads(_fused(), scene, opts, device=DEV)
        assert sorted(got) == sorted(k for k in rec if k != "error"), oname
        n1 = opts["norm"] == 1
        want = restated(scene, opts, (ix1 if n1 else ix).cpu(), (iy1 if n1 else iy).cpu())
        for k in got:
            assert got[k].shape == rec[k].shape, (oname, k)
            if k.startswith("loss"):
                assert _rel_err(got[k], rec[k]) < TOL, (sname, oname, k, _rel_err(got[k], rec[k]))
            if opts["weights"] == "w0":
                assert np.array_equal(got[k], rec[k]), (oname, k)
                continue
            assert _rel_err(got[k], want[k]) < TOL, (sname, oname, k, _rel_err(got[k], want[k]))


@pytest.mark.gpu
def test_point_terms_bit_identical_to_device_reference(built_lib):
    ref = _ref_cuda()
    scene = chamfer_scenes()["ragged"]
    x, y = scene["x"].to(DEV), scene["y"].to(DEV)
    xl, yl, w = scene["xl"].to(DEV), scene["yl"].to(DEV), torch.tensor([1.5, 0.25, 3.0], device=DEV)
    (lx, ly), _ = _fused()(x, y, x_lengths=xl, y_lengths=yl, weights=w, point_reduction=None, batch_reduction=None)
    for got, a, b, la, lb in ((lx, x, y, xl, yl), (ly, y, x, yl, xl)):
        _, d = ref.knn_points_idx(a, b, la, lb, 2, 1, -1)
        d = d[..., 0].clone()
        d[torch.arange(a.shape[1], device=DEV)[None] >= la[:, None]] = 0.0
        d *= w.view(-1, 1)
        assert _same_bits(got, d)


@pytest.mark.gpu
def test_deterministic(built_lib):
    g = torch.Generator().manual_seed(9)
    x, y = torch.randn(4, 3000, 3, generator=g).to(DEV), torch.randn(4, 2500, 3, generator=g).to(DEV)
    xn, yn = torch.randn(4, 3000, 3, generator=g).to(DEV), torch.randn(4, 2500, 3, generator=g).to(DEV)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        runs = []
        for _ in range(2):
            leaves = [t.clone().requires_grad_() for t in (x, y, xn, yn)]
            loss, ln = _fused()(leaves[0], leaves[1], x_normals=leaves[2], y_normals=leaves[3])
            grads = torch.autograd.grad(loss + 0.5 * ln, leaves)
            runs.append([loss, ln] + list(grads))
    finally:
        torch.use_deterministic_algorithms(prev)
    for a, b in zip(*runs):
        assert _same_bits(a, b)


def _count_syncs(fn):
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("warn")
    try:
        with warnings.catch_warnings(record=True) as rec:
            warnings.simplefilter("always")
            fn()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    return len([w for w in rec if "synchroniz" in str(w.message)])


@pytest.mark.gpu
def test_host_synchronisations(built_lib):
    g = torch.Generator().manual_seed(10)
    x = torch.randn(2, 500, 3, generator=g).to(DEV).requires_grad_()
    y = torch.randn(2, 400, 3, generator=g).to(DEV).requires_grad_()
    xl, yl = torch.tensor([500, 300], device=DEV), torch.tensor([100, 400], device=DEV)
    w = torch.tensor([1.0, 2.0], device=DEV)
    out = {}
    assert _count_syncs(lambda: out.setdefault("a", _fused()(x, y))) == 0
    assert _count_syncs(lambda: out["a"][0].backward()) == 0
    assert _count_syncs(lambda: out.setdefault("b", _fused()(x, y, x_lengths=xl, y_lengths=yl, weights=w))) == 1
    assert _count_syncs(lambda: out["b"][0].backward()) == 0


@pytest.mark.gpu
def test_fitting_step(built_lib):
    """One step of the mesh-to-mesh fitting loop: ico_sphere(4) offset by deform_verts, sampled on the GPU, chamfer to
    a target cloud with normals; the loss and the gradient are finite and the gradient reaches every vertex."""
    from pytorch3d_b200 import PackedMeshes, sampling, synthetic
    v, f = synthetic.ico_sphere(4)
    v, f = v.float().to(DEV), f.to(DEV)
    deform = torch.zeros_like(v, requires_grad=True)
    g = torch.Generator().manual_seed(11)
    target = (torch.randn(1, 5000, 3, generator=g) * torch.tensor([1.0, 0.7, 1.3])).to(DEV)
    tn = torch.nn.functional.normalize(target, dim=2)
    mesh = PackedMeshes([v + deform], [f])
    pts, nrm = sampling.sample_points_from_meshes(mesh, 5000, return_normals=True)
    loss, ln = _fused()(pts, target, x_normals=nrm, y_normals=tn)
    (loss + 0.01 * ln).backward()
    assert torch.isfinite(loss) and torch.isfinite(ln)
    assert torch.isfinite(deform.grad).all() and deform.grad.abs().sum() > 0
