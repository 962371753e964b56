"""Fused frustum culling and z-clipping (DESIGN.md section 14): `clip_faces_fused` / `convert_clipped_fused` against the
torch restatement in pytorch3d_b200/clip.py, and both against the reference's own clip.py, whose CPU results on the
seeded scenes below are stored in tests/golden/reference_clip.npz (tests/golden/make_clip_golden.py)."""
import math
import os
import sys
import types
import warnings

import numpy as np
import pytest
import torch

from conftest import ROOT
from pytorch3d_b200 import clip as mclip

# ------------------------------------------------------------------------------------------------ scenes
Z_CLIP = 1.05  # not a float32 value, and rn(1 / 1.05) differs from rn(1 / rn(1.05)): pins the perspective divide
MIX = ["mix-p%d-c%d-z%d" % (p, c, z) for p in (0, 1) for c in (0, 1) for z in (0, 1)]
SCENES = MIX + ["on_plane", "equal_z", "only_culled", "nothing", "all_culled", "empty_first", "single_mesh",
                "no_faces", "near_far"]
FIELDS = ("face_verts", "mesh_to_face_first_idx", "num_faces_per_mesh", "faces_clipped_to_unclipped_idx",
          "barycentric_conversion", "faces_clipped_to_conversion_idx", "clipped_faces_neighbor_idx")
FRAGMENTS = (2, 5, 6, 3)  # N, H, W, K of the seeded Fragments over the clipped faces


def clip_scene(name):
    """A dict: face_verts (F,3,3) with z in [-0.4, 1.6), per-mesh ranges (an empty mesh in the middle unless the scene
    says otherwise), the frustum as planes (6,) float64 (NaN = unused), flags (perspective, cull, has z_clip) and
    z_clip.  A few faces have vertex 0 at (1.2, 1.3, 1.5): the reference culls them at the right plane (it tests the
    coordinates of VERTEX `axis`)."""
    g = torch.Generator().manual_seed(SCENES.index(name) + 7)
    nums = {"empty_first": [0, 30, 34], "single_mesh": [64], "no_faces": [0, 0]}.get(name, [20, 0, 44])
    F = sum(nums)
    fv = torch.rand(F, 3, 3, generator=g) * 3.0 - 1.5
    fv[..., 2] = torch.rand(F, 3, generator=g) * 2.0 - 0.4
    persp, cull, has_z = 1, 1, 1
    planes = [-1.0, 1.0, -1.0, 1.0, float("nan"), float("nan")]
    if name.startswith("mix"):
        persp, cull, has_z = (int(c) for c in name[5::3])
    if F > 0 and name != "nothing":
        fv[3] = fv[17] = fv[40 % F] = torch.tensor([[1.2, 1.3, 1.5], [0.2, 0.1, 0.9], [0.5, -0.2, 1.1]])
    if name == "on_plane":
        fv[::3, 0, 2] = Z_CLIP  # rounded to float32: exactly on the plane, counts as in front
        fv[1::5, :, 2] = Z_CLIP
        cull = 0
    elif name == "equal_z":
        fv[::2, :, 2] = fv[::2, :1, 2]  # three equal depths, in front or behind
    elif name == "only_culled":
        fv[..., 2] = fv[..., 2].abs() + Z_CLIP + 0.2
    elif name == "nothing":
        fv[..., :2] *= 0.6
        fv[..., 2] = fv[..., 2].abs() + Z_CLIP + 0.2
    elif name == "all_culled":
        fv[:, 0] = torch.tensor([1.2, 1.3, 1.5])
    elif name == "near_far":
        planes[4:] = [0.2, 1.4]
    return {"face_verts": fv, "first": torch.tensor([0] + list(np.cumsum(nums)[:-1]), dtype=torch.int64),
            "num": torch.tensor(nums, dtype=torch.int64), "planes": torch.tensor(planes, dtype=torch.float64),
            "flags": torch.tensor([persp, cull, has_z]), "z_clip": torch.tensor([Z_CLIP], dtype=torch.float64)}


def frustum_kwargs(s):
    planes = [None if math.isnan(v) else float(v) for v in s["planes"].tolist()]
    persp, cull, has_z = (int(v) for v in s["flags"])
    return dict(left=planes[0], right=planes[1], top=planes[2], bottom=planes[3], znear=planes[4], zfar=planes[5],
                perspective_correct=bool(persp), cull=bool(cull),
                z_clip_value=float(s["z_clip"][0]) if has_z else None)


def fragments(name, F_clipped):
    """(pix_to_face, bary, upstream gradient on the clipped face_verts, upstream gradient on the converted bary):
    seeded, about 30 % background slots (pix_to_face -1, bary -1 as the rasterizer pads)."""
    g = torch.Generator().manual_seed(1000 + SCENES.index(name))
    shape = FRAGMENTS
    p2f = torch.randint(0, max(F_clipped, 1), shape, generator=g)
    background = (torch.rand(shape, generator=g) < 0.3) | (F_clipped == 0)
    p2f = torch.where(background, torch.full_like(p2f, -1), p2f)
    bary = torch.rand(shape + (3,), generator=g)
    bary = bary / bary.sum(-1, keepdim=True)
    bary = torch.where(background[..., None], torch.full_like(bary, -1.0), bary)
    return p2f, bary, torch.randn(F_clipped, 3, 3, generator=g), torch.randn(shape + (3,), generator=g)


@pytest.fixture(scope="module")
def records():
    data = np.load(os.path.join(ROOT, "tests", "golden", "reference_clip.npz"))
    out = {}
    for key in data.files:
        _, name, _, field = key.split("/")
        out.setdefault(name, {})[field] = data[key]
    assert sorted(out) == sorted(SCENES)
    return out


def _frustum(rec):
    s = {k: torch.from_numpy(rec[k]) for k in ("planes", "flags", "z_clip")}
    return mclip.ClipFrustum(**frustum_kwargs(s))


def _inputs(rec, device="cpu"):
    return [torch.from_numpy(rec[k]).to(device) for k in ("face_verts_in", "first_in", "num_in")]


def _loss(cf, p2f, bary, g_fv, g_bary, convert):
    p2f_u, bary_u = convert(p2f, bary, cf)
    return p2f_u, bary_u, (cf.face_verts * g_fv).sum() + (bary_u * g_bary).sum()


# ------------------------------------------------------------------------------------------------ CPU part

def test_scene_records_cover_the_cases(records):
    seen = set()
    for name, rec in records.items():
        if "out_faces_clipped_to_unclipped_idx" not in rec:
            seen.add("identity")
        elif "out_barycentric_conversion" not in rec:
            seen.add("culled only" if rec["out_face_verts"].shape[0] else "all culled")
        else:
            seen.add("clipped")
            conv = rec["out_faces_clipped_to_conversion_idx"]
            assert sorted(conv[conv >= 0].tolist()) == list(range(rec["out_barycentric_conversion"].shape[0]))
    assert seen == {"identity", "culled only", "all culled", "clipped"}


def test_restatement_matches_the_reference_records(records):
    """The torch restatement against the reference: bit for bit in the fields it shares the layout of, and its own
    layout of the conversion gives the same conversion and gradients."""
    for name, rec in records.items():
        fv, first, num = _inputs(rec)
        out = mclip.clip_faces(fv, first, num, _frustum(rec))
        if "out_faces_clipped_to_unclipped_idx" not in rec:
            assert out.face_verts is fv and out.faces_clipped_to_unclipped_idx is None, name
        for f in FIELDS:
            if f == "barycentric_conversion" or f == "faces_clipped_to_conversion_idx" or "out_" + f not in rec:
                continue
            assert np.array_equal(getattr(out, f).numpy(), rec["out_" + f]), (name, f)
        fv = fv.clone().requires_grad_(True)
        out = mclip.clip_faces(fv, first, num, _frustum(rec))
        p2f, bary, g_fv, g_bary = (torch.from_numpy(rec[k]) for k in
                                   ("p2f_in", "bary_in", "grad_fv_clipped_in", "grad_bary_unclipped_in"))
        bary = bary.clone().requires_grad_(True)
        p2f_u, bary_u, loss = _loss(out, p2f, bary, g_fv, g_bary,
                                    mclip.convert_clipped_rasterization_to_original_faces)
        assert np.array_equal(p2f_u.numpy(), rec["p2f_out"]), name
        np.testing.assert_allclose(bary_u.detach().numpy(), rec["bary_out"], rtol=1e-6, atol=1e-7, err_msg=name)
        loss.backward()
        np.testing.assert_allclose(fv.grad.numpy(), rec["grad_face_verts"], rtol=1e-5, atol=1e-5, err_msg=name)
        np.testing.assert_allclose(bary.grad.numpy(), rec["grad_bary_in"], rtol=1e-5, atol=1e-6, err_msg=name)


# ------------------------------------------------------------------------------------------------ GPU part

@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def _assert_same_clip(fused, torch_cf, tag):
    """Fused output (reference layout) == restatement output (per-face conversion layout), bit for bit."""
    for f in ("face_verts", "mesh_to_face_first_idx", "num_faces_per_mesh", "faces_clipped_to_unclipped_idx"):
        a, b = getattr(fused, f), getattr(torch_cf, f)
        assert (a is None) == (b is None), (tag, f)
        if a is not None:
            assert torch.equal(a, b), (tag, f)
    if fused.barycentric_conversion is None:
        # culled only (the reference returns no conversion; the restatement may return rows that are all unused)
        assert fused.faces_clipped_to_conversion_idx is None and fused.clipped_faces_neighbor_idx is None, tag
        for t in (torch_cf.faces_clipped_to_conversion_idx, torch_cf.clipped_faces_neighbor_idx):
            assert t is None or (t == -1).all(), tag
        return
    assert torch.equal(fused.clipped_faces_neighbor_idx, torch_cf.clipped_faces_neighbor_idx), tag
    ci = fused.faces_clipped_to_conversion_idx
    m = torch_cf.faces_clipped_to_conversion_idx >= 0
    assert torch.equal(ci >= 0, m), tag
    assert torch.equal(fused.barycentric_conversion[ci[m]], torch_cf.barycentric_conversion[m]), tag
    n = int(m.sum())
    assert fused.barycentric_conversion.shape == (n, 3, 3) and torch.equal(ci[m].sort().values,
                                                                           torch.arange(n, device=ci.device)), tag


def _random_scene(F, seed, device, n_meshes=3):
    g = torch.Generator().manual_seed(seed)
    fv = torch.rand(F, 3, 3, generator=g) * 3.0 - 1.5
    fv[..., 2] = torch.rand(F, 3, generator=g) * 2.0 - 0.4
    cuts = torch.sort(torch.randint(0, F + 1, (n_meshes - 1,), generator=g)).values.tolist()
    first = torch.tensor([0] + cuts, dtype=torch.int64)
    num = torch.tensor(cuts + [F], dtype=torch.int64) - first
    return fv.to(device), first.to(device), num.to(device)


@pytest.mark.gpu
def test_fused_forward_matches_restatement_and_records(built_lib, dev, records):
    for name, rec in records.items():
        fv, first, num = _inputs(rec, dev)
        fr = _frustum(rec)
        fused = mclip.clip_faces_fused(fv, first, num, fr)
        _assert_same_clip(fused, mclip.clip_faces(fv, first, num, fr), name)
        if "out_faces_clipped_to_unclipped_idx" not in rec:
            assert fused.face_verts is fv and fused.faces_clipped_to_unclipped_idx is None, name
            continue
        for f in FIELDS[1:]:
            if "out_" + f in rec:
                assert np.array_equal(getattr(fused, f).cpu().numpy(), rec["out_" + f]), (name, f)
            else:
                assert getattr(fused, f) is None, (name, f)
        # face_verts: bit for bit, except the perspective xy of p4 / p5, which the CPU divides by z_clip where CUDA
        # multiplies by its reciprocal (<= 1 ulp)
        got, want = fused.face_verts.cpu().numpy(), rec["out_face_verts"]
        diff = got != want
        if diff.any():
            assert fr.perspective_correct, name
            assert not diff[..., 2].any(), name
            ulp = np.abs(got.view(np.int32).astype(np.int64) - want.view(np.int32).astype(np.int64))
            assert ulp[diff].max() <= 1, name
            clipped = np.isin(np.arange(len(got)), np.nonzero(rec.get("out_faces_clipped_to_conversion_idx",
                                                                      np.full(len(got), -1)) >= 0)[0])
            assert not diff[~clipped].any(), name
            assert diff.sum() <= 4 * clipped.sum(), name


@pytest.mark.gpu
@pytest.mark.parametrize("F", [1, 255, 256, 257, 10_000, 1_000_000])
def test_fused_forward_random_scenes(built_lib, dev, F):
    fv, first, num = _random_scene(F, F, dev)
    for persp in (False, True):
        for cull in (False, True):
            fr = mclip.ClipFrustum(left=-1, right=1, top=-1, bottom=1, znear=0.1 if cull else None,
                                   perspective_correct=persp, cull=cull, z_clip_value=Z_CLIP)
            _assert_same_clip(mclip.clip_faces_fused(fv, first, num, fr), mclip.clip_faces(fv, first, num, fr),
                              (F, persp, cull))


def _clip_losses(fv, first, num, fr, seed):
    """Gradients of sum(face_verts * G1) + sum(conversion * G2) through the fused op and through the restatement (G2
    moved to the restatement's per-face rows)."""
    x = fv.clone().requires_grad_(True)
    fused = mclip.clip_faces_fused(x, first, num, fr)
    g = torch.Generator(device=fv.device).manual_seed(seed)
    g1 = torch.randn(fused.face_verts.shape, generator=g, device=fv.device)
    loss = (fused.face_verts * g1).sum()
    conv = fused.barycentric_conversion
    g2 = None
    if conv is not None:
        g2 = torch.randn(conv.shape, generator=g, device=fv.device)
        loss = loss + (conv * g2).sum()
    (grad_fused,) = torch.autograd.grad(loss, x)
    y = fv.clone().requires_grad_(True)
    ref = mclip.clip_faces(y, first, num, fr)
    loss_r = (ref.face_verts * g1).sum()
    if g2 is not None:
        ci = fused.faces_clipped_to_conversion_idx
        g2r = torch.where((ci >= 0)[:, None, None], g2[ci.clamp(min=0)], torch.zeros_like(g2[:1]))
        loss_r = loss_r + (ref.barycentric_conversion * g2r).sum()
    (grad_ref,) = torch.autograd.grad(loss_r, y)
    return x, fused, grad_fused, grad_ref


@pytest.mark.gpu
@pytest.mark.parametrize("F", [64, 257, 100_000])
def test_clip_backward_matches_autograd_of_restatement(built_lib, dev, F):
    fv, first, num = _random_scene(F, 3 * F, dev)
    fv[::7, :, 2] = fv[::7, :1, 2]  # equal depths
    for persp in (False, True):
        for cull in (False, True):
            fr = mclip.ClipFrustum(left=-1, right=1, top=-1, bottom=1, perspective_correct=persp, cull=cull,
                                   z_clip_value=Z_CLIP)
            x, fused, grad, want = _clip_losses(fv, first, num, fr, F)
            assert torch.isfinite(grad).all()
            torch.testing.assert_close(grad, want, rtol=1e-5, atol=1e-6 * float(want.abs().max()))
            # faces without an output face (culled, all behind) get exactly 0
            kept = torch.zeros(F, dtype=torch.bool, device=dev)
            kept[fused.faces_clipped_to_unclipped_idx] = True
            assert (grad[~kept] == 0).all() and (grad[~kept].view(-1).view(torch.int32) == 0).all()
            # bitwise repeatable
            _, _, again, _ = _clip_losses(fv, first, num, fr, F)
            assert torch.equal(grad, again)


@pytest.mark.gpu
def test_fused_pair_matches_reference_records_end_to_end(built_lib, dev, records):
    """clip_faces_fused + convert_clipped_fused on the records' Fragments and upstream gradients."""
    for name, rec in records.items():
        fv, first, num = _inputs(rec, dev)
        fv = fv.clone().requires_grad_(True)
        cf = mclip.clip_faces_fused(fv, first, num, _frustum(rec))
        p2f, bary, g_fv, g_bary = (torch.from_numpy(rec[k]).to(dev) for k in
                                   ("p2f_in", "bary_in", "grad_fv_clipped_in", "grad_bary_unclipped_in"))
        bary = bary.clone().requires_grad_(True)
        p2f_u, bary_u, loss = _loss(cf, p2f, bary, g_fv, g_bary, mclip.convert_clipped_fused)
        assert np.array_equal(p2f_u.cpu().numpy(), rec["p2f_out"]), name
        np.testing.assert_allclose(bary_u.detach().cpu().numpy(), rec["bary_out"], rtol=1e-6, atol=1e-6, err_msg=name)
        loss.backward()
        np.testing.assert_allclose(fv.grad.cpu().numpy(), rec["grad_face_verts"], rtol=1e-4, atol=1e-5, err_msg=name)
        np.testing.assert_allclose(bary.grad.cpu().numpy(), rec["grad_bary_in"], rtol=1e-5, atol=1e-6, err_msg=name)


@pytest.mark.gpu
@pytest.mark.parametrize("F,K", [(300, 1), (5000, 8), (100_000, 20)])
def test_convert_matches_the_bmm_chain(built_lib, dev, F, K):
    fv, first, num = _random_scene(F, F + K, dev)
    fr = mclip.ClipFrustum(perspective_correct=True, cull=False, z_clip_value=Z_CLIP)
    cf = mclip.clip_faces_fused(fv, first, num, fr)
    Fc = cf.face_verts.shape[0]
    g = torch.Generator(device=dev).manual_seed(F)
    shape = (2, 33, 17, K)
    p2f = torch.randint(0, Fc, shape, generator=g, device=dev)
    p2f = torch.where(torch.rand(shape, generator=g, device=dev) < 0.3, torch.full_like(p2f, -1), p2f)
    bary = torch.rand(shape + (3,), generator=g, device=dev)
    conv = cf.barycentric_conversion.clone().requires_grad_(True)
    cfa = mclip.ClippedFaces(cf.face_verts, cf.mesh_to_face_first_idx, cf.num_faces_per_mesh,
                             cf.faces_clipped_to_unclipped_idx, conv, cf.faces_clipped_to_conversion_idx,
                             cf.clipped_faces_neighbor_idx)
    b1, b2 = bary.clone().requires_grad_(True), bary.clone().requires_grad_(True)
    p_f, bary_f = mclip.convert_clipped_fused(p2f, b1, cfa)
    p_r, bary_r = mclip.convert_clipped_rasterization_to_original_faces(p2f, b2, cfa)
    assert torch.equal(p_f, p_r)
    converted = (p2f >= 0) & (cf.faces_clipped_to_conversion_idx[p2f.clamp(min=0)] >= 0)
    assert converted.any() and (~converted).any()
    assert torch.equal(bary_f[~converted], bary[~converted])
    torch.testing.assert_close(bary_f, bary_r, rtol=1e-6, atol=1e-7)
    gb = torch.randn(shape + (3,), generator=g, device=dev)
    gf = torch.autograd.grad((bary_f * gb).sum(), (b1, conv))
    gr = torch.autograd.grad((bary_r * gb).sum(), (b2, conv))
    torch.testing.assert_close(gf[0], gr[0], rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(gf[1], gr[1], rtol=1e-4, atol=1e-5 * float(gr[1].abs().max()))
    # only pix_to_face (culling only: no conversion)
    fr_cull = mclip.ClipFrustum(left=-1, right=1, top=-1, bottom=1, cull=True)
    fv2 = fv.clone()
    fv2[::5, 0] = torch.tensor([1.2, 1.3, 1.5], device=dev)
    cf2 = mclip.clip_faces_fused(fv2, first, num, fr_cull)
    assert cf2.barycentric_conversion is None
    p2, b2 = mclip.convert_clipped_fused(p2f.clamp(max=cf2.face_verts.shape[0] - 1), bary, cf2)
    assert b2 is bary and torch.equal(p2, torch.where(p2f >= 0, cf2.faces_clipped_to_unclipped_idx[
        p2f.clamp(0, cf2.face_verts.shape[0] - 1)], p2f))


def _torus_scene(dev, n=4, rings=40, sides=24, seed=0):
    """Per-mesh vertices (leaves that require grad) and faces of n randomly rotated tori, projected with a perspective
    divide; their depths run from about 0.2 to 2.4, so the plane z = 0.5 cuts every torus."""
    from pytorch3d_b200 import synthetic
    verts, faces = synthetic.torus(rings, sides)
    g = torch.Generator().manual_seed(seed)
    vs = []
    for _ in range(n):
        q = torch.linalg.qr(torch.randn(3, 3, generator=g))[0]
        v = verts @ q.T
        v[:, 2] = v[:, 2] * 0.8 + 1.2
        v[:, :2] = v[:, :2] / v[:, 2:3].clamp(min=0.3)
        vs.append(v.to(dev).requires_grad_(True))
    return vs, [faces.to(dev)] * n


def _torch_path(meshes, image_size, blur, K, persp, z_clip, cull):
    """rasterize_meshes with the restatement's clip_faces / conversion (what the wrapper ran before the fused pair)."""
    import importlib
    rm = importlib.import_module("pytorch3d_b200.rasterize_meshes")
    fv = meshes.verts_packed()[meshes.faces_packed()]
    fr = mclip.ClipFrustum(left=-1, right=1, top=-1, bottom=1, perspective_correct=persp, z_clip_value=z_clip,
                           cull=cull)
    cf = mclip.clip_faces(fv, meshes.mesh_to_faces_packed_first_idx(), meshes.num_faces_per_mesh(), fr)
    nb = cf.clipped_faces_neighbor_idx
    if nb is None:
        nb = torch.full((cf.face_verts.shape[0],), -1, dtype=torch.int64, device=fv.device)
        nb._b200_all_minus_one = True
    p2f, zbuf, bary, dists = rm._RasterizeFaceVerts.apply(
        cf.face_verts, cf.mesh_to_face_first_idx, cf.num_faces_per_mesh, nb, image_size, blur, K, 0, 0, persp,
        False, False)
    p2f, bary = mclip.convert_clipped_rasterization_to_original_faces(p2f, bary, cf)
    return p2f, zbuf, bary, dists


@pytest.mark.gpu
def test_rasterize_meshes_with_clipping_matches_the_torch_path(built_lib, dev):
    import pytorch3d_b200 as p3b
    vs, fs = _torus_scene(dev)
    m = p3b.PackedMeshes(vs, fs)
    outs = []
    for fused in (True, False):
        args = ((64, 80), 1e-4, 4, True, 0.5, True)
        if fused:
            o = p3b.rasterize_meshes(m, args[0], args[1], args[2], None, None, args[3], False, False, args[4], args[5])
        else:
            o = _torch_path(m, *args)
        loss = (o[1].clamp_min(0) * 0.3).sum() + (o[2] * 0.7).sum() + o[3].clamp(-1, 1).sum()
        outs.append((o, torch.cat(torch.autograd.grad(loss, vs))))
    (a, ga), (b, gb) = outs
    assert (a[0] >= 0).any()
    for i in (0, 1, 3):
        assert torch.equal(a[i], b[i]), i
    torch.testing.assert_close(a[2], b[2], rtol=1e-6, atol=1e-7)
    torch.testing.assert_close(ga, gb, rtol=1e-4, atol=1e-4 * float(gb.abs().max()))


@pytest.mark.gpu
def test_identity_scene_takes_the_indexed_path(built_lib, dev, monkeypatch):
    import importlib
    import pytorch3d_b200 as p3b
    from pytorch3d_b200 import synthetic
    rm = importlib.import_module("pytorch3d_b200.rasterize_meshes")
    m = synthetic.torus_batch(3, 20, 12, device=dev)  # depths 1 .. 3: wholly in front of z = 0.01
    plain = p3b.rasterize_meshes(m, 48, 1e-4, 3, perspective_correct=True)
    calls = []
    monkeypatch.setattr(rm._C, "rasterize_meshes", lambda *a, **k: calls.append(1))
    clipped = p3b.rasterize_meshes(m, 48, 1e-4, 3, perspective_correct=True, z_clip_value=0.01)
    assert calls == []
    for x, y in zip(plain, clipped):
        assert torch.equal(x, y)


@pytest.mark.gpu
def test_one_host_sync_per_forward_and_none_in_backward(built_lib, dev):
    import pytorch3d_b200 as p3b
    vs, fs = _torus_scene(dev)
    m = p3b.PackedMeshes(vs, fs)
    torch.cuda.synchronize()
    prev = torch.cuda.get_sync_debug_mode()
    try:
        torch.cuda.set_sync_debug_mode("warn")
        with warnings.catch_warnings(record=True) as fw:
            warnings.simplefilter("always")
            o = p3b.rasterize_meshes(m, 64, 1e-4, 4, None, None, True, False, False, 0.5, True)
            loss = o[1].clamp_min(0).sum() + o[2].sum() + o[3].clamp(-1, 1).sum()
        with warnings.catch_warnings(record=True) as bw:
            warnings.simplefilter("always")
            loss.backward()
    finally:
        torch.cuda.set_sync_debug_mode(prev)
    sync = [w for w in fw if "synchroniz" in str(w.message)]
    assert len(sync) == 1, [str(w.message) for w in fw]
    assert not [w for w in bw if "synchroniz" in str(w.message)]
    assert all(torch.isfinite(v.grad).all() for v in vs) and sum(float(v.grad.abs().sum()) for v in vs) > 0


# ------------------------------------------------------------------------------------- errors and determinism

@pytest.mark.gpu
def test_argument_errors(built_lib, dev):
    from pytorch3d_b200 import _C
    fr = mclip.ClipFrustum(z_clip_value=0.3)
    fv, first, num = _random_scene(10, 0, dev)
    with pytest.raises(RuntimeError, match="face_verts"):
        _C.clip_faces_count(fr, face_verts=fv.double())
    with pytest.raises(RuntimeError, match="face_verts"):
        _C.clip_faces_count(fr, face_verts=fv.reshape(10, 9))
    with pytest.raises(RuntimeError, match="face_verts must be a CUDA tensor"):
        _C.clip_faces_count(fr, face_verts=fv.cpu())
    with pytest.raises(RuntimeError, match="faces"):
        _C.clip_faces_count(fr, verts=fv.reshape(-1, 3), faces=torch.zeros(4, 3, dtype=torch.int32, device=dev))
    ws = _C.clip_faces_count(fr, face_verts=fv)
    rec = ws[:4].tolist()
    with pytest.raises(RuntimeError, match="mesh_to_face_first_idx"):
        _C.clip_faces_fill(fv, first.int(), num, fr, ws, rec)
    with pytest.raises(RuntimeError, match="num_faces_per_mesh"):
        _C.clip_faces_fill(fv, first, num.cpu(), fr, ws, rec)
    with pytest.raises(RuntimeError, match="pix_to_face"):
        _C.clip_convert_forward(torch.zeros(2, 2, 2, 1, dtype=torch.int32, device=dev),
                                torch.zeros(2, 2, 2, 1, 3, device=dev), torch.zeros(3, dtype=torch.int64, device=dev))
    with pytest.raises(RuntimeError, match="barycentric_coords"):
        _C.clip_convert_forward(torch.zeros(2, 2, 2, 1, dtype=torch.int64, device=dev),
                                torch.zeros(2, 2, 2, 2, 3, device=dev), torch.zeros(3, dtype=torch.int64, device=dev))


@pytest.mark.gpu
def test_deterministic_mode(built_lib, dev):
    fv, first, num = _random_scene(500, 5, dev)
    fr = mclip.ClipFrustum(perspective_correct=True, cull=False, z_clip_value=Z_CLIP)
    x = fv.clone().requires_grad_(True)
    prev = torch.are_deterministic_algorithms_enabled()
    try:
        torch.use_deterministic_algorithms(True)
        cf = mclip.clip_faces_fused(x, first, num, fr)
        (cf.face_verts.sum() + cf.barycentric_conversion.sum()).backward()  # the clip backward has no atomics
        p2f = torch.zeros(1, 4, 4, 2, dtype=torch.int64, device=dev)
        bary = torch.rand(1, 4, 4, 2, 3, device=dev)
        _, b = mclip.convert_clipped_fused(p2f, bary, cf)
        with pytest.raises(RuntimeError, match="deterministic"):
            b.sum().backward()
    finally:
        torch.use_deterministic_algorithms(prev)


# ------------------------------------------------------------------------------------------------ install

def _stand_in(shape, dtype=torch.float32, is_cuda=True):
    return types.SimpleNamespace(is_cuda=is_cuda, dtype=dtype, shape=torch.Size(shape))


def _fake_pytorch3d(monkeypatch):
    names = ("pytorch3d", "pytorch3d.renderer", "pytorch3d.renderer.mesh")
    for n in names:
        mod = types.ModuleType(n)
        mod.__path__ = []
        monkeypatch.setitem(sys.modules, n, mod)
    clip_mod = types.ModuleType("pytorch3d.renderer.mesh.clip")

    class RefClippedFaces:
        def __init__(self, **kw):
            self.__dict__.update(kw)

    clip_mod.ClippedFaces = RefClippedFaces
    rm = types.ModuleType("pytorch3d.renderer.mesh.rasterize_meshes")
    rm.clip_faces = lambda *a: "ref-clip"
    rm.convert_clipped_rasterization_to_original_faces = lambda *a: "ref-convert"
    monkeypatch.setitem(sys.modules, clip_mod.__name__, clip_mod)
    monkeypatch.setitem(sys.modules, rm.__name__, rm)
    return rm, RefClippedFaces


@pytest.mark.gpu
def test_install_clipping_routes_and_uninstalls(monkeypatch, built_lib):
    from pytorch3d_b200 import install as inst
    rm, RefClippedFaces = _fake_pytorch3d(monkeypatch)
    original_clip, original_convert = rm.clip_faces, rm.convert_clipped_rasterization_to_original_faces
    fused_cf = mclip.ClippedFaces("fv", "first", "num")
    monkeypatch.setattr(mclip, "clip_faces_fused", lambda *a: fused_cf)
    monkeypatch.setattr(mclip, "convert_clipped_fused", lambda *a: "b200-convert")
    try:
        assert inst.install_clipping() == ["pytorch3d.renderer.mesh.rasterize_meshes"]
        assert inst._saved == {} and inst._saved_methods == {}
        out = rm.clip_faces(_stand_in((5, 3, 3)), None, None, None)
        assert isinstance(out, RefClippedFaces) and out.face_verts == "fv" and out.barycentric_conversion is None
        assert rm.clip_faces(_stand_in((5, 3, 3), is_cuda=False), None, None, None) == "ref-clip"
        assert rm.clip_faces(_stand_in((5, 3, 3), torch.float64), None, None, None) == "ref-clip"
        cf = types.SimpleNamespace(barycentric_conversion=_stand_in((2, 3, 3)))
        p2f, bary = _stand_in((1, 2, 2, 1), torch.int64), _stand_in((1, 2, 2, 1, 3))
        assert rm.convert_clipped_rasterization_to_original_faces(p2f, bary, cf) == "b200-convert"
        assert rm.convert_clipped_rasterization_to_original_faces(
            _stand_in((1, 2, 2, 1), torch.int64, is_cuda=False), bary, cf) == "ref-convert"
        assert rm.convert_clipped_rasterization_to_original_faces(
            p2f, _stand_in((1, 2, 2, 1, 3), torch.float64), cf) == "ref-convert"
    finally:
        inst.uninstall()
    assert rm.clip_faces is original_clip
    assert rm.convert_clipped_rasterization_to_original_faces is original_convert
