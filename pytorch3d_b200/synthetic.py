"""Seeded synthetic inputs for tests and bench.py (pure torch; no dependency on pytorch3d.utils).

The workloads follow SURVEY.md 8(d): torus meshes with a chosen face count placed in NDC
(xy in [-0.9, 0.9], z in [1, 3]) with a per-mesh random rotation, ico-spheres, and uniform point clouds.
"""
import math

import torch

from .structures import PackedMeshes, PackedPointclouds


def _rotation(gen):
    """Random rotation matrix from a seeded generator (QR of a Gaussian matrix)."""
    a = torch.randn(3, 3, generator=gen, dtype=torch.float64)
    q, r = torch.linalg.qr(a)
    q = q * torch.sign(torch.diagonal(r))
    if torch.det(q) < 0:
        q[:, 0] = -q[:, 0]
    return q.to(torch.float32)


def torus(rings: int, sides: int, R: float = 1.0, r: float = 0.45):
    """Torus with rings*sides*2 triangles; returns (verts (V,3) f32, faces (F,3) i64)."""
    u = torch.arange(rings, dtype=torch.float64) * (2 * math.pi / rings)
    v = torch.arange(sides, dtype=torch.float64) * (2 * math.pi / sides)
    uu, vv = torch.meshgrid(u, v, indexing="ij")
    x = (R + r * torch.cos(vv)) * torch.cos(uu)
    y = (R + r * torch.cos(vv)) * torch.sin(uu)
    z = r * torch.sin(vv)
    verts = torch.stack([x, y, z], -1).reshape(-1, 3).to(torch.float32)
    i = torch.arange(rings).reshape(-1, 1)
    j = torch.arange(sides).reshape(1, -1)
    a = (i * sides + j).reshape(-1)
    b = (((i + 1) % rings) * sides + j).reshape(-1)
    c = (((i + 1) % rings) * sides + (j + 1) % sides).reshape(-1)
    d = (i * sides + (j + 1) % sides).reshape(-1)
    faces = torch.cat([torch.stack([a, b, c], 1), torch.stack([a, c, d], 1)], 0).to(torch.int64)
    return verts, faces


def fit_to_ndc(verts, rot=None, xy_extent=0.9, z_range=(1.0, 3.0)):
    """Rotate, then scale/shift so that xy spans [-xy_extent, xy_extent] and z spans z_range."""
    if rot is not None:
        verts = verts @ rot.T
    lo, hi = verts.min(0).values, verts.max(0).values
    ctr = (lo + hi) / 2
    out = verts - ctr
    s = xy_extent / torch.max(hi[:2] - ctr[:2])
    out[:, :2] = out[:, :2] * s
    zspan = torch.clamp(hi[2] - lo[2], min=1e-6)
    out[:, 2] = (out[:, 2] / zspan + 0.5) * (z_range[1] - z_range[0]) + z_range[0]
    return out.contiguous()


def torus_batch(n_meshes: int, rings: int, sides: int, seed: int = 0, device="cpu"):
    """Batch of n identical-topology tori with per-mesh random rotations (seeded) in NDC."""
    gen = torch.Generator().manual_seed(seed)
    verts, faces = torus(rings, sides)
    vs, fs = [], []
    for _ in range(n_meshes):
        vs.append(fit_to_ndc(verts, _rotation(gen)).to(device))
        fs.append(faces.to(device))
    return PackedMeshes(vs, fs)


def torus_uvs(rings: int, sides: int):
    """UVs of `torus(rings, sides)` from its (ring, side) parametrisation: (verts_uvs ((rings+1)*(sides+1), 2) f32,
    faces_uvs (F, 3) i64), faces in the order of `torus`.  The UV grid has one more row and column than the vertex grid,
    so the vertices on the two seams are duplicated in UV space and `faces_uvs` differs from `faces` there."""
    uu, vv = torch.meshgrid(torch.arange(rings + 1, dtype=torch.float64) / rings,
                            torch.arange(sides + 1, dtype=torch.float64) / sides, indexing="ij")
    verts_uvs = torch.stack([uu, vv], -1).reshape(-1, 2).to(torch.float32)
    S = sides + 1
    i = torch.arange(rings).reshape(-1, 1)
    j = torch.arange(sides).reshape(1, -1)
    a = (i * S + j).reshape(-1)
    b = ((i + 1) * S + j).reshape(-1)
    c = ((i + 1) * S + j + 1).reshape(-1)
    d = (i * S + j + 1).reshape(-1)
    faces_uvs = torch.cat([torch.stack([a, b, c], 1), torch.stack([a, c, d], 1)], 0).to(torch.int64)
    return verts_uvs, faces_uvs


def textured_torus_batch(n_meshes: int, rings: int, sides: int, map_size=(64, 64), channels: int = 3, seed: int = 0,
                         device="cpu"):
    """`torus_batch` with UV texture coordinates and maps: (meshes, verts_uvs list of (V_uv, 2), faces_uvs list of
    (F, 3), maps (n_meshes, H_in, W_in, channels) f32 in [0, 1), one seeded map per mesh)."""
    meshes = torus_batch(n_meshes, rings, sides, seed=seed, device=device)
    verts_uvs, faces_uvs = torus_uvs(rings, sides)
    gen = torch.Generator().manual_seed(seed + 1)
    maps = torch.rand((n_meshes, int(map_size[0]), int(map_size[1]), channels), generator=gen).to(device)
    return meshes, [verts_uvs.to(device)] * n_meshes, [faces_uvs.to(device)] * n_meshes, maps


def torus_batch_hetero(face_counts, seed: int = 0, device="cpu"):
    """Batch of tori whose face counts approximate `face_counts` (rings = sides = sqrt(F/2))."""
    gen = torch.Generator().manual_seed(seed)
    vs, fs = [], []
    for fc in face_counts:
        s = max(3, int(round(math.sqrt(fc / 2))))
        verts, faces = torus(s, s)
        vs.append(fit_to_ndc(verts, _rotation(gen)).to(device))
        fs.append(faces.to(device))
    return PackedMeshes(vs, fs)


def ico_sphere(level: int = 0):
    """Icosphere by recursive 4-way subdivision: level 4 = 2562 verts / 5120 faces."""
    t = (1.0 + math.sqrt(5.0)) / 2.0
    verts = torch.tensor(
        [[-1, t, 0], [1, t, 0], [-1, -t, 0], [1, -t, 0], [0, -1, t], [0, 1, t], [0, -1, -t], [0, 1, -t],
         [t, 0, -1], [t, 0, 1], [-t, 0, -1], [-t, 0, 1]], dtype=torch.float64)
    verts = verts / verts.norm(dim=1, keepdim=True)
    faces = torch.tensor(
        [[0, 11, 5], [0, 5, 1], [0, 1, 7], [0, 7, 10], [0, 10, 11], [1, 5, 9], [5, 11, 4], [11, 10, 2],
         [10, 7, 6], [7, 1, 8], [3, 9, 4], [3, 4, 2], [3, 2, 6], [3, 6, 8], [3, 8, 9], [4, 9, 5], [2, 4, 11],
         [6, 2, 10], [8, 6, 7], [9, 8, 1]], dtype=torch.int64)
    for _ in range(level):
        v = verts.shape[0]
        e = torch.cat([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]], 0)
        e = torch.sort(e, dim=1).values
        key = e[:, 0] * v + e[:, 1]
        uniq, inv = torch.unique(key, return_inverse=True)
        mid = (verts[uniq // v] + verts[uniq % v]) / 2
        mid = mid / mid.norm(dim=1, keepdim=True)
        verts = torch.cat([verts, mid], 0)
        nf = faces.shape[0]
        m01, m12, m20 = inv[:nf] + v, inv[nf:2 * nf] + v, inv[2 * nf:] + v
        f0, f1, f2 = faces[:, 0], faces[:, 1], faces[:, 2]
        faces = torch.cat([torch.stack([f0, m01, m20], 1), torch.stack([f1, m12, m01], 1),
                           torch.stack([f2, m20, m12], 1), torch.stack([m01, m12, m20], 1)], 0)
    return verts.to(torch.float32), faces


def ico_sphere_batch(n_meshes: int, level: int, device="cpu", xy_scale=0.8, z_offset=2.0):
    """The reference CPU benchmark scene: ico_sphere scaled 0.8 in xy, z += 2 (BASELINE.md section 2)."""
    verts, faces = ico_sphere(level)
    verts = verts.clone()
    verts[:, :2] *= xy_scale
    verts[:, 2] += z_offset
    return PackedMeshes([verts.to(device)] * n_meshes, [faces.to(device)] * n_meshes)


def random_pointclouds(n_clouds: int, n_points: int, seed: int = 0, device="cpu", z_range=(0.5, 1.5)):
    """Uniform points in [-1,1]^2 x z_range (SURVEY.md 8d, config C3)."""
    gen = torch.Generator().manual_seed(seed)
    clouds = []
    for _ in range(n_clouds):
        p = torch.rand(n_points, 3, generator=gen)
        p[:, :2] = p[:, :2] * 2 - 1
        p[:, 2] = p[:, 2] * (z_range[1] - z_range[0]) + z_range[0]
        clouds.append(p.to(device))
    return PackedPointclouds(clouds)


def face_verts_of(meshes):
    """(F,3,3) packed face vertices, the operator-level input."""
    return meshes.verts_packed()[meshes.faces_packed()].contiguous()
