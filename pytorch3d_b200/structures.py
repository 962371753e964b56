"""Minimal packed-batch containers with the accessor surface of PyTorch3D's Meshes / Pointclouds.

The rasterizer only needs the *packed* layout of pytorch3d/structures/meshes.py and pointclouds.py
(verts_packed / faces_packed / mesh_to_faces_packed_first_idx / num_faces_per_mesh, and the points
analogue), which is reused unchanged.  When PyTorch3D is installed its own `Meshes` / `Pointclouds`
objects can be passed to every function of this package instead; these classes exist so that the
package, its tests and the benchmark are standalone.
"""
from typing import List, Sequence

import torch


class PackedMeshes:
    """A batch of triangle meshes in packed form (same fields as pytorch3d.structures.Meshes)."""

    def __init__(self, verts: Sequence[torch.Tensor], faces: Sequence[torch.Tensor]):
        assert len(verts) == len(faces)
        self._N = len(verts)
        self.device = verts[0].device if self._N else torch.device("cpu")
        v_counts = [int(v.shape[0]) for v in verts]
        f_counts = [int(f.shape[0]) for f in faces]
        v_off, acc = [], 0
        for c in v_counts:
            v_off.append(acc)
            acc += c
        self._verts_packed = (torch.cat(list(verts), 0) if self._N else torch.zeros((0, 3))).to(torch.float32)
        self._faces_packed = (
            torch.cat([f.to(torch.int64) + o for f, o in zip(faces, v_off)], 0)
            if self._N else torch.zeros((0, 3), dtype=torch.int64))
        self._num_faces_per_mesh = torch.tensor(f_counts, dtype=torch.int64, device=self.device)
        first = torch.zeros((self._N,), dtype=torch.int64, device=self.device)
        if self._N > 1:
            first[1:] = torch.cumsum(self._num_faces_per_mesh, 0)[:-1]
        self._mesh_to_faces_packed_first_idx = first
        self._num_verts_per_mesh = torch.tensor(v_counts, dtype=torch.int64, device=self.device)
        self._mesh_to_verts_packed_first_idx = torch.tensor(v_off, dtype=torch.int64, device=self.device)
        self._F = max(f_counts) if f_counts else 0
        self._V = max(v_counts) if v_counts else 0

    def __len__(self):
        return self._N

    def verts_packed(self):
        return self._verts_packed

    def faces_packed(self):
        return self._faces_packed

    def mesh_to_faces_packed_first_idx(self):
        return self._mesh_to_faces_packed_first_idx

    def num_faces_per_mesh(self):
        return self._num_faces_per_mesh

    def num_verts_per_mesh(self):
        return self._num_verts_per_mesh

    def mesh_to_verts_packed_first_idx(self):
        return self._mesh_to_verts_packed_first_idx

    def isempty(self):
        return self._N == 0 or self._verts_packed.shape[0] == 0

    def verts_normals_packed(self):
        """(V, 3) unit vertex normals, as pytorch3d.structures.Meshes computes them: the sum of the area-weighted normals
        (v2 - v1) x (v0 - v1) of the faces around each vertex, normalised with eps 1e-6.  Differentiable in the
        vertices; computed on every call."""
        verts, faces = self.verts_packed(), self.faces_packed()
        if self.isempty():
            return torch.zeros((self._N, 3), dtype=torch.int64, device=self.device)  # what Meshes returns when empty
        corners = verts[faces]
        face_normals = torch.cross(corners[:, 2] - corners[:, 1], corners[:, 0] - corners[:, 1], dim=1)
        normals = torch.zeros_like(verts)
        for j in range(3):
            normals = normals.index_add(0, faces[:, j], face_normals)
        return torch.nn.functional.normalize(normals, eps=1e-6, dim=1)

    def requires_grad_(self, flag=True):
        self._verts_packed.requires_grad_(flag)
        return self


class PackedPointclouds:
    """A batch of point clouds in packed form (same fields as pytorch3d.structures.Pointclouds)."""

    def __init__(self, points: Sequence[torch.Tensor]):
        self._N = len(points)
        self.device = points[0].device if self._N else torch.device("cpu")
        counts = [int(p.shape[0]) for p in points]
        self._P = max(counts) if counts else 0
        self._points_packed = (torch.cat(list(points), 0) if self._N else torch.zeros((0, 3))).to(torch.float32)
        self._num_points_per_cloud = torch.tensor(counts, dtype=torch.int64, device=self.device)
        first = torch.zeros((self._N,), dtype=torch.int64, device=self.device)
        if self._N > 1:
            first[1:] = torch.cumsum(self._num_points_per_cloud, 0)[:-1]
        self._cloud_to_packed_first_idx = first
        idx: List[torch.Tensor] = []
        for n, c in enumerate(counts):
            idx.append(torch.arange(c, dtype=torch.int64, device=self.device) + n * self._P)
        self._padded_to_packed_idx = torch.cat(idx, 0) if idx else torch.zeros((0,), dtype=torch.int64)

    def __len__(self):
        return self._N

    def points_packed(self):
        return self._points_packed

    def cloud_to_packed_first_idx(self):
        return self._cloud_to_packed_first_idx

    def num_points_per_cloud(self):
        return self._num_points_per_cloud

    def padded_to_packed_idx(self):
        return self._padded_to_packed_idx
