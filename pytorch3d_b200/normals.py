"""Mesh normals on the GPU: face areas and normals, and vertex normals, with the results of the reference's
`mesh_face_areas_normals` (pytorch3d/ops/mesh_face_areas_normals.py) and `Meshes._compute_vertex_normals`
(pytorch3d/structures/meshes.py).

Both ops build a vertex -> corner table (a stable radix sort of the 3F corners by vertex) and sum each vertex's corners
in one thread, in the order the reference's serial CPU `index_add` calls use (DESIGN.md section 17).  So the backward
passes have no float atomics and are deterministic, and nothing synchronises the host.

- `face_areas_normals(verts, faces)`: the reference's `_MeshFaceAreasNormals`; the forward is bit-identical to the
  reference's CUDA kernel, the backward sums the reference's per-corner gradients in a fixed order.
- `verts_normals(verts, faces)`: the (V, 3) unit vertex normals, bit-identical to the reference's torch chain on the
  CPU, with gradients to `verts`.  The forward's table is saved for the backward, which does not sort again.
"""
import torch
from torch.autograd.function import once_differentiable

from . import _C

__all__ = ["face_areas_normals", "verts_normals", "verts_normals_packed", "faces_areas_normals_packed"]


class _FaceAreasNormals(torch.autograd.Function):
    """The reference's `_MeshFaceAreasNormals` on `pytorch3d_b200._C`: the same argument checks, the float cast, and a
    once-differentiable backward."""

    @staticmethod
    def forward(ctx, verts, faces):
        if not (verts.dim() == 2):
            raise ValueError("verts need to be of shape Vx3.")
        if not (verts.shape[1] == 3):
            raise ValueError("verts need to be of shape Vx3.")
        if not (faces.dim() == 2):
            raise ValueError("faces need to be of shape Fx3.")
        if not (faces.shape[1] == 3):
            raise ValueError("faces need to be of shape Fx3.")
        if not (faces.dtype == torch.int64):
            raise ValueError("faces need to be of type torch.int64.")
        if not (verts.dtype == torch.float32):
            verts = verts.float()
        ctx.save_for_backward(verts, faces)
        return _C.face_areas_normals_forward(verts, faces)

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_areas, grad_normals):
        grad_areas = grad_areas.contiguous()
        grad_normals = grad_normals.contiguous()
        verts, faces = ctx.saved_tensors
        if not (grad_areas.dtype == torch.float32):
            grad_areas = grad_areas.float()
        if not (grad_normals.dtype == torch.float32):
            grad_normals = grad_normals.float()
        return _C.face_areas_normals_backward(grad_areas, grad_normals, verts, faces), None


def face_areas_normals(verts: torch.Tensor, faces: torch.Tensor):
    """(areas (F,), normals (F, 3)) of the packed faces: verts (V, 3) float, faces (F, 3) int64, both CUDA."""
    return _FaceAreasNormals.apply(verts, faces)


class _VertsNormals(torch.autograd.Function):
    @staticmethod
    def forward(ctx, verts, faces):
        normals, table, sums = _C.verts_normals_forward(verts, faces)
        ctx.save_for_backward(verts, faces, table, sums)
        return normals

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_normals):
        verts, faces, table, sums = ctx.saved_tensors
        grad_verts = None
        if ctx.needs_input_grad[0]:
            grad_verts = _C.verts_normals_backward(grad_normals.contiguous(), verts, faces, table, sums)
        return grad_verts, None


def verts_normals(verts: torch.Tensor, faces: torch.Tensor) -> torch.Tensor:
    """(V, 3) unit vertex normals: each vertex's sum of the area-weighted face normals (v2 - v1) x (v0 - v1) of its
    faces, divided by max(|sum|, 1e-6).  verts (V, 3) float32 and faces (F, 3) int64 on one CUDA device; gradients
    reach `verts`."""
    return _VertsNormals.apply(verts, faces)


def verts_normals_packed(meshes) -> torch.Tensor:
    """`verts_normals` of an object with `verts_packed()` and `faces_packed()` (a PyTorch3D `Meshes`, or
    `PackedMeshes`)."""
    return verts_normals(meshes.verts_packed(), meshes.faces_packed())


def faces_areas_normals_packed(meshes):
    """`face_areas_normals` of an object with `verts_packed()` and `faces_packed()`: (areas (F,), normals (F, 3))."""
    return face_areas_normals(meshes.verts_packed(), meshes.faces_packed())
