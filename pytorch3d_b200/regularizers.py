"""Mesh regularisers on the GPU: `mesh_edge_loss`, `mesh_laplacian_smoothing` and `mesh_normal_consistency`, with the
signatures, keyword defaults and results of pytorch3d/loss/mesh_edge_loss.py, mesh_laplacian_smoothing.py and
mesh_normal_consistency.py.

Each loss builds its topology in fused kernels (DESIGN.md section 18): a stable radix sort of the face-edges gives the
edges in the reference's order, and per-vertex tables give each vertex its incident edges or corners.  No kernel uses
float atomics, nothing synchronises the host (the reference's normal consistency copies the edge counts to the host
and enumerates the face pairs on the CPU), and the backward reads the tables its forward built.

The functions take a PyTorch3D `Meshes` or a `PackedMeshes`: anything with `verts_packed()`, `faces_packed()`,
`num_verts_per_mesh()`, `mesh_to_verts_packed_first_idx()` and `len()`, on a CUDA device, with float32 verts and int64
faces.  Gradients reach `verts_packed()`.

One divergence: where no edge has two faces (a triangle soup), the reference's normal consistency returns a detached
`tensor([0.])`; telling that case apart needs a device read, so here it is a 0-dim zero connected to the verts, whose
gradient is zero.
"""
import torch
from torch.autograd.function import once_differentiable

from . import _C

__all__ = ["mesh_edge_loss", "mesh_laplacian_smoothing", "mesh_normal_consistency"]


def _empty(meshes):
    """The reference's result for a batch with no meshes or no faces at all, decided from host state only: the
    number of meshes and the faces' row count (Meshes keeps the largest face count per mesh, `_F`, on the host)."""
    if len(meshes) == 0:
        return True
    F = getattr(meshes, "_F", None)
    return (F == 0) if isinstance(F, int) else meshes.faces_packed().shape[0] == 0


def _zero(meshes):
    device = getattr(meshes, "device", None) or meshes.verts_packed().device
    return torch.tensor([0.0], dtype=torch.float32, device=device, requires_grad=True)


def _packed(meshes):
    return (meshes.verts_packed(), meshes.faces_packed(), meshes.mesh_to_verts_packed_first_idx(),
            meshes.num_verts_per_mesh())


class _EdgeLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, verts, faces, first, num, target_length):
        loss, ws = _C.mesh_edge_loss_forward(verts, faces, first, num, target_length)
        ctx.save_for_backward(verts, faces, first, num, ws)
        ctx.target_length = target_length
        return loss

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_loss):
        verts, faces, first, num, ws = ctx.saved_tensors
        grad = None
        if ctx.needs_input_grad[0]:
            grad = _C.mesh_edge_loss_backward(grad_loss, verts, faces, first, num, ctx.target_length, ws)
        return grad, None, None, None, None


class _LaplacianSmoothing(torch.autograd.Function):
    @staticmethod
    def forward(ctx, verts, faces, first, num, method):
        loss, ws = _C.mesh_laplacian_smoothing_forward(verts, faces, first, num, method)
        ctx.save_for_backward(verts, faces, first, num, ws)
        ctx.method = method
        return loss

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_loss):
        verts, faces, first, num, ws = ctx.saved_tensors
        grad = None
        if ctx.needs_input_grad[0]:
            grad = _C.mesh_laplacian_smoothing_backward(grad_loss, verts, faces, first, num, ctx.method, ws)
        return grad, None, None, None, None


class _NormalConsistency(torch.autograd.Function):
    @staticmethod
    def forward(ctx, verts, faces, first, num):
        loss, ws = _C.mesh_normal_consistency_forward(verts, faces, first, num)
        ctx.save_for_backward(verts, faces, first, num, ws)
        return loss

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_loss):
        verts, faces, first, num, ws = ctx.saved_tensors
        grad = None
        if ctx.needs_input_grad[0]:
            grad = _C.mesh_normal_consistency_backward(grad_loss, verts, faces, first, num, ws)
        return grad, None, None, None


def mesh_edge_loss(meshes, target_length: float = 0.0):
    """Sum over each mesh's edges of (|v0 - v1| - target_length)^2 / (its edge count), averaged over len(meshes)."""
    if _empty(meshes):
        return _zero(meshes)
    return _EdgeLoss.apply(*_packed(meshes), float(target_length))


def mesh_laplacian_smoothing(meshes, method: str = "uniform"):
    """Sum over each mesh's vertices of |L v| / (its vertex count), averaged over len(meshes), with the uniform,
    cotangent ("cot") or cotangent-curvature ("cotcurv") Laplacian of the reference; L is a constant of the
    gradient."""
    if _empty(meshes):
        return _zero(meshes)  # before the method check, as in the reference
    if method not in _C.LAPLACIAN_METHODS:
        raise ValueError("Method should be one of {uniform, cot, cotcurv}")
    return _LaplacianSmoothing.apply(*_packed(meshes), method)


def mesh_normal_consistency(meshes):
    """Over every pair of faces around an edge, 1 - cos(n_a, -n_b), weighted by 1 / (the pairs of its mesh) and
    averaged over len(meshes)."""
    if _empty(meshes):
        return _zero(meshes)
    return _NormalConsistency.apply(*_packed(meshes))
