"""Mesh surface sampling on the GPU: `sample_points_from_meshes`, with the signature, return tuple, shapes, dtypes and
errors of pytorch3d/ops/sample_points_from_meshes.py.

Three fused kernels (DESIGN.md section 20) compute the face areas (the arithmetic of the reference's CUDA
face_areas_normals, bit for bit), a reproducible float64 prefix of them per mesh, and then every sample in one thread:
its face, its barycentrics, its position and, optionally, its normal.  The backward sums per-sample corner gradients
per vertex in a fixed order, with no float atomics.  The forward synchronises the host exactly once, to read the one
status word that decides the reference's error checks; the backward never does.

One divergence: the draws come from a counter-based generator (Philox4x32-10, one evaluation per sample, keyed by a
seed drawn from torch's default CUDA generator), not from torch's multinomial and rand streams.  For a given
`torch.manual_seed` the samples differ from the reference's; their distribution is the same, and given the same face
and (u, v) the positions are bit-identical.  Unlike the reference (torch.multinomial takes at most 2^24 categories),
meshes with more than 2^24 faces are sampled.

The function takes a PyTorch3D `Meshes` or a `PackedMeshes`: anything with `verts_packed()`, `faces_packed()`,
`mesh_to_faces_packed_first_idx()`, `num_faces_per_mesh()` and `len()` (and `textures` / `sample_textures` for
`return_textures`), on a CUDA device, with float32 verts and int64 faces.  Gradients reach `verts_packed()`.
"""
import torch
from torch.autograd.function import once_differentiable

from . import _C

__all__ = ["sample_points_from_meshes"]


class EmptyMeshWithTextures(RuntimeError):
    """`return_textures=True` on a batch with a mesh without faces: the reference fails there (reshaping its face draws
    of the non-empty meshes to (N, S, 1, 1)), so `install_sampling()` sends such a call to it."""


class _SamplePoints(torch.autograd.Function):
    @staticmethod
    def forward(ctx, verts, faces, first, num, num_samples, return_normals, seed, draws):
        if draws is None:
            samples, normals, face_idx, bary, status = _C.sample_points_forward(verts, faces, first, num, num_samples,
                                                                                return_normals, seed)
        else:
            samples, normals, face_idx, bary, status = _C._sample_points_from_draws(verts, faces, first, num,
                                                                                    return_normals, *draws)
        ctx.save_for_backward(verts, faces, face_idx, bary)
        ctx.return_normals = return_normals
        ctx.mark_non_differentiable(face_idx, bary, status)
        if normals is None:
            return samples, face_idx, bary, status
        return samples, normals, face_idx, bary, status

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_samples, *rest):
        verts, faces, face_idx, bary = ctx.saved_tensors
        grad = None
        if ctx.needs_input_grad[0]:
            grad_normals = rest[0].contiguous() if ctx.return_normals else None
            grad = _C.sample_points_backward(grad_samples.contiguous(), grad_normals, verts, faces, face_idx, bary)
        return grad, None, None, None, None, None, None, None


def _check_status(status, meshes, return_textures):
    """The reference's checks, in its order, decided by the status word read once."""
    s = int(status.item())
    if not s & _C.SAMPLE_HAS_VALID:
        raise ValueError("Meshes are empty.")
    if s & _C.SAMPLE_NONFINITE:
        raise ValueError("Meshes contain nan or inf.")
    if return_textures and meshes.textures is None:
        raise ValueError("Meshes do not contain textures.")
    if s & _C.SAMPLE_BAD_TOTAL:
        raise RuntimeError("invalid multinomial distribution (sum of probabilities <= 0)")
    if return_textures and s & _C.SAMPLE_HAS_EMPTY:
        raise EmptyMeshWithTextures("sample_points_from_meshes: return_textures needs every mesh to have a face")


def _fragments(face_idx, bary):
    try:
        from pytorch3d.renderer.mesh.rasterizer import Fragments
    except ImportError:
        from .rasterizer import Fragments
    N, S = face_idx.shape
    dummy = torch.zeros((N, S, 1, 1), device=face_idx.device, dtype=torch.float32)
    return Fragments(pix_to_face=face_idx.view(N, S, 1, 1), zbuf=dummy, bary_coords=bary.view(N, S, 1, 1, 3),
                     dists=dummy)


def _sample(meshes, num_samples, return_normals, return_textures, draws):
    if len(meshes) == 0:
        raise ValueError("Meshes are empty.")
    verts, faces = meshes.verts_packed(), meshes.faces_packed()
    first, num = meshes.mesh_to_faces_packed_first_idx(), meshes.num_faces_per_mesh()
    seed = None
    if draws is None:  # drawn on the device, so that the host never waits for it
        seed = torch.randint(0, 1 << 32, (2,), dtype=torch.int64, device=verts.device)
    out = _SamplePoints.apply(verts, faces, first, num, int(num_samples), bool(return_normals), seed, draws)
    samples, normals = out[0], (out[1] if return_normals else None)
    face_idx, bary, status = out[-3:]
    _check_status(status, meshes, return_textures)
    textures = None
    if return_textures:
        textures = meshes.sample_textures(_fragments(face_idx, bary))[:, :, 0, 0, :]
    if return_normals and return_textures:
        return samples, normals, textures
    if return_normals:
        return samples, normals
    if return_textures:
        return samples, textures
    return samples


def sample_points_from_meshes(meshes, num_samples: int = 10000, return_normals: bool = False,
                              return_textures: bool = False):
    """`num_samples` points on the surface of each mesh, each face drawn with probability proportional to its area and
    the point uniform on it: samples (N, S, 3), and normals (N, S, 3) and textures (N, S, C) when asked for, as in the
    reference.  Rows of meshes without faces are zeros, with zero gradient."""
    return _sample(meshes, num_samples, return_normals, return_textures, None)


def _sample_from_draws(meshes, face_idx, u, v, return_normals=False, return_textures=False):
    """Test hook: `sample_points_from_meshes` with the draws given -- face_idx (N, S) int64 packed faces, u and v
    (N, S) float32 -- instead of drawn, differentiable like it."""
    return _sample(meshes, face_idx.shape[1], return_normals, return_textures, (face_idx, u, v))
