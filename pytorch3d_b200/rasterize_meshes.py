"""`rasterize_meshes` with the reference's keyword signature, on the H100-native kernels.

Mirrors pytorch3d/renderer/mesh/rasterize_meshes.py:32-357 (wrapper + torch.autograd.Function); the
native ops come from `pytorch3d_b200._C` instead of `pytorch3d._C`.
"""
from typing import List, Optional, Tuple, Union

import numpy as np
import torch

from . import _C
from .clip import (ClipFrustum, _clip_faces_counted, clip_faces, convert_clipped_fused,
                   convert_clipped_rasterization_to_original_faces)

# kMaxItemsPerBin (rasterization_utils.cuh:50); mirrored by rasterize_meshes.py:24-27 of the reference
kMaxFacesPerBin = 22


def parse_image_size(image_size: Union[List[int], Tuple[int, int], int]) -> Tuple[int, int]:
    """(H, W) from an int or a 2-sequence; same checks as pytorch3d/renderer/utils.py:432-457."""
    if not isinstance(image_size, (tuple, list)):
        return (image_size, image_size)
    if len(image_size) != 2:
        raise ValueError("Image size can only be a tuple/list of (H, W)")
    if not all(i > 0 for i in image_size):
        raise ValueError("Image sizes must be greater than 0; got %d, %d" % tuple(image_size))
    if not all(isinstance(i, int) for i in image_size):
        raise ValueError("Image sizes must be integers; got %f, %f" % tuple(image_size))
    return tuple(image_size)


def rasterize_meshes(
    meshes,
    image_size: Union[int, List[int], Tuple[int, int]] = 256,
    blur_radius: float = 0.0,
    faces_per_pixel: int = 8,
    bin_size: Optional[int] = None,
    max_faces_per_bin: Optional[int] = None,
    perspective_correct: bool = False,
    clip_barycentric_coords: bool = False,
    cull_backfaces: bool = False,
    z_clip_value: Optional[float] = None,
    cull_to_frustum: bool = False,
):
    """
    Rasterize a batch of meshes (NDC coordinates, +X left, +Y up) to (N, H, W, faces_per_pixel) buffers.

    Same arguments, return values and error behaviour as the reference function
    (pytorch3d/renderer/mesh/rasterize_meshes.py:32-251).  `meshes` is any object exposing the packed
    accessors of pytorch3d.structures.Meshes.  `bin_size` / `max_faces_per_bin` are validated like in the
    reference but are only hints: tiling is exact, faces are never dropped and the result does not depend
    on them.

    Returns (pix_to_face int64, zbuf, barycentric_coords, pix_dists), each (N, H, W, K[, 3]), -1 padded.
    """
    verts_packed = meshes.verts_packed()
    faces_packed = meshes.faces_packed()
    mesh_to_face_first_idx = meshes.mesh_to_faces_packed_first_idx()
    num_faces_per_mesh = meshes.num_faces_per_mesh()

    im_size = parse_image_size(image_size)
    max_image_size = max(*im_size)

    if bin_size is None:
        if max_image_size <= 64:
            bin_size = 8
        else:
            bin_size = int(2 ** max(np.ceil(np.log2(max_image_size)) - 4, 4))
    if bin_size != 0:
        faces_per_bin = 1 + (max_image_size - 1) // bin_size
        if faces_per_bin >= kMaxFacesPerBin:
            raise ValueError(
                "bin_size too small, number of faces per bin must be less than %d; got %d"
                % (kMaxFacesPerBin, faces_per_bin))
    if max_faces_per_bin is None:
        max_faces_per_bin = int(max(10000, getattr(meshes, "_F", 0) / 5))

    if z_clip_value is None and not cull_to_frustum:
        # no clipping: the gather `verts_packed[faces_packed]` (rasterize_meshes.py:144-148 of the reference) and
        # its backward scatter run inside the native op (b200r_rasterize_meshes_*_indexed)
        return _RasterizeMeshesIndexed.apply(
            verts_packed, faces_packed, mesh_to_face_first_idx, num_faces_per_mesh, im_size, blur_radius,
            faces_per_pixel, perspective_correct, clip_barycentric_coords, cull_backfaces)

    # Cull faces outside the view frustum and clip faces that are partially behind the camera to
    # z >= z_clip_value; this may change the number of faces (rasterize_meshes.py:160-183 of the reference)
    frustum = ClipFrustum(left=-1, right=1, top=-1, bottom=1, perspective_correct=perspective_correct,
                          z_clip_value=z_clip_value, cull=cull_to_frustum)
    fused = verts_packed.is_cuda and verts_packed.dtype == torch.float32
    if fused:
        # count pass on verts[faces] in place; its record is the forward's one host read
        workspace = _C.clip_faces_count(frustum, verts=verts_packed, faces=faces_packed)
        record = workspace[:4].tolist()
        if record[3] == 0:
            # nothing culled or clipped: clip_faces would return its input unchanged, so the fused gather path
            # computes the same Fragments without materialising face_verts
            return _RasterizeMeshesIndexed.apply(
                verts_packed, faces_packed, mesh_to_face_first_idx, num_faces_per_mesh, im_size, blur_radius,
                faces_per_pixel, perspective_correct, clip_barycentric_coords, cull_backfaces)
        face_verts = verts_packed[faces_packed]
        clipped_faces = _clip_faces_counted(face_verts, mesh_to_face_first_idx, num_faces_per_mesh, frustum,
                                            workspace, record)
    else:
        face_verts = verts_packed[faces_packed]
        clipped_faces = clip_faces(face_verts, mesh_to_face_first_idx, num_faces_per_mesh, frustum=frustum)
    face_verts = clipped_faces.face_verts
    mesh_to_face_first_idx = clipped_faces.mesh_to_face_first_idx
    num_faces_per_mesh = clipped_faces.num_faces_per_mesh
    # the two halves of a face that was clipped to a quad name each other: only one may enter the top K
    clipped_faces_neighbor_idx = clipped_faces.clipped_faces_neighbor_idx
    if clipped_faces_neighbor_idx is None:
        clipped_faces_neighbor_idx = torch.full(
            size=(face_verts.shape[0],), fill_value=-1, device=face_verts.device, dtype=torch.int64)
        clipped_faces_neighbor_idx._b200_all_minus_one = True  # selects the kernel variant without that logic

    pix_to_face, zbuf, barycentric_coords, dists = _RasterizeFaceVerts.apply(
        face_verts, mesh_to_face_first_idx, num_faces_per_mesh, clipped_faces_neighbor_idx, im_size, blur_radius,
        faces_per_pixel, bin_size, max_faces_per_bin, perspective_correct, clip_barycentric_coords, cull_backfaces)

    # express face indices and barycentrics in terms of the original, unclipped faces
    # (rasterize_meshes.py:239-249 of the reference)
    convert = convert_clipped_fused if fused else convert_clipped_rasterization_to_original_faces
    pix_to_face, barycentric_coords = convert(pix_to_face, barycentric_coords, clipped_faces)
    return pix_to_face, zbuf, barycentric_coords, dists


def _zeros_where_none(pix_to_face, grad_zbuf, grad_bary, grad_dists):
    """Outputs that did not take part in the loss arrive as None (set_materialize_grads(False))."""
    shape, dev = tuple(pix_to_face.shape), pix_to_face.device
    if grad_zbuf is None:
        grad_zbuf = torch.zeros(shape, dtype=torch.float32, device=dev)
    if grad_bary is None:
        grad_bary = torch.zeros(shape + (3,), dtype=torch.float32, device=dev)
    if grad_dists is None:
        grad_dists = torch.zeros(shape, dtype=torch.float32, device=dev)
    return grad_zbuf, grad_bary, grad_dists


class _RasterizeMeshesIndexed(torch.autograd.Function):
    """`_RasterizeFaceVerts` fused with the face gather that precedes it: differentiable w.r.t. verts_packed."""

    @staticmethod
    def forward(ctx, verts_packed, faces_packed, mesh_to_face_first_idx, num_faces_per_mesh, image_size, blur_radius,
                faces_per_pixel, perspective_correct, clip_barycentric_coords, cull_backfaces):
        pix_to_face, zbuf, barycentric_coords, dists, face_verts = _C.rasterize_meshes_indexed(
            verts_packed, faces_packed, mesh_to_face_first_idx, num_faces_per_mesh, image_size, blur_radius,
            faces_per_pixel, perspective_correct, clip_barycentric_coords, cull_backfaces)
        ctx.save_for_backward(face_verts, faces_packed, pix_to_face)
        ctx.mark_non_differentiable(pix_to_face)
        # no zero-filled "gradient" for pix_to_face (134 MB of int64 zeros per step at the north-star size)
        ctx.set_materialize_grads(False)
        ctx.num_verts = int(verts_packed.shape[0])
        ctx.perspective_correct = perspective_correct
        ctx.clip_barycentric_coords = clip_barycentric_coords
        return pix_to_face, zbuf, barycentric_coords, dists

    @staticmethod
    def backward(ctx, grad_pix_to_face, grad_zbuf, grad_barycentric_coords, grad_dists):
        face_verts, faces_packed, pix_to_face = ctx.saved_tensors
        grad_zbuf, grad_barycentric_coords, grad_dists = _zeros_where_none(
            pix_to_face, grad_zbuf, grad_barycentric_coords, grad_dists)
        grad_verts = _C.rasterize_meshes_backward_indexed(
            face_verts, faces_packed, ctx.num_verts, pix_to_face, grad_zbuf, grad_barycentric_coords, grad_dists,
            ctx.perspective_correct, ctx.clip_barycentric_coords)
        return (grad_verts,) + (None,) * 9


class _RasterizeFaceVerts(torch.autograd.Function):
    """Autograd glue, same contract as the reference class (rasterize_meshes.py:254-357)."""

    @staticmethod
    def forward(ctx, face_verts, mesh_to_face_first_idx, num_faces_per_mesh, clipped_faces_neighbor_idx,
                image_size=(256, 256), blur_radius=0.01, faces_per_pixel=0, bin_size=0, max_faces_per_bin=0,
                perspective_correct=False, clip_barycentric_coords=False, cull_backfaces=False):
        pix_to_face, zbuf, barycentric_coords, dists = _C.rasterize_meshes(
            face_verts, mesh_to_face_first_idx, num_faces_per_mesh, clipped_faces_neighbor_idx, image_size,
            blur_radius, faces_per_pixel, bin_size, max_faces_per_bin, perspective_correct,
            clip_barycentric_coords, cull_backfaces)
        ctx.save_for_backward(face_verts, pix_to_face)
        ctx.mark_non_differentiable(pix_to_face)
        ctx.set_materialize_grads(False)
        ctx.perspective_correct = perspective_correct
        ctx.clip_barycentric_coords = clip_barycentric_coords
        return pix_to_face, zbuf, barycentric_coords, dists

    @staticmethod
    def backward(ctx, grad_pix_to_face, grad_zbuf, grad_barycentric_coords, grad_dists):
        face_verts, pix_to_face = ctx.saved_tensors
        grad_zbuf, grad_barycentric_coords, grad_dists = _zeros_where_none(
            pix_to_face, grad_zbuf, grad_barycentric_coords, grad_dists)
        grad_face_verts = _C.rasterize_meshes_backward(
            face_verts, pix_to_face, grad_zbuf, grad_barycentric_coords, grad_dists, ctx.perspective_correct,
            ctx.clip_barycentric_coords)
        return (grad_face_verts,) + (None,) * 11


def non_square_ndc_range(S1, S2):
    """NDC range of the axis with S1 pixels (rasterize_meshes.py:360-377 of the reference)."""
    ndc_range = 2.0
    if S1 > S2:
        ndc_range = (S1 / S2) * ndc_range
    return ndc_range


def pix_to_non_square_ndc(i, S1, S2):
    """NDC coordinate of the centre of pixel i (rasterize_meshes.py:380-401 of the reference)."""
    ndc_range = non_square_ndc_range(S1, S2)
    offset = ndc_range / 2.0
    return -offset + (ndc_range * i + offset) / S1
