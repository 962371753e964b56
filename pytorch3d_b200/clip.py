"""Frustum culling and z-clipping of faces before rasterization, and mapping the result back.

Row f1 of the scope table (SURVEY.md 8f): the pre/post step that `rasterize_meshes(z_clip_value=...,
cull_to_frustum=...)` runs around the native op, and that `MeshRasterizer` switches on by default for
perspective cameras.  Same public surface as pytorch3d/renderer/mesh/clip.py (ClipFrustum :84-148, ClippedFaces
:20-82, clip_faces :324-615, convert_clipped_rasterization_to_original_faces :618-734).

Faces fall into four cases (clip.py:386-423 of the reference):
  1  entirely in front of z_clip_value and not culled   -> kept
  2  entirely behind, or outside the frustum            -> dropped
  3  two vertices behind                                -> replaced by the triangle (p4, p5, p1)
  4  one vertex behind                                  -> the remaining quad becomes (p4, p2, p5) and (p5, p2, p3),
                                                           which name each other in clipped_faces_neighbor_idx
where p4 / p5 are the intersections of the edges p1-p2 / p1-p3 with the plane z = z_clip_value (interpolated in
world space when the camera is a perspective one).

This implementation is written for the GPU: it is one vectorised pass over all faces with no boolean-mask
indexing and no `nonzero` -- every face computes its output slot(s) from an exclusive prefix sum and writes through
`index_copy_` into arrays with one spare slot for "nothing to write" -- so the only host synchronisation is the single
read of the output size (the reference syncs five times).  All arithmetic that produces vertex positions and
barycentric conversions uses the reference's formulas and stays differentiable.
"""
from typing import Optional, Tuple

import torch

from . import _C


class ClippedFaces:
    """Clipped faces plus what is needed to map rasterization results back to the unclipped faces
    (same fields as the reference class, clip.py:20-82)."""

    __slots__ = [
        "face_verts",
        "mesh_to_face_first_idx",
        "num_faces_per_mesh",
        "faces_clipped_to_unclipped_idx",
        "barycentric_conversion",
        "faces_clipped_to_conversion_idx",
        "clipped_faces_neighbor_idx",
    ]

    def __init__(self, face_verts, mesh_to_face_first_idx, num_faces_per_mesh, faces_clipped_to_unclipped_idx=None,
                 barycentric_conversion=None, faces_clipped_to_conversion_idx=None,
                 clipped_faces_neighbor_idx=None) -> None:
        self.face_verts = face_verts
        self.mesh_to_face_first_idx = mesh_to_face_first_idx
        self.num_faces_per_mesh = num_faces_per_mesh
        self.faces_clipped_to_unclipped_idx = faces_clipped_to_unclipped_idx
        self.barycentric_conversion = barycentric_conversion
        self.faces_clipped_to_conversion_idx = faces_clipped_to_conversion_idx
        self.clipped_faces_neighbor_idx = clipped_faces_neighbor_idx


class ClipFrustum:
    """View frustum (left, right, top, bottom, znear, zfar) + clipping behaviour (clip.py:84-148 of the reference)."""

    __slots__ = ["left", "right", "top", "bottom", "znear", "zfar", "perspective_correct", "cull", "z_clip_value"]

    def __init__(self, left: Optional[float] = None, right: Optional[float] = None, top: Optional[float] = None,
                 bottom: Optional[float] = None, znear: Optional[float] = None, zfar: Optional[float] = None,
                 perspective_correct: bool = False, cull: bool = True, z_clip_value: Optional[float] = None) -> None:
        self.left = left
        self.right = right
        self.top = top
        self.bottom = bottom
        self.znear = znear
        self.zfar = zfar
        self.perspective_correct = perspective_correct
        self.cull = cull
        self.z_clip_value = z_clip_value


def _get_culled_faces(face_verts: torch.Tensor, frustum: ClipFrustum) -> torch.Tensor:
    """Faces to cull (clip.py:151-195 of the reference).

    Bug-compatible on purpose: the reference indexes `face_verts[:, axis]` on an (F,3,3) tensor, i.e. it takes
    VERTEX number `axis` of every face and requires all three of that vertex's coordinates to be beyond the
    plane value -- not "coordinate `axis` of all three vertices" as its comment says.  A drop-in has to make the
    same decisions, so the same expression is used here."""
    planes = ((frustum.left, 0, "<"), (frustum.right, 0, ">"), (frustum.top, 1, "<"), (frustum.bottom, 1, ">"),
              (frustum.znear, 2, "<"), (frustum.zfar, 2, ">"))
    culled = torch.zeros([face_verts.shape[0]], dtype=torch.bool, device=face_verts.device)
    if not frustum.cull:
        return culled
    for value, axis, op in planes:
        if value is None:
            continue
        out = face_verts[:, axis] < value if op == "<" else face_verts[:, axis] > value
        culled |= out.sum(1) == 3
    return culled


def _intersections(face_verts, p1_ind, active, clip_value: float, perspective_correct: bool):
    """p1..p5 and their barycentric weights w.r.t. the original triangle, for EVERY face; rows of faces that are
    not case 3/4 (`active` False) are never used and get a harmless denominator so that no NaN can reach the
    gradients through torch.where.  Formulas of clip.py:198-321."""
    F = face_verts.shape[0]
    p2_ind = torch.remainder(p1_ind + 1, 3)
    p3_ind = torch.remainder(p1_ind + 2, 3)

    def pick(ind):
        return face_verts.gather(1, ind[:, None, None].expand(-1, -1, 3)).squeeze(1)

    p1, p2, p3 = pick(p1_ind), pick(p2_ind), pick(p3_ind)
    one = torch.ones_like(p1[:, 2])
    w2 = (p1[:, 2] - clip_value) / torch.where(active, p1[:, 2] - p2[:, 2], one)
    p4 = p1 * (1 - w2[:, None]) + p2 * w2[:, None]
    if perspective_correct:
        p1_world = p1[:, :2] * p1[:, 2:3]
        p2_world = p2[:, :2] * p2[:, 2:3]
        p4 = torch.cat([(p1_world * (1 - w2[:, None]) + p2_world * w2[:, None]) / clip_value, p4[:, 2:3]], 1)
    w3 = ((p1[:, 2] - clip_value) / torch.where(active, p1[:, 2] - p3[:, 2], one)).detach()  # detached in the reference too (:287)
    p5 = p1 * (1 - w3[:, None]) + p3 * w3[:, None]
    if perspective_correct:
        p1_world = p1[:, :2] * p1[:, 2:3]
        p3_world = p3[:, :2] * p3[:, 2:3]
        p5 = torch.cat([(p1_world * (1 - w3[:, None]) + p3_world * w3[:, None]) / clip_value, p5[:, 2:3]], 1)

    def onehot(ind, value=None):
        o = torch.zeros((F, 3), device=face_verts.device, dtype=face_verts.dtype)
        src = torch.ones((F, 1), device=face_verts.device, dtype=face_verts.dtype) if value is None else value[:, None]
        return o.scatter(1, ind[:, None], src)

    b1, b2, b3 = onehot(p1_ind), onehot(p2_ind), onehot(p3_ind)
    b4 = onehot(p1_ind, 1 - w2) + onehot(p2_ind, w2)
    b5 = onehot(p1_ind, 1 - w3) + onehot(p3_ind, w3)
    return (p1, p2, p3, p4, p5), (b1, b2, b3, b4, b5)


def clip_faces(face_verts_unclipped: torch.Tensor, mesh_to_face_first_idx: torch.Tensor,
               num_faces_per_mesh: torch.Tensor, frustum: ClipFrustum) -> ClippedFaces:
    """Cull faces outside the frustum and clip faces to z >= frustum.z_clip_value (clip.py:324-615)."""
    F = face_verts_unclipped.shape[0]
    device = face_verts_unclipped.device
    fv = face_verts_unclipped
    culled = _get_culled_faces(fv, frustum)
    z_clip = frustum.z_clip_value
    if z_clip is not None:
        behind = fv[:, :, 2] < z_clip
        n_behind = behind.sum(1)
    else:
        behind = torch.zeros((F, 3), dtype=torch.bool, device=device)
        n_behind = torch.zeros([F], dtype=torch.int64, device=device)

    keep = ~culled
    case1 = (n_behind == 0) & keep
    case3 = (n_behind == 2) & keep
    case4 = (n_behind == 1) & keep
    out_count = case1.long() + case3.long() + 2 * case4.long()
    first_out = out_count.cumsum(0) - out_count  # faces_unclipped_to_clipped_idx
    # the only host synchronisation: output size (and the "nothing to do" early exit, clip.py:373-378)
    F_clipped, n_changed = (int(v) for v in torch.stack([out_count.sum(), (~case1).sum()]).tolist())
    if n_changed == 0:
        return ClippedFaces(face_verts=fv, mesh_to_face_first_idx=mesh_to_face_first_idx,
                            num_faces_per_mesh=num_faces_per_mesh)

    # per-mesh ranges in the clipped numbering (empty meshes keep first == next first)
    N = mesh_to_face_first_idx.shape[0]
    first_ext = torch.cat([first_out, first_out.new_full((1,), F_clipped)])
    first_clipped = first_ext[mesh_to_face_first_idx.clamp(max=F)]
    end_clipped = first_ext[(mesh_to_face_first_idx + num_faces_per_mesh).clamp(max=F)]
    num_clipped = end_clipped - first_clipped
    arange_f = torch.arange(F, device=device)

    if z_clip is None or F == 0:
        # culling only: compact case 1 faces
        dest = torch.where(case1, first_out, first_out.new_full((1,), F_clipped))
        verts = fv.new_zeros((F_clipped + 1, 3, 3)).index_copy(0, dest, fv)[:F_clipped]
        c2u = torch.zeros([F_clipped + 1], dtype=torch.int64, device=device).index_copy(0, dest, arange_f)[:F_clipped]
        return ClippedFaces(face_verts=verts, mesh_to_face_first_idx=first_clipped, num_faces_per_mesh=num_clipped,
                            faces_clipped_to_unclipped_idx=c2u)

    # p1 = the vertex that is alone on its side of the plane: case 3 -> the one in front, case 4 -> the one behind
    lone = torch.where(case3[:, None], ~behind, behind)
    p1_ind = lone.long().argmax(1)
    (p1, p2, p3, p4, p5), (b1, b2, b3, b4, b5) = _intersections(fv, p1_ind, case3 | case4, float(z_clip),
                                                                frustum.perspective_correct)

    # output triangle A of every face, and triangle B of case-4 faces
    tri_a = torch.where(case3[:, None, None], torch.stack((p4, p5, p1), 1),
                        torch.where(case4[:, None, None], torch.stack((p4, p2, p5), 1), fv))
    tri_b = torch.stack((p5, p2, p3), 1)
    bary_a = torch.where(case3[:, None, None], torch.stack((b4, b5, b1), 2), torch.stack((b4, b2, b5), 2))
    bary_b = torch.stack((b5, b2, b3), 2)

    spare = first_out.new_full((1,), F_clipped)
    dest_a = torch.where(out_count > 0, first_out, spare)
    dest_b = torch.where(case4, first_out + 1, spare)
    # NaN/inf rows of faces that are not case 3/4 must not leak through the spare slot into gradients
    tri_b = torch.where(case4[:, None, None], tri_b, torch.zeros_like(tri_b))
    converts = case3 | case4
    bary_a = torch.where(converts[:, None, None], bary_a, torch.zeros_like(bary_a))
    bary_b = torch.where(case4[:, None, None], bary_b, torch.zeros_like(bary_b))

    verts = fv.new_zeros((F_clipped + 1, 3, 3)).index_copy(0, dest_a, tri_a).index_copy(0, dest_b, tri_b)[:F_clipped]
    c2u = torch.zeros([F_clipped + 1], dtype=torch.int64, device=device)
    c2u = c2u.index_copy(0, dest_a, arange_f).index_copy(0, dest_b, arange_f)[:F_clipped]

    # barycentric conversion: one row per clipped face (identity rows are marked -1 in the index and never used)
    conv = fv.new_zeros((F_clipped + 1, 3, 3)).index_copy(0, dest_a, bary_a).index_copy(0, dest_b, bary_b)[:F_clipped]
    conv_idx = torch.full([F_clipped + 1], -1, dtype=torch.int64, device=device)
    conv_idx = conv_idx.index_copy(0, torch.where(converts, first_out, spare), first_out)
    conv_idx = conv_idx.index_copy(0, dest_b, first_out + 1)
    conv_idx = torch.cat([conv_idx[:F_clipped], conv_idx.new_full((1,), -1)])[:F_clipped]

    neighbor = torch.full([F_clipped + 1], -1, dtype=torch.int64, device=device)
    dest_a4 = torch.where(case4, first_out, spare)
    neighbor = neighbor.index_copy(0, dest_a4, first_out + 1).index_copy(0, dest_b, first_out)
    neighbor = torch.cat([neighbor[:F_clipped], neighbor.new_full((1,), -1)])[:F_clipped]

    return ClippedFaces(face_verts=verts, mesh_to_face_first_idx=first_clipped, num_faces_per_mesh=num_clipped,
                        faces_clipped_to_unclipped_idx=c2u, barycentric_conversion=conv,
                        faces_clipped_to_conversion_idx=conv_idx, clipped_faces_neighbor_idx=neighbor)


def convert_clipped_rasterization_to_original_faces(pix_to_face_clipped, bary_coords_clipped,
                                                    clipped_faces: ClippedFaces) -> Tuple[torch.Tensor, torch.Tensor]:
    """Map face indices and barycentrics of a rasterization of the clipped faces back to the unclipped faces
    (clip.py:618-734): alpha_unclipped = barycentric_conversion[f] @ alpha_clipped."""
    c2u = clipped_faces.faces_clipped_to_unclipped_idx
    if c2u is None or c2u.numel() == 0:
        return pix_to_face_clipped, bary_coords_clipped
    valid = pix_to_face_clipped != -1
    safe = pix_to_face_clipped.clamp(min=0)
    pix_to_face_unclipped = torch.where(valid, c2u[safe], torch.full_like(pix_to_face_clipped, -1))
    conversion = clipped_faces.barycentric_conversion
    if conversion is None:
        return pix_to_face_unclipped, bary_coords_clipped
    conv_idx = torch.where(valid, clipped_faces.faces_clipped_to_conversion_idx[safe],
                           torch.full_like(pix_to_face_clipped, -1))
    mask = conv_idx != -1
    rows = conv_idx[mask]  # (boolean indexing: the one sync of this step, as in the reference)
    sub = bary_coords_clipped[mask]  # (M, 3)
    converted = torch.bmm(conversion[rows], sub[:, :, None])[:, :, 0]
    bary_unclipped = bary_coords_clipped.clone()
    bary_unclipped[mask] = converted
    return pix_to_face_unclipped, bary_unclipped


# ------------------------------------------------------------------------------------------ fused (CUDA) versions
# The same two steps on the GPU kernels of csrc/clip.cu (DESIGN.md section 14), with the reference's output layout:
# barycentric_conversion has one row per clipped face that needs one -- case-3 faces, then the first and then the
# second halves of case-4 faces -- and faces_clipped_to_conversion_idx points into it.  The host reads one four-word
# record per forward call (output sizes, and whether anything was culled or clipped at all); nothing else synchronises.

class _ClipFacesFused(torch.autograd.Function):
    """Fill pass and its backward; differentiable outputs: face_verts and barycentric_conversion."""

    @staticmethod
    def forward(ctx, face_verts, mesh_to_face_first_idx, num_faces_per_mesh, frustum, workspace, record):
        outs = _C.clip_faces_fill(face_verts, mesh_to_face_first_idx, num_faces_per_mesh, frustum, workspace, record)
        ctx.save_for_backward(face_verts, workspace)
        ctx.frustum, ctx.record = frustum, tuple(record)
        ctx.mark_non_differentiable(outs[1], outs[2], outs[3], outs[5], outs[6])
        ctx.set_materialize_grads(False)
        return outs

    @staticmethod
    def backward(ctx, grad_face_verts, _g1, _g2, _g3, grad_conversion, _g5, _g6):
        face_verts, workspace = ctx.saved_tensors
        grad = None
        if ctx.needs_input_grad[0] and (grad_face_verts is not None or grad_conversion is not None):
            grad = _C.clip_faces_backward(face_verts, ctx.frustum, workspace, ctx.record, grad_face_verts,
                                          grad_conversion)
        return grad, None, None, None, None, None


def _clip_faces_counted(face_verts, mesh_to_face_first_idx, num_faces_per_mesh, frustum, workspace, record):
    """clip_faces_fused after its count pass; `record` is the workspace's first four words, read by the caller."""
    F_clipped, n3, n4, changed = (int(v) for v in record)
    if changed == 0:  # nothing culled or clipped: the reference returns its inputs (clip.py:384-389)
        return ClippedFaces(face_verts=face_verts, mesh_to_face_first_idx=mesh_to_face_first_idx,
                            num_faces_per_mesh=num_faces_per_mesh)
    fv, first, num, c2u, conv, conv_idx, neighbor = _ClipFacesFused.apply(
        face_verts, mesh_to_face_first_idx, num_faces_per_mesh, frustum, workspace, record)
    if n3 + n4 == 0:  # only culled (clip.py:465-471)
        return ClippedFaces(face_verts=fv, mesh_to_face_first_idx=first, num_faces_per_mesh=num,
                            faces_clipped_to_unclipped_idx=c2u)
    return ClippedFaces(face_verts=fv, mesh_to_face_first_idx=first, num_faces_per_mesh=num,
                        faces_clipped_to_unclipped_idx=c2u, barycentric_conversion=conv,
                        faces_clipped_to_conversion_idx=conv_idx, clipped_faces_neighbor_idx=neighbor)


def clip_faces_fused(face_verts_unclipped: torch.Tensor, mesh_to_face_first_idx: torch.Tensor,
                     num_faces_per_mesh: torch.Tensor, frustum: ClipFrustum) -> ClippedFaces:
    """`clip_faces` on the GPU for float32 CUDA tensors, in the reference's layout (a drop-in for
    pytorch3d.renderer.mesh.clip.clip_faces).  Differentiable w.r.t. face_verts_unclipped through the clipped
    face_verts and barycentric_conversion.  One host synchronisation: the read of the count pass's record."""
    workspace = _C.clip_faces_count(frustum, face_verts=face_verts_unclipped)
    record = workspace[:4].tolist()
    return _clip_faces_counted(face_verts_unclipped, mesh_to_face_first_idx, num_faces_per_mesh, frustum, workspace,
                               record)


class _ConvertClippedFused(torch.autograd.Function):
    """Barycentric conversion of a rasterization of clipped faces; differentiable w.r.t. bary and the conversion."""

    @staticmethod
    def forward(ctx, pix_to_face, bary, conversion, c2u, conv_idx):
        p2f, bary_u = _C.clip_convert_forward(pix_to_face, bary, c2u, conversion, conv_idx)
        ctx.save_for_backward(pix_to_face, bary, conversion, conv_idx)
        ctx.mark_non_differentiable(p2f)
        ctx.set_materialize_grads(False)
        return p2f, bary_u

    @staticmethod
    def backward(ctx, _grad_p2f, grad_bary):
        pix_to_face, bary, conversion, conv_idx = ctx.saved_tensors
        need = (ctx.needs_input_grad[1], ctx.needs_input_grad[2])
        if grad_bary is None or not any(need):
            return None, None, None, None, None
        g_bary, g_conv = _C.clip_convert_backward(grad_bary, pix_to_face, bary, conversion, conv_idx, need)
        return None, g_bary, g_conv, None, None


def convert_clipped_fused(pix_to_face_clipped: torch.Tensor, bary_coords_clipped: torch.Tensor,
                          clipped_faces) -> Tuple[torch.Tensor, torch.Tensor]:
    """`convert_clipped_rasterization_to_original_faces` on the GPU, for any ClippedFaces in the reference's layout
    (from clip_faces_fused or from the reference's own clip_faces).  No host synchronisation."""
    c2u = clipped_faces.faces_clipped_to_unclipped_idx
    if c2u is None or c2u.numel() == 0:
        return pix_to_face_clipped, bary_coords_clipped
    conversion = clipped_faces.barycentric_conversion
    if conversion is None:
        return _C.clip_convert_forward(pix_to_face_clipped, bary_coords_clipped, c2u)[0], bary_coords_clipped
    return _ConvertClippedFused.apply(pix_to_face_clipped, bary_coords_clipped, conversion, c2u,
                                      clipped_faces.faces_clipped_to_conversion_idx)
