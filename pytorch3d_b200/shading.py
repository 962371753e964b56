"""Phong, flat and Gouraud shading, same API as the reference's pytorch3d/renderer/mesh/shading.py: `phong_shading`,
`_phong_shading_with_pixels`, `flat_shading` and `gouraud_shading`, with the light models of
pytorch3d/renderer/lighting.py.

Each slot's position and normal are interpolated from its face (phong) or taken from the face (flat) and lit by one
point, directional or ambient light; the colour is `(ambient + diffuse) * texel + specular`.  The reference writes about
two dozen (N,H,W,K[,3]) tensors for this; here the forward is one kernel and the backward one kernel plus, when a light,
material or camera tensor requires grad, a small reduction (DESIGN.md section 12).  Neither synchronises the host.

Objects are duck-typed.  `meshes` needs `verts_packed`, `faces_packed` and `verts_normals_packed` (phong) or
`faces_normals_packed` (flat); `cameras` needs `get_camera_center`; `materials` needs `ambient_color`,
`diffuse_color`, `specular_color` and `shininess`.  A light with a `location` is a point light, one with a `direction`
a directional light, and one with neither an ambient light.  Gradients reach the texels, the barycentric coordinates,
the vertices and normals, and every light, material and camera tensor.

`gouraud_shading` lights every vertex instead (one kernel), then interpolates the shaded vertex colours at the slots
(a second one), with no (F, 3, 3) gather (DESIGN.md section 16).  Its `meshes` also needs `textures` with
`verts_features_packed`, `num_verts_per_mesh` and `mesh_to_verts_packed_first_idx`; its parameter rows are per mesh.
"""
from typing import Tuple

import torch

from . import _C

__all__ = ["phong_shading", "_phong_shading_with_pixels", "flat_shading", "gouraud_shading", "light_kind"]


class _Shading(torch.autograd.Function):
    @staticmethod
    def forward(ctx, texels, bary, face_positions, face_normals, params, pix_to_face, flat, light, return_positions):
        colors, positions = _C.shading_forward(pix_to_face, bary, face_positions, face_normals, texels, params, flat,
                                               light, return_positions)
        ctx.save_for_backward(texels, bary, face_positions, face_normals, params, pix_to_face)
        ctx.args = (flat, light)
        return (colors, positions) if return_positions else colors

    @staticmethod
    def backward(ctx, grad_colors, grad_positions=None):
        texels, bary, face_positions, face_normals, params, pix_to_face = ctx.saved_tensors
        flat, light = ctx.args
        grads = _C.shading_backward(grad_colors.contiguous(), grad_positions, pix_to_face, bary, face_positions,
                                    face_normals, texels, params, flat, light, ctx.needs_input_grad[:5])
        return grads + (None, None, None, None)


def light_kind(lights) -> str:
    """"point" for a light with a `location`, "directional" for one with a `direction`, "ambient" otherwise."""
    if hasattr(lights, "location"):
        return "point"
    if hasattr(lights, "direction"):
        return "directional"
    return "ambient"


def _rows(name, x, width, device):
    """A light, material or camera value as a float32 (B, width) tensor on `device`: a number or a (B,) / (width,)
    vector is reshaped, a (B, width) tensor kept."""
    t = (x if torch.is_tensor(x) else torch.tensor(x)).to(device=device, dtype=torch.float32)
    if t.dim() <= 1:
        t = t.reshape(-1, width) if t.numel() % width == 0 else t
    if t.dim() != 2 or t.shape[1] != width:
        raise ValueError("Expected %s to have shape (N, %d); got %r" % (name, width, tuple(t.shape)))
    return t


def _params(N, lights, cameras, materials, kind, device, batched_material_colors=False):
    """The per-image (per-mesh for Gouraud) parameter row (N, 22) of the shading kernels, with the reference's batch
    rules: every piece has batch 1 or N (ValueError "Got non-broadcastable sizes" otherwise).  `ambient` is formed as
    the reference forms it, `materials.ambient_color * lights.ambient_color`; autograd returns each piece's gradient to
    its source, summed over the batch where the source has batch 1.  Material diffuse and specular colours must have
    batch 1 unless `batched_material_colors` (Gouraud shading, where the reference gathers them per vertex)."""
    ambient = _rows("ambient_color", materials.ambient_color * lights.ambient_color, 3, device)
    md = _rows("diffuse_color", materials.diffuse_color, 3, device)
    ms = _rows("specular_color", materials.specular_color, 3, device)
    zeros = torch.zeros((1, 3), dtype=torch.float32, device=device)
    if kind == "ambient":  # no diffuse or specular term: the light colours, camera and shininess take no part
        ld = ls = where = cam = zeros
        shininess = zeros[:, :1]
    else:
        ld = _rows("diffuse_color", lights.diffuse_color, 3, device)
        ls = _rows("specular_color", lights.specular_color, 3, device)
        where = _rows(kind == "point" and "location" or "direction",
                      lights.location if kind == "point" else lights.direction, 3, device)
        cam = _rows("camera center", cameras.get_camera_center(), 3, device)
        shininess = _rows("shininess", materials.shininess, 1, device)
    pieces = [ambient, ld, ls, md, ms, where, cam, shininess]
    sizes = [N] + [int(p.shape[0]) for p in pieces]
    if any(s not in (1, N) for s in sizes):
        raise ValueError("Got non-broadcastable sizes %r" % sizes)
    if not batched_material_colors and (md.shape[0] != 1 or ms.shape[0] != 1):
        # the reference multiplies these (B, 3) colours into the (N, H, W, K, 3) light colours, which only broadcasts
        # for B = 1
        raise ValueError("Got non-broadcastable sizes %r: material diffuse and specular colours must have batch 1"
                         % sizes)
    return torch.cat([p.expand(N, p.shape[1]) for p in pieces], dim=1)


def _check_texels(texels, fragments):
    want = tuple(fragments.pix_to_face.shape) + (3,)
    if tuple(texels.shape) != want:
        raise ValueError("texels must have shape %r (N, H, W, K, 3); got %r" % (want, tuple(texels.shape)))


def _shade_phong(meshes, fragments, lights, cameras, materials, texels, return_positions):
    _check_texels(texels, fragments)
    kind = light_kind(lights)
    verts, faces = meshes.verts_packed(), meshes.faces_packed()
    faces_verts = verts[faces]
    faces_normals = None if kind == "ambient" else meshes.verts_normals_packed()[faces]
    N = int(fragments.pix_to_face.shape[0])
    params = _params(N, lights, cameras, materials, kind, texels.device)
    return _Shading.apply(texels, fragments.bary_coords, faces_verts, faces_normals, params, fragments.pix_to_face,
                          False, kind, return_positions)


def _phong_shading_with_pixels(meshes, fragments, lights, cameras, materials, texels
                               ) -> Tuple[torch.Tensor, torch.Tensor]:
    """Per-pixel Phong shading.  Returns (colors (N,H,W,K,3), pixel_coords (N,H,W,K,3)), the latter the interpolated
    positions (camera coordinates of each intersection, 0 in background slots), bit-identical to
    `interpolate_face_attributes(pix_to_face, bary_coords, verts[faces])`."""
    return _shade_phong(meshes, fragments, lights, cameras, materials, texels, True)


def phong_shading(meshes, fragments, lights, cameras, materials, texels) -> torch.Tensor:
    """Per-pixel Phong shading: positions and normals interpolated with the barycentric coordinates, then lit.
    texels (N,H,W,K,3) -> colors (N,H,W,K,3)."""
    return _shade_phong(meshes, fragments, lights, cameras, materials, texels, False)


def flat_shading(meshes, fragments, lights, cameras, materials, texels) -> torch.Tensor:
    """Per-face shading: the mean of the face's vertices and the face normal, lit.  texels (N,H,W,K,3) ->
    colors (N,H,W,K,3)."""
    _check_texels(texels, fragments)
    kind = light_kind(lights)
    verts, faces = meshes.verts_packed(), meshes.faces_packed()
    face_coords = verts[faces].mean(dim=-2)  # (F, 3), as the reference forms it
    face_normals = None if kind == "ambient" else meshes.faces_normals_packed()
    N = int(fragments.pix_to_face.shape[0])
    params = _params(N, lights, cameras, materials, kind, texels.device)
    return _Shading.apply(texels, None, face_coords, face_normals, params, fragments.pix_to_face, True, kind, False)


class _Gouraud(torch.autograd.Function):
    @staticmethod
    def forward(ctx, verts, normals, verts_colors, bary, params, first, num, faces, pix_to_face, light):
        colors, shaded = _C.gouraud_forward(verts, normals, verts_colors, first, num, params, faces, pix_to_face, bary,
                                            light)
        ctx.save_for_backward(verts, normals, verts_colors, bary, params, first, num, faces, pix_to_face, shaded)
        ctx.light = light
        return colors

    @staticmethod
    def backward(ctx, grad_colors):
        verts, normals, verts_colors, bary, params, first, num, faces, pix_to_face, shaded = ctx.saved_tensors
        grads = _C.gouraud_backward(grad_colors.contiguous(), verts, normals, verts_colors, first, num, params, faces,
                                    pix_to_face, bary, ctx.light, shaded, ctx.needs_input_grad[:5])
        return grads + (None, None, None, None, None)


def gouraud_shading(meshes, fragments, lights, cameras, materials) -> torch.Tensor:
    """Per-vertex shading: every vertex lit with its mesh's lights, camera and material, its colour
    `verts_colors * (ambient + diffuse) + specular`, then interpolated with the barycentric coordinates.  The vertex
    colours come from a `TexturesVertex` with 3 channels.  -> colors (N,H,W,K,3)."""
    textures = getattr(meshes, "textures", None)
    if not hasattr(textures, "verts_features_packed"):
        raise ValueError("Mesh textures must be an instance of TexturesVertex")
    verts, faces = meshes.verts_packed(), meshes.faces_packed()
    verts_colors = textures.verts_features_packed()
    if tuple(verts_colors.shape) != (verts.shape[0], 3):
        raise ValueError("Gouraud shading needs vertex colours of shape (V, 3) = %r; got %r"
                         % ((int(verts.shape[0]), 3), tuple(verts_colors.shape)))
    kind = light_kind(lights)
    normals = None if kind == "ambient" else meshes.verts_normals_packed()
    params = _params(len(meshes), lights, cameras, materials, kind, verts.device, batched_material_colors=True)
    return _Gouraud.apply(verts, normals, verts_colors, fragments.bary_coords, params,
                          meshes.mesh_to_verts_packed_first_idx(), meshes.num_verts_per_mesh(), faces,
                          fragments.pix_to_face, kind)
