"""UV texture sampling, same results as the reference's `TexturesUV.sample_textures`
(pytorch3d/renderer/mesh/textures.py) for a texture with one map per mesh.

Each slot's UV is interpolated from its face's corner UVs, mapped to grid_sample's coordinates with the y flip, and the
map of the slot's image is sampled there with `F.grid_sample`'s rules ("bilinear" or "nearest"; "zeros", "border" or
"reflection" padding; either `align_corners`).  The reference expands the maps K times into an (N*K, C, H_in, W_in) copy
for this; here the forward is one kernel that reads the maps in place and the backward one kernel (DESIGN.md
section 13).  Neither synchronises the host.

As in the reference, background slots (pix_to_face < 0) sample UV (0, 0), so they get a real texel (`maps[n, H_in-1, 0]`
with align_corners=True) and their upstream gradient reaches that texel.  The texels come back contiguous, (N,H,W,K,C);
the reference returns a permuted view with the same values.
"""
import torch

from . import _C

__all__ = ["sample_textures_uv", "sample_textures"]


class _SampleUV(torch.autograd.Function):
    @staticmethod
    def forward(ctx, maps, bary, face_uvs, pix_to_face, sampling_mode, padding_mode, align_corners):
        texels = _C.texture_uv_forward(pix_to_face, bary, face_uvs, maps, sampling_mode, padding_mode, align_corners)
        ctx.save_for_backward(maps, bary, face_uvs, pix_to_face)
        ctx.args = (sampling_mode, padding_mode, align_corners)
        return texels

    @staticmethod
    def backward(ctx, grad_texels):
        maps, bary, face_uvs, pix_to_face = ctx.saved_tensors
        grads = _C.texture_uv_backward(grad_texels.contiguous(), pix_to_face, bary, face_uvs, maps, *ctx.args,
                                       needs_input_grad=ctx.needs_input_grad[:3])
        return grads + (None, None, None, None)


def sample_textures_uv(fragments, maps, face_uvs, *, sampling_mode="bilinear", padding_mode="border",
                       align_corners=True) -> torch.Tensor:
    """Sample `maps` (N, H_in, W_in, C), one map per image, at the UVs of the rasterized slots.

    fragments: `pix_to_face` (N,H,W,K) int64 and `bary_coords` (N,H,W,K,3) float32; face_uvs (F,3,2) float32, the UVs
    of each packed face's corners.  Returns texels (N,H,W,K,C).  Gradients reach the maps, the barycentric coordinates
    and the face UVs."""
    return _SampleUV.apply(maps, fragments.bary_coords, face_uvs, fragments.pix_to_face, sampling_mode, padding_mode,
                           align_corners)


def sample_textures(textures, fragments, **kwargs) -> torch.Tensor:
    """Drop-in for `TexturesUV.sample_textures(fragments)` of a texture without `maps_ids`.  `textures` needs
    `verts_uvs_list()`, `faces_uvs_list()`, `maps_padded()`, `isempty()` and the attributes `sampling_mode`,
    `padding_mode` and `align_corners`; the face UVs are formed as the reference forms them, so autograd takes their
    gradient back to the vertex UVs."""
    if textures.isempty():
        face_uvs = torch.zeros((textures._N, 3, 2), dtype=torch.float32, device=textures.device)
    else:
        face_uvs = torch.cat([v[f] for v, f in zip(textures.verts_uvs_list(), textures.faces_uvs_list())])
    return sample_textures_uv(fragments, textures.maps_padded(), face_uvs, sampling_mode=textures.sampling_mode,
                              padding_mode=textures.padding_mode, align_corners=textures.align_corners)
