"""Texture atlas sampling, same results as the reference's `TexturesAtlas.sample_textures`
(pytorch3d/renderer/mesh/textures.py).

Each face has an R x R patch of texels.  A slot reads the cell of its face's patch that its barycentrics (b0, b1) fall
in, with the reference's truncation, clamp to R - 1 and flip across the diagonal, and multiplies it by
float(pix_to_face >= 0).  The reference does this with a dozen elementwise torch ops and an advanced-indexing gather;
here the forward is one kernel and the backward a key pass, a stable radix sort and a segmented sum (DESIGN.md section
15), so the atlas gradient is deterministic, as the reference's is.  Neither synchronises the host.

As in the reference, the barycentrics get no gradient, and background slots read `atlas[F-1, 0, 0]` times 0 (so -0.0
where that value is negative), whose gradient is 0 unless the upstream gradient is not finite.  One divergence: a cell
the reference cannot index (blurred barycentrics outside [-1, 1]; it raises) gives texel 0 and no gradient.  The texels
come back contiguous, (N,H,W,K,C).
"""
import torch

from . import _C

__all__ = ["sample_textures_atlas", "sample_textures"]


class _SampleAtlas(torch.autograd.Function):
    @staticmethod
    def forward(ctx, atlas, bary, pix_to_face):
        texels = _C.texture_atlas_forward(pix_to_face, bary, atlas)
        ctx.save_for_backward(atlas, bary, pix_to_face)
        return texels

    @staticmethod
    def backward(ctx, grad_texels):
        atlas, bary, pix_to_face = ctx.saved_tensors
        grad_atlas = None
        if ctx.needs_input_grad[0]:
            grad_atlas = _C.texture_atlas_backward(grad_texels.contiguous(), pix_to_face, bary, atlas)
        return grad_atlas, None, None


def sample_textures_atlas(fragments, atlas_packed) -> torch.Tensor:
    """Sample the packed atlas (F, R, R, C) at the rasterized slots.

    fragments: `pix_to_face` (N,H,W,K) int64 into the packed faces and `bary_coords` (N,H,W,K,3) float32.  Returns
    texels (N,H,W,K,C).  Gradients reach the atlas only."""
    return _SampleAtlas.apply(atlas_packed, fragments.bary_coords, fragments.pix_to_face)


def sample_textures(textures, fragments, **kwargs) -> torch.Tensor:
    """Drop-in for `TexturesAtlas.sample_textures(fragments)`.  `textures` needs `atlas_packed()`, which is called once,
    as the reference calls it, so autograd takes the gradient back to the list or padded atlas the texture was built
    from."""
    return sample_textures_atlas(fragments, textures.atlas_packed())
