"""Mesh blending (SURVEY.md 8f-5), same API as the reference's pytorch3d/renderer/blending.py: `BlendParams`,
`hard_rgb_blend`, `sigmoid_alpha_blend` and `softmax_rgb_blend`; and the depth blends of the reference's
SoftDepthShader and HardDepthShader (pytorch3d/renderer/mesh/shader.py): `soft_depth` and `hard_depth`.

`sigmoid_alpha_blend` runs the drop-in `_C.sigmoid_alpha_blend[_backward]` kernels (bit-identical to the reference's);
`softmax_rgb_blend` runs one fused kernel per direction instead of the reference's chain of some twenty torch kernels;
`hard_rgb_blend` needs no kernel of its own; `soft_depth` and `hard_depth` run one fused kernel per direction (DESIGN.md
section 19).  None of them synchronises the host.
"""
from typing import NamedTuple, Sequence, Union

import torch

from . import _C


class BlendParams(NamedTuple):
    """sigma: width of the sigmoid of the 2D distance (sharpness of the edges); gamma: scale of the exponential of the
    inverse depth (higher => faces are more transparent); background_color: RGB as a tuple or a tensor of three
    floats.  Same fields and defaults as the reference."""

    sigma: float = 1e-4
    gamma: float = 1e-4
    background_color: Union[torch.Tensor, Sequence[float]] = (1.0, 1.0, 1.0)


def _background_tensor(background_color, like: torch.Tensor) -> torch.Tensor:
    """The background colour as a (3,) tensor on `like`'s device.  A sequence of numbers is written on the device by
    fill kernels: a host-to-device copy from pageable memory would synchronise the host."""
    if torch.is_tensor(background_color):
        return background_color.to(like.device)
    return torch.stack([like.new_full((), float(v), dtype=torch.float32) for v in background_color])


def hard_rgb_blend(colors: torch.Tensor, fragments, blend_params: BlendParams) -> torch.Tensor:
    """RGB of the closest face (slot 0), the background colour where no face covers the pixel; alpha 1 on covered
    pixels, 0 elsewhere.  colors (N,H,W,K,3) -> (N,H,W,4).  Same values and gradients as the reference's
    `masked_scatter` form, without counting the background pixels on the host."""
    is_background = fragments.pix_to_face[..., 0] < 0  # (N, H, W)
    background_color = _background_tensor(blend_params.background_color, fragments.pix_to_face)
    pixel_colors = torch.where(is_background[..., None], background_color.to(colors.dtype), colors[..., 0, :])
    alpha = (~is_background).type_as(pixel_colors)[..., None]
    return torch.cat([pixel_colors, alpha], dim=-1)


class _SigmoidAlphaBlend(torch.autograd.Function):
    @staticmethod
    def forward(ctx, dists, pix_to_face, sigma):
        alphas = _C.sigmoid_alpha_blend(dists, pix_to_face, sigma)
        ctx.save_for_backward(dists, pix_to_face, alphas)
        ctx.sigma = sigma
        return alphas

    @staticmethod
    def backward(ctx, grad_alphas):
        dists, pix_to_face, alphas = ctx.saved_tensors
        grad_dists = _C.sigmoid_alpha_blend_backward(grad_alphas, alphas, dists, pix_to_face, ctx.sigma)
        return grad_dists, None, None


_sigmoid_alpha = _SigmoidAlphaBlend.apply


def sigmoid_alpha_blend(colors, fragments, blend_params: BlendParams) -> torch.Tensor:
    """Silhouette blending: RGB of the closest face, alpha = 1 - prod_k (1 - sigmoid(-dists_k / sigma)) over the valid
    slots (Liu et al., Soft Rasterizer, ICCV 2019).  colors (N,H,W,K,3) -> (N,H,W,4); gradients flow to
    `fragments.dists` through the alpha channel and to `colors` through the RGB channels."""
    N, H, W, K = fragments.pix_to_face.shape
    pixel_colors = torch.ones((N, H, W, 4), dtype=colors.dtype, device=colors.device)
    pixel_colors[..., :3] = colors[..., 0, :]
    alpha = _sigmoid_alpha(fragments.dists, fragments.pix_to_face, blend_params.sigma)
    pixel_colors[..., 3] = alpha
    return pixel_colors


class _SoftmaxRGBBlend(torch.autograd.Function):
    @staticmethod
    def forward(ctx, colors, zbuf, dists, pix_to_face, sigma, gamma, background, znear, zfar):
        out = _C.softmax_rgb_blend(colors, pix_to_face, zbuf, dists, sigma, gamma, background, znear, zfar)
        ctx.save_for_backward(colors, zbuf, dists, pix_to_face)
        ctx.args = (sigma, gamma, background, znear, zfar)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        colors, zbuf, dists, pix_to_face = ctx.saved_tensors
        grad_colors, grad_dists, grad_zbuf = _C.softmax_rgb_blend_backward(grad_out, colors, pix_to_face, zbuf, dists,
                                                                           *ctx.args)
        return grad_colors, grad_zbuf, grad_dists, None, None, None, None, None, None


def _as_device_float(x, device):
    return x.to(device=device, dtype=torch.float32) if torch.is_tensor(x) else x


def softmax_rgb_blend(colors: torch.Tensor, fragments, blend_params: BlendParams,
                      znear: Union[float, torch.Tensor] = 1.0, zfar: Union[float, torch.Tensor] = 100) -> torch.Tensor:
    """RGB blended by the softmax of the inverse depth weighted with the sigmoid of the 2D distance, alpha from the
    distances alone (Liu et al., Soft Rasterizer, ICCV 2019) -- the reference's `softmax_rgb_blend`, one fused kernel
    per direction.

    colors (N,H,W,K,3); `fragments` with pix_to_face, zbuf and dists (N,H,W,K); znear / zfar numbers or (N,) tensors.
    Returns (N,H,W,4).  Gradients flow to `colors`, `fragments.dists` and `fragments.zbuf`.  The background colour,
    znear and zfar are constants here: a tensor among them that requires grad raises ValueError.
    """
    for name, x in (("background_color", blend_params.background_color), ("znear", znear), ("zfar", zfar)):
        if torch.is_tensor(x) and x.requires_grad:
            raise ValueError("softmax_rgb_blend: %s must not require grad (gradients flow to colors, dists and zbuf "
                             "only)" % name)
    device = fragments.pix_to_face.device
    background = _as_device_float(blend_params.background_color, device)
    return _SoftmaxRGBBlend.apply(colors, fragments.zbuf, fragments.dists, fragments.pix_to_face,
                                  float(blend_params.sigma), float(blend_params.gamma), background,
                                  _as_device_float(znear, device), _as_device_float(zfar, device))


def _check_zfar(zfar, fn):
    if torch.is_tensor(zfar) and zfar.requires_grad:
        raise ValueError("%s: zfar must not require grad (gradients flow to zbuf and dists only)" % fn)


class _SoftDepth(torch.autograd.Function):
    @staticmethod
    def forward(ctx, zbuf, dists, pix_to_face, sigma, zfar):
        out = _C.soft_depth_blend(pix_to_face, zbuf, dists, sigma, zfar)
        ctx.save_for_backward(zbuf, dists, pix_to_face)
        ctx.args = (sigma, zfar)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        zbuf, dists, pix_to_face = ctx.saved_tensors
        grad_zbuf, grad_dists = _C.soft_depth_blend_backward(grad_out, pix_to_face, zbuf, dists, *ctx.args)
        return grad_zbuf, grad_dists, None, None, None


def soft_depth(fragments, sigma: float, zfar: Union[float, torch.Tensor]) -> torch.Tensor:
    """Depth blended over the K faces of each pixel and a background at `zfar` -- the reference's SoftDepthShader.
    Each face's coverage is sigmoid(-dists / sigma) (0 for empty slots); the faces are taken nearest first until their
    cumulative coverage reaches 1, and the background gets what is left.

    `fragments` with pix_to_face, zbuf and dists (N,H,W,K), 1 <= K <= 150; zfar a number or a 1-element float32 tensor
    on the same device (read on the device).  Returns (N,H,W,1).  Gradients flow to `fragments.zbuf` and
    `fragments.dists`; a zfar that requires grad raises ValueError.
    """
    _check_zfar(zfar, "soft_depth")
    return _SoftDepth.apply(fragments.zbuf, fragments.dists, fragments.pix_to_face, float(sigma), zfar)


class _HardDepth(torch.autograd.Function):
    @staticmethod
    def forward(ctx, zbuf, pix_to_face, zfar):
        out = _C.hard_depth(pix_to_face, zbuf, zfar)
        ctx.save_for_backward(pix_to_face)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        pix_to_face, = ctx.saved_tensors
        return _C.hard_depth_backward(grad_out, pix_to_face), None, None


def hard_depth(fragments, zfar: Union[float, torch.Tensor]) -> torch.Tensor:
    """Depth of the closest face, `zfar` where no face covers the pixel -- the reference's HardDepthShader.
    `fragments` with pix_to_face and zbuf (N,H,W,K), 1 <= K <= 150; zfar as for `soft_depth`.  Returns (N,H,W,1);
    the gradient flows to slot 0 of `fragments.zbuf` on covered pixels."""
    _check_zfar(zfar, "hard_depth")
    return _HardDepth.apply(fragments.zbuf, fragments.pix_to_face, zfar)
