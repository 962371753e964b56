"""Splatter blending, same API as the reference's pytorch3d/renderer/splatter_blend.py: `SplatterBlender`, the blend of
`SplatterPhongShader` (Cole et al., "Differentiable Surface Rendering via Non-Differentiable Sampling").

Each pixel's K layers splat their colour onto the 3 x 3 neighbourhood with a Gaussian of the distance between the
layer's projected position and the pixel centre.  The splats a pixel receives are sorted into three occlusion layers
by comparing depths with the neighbour, normalised per layer and composed over the background.  Gradients reach the
projected positions -- and through them the vertices -- even though the rasterizer itself is not differentiable.

The reference builds several (N,H,W,K,9,5) tensors per call (3 GB each at 8 x 512 x 512, K = 8); here the forward is one
kernel and the backward two (DESIGN.md section 11).  Neither synchronises the host.
"""
from typing import Tuple

import torch

from . import _C
from .blending import BlendParams, _as_device_float

__all__ = ["SplatterBlender", "splatter_blend"]


class _SplatterBlend(torch.autograd.Function):
    @staticmethod
    def forward(ctx, colors, pixel_coords_screen, background_mask, sigma, background):
        out = _C.splatter_blend(colors, pixel_coords_screen, background_mask, sigma, background)
        ctx.save_for_backward(colors, pixel_coords_screen, background_mask)
        ctx.args = (sigma, background)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        colors, pixel_coords_screen, background_mask = ctx.saved_tensors
        grad_colors, grad_coords = _C.splatter_blend_backward(grad_out, colors, pixel_coords_screen, background_mask,
                                                              *ctx.args)
        return grad_colors, grad_coords, None, None, None


def splatter_blend(colors: torch.Tensor, pixel_coords_screen: torch.Tensor, background_mask: torch.Tensor,
                   blend_params: BlendParams) -> torch.Tensor:
    """The splatter blend of already projected positions: what `SplatterBlender.forward` computes after it has called
    `cameras.transform_points_screen`.

    colors (N,H,W,K,3) and pixel_coords_screen (N,H,W,K,3) float32 CUDA tensors (x, y in pixels, without the xy flip,
    z the depth); background_mask (N,H,W,K) bool, True in slots without a face.  From `blend_params` it uses sigma (the
    splat's standard deviation in pixels) and background_color.  Returns (N,H,W,4) RGBA.  Gradients flow to `colors`
    and to the x, y of `pixel_coords_screen`; the background colour is a constant, so a tensor that requires grad
    raises ValueError.
    """
    sigma = float(blend_params.sigma)
    if sigma <= 0.0:
        raise ValueError("Only positive standard deviations make sense.")
    background = blend_params.background_color
    if torch.is_tensor(background) and background.requires_grad:
        raise ValueError("splatter_blend: background_color must not require grad (gradients flow to colors and "
                         "pixel_coords_screen only)")
    return _SplatterBlend.apply(colors, pixel_coords_screen, background_mask, sigma,
                                _as_device_float(background, colors.device))


class SplatterBlender(torch.nn.Module):
    """Drop-in for the reference's `SplatterBlender`.  `input_shape` (N, H, W, K) is accepted for compatibility; nothing
    depends on it, so one blender serves inputs of any shape."""

    def __init__(self, input_shape: Tuple[int, int, int, int], device=None):
        super().__init__()
        self.input_shape = tuple(input_shape)
        self.device = device

    def to(self, device):
        self.device = device
        return super().to(device)

    def forward(self, colors: torch.Tensor, pixel_coords_cameras: torch.Tensor, cameras, background_mask: torch.Tensor,
                blend_params: BlendParams) -> torch.Tensor:
        """colors, pixel_coords_cameras (N,H,W,K,3) (positions in the camera frame, interpolated from the vertices with
        the barycentrics so that gradients reach the vertices); `cameras` anything with PyTorch3D's
        `transform_points_screen`; background_mask (N,H,W,K) bool.  Returns (N,H,W,4) RGBA, alpha 0 in the
        background."""
        N, H, W, K, _ = colors.shape
        pixel_coords_screen = cameras.transform_points_screen(
            pixel_coords_cameras.view([N, -1, 3]), image_size=(H, W), with_xyflip=False
        ).reshape(pixel_coords_cameras.shape)
        return splatter_blend(colors, pixel_coords_screen, background_mask, blend_params)
