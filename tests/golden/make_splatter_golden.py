"""Writes tests/golden/reference_golden_splatter.npz: the outputs of the reference's own SplatterBlender
(pytorch3d/renderer/splatter_blend.py) on the seeded scenes of tests/test_splatter_blend.py, in the record format of
make_reference_golden.py (tests/helpers.py: reference_record).

The reference module is pure torch.  It is imported on the CPU with stand-ins for the modules it imports
(pytorch3d.common.datatypes, pytorch3d.renderer.BlendParams, pytorch3d.renderer.cameras and
pytorch3d.renderer.blending._get_background_color, the latter two from the reference's own blending.py) and run with
an identity camera, so its positions are the scene's screen positions.  For every scene it stores the RGBA output and
the gradients of the colours and positions under the scene's seeded upstream gradient.

    python tests/golden/make_splatter_golden.py [OUT_DIR]
"""
import importlib.util
import os
import sys
import types
from typing import Union

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.dirname(HERE)]

from helpers import reference_record  # noqa: E402
from oracle import build_ref  # noqa: E402

SAMPLE_ROWS = 1024


def put(store, case, arrays):
    for i, rec in enumerate(reference_record(arrays, 3, SAMPLE_ROWS)):
        for field, v in rec.items():
            store["%s/%d/%s" % (case, i, field)] = v


def _load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod
    spec.loader.exec_module(mod)
    return mod


def reference_splatter_module():
    """The reference's splatter_blend.py with stand-ins for the PyTorch3D modules it imports."""
    renderer = os.path.join(build_ref.REF, "pytorch3d", "renderer")
    names = ("pytorch3d", "pytorch3d.common", "pytorch3d.common.datatypes", "pytorch3d.renderer",
             "pytorch3d.renderer.cameras", "pytorch3d.renderer.blending", "pytorch3d.renderer.splatter_blend")
    saved = {n: sys.modules.get(n) for n in names}
    stubs = {n: types.ModuleType(n) for n in names[:5]}
    for m in stubs.values():
        m.__path__ = []
    stubs["pytorch3d"]._C = types.SimpleNamespace()
    stubs["pytorch3d.common.datatypes"].Device = Union[str, torch.device]
    stubs["pytorch3d.renderer.cameras"].FoVPerspectiveCameras = object
    sys.modules.update(stubs)
    try:
        blending = _load("pytorch3d.renderer.blending", os.path.join(renderer, "blending.py"))
        stubs["pytorch3d.renderer"].BlendParams = blending.BlendParams
        splatter = _load("pytorch3d.renderer.splatter_blend", os.path.join(renderer, "splatter_blend.py"))
    finally:
        for n, m in saved.items():
            if m is None:
                sys.modules.pop(n, None)
            else:
                sys.modules[n] = m
    return splatter, blending.BlendParams


class IdentityCamera:
    def transform_points_screen(self, points, image_size, with_xyflip=True):
        return points * 1.0


def run_reference(sb, BlendParams, colors, coords, mask, grad, sigma, background):
    N, H, W, K, _ = colors.shape
    c, x = colors.clone().requires_grad_(True), coords.clone().requires_grad_(True)
    out = sb.SplatterBlender((N, H, W, K), "cpu")(c, x, IdentityCamera(), mask,
                                                   BlendParams(sigma=sigma, background_color=background))
    out.backward(grad)
    return [out.detach(), c.grad, x.grad]


def main():
    import test_splatter_blend as ts
    out_dir = sys.argv[1] if len(sys.argv) > 1 else HERE
    torch.set_grad_enabled(True)
    sb, BlendParams = reference_splatter_module()
    store = {}
    for args in ts.SPLATTER_CASES:
        colors, coords, mask, grad = ts.splatter_scene(*args)
        put(store, ts.splatter_case(args), run_reference(sb, BlendParams, colors, coords, mask, grad, args[4],
                                                         ts.BACKGROUND))
    colors, coords, mask, grad = ts.quirk_scene()
    put(store, "splatter/quirk", run_reference(sb, BlendParams, colors, coords, mask, grad, 0.5, ts.BACKGROUND))
    out = os.path.join(out_dir, "reference_golden_splatter.npz")
    np.savez_compressed(out, **store)
    print("wrote %s: %d arrays, %d bytes" % (out, len(store), os.path.getsize(out)))
    assert os.path.getsize(out) < 1 << 20, "%s is larger than 1 MB: store fewer rows" % out


if __name__ == "__main__":
    main()
