"""Writes tests/golden/reference_golden_depth.npz: the outputs and autograd gradients of the reference's own
SoftDepthShader and HardDepthShader (pytorch3d/renderer/mesh/shader.py, with its renderer/blending.py) on the seeded
scenes of tests/test_depth_shading.py (DEPTH_CASES), in the record format of make_reference_golden.py
(tests/helpers.py: reference_record).

The shaders are pure torch.  They are imported on the CPU with stand-ins for the modules around them that their
forward passes do not use (lights, materials, meshes, the other shaders' helpers); pytorch3d.common is the reference's
own package.  zfar reaches each shader the way the scene says: as the camera's number, as the camera's 1-element
tensor, or as the forward's `zfar=` overriding the camera's.  Cases: "depth_soft/<case>" (depth, grad zbuf, grad dists)
and "depth_hard/<case>" (depth, grad zbuf).

    python tests/golden/make_depth_golden.py [OUT_DIR]
"""
import importlib.util
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.dirname(HERE)]

from helpers import reference_record  # noqa: E402
from oracle import build_ref  # noqa: E402

SAMPLE_ROWS = 256


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


def reference_shader_module():
    """The reference's pytorch3d/renderer/mesh/shader.py and the blending module it imports."""
    ref = os.path.join(build_ref.REF, "pytorch3d")
    saved = {n: m for n, m in sys.modules.items() if n == "pytorch3d" or n.startswith("pytorch3d.")}

    class _Stand:
        def __init__(self, *args, **kwargs):
            pass

    stub_names = ("pytorch3d", "pytorch3d.structures", "pytorch3d.structures.meshes", "pytorch3d.renderer",
                  "pytorch3d.renderer.lighting", "pytorch3d.renderer.materials", "pytorch3d.renderer.splatter_blend",
                  "pytorch3d.renderer.utils", "pytorch3d.renderer.mesh", "pytorch3d.renderer.mesh.rasterizer",
                  "pytorch3d.renderer.mesh.shading")
    stubs = {n: types.ModuleType(n) for n in stub_names}
    for m in stubs.values():
        m.__path__ = []
    stubs["pytorch3d"].__path__ = [ref]  # pytorch3d.common imports as the reference's own
    stubs["pytorch3d"]._C = types.SimpleNamespace()
    stubs["pytorch3d.structures.meshes"].Meshes = _Stand
    stubs["pytorch3d.renderer.lighting"].PointLights = _Stand
    stubs["pytorch3d.renderer.materials"].Materials = _Stand
    stubs["pytorch3d.renderer.splatter_blend"].SplatterBlender = _Stand
    stubs["pytorch3d.renderer.utils"].TensorProperties = _Stand
    stubs["pytorch3d.renderer.mesh.rasterizer"].Fragments = _Stand
    for n in ("_phong_shading_with_pixels", "flat_shading", "gouraud_shading", "phong_shading"):
        setattr(stubs["pytorch3d.renderer.mesh.shading"], n, None)
    sys.modules.update(stubs)
    try:
        _load("pytorch3d.renderer.blending", os.path.join(ref, "renderer", "blending.py"))
        shader = _load("pytorch3d.renderer.mesh.shader", os.path.join(ref, "renderer", "mesh", "shader.py"))
    finally:
        for n in [n for n in sys.modules if n == "pytorch3d" or n.startswith("pytorch3d.")]:
            del sys.modules[n]
        sys.modules.update(saved)
    return shader


def main():
    import test_depth_shading as td
    out_dir = sys.argv[1] if len(sys.argv) > 1 else HERE
    sh = reference_shader_module()
    torch.set_grad_enabled(True)
    store = {}
    for args in td.DEPTH_CASES:
        N, H, W, K, sigma, zk = args
        p2f, zbuf, dists, grad = td.depth_scene(N, H, W, K, sigma)
        camera_zfar, kwargs, _ = td.scene_zfar(zk)
        cameras = types.SimpleNamespace(zfar=camera_zfar)
        params = sh.BlendParams(sigma=sigma)
        soft = sh.SoftDepthShader(device="cpu", cameras=cameras, blend_params=params)
        got = td.soft_with_grads(lambda p, z, d: soft(td.frags(p, z, d), None, **kwargs), p2f, zbuf, dists, grad)
        put(store, "depth_soft/" + td.depth_case(args), got)
        hard = sh.HardDepthShader(device="cpu", cameras=cameras)
        got = td.hard_with_grads(lambda p, z: hard(td.frags(p, z, dists), None, **kwargs), p2f, zbuf, grad)
        put(store, "depth_hard/" + td.depth_case(args), got)
    out = os.path.join(out_dir, "reference_golden_depth.npz")
    np.savez_compressed(out, **store)
    print("wrote %s: %d arrays, %d bytes" % (out, len(store), os.path.getsize(out)))
    assert os.path.getsize(out) < 1 << 20, "%s is larger than 1 MB: store fewer rows" % out


if __name__ == "__main__":
    main()
