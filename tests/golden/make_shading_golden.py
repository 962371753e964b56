"""Writes tests/golden/reference_golden_shading.npz: the outputs and gradients of the reference's own phong_shading,
_phong_shading_with_pixels and flat_shading (pytorch3d/renderer/mesh/shading.py, with renderer/lighting.py,
renderer/materials.py and renderer/utils.py) on the seeded scenes of tests/test_shading.py, and the reference's
Meshes.verts_normals_packed() (structures/meshes.py) of a seeded torus batch, in the record format of
make_reference_golden.py (tests/helpers.py: reference_record).

The reference modules are pure torch.  They are imported on the CPU with stand-ins for what they import:
pytorch3d._C (empty: on the CPU interpolate_face_attributes takes the reference's own python path),
pytorch3d.common.datatypes and a TexturesVertex placeholder.  Every input -- texels, barycentrics, vertices, vertex and
face normals, and every light, material and camera tensor -- requires grad; each output and each gradient the reference
produces is stored as its own case, "shading/<mode>-<light>-<batch>-<shininess>/<field>".

    python tests/golden/make_shading_golden.py [OUT_DIR]
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

SAMPLE_ROWS = 64
LEAD = {"colors": 4, "pixel_coords": 4, "grad_texels": 4, "grad_bary": 4}  # everything else: one row per vertex / face


def put(store, case, array, lead):
    for field, v in reference_record([array], lead, SAMPLE_ROWS)[0].items():
        store["%s/0/%s" % (case, field)] = v


def _load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod
    spec.loader.exec_module(mod)
    return mod


def reference_modules():
    """(shading, lighting, materials, meshes): the reference's modules with stand-ins for what they import."""
    ref = os.path.join(build_ref.REF, "pytorch3d")
    names = ("pytorch3d", "pytorch3d.common", "pytorch3d.common.datatypes", "pytorch3d.ops", "pytorch3d.renderer",
             "pytorch3d.renderer.mesh", "pytorch3d.renderer.mesh.textures", "pytorch3d.structures",
             "pytorch3d.ops.interp_face_attrs", "pytorch3d.renderer.utils", "pytorch3d.renderer.lighting",
             "pytorch3d.renderer.materials", "pytorch3d.renderer.mesh.shading", "pytorch3d.structures.utils",
             "pytorch3d.structures.meshes")
    saved = {n: sys.modules.get(n) for n in names}
    stubs = {n: types.ModuleType(n) for n in names[:8]}
    for m in stubs.values():
        m.__path__ = []
    stubs["pytorch3d"]._C = types.SimpleNamespace()
    dt = stubs["pytorch3d.common.datatypes"]
    dt.Device = Union[str, torch.device]
    dt.make_device = lambda d: torch.device(d) if isinstance(d, str) else d
    stubs["pytorch3d.renderer.mesh.textures"].TexturesVertex = type("TexturesVertex", (), {})
    sys.modules.update(stubs)
    try:
        interp = _load("pytorch3d.ops.interp_face_attrs", os.path.join(ref, "ops", "interp_face_attrs.py"))
        stubs["pytorch3d.ops"].interpolate_face_attributes = interp.interpolate_face_attributes
        _load("pytorch3d.renderer.utils", os.path.join(ref, "renderer", "utils.py"))
        lighting = _load("pytorch3d.renderer.lighting", os.path.join(ref, "renderer", "lighting.py"))
        materials = _load("pytorch3d.renderer.materials", os.path.join(ref, "renderer", "materials.py"))
        shading = _load("pytorch3d.renderer.mesh.shading", os.path.join(ref, "renderer", "mesh", "shading.py"))
        _load("pytorch3d.structures.utils", os.path.join(ref, "structures", "utils.py"))
        meshes = _load("pytorch3d.structures.meshes", os.path.join(ref, "structures", "meshes.py"))
    finally:
        for n, m in saved.items():
            if m is None:
                sys.modules.pop(n, None)
            else:
                sys.modules[n] = m
    return shading, lighting, materials, meshes


def run_reference(mods, ts, args):
    """[(field, tensor)] of one case, in the order of tests/test_shading.py: with_grads."""
    shading, lighting, materials_mod, _ = mods
    mode, kind, batch, shininess = args
    s = ts.shading_scene(*ts.SCENE, batch, shininess)
    leaves = {k: s[k].clone().requires_grad_(True) for k in ts.LEAVES}
    meshes, fragments, _, cameras, _ = ts.scene_objects(s, kind, leaves)
    if kind == "point":
        lights = lighting.PointLights(ambient_color=leaves["light_ambient"], diffuse_color=leaves["light_diffuse"],
                                      specular_color=leaves["light_specular"], location=leaves["light_where"])
    elif kind == "directional":
        lights = lighting.DirectionalLights(ambient_color=leaves["light_ambient"],
                                            diffuse_color=leaves["light_diffuse"],
                                            specular_color=leaves["light_specular"], direction=leaves["light_where"])
    else:
        lights = lighting.AmbientLights(ambient_color=leaves["light_ambient"])
    materials = materials_mod.Materials(ambient_color=leaves["material_ambient"],
                                        diffuse_color=leaves["material_diffuse"],
                                        specular_color=leaves["material_specular"], shininess=leaves["shininess"])
    fn = {"phong": shading.phong_shading, "pixels": shading._phong_shading_with_pixels,
          "flat": shading.flat_shading}[mode]
    out = fn(meshes, fragments, lights, cameras, materials, leaves["texels"])
    outs = list(out) if isinstance(out, tuple) else [out]
    loss = (outs[0] * s["grad_colors"]).sum()
    if len(outs) > 1:
        loss = loss + (outs[1] * s["grad_positions"]).sum()
    loss.backward()
    named = [("colors", outs[0].detach())] + ([("pixel_coords", outs[1].detach())] if len(outs) > 1 else [])
    return named + [("grad_" + k, leaves[k].grad) for k in ts.LEAVES if leaves[k].grad is not None]


def main():
    import test_shading as ts
    from pytorch3d_b200 import synthetic
    out_dir = sys.argv[1] if len(sys.argv) > 1 else HERE
    torch.set_grad_enabled(True)
    mods = reference_modules()
    store = {}
    for args in ts.SHADING_CASES:
        for field, t in run_reference(mods, ts, args):
            put(store, ts.shading_case(args) + "/" + field, t, LEAD.get(field, 1))
    m = synthetic.torus_batch(2, 7, 9, seed=3)
    nv = m.verts_packed().shape[0] // 2
    nf = m.faces_packed().shape[0] // 2
    ref_mesh = mods[3].Meshes(verts=[m.verts_packed()[:nv], m.verts_packed()[nv:]],
                              faces=[m.faces_packed()[:nf], m.faces_packed()[nf:] - nv])
    put(store, "shading/torus_verts_normals", ref_mesh.verts_normals_packed(), 1)
    out = os.path.join(out_dir, "reference_golden_shading.npz")
    np.savez_compressed(out, **store)
    print("wrote %s: %d arrays, %d bytes" % (out, len(store), os.path.getsize(out)))
    assert os.path.getsize(out) < 1 << 20, "%s is larger than 1 MB: store fewer rows" % out


if __name__ == "__main__":
    main()
