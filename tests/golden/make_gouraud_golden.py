"""Writes tests/golden/reference_golden_gouraud.npz: the colours and gradients of the reference's own gouraud_shading
(pytorch3d/renderer/mesh/shading.py, with renderer/lighting.py, renderer/materials.py, renderer/utils.py,
renderer/cameras.py with transforms/, the real TexturesVertex of renderer/mesh/textures.py and structures/meshes.py) on
the seeded scenes of tests/test_gouraud.py (golden_scene), in the record format of make_reference_golden.py
(tests/helpers.py: reference_record).

The reference modules are pure torch.  They are imported on the CPU with stand-ins only for the packages around them
(pytorch3d._C is empty: on the CPU interpolate_face_attributes takes the reference's own python path); pytorch3d.common
and pytorch3d.transforms are the reference's own packages.  The cameras are real FoVPerspectiveCameras whose R and T
require grad, like every vertex, vertex colour, barycentric, light and material tensor.  Each output and gradient is its
own case, "gouraud/<light>-<batch>-<shininess>-<meshes>/<field>".  Two more fields per case record the camera centres:
`camera_center_mesh`, what get_camera_center() returns for the N cameras, and `camera_center_vertex` with its gradient
`grad_camera_center_vertex`, what gouraud_shading forms from the cameras gathered per vertex (len(meshes) > 1) or the
single camera.

    python tests/golden/make_gouraud_golden.py [OUT_DIR]
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

SAMPLE_ROWS = 64
LEAD = {"colors": 4, "grad_bary": 4}  # everything else: one row per vertex / batch entry


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
    """The reference's modules, by short name, with stand-ins for the packages around them."""
    ref = os.path.join(build_ref.REF, "pytorch3d")
    stub_names = ("pytorch3d", "pytorch3d.ops", "pytorch3d.structures", "pytorch3d.renderer", "pytorch3d.renderer.mesh")
    saved = {n: m for n, m in sys.modules.items() if n == "pytorch3d" or n.startswith("pytorch3d.")}
    stubs = {n: types.ModuleType(n) for n in stub_names}
    for m in stubs.values():
        m.__path__ = []
    stubs["pytorch3d"].__path__ = [ref]  # pytorch3d.common and pytorch3d.transforms import as the reference's own
    stubs["pytorch3d"]._C = types.SimpleNamespace()
    sys.modules.update(stubs)
    mods = {}
    try:
        interp = _load("pytorch3d.ops.interp_face_attrs", os.path.join(ref, "ops", "interp_face_attrs.py"))
        stubs["pytorch3d.ops"].interpolate_face_attributes = interp.interpolate_face_attributes
        _load("pytorch3d.structures.utils", os.path.join(ref, "structures", "utils.py"))
        _load("pytorch3d.renderer.utils", os.path.join(ref, "renderer", "utils.py"))
        _load("pytorch3d.renderer.mesh.utils", os.path.join(ref, "renderer", "mesh", "utils.py"))
        for short, name, path in (
                ("textures", "pytorch3d.renderer.mesh.textures", ("renderer", "mesh", "textures.py")),
                ("lighting", "pytorch3d.renderer.lighting", ("renderer", "lighting.py")),
                ("materials", "pytorch3d.renderer.materials", ("renderer", "materials.py")),
                ("cameras", "pytorch3d.renderer.cameras", ("renderer", "cameras.py")),
                ("shading", "pytorch3d.renderer.mesh.shading", ("renderer", "mesh", "shading.py")),
                ("meshes", "pytorch3d.structures.meshes", ("structures", "meshes.py"))):
            mods[short] = _load(name, os.path.join(ref, *path))
    finally:
        for n in [n for n in sys.modules if n == "pytorch3d" or n.startswith("pytorch3d.")]:
            del sys.modules[n]
        sys.modules.update(saved)
    return types.SimpleNamespace(**mods)


def run_reference(ref, tg, args):
    """[(field, tensor)] of one case: the colours, the gradients of the leaves, and the camera centres."""
    kind, batch, shininess, meshes = args
    s = tg.golden_scene(*args)
    leaves = tg.golden_leaves(s)
    bounds = [sum(s["sizes"][:i]) for i in range(len(s["sizes"]) + 1)]
    split = list(zip(bounds[:-1], bounds[1:]))
    mesh = ref.meshes.Meshes(verts=[leaves["verts"][a:b] for a, b in split], faces=s["faces"],
                             textures=ref.textures.TexturesVertex(verts_features=[leaves["colors"][a:b]
                                                                                  for a, b in split]))
    fragments = types.SimpleNamespace(pix_to_face=s["pix_to_face"], bary_coords=leaves["bary"])
    if kind == "point":
        lights = ref.lighting.PointLights(ambient_color=leaves["light_ambient"], diffuse_color=leaves["light_diffuse"],
                                          specular_color=leaves["light_specular"], location=leaves["light_where"])
    elif kind == "directional":
        lights = ref.lighting.DirectionalLights(ambient_color=leaves["light_ambient"],
                                                diffuse_color=leaves["light_diffuse"],
                                                specular_color=leaves["light_specular"],
                                                direction=leaves["light_where"])
    else:
        lights = ref.lighting.AmbientLights(ambient_color=leaves["light_ambient"])
    materials = ref.materials.Materials(ambient_color=leaves["material_ambient"],
                                        diffuse_color=leaves["material_diffuse"],
                                        specular_color=leaves["material_specular"], shininess=leaves["shininess"])
    cameras = ref.cameras.FoVPerspectiveCameras(R=leaves["R"], T=leaves["T"])
    with torch.no_grad():
        center_mesh = cameras.get_camera_center().clone()
    seen = []
    cls = ref.cameras.FoVPerspectiveCameras
    original = cls.get_camera_center

    def recording(self, **kwargs):  # the centre gouraud_shading forms, kept with its gradient
        c = original(self, **kwargs)
        if c.requires_grad:
            c.retain_grad()
        seen.append(c)
        return c

    cls.get_camera_center = recording
    try:
        out = ref.shading.gouraud_shading(mesh, fragments, lights, cameras, materials)
    finally:
        cls.get_camera_center = original
    (out * s["grad_colors"]).sum().backward()
    named = [("colors", out.detach())]
    named += [("grad_" + k, leaves[k].grad) for k in tg.GOLDEN_LEAVES if leaves[k].grad is not None]
    assert len(seen) == 1
    named += [("camera_center_mesh", center_mesh), ("camera_center_vertex", seen[0].detach())]
    if seen[0].grad is not None:
        named.append(("grad_camera_center_vertex", seen[0].grad))
    return named


def main():
    import test_gouraud as tg
    out_dir = sys.argv[1] if len(sys.argv) > 1 else HERE
    torch.set_grad_enabled(True)
    ref = reference_modules()
    store = {}
    for args in tg.GOLDEN_CASES:
        for field, t in run_reference(ref, tg, args):
            put(store, tg.golden_case(args) + "/" + field, t, LEAD.get(field, 1))
    out = os.path.join(out_dir, "reference_golden_gouraud.npz")
    np.savez_compressed(out, **store)
    print("wrote %s: %d arrays, %d bytes" % (out, len(store), os.path.getsize(out)))
    assert os.path.getsize(out) < 1 << 20, "%s is larger than 1 MB: store fewer rows" % out


if __name__ == "__main__":
    main()
