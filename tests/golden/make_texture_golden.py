"""Writes tests/golden/reference_golden_textures.npz: the texels and gradients of the reference's own
TexturesUV.sample_textures (pytorch3d/renderer/mesh/textures.py, with structures/utils.py, renderer/mesh/utils.py and
ops/interp_face_attrs.py) on the seeded scenes of tests/test_textures.py, in the record format of
make_reference_golden.py (tests/helpers.py: reference_record).

The reference modules are pure torch.  They are imported on the CPU with stand-ins for what they import: empty
pytorch3d, pytorch3d.ops and pytorch3d.structures packages and an empty pytorch3d._C (so interpolate_face_attributes
takes the reference's own python path).  The maps, the vertex UVs and the barycentrics require grad; each output and
each gradient is stored as its own case, "textures/<mode>-<padding>-<align>-C<channels>-<H_in>x<W_in>/<field>".

    python tests/golden/make_texture_golden.py [OUT_DIR]
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
LEAD = {"texels": 4, "grad_bary": 4}  # the map and vertex-UV gradients: one row per image


def put(store, case, array, lead):
    for field, v in reference_record([array], lead, SAMPLE_ROWS)[0].items():
        store["%s/0/%s" % (case, field)] = v


def _load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod
    spec.loader.exec_module(mod)
    return mod


def reference_textures():
    """The reference's textures module with stand-ins for what it imports."""
    ref = os.path.join(build_ref.REF, "pytorch3d")
    stub_names = ("pytorch3d", "pytorch3d.ops", "pytorch3d.structures", "pytorch3d.renderer", "pytorch3d.renderer.mesh")
    names = stub_names + ("pytorch3d.ops.interp_face_attrs", "pytorch3d.structures.utils", "pytorch3d.renderer.mesh.utils",
                          "pytorch3d.renderer.mesh.textures")
    saved = {n: sys.modules.get(n) for n in names}
    stubs = {n: types.ModuleType(n) for n in stub_names}
    for m in stubs.values():
        m.__path__ = []
    stubs["pytorch3d"]._C = types.SimpleNamespace()
    sys.modules.update(stubs)
    try:
        interp = _load("pytorch3d.ops.interp_face_attrs", os.path.join(ref, "ops", "interp_face_attrs.py"))
        stubs["pytorch3d.ops"].interpolate_face_attributes = interp.interpolate_face_attributes
        _load("pytorch3d.structures.utils", os.path.join(ref, "structures", "utils.py"))
        _load("pytorch3d.renderer.mesh.utils", os.path.join(ref, "renderer", "mesh", "utils.py"))
        textures = _load("pytorch3d.renderer.mesh.textures", os.path.join(ref, "renderer", "mesh", "textures.py"))
    finally:
        for n, m in saved.items():
            if m is None:
                sys.modules.pop(n, None)
            else:
                sys.modules[n] = m
    return textures


def run_reference(textures, tt, args):
    """[(field, tensor)] of one case, in the order of tests/test_textures.py: with_grads."""
    mode, pad, align, _, _ = args
    s = tt.case_scene(args)
    maps = s["maps"].clone().requires_grad_(True)
    verts_uvs = s["verts_uvs"].clone().requires_grad_(True)
    bary = s["bary"].clone().requires_grad_(True)
    tex = textures.TexturesUV(maps=maps, faces_uvs=s["faces_uvs"], verts_uvs=verts_uvs, padding_mode=pad,
                              align_corners=align, sampling_mode=mode)
    frags = types.SimpleNamespace(pix_to_face=s["pix_to_face"], bary_coords=bary)
    texels = tex.sample_textures(frags)
    (texels * s["grad_texels"]).sum().backward()
    grads = [torch.zeros_like(t) if t.grad is None else t.grad for t in (maps, verts_uvs, bary)]
    return list(zip(tt.FIELDS, [texels.detach()] + grads))


def main():
    import test_textures as tt
    out_dir = sys.argv[1] if len(sys.argv) > 1 else HERE
    torch.set_grad_enabled(True)
    textures = reference_textures()
    store = {}
    for args in tt.TEXTURE_CASES:
        for field, t in run_reference(textures, tt, args):
            put(store, tt.texture_case(args) + "/" + field, t, LEAD.get(field, 1))
    out = os.path.join(out_dir, "reference_golden_textures.npz")
    np.savez_compressed(out, **store)
    print("wrote %s: %d arrays, %d bytes" % (out, len(store), os.path.getsize(out)))
    assert os.path.getsize(out) < 1 << 20, "%s is larger than 1 MB: store fewer rows" % out


if __name__ == "__main__":
    main()
