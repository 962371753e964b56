"""Writes tests/golden/reference_golden_atlas.npz: the texels and atlas gradients of the reference's own
TexturesAtlas.sample_textures (pytorch3d/renderer/mesh/textures.py, with structures/utils.py) on the seeded scenes of
tests/test_texture_atlas.py, in the record format of make_reference_golden.py (tests/helpers.py: reference_record).

The reference's textures module is loaded on the CPU with the stand-ins of make_texture_golden.py.  Each scene builds
its TexturesAtlas from a list of per-mesh atlases or from a padded tensor (with the meshes' face counts set, as Meshes
sets them), and the gradient is taken back to that input; each output is stored as its own case,
"atlas/R<R>-C<C>-<list|padded>/<field>".  "atlas/out_of_range/raises" records that the reference raises IndexError on
a slot whose cell lies past the end of the patch.

    python tests/golden/make_atlas_golden.py [OUT_DIR]
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [HERE, os.path.dirname(HERE)]

from make_texture_golden import put, reference_textures  # noqa: E402

LEAD = {"texels": 4, "grad_atlas": 1}


def run_reference(textures, ta, args):
    """[(field, tensor)] of one case, in the order of tests/test_texture_atlas.py: with_grads."""
    _, _, build = args
    s = ta.case_scene(args)
    if build == "list":
        leaves = [a.clone().requires_grad_(True) for a in s["atlases"]]
        tex = textures.TexturesAtlas(atlas=leaves)
    else:
        F = max(a.shape[0] for a in s["atlases"])
        padded = torch.zeros((len(s["atlases"]), F) + tuple(s["atlases"][0].shape[1:]))
        for i, a in enumerate(s["atlases"]):
            padded[i, :a.shape[0]] = a
        leaves = padded.requires_grad_(True)
        tex = textures.TexturesAtlas(atlas=leaves)
        tex._num_faces_per_mesh = [a.shape[0] for a in s["atlases"]]
    bary = s["bary"].clone().requires_grad_(True)
    texels = tex.sample_textures(types.SimpleNamespace(pix_to_face=s["pix_to_face"], bary_coords=bary))
    (texels * s["grad_texels"]).sum().backward()
    assert bary.grad is None
    grad = torch.cat([t.grad for t in leaves]) if build == "list" else leaves.grad
    return list(zip(ta.FIELDS, [texels.detach(), grad]))


def out_of_range_raises(textures, ta):
    s = ta.out_of_range_scene()
    tex = textures.TexturesAtlas(atlas=s["atlases"])
    try:
        tex.sample_textures(types.SimpleNamespace(pix_to_face=s["pix_to_face"], bary_coords=s["bary"]))
    except IndexError:
        return 1
    return 0


def main():
    import test_texture_atlas as ta
    out_dir = sys.argv[1] if len(sys.argv) > 1 else HERE
    torch.set_grad_enabled(True)
    textures = reference_textures()
    store = {}
    for args in ta.ATLAS_CASES:
        for field, t in run_reference(textures, ta, args):
            put(store, ta.atlas_case(args) + "/" + field, t, LEAD[field])
    put(store, "atlas/out_of_range/raises", np.array([out_of_range_raises(textures, ta)], np.int64), 1)
    out = os.path.join(out_dir, "reference_golden_atlas.npz")
    np.savez_compressed(out, **store)
    print("wrote %s: %d arrays, %d bytes" % (out, len(store), os.path.getsize(out)))
    assert os.path.getsize(out) < 1 << 20, "%s is larger than 1 MB: store fewer rows" % out


if __name__ == "__main__":
    main()
