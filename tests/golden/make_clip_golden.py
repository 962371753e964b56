"""Writes tests/golden/reference_clip.npz (not named reference_golden*.npz: those hold rasterizer records in the format
of tests/helpers.py): what the reference's own clip_faces and
convert_clipped_rasterization_to_original_faces (pytorch3d/renderer/mesh/clip.py) compute on the CPU for the seeded
scenes of tests/test_clip_fused.py.

clip.py imports only torch, so it is loaded by file path.  Per scene "clip_faces/<name>/0/..." it stores the inputs, the seven
ClippedFaces fields (absent when the reference returns None), a seeded Fragments over the clipped faces (about 30 %
background) with its conversion, and the gradient of face_verts_unclipped (and of the clipped barycentrics) for seeded
upstream gradients on the clipped face_verts and on the converted barycentrics.

    python tests/golden/make_clip_golden.py [OUT_DIR]
"""
import importlib.util
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.dirname(HERE)]

from oracle import build_ref  # noqa: E402

FIELDS = ("face_verts", "mesh_to_face_first_idx", "num_faces_per_mesh", "faces_clipped_to_unclipped_idx",
          "barycentric_conversion", "faces_clipped_to_conversion_idx", "clipped_faces_neighbor_idx")


def reference_clip():
    path = os.path.join(build_ref.REF, "pytorch3d", "renderer", "mesh", "clip.py")
    spec = importlib.util.spec_from_file_location("reference_clip", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def run_reference(clip, tc, name):
    s = tc.clip_scene(name)
    fv = s["face_verts"].clone().requires_grad_(True)
    fr = clip.ClipFrustum(**tc.frustum_kwargs(s))
    out = clip.clip_faces(fv, s["first"], s["num"], fr)
    rec = {"face_verts_in": s["face_verts"], "first_in": s["first"], "num_in": s["num"], "planes": s["planes"],
           "flags": s["flags"], "z_clip": s["z_clip"]}
    for f in FIELDS:
        v = getattr(out, f)
        if v is not None:
            rec["out_" + f] = v.detach()
    p2f, bary, g_fv, g_bary = tc.fragments(name, int(out.face_verts.shape[0]))
    bary = bary.clone().requires_grad_(True)
    p2f_u, bary_u = clip.convert_clipped_rasterization_to_original_faces(p2f, bary, out)
    loss = (out.face_verts * g_fv).sum() + (bary_u * g_bary).sum()
    if loss.requires_grad:
        loss.backward()
    rec.update(p2f_in=p2f, bary_in=bary.detach(), grad_fv_clipped_in=g_fv, grad_bary_unclipped_in=g_bary,
               p2f_out=p2f_u, bary_out=bary_u.detach(),
               grad_face_verts=fv.grad if fv.grad is not None else torch.zeros_like(fv),
               grad_bary_in=bary.grad if bary.grad is not None else torch.zeros_like(bary))
    return rec


def main():
    import test_clip_fused as tc
    out_dir = sys.argv[1] if len(sys.argv) > 1 else HERE
    clip = reference_clip()
    store = {}
    for name in tc.SCENES:
        for k, v in run_reference(clip, tc, name).items():
            store["clip_faces/%s/0/%s" % (name, k)] = v.numpy() if torch.is_tensor(v) else np.asarray(v)
    out = os.path.join(out_dir, "reference_clip.npz")
    np.savez_compressed(out, **store)
    print("wrote %s: %d arrays, %d bytes" % (out, len(store), os.path.getsize(out)))
    assert os.path.getsize(out) < 1 << 20, "%s is larger than 1 MB" % out


if __name__ == "__main__":
    main()
