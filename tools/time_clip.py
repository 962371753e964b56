"""Times the fused frustum culling / z-clipping (pytorch3d_b200.clip: clip_faces_fused, convert_clipped_fused) on the GPU
against the torch restatement (clip_faces, convert_clipped_rasterization_to_original_faces) that rasterize_meshes ran
before.  CUDA events, 20 iterations after warm-up; peak memory and host synchronisations (torch's sync debug mode) of
forward + backward; the card's name and power limit are read in the same run.

    python tools/time_clip.py OUT_DIR        -> OUT_DIR/time_clip.json

Workloads: the north-star torus batch (8 tori of 187 x 187, about 70 k faces each, depths 1 .. 3, 512 x 512, K = 8,
perspective-correct, cull_to_frustum) with z_clip = 1.05, where a few percent of the faces cross the plane, and the same
batch with z_clip = 0.5, where none does.  Rows:
  clip        clip step forward + backward on face_verts (F,3,3), upstream gradient on face_verts and the conversion
  convert     conversion forward + backward on the Fragments of the clipped faces, upstream gradient on bary
  end_to_end  rasterize_meshes(z_clip_value, cull_to_frustum) forward + backward to the vertices, new vs the previous
              wrapper (restatement + face_verts rasterizer)
"""
import json
import os
import subprocess
import sys
import warnings

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools")]

from time_blend import _events_ms, _peak_bytes  # noqa: E402

IMAGE, K, ITERS = (512, 512), 8, 20


def _frustum(z_clip):
    from pytorch3d_b200 import clip
    return clip.ClipFrustum(left=-1, right=1, top=-1, bottom=1, perspective_correct=True, z_clip_value=z_clip,
                            cull=True)


def previous_wrapper(meshes, z_clip):
    """rasterize_meshes as it ran before the fused pair: torch clip_faces, face_verts rasterizer, torch conversion."""
    import importlib
    from pytorch3d_b200 import clip
    rm = importlib.import_module("pytorch3d_b200.rasterize_meshes")
    fv = meshes.verts_packed()[meshes.faces_packed()]
    cf = clip.clip_faces(fv, meshes.mesh_to_faces_packed_first_idx(), meshes.num_faces_per_mesh(), _frustum(z_clip))
    nb = cf.clipped_faces_neighbor_idx
    if nb is None:
        nb = torch.full((cf.face_verts.shape[0],), -1, dtype=torch.int64, device=fv.device)
        nb._b200_all_minus_one = True
    p2f, zbuf, bary, dists = rm._RasterizeFaceVerts.apply(
        cf.face_verts, cf.mesh_to_face_first_idx, cf.num_faces_per_mesh, nb, IMAGE, 0.0, K, 0, 0, True, False, False)
    p2f, bary = clip.convert_clipped_rasterization_to_original_faces(p2f, bary, cf)
    return p2f, zbuf, bary, dists


def new_wrapper(meshes, z_clip):
    import pytorch3d_b200 as p3b
    return p3b.rasterize_meshes(meshes, IMAGE, 0.0, K, None, None, True, False, False, z_clip, True)


def _syncs(fn):
    torch.cuda.synchronize()
    prev = torch.cuda.get_sync_debug_mode()
    try:
        torch.cuda.set_sync_debug_mode("warn")
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            fn()
    finally:
        torch.cuda.set_sync_debug_mode(prev)
    return sum("synchroniz" in str(x.message) for x in w)


def _measure(fn):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    return {"us": _events_ms(fn, ITERS) * 1e3, "peak_mb": _peak_bytes(fn) / 2 ** 20, "host_syncs": _syncs(fn)}


def measure(meshes, z_clip):
    from pytorch3d_b200 import _C, clip
    fr = _frustum(z_clip)
    vp = meshes.verts_packed().detach().clone().requires_grad_(True)
    faces, first, num = meshes.faces_packed(), meshes.mesh_to_faces_packed_first_idx(), meshes.num_faces_per_mesh()
    fv0 = vp.detach()[faces]
    out = {"faces": int(faces.shape[0])}

    def clip_step(fn):
        def run():
            x = fv0.clone().requires_grad_(True)
            cf = fn(x, first, num, fr)
            loss = cf.face_verts.sum()
            if cf.barycentric_conversion is not None:
                loss = loss + cf.barycentric_conversion.sum()
            torch.autograd.grad(loss, x)
        return run

    cf = clip.clip_faces_fused(fv0, first, num, fr)
    out["faces_clipped"] = int(cf.face_verts.shape[0])
    out["faces_with_conversion"] = 0 if cf.barycentric_conversion is None else int(cf.barycentric_conversion.shape[0])
    out["clip_fused"] = _measure(clip_step(clip.clip_faces_fused))
    out["clip_restatement"] = _measure(clip_step(clip.clip_faces))

    if cf.faces_clipped_to_unclipped_idx is not None:
        nb = cf.clipped_faces_neighbor_idx
        if nb is None:
            nb = torch.full((cf.face_verts.shape[0],), -1, dtype=torch.int64, device=fv0.device)
        p2f, _, bary, _ = _C.rasterize_meshes(cf.face_verts, cf.mesh_to_face_first_idx, cf.num_faces_per_mesh, nb,
                                              IMAGE, 0.0, K, 0, 0, True, False, False)
        cf_t = clip.clip_faces(fv0, first, num, fr)

        def convert_step(fn, c):
            def run():
                b = bary.clone().requires_grad_(True)
                _, bu = fn(p2f, b, c)
                torch.autograd.grad(bu.sum(), b)
            return run

        out["convert_fused"] = _measure(convert_step(clip.convert_clipped_fused, cf))
        out["convert_restatement"] = _measure(convert_step(clip.convert_clipped_rasterization_to_original_faces, cf_t))

    def e2e(fn):
        def run():
            from pytorch3d_b200 import PackedMeshes
            m = PackedMeshes([vp], [faces])  # (one packed mesh list entry per call keeps the graph fresh)
            m._num_faces_per_mesh, m._mesh_to_faces_packed_first_idx = num, first
            o = fn(m, z_clip)
            torch.autograd.grad(o[1].clamp_min(0).sum() + o[2].sum() + o[3].sum(), vp)
        return run

    out["end_to_end_new"] = _measure(e2e(new_wrapper))
    out["end_to_end_previous"] = _measure(e2e(previous_wrapper))
    # same results: the new wrapper against the previous one on this workload
    a, b, c = new_wrapper(meshes, z_clip), previous_wrapper(meshes, z_clip), previous_wrapper(meshes, z_clip)
    for name, x, y in (("new_vs_previous", a, b), ("previous_vs_previous_rerun", b, c)):
        out[name] = {"differing_pix_to_face": int((x[0] != y[0]).sum()), "differing_zbuf": int((x[1] != y[1]).sum()),
                     "differing_dists": int((x[3] != y[3]).sum()),
                     "max_abs_bary_diff_where_same_face": float((x[2] - y[2]).abs()[x[0] == y[0]].max())}
    return out


def main():
    from pytorch3d_b200 import synthetic
    out_dir = sys.argv[1] if len(sys.argv) > 1 else "."
    dev = torch.device("cuda:0")
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               stdout=subprocess.PIPE, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = "not measured"
    meshes = synthetic.torus_batch(8, 187, 187, seed=0, device=dev)
    report = {"device": torch.cuda.get_device_name(dev), "power_limit": power, "workloads": {}}
    report["workloads"]["torus_8x70k_512_K8_zclip1.05"] = measure(meshes, 1.05)
    report["workloads"]["torus_8x70k_512_K8_zclip0.5_nothing_crosses"] = measure(meshes, 0.5)
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "time_clip.json"), "w") as fh:
        json.dump(report, fh, indent=1)
    print(json.dumps(report, indent=1))


if __name__ == "__main__":
    main()
