"""Writes tests/golden/reference_golden_normals.npz: the vertex normals, face areas and face normals of the reference's
own `Meshes` (pytorch3d/structures/meshes.py, with ops/mesh_face_areas_normals.py and structures/utils.py) on the seeded
scenes of tests/test_normals.py (SCENES), and the vertex gradients under seeded upstream gradients, in the record format
of make_reference_golden.py (tests/helpers.py: reference_record).

The reference modules are imported on the CPU with stand-ins only for the packages around them, as
make_gouraud_golden.py does; `pytorch3d._C` is the reference's own CPU face_areas_normals op, built by
oracle/build_ref_normals.py.  Each output is its own case, "normals/<scene>/<field>":
  verts_normals          Meshes.verts_normals_packed()
  grad_verts_normals     d/d verts of (verts_normals_packed() * g_vn).sum()
  faces_areas, faces_normals, grad_faces              faces_areas_packed(), faces_normals_packed() and d/d verts of
                                                       (areas * g_a).sum() + (normals * g_n).sum()

With --cuda (on an H100, with oracle/_ref/ref_normals_cuda.so) it writes reference_golden_normals_cuda.npz instead:
"normals_cuda/<scene>/<field>" for the reference's CUDA kernels, called as `_MeshFaceAreasNormals` calls them, on the
same scenes and upstream gradients: faces_areas, faces_normals and grad_faces.

    python tests/golden/make_normals_golden.py [--cuda] [OUT_DIR]
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
from oracle import build_ref, build_ref_normals  # noqa: E402

SAMPLE_ROWS = 64


def put(store, case, array):
    for field, v in reference_record([array], 1, SAMPLE_ROWS)[0].items():
        store["%s/0/%s" % (case, field)] = v


def _load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod
    spec.loader.exec_module(mod)
    return mod


def record_cpu(tn):
    ref = os.path.join(build_ref.REF, "pytorch3d")
    op = build_ref_normals.load(cuda=False)
    assert op is not None, "build oracle/_ref/ref_normals_cpu.so first (python oracle/build_ref_normals.py)"
    stub_names = ("pytorch3d", "pytorch3d.ops", "pytorch3d.structures")
    saved = {n: m for n, m in sys.modules.items() if n == "pytorch3d" or n.startswith("pytorch3d.")}
    stubs = {n: types.ModuleType(n) for n in stub_names}
    for m in stubs.values():
        m.__path__ = []
    stubs["pytorch3d"].__path__ = [ref]  # pytorch3d.common imports as the reference's own
    stubs["pytorch3d"]._C = op
    sys.modules.update(stubs)
    store = {}
    try:
        # meshes.py imports the op module lazily, inside _compute_face_areas_normals: keep it loaded while recording
        _load("pytorch3d.ops.mesh_face_areas_normals", os.path.join(ref, "ops", "mesh_face_areas_normals.py"))
        _load("pytorch3d.structures.utils", os.path.join(ref, "structures", "utils.py"))
        meshes = _load("pytorch3d.structures.meshes", os.path.join(ref, "structures", "meshes.py"))
        for name in tn.SCENES:
            s = tn.scene(name)
            g = tn.upstream_grads(s)
            for which in ("verts", "faces"):
                leaf = s["verts"].clone().requires_grad_(True)
                m = meshes.Meshes(verts=list(torch.split(leaf, s["nverts"])), faces=s["faces_list"])
                if which == "verts":
                    n = m.verts_normals_packed()
                    (n * g["verts_normals"]).sum().backward()
                    put(store, "normals/%s/verts_normals" % name, n.detach())
                    put(store, "normals/%s/grad_verts_normals" % name, leaf.grad)
                else:
                    a, fn = m.faces_areas_packed(), m.faces_normals_packed()
                    ((a * g["faces_areas"]).sum() + (fn * g["faces_normals"]).sum()).backward()
                    put(store, "normals/%s/faces_areas" % name, a.detach())
                    put(store, "normals/%s/faces_normals" % name, fn.detach())
                    put(store, "normals/%s/grad_faces" % name, leaf.grad)
    finally:
        for n in [n for n in sys.modules if n == "pytorch3d" or n.startswith("pytorch3d.")]:
            del sys.modules[n]
        sys.modules.update(saved)
    return store, "reference_golden_normals.npz"


def record_cuda(tn):
    op = build_ref_normals.load(cuda=True)
    assert op is not None and op.with_cuda, "build oracle/_ref/ref_normals_cuda.so first"
    dev = torch.device("cuda:0")
    store = {}
    for name in tn.SCENES:
        s = tn.scene(name)
        g = tn.upstream_grads(s)
        verts, faces = s["verts"].to(dev), s["faces"].to(dev)
        areas, normals = op.face_areas_normals_forward(verts, faces)
        grad = op.face_areas_normals_backward(g["faces_areas"].to(dev), g["faces_normals"].to(dev), verts, faces)
        put(store, "normals_cuda/%s/faces_areas" % name, areas.cpu())
        put(store, "normals_cuda/%s/faces_normals" % name, normals.cpu())
        put(store, "normals_cuda/%s/grad_faces" % name, grad.cpu())
    return store, "reference_golden_normals_cuda.npz"


def main():
    import test_normals as tn
    args = [a for a in sys.argv[1:] if a != "--cuda"]
    out_dir = args[0] if args else HERE
    torch.set_grad_enabled(True)
    store, fname = record_cuda(tn) if "--cuda" in sys.argv else record_cpu(tn)
    out = os.path.join(out_dir, fname)
    np.savez_compressed(out, **store)
    print("wrote %s: %d arrays, %d bytes" % (out, len(store), os.path.getsize(out)))
    assert os.path.getsize(out) < 1 << 20, "%s is larger than 1 MB: store fewer rows" % out


if __name__ == "__main__":
    main()
