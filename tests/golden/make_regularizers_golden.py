"""Writes tests/golden/reference_golden_regularizers.npz: the reference's own mesh_edge_loss, mesh_laplacian_smoothing
and mesh_normal_consistency (pytorch3d/loss/*.py, with ops/laplacian_matrices.py, structures/meshes.py and
structures/utils.py) on the seeded scenes of tests/test_regularizers.py (SCENES), in the record format of
make_reference_golden.py (tests/helpers.py: reference_record).

The reference modules are imported on the CPU with stand-ins only for the packages around them, as
make_normals_golden.py does; `pytorch3d._C` is the reference's own CPU face-pair op, built by
oracle/build_ref_regularizers.py.  Each output is its own case:
  regularizers/<scene>/edges, faces_to_edges, num_edges_per_mesh     Meshes.edges_packed(),
                                                                      faces_packed_to_edges_packed(), num_edges_per_mesh()
  regularizers/<scene>/<case>/loss      the loss of case (edge_t0, edge_t005, lap_uniform, lap_cot, lap_cotcurv, normal)
  regularizers/<scene>/<case>/grad      d/d verts of loss * g, g the seeded scalar of test_regularizers.upstream (zeros
                                        where the reference's result is not connected to the verts)

    python tests/golden/make_regularizers_golden.py [OUT_DIR]
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
from oracle import build_ref, build_ref_regularizers  # noqa: E402

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


def record(tr):
    ref = os.path.join(build_ref.REF, "pytorch3d")
    op = build_ref_regularizers.load()
    assert op is not None, "build oracle/_ref/ref_regularizers_cpu.so first (python oracle/build_ref_regularizers.py)"
    stub_names = ("pytorch3d", "pytorch3d.ops", "pytorch3d.structures", "pytorch3d.loss")
    saved = {n: m for n, m in sys.modules.items() if n == "pytorch3d" or n.startswith("pytorch3d.")}
    stubs = {n: types.ModuleType(n) for n in stub_names}
    for m in stubs.values():
        m.__path__ = []
    stubs["pytorch3d"].__path__ = [ref]  # pytorch3d.common imports as the reference's own
    stubs["pytorch3d"]._C = op
    sys.modules.update(stubs)
    store = {}
    try:
        lap = _load("pytorch3d.ops.laplacian_matrices", os.path.join(ref, "ops", "laplacian_matrices.py"))
        for n in ("laplacian", "cot_laplacian", "norm_laplacian"):
            setattr(stubs["pytorch3d.ops"], n, getattr(lap, n))
        _load("pytorch3d.structures.utils", os.path.join(ref, "structures", "utils.py"))
        meshes = _load("pytorch3d.structures.meshes", os.path.join(ref, "structures", "meshes.py"))
        losses = {n: _load("pytorch3d.loss." + n, os.path.join(ref, "loss", n + ".py"))
                  for n in ("mesh_edge_loss", "mesh_laplacian_smoothing", "mesh_normal_consistency")}
        for name in tr.SCENES:
            s = tr.scene(name)
            m = meshes.Meshes(verts=list(torch.split(s["verts"], s["nverts"])), faces=s["faces_list"])
            put(store, "regularizers/%s/edges" % name, m.edges_packed())
            put(store, "regularizers/%s/faces_to_edges" % name, m.faces_packed_to_edges_packed())
            put(store, "regularizers/%s/num_edges_per_mesh" % name, m.num_edges_per_mesh().to(torch.int64))
            for case, loss, arg in tr.CASES:
                leaf = s["verts"].clone().requires_grad_(True)
                m = meshes.Meshes(verts=list(torch.split(leaf, s["nverts"])), faces=s["faces_list"])
                if loss == "edge":
                    out = losses["mesh_edge_loss"].mesh_edge_loss(m, target_length=arg)
                elif loss == "laplacian":
                    out = losses["mesh_laplacian_smoothing"].mesh_laplacian_smoothing(m, method=arg)
                else:
                    out = losses["mesh_normal_consistency"].mesh_normal_consistency(m)
                (out.sum() * tr.upstream(name, case)).backward()
                grad = leaf.grad if leaf.grad is not None else torch.zeros_like(leaf)
                put(store, "regularizers/%s/%s/loss" % (name, case), out.detach().reshape(1, 1))
                put(store, "regularizers/%s/%s/grad" % (name, case), grad)
    finally:
        for n in [n for n in sys.modules if n == "pytorch3d" or n.startswith("pytorch3d.")]:
            del sys.modules[n]
        sys.modules.update(saved)
    return store


def main():
    import test_regularizers as tr
    out_dir = sys.argv[1] if len(sys.argv) > 1 else HERE
    torch.set_grad_enabled(True)
    store = record(tr)
    out = os.path.join(out_dir, "reference_golden_regularizers.npz")
    np.savez_compressed(out, **store)
    print("wrote %s: %d arrays, %d bytes" % (out, len(store), os.path.getsize(out)))
    assert os.path.getsize(out) < 1 << 20, "%s is larger than 1 MB: store fewer rows" % out


if __name__ == "__main__":
    main()
