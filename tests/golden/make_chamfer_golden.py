"""Writes tests/golden/reference_golden_chamfer.npz: the reference's own chamfer_distance (pytorch3d/loss/chamfer.py
with ops/knn.py) on the CPU, on the seeded scenes of tests/test_chamfer.py (chamfer_scenes), for every option
combination of test_chamfer.OPTIONS, with the gradients of test_chamfer.upstream-weighted outputs.

The reference modules are imported with stand-ins only for the packages around them, as make_sampling_golden.py
does; `pytorch3d._C` is the reference's own CPU knn op, built by oracle/build_ref_knn.py.  Keys:
  chamfer/<scene>/<option>/0/loss, loss_normals (and loss_y, loss_normals_y for point_reduction None)
  chamfer/<scene>/<option>/0/grad_x, grad_y, grad_x_normals, grad_y_normals
  chamfer/<scene>/<option>/0/error      the reference's error message, for calls it rejects (bytes)
(the name/index/field layout of the other records, so tests/helpers.py: reference reads them).

    python tests/golden/make_chamfer_golden.py [OUT_DIR]
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

from oracle import build_ref, build_ref_knn  # noqa: E402


def _load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod
    spec.loader.exec_module(mod)
    return mod


class _Pointclouds:
    """Stand-in for the reference's Pointclouds (chamfer.py only tests isinstance against it)."""


def reference_chamfer():
    ref = os.path.join(build_ref.REF, "pytorch3d")
    op = build_ref_knn.load()
    assert op is not None, "build oracle/_ref/ref_knn_cpu.so first (python oracle/build_ref_knn.py)"
    stub_names = ("pytorch3d", "pytorch3d.ops", "pytorch3d.structures", "pytorch3d.structures.pointclouds",
                  "pytorch3d.loss")
    stubs = {n: types.ModuleType(n) for n in stub_names}
    for m in stubs.values():
        m.__path__ = []
    stubs["pytorch3d"]._C = op
    stubs["pytorch3d.structures.pointclouds"].Pointclouds = _Pointclouds
    sys.modules.update(stubs)
    _load("pytorch3d.ops.knn", os.path.join(ref, "ops", "knn.py"))
    return _load("pytorch3d.loss.chamfer", os.path.join(ref, "loss", "chamfer.py")).chamfer_distance


def main(out_dir):
    import test_chamfer as T
    cd = reference_chamfer()
    store = {}
    for sname, scene in T.chamfer_scenes().items():
        for oname, opts in T.OPTIONS.items():
            key = "chamfer/%s/%s/0" % (sname, oname)
            try:
                res = T.run_with_grads(cd, scene, opts)
            except Exception as e:  # noqa: BLE001 -- the reference's own rejection is the record
                store[key + "/error"] = np.frombuffer(str(e).encode(), dtype=np.uint8)
                continue
            for k, v in res.items():
                store["%s/%s" % (key, k)] = v
    path = os.path.join(out_dir, "reference_golden_chamfer.npz")
    np.savez_compressed(path, **store)
    print("wrote %s (%d arrays)" % (path, len(store)))


if __name__ == "__main__":
    torch.set_num_threads(1)
    main(sys.argv[1] if len(sys.argv) > 1 else HERE)
