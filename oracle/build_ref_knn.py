"""TEST INFRASTRUCTURE ONLY -- builds the UNMODIFIED reference k-nearest-neighbour op behind chamfer_distance into
oracle/_ref/.

Compiles, from the sources where they lie in the reference tree (never copied):
  pytorch3d/csrc/knn/knn_cpu.cpp  (included by oracle/ref_knn_shim.cpp, so that one compiler run parses the torch
                                   headers once per module)
  pytorch3d/csrc/knn/knn.cu       (sm_90a)
into

  oracle/_ref/ref_knn_cpu.so    CPU only
  oracle/_ref/ref_knn_cuda.so   CPU+CUDA (the reference's own kernels recompiled for sm_90a)

with `build_op_pair` of oracle/build_ref_normals.py.  tests/golden/make_chamfer_golden.py records the reference's
chamfer_distance on the CPU with the first; tests/test_chamfer.py compares the fused search with the second.

Usage:  python oracle/build_ref_knn.py [--cpu-only] [--force]
"""
import argparse
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import build_ref, build_ref_normals  # noqa: E402

CPU_SOURCES = [os.path.join(build_ref.CSRC, "knn", "knn_cpu.cpp")]  # compiled through the shim
CUDA_SOURCES = [os.path.join(build_ref.CSRC, "knn", "knn.cu")]
SHIM = os.path.join(HERE, "ref_knn_shim.cpp")
NAME = "ref_knn"


def reference_present():
    return all(os.path.exists(p) for p in CPU_SOURCES + CUDA_SOURCES)


def build(cpu_only=False, force=False):
    if not reference_present():
        print("[build_ref_knn] reference sources not found under %s -- nothing to do" % build_ref.REF)
        return False
    return build_ref_normals.build_op_pair(NAME, [], CUDA_SOURCES, SHIM, cpu_only=cpu_only, force=force)


def load(cuda=False):
    """The built module (None if absent)."""
    return build_ref_normals.load_module(NAME + ("_cuda" if cuda else "_cpu"))


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--cpu-only", action="store_true")
    ap.add_argument("--force", action="store_true")
    a = ap.parse_args()
    sys.exit(0 if build(cpu_only=a.cpu_only, force=a.force) else 1)
