"""TEST INFRASTRUCTURE ONLY -- builds the UNMODIFIED reference farthest point sampling and ball query ops into
oracle/_ref/.

Compiles, from the sources where they lie in the reference tree (never copied):
  pytorch3d/csrc/sample_farthest_points/sample_farthest_points_cpu.cpp  (both included by
  pytorch3d/csrc/ball_query/ball_query_cpu.cpp                          oracle/ref_point_ops_shim.cpp)
  pytorch3d/csrc/sample_farthest_points/sample_farthest_points.cu       (sm_90a)
  pytorch3d/csrc/ball_query/ball_query.cu                               (sm_90a)
into

  oracle/_ref/ref_point_ops_cpu.so    CPU only
  oracle/_ref/ref_point_ops_cuda.so   CPU+CUDA (the reference's own kernels recompiled for sm_90a)

with `build_op_pair` of oracle/build_ref_normals.py.  Ball query's backward, knn_points_backward, is
oracle/_ref/ref_knn_*.so (oracle/build_ref_knn.py).  tests/golden/make_point_ops_golden.py records the reference's ops
on the CPU with the first; tests/test_point_ops.py compares the fused kernels with the second.

Usage:  python oracle/build_ref_point_ops.py [--cpu-only] [--force]
"""
import argparse
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import build_ref, build_ref_normals  # noqa: E402

CPU_SOURCES = [os.path.join(build_ref.CSRC, "sample_farthest_points", "sample_farthest_points_cpu.cpp"),
               os.path.join(build_ref.CSRC, "ball_query", "ball_query_cpu.cpp")]  # compiled through the shim
CUDA_SOURCES = [os.path.join(build_ref.CSRC, "sample_farthest_points", "sample_farthest_points.cu"),
                os.path.join(build_ref.CSRC, "ball_query", "ball_query.cu")]
SHIM = os.path.join(HERE, "ref_point_ops_shim.cpp")
NAME = "ref_point_ops"


def reference_present():
    return all(os.path.exists(p) for p in CPU_SOURCES + CUDA_SOURCES)


def build(cpu_only=False, force=False):
    if not reference_present():
        print("[build_ref_point_ops] reference sources not found under %s -- nothing to do" % build_ref.REF)
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
