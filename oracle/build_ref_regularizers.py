"""TEST INFRASTRUCTURE ONLY -- builds the UNMODIFIED reference face-pair enumeration of mesh_normal_consistency into
oracle/_ref/.

Compiles, from the source where it lies in the reference tree (never copied):
  pytorch3d/csrc/mesh_normal_consistency/mesh_normal_consistency_cpu.cpp
plus oracle/ref_regularizers_shim.cpp, into

  oracle/_ref/ref_regularizers_cpu.so    CPU only (the reference has no CUDA version of this op)

with `build_op_pair` of oracle/build_ref_normals.py.  tests/golden/make_regularizers_golden.py records the reference's
losses on it, and tools/time_regularizers.py times the reference's normal-consistency chain with it.

Usage:  python oracle/build_ref_regularizers.py [--force]
"""
import argparse
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import build_ref, build_ref_normals  # noqa: E402

CPU_SOURCES = [os.path.join(build_ref.CSRC, "mesh_normal_consistency", "mesh_normal_consistency_cpu.cpp")]
SHIM = os.path.join(HERE, "ref_regularizers_shim.cpp")
NAME = "ref_regularizers"


def reference_present():
    return all(os.path.exists(p) for p in CPU_SOURCES)


def build(force=False):
    if not reference_present():
        print("[build_ref_regularizers] reference sources not found under %s -- nothing to do" % build_ref.REF)
        return False
    return build_ref_normals.build_op_pair(NAME, CPU_SOURCES, [], SHIM, cpu_only=True, force=force)


def load():
    """The built module (None if absent)."""
    return build_ref_normals.load_module(NAME + "_cpu")


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--force", action="store_true")
    a = ap.parse_args()
    sys.exit(0 if build(force=a.force) else 1)
