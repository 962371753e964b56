"""TEST INFRASTRUCTURE ONLY -- builds the UNMODIFIED reference packed-to-padded op behind sample_points_from_meshes
into oracle/_ref/.

Compiles, from the source where it lies in the reference tree (never copied; oracle/ref_sampling_shim.cpp includes it,
so that one compiler run parses the torch headers once):
  pytorch3d/csrc/packed_to_padded_tensor/packed_to_padded_tensor_cpu.cpp
with the shim, into

  oracle/_ref/ref_sampling_cpu.so    CPU only

with `build_op_pair` of oracle/build_ref_normals.py.  The sampler's other native op, face_areas_normals, is
oracle/_ref/ref_normals_cpu.so (oracle/build_ref_normals.py), so it is not compiled a second time.
tests/golden/make_sampling_golden.py records the reference's sample_points_from_meshes on the CPU with the two.

Usage:  python oracle/build_ref_sampling.py [--force]
"""
import argparse
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import build_ref, build_ref_normals  # noqa: E402

CPU_SOURCES = [os.path.join(build_ref.CSRC, "packed_to_padded_tensor", "packed_to_padded_tensor_cpu.cpp")]
SHIM = os.path.join(HERE, "ref_sampling_shim.cpp")
NAME = "ref_sampling"


def reference_present():
    return all(os.path.exists(p) for p in CPU_SOURCES)


def build(force=False):
    if not reference_present():
        print("[build_ref_sampling] reference sources not found under %s -- nothing to do" % build_ref.REF)
        return False
    return build_ref_normals.build_op_pair(NAME, [], [], SHIM, cpu_only=True, force=force)


def load():
    """The built module (None if absent)."""
    return build_ref_normals.load_module(NAME + "_cpu")


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--force", action="store_true")
    a = ap.parse_args()
    sys.exit(0 if build(force=a.force) else 1)
