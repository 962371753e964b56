"""Builds pytorch3d_b200/lib/libb200raster.so (hand-written sm_90a kernels + C ABI) with nvcc, and the torch C++
extension over it (csrc/torch_ext.cpp) with g++.

nvcc cross-compiles without a GPU; the built .so files are git-ignored.
Usage: python -m pytorch3d_b200.build [--force] [--verbose]
"""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB_DIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIB_DIR, "libb200raster.so")
SOURCES = ["raster_meshes.cu", "raster_points.cu", "compositing.cu", "blending.cu", "splatter_blend.cu", "shading.cu", "textures.cu", "texture_atlas.cu", "normals.cu", "regularizers.cu", "sampling.cu", "chamfer.cu", "point_ops.cu", "clip.cu", "interp_face_attrs.cu", "peer_exchange.cu",
           "coarse_hooks.cu", "host_api.cu"]
HEADERS = ["raster_math.cuh", "bulk_copy.cuh", "binning.cuh", "common.cuh", "keyed_runs.cuh", "mesh_tables.cuh", "point_pairs.cuh", os.path.join("..", "..", "include", "b200_raster.h")]


# The one architecture the library is built for (H100, sm_90a); tools/variant_time.py builds its variants with it too.
ARCH_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a"]


def _nvcc():
    return shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"


def is_stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(os.path.join(CSRC, f)) > t for f in SOURCES + HEADERS)


def build(force=False, verbose=False):
    """libb200raster.so, then the torch extension over it, each rebuilt when stale; returns the library's path."""
    if force or is_stale():
        _build_lib(verbose)
    _build_ext(force, verbose)
    return LIB


def _build_lib(verbose):
    os.makedirs(LIB_DIR, exist_ok=True)
    cmd = [_nvcc(), "-O3", "-std=c++17"] + ARCH_FLAGS + ["-lineinfo",
           "-Xcompiler", "-fPIC", "-shared", "-Xptxas", "-v", "-o", LIB] + [os.path.join(CSRC, f) for f in SOURCES]
    res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    with open(os.path.join(LIB_DIR, "build.log"), "w") as fh:
        fh.write(" ".join(cmd) + "\n" + res.stdout)
    if verbose or res.returncode != 0:
        print(res.stdout)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed building libb200raster.so (see output above)")


EXT_NAME = "_b200_ext"
EXT_SRC = os.path.join(CSRC, "torch_ext.cpp")


def ext_path():
    import sysconfig
    return os.path.join(LIB_DIR, EXT_NAME + (sysconfig.get_config_var("EXT_SUFFIX") or ".so"))


def _build_ext(force, verbose):
    """The torch C++ extension over the C ABI (csrc/torch_ext.cpp): what `pytorch3d_b200._C` binds the rasterizer ops
    to, like `pytorch3d._C` in the reference (ext.cpp, setup.py:143-151).  Plain g++ with torch's own include / library
    paths (the same the reference's setup.py passes through torch.utils.cpp_extension); links libb200raster.so by
    $ORIGIN."""
    out = ext_path()
    deps = [EXT_SRC, os.path.join(HERE, "..", "include", "b200_raster.h")]
    if not force and os.path.exists(out) and all(os.path.getmtime(d) <= os.path.getmtime(out) for d in deps):
        return out
    import sysconfig

    import torch
    from torch.utils import cpp_extension as ce
    inc = ce.include_paths(device_type="cuda") + [sysconfig.get_paths()["include"]]
    libdirs = ce.library_paths(device_type="cuda")
    abi = "-D_GLIBCXX_USE_CXX11_ABI=%d" % int(torch.compiled_with_cxx11_abi())
    cmd = ["g++", "-O2", "-fPIC", "-std=c++17", "-shared", abi, "-DTORCH_EXTENSION_NAME=" + EXT_NAME,
           "-DTORCH_API_INCLUDE_EXTENSION_H", EXT_SRC, "-o", out]
    for i in inc:
        cmd += ["-isystem", i]
    for d in libdirs:
        cmd += ["-L" + d, "-Wl,-rpath," + d]
    cmd += ["-L" + LIB_DIR, "-Wl,-rpath,$ORIGIN", "-lb200raster", "-lc10", "-lc10_cuda", "-ltorch_cpu", "-ltorch_cuda",
            "-ltorch", "-ltorch_python", "-lcudart"]
    res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    with open(os.path.join(LIB_DIR, "build_ext.log"), "w") as fh:
        fh.write(" ".join(cmd) + "\n" + res.stdout)
    if verbose or res.returncode != 0:
        print(res.stdout)
    if res.returncode != 0:
        raise RuntimeError("g++ failed building the torch extension (see output above)")
    return out


if __name__ == "__main__":
    build(force="--force" in sys.argv, verbose=True)
    print("built", LIB)
    print("built", ext_path())
