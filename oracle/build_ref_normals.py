"""TEST INFRASTRUCTURE ONLY -- builds the UNMODIFIED reference face areas / normals op into oracle/_ref/.

Compiles, from the sources where they lie in the reference tree (never copied):
  pytorch3d/csrc/face_areas_normals/face_areas_normals_cpu.cpp
  pytorch3d/csrc/face_areas_normals/face_areas_normals.cu      (sm_90a)
plus oracle/ref_normals_shim.cpp, into

  oracle/_ref/ref_normals_cpu.so    CPU only
  oracle/_ref/ref_normals_cuda.so   CPU+CUDA (the reference's own kernels recompiled for sm_90a)

with the flags of oracle/build_ref.py (the reference's setup.py).  `build_op_pair` is the recipe of
oracle/build_ref_blend.py with the sources and the module name as parameters, so that further single-op oracles need
no copy of it.  tests/golden/make_normals_golden.py stores what the tests compare against.

Usage:  python oracle/build_ref_normals.py [--cpu-only] [--force]
"""
import argparse
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import build_ref  # noqa: E402

CPU_SOURCES = [os.path.join(build_ref.CSRC, "face_areas_normals", "face_areas_normals_cpu.cpp")]
CUDA_SOURCES = [os.path.join(build_ref.CSRC, "face_areas_normals", "face_areas_normals.cu")]
SHIM = os.path.join(HERE, "ref_normals_shim.cpp")
NAME = "ref_normals"


def reference_present():
    return all(os.path.exists(p) for p in CPU_SOURCES + CUDA_SOURCES)


def build_op_pair(name, cpu_sources, cuda_sources, shim, cpu_only=False, force=False):
    """oracle/_ref/<name>_cpu.so from `cpu_sources` + `shim`, and (unless cpu_only) <name>_cuda.so from those and
    `cuda_sources` compiled for sm_90a; each rebuilt when older than a source."""
    os.makedirs(build_ref.OUT, exist_ok=True)
    torch, inc, lib = build_ref._torch_paths()
    abi = "-D_GLIBCXX_USE_CXX11_ABI=%d" % int(torch._C._GLIBCXX_USE_CXX11_ABI)
    ldflags = []
    for p in lib:
        ldflags += ["-L" + p, "-Wl,-rpath," + p]
    ldflags += ["-lc10", "-ltorch_cpu", "-ltorch", "-ltorch_python"]

    def stale(target, srcs):
        return force or not os.path.exists(target) or any(os.path.getmtime(s) > os.path.getmtime(target) for s in srcs)

    for module, cuda in ((name + "_cpu", False), (name + "_cuda", True)):
        if cuda and cpu_only:
            break
        target = os.path.join(build_ref.OUT, module + ".so")
        srcs = cpu_sources + [shim] + (cuda_sources if cuda else [])
        if not stale(target, srcs):
            continue
        objs = []
        for i, src in enumerate(cpu_sources + [shim]):
            obj = os.path.join(build_ref.OUT, "%s_%d.o" % (module, i))
            build_ref._run(["g++", "-O2", "-fPIC", "-std=c++17", abi] + (["-DWITH_CUDA"] if cuda else [])
                           + ["-c", src, "-o", obj] + build_ref._common(module, inc))
            objs.append(obj)
        extra = []
        if cuda:
            nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
            for i, src in enumerate(cuda_sources):
                obj = os.path.join(build_ref.OUT, "%s_cu%d.o" % (module, i))
                build_ref._run([nvcc, "-O3", "-std=c++17", "-Xcompiler", "-fPIC", abi, "-DWITH_CUDA",
                                "-DCUDA_HAS_FP16=1", "-D__CUDA_NO_HALF_OPERATORS__", "-D__CUDA_NO_HALF_CONVERSIONS__",
                                "-D__CUDA_NO_HALF2_OPERATORS__", "-DTHRUST_IGNORE_CUB_VERSION_CHECK",
                                "--expt-relaxed-constexpr", "-gencode", "arch=compute_90a,code=sm_90a", "-c", src,
                                "-o", obj] + build_ref._common(module, inc))
                objs.append(obj)
            extra = ["-L/usr/local/cuda/lib64", "-lcudart", "-lc10_cuda", "-ltorch_cuda"]
        build_ref._run(["g++", "-shared", "-o", target] + objs + ldflags + extra)
    return True


def load_module(module):
    """oracle/_ref/<module>.so imported (None if absent)."""
    import importlib.util
    import torch  # noqa: F401  (the .so links against libtorch)
    path = os.path.join(build_ref.OUT, module + ".so")
    if not os.path.exists(path):
        return None
    spec = importlib.util.spec_from_file_location(module, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def build(cpu_only=False, force=False):
    if not reference_present():
        print("[build_ref_normals] reference sources not found under %s -- nothing to do" % build_ref.REF)
        return False
    return build_op_pair(NAME, CPU_SOURCES, CUDA_SOURCES, SHIM, cpu_only=cpu_only, force=force)


def load(cuda=False):
    """The built module (None if absent)."""
    return load_module(NAME + ("_cuda" if cuda else "_cpu"))


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--cpu-only", action="store_true")
    ap.add_argument("--force", action="store_true")
    a = ap.parse_args()
    sys.exit(0 if build(cpu_only=a.cpu_only, force=a.force) else 1)
