"""TEST INFRASTRUCTURE ONLY -- builds the UNMODIFIED reference blending ops into oracle/_ref/.

Compiles, from the sources where they lie in the reference tree (never copied):
  pytorch3d/csrc/blending/sigmoid_alpha_blend_cpu.cpp
  pytorch3d/csrc/blending/sigmoid_alpha_blend.cu           (sm_90a)
plus oracle/ref_blend_shim.cpp, into

  oracle/_ref/ref_blend_cpu.so    CPU only
  oracle/_ref/ref_blend_cuda.so   CPU+CUDA (the reference's own kernels recompiled for sm_90a)

with the flags of oracle/build_ref.py (the reference's setup.py).  A module of its own, so that the rasterizer's
reference build and the golden files made from it stay as they are.  tests/golden/make_blend_golden.py stores what the
tests compare against.

Usage:  python oracle/build_ref_blend.py [--cpu-only] [--force]
"""
import argparse
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import build_ref  # noqa: E402

CPU_SOURCES = [os.path.join(build_ref.CSRC, "blending", "sigmoid_alpha_blend_cpu.cpp")]
CUDA_SOURCES = [os.path.join(build_ref.CSRC, "blending", "sigmoid_alpha_blend.cu")]
SHIM = os.path.join(HERE, "ref_blend_shim.cpp")


def reference_present():
    return all(os.path.exists(p) for p in CPU_SOURCES + CUDA_SOURCES)


def build(cpu_only=False, force=False):
    if not reference_present():
        print("[build_ref_blend] reference sources not found under %s -- nothing to do" % build_ref.REF)
        return False
    os.makedirs(build_ref.OUT, exist_ok=True)
    torch, inc, lib = build_ref._torch_paths()
    abi = "-D_GLIBCXX_USE_CXX11_ABI=%d" % int(torch._C._GLIBCXX_USE_CXX11_ABI)
    ldflags = []
    for p in lib:
        ldflags += ["-L" + p, "-Wl,-rpath," + p]
    ldflags += ["-lc10", "-ltorch_cpu", "-ltorch", "-ltorch_python"]

    def stale(target, srcs):
        return force or not os.path.exists(target) or any(os.path.getmtime(s) > os.path.getmtime(target) for s in srcs)

    for name, cuda in (("ref_blend_cpu", False), ("ref_blend_cuda", True)):
        if cuda and cpu_only:
            break
        target = os.path.join(build_ref.OUT, name + ".so")
        srcs = CPU_SOURCES + [SHIM] + (CUDA_SOURCES if cuda else [])
        if not stale(target, srcs):
            continue
        objs = []
        for i, src in enumerate(CPU_SOURCES + [SHIM]):
            obj = os.path.join(build_ref.OUT, "%s_%d.o" % (name, i))
            build_ref._run(["g++", "-O2", "-fPIC", "-std=c++17", abi] + (["-DWITH_CUDA"] if cuda else [])
                           + ["-c", src, "-o", obj] + build_ref._common(name, inc))
            objs.append(obj)
        extra = []
        if cuda:
            nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
            for i, src in enumerate(CUDA_SOURCES):
                obj = os.path.join(build_ref.OUT, "%s_cu%d.o" % (name, i))
                build_ref._run([nvcc, "-O3", "-std=c++17", "-Xcompiler", "-fPIC", abi, "-DWITH_CUDA",
                                "-DCUDA_HAS_FP16=1", "-D__CUDA_NO_HALF_OPERATORS__", "-D__CUDA_NO_HALF_CONVERSIONS__",
                                "-D__CUDA_NO_HALF2_OPERATORS__", "-DTHRUST_IGNORE_CUB_VERSION_CHECK",
                                "--expt-relaxed-constexpr", "-gencode", "arch=compute_90a,code=sm_90a", "-c", src,
                                "-o", obj] + build_ref._common(name, inc))
                objs.append(obj)
            extra = ["-L/usr/local/cuda/lib64", "-lcudart", "-lc10_cuda", "-ltorch_cuda"]
        build_ref._run(["g++", "-shared", "-o", target] + objs + ldflags + extra)
    return True


def load(cuda=False):
    """The built module (None if absent)."""
    import importlib.util
    import torch  # noqa: F401  (the .so links against libtorch)
    name = "ref_blend_cuda" if cuda else "ref_blend_cpu"
    path = os.path.join(build_ref.OUT, name + ".so")
    if not os.path.exists(path):
        return None
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--cpu-only", action="store_true")
    ap.add_argument("--force", action="store_true")
    a = ap.parse_args()
    sys.exit(0 if build(cpu_only=a.cpu_only, force=a.force) else 1)
