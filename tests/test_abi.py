"""The C-ABI library loads on a CPU-only machine and exports every symbol include/b200_raster.h declares."""
import ctypes
import os
import re

from conftest import ROOT


def _declared_symbols():
    text = open(os.path.join(ROOT, "include", "b200_raster.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(b200r_[a-z_0-9]+)\s*\(", text)))


def test_header_declares_expected_entry_points():
    syms = _declared_symbols()
    for s in ("b200r_rasterize_meshes_forward", "b200r_rasterize_meshes_backward", "b200r_rasterize_points_forward",
              "b200r_rasterize_points_backward", "b200r_rasterize_meshes_forward_host",
              "b200r_rasterize_points_forward_host", "b200r_last_error", "b200r_version"):
        assert s in syms


def test_library_exports_every_declared_symbol(built_lib):
    lib = ctypes.CDLL(built_lib)
    for s in _declared_symbols():
        assert hasattr(lib, s), "libb200raster.so does not export %s" % s


def test_ctypes_prototypes_cover_the_header(built_lib):
    from pytorch3d_b200 import _lib
    assert sorted(_lib.SIGNATURES) == _declared_symbols()
    lib = _lib.load()
    assert lib.b200r_version().startswith(b"b200raster")
    assert lib.b200r_kernel_launch_count() == 0


def test_workspace_size_query_is_pure_host_code(built_lib):
    from pytorch3d_b200 import _lib
    lib = _lib.load()
    small = lib.b200r_rasterize_meshes_workspace_bytes(1000, 2, 64, 64, 0)
    big = lib.b200r_rasterize_meshes_workspace_bytes(100000, 8, 512, 512, 0)
    assert 0 < small < big
    explicit = lib.b200r_rasterize_meshes_workspace_bytes(1000, 2, 64, 64, 12345)
    assert explicit != small
    assert lib.b200r_rasterize_points_workspace_bytes(1000, 2, 64, 64, 0) > 0


def test_sass_contains_tma_bulk_copy(built_lib):
    """The setup kernels stage packed face_verts with cp.async.bulk (SASS: UBLKCP)."""
    import shutil
    import subprocess
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        import pytest
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", built_lib], stdout=subprocess.PIPE, text=True).stdout
    assert "UBLKCP" in sass
    assert "sm_90a" in sass or "SM90" in sass.upper() or "EF_CUDA_SM90" in sass


def test_torch_extension_loads_and_mirrors_the_reference_ops(built_lib):
    """csrc/torch_ext.cpp: the pybind11 / torch C++ extension over the C ABI (the binding pytorch3d/csrc/ext.cpp:53-56
    is for the reference) is built next to the library, loads on a CPU-only machine and exports the four ops of the path
    (+ the fused indexed pair); like a CUDA-less build of the reference it raises RuntimeError for CPU tensors."""
    import pytest
    import torch
    from pytorch3d_b200 import _C
    ext = _C._ext()
    for name in ("rasterize_meshes", "rasterize_meshes_backward", "rasterize_points", "rasterize_points_backward",
                 "rasterize_meshes_indexed", "rasterize_meshes_backward_indexed"):
        assert callable(getattr(ext, name))
    fv = torch.zeros(2, 3, 3)
    with pytest.raises(RuntimeError, match="must be a CUDA tensor"):
        ext.rasterize_meshes(fv, torch.zeros(1, dtype=torch.int64), torch.tensor([2]), None, (8, 8), 0.0, 2, 0, 0, False,
                             False, False)
    with pytest.raises(RuntimeError, match=r"face_verts must have dimensions \(num_faces, 3, 3\)"):
        ext.rasterize_meshes(torch.zeros(2, 3), torch.zeros(1, dtype=torch.int64), torch.tensor([2]), None, (8, 8), 0.0,
                             2, 0, 0, False, False, False)
    with pytest.raises(RuntimeError, match="Must have points_per_pixel <= 150"):
        ext.rasterize_meshes(fv, torch.zeros(1, dtype=torch.int64), torch.tensor([2]), None, (8, 8), 0.0, 151, 0, 0,
                             False, False, False)


def test_missing_torch_extension_raises_import_error(built_lib, monkeypatch, tmp_path):
    """The rasterizer ops have one binding: without the torch extension they fail loudly with the build command, and
    never fall back to another binding."""
    import pytest
    import torch
    from pytorch3d_b200 import _C, build
    monkeypatch.setattr(build, "ext_path", lambda: str(tmp_path / "missing_ext.so"))
    monkeypatch.setattr(_C, "_EXT", None)  # forget an extension loaded by an earlier test
    with pytest.raises(ImportError, match=r"python -m pytorch3d_b200\.build"):
        _C.rasterize_meshes(torch.zeros(2, 3, 3), torch.zeros(1, dtype=torch.int64), torch.tensor([2]),
                            torch.full((2,), -1), (8, 8), 0.0, 2, 0, 0, False, False, False)


def test_tagged_neighbour_tensor_is_still_checked(built_lib):
    """A clipped_faces_neighbor_idx tagged as all -1 only selects the kernel variant; the extension checks its length
    like that of an untagged one."""
    import pytest
    import torch
    from pytorch3d_b200 import _C
    z = torch.zeros(1, dtype=torch.int64)
    nb = torch.full((3,), -1, dtype=torch.int64)
    nb._b200_all_minus_one = True
    with pytest.raises(RuntimeError, match="clipped_faces_neighbor_idx must have save size first dimension"):
        _C.rasterize_meshes(torch.zeros(4, 3, 3), z, z, nb, (8, 8), 0.0, 1, 0, 0, False, False, False)
