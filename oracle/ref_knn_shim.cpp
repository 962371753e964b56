// TEST INFRASTRUCTURE ONLY -- not part of the product path.
//
// pybind11 shim exposing the UNMODIFIED reference k-nearest-neighbour op (compiled from the sources where they lie
// under the reference tree by oracle/build_ref_knn.py), so that tests/golden/make_chamfer_golden.py can run the
// reference's own chamfer_distance on the CPU and tests/test_chamfer.py can compare the fused search with the
// reference's CUDA kernel recompiled for sm_90a.  The declarations and the dispatch come from the reference's own
// header
//   pytorch3d/csrc/knn/knn.h   (KNearestNeighborIdx, KNearestNeighborBackward)
// and the registration mirrors pytorch3d/csrc/ext.cpp (knn_points_idx, knn_points_backward).  The reference's CPU
// source is compiled in this translation unit (included from where it lies, by the -I of the reference's csrc), so that
// the torch headers are parsed once per module.
#include <torch/extension.h>
#include "knn/knn.h"
#include "knn/knn_cpu.cpp"

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.def("knn_points_idx", &KNearestNeighborIdx);
  m.def("knn_points_backward", &KNearestNeighborBackward);
#ifdef WITH_CUDA
  m.attr("with_cuda") = true;
#else
  m.attr("with_cuda") = false;
#endif
}
