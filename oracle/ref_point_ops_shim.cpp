// TEST INFRASTRUCTURE ONLY -- not part of the product path.
//
// pybind11 shim exposing the UNMODIFIED reference farthest point sampling and ball query ops (compiled from the
// sources where they lie under the reference tree by oracle/build_ref_point_ops.py), so that
// tests/golden/make_point_ops_golden.py can run the reference's own ops on the CPU and tests/test_point_ops.py can
// compare the fused kernels with the reference's CUDA kernels recompiled for sm_90a.  The declarations and the dispatch
// come from the reference's own headers
//   pytorch3d/csrc/sample_farthest_points/sample_farthest_points.h   (FarthestPointSampling)
//   pytorch3d/csrc/ball_query/ball_query.h                           (BallQuery)
// and the registration mirrors pytorch3d/csrc/ext.cpp (sample_farthest_points, ball_query).  The reference's CPU
// sources are compiled in this translation unit (included from where they lie, by the -I of the reference's csrc), so
// that the torch headers are parsed once per module.  Ball query's backward is knn_points_backward, which
// oracle/_ref/ref_knn_*.so (oracle/build_ref_knn.py) provides.
#include <torch/extension.h>
#include "ball_query/ball_query.h"
#include "ball_query/ball_query_cpu.cpp"
#include "sample_farthest_points/sample_farthest_points.h"
#include "sample_farthest_points/sample_farthest_points_cpu.cpp"

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.def("ball_query", &BallQuery);
  m.def("sample_farthest_points", &FarthestPointSampling);
#ifdef WITH_CUDA
  m.attr("with_cuda") = true;
#else
  m.attr("with_cuda") = false;
#endif
}
