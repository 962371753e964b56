// TEST INFRASTRUCTURE ONLY -- not part of the product path.
//
// pybind11 shim exposing the UNMODIFIED reference face areas / normals op (compiled from the sources where they lie
// under the reference tree by oracle/build_ref_normals.py), so that tests/golden/make_normals_golden.py can run the
// reference's own Meshes on it and store the outputs.  The declarations and the dispatch come from the reference's own
// header
//   pytorch3d/csrc/face_areas_normals/face_areas_normals.h   (FaceAreasNormalsForward, FaceAreasNormalsBackward)
// and the registration mirrors pytorch3d/csrc/ext.cpp (face_areas_normals_forward, face_areas_normals_backward).
#include <torch/extension.h>
#include "face_areas_normals/face_areas_normals.h"

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.def("face_areas_normals_forward", &FaceAreasNormalsForward);
  m.def("face_areas_normals_backward", &FaceAreasNormalsBackward);
#ifdef WITH_CUDA
  m.attr("with_cuda") = true;
#else
  m.attr("with_cuda") = false;
#endif
}
