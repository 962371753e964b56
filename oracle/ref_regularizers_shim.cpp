// TEST INFRASTRUCTURE ONLY -- not part of the product path.
//
// pybind11 shim exposing the UNMODIFIED reference face-pair enumeration of mesh_normal_consistency (compiled from the
// source where it lies under the reference tree by oracle/build_ref_regularizers.py), so that
// tests/golden/make_regularizers_golden.py can run the reference's own loss on it and tools/time_regularizers.py can
// time the reference's chain.  The declaration and the dispatch come from the reference's own header
//   pytorch3d/csrc/mesh_normal_consistency/mesh_normal_consistency.h   (MeshNormalConsistencyFindVertices)
// and the registration mirrors pytorch3d/csrc/ext.cpp (mesh_normal_consistency_find_verts).
#include <torch/extension.h>
#include "mesh_normal_consistency/mesh_normal_consistency.h"

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.def("mesh_normal_consistency_find_verts", &MeshNormalConsistencyFindVertices);
}
