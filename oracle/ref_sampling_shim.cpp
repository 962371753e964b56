// TEST INFRASTRUCTURE ONLY -- not part of the product path.
//
// pybind11 shim exposing the UNMODIFIED reference packed-to-padded op (compiled from the source where it lies under
// the reference tree by oracle/build_ref_sampling.py), so that tests/golden/make_sampling_golden.py can run the
// reference's own sample_points_from_meshes on the CPU; its face areas come from oracle/_ref/ref_normals_cpu.so.  The
// declarations and the dispatch come from the reference's own header
//   pytorch3d/csrc/packed_to_padded_tensor/packed_to_padded_tensor.h   (PackedToPadded, PaddedToPacked)
// and the registration mirrors pytorch3d/csrc/ext.cpp.  The reference's CPU source is compiled in this translation unit
// (included from where it lies, by the -I of the reference's csrc), so that the torch headers are parsed once.
#include <torch/extension.h>
#include "packed_to_padded_tensor/packed_to_padded_tensor.h"
#include "packed_to_padded_tensor/packed_to_padded_tensor_cpu.cpp"

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.def("packed_to_padded", &PackedToPadded);
  m.def("padded_to_packed", &PaddedToPacked);
}
