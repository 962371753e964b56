// TEST INFRASTRUCTURE ONLY -- not part of the product path.
//
// pybind11 shim exposing the UNMODIFIED reference blending ops (compiled from the sources where they lie under the
// reference tree by oracle/build_ref_blend.py), so that tests/golden/make_blend_golden.py can store their outputs.
// The declarations and the dispatch come from the reference's own header
//   pytorch3d/csrc/blending/sigmoid_alpha_blend.h   (SigmoidAlphaBlend, SigmoidAlphaBlendBackward)
// and the registration mirrors pytorch3d/csrc/ext.cpp (sigmoid_alpha_blend, sigmoid_alpha_blend_backward).
#include <torch/extension.h>
#include "utils/pytorch3d_cutils.h"  // CHECK_CPU, used by the header below (ext.cpp includes it first as well)
#include "blending/sigmoid_alpha_blend.h"

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.def("sigmoid_alpha_blend", &SigmoidAlphaBlend);
  m.def("sigmoid_alpha_blend_backward", &SigmoidAlphaBlendBackward);
#ifdef WITH_CUDA
  m.attr("with_cuda") = true;
#else
  m.attr("with_cuda") = false;
#endif
}
