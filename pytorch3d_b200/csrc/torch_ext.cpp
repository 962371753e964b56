// torch C++ extension over the C ABI of libb200raster.so: the binding the reference itself uses for this path
// (pybind11 module built with torch.utils.cpp_extension, pytorch3d/csrc/ext.cpp:34,53-56).  Same op names, positional
// arguments, return values and error texts as RasterizeMeshes / RasterizeMeshesBackward / RasterizePoints /
// RasterizePointsBackward (rasterize_meshes.h:513-562, 211-218; rasterize_points.h:343-374, 281-285).  This file
// contains no kernel and no CPU path: it checks arguments, allocates the outputs and the scratch workspace from
// torch's caching allocator, takes the current CUDA stream and calls include/b200_raster.h.
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include <tuple>

#include "../../include/b200_raster.h"

namespace {

constexpr int kMaxPointsPerPixel = 150;  // rasterization_utils.cuh:48

void check_status(int rc) {
  if (rc != B200R_OK) {
    const char* msg = b200r_last_error();
    TORCH_CHECK(false, (msg && *msg) ? msg : "libb200raster error");
  }
}

void require_cuda(const at::Tensor& t, const char* name) {
  TORCH_CHECK(t.is_cuda(), name,
              " must be a CUDA tensor: pytorch3d_b200 is an H100-native (sm_90a) rasterizer and has no CPU "
              "implementation.");
}

void require_same_device(const at::Tensor& a, const at::Tensor& b, const char* name) {
  TORCH_CHECK(a.device() == b.device(), "Expected all tensors to be on the same device (", name, " is on ", b.device(),
              ", expected ", a.device(), ")");
}

int64_t* i64_or_null(const at::Tensor& t) { return t.numel() > 0 ? t.data_ptr<int64_t>() : nullptr; }
float* f32_or_null(const at::Tensor& t) { return t.numel() > 0 ? t.data_ptr<float>() : nullptr; }

void check_not_deterministic(const char* what) {
  // same non-determinism contract as the reference (rasterize_meshes.cu:587, rasterize_points.cu:428)
  if (at::globalContext().deterministicAlgorithms() && !at::globalContext().deterministicAlgorithmsWarnOnly())
    TORCH_CHECK(false, what, " does not have a deterministic implementation, but you set "
                             "'torch.use_deterministic_algorithms(True)'.");
}

// ---------------------------------------------------------------------------------------------- meshes

std::tuple<at::Tensor, at::Tensor, at::Tensor, at::Tensor> rasterize_meshes(
    const at::Tensor& face_verts, const at::Tensor& mesh_to_face_first_idx, const at::Tensor& num_faces_per_mesh,
    const c10::optional<at::Tensor>& clipped_faces_neighbor_idx, const std::tuple<int, int> image_size,
    const double blur_radius, const int64_t faces_per_pixel, const int64_t bin_size, const int64_t max_faces_per_bin,
    const bool perspective_correct, const bool clip_barycentric_coords, const bool cull_backfaces,
    const int64_t pair_capacity, const bool neighbors_all_minus_one) {
  TORCH_CHECK(face_verts.dim() == 3 && face_verts.size(1) == 3 && face_verts.size(2) == 3,
              "face_verts must have dimensions (num_faces, 3, 3)");
  TORCH_CHECK(num_faces_per_mesh.size(0) == mesh_to_face_first_idx.size(0),
              "num_faces_per_mesh must have save size first dimension as mesh_to_faces_packed_first_idx");
  if (clipped_faces_neighbor_idx.has_value())
    TORCH_CHECK(clipped_faces_neighbor_idx->size(0) == face_verts.size(0),
                "clipped_faces_neighbor_idx must have save size first dimension as face_verts");
  TORCH_CHECK(faces_per_pixel <= kMaxPointsPerPixel, "Must have points_per_pixel <= ", kMaxPointsPerPixel);
  TORCH_CHECK(face_verts.scalar_type() == at::kFloat, "expected scalar type Float but found ",
              face_verts.scalar_type());
  require_cuda(face_verts, "face_verts");
  require_cuda(mesh_to_face_first_idx, "mesh_to_faces_packed_first_idx");
  require_cuda(num_faces_per_mesh, "num_faces_per_mesh");
  require_same_device(face_verts, mesh_to_face_first_idx, "mesh_to_faces_packed_first_idx");
  require_same_device(face_verts, num_faces_per_mesh, "num_faces_per_mesh");
  if (clipped_faces_neighbor_idx.has_value()) {
    require_cuda(*clipped_faces_neighbor_idx, "clipped_faces_neighbor_idx");
    require_same_device(face_verts, *clipped_faces_neighbor_idx, "clipped_faces_neighbor_idx");
  }
  c10::cuda::CUDAGuard guard(face_verts.device());
  cudaStream_t stream = at::cuda::getCurrentCUDAStream();
  const int H = std::get<0>(image_size), W = std::get<1>(image_size);
  const int64_t N = num_faces_per_mesh.size(0), F = face_verts.size(0), K = faces_per_pixel;
  const at::Tensor fv = face_verts.contiguous();
  const at::Tensor first = mesh_to_face_first_idx.contiguous().to(at::kLong);
  const at::Tensor num = num_faces_per_mesh.contiguous().to(at::kLong);
  // A neighbour tensor the caller knows to be all -1 is checked like any other but not passed on: NULL selects the
  // kernel variant without the clipped-face neighbour logic.
  at::Tensor nb;
  if (clipped_faces_neighbor_idx.has_value() && !neighbors_all_minus_one && F > 0)
    nb = clipped_faces_neighbor_idx->contiguous().to(at::kLong);
  const auto fopt = fv.options();
  at::Tensor pix_to_face = at::empty({N, H, W, K}, fopt.dtype(at::kLong));
  at::Tensor zbuf = at::empty({N, H, W, K}, fopt);
  at::Tensor bary = at::empty({N, H, W, K, 3}, fopt);
  at::Tensor dists = at::empty({N, H, W, K}, fopt);
  if (pix_to_face.numel() == 0) return std::make_tuple(pix_to_face, zbuf, bary, dists);
  const size_t ws_bytes = b200r_rasterize_meshes_workspace_bytes(F, (int32_t)N, H, W, pair_capacity);
  at::Tensor ws = at::empty({(int64_t)ws_bytes}, fopt.dtype(at::kByte));
  check_status(b200r_rasterize_meshes_forward(
      f32_or_null(fv), F, i64_or_null(first), i64_or_null(num), nb.defined() ? i64_or_null(nb) : nullptr, (int32_t)N, H,
      W, (float)blur_radius, (int32_t)K, (int32_t)bin_size, (int32_t)max_faces_per_bin, perspective_correct,
      clip_barycentric_coords, cull_backfaces, pix_to_face.data_ptr<int64_t>(), zbuf.data_ptr<float>(),
      bary.data_ptr<float>(), dists.data_ptr<float>(), ws.data_ptr(), ws_bytes, pair_capacity, stream));
  // (the workspace is only used by kernels already enqueued on `stream`, the stream it was allocated on)
  return std::make_tuple(pix_to_face, zbuf, bary, dists);
}

void check_backward_inputs(const at::Tensor& face_verts, const at::Tensor& pix_to_face, const at::Tensor& grad_zbuf,
                           const at::Tensor& grad_bary, const at::Tensor& grad_dists) {
  const at::Tensor* ts[] = {&face_verts, &pix_to_face, &grad_zbuf, &grad_bary, &grad_dists};
  const char* names[] = {"face_verts", "pix_to_face", "grad_zbuf", "grad_bary", "grad_dists"};
  for (int i = 0; i < 5; ++i) {
    require_cuda(*ts[i], names[i]);
    require_same_device(face_verts, *ts[i], names[i]);
    if (i != 1)
      TORCH_CHECK(ts[i]->scalar_type() == at::kFloat, "Expected tensor for ", names[i],
                  " to have scalar type Float; but got ", ts[i]->scalar_type());
  }
  TORCH_CHECK(pix_to_face.scalar_type() == at::kLong, "expected scalar type Long but found ",
              pix_to_face.scalar_type());
  TORCH_CHECK(pix_to_face.dim() == 4, "pix_to_face must have dimensions (N, H, W, K)");
  check_not_deterministic("RasterizeMeshesBackwardCuda");
}

at::Tensor rasterize_meshes_backward(const at::Tensor& face_verts, const at::Tensor& pix_to_face,
                                     const at::Tensor& grad_zbuf, const at::Tensor& grad_bary,
                                     const at::Tensor& grad_dists, const bool perspective_correct,
                                     const bool clip_barycentric_coords) {
  check_backward_inputs(face_verts, pix_to_face, grad_zbuf, grad_bary, grad_dists);
  c10::cuda::CUDAGuard guard(face_verts.device());
  cudaStream_t stream = at::cuda::getCurrentCUDAStream();
  const int64_t F = face_verts.size(0);
  const at::Tensor fv = face_verts.contiguous(), p2f = pix_to_face.contiguous();
  const at::Tensor gz = grad_zbuf.contiguous(), gb = grad_bary.contiguous(), gd = grad_dists.contiguous();
  at::Tensor grad_face_verts = at::empty({F, 3, 3}, fv.options());
  if (F == 0) return grad_face_verts;
  check_status(b200r_rasterize_meshes_backward(
      fv.data_ptr<float>(), F, i64_or_null(p2f), f32_or_null(gz), f32_or_null(gb), f32_or_null(gd),
      (int32_t)p2f.size(0), (int32_t)p2f.size(1), (int32_t)p2f.size(2), (int32_t)p2f.size(3), perspective_correct,
      clip_barycentric_coords, grad_face_verts.data_ptr<float>(), stream));
  return grad_face_verts;
}

// fused `rasterize_meshes(verts_packed[faces_packed], ...)` (no counterpart in pytorch3d._C; SURVEY.md 8 f-4)
std::tuple<at::Tensor, at::Tensor, at::Tensor, at::Tensor, at::Tensor> rasterize_meshes_indexed(
    const at::Tensor& verts_packed, const at::Tensor& faces_packed, const at::Tensor& mesh_to_face_first_idx,
    const at::Tensor& num_faces_per_mesh, const std::tuple<int, int> image_size, const double blur_radius,
    const int64_t faces_per_pixel, const bool perspective_correct, const bool clip_barycentric_coords,
    const bool cull_backfaces, const int64_t pair_capacity) {
  TORCH_CHECK(verts_packed.dim() == 2 && verts_packed.size(1) == 3, "verts_packed must have dimensions (num_verts, 3)");
  TORCH_CHECK(faces_packed.dim() == 2 && faces_packed.size(1) == 3, "faces_packed must have dimensions (num_faces, 3)");
  TORCH_CHECK(num_faces_per_mesh.size(0) == mesh_to_face_first_idx.size(0),
              "num_faces_per_mesh must have save size first dimension as mesh_to_faces_packed_first_idx");
  TORCH_CHECK(faces_per_pixel <= kMaxPointsPerPixel, "Must have points_per_pixel <= ", kMaxPointsPerPixel);
  TORCH_CHECK(verts_packed.scalar_type() == at::kFloat, "expected scalar type Float but found ",
              verts_packed.scalar_type());
  require_cuda(verts_packed, "verts_packed");
  require_cuda(faces_packed, "faces_packed");
  require_cuda(mesh_to_face_first_idx, "mesh_to_faces_packed_first_idx");
  require_cuda(num_faces_per_mesh, "num_faces_per_mesh");
  require_same_device(verts_packed, faces_packed, "faces_packed");
  require_same_device(verts_packed, mesh_to_face_first_idx, "mesh_to_faces_packed_first_idx");
  require_same_device(verts_packed, num_faces_per_mesh, "num_faces_per_mesh");
  c10::cuda::CUDAGuard guard(verts_packed.device());
  cudaStream_t stream = at::cuda::getCurrentCUDAStream();
  const int H = std::get<0>(image_size), W = std::get<1>(image_size);
  const int64_t N = num_faces_per_mesh.size(0), F = faces_packed.size(0), V = verts_packed.size(0), K = faces_per_pixel;
  const at::Tensor verts = verts_packed.contiguous(), faces = faces_packed.contiguous().to(at::kLong);
  const at::Tensor first = mesh_to_face_first_idx.contiguous().to(at::kLong);
  const at::Tensor num = num_faces_per_mesh.contiguous().to(at::kLong);
  const auto fopt = verts.options();
  at::Tensor pix_to_face = at::empty({N, H, W, K}, fopt.dtype(at::kLong));
  at::Tensor zbuf = at::empty({N, H, W, K}, fopt);
  at::Tensor bary = at::empty({N, H, W, K, 3}, fopt);
  at::Tensor dists = at::empty({N, H, W, K}, fopt);
  at::Tensor face_verts = at::empty({F, 3, 3}, fopt);
  const size_t ws_bytes = b200r_rasterize_meshes_workspace_bytes(F, (int32_t)N, H, W, pair_capacity);
  at::Tensor ws = at::empty({(int64_t)ws_bytes}, fopt.dtype(at::kByte));
  check_status(b200r_rasterize_meshes_forward_indexed(
      f32_or_null(verts), V, i64_or_null(faces), F, i64_or_null(first), i64_or_null(num), nullptr, (int32_t)N, H, W,
      (float)blur_radius, (int32_t)K, perspective_correct, clip_barycentric_coords, cull_backfaces,
      pix_to_face.numel() > 0 ? pix_to_face.data_ptr<int64_t>() : nullptr, f32_or_null(zbuf), f32_or_null(bary),
      f32_or_null(dists), f32_or_null(face_verts), ws.data_ptr(), ws_bytes, pair_capacity, stream));
  return std::make_tuple(pix_to_face, zbuf, bary, dists, face_verts);
}

at::Tensor rasterize_meshes_backward_indexed(const at::Tensor& face_verts, const at::Tensor& faces_packed,
                                             const int64_t num_verts, const at::Tensor& pix_to_face,
                                             const at::Tensor& grad_zbuf, const at::Tensor& grad_bary,
                                             const at::Tensor& grad_dists, const bool perspective_correct,
                                             const bool clip_barycentric_coords) {
  check_backward_inputs(face_verts, pix_to_face, grad_zbuf, grad_bary, grad_dists);
  require_cuda(faces_packed, "faces_packed");
  require_same_device(face_verts, faces_packed, "faces_packed");
  c10::cuda::CUDAGuard guard(face_verts.device());
  cudaStream_t stream = at::cuda::getCurrentCUDAStream();
  const int64_t F = face_verts.size(0), V = num_verts;
  const at::Tensor fv = face_verts.contiguous(), faces = faces_packed.contiguous().to(at::kLong);
  const at::Tensor p2f = pix_to_face.contiguous();
  const at::Tensor gz = grad_zbuf.contiguous(), gb = grad_bary.contiguous(), gd = grad_dists.contiguous();
  at::Tensor grad_verts = at::empty({V, 3}, fv.options());
  check_status(b200r_rasterize_meshes_backward_indexed(
      f32_or_null(fv), i64_or_null(faces), F, V, i64_or_null(p2f), f32_or_null(gz), f32_or_null(gb), f32_or_null(gd),
      (int32_t)p2f.size(0), (int32_t)p2f.size(1), (int32_t)p2f.size(2), (int32_t)p2f.size(3), perspective_correct,
      clip_barycentric_coords, f32_or_null(grad_verts), stream));
  return grad_verts;
}

// ---------------------------------------------------------------------------------------------- points

std::tuple<at::Tensor, at::Tensor, at::Tensor> rasterize_points(
    const at::Tensor& points, const at::Tensor& cloud_to_packed_first_idx, const at::Tensor& num_points_per_cloud,
    const std::tuple<int, int> image_size, const at::Tensor& radius, const int64_t points_per_pixel,
    const int64_t bin_size, const int64_t max_points_per_bin, const int64_t pair_capacity) {
  TORCH_CHECK(points.dim() == 2 && points.size(1) == 3, "points must have dimensions (num_points, 3)");
  TORCH_CHECK(num_points_per_cloud.size(0) == cloud_to_packed_first_idx.size(0),
              "num_points_per_cloud must have same size first dimension as cloud_to_packed_first_idx");
  TORCH_CHECK(radius.dim() == 1 && radius.size(0) == points.size(0), "radius must be of shape (P,)");
  TORCH_CHECK(points_per_pixel <= kMaxPointsPerPixel, "Must have num_closest <= ", kMaxPointsPerPixel);
  TORCH_CHECK(points.scalar_type() == at::kFloat && radius.scalar_type() == at::kFloat, "expected scalar type Float");
  require_cuda(points, "points");
  require_cuda(cloud_to_packed_first_idx, "cloud_to_packed_first_idx");
  require_cuda(num_points_per_cloud, "num_points_per_cloud");
  require_cuda(radius, "radius");
  require_same_device(points, cloud_to_packed_first_idx, "cloud_to_packed_first_idx");
  require_same_device(points, num_points_per_cloud, "num_points_per_cloud");
  require_same_device(points, radius, "radius");
  c10::cuda::CUDAGuard guard(points.device());
  cudaStream_t stream = at::cuda::getCurrentCUDAStream();
  const int H = std::get<0>(image_size), W = std::get<1>(image_size);
  const int64_t N = num_points_per_cloud.size(0), P = points.size(0), K = points_per_pixel;
  const at::Tensor pts = points.contiguous(), rad = radius.contiguous();
  const at::Tensor first = cloud_to_packed_first_idx.contiguous().to(at::kLong);
  const at::Tensor num = num_points_per_cloud.contiguous().to(at::kLong);
  const auto fopt = pts.options();
  at::Tensor idx = at::empty({N, H, W, K}, fopt.dtype(at::kInt));
  at::Tensor zbuf = at::empty({N, H, W, K}, fopt);
  at::Tensor dists = at::empty({N, H, W, K}, fopt);
  if (idx.numel() == 0) return std::make_tuple(idx, zbuf, dists);
  const size_t ws_bytes = b200r_rasterize_points_workspace_bytes(P, (int32_t)N, H, W, pair_capacity);
  at::Tensor ws = at::empty({(int64_t)ws_bytes}, fopt.dtype(at::kByte));
  check_status(b200r_rasterize_points_forward(f32_or_null(pts), P, i64_or_null(first), i64_or_null(num),
                                              f32_or_null(rad), (int32_t)N, H, W, (int32_t)K, (int32_t)bin_size,
                                              (int32_t)max_points_per_bin, idx.data_ptr<int32_t>(),
                                              zbuf.data_ptr<float>(), dists.data_ptr<float>(), ws.data_ptr(), ws_bytes,
                                              pair_capacity, stream));
  return std::make_tuple(idx, zbuf, dists);
}

at::Tensor rasterize_points_backward(const at::Tensor& points, const at::Tensor& idxs, const at::Tensor& grad_zbuf,
                                     const at::Tensor& grad_dists) {
  require_cuda(points, "points");
  require_cuda(idxs, "idxs");
  require_cuda(grad_zbuf, "grad_zbuf");
  require_cuda(grad_dists, "grad_dists");
  require_same_device(points, idxs, "idxs");
  require_same_device(points, grad_zbuf, "grad_zbuf");
  require_same_device(points, grad_dists, "grad_dists");
  TORCH_CHECK(idxs.scalar_type() == at::kInt, "expected scalar type Int but found ", idxs.scalar_type());
  TORCH_CHECK(idxs.dim() == 4, "idxs must have dimensions (N, H, W, K)");
  check_not_deterministic("RasterizePointsBackwardCuda");
  c10::cuda::CUDAGuard guard(points.device());
  cudaStream_t stream = at::cuda::getCurrentCUDAStream();
  const int64_t P = points.size(0);
  const at::Tensor pts = points.contiguous(), idx = idxs.contiguous();
  const at::Tensor gz = grad_zbuf.contiguous(), gd = grad_dists.contiguous();
  at::Tensor grad_points = at::empty({P, 3}, pts.options());
  if (P == 0) return grad_points;
  check_status(b200r_rasterize_points_backward(pts.data_ptr<float>(), P, idx.numel() > 0 ? idx.data_ptr<int32_t>() : nullptr,
                                               f32_or_null(gz), f32_or_null(gd), (int32_t)idx.size(0),
                                               (int32_t)idx.size(1), (int32_t)idx.size(2), (int32_t)idx.size(3),
                                               grad_points.data_ptr<float>(), stream));
  return grad_points;
}

}  // namespace

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.doc() = "torch C++ extension over libb200raster.so (include/b200_raster.h); mirrors pytorch3d/csrc/ext.cpp:53-56";
  m.def("rasterize_meshes", &rasterize_meshes, py::arg("face_verts"), py::arg("mesh_to_face_first_idx"),
        py::arg("num_faces_per_mesh"), py::arg("clipped_faces_neighbor_idx"), py::arg("image_size"),
        py::arg("blur_radius"), py::arg("faces_per_pixel"), py::arg("bin_size"), py::arg("max_faces_per_bin"),
        py::arg("perspective_correct"), py::arg("clip_barycentric_coords"), py::arg("cull_backfaces"),
        py::arg("pair_capacity") = 0, py::arg("neighbors_all_minus_one") = false);
  m.def("rasterize_meshes_backward", &rasterize_meshes_backward);
  m.def("rasterize_meshes_indexed", &rasterize_meshes_indexed, py::arg("verts_packed"), py::arg("faces_packed"),
        py::arg("mesh_to_face_first_idx"), py::arg("num_faces_per_mesh"), py::arg("image_size"),
        py::arg("blur_radius"), py::arg("faces_per_pixel"), py::arg("perspective_correct"),
        py::arg("clip_barycentric_coords"), py::arg("cull_backfaces"), py::arg("pair_capacity") = 0);
  m.def("rasterize_meshes_backward_indexed", &rasterize_meshes_backward_indexed);
  m.def("rasterize_points", &rasterize_points, py::arg("points"), py::arg("cloud_to_packed_first_idx"),
        py::arg("num_points_per_cloud"), py::arg("image_size"), py::arg("radius"), py::arg("points_per_pixel"),
        py::arg("bin_size"), py::arg("max_points_per_bin"), py::arg("pair_capacity") = 0);
  m.def("rasterize_points_backward", &rasterize_points_backward);
}
