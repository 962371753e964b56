// Mesh normals: vertex normals and face areas / normals, forward and deterministic backward (DESIGN.md section 17).
//
// Both ops rest on one structure, the vertex -> corner table (mesh_tables.cuh, keyed_runs.cuh).  Corner j of face f has the id
// c = j * F + f and the key faces[f, j]; a stable radix sort of the 3F (key, id) pairs over ceil(log2(V + 1)) key bits,
// and an offset array of V + 1 entries, give every vertex the run of its corners in (j, f) order.  That is the order in
// which the three serial index_add calls of pytorch3d/structures/meshes.py Meshes._compute_vertex_normals accumulate on
// the CPU.  Every per-vertex sum is one thread walking its run from +0 with __fadd_rn (segmented_sum_kernel, shared by
// both ops), so there are no float atomics and the results do not depend on scheduling.  Nothing synchronises the
// host, and the workspace depends only on (V, F).
//
// Vertex normals (Meshes._compute_vertex_normals, restated with explicit rounding):
//   n_f = (v2 - v1) x (v0 - v1), each component fma(a_i, b_j, -rn(a_j * b_i)) with a = v2 - v1, b = v0 - v1
//   s_v = the sum of n_f over the corners of v, in (j, f) order from +0
//   out = s_v / max(|s_v|, 1e-6), |s| = sqrt_rn(fma(z, z, fma(y, y, rn(x * x)))), an IEEE divide
// The backward is autograd's through F.normalize (x / clamp_min(norm, eps)), the cross product and the two
// subtractions, with the per-corner gradients summed per vertex over the forward's table.
//
// Face areas and normals (pytorch3d/csrc/face_areas_normals/face_areas_normals.cu): the forward restates
// FaceAreasNormalsForwardKernel<float> as nvcc compiles it for sm_90a (its FMA contraction, the double compare against
// 1e-6, norm / 2.0), so the results are bit-identical.  The backward writes the reference's nine per-corner expressions,
// in its arithmetic, to an (F, 3, 3) workspace, and sums them per vertex over a table built in the same call instead of
// adding them with float atomics.
#include "mesh_tables.cuh"

namespace b200r {
namespace {

// ---- vertex normals -----------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(kThreads)
    face_normal_rows_kernel(const float* __restrict__ verts, const int64_t* __restrict__ faces, int64_t V, int64_t F,
                            float* __restrict__ rows) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; f < F; f += stride) {
    float3 p[3];
    face_corners(verts, faces, V, f, p);
    store3(rows, f, cross_fma(sub_rn(p[2], p[1]), sub_rn(p[0], p[1])));
  }
}

// d loss / d s for y = s / clamp_min(|s|, 1e-6) (mesh_tables.cuh normalize_backward).
__global__ void __launch_bounds__(kThreads)
    normalize_backward_kernel(const float* __restrict__ grad_normals, const float* __restrict__ sums, int64_t V,
                              float* __restrict__ grad_sums) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < V; v += stride)
    store3(grad_sums, v, normalize_backward(load3(sums, v), load3(grad_normals, v), kNormalizeEps));
}

// Per face: the gradient of n_f (the sum of grad_sums over its three corners), through the cross product and the two
// subtractions, as rows (f, j) = d loss / d corner j.
__global__ void __launch_bounds__(kThreads)
    cross_backward_rows_kernel(const float* __restrict__ verts, const int64_t* __restrict__ faces, int64_t V,
                               int64_t F, const float* __restrict__ grad_sums, float* __restrict__ rows) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; f < F; f += stride) {
    float3 p[3];
    face_corners(verts, faces, V, f, p);
    float3 gs = make_float3(0.0f, 0.0f, 0.0f);
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      const int64_t v = __ldg(faces + 3 * f + j);
      const float3 g = (v >= 0 && v < V) ? load3(grad_sums, v) : make_float3(0.0f, 0.0f, 0.0f);
      gs = make_float3(__fadd_rn(gs.x, g.x), __fadd_rn(gs.y, g.y), __fadd_rn(gs.z, g.z));
    }
    const float3 a = sub_rn(p[2], p[1]), b = sub_rn(p[0], p[1]);
    const float3 ga = cross_fma(b, gs);  // cross(a, b) backward: a gets b x g, b gets g x a
    const float3 gb = cross_fma(gs, a);
    store3(rows, f * 3 + 0, gb);
    store3(rows, f * 3 + 1,
           make_float3(__fsub_rn(-ga.x, gb.x), __fsub_rn(-ga.y, gb.y), __fsub_rn(-ga.z, gb.z)));
    store3(rows, f * 3 + 2, ga);
  }
}

// ---- face areas and normals ---------------------------------------------------------------------------------------

// FaceAreasNormalsForwardKernel<float> as nvcc compiles it for sm_90a: the cross product, norm and area of
// face_cross_norm (mesh_tables.cuh).  The clamp compares in double (NaN passes) and clamps to (float)1e-6; the normal is
// an IEEE divide.
__global__ void __launch_bounds__(kThreads)
    face_areas_normals_forward_kernel(const float* __restrict__ verts, const int64_t* __restrict__ faces, int64_t V,
                                      int64_t F, float* __restrict__ areas, float* __restrict__ normals) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; f < F; f += stride) {
    float3 p[3], c;
    face_corners(verts, faces, V, f, p);
    float norm = face_cross_norm(p, c);
    areas[f] = __fmul_rn(norm, 0.5f);
    norm = ((double)norm < 1e-6) ? (float)1e-6 : norm;
    store3(normals, f, make_float3(__fdiv_rn(c.x, norm), __fdiv_rn(c.y, norm), __fdiv_rn(c.z, norm)));
  }
}

// The reference backward's per-corner expressions (FaceAreasNormalsBackwardKernel), in its arithmetic: float
// products, the area term divided by 2.0 in double, pow() for the inverse norm's powers, and the sum of the four terms
// rounded to float once.  Row (f, j) = the gradient of corner j.
__global__ void __launch_bounds__(kThreads)
    face_areas_normals_backward_rows_kernel(const float* __restrict__ grad_areas,
                                            const float* __restrict__ grad_normals, const float* __restrict__ verts,
                                            const int64_t* __restrict__ faces, int64_t V, int64_t F,
                                            float* __restrict__ rows) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; f < F; f += stride) {
    float3 p[3];
    face_corners(verts, faces, V, f, p);
    const float ax = p[1].x - p[0].x, ay = p[1].y - p[0].y, az = p[1].z - p[0].z;
    const float bx = p[2].x - p[0].x, by = p[2].y - p[0].y, bz = p[2].z - p[0].z;
    const float cx = ay * bz - az * by;
    const float cy = az * bx - ax * bz;
    const float cz = ax * by - ay * bx;
    float norm = sqrtf(cx * cx + cy * cy + cz * cz);
    norm = (norm < 1e-6) ? 1e-6 : norm;
    const float inv = 1. / norm;
    const float inv2 = powf(inv, 2.0f);
    const float inv3 = powf(inv, 3.0f);
    const float ga = __ldg(grad_areas + f);
    const float g0 = __ldg(grad_normals + 3 * f + 0), g1 = __ldg(grad_normals + 3 * f + 1),
                g2 = __ldg(grad_normals + 3 * f + 2);
    // t is d(c)/d(coordinate) . c; each component's gradient is
    //   t / 2.0 * inv * ga + sum_k (term of normal component k)
    // where the component of c that the coordinate does not move gets -c_k * t * inv3 * g_k and the other two
    // (d_k - c_k * t * inv2) * inv * g_k, each written out as the reference writes it.
    float* r = rows + 9 * f;
    float t;
    // corner 0
    t = (-az + bz) * cy + (-by + ay) * cz;
    r[0] = t / 2.0 * inv * ga + -cx * t * inv3 * g0 + ((-az + bz) - cy * t * inv2) * inv * g1 +
           ((-by + ay) - cz * t * inv2) * inv * g2;
    t = (-bz + az) * cx + (-ax + bx) * cz;
    r[1] = t / 2.0 * inv * ga + ((-bz + az) - cx * t * inv2) * inv * g0 + -cy * t * inv3 * g1 +
           ((-ax + bx) - cz * t * inv2) * inv * g2;
    t = (-ay + by) * cx + (-bx + ax) * cy;
    r[2] = t / 2.0 * inv * ga + ((-ay + by) - cx * t * inv2) * inv * g0 + ((-bx + ax) - cy * t * inv2) * inv * g1 +
           -cz * t * inv3 * g2;
    // corner 1
    t = by * cz - bz * cy;
    r[3] = t / 2.0 * inv * ga + -cx * t * inv3 * g0 + (-bz - cy * t * inv2) * inv * g1 + (by - cz * t * inv2) * inv * g2;
    t = bz * cx - bx * cz;
    r[4] = t / 2.0 * inv * ga + (bz - cx * t * inv2) * inv * g0 + -cy * t * inv3 * g1 + (-bx - cz * t * inv2) * inv * g2;
    t = bx * cy - by * cx;
    // the reference multiplies the second normal component's term by cx, not cy; kept, the records depend on it
    r[5] = t / 2.0 * inv * ga + (-by - cx * t * inv2) * inv * g0 + (bx - cx * t * inv2) * inv * g1 + -cz * t * inv3 * g2;
    // corner 2
    t = az * cy - ay * cz;
    r[6] = t / 2.0 * inv * ga + -cx * t * inv3 * g0 + (az - cy * t * inv2) * inv * g1 + (-ay - cz * t * inv2) * inv * g2;
    t = ax * cz - az * cx;
    r[7] = t / 2.0 * inv * ga + (-az - cx * t * inv2) * inv * g0 + -cy * t * inv3 * g1 + (ax - cz * t * inv2) * inv * g2;
    t = ay * cx - ax * cy;
    r[8] = t / 2.0 * inv * ga + (ay - cx * t * inv2) * inv * g0 + (-ax - cy * t * inv2) * inv * g1 + -cz * t * inv3 * g2;
  }
}

// ---- host side ----------------------------------------------------------------------------------------------------

// Workspace: rows (9F floats), a table (V + 1 + 3F ints), keys in / out and ids (3F each), then cub's temporary
// storage.  Returns false when cub cannot size its storage (no device).
struct Layout {
  size_t rows, table, keys_in, keys_out, ids_in, cub, cub_bytes, total;
};

bool layout(int64_t V, int64_t F, Layout& L) {
  const size_t n = 3 * (size_t)F;
  Carver c;
  L.rows = c.take(sizeof(float) * 9 * (size_t)F);
  L.table = c.take(sizeof(int32_t) * ((size_t)V + 1 + n));
  L.keys_in = c.take(sizeof(uint32_t) * n);
  L.keys_out = c.take(sizeof(uint32_t) * n);
  L.ids_in = c.take(sizeof(int32_t) * n);
  const bool sized = run_sort_bytes(V, (int64_t)n, L.cub_bytes);
  L.cub = c.take(L.cub_bytes);
  L.total = c.used;
  return sized;
}

int check_sizes(const char* op, int64_t V, int64_t F) {
  if (V < 0 || F < 0) return fail(B200R_ERR_INVALID_ARGUMENT, std::string(op) + ": negative size");
  if (V >= ((int64_t)1 << 31) - 1)
    return fail(B200R_ERR_INVALID_ARGUMENT, std::string(op) + ": at most 2^31 - 2 vertices");
  if (3 * F >= ((int64_t)1 << 31))
    return fail(B200R_ERR_INVALID_ARGUMENT, std::string(op) + ": at most (2^31 - 1) / 3 faces (3F < 2^31 corners)");
  return B200R_OK;
}

int checked_layout(const char* op, int64_t V, int64_t F, size_t workspace_bytes, const void* workspace, Layout& L) {
  const bool sized = layout(V, F, L);
  return check_workspace(op, "b200r_normals_workspace_bytes", sized, L.total, workspace, workspace_bytes);
}

// Builds the table (offsets[V + 1], then the 3F corner ids in run order) at `table`.
int build_table(const int64_t* faces, int64_t V, int64_t F, char* ws, const Layout& L, int32_t* table,
                cudaStream_t stream) {
  return build_table(faces, V, F, reinterpret_cast<uint32_t*>(ws + L.keys_in),
                     reinterpret_cast<uint32_t*>(ws + L.keys_out), reinterpret_cast<int32_t*>(ws + L.ids_in),
                     ws + L.cub, L.cub_bytes, table, stream);
}

}  // namespace
}  // namespace b200r

using namespace b200r;

extern "C" size_t b200r_normals_workspace_bytes(int64_t V, int64_t F) {
  if (V < 0 || F < 0) return 0;
  Layout L;
  const bool sized = layout(V, F, L);
  return workspace_size(sized, L.total);
}

extern "C" int b200r_verts_normals_forward(const float* verts, int64_t V, const int64_t* faces, int64_t F,
                                           void* workspace, size_t workspace_bytes, int32_t* table, float* sums,
                                           float* normals, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int rc = check_sizes("verts_normals_forward", V, F);
  if (rc != B200R_OK) return rc;
  if (V == 0) return B200R_OK;
  Layout L;
  rc = checked_layout("verts_normals_forward", V, F, workspace_bytes, workspace, L);
  if (rc != B200R_OK) return rc;
  char* ws = static_cast<char*>(workspace);
  float* rows = reinterpret_cast<float*>(ws + L.rows);
  rc = build_table(faces, V, F, ws, L, table, stream);
  if (rc != B200R_OK) return rc;
  if (F > 0) {
    face_normal_rows_kernel<<<grid_for(F), kThreads, 0, stream>>>(verts, faces, V, F, rows);
    B200R_LAUNCHED("face_normal_rows_kernel");
  }
  segmented_sum_kernel<Mode::kNormalize>
      <<<grid_for(V), kThreads, 0, stream>>>(table, table + V + 1, V, CornerRows<false>{{}, rows, F}, sums, normals);
  B200R_LAUNCHED("segmented_sum_kernel");
  return B200R_OK;
}

extern "C" int b200r_verts_normals_backward(const float* grad_normals, const float* verts, int64_t V,
                                            const int64_t* faces, int64_t F, const int32_t* table, const float* sums,
                                            void* workspace, size_t workspace_bytes, float* grad_verts,
                                            void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int rc = check_sizes("verts_normals_backward", V, F);
  if (rc != B200R_OK) return rc;
  if (V == 0) return B200R_OK;
  Layout L;
  rc = checked_layout("verts_normals_backward", V, F, workspace_bytes, workspace, L);
  if (rc != B200R_OK) return rc;
  char* ws = static_cast<char*>(workspace);
  float* rows = reinterpret_cast<float*>(ws + L.rows);
  float* grad_sums = grad_verts;  // read by the rows kernel before the segmented sum overwrites it
  normalize_backward_kernel<<<grid_for(V), kThreads, 0, stream>>>(grad_normals, sums, V, grad_sums);
  B200R_LAUNCHED("normalize_backward_kernel");
  if (F > 0) {
    cross_backward_rows_kernel<<<grid_for(F), kThreads, 0, stream>>>(verts, faces, V, F, grad_sums, rows);
    B200R_LAUNCHED("cross_backward_rows_kernel");
  }
  segmented_sum_kernel<Mode::kSum>
      <<<grid_for(V), kThreads, 0, stream>>>(table, table + V + 1, V, CornerRows<true>{{}, rows, F}, nullptr, grad_verts);
  B200R_LAUNCHED("segmented_sum_kernel");
  return B200R_OK;
}

extern "C" int b200r_face_areas_normals_forward(const float* verts, int64_t V, const int64_t* faces, int64_t F,
                                                float* areas, float* normals, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int rc = check_sizes("face_areas_normals_forward", V, F);
  if (rc != B200R_OK) return rc;
  if (F == 0) return B200R_OK;
  face_areas_normals_forward_kernel<<<grid_for(F), kThreads, 0, stream>>>(verts, faces, V, F, areas, normals);
  B200R_LAUNCHED("face_areas_normals_forward_kernel");
  return B200R_OK;
}

extern "C" int b200r_face_areas_normals_backward(const float* grad_areas, const float* grad_normals,
                                                 const float* verts, int64_t V, const int64_t* faces, int64_t F,
                                                 void* workspace, size_t workspace_bytes, float* grad_verts,
                                                 void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int rc = check_sizes("face_areas_normals_backward", V, F);
  if (rc != B200R_OK) return rc;
  if (V == 0) return B200R_OK;
  Layout L;
  rc = checked_layout("face_areas_normals_backward", V, F, workspace_bytes, workspace, L);
  if (rc != B200R_OK) return rc;
  char* ws = static_cast<char*>(workspace);
  float* rows = reinterpret_cast<float*>(ws + L.rows);
  int32_t* table = reinterpret_cast<int32_t*>(ws + L.table);
  rc = build_table(faces, V, F, ws, L, table, stream);
  if (rc != B200R_OK) return rc;
  if (F > 0) {
    face_areas_normals_backward_rows_kernel<<<grid_for(F), kThreads, 0, stream>>>(grad_areas, grad_normals, verts,
                                                                                  faces, V, F, rows);
    B200R_LAUNCHED("face_areas_normals_backward_rows_kernel");
  }
  segmented_sum_kernel<Mode::kSum>
      <<<grid_for(V), kThreads, 0, stream>>>(table, table + V + 1, V, CornerRows<true>{{}, rows, F}, nullptr, grad_verts);
  B200R_LAUNCHED("segmented_sum_kernel");
  return B200R_OK;
}
