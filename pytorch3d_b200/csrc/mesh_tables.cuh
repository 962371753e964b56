// Mesh arithmetic shared by the normals (normals.cu, DESIGN.md section 17), the mesh regularisers (regularizers.cu,
// section 18) and the surface sampler (sampling.cu, section 20): the face corners, the face-area and normalisation
// arithmetic, and the vertex -> corner table.
//
// Corner j of face f has the id c = j * F + f and the key faces[f, j]; sort_into_runs (keyed_runs.cuh) over the 3F
// (key, id) pairs gives every vertex the run of its corners in (j, f) order, and segmented_sum_kernel sums a per-face
// or per-corner row over it.
#pragma once

#include "keyed_runs.cuh"

namespace b200r {
namespace {

// The three corners of face f.  A face index outside [0, V) (the reference does not check them either) gives NaN
// corners instead of a read out of bounds.
__device__ __forceinline__ void face_corners(const float* __restrict__ verts, const int64_t* __restrict__ faces,
                                             int64_t V, int64_t f, float3 p[3]) {
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    const int64_t v = __ldg(faces + 3 * f + j);
    if (v >= 0 && v < V) {
      p[j] = make_float3(__ldg(verts + 3 * v + 0), __ldg(verts + 3 * v + 1), __ldg(verts + 3 * v + 2));
    } else {
      const float nan = __int_as_float(0x7fc00000);
      p[j] = make_float3(nan, nan, nan);
    }
  }
}

// a x b with each component fma(a_i, b_j, -rn(a_j * b_i)): torch.cross on float32 as compiled for the CPU, and autograd's
// cross backward.
__device__ __forceinline__ float3 cross_fma(float3 a, float3 b) {
  return make_float3(__fmaf_rn(a.y, b.z, -__fmul_rn(a.z, b.y)), __fmaf_rn(a.z, b.x, -__fmul_rn(a.x, b.z)),
                     __fmaf_rn(a.x, b.y, -__fmul_rn(a.y, b.x)));
}

__device__ __forceinline__ float3 sub_rn(float3 a, float3 b) {
  return make_float3(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y), __fsub_rn(a.z, b.z));
}

// The cross product c = (p1 - p0) x (p2 - p0) and its norm as FaceAreasNormalsForwardKernel<float>
// (pytorch3d/csrc/face_areas_normals/face_areas_normals.cu) is compiled by nvcc for sm_90a: each cross component is
// FFMA(first product, -FMUL(second product)), the squared norm FFMA(cz, cz, FFMA(cx, cx, FMUL(cy, cy))), then an
// IEEE square root.  The face's area is FMUL(norm, 0.5) (the reference's norm / 2.0 formed in double and rounded to
// float is exactly that).  Shared by the face-area op (normals.cu) and the sampler (sampling.cu).
__device__ __forceinline__ float face_cross_norm(const float3 p[3], float3& c) {
  const float3 a = sub_rn(p[1], p[0]), b = sub_rn(p[2], p[0]);
  c.x = __fmaf_rn(a.y, b.z, -__fmul_rn(a.z, b.y));
  c.y = __fmaf_rn(a.z, b.x, -__fmul_rn(a.x, b.z));
  c.z = __fmaf_rn(a.x, b.y, -__fmul_rn(a.y, b.x));
  return __fsqrt_rn(__fmaf_rn(c.z, c.z, __fmaf_rn(c.x, c.x, __fmul_rn(c.y, c.y))));
}

// d loss / d s for y = s / clamp_min(|s|, eps), as autograd forms it: the quotient's two gradients, clamp_min's
// (none below eps), and the norm's (none where |s| = 0).
__device__ __forceinline__ float3 normalize_backward(float3 s, float3 g, float eps) {
  const float n = norm3(s);
  const float m = n < eps ? eps : n;
  // div's gradient to the divisor, -g * ((s / m) / m), summed over the three components by expand_as's backward
  const float gm = __fadd_rn(__fadd_rn(-__fmul_rn(g.x, __fdiv_rn(__fdiv_rn(s.x, m), m)),
                                       -__fmul_rn(g.y, __fdiv_rn(__fdiv_rn(s.y, m), m))),
                             -__fmul_rn(g.z, __fdiv_rn(__fdiv_rn(s.z, m), m)));
  const float gn = n >= eps ? gm : 0.0f;               // clamp_min(norm, eps): where(norm >= eps, grad, 0)
  const float k = n == 0.0f ? 0.0f : __fdiv_rn(gn, n);  // the norm's backward: s * (grad / norm), 0 where norm == 0
  return make_float3(__fadd_rn(__fdiv_rn(g.x, m), __fmul_rn(s.x, k)), __fadd_rn(__fdiv_rn(g.y, m), __fmul_rn(s.y, k)),
                     __fadd_rn(__fdiv_rn(g.z, m), __fmul_rn(s.z, k)));
}

// ---- the vertex -> corner table ---------------------------------------------------------------------------------

// (key, corner id) of every corner; a face index outside [0, V) gets the key V, which sorts after every vertex and
// belongs to no run.
__global__ void __launch_bounds__(kThreads)
    corner_keys_kernel(const int64_t* __restrict__ faces, int64_t F, int64_t V, uint32_t* __restrict__ keys,
                       int32_t* __restrict__ ids) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; f < F; f += stride) {
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      const int64_t v = __ldg(faces + 3 * f + j);
      const int64_t c = j * F + f;
      keys[c] = (uint32_t)((v >= 0 && v < V) ? v : V);
      ids[c] = (int32_t)c;
    }
  }
}

// Rows of corner ids c = j * n + i (i < n, j < 3): rows[i] of (n, 3) per item, or rows[i * 3 + j] of (n, 3, 3) per
// corner.  The items are faces, or the sampler's samples.
template <bool PER_CORNER>
struct CornerRows : AddedRows {
  const float* rows;
  int64_t n;
  __device__ float3 operator()(int64_t, int32_t c) const {
    const int64_t j = c >= 2 * n ? 2 : (c >= n ? 1 : 0), i = c - j * n;
    return load3(rows, PER_CORNER ? i * 3 + j : i);
  }
};

// ---- host side ----------------------------------------------------------------------------------------------------

// Builds the vertex -> corner table (offsets[V + 1], then the 3F corner ids in run order) at `table`, with keys_in,
// keys_out and ids_in of 3F entries and cub's storage of run_sort_bytes(V, 3F) bytes as scratch.
int build_table(const int64_t* faces, int64_t V, int64_t F, uint32_t* keys_in, uint32_t* keys_out, int32_t* ids_in,
                void* cub_storage, size_t cub_bytes, int32_t* table, cudaStream_t stream) {
  if (F > 0) {
    corner_keys_kernel<<<grid_for(F), kThreads, 0, stream>>>(faces, F, V, keys_in, ids_in);
    B200R_LAUNCHED("corner_keys_kernel");
  }
  return sort_into_runs(keys_in, keys_out, ids_in, table + V + 1, 3 * F, V, cub_storage, cub_bytes, table, stream);
}

}  // namespace
}  // namespace b200r
