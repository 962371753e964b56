// Mesh topology tables shared by the normals (normals.cu, DESIGN.md section 17), the mesh regularisers
// (regularizers.cu, section 18) and the surface sampler (sampling.cu, section 20): the vertex -> corner table, the one
// segmented sum over it, and the face-area and normalisation arithmetic they have in common.
//
// Corner j of face f has the id c = j * F + f and the key faces[f, j]; a stable radix sort of the 3F (key, id) pairs
// over key_bits(V) bits, and an offset array of V + 1 entries, give every vertex the run of its corners in (j, f)
// order.  Every per-vertex sum is one thread walking its run from +0 with __fadd_rn, so there are no float atomics and
// the results do not depend on scheduling.
#pragma once

#include <cub/device/device_radix_sort.cuh>

#include "common.cuh"

namespace b200r {
namespace {

constexpr int kThreads = 256;
constexpr float kNormalizeEps = 1e-6f;  // F.normalize(..., eps=1e-6) in Meshes._compute_vertex_normals

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

// |s| as torch's 2-norm over dim 1 of a float32 (V, 3) tensor computes it.
__device__ __forceinline__ float norm3(float3 s) {
  return __fsqrt_rn(__fmaf_rn(s.z, s.z, __fmaf_rn(s.y, s.y, __fmul_rn(s.x, s.x))));
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

__device__ __forceinline__ float3 load3(const float* __restrict__ p, int64_t i) {
  return make_float3(__ldg(p + 3 * i + 0), __ldg(p + 3 * i + 1), __ldg(p + 3 * i + 2));
}

__device__ __forceinline__ void store3(float* __restrict__ p, int64_t i, float3 v) {
  p[3 * i + 0] = v.x;
  p[3 * i + 1] = v.y;
  p[3 * i + 2] = v.z;
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

// offsets[v] = the first sorted position whose key is >= v, for v in [0, V]: position i writes the offsets of the
// vertices after the previous key up to its own (the end, n, stands for the key V).
__global__ void __launch_bounds__(kThreads)
    run_offsets_kernel(const uint32_t* __restrict__ keys, int64_t n, int64_t V, int32_t* __restrict__ offsets) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i <= n; i += stride) {
    const int64_t prev = i > 0 ? (int64_t)keys[i - 1] : -1;
    const int64_t cur = i < n ? (int64_t)keys[i] : V;
    for (int64_t v = prev + 1; v <= cur; ++v) offsets[v] = (int32_t)i;
  }
}

// ---- the one segmented sum --------------------------------------------------------------------------------------

enum class RowOf { kFace, kCorner };   // rows[f] (F, 3) or rows[f * 3 + j] (F, 3, 3)
enum class Epilogue { kSum, kNormalize };

// Per vertex: the sum of its corners' rows in run order from +0.  kNormalize also stores the sum in `sums` and writes
// sum / max(|sum|, 1e-6) to `out`.
template <RowOf ROW, Epilogue EPI>
__global__ void __launch_bounds__(kThreads)
    segmented_sum_kernel(const int32_t* __restrict__ offsets, const int32_t* __restrict__ corners, int64_t V,
                         int64_t F, const float* __restrict__ rows, float* __restrict__ sums,
                         float* __restrict__ out) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < V; v += stride) {
    const int32_t end = __ldg(offsets + v + 1);
    float3 acc = make_float3(0.0f, 0.0f, 0.0f);
    for (int32_t i = __ldg(offsets + v); i < end; ++i) {
      const int64_t c = __ldg(corners + i);
      const int64_t j = c >= 2 * F ? 2 : (c >= F ? 1 : 0);
      const int64_t f = c - j * F;
      const float3 r = load3(rows, ROW == RowOf::kFace ? f : f * 3 + j);
      acc = make_float3(__fadd_rn(acc.x, r.x), __fadd_rn(acc.y, r.y), __fadd_rn(acc.z, r.z));
    }
    if (EPI == Epilogue::kNormalize) {
      store3(sums, v, acc);
      const float n = norm3(acc);
      const float m = n < kNormalizeEps ? kNormalizeEps : n;  // clamp_min: NaN stays NaN
      acc = make_float3(__fdiv_rn(acc.x, m), __fdiv_rn(acc.y, m), __fdiv_rn(acc.z, m));
    }
    store3(out, v, acc);
  }
}

// ---- host side ----------------------------------------------------------------------------------------------------

// ceil(log2(V + 1)): the key bits the sort looks at (the key V, for faces out of range, included).
int key_bits(int64_t V) {
  int bits = 1;
  while (bits < 32 && (V >> bits) != 0) ++bits;
  return bits;
}

dim3 grid_for(int64_t n) { return dim3((unsigned)cap_grid_stride_blocks((n + kThreads - 1) / kThreads)); }

// cub's temporary storage for sorting n (uint32 key, int32 id) pairs over key_bits(V) bits; false when cub cannot size
// it (no device).
bool corner_sort_bytes(int64_t V, size_t n, size_t& bytes) {
  bytes = 0;
  return n == 0 || cub::DeviceRadixSort::SortPairs(nullptr, bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr,
                                                   (const int32_t*)nullptr, (int32_t*)nullptr, (int)n, 0,
                                                   key_bits(V)) == cudaSuccess;
}

// Builds the vertex -> corner table (offsets[V + 1], then the 3F corner ids in run order) at `table`, with keys_in,
// keys_out and ids_in of 3F entries and cub's storage of corner_sort_bytes(V, 3F) bytes as scratch.
int build_table(const int64_t* faces, int64_t V, int64_t F, uint32_t* keys_in, uint32_t* keys_out, int32_t* ids_in,
                void* cub_storage, size_t cub_bytes, int32_t* table, cudaStream_t stream) {
  const int64_t n = 3 * F;
  int32_t* offsets = table;
  int32_t* corners = table + V + 1;
  if (n > 0) {
    corner_keys_kernel<<<grid_for(F), kThreads, 0, stream>>>(faces, F, V, keys_in, ids_in);
    B200R_LAUNCHED("corner_keys_kernel");
    B200R_CUDA_OK(cub::DeviceRadixSort::SortPairs(cub_storage, cub_bytes, keys_in, keys_out, ids_in, corners, (int)n,
                                                  0, key_bits(V), stream));
  }
  run_offsets_kernel<<<grid_for(n + 1), kThreads, 0, stream>>>(keys_out, n, V, offsets);
  B200R_LAUNCHED("run_offsets_kernel");
  return B200R_OK;
}

}  // namespace
}  // namespace b200r
