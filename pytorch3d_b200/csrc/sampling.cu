// Mesh surface sampling: pytorch3d.ops.sample_points_from_meshes, forward and deterministic backward (DESIGN.md
// section 20).
//
// Forward, three kernels and no host synchronisation:
//   1. scan_chunks_kernel: the face areas (face_cross_norm of mesh_tables.cuh, bit-identical to the reference's CUDA
//      face_areas_normals) and their float64 inclusive prefix within fixed chunks of kChunk faces of one mesh.  The same
//      launch checks every vertex coordinate for NaN / inf and marks which meshes have faces, in the status word.
//   2. mesh_totals_kernel: one thread per mesh turns its chunk totals into chunk carries, serially, and writes the
//      mesh's total area; a mesh with faces whose total is not positive and finite sets a status bit.
//   3. sample_kernel: one thread per sample.  One Philox4x32-10 evaluation (key: the per-call seed, counter: the
//      sample's global index) gives a 53-bit face draw x = u * total and the 24-bit u, v of the barycentrics; a binary
//      search finds the first face whose prefix exceeds x; then the barycentrics, the position and the normal in the
//      reference's float32 arithmetic.  Samples of meshes without faces are written as zeros.
//
// The prefix of face i is carry(chunk) + (warp carry + (lane carry + serial prefix within the thread)), every carry
// a serial exclusive sum of the totals of the level below, and every total the prefix of the level's last element.  So
// the association depends on the face counts only (the prefix is bitwise reproducible), the prefix never decreases,
// and a zero-area face has exactly the prefix of the face before it: it is never drawn.
//
// Backward: one thread per sample writes its three corner rows (w_j * grad_sample, plus the normalise and
// cross-product backward of grad_normal) and keys them by vertex; sort_into_runs and the segmented sum of
// keyed_runs.cuh add each vertex's rows in one thread, so there are no float atomics and the cost scales with the
// samples, not the faces.
#include "mesh_tables.cuh"

namespace b200r {
namespace {

constexpr int kScanItems = 16;                                // faces per thread of the chunk scan
constexpr int64_t kChunk = (int64_t)kThreads * kScanItems;   // 4096 faces per chunk
constexpr int kWarps = kThreads / 32;
constexpr float kSampleNormalEps = 2.220446049250313e-16f;  // sys.float_info.epsilon, as clamp casts it to float32

// Chunk slots of mesh m start at first[m] / kChunk + m: strictly increasing in m, and ceil(num[m] / kChunk) slots fit
// before the next mesh's, so F / kChunk + N + 1 slots cover any batch.
__host__ __device__ __forceinline__ int64_t slot_base(int64_t first, int64_t m) { return first / kChunk + m; }
int64_t num_slots(int64_t F, int64_t N) { return F / kChunk + N + 1; }

// ---- Philox4x32-10 ------------------------------------------------------------------------------------------------

__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t lo0 = 0xD2511F53u * c.x, hi0 = __umulhi(0xD2511F53u, c.x);
    const uint32_t lo1 = 0xCD9E8D57u * c.z, hi1 = __umulhi(0xCD9E8D57u, c.z);
    c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
    k.x += 0x9E3779B9u;
    k.y += 0xBB67AE85u;
  }
  return c;
}

// ---- 1. areas and chunk prefixes ----------------------------------------------------------------------------------

__global__ void __launch_bounds__(kThreads)
    scan_chunks_kernel(const float* __restrict__ verts, int64_t V, const int64_t* __restrict__ faces, int64_t F,
                       const int64_t* __restrict__ first, const int64_t* __restrict__ num, int64_t N,
                       double* __restrict__ prefix, double* __restrict__ chunk_total, int32_t* __restrict__ status) {
  const int64_t gtid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  bool finite = true;
  for (int64_t i = gtid; i < 3 * V; i += stride) finite &= isfinite(__ldg(verts + i));
  if (!finite) atomicOr(status, B200R_SAMPLE_NONFINITE);
  for (int64_t m = gtid; m < N; m += stride)
    atomicOr(status, __ldg(num + m) > 0 ? B200R_SAMPLE_HAS_VALID : B200R_SAMPLE_HAS_EMPTY);

  // the mesh owning this slot: the last m with slot_base(first[m], m) <= slot
  const int64_t slot = blockIdx.x;
  int64_t lo = 0, hi = N;
  while (hi - lo > 1) {
    const int64_t mid = (lo + hi) >> 1;
    if (slot_base(__ldg(first + mid), mid) <= slot) lo = mid; else hi = mid;
  }
  const int64_t k = slot - slot_base(__ldg(first + lo), lo);
  const int64_t count = min(__ldg(num + lo) - k * kChunk, kChunk);
  if (k < 0 || count <= 0) return;  // a slot no mesh uses (uniform over the block)
  const int64_t f0 = __ldg(first + lo) + k * kChunk + (int64_t)threadIdx.x * kScanItems;
  const int n = (int)max(min(count - (int64_t)threadIdx.x * kScanItems, (int64_t)kScanItems), (int64_t)0);

  double local[kScanItems];
  double run = 0.0;
#pragma unroll
  for (int i = 0; i < kScanItems; ++i) {
    if (i < n) {
      float3 p[3], c;
      face_corners(verts, faces, V, f0 + i, p);
      run = run + (double)__fmul_rn(face_cross_norm(p, c), 0.5f);
    }
    local[i] = run;
  }

  __shared__ double lane_total[kThreads];
  __shared__ double warp_total[kWarps];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  lane_total[threadIdx.x] = run;
  __syncthreads();
  if (lane == 0) {  // lane carries of this warp, serially; the warp's total is its last lane's prefix
    double carry = 0.0;
    for (int l = 0; l < 32; ++l) {
      const double t = lane_total[threadIdx.x + l];
      lane_total[threadIdx.x + l] = carry;
      carry = carry + t;
    }
    warp_total[warp] = carry;
  }
  __syncthreads();
  if (threadIdx.x == 0) {  // warp carries, serially; the chunk's total is its last warp's prefix
    double carry = 0.0;
    for (int w = 0; w < kWarps; ++w) {
      const double t = warp_total[w];
      warp_total[w] = carry;
      carry = carry + t;
    }
    chunk_total[slot] = carry;
  }
  __syncthreads();
  const double lane_carry = lane_total[threadIdx.x], warp_carry = warp_total[warp];
#pragma unroll
  for (int i = 0; i < kScanItems; ++i)
    if (i < n) prefix[f0 + i] = warp_carry + (lane_carry + local[i]);
}

// ---- 2. chunk carries and mesh totals -----------------------------------------------------------------------------

__global__ void __launch_bounds__(kThreads)
    mesh_totals_kernel(const int64_t* __restrict__ first, const int64_t* __restrict__ num, int64_t N,
                       const double* __restrict__ chunk_total, double* __restrict__ chunk_carry,
                       double* __restrict__ mesh_total, int32_t* __restrict__ status) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t m = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; m < N; m += stride) {
    const int64_t n = __ldg(num + m);
    const int64_t base = slot_base(__ldg(first + m), m);
    double carry = 0.0;
    for (int64_t k = 0; k * kChunk < n; ++k) {
      const double t = __ldg(chunk_total + base + k);
      chunk_carry[base + k] = carry;
      carry = carry + t;
    }
    mesh_total[m] = carry;
    if (n > 0 && !(carry > 0.0 && carry <= 1.7976931348623157e308)) atomicOr(status, B200R_SAMPLE_BAD_TOTAL);
  }
}

// ---- 3. samples ---------------------------------------------------------------------------------------------------

__device__ __forceinline__ double face_prefix(const double* __restrict__ prefix, const double* __restrict__ chunk_carry,
                                              int64_t f0, int64_t base, int64_t i) {
  return __ldg(chunk_carry + base + i / kChunk) + __ldg(prefix + f0 + i);
}

template <bool NORMALS, bool DRAWS>
__global__ void __launch_bounds__(kThreads)
    sample_kernel(const float* __restrict__ verts, int64_t V, const int64_t* __restrict__ faces, int64_t F,
                  const int64_t* __restrict__ first, const int64_t* __restrict__ num, int64_t S, int64_t M,
                  const int64_t* __restrict__ seed, const double* __restrict__ prefix,
                  const double* __restrict__ chunk_carry, const double* __restrict__ mesh_total,
                  const int64_t* __restrict__ draw_face, const float* __restrict__ draw_u,
                  const float* __restrict__ draw_v, float* __restrict__ samples, float* __restrict__ normals,
                  int64_t* __restrict__ face_idx, float* __restrict__ bary) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  uint2 key = make_uint2(0u, 0u);
  if (!DRAWS) key = make_uint2((uint32_t)__ldg(seed + 0), (uint32_t)__ldg(seed + 1));
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < M; g += stride) {
    const int64_t m = g / S;
    const int64_t n = __ldg(num + m);
    if (n <= 0) {  // a mesh without faces: zero rows
      const float3 z = make_float3(0.0f, 0.0f, 0.0f);
      store3(samples, g, z);
      if (NORMALS) store3(normals, g, z);
      store3(bary, g, z);
      face_idx[g] = -1;
      continue;
    }
    int64_t f;
    float u, v;
    if (DRAWS) {
      f = __ldg(draw_face + g);
      u = __ldg(draw_u + g);
      v = __ldg(draw_v + g);
    } else {
      const uint4 r = philox4x32_10(make_uint4((uint32_t)g, (uint32_t)((uint64_t)g >> 32), 0u, 0u), key);
      const double uf = ((double)(r.x >> 5) * 67108864.0 + (double)(r.y >> 6)) * 0x1.0p-53;  // 27 + 26 bits
      u = (float)(r.z & 0xFFFFFFu) * 0x1.0p-24f;  // torch.rand's float32: 24 random bits
      v = (float)(r.w & 0xFFFFFFu) * 0x1.0p-24f;
      const int64_t f_first = __ldg(first + m), base = slot_base(f_first, m);
      const double total = __ldg(mesh_total + m), x = uf * total;
      // the first face whose prefix exceeds x; when x rounds up to the total, the first that reaches it (the last
      // face of positive area)
      const bool at_end = !(x < total);
      int64_t lo = 0, hi = n - 1;
      while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        const double p = face_prefix(prefix, chunk_carry, f_first, base, mid);
        if (at_end ? p >= total : p > x) hi = mid; else lo = mid + 1;
      }
      f = f_first + lo;
    }
    float3 p[3];
    if (f >= 0 && f < F) {
      face_corners(verts, faces, V, f, p);
    } else {
      const float nan = __int_as_float(0x7fc00000);
      p[0] = p[1] = p[2] = make_float3(nan, nan, nan);
    }
    // _rand_barycentric_coords and w0 * a + w1 * b + w2 * c, one rounding per torch op
    const float s = __fsqrt_rn(u);
    const float w0 = __fsub_rn(1.0f, s), w1 = __fmul_rn(s, __fsub_rn(1.0f, v)), w2 = __fmul_rn(s, v);
    store3(samples, g,
           make_float3(__fadd_rn(__fadd_rn(__fmul_rn(w0, p[0].x), __fmul_rn(w1, p[1].x)), __fmul_rn(w2, p[2].x)),
                       __fadd_rn(__fadd_rn(__fmul_rn(w0, p[0].y), __fmul_rn(w1, p[1].y)), __fmul_rn(w2, p[2].y)),
                       __fadd_rn(__fadd_rn(__fmul_rn(w0, p[0].z), __fmul_rn(w1, p[1].z)), __fmul_rn(w2, p[2].z))));
    if (NORMALS) {  // (v1 - v0) x (v2 - v1) / clamp_min(|.|, eps)
      const float3 c = cross_fma(sub_rn(p[1], p[0]), sub_rn(p[2], p[1]));
      const float nr = norm3(c);
      const float d = nr < kSampleNormalEps ? kSampleNormalEps : nr;  // clamp: NaN stays NaN
      store3(normals, g, make_float3(__fdiv_rn(c.x, d), __fdiv_rn(c.y, d), __fdiv_rn(c.z, d)));
    }
    face_idx[g] = f;
    store3(bary, g, make_float3(w0, w1, w2));
  }
}

// ---- backward -----------------------------------------------------------------------------------------------------

// Per sample g: rows (g, j) = d loss / d corner j and keys[j * M + g] = its vertex (V for a sample of an empty mesh
// or a face index out of range, which sorts after every vertex and belongs to no run).
template <bool NORMALS>
__global__ void __launch_bounds__(kThreads)
    corner_rows_kernel(const float* __restrict__ grad_samples, const float* __restrict__ grad_normals,
                       const float* __restrict__ verts, int64_t V, const int64_t* __restrict__ faces, int64_t F,
                       const int64_t* __restrict__ face_idx, const float* __restrict__ bary, int64_t M,
                       float* __restrict__ rows, uint32_t* __restrict__ keys, int32_t* __restrict__ ids) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < M; g += stride) {
    const int64_t f = __ldg(face_idx + g);
    const bool ok = f >= 0 && f < F;
    const float3 w = load3(bary, g), gp = load3(grad_samples, g);
    float3 r[3] = {make_float3(__fmul_rn(gp.x, w.x), __fmul_rn(gp.y, w.x), __fmul_rn(gp.z, w.x)),
                   make_float3(__fmul_rn(gp.x, w.y), __fmul_rn(gp.y, w.y), __fmul_rn(gp.z, w.y)),
                   make_float3(__fmul_rn(gp.x, w.z), __fmul_rn(gp.y, w.z), __fmul_rn(gp.z, w.z))};
    if (NORMALS && ok) {
      float3 p[3];
      face_corners(verts, faces, V, f, p);
      const float3 a = sub_rn(p[1], p[0]), b = sub_rn(p[2], p[1]);
      const float3 gc = normalize_backward(cross_fma(a, b), load3(grad_normals, g), kSampleNormalEps);
      const float3 ga = cross_fma(b, gc), gb = cross_fma(gc, a);  // cross(a, b): a gets b x g, b gets g x a
      r[0] = sub_rn(r[0], ga);
      r[1] = make_float3(__fadd_rn(r[1].x, __fsub_rn(ga.x, gb.x)), __fadd_rn(r[1].y, __fsub_rn(ga.y, gb.y)),
                         __fadd_rn(r[1].z, __fsub_rn(ga.z, gb.z)));
      r[2] = make_float3(__fadd_rn(r[2].x, gb.x), __fadd_rn(r[2].y, gb.y), __fadd_rn(r[2].z, gb.z));
    }
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      const int64_t v = ok ? __ldg(faces + 3 * f + j) : V;
      const int64_t c = j * M + g;
      keys[c] = (uint32_t)((v >= 0 && v < V) ? v : V);
      ids[c] = (int32_t)c;
      store3(rows, g * 3 + j, r[j]);
    }
  }
}

// ---- host side ----------------------------------------------------------------------------------------------------

// Forward workspace: the face prefixes (F doubles), chunk totals and carries (num_slots doubles each), mesh totals (N
// doubles).  Backward: rows (9M floats), keys in / out, ids in / sorted ids (3M each), offsets (V + 1), cub's storage.
struct Layout {
  size_t prefix, chunk_total, chunk_carry, mesh_total;                 // forward
  size_t rows, keys_in, keys_out, ids_in, corners, offsets, cub, cub_bytes;  // backward
  size_t total;
};

bool layout(int64_t V, int64_t F, int64_t N, int64_t S, int pass, Layout& L) {
  L = Layout{};
  Carver c;
  if (pass == 0) {
    const size_t slots = (size_t)num_slots(F, N);
    L.prefix = c.take(sizeof(double) * (size_t)F);
    L.chunk_total = c.take(sizeof(double) * slots);
    L.chunk_carry = c.take(sizeof(double) * slots);
    L.mesh_total = c.take(sizeof(double) * (size_t)N);
    L.total = c.used;
    return true;
  }
  const size_t n = 3 * (size_t)N * (size_t)S;
  L.rows = c.take(sizeof(float) * 3 * n);
  L.keys_in = c.take(sizeof(uint32_t) * n);
  L.keys_out = c.take(sizeof(uint32_t) * n);
  L.ids_in = c.take(sizeof(int32_t) * n);
  L.corners = c.take(sizeof(int32_t) * n);
  L.offsets = c.take(sizeof(int32_t) * ((size_t)V + 1));
  const bool sized = run_sort_bytes(V, (int64_t)n, L.cub_bytes);
  L.cub = c.take(L.cub_bytes);
  L.total = c.used;
  return sized;
}

int check_sizes(const char* op, int64_t V, int64_t F, int64_t N, int64_t S, bool backward) {
  if (V < 0 || F < 0 || N < 1 || S < 1) return fail(B200R_ERR_INVALID_ARGUMENT, std::string(op) + ": bad sizes");
  if (V >= ((int64_t)1 << 31) - 1) return fail(B200R_ERR_INVALID_ARGUMENT, std::string(op) + ": at most 2^31 - 2 vertices");
  if (N >= ((int64_t)1 << 31) || num_slots(F, N) >= ((int64_t)1 << 31) || S > ((int64_t)1 << 40) / N)
    return fail(B200R_ERR_INVALID_ARGUMENT, std::string(op) + ": at most 2^31 - 1 meshes and 2^40 samples");
  if (backward && 3 * N * S >= ((int64_t)1 << 31))
    return fail(B200R_ERR_INVALID_ARGUMENT, std::string(op) + ": the backward takes 3 N S < 2^31 sample corners");
  return B200R_OK;
}

int checked_layout(const char* op, int64_t V, int64_t F, int64_t N, int64_t S, int pass, size_t workspace_bytes,
                   const void* workspace, Layout& L) {
  const bool sized = layout(V, F, N, S, pass, L);
  return check_workspace(op, "b200r_sample_points_workspace_bytes", sized, L.total, workspace, workspace_bytes);
}

}  // namespace
}  // namespace b200r

using namespace b200r;

extern "C" size_t b200r_sample_points_workspace_bytes(int64_t V, int64_t F, int64_t N, int64_t S, int32_t pass) {
  if (V < 0 || F < 0 || N < 1 || S < 1 || (pass != 0 && pass != 1)) return 0;
  Layout L;
  const bool sized = layout(V, F, N, S, pass, L);
  return workspace_size(sized, L.total);
}

extern "C" int b200r_sample_points_forward(const float* verts, int64_t V, const int64_t* faces, int64_t F,
                                           const int64_t* mesh_first_face, const int64_t* mesh_num_faces, int64_t N,
                                           int64_t S, const int64_t* seed, const int64_t* draw_face,
                                           const float* draw_u, const float* draw_v, void* workspace,
                                           size_t workspace_bytes, float* samples, float* normals, int64_t* face_idx,
                                           float* bary, int32_t* status, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int rc = check_sizes("sample_points_forward", V, F, N, S, false);
  if (rc != B200R_OK) return rc;
  const bool draws = draw_face != nullptr;
  if (draws != (draw_u != nullptr) || draws != (draw_v != nullptr) || (!draws && seed == nullptr))
    return fail(B200R_ERR_INVALID_ARGUMENT, "sample_points_forward: give a seed, or all three of the draws");
  Layout L;
  rc = checked_layout("sample_points_forward", V, F, N, S, 0, workspace_bytes, workspace, L);
  if (rc != B200R_OK) return rc;
  char* ws = static_cast<char*>(workspace);
  double* prefix = reinterpret_cast<double*>(ws + L.prefix);
  double* chunk_total = reinterpret_cast<double*>(ws + L.chunk_total);
  double* chunk_carry = reinterpret_cast<double*>(ws + L.chunk_carry);
  double* mesh_total = reinterpret_cast<double*>(ws + L.mesh_total);
  B200R_CUDA_OK(cudaMemsetAsync(status, 0, sizeof(int32_t), stream));
  scan_chunks_kernel<<<dim3((unsigned)num_slots(F, N)), kThreads, 0, stream>>>(verts, V, faces, F, mesh_first_face,
                                                                                mesh_num_faces, N, prefix, chunk_total,
                                                                                status);
  B200R_LAUNCHED("scan_chunks_kernel");
  mesh_totals_kernel<<<grid_for(N), kThreads, 0, stream>>>(mesh_first_face, mesh_num_faces, N, chunk_total,
                                                           chunk_carry, mesh_total, status);
  B200R_LAUNCHED("mesh_totals_kernel");
  const int64_t M = N * S;
  const dim3 grid = grid_for(M);
#define B200R_SAMPLE_LAUNCH(NRM, DRW)                                                                              \
  sample_kernel<NRM, DRW><<<grid, kThreads, 0, stream>>>(verts, V, faces, F, mesh_first_face, mesh_num_faces, S, M, \
                                                         seed, prefix, chunk_carry, mesh_total, draw_face, draw_u,   \
                                                         draw_v, samples, normals, face_idx, bary)
  if (normals != nullptr) {
    if (draws) B200R_SAMPLE_LAUNCH(true, true); else B200R_SAMPLE_LAUNCH(true, false);
  } else {
    if (draws) B200R_SAMPLE_LAUNCH(false, true); else B200R_SAMPLE_LAUNCH(false, false);
  }
#undef B200R_SAMPLE_LAUNCH
  B200R_LAUNCHED("sample_kernel");
  return B200R_OK;
}

extern "C" int b200r_sample_points_backward(const float* grad_samples, const float* grad_normals, const float* verts,
                                            int64_t V, const int64_t* faces, int64_t F, int64_t N, int64_t S,
                                            const int64_t* face_idx, const float* bary, void* workspace,
                                            size_t workspace_bytes, float* grad_verts, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int rc = check_sizes("sample_points_backward", V, F, N, S, true);
  if (rc != B200R_OK) return rc;
  if (V == 0) return B200R_OK;
  Layout L;
  rc = checked_layout("sample_points_backward", V, F, N, S, 1, workspace_bytes, workspace, L);
  if (rc != B200R_OK) return rc;
  char* ws = static_cast<char*>(workspace);
  float* rows = reinterpret_cast<float*>(ws + L.rows);
  uint32_t* keys_in = reinterpret_cast<uint32_t*>(ws + L.keys_in);
  uint32_t* keys_out = reinterpret_cast<uint32_t*>(ws + L.keys_out);
  int32_t* ids_in = reinterpret_cast<int32_t*>(ws + L.ids_in);
  int32_t* corners = reinterpret_cast<int32_t*>(ws + L.corners);
  int32_t* offsets = reinterpret_cast<int32_t*>(ws + L.offsets);
  const int64_t M = N * S, n = 3 * M;
  if (grad_normals != nullptr)
    corner_rows_kernel<true><<<grid_for(M), kThreads, 0, stream>>>(grad_samples, grad_normals, verts, V, faces, F,
                                                                   face_idx, bary, M, rows, keys_in, ids_in);
  else
    corner_rows_kernel<false><<<grid_for(M), kThreads, 0, stream>>>(grad_samples, nullptr, verts, V, faces, F,
                                                                    face_idx, bary, M, rows, keys_in, ids_in);
  B200R_LAUNCHED("corner_rows_kernel");
  rc = sort_into_runs(keys_in, keys_out, ids_in, corners, n, V, ws + L.cub, L.cub_bytes, offsets, stream);
  if (rc != B200R_OK) return rc;
  // corner id c = j * M + g, rows (g, j)
  segmented_sum_kernel<Mode::kSum>
      <<<grid_for(V), kThreads, 0, stream>>>(offsets, corners, V, CornerRows<true>{{}, rows, M}, nullptr, grad_verts);
  B200R_LAUNCHED("segmented_sum_kernel");
  return B200R_OK;
}
