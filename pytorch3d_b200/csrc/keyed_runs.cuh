// Keyed runs: the deterministic gradient scatter shared by the normals (normals.cu, DESIGN.md section 17), the mesh
// regularisers (regularizers.cu, section 18), the surface sampler (sampling.cu, section 20), chamfer (chamfer.cu,
// section 21) and ball query (point_ops.cu, section 22), and the workspace arithmetic they and the texture atlas
// (texture_atlas.cu, section 15) have in common.
//
// Each gradient row gets a (key, id) pair, the key being the output row it adds to.  A stable radix sort of the pairs
// over key_bits(num_keys) bits and an offset array of num_keys + 1 entries give every key the run of its ids in id
// order (sort_into_runs); the key num_keys sorts after every other and belongs to no run.  Every per-key sum is one
// thread walking its run from +0 with __fadd_rn (segmented_sum_kernel), so there are no float atomics and the results
// do not depend on scheduling.
#pragma once

#include <cub/device/device_radix_sort.cuh>

#include "common.cuh"

namespace b200r {
namespace {

constexpr int kThreads = 256;
constexpr size_t kAlign = 256;  // workspace region alignment
constexpr float kNormalizeEps = 1e-6f;  // F.normalize(..., eps=1e-6) in Meshes._compute_vertex_normals

__device__ __forceinline__ float3 load3(const float* __restrict__ p, int64_t i) {
  return make_float3(__ldg(p + 3 * i + 0), __ldg(p + 3 * i + 1), __ldg(p + 3 * i + 2));
}

__device__ __forceinline__ void store3(float* __restrict__ p, int64_t i, float3 v) {
  p[3 * i + 0] = v.x;
  p[3 * i + 1] = v.y;
  p[3 * i + 2] = v.z;
}

// |s| as torch's 2-norm over dim 1 of a float32 (V, 3) tensor computes it.
__device__ __forceinline__ float norm3(float3 s) {
  return __fsqrt_rn(__fmaf_rn(s.z, s.z, __fmaf_rn(s.y, s.y, __fmul_rn(s.x, s.x))));
}

// ---- the runs ---------------------------------------------------------------------------------------------------

// offsets[k] = the first sorted position whose key is >= k, for k in [0, num_keys]: position i writes the offsets of
// the keys after the previous key up to its own (the end, n, stands for the key num_keys).
__global__ void __launch_bounds__(kThreads)
    run_offsets_kernel(const uint32_t* __restrict__ keys, int64_t n, int64_t num_keys, int32_t* __restrict__ offsets) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i <= n; i += stride) {
    const int64_t prev = i > 0 ? (int64_t)keys[i - 1] : -1;
    const int64_t cur = i < n ? (int64_t)keys[i] : num_keys;
    for (int64_t k = prev + 1; k <= cur; ++k) offsets[k] = (int32_t)i;
  }
}

// A row functor gives segmented_sum_kernel the row that id adds to key v's sum, row(at_key(v), id): at_key reads what
// the rows of one run share once per key.  Where negated(id), the row is subtracted instead.
struct AddedRows {
  __device__ static int64_t at_key(int64_t v) { return v; }
  __device__ static bool negated(int32_t) { return false; }
};

// Rows by id: rows[id].
struct RowsById : AddedRows {
  const float* rows;
  __device__ float3 operator()(int64_t, int32_t id) const { return load3(rows, id); }
};

enum class Mode {
  kSum,        // out[v] = the sum of v's run
  kContinue,   // out[v] += the sum of v's run, added in order to the value out[v] holds; an empty run leaves it
  kNormalize,  // sums[v] = the sum, out[v] = sum / max(|sum|, kNormalizeEps)
};

// Per key v: the rows of its run in run order, from +0 (or from out[v] for kContinue).
template <Mode MODE, typename Row>
__global__ void __launch_bounds__(kThreads)
    segmented_sum_kernel(const int32_t* __restrict__ offsets, const int32_t* __restrict__ ids, int64_t num_keys,
                         Row row, float* __restrict__ sums, float* __restrict__ out) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < num_keys; v += stride) {
    const int32_t end = __ldg(offsets + v + 1);
    int32_t i = __ldg(offsets + v);
    if (MODE == Mode::kContinue && i == end) continue;
    float3 acc = MODE == Mode::kContinue ? load3(out, v) : make_float3(0.0f, 0.0f, 0.0f);
    const auto key = row.at_key(v);
    for (; i < end; ++i) {
      const int32_t id = __ldg(ids + i);
      const float3 r = row(key, id);
      acc = row.negated(id) ? make_float3(__fsub_rn(acc.x, r.x), __fsub_rn(acc.y, r.y), __fsub_rn(acc.z, r.z))
                            : make_float3(__fadd_rn(acc.x, r.x), __fadd_rn(acc.y, r.y), __fadd_rn(acc.z, r.z));
    }
    if (MODE == Mode::kNormalize) {
      store3(sums, v, acc);
      const float n = norm3(acc);
      const float m = n < kNormalizeEps ? kNormalizeEps : n;  // clamp_min: NaN stays NaN
      acc = make_float3(__fdiv_rn(acc.x, m), __fdiv_rn(acc.y, m), __fdiv_rn(acc.z, m));
    }
    store3(out, v, acc);
  }
}

// ---- host side ----------------------------------------------------------------------------------------------------

// ceil(log2(max_key + 1)): the key bits a sort looks at for keys in [0, max_key].
inline int key_bits(int64_t max_key) {
  int bits = 1;
  while (bits < 64 && (max_key >> bits) != 0) ++bits;
  return bits;
}

inline dim3 grid_for(int64_t n) { return dim3((unsigned)cap_grid_stride_blocks((n + kThreads - 1) / kThreads)); }

// Lays a workspace out as consecutive regions, each rounded up to kAlign bytes: take() returns a region's offset, and
// `used` is the workspace's size so far.
struct Carver {
  size_t used = 0;
  size_t take(size_t bytes) {
    const size_t at = used;
    used += align_up(bytes, kAlign);
    return at;
  }
};

// cub's temporary storage for a stable radix sort of n (Key, Id) pairs over `bits` key bits (n's type is cub's item
// count type); false when cub cannot size it (no device).
template <typename Key, typename Id, typename Count>
bool sort_bytes(Count n, int bits, size_t& bytes) {
  bytes = 0;
  return n == 0 || cub::DeviceRadixSort::SortPairs(nullptr, bytes, (const Key*)nullptr, (Key*)nullptr,
                                                   (const Id*)nullptr, (Id*)nullptr, n, 0, bits) == cudaSuccess;
}

inline bool run_sort_bytes(int64_t num_keys, int64_t n, size_t& bytes) {  // sort_into_runs' storage
  return sort_bytes<uint32_t, int32_t>((int)n, key_bits(num_keys), bytes);
}

// b200r_<op>_workspace_bytes' result for a layout of `need` bytes: 0 when cub could not size its storage (`sized`
// false; the error is cleared).
inline size_t workspace_size(bool sized, size_t need) {
  if (sized) return need;
  cudaGetLastError();
  return 0;
}

// An op's checks of its workspace: cub could size its storage, and the caller's workspace holds `need` bytes, the
// size that `bytes_fn` reports.
inline int check_workspace(const char* op, const char* bytes_fn, bool sized, size_t need, const void* workspace,
                           size_t workspace_bytes) {
  if (!sized) {
    cudaGetLastError();
    return fail(B200R_ERR_CUDA, std::string(op) + ": cub could not size its temporary storage");
  }
  if (workspace == nullptr || workspace_bytes < need)
    return fail(B200R_ERR_INVALID_ARGUMENT, std::string(op) + ": workspace smaller than " + bytes_fn);
  return B200R_OK;
}

// Sorts the n (key, id) pairs in keys_in / ids_in stably by key, over key_bits(num_keys) bits, into keys_out /
// ids_out, and writes offsets[num_keys + 1]: the run of key k is ids_out[offsets[k], offsets[k + 1]).  cub's storage
// holds run_sort_bytes(num_keys, n).  With n == 0 only the offsets are written.
int sort_into_runs(uint32_t* keys_in, uint32_t* keys_out, int32_t* ids_in, int32_t* ids_out, int64_t n,
                   int64_t num_keys, void* cub_storage, size_t cub_bytes, int32_t* offsets, cudaStream_t stream) {
  if (n > 0)
    B200R_CUDA_OK(cub::DeviceRadixSort::SortPairs(cub_storage, cub_bytes, keys_in, keys_out, ids_in, ids_out, (int)n,
                                                  0, key_bits(num_keys), stream));
  run_offsets_kernel<<<grid_for(n + 1), kThreads, 0, stream>>>(keys_out, n, num_keys, offsets);
  B200R_LAUNCHED("run_offsets_kernel");
  return B200R_OK;
}

}  // namespace
}  // namespace b200r
