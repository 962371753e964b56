// Texture atlas sampling, forward and deterministic backward (DESIGN.md section 15).
//
// What pytorch3d/renderer/mesh/textures.py TexturesAtlas.sample_textures computes, per slot, with p = pix_to_face,
// b = barycentric_coords and the packed (F, R, R, C) atlas:
//
//   (b0, b1) = (0, 0) where p < 0
//   w        = min(trunc_to_int64((b0, b1) * R), R - 1)               (no lower clamp)
//   below    = (b0 + b1) * R - (float(w0) + float(w1)) <= 1           (separately rounded float32 ops)
//   w        = below ? w : R - 1 - w
//   texel    = atlas[p, w1, w0] * float(p >= 0)                       (negative indices wrap, as torch indexing does)
//
// The reference is a chain of a dozen elementwise torch ops and an advanced-indexing gather; here the forward is one
// thread per slot.  Cells the reference cannot index (it raises) give texel 0 and no gradient.
//
// The backward must be deterministic, as autograd's backward of that gather (a sort-based index_put_) is.  So there
// are no float atomics: a key pass gives each slot the index of the cell it sampled (or a sentinel when its
// contribution is exactly ±0 in every channel, or the cell is out of range), a stable radix sort orders the
// (cell, slot) pairs, and a segmented pass sums each cell's run in ascending slot order from +0 and writes it once.
#include "keyed_runs.cuh"

namespace b200r {
namespace {

constexpr uint32_t kBackgroundBit = 0x80000000u;  // in the sorted slot index: the slot's texel was multiplied by 0

struct AtlasGeometry {
  const int64_t* pix_to_face;
  const float* bary;
  int64_t total, F;
  int R, C;
};

// The cell (f * R + w_y) * R + w_x the reference reads for slot s, or -1 where it cannot index the atlas.
// `foreground` is p >= 0, the reference's mask.
__device__ __forceinline__ int64_t atlas_cell(const AtlasGeometry& g, int64_t s, bool& foreground) {
  int64_t f = __ldg(g.pix_to_face + s);
  foreground = f >= 0;
  float b0 = 0.0f, b1 = 0.0f;
  if (foreground) {
    b0 = __ldg(g.bary + s * 3 + 0);
    b1 = __ldg(g.bary + s * 3 + 1);
  }
  const int64_t R = g.R;
  const float Rf = (float)g.R;
  int64_t wx = (int64_t)__fmul_rn(b0, Rf), wy = (int64_t)__fmul_rn(b1, Rf);
  wx = wx < R - 1 ? wx : R - 1;
  wy = wy < R - 1 ? wy : R - 1;
  const float lhs = __fsub_rn(__fmul_rn(__fadd_rn(b0, b1), Rf), __fadd_rn((float)wx, (float)wy));
  // below -R nothing indexes (flipped or not); checked first so that the flip cannot overflow
  if (wx < -R || wy < -R) return -1;
  if (!(lhs <= 1.0f)) {  // NaN compares false: flipped, as torch.where does
    wx = R - 1 - wx;
    wy = R - 1 - wy;
  }
  if (wx >= R || wy >= R) return -1;  // a negative index flipped past the end
  if (wx < 0) wx += R;
  if (wy < 0) wy += R;
  if (f < 0) f += g.F;
  if (f < 0 || f >= g.F) return -1;
  return (f * R + wy) * R + wx;
}

// One thread per slot.  CT channels per pass: C itself for C <= 4 (registers, one pass), 4 for larger C.
template <int CT>
__global__ void __launch_bounds__(kThreads)
    texture_atlas_forward_kernel(const AtlasGeometry g, const float* __restrict__ atlas, float* __restrict__ texels) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; s < g.total; s += stride) {
    bool foreground;
    const int64_t cell = atlas_cell(g, s, foreground);
    const float mask = foreground ? 1.0f : 0.0f;
    const float* src = atlas + (cell < 0 ? 0 : cell) * g.C;
    float* out = texels + s * g.C;
    for (int c0 = 0; c0 < g.C; c0 += CT) {
#pragma unroll
      for (int i = 0; i < CT; ++i)
        if (c0 + i < g.C) out[c0 + i] = cell < 0 ? 0.0f : __fmul_rn(__ldg(src + c0 + i), mask);
    }
  }
}

// Key pass: (cell or sentinel, slot index | background bit) per slot.
template <typename KeyT>
__global__ void __launch_bounds__(kThreads)
    texture_atlas_keys_kernel(const AtlasGeometry g, const float* __restrict__ grad_texels, KeyT sentinel,
                              KeyT* __restrict__ keys, uint32_t* __restrict__ slots) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; s < g.total; s += stride) {
    bool foreground;
    const int64_t cell = atlas_cell(g, s, foreground);
    bool any = false;
    if (cell >= 0) {
      const float mask = foreground ? 1.0f : 0.0f;
      const float* go = grad_texels + s * g.C;
      for (int c = 0; c < g.C && !any; ++c) any = __fmul_rn(__ldg(go + c), mask) != 0.0f;  // NaN counts
    }
    keys[s] = any ? (KeyT)cell : sentinel;
    slots[s] = (uint32_t)s | (foreground ? 0u : kBackgroundBit);
  }
}

// Segmented pass: the first position of each run of equal keys sums the run in order (ascending slot index, the sort is
// stable) from +0 and writes the cell once.
template <typename KeyT, int CT>
__global__ void __launch_bounds__(kThreads)
    texture_atlas_reduce_kernel(const KeyT* __restrict__ keys, const uint32_t* __restrict__ slots, int64_t total,
                                KeyT sentinel, int C, const float* __restrict__ grad_texels,
                                float* __restrict__ grad_atlas) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
    const KeyT key = keys[i];
    if (key == sentinel || (i > 0 && keys[i - 1] == key)) continue;
    for (int c0 = 0; c0 < C; c0 += CT) {
      float acc[CT];
#pragma unroll
      for (int k = 0; k < CT; ++k) acc[k] = 0.0f;
      for (int64_t j = i; j < total && keys[j] == key; ++j) {
        const uint32_t v = slots[j];
        const float mask = (v & kBackgroundBit) ? 0.0f : 1.0f;
        const float* go = grad_texels + (int64_t)(v & ~kBackgroundBit) * C + c0;
#pragma unroll
        for (int k = 0; k < CT; ++k)
          if (c0 + k < C) acc[k] = __fadd_rn(acc[k], __fmul_rn(__ldg(go + k), mask));
      }
      float* out = grad_atlas + (int64_t)key * C + c0;
#pragma unroll
      for (int k = 0; k < CT; ++k)
        if (c0 + k < C) out[k] = acc[k];
    }
  }
}

// Workspace layout: keys in / out, slot indices in / out, then cub's temporary storage of a sort over key_bits(cells)
// bits.  Returns false when cub cannot size its storage (no device).
struct Layout {
  size_t keys_in, keys_out, slots_in, slots_out, cub, cub_bytes, total;
};

template <typename KeyT>
bool layout(int64_t total, int64_t cells, Layout& L) {
  Carver c;
  L.keys_in = c.take(sizeof(KeyT) * (size_t)total);
  L.keys_out = c.take(sizeof(KeyT) * (size_t)total);
  L.slots_in = c.take(sizeof(uint32_t) * (size_t)total);
  L.slots_out = c.take(sizeof(uint32_t) * (size_t)total);
  const bool sized = sort_bytes<KeyT, uint32_t>(total, key_bits(cells), L.cub_bytes);
  L.cub = c.take(L.cub_bytes);
  L.total = c.used;
  return sized;
}

template <typename KeyT>
int backward_sorted(const AtlasGeometry& g, const float* grad_texels, int64_t cells, void* workspace,
                    size_t workspace_bytes, float* grad_atlas, cudaStream_t stream) {
  Layout L;
  const bool sized = layout<KeyT>(g.total, cells, L);
  const int rc = check_workspace("texture_atlas_backward", "b200r_texture_atlas_workspace_bytes", sized, L.total,
                                 workspace, workspace_bytes);
  if (rc != B200R_OK) return rc;
  char* ws = static_cast<char*>(workspace);
  KeyT* keys_in = reinterpret_cast<KeyT*>(ws + L.keys_in);
  KeyT* keys_out = reinterpret_cast<KeyT*>(ws + L.keys_out);
  uint32_t* slots_in = reinterpret_cast<uint32_t*>(ws + L.slots_in);
  uint32_t* slots_out = reinterpret_cast<uint32_t*>(ws + L.slots_out);
  const KeyT sentinel = (KeyT)cells;
  const dim3 grid = grid_for(g.total);
  texture_atlas_keys_kernel<KeyT><<<grid, kThreads, 0, stream>>>(g, grad_texels, sentinel, keys_in, slots_in);
  B200R_LAUNCHED("texture_atlas_keys_kernel");
  B200R_CUDA_OK(cub::DeviceRadixSort::SortPairs(ws + L.cub, L.cub_bytes, keys_in, keys_out, slots_in, slots_out,
                                                g.total, 0, key_bits(cells), stream));
#define B200R_ATLAS_LAUNCH(CT)                                                                                     \
  texture_atlas_reduce_kernel<KeyT, CT><<<grid, kThreads, 0, stream>>>(keys_out, slots_out, g.total, sentinel, g.C, \
                                                                       grad_texels, grad_atlas);
  switch (g.C) {
    case 1: B200R_ATLAS_LAUNCH(1) break;
    case 2: B200R_ATLAS_LAUNCH(2) break;
    case 3: B200R_ATLAS_LAUNCH(3) break;
    default: B200R_ATLAS_LAUNCH(4) break;
  }
#undef B200R_ATLAS_LAUNCH
  B200R_LAUNCHED("texture_atlas_reduce_kernel");
  return B200R_OK;
}

int check_atlas_args(int32_t N, int32_t H, int32_t W, int32_t K, int64_t F, int32_t R, int32_t C) {
  if (N < 0 || H < 0 || W < 0 || K < 0 || F < 0) return fail(B200R_ERR_INVALID_ARGUMENT, "negative size");
  if (R < 1 || C < 1) return fail(B200R_ERR_INVALID_ARGUMENT, "the atlas must have R >= 1 and C >= 1");
  return B200R_OK;
}

}  // namespace
}  // namespace b200r

using namespace b200r;

extern "C" size_t b200r_texture_atlas_workspace_bytes(int32_t N, int32_t H, int32_t W, int32_t K, int64_t F,
                                                      int32_t R) {
  const int64_t total = (int64_t)N * H * W * K, cells = F * R * (int64_t)R;
  if (total <= 0 || cells <= 0 || R < 1) return 0;
  Layout L;
  const bool sized = key_bits(cells) > 32 ? layout<uint64_t>(total, cells, L) : layout<uint32_t>(total, cells, L);
  return workspace_size(sized, L.total);
}

extern "C" int b200r_texture_atlas_forward(const int64_t* pix_to_face, const float* barycentric_coords,
                                           const float* atlas, int64_t F, int32_t R, int32_t C, int32_t N, int32_t H,
                                           int32_t W, int32_t K, float* texels, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int rc = check_atlas_args(N, H, W, K, F, R, C);
  if (rc != B200R_OK) return rc;
  const int64_t total = (int64_t)N * H * W * K;
  if (total == 0) return B200R_OK;
  const AtlasGeometry g{pix_to_face, barycentric_coords, total, F, R, C};
  const dim3 grid = grid_for(total);
  switch (C) {
    case 1: texture_atlas_forward_kernel<1><<<grid, kThreads, 0, stream>>>(g, atlas, texels); break;
    case 2: texture_atlas_forward_kernel<2><<<grid, kThreads, 0, stream>>>(g, atlas, texels); break;
    case 3: texture_atlas_forward_kernel<3><<<grid, kThreads, 0, stream>>>(g, atlas, texels); break;
    default: texture_atlas_forward_kernel<4><<<grid, kThreads, 0, stream>>>(g, atlas, texels); break;
  }
  B200R_LAUNCHED("texture_atlas_forward_kernel");
  return B200R_OK;
}

extern "C" int b200r_texture_atlas_backward(const float* grad_texels, const int64_t* pix_to_face,
                                            const float* barycentric_coords, int64_t F, int32_t R, int32_t C,
                                            int32_t N, int32_t H, int32_t W, int32_t K, void* workspace,
                                            size_t workspace_bytes, float* grad_atlas, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int rc = check_atlas_args(N, H, W, K, F, R, C);
  if (rc != B200R_OK) return rc;
  const int64_t total = (int64_t)N * H * W * K, cells = F * R * (int64_t)R;
  if (total >= (int64_t)kBackgroundBit)
    return fail(B200R_ERR_INVALID_ARGUMENT, "texture_atlas_backward: at most 2^31 - 1 slots (N*H*W*K)");
  if (cells == 0) return B200R_OK;
  B200R_CUDA_OK(cudaMemsetAsync(grad_atlas, 0, sizeof(float) * (size_t)cells * C, stream));
  if (total == 0) return B200R_OK;
  const AtlasGeometry g{pix_to_face, barycentric_coords, total, F, R, C};
  return key_bits(cells) > 32
             ? backward_sorted<uint64_t>(g, grad_texels, cells, workspace, workspace_bytes, grad_atlas, stream)
             : backward_sorted<uint32_t>(g, grad_texels, cells, workspace, workspace_bytes, grad_atlas, stream);
}
