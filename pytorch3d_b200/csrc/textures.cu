// UV texture sampling, forward and backward (DESIGN.md section 13).
//
// What pytorch3d/renderer/mesh/textures.py TexturesUV.sample_textures computes for a single-map texture, per slot:
//
//   uv      = barycentric interpolation of the face's three corner UVs, (0, 0) where pix_to_face < 0
//   grid    = (lerp(-1, 1, u), lerp(1, -1, v))                                   (torch.lerp, y flipped)
//   texel   = F.grid_sample(map of image n, grid, mode, padding_mode, align_corners)
//
// The reference expands the (N, H_in, W_in, C) maps K times into an (N*K, C, H_in, W_in) copy so that grid_sample has
// one batch entry per (image, slot); here one thread per slot reads the channel-last maps of its image in place and
// writes its C texels.  The backward recomputes the sample and writes grad_barycentric_coords once per slot; the map
// and face-UV gradients are scattered with warp-merged atomics.  Nothing synchronises the host.
//
// The UV uses the FMA chain of interp_face_attrs_forward_kernel (bit-identical to interpolate_face_attributes).  The
// coordinate helpers restate torch's ATen/native/cuda/GridSampler.cuh; the four-corner weights, their summation order
// (an FMA chain nw, ne, sw, se from 0) and the unnormalisation's contraction follow what torch's grid_sampler_2d_kernel
// compiles to for sm_90, so the texels equal the chain's.  "nearest" rounds half to even (nearbyint).
#include <climits>

#include "common.cuh"
#include "raster_math.cuh"

namespace b200r {
namespace {

constexpr int kThreads = 256;

// (u, v) of slot s on face f (>= 0): fma(w2,a2, fma(w1,a1, fma(w0,a0,0))), corners 2 floats apart
__device__ __forceinline__ void interp_uv(const float* __restrict__ face_uvs, int64_t f, float w0, float w1, float w2,
                                          float& u, float& v) {
  const float* a = face_uvs + f * 6;
  u = ffma(w2, __ldg(a + 4), ffma(w1, __ldg(a + 2), ffma(w0, __ldg(a + 0), 0.0f)));
  v = ffma(w2, __ldg(a + 5), ffma(w1, __ldg(a + 3), ffma(w0, __ldg(a + 1), 0.0f)));
}

// torch.lerp(start, end, weight) for float: start + weight * (end - start) where |weight| < 0.5, else
// end - (end - start) * (1 - weight)
__device__ __forceinline__ float torch_lerp(float start, float end, float w) {
  const float d = fsub(end, start);
  return fabsf(w) < 0.5f ? fadd(start, fmul(w, d)) : fsub(end, fmul(d, fsub(1.0f, w)));
}

// grid_sampler_unnormalize; the non-aligned branch's (coord + 1) * size - 1 is one FMA in torch's build
__device__ __forceinline__ float unnormalize(float coord, int size, bool align_corners) {
  const float c1 = fadd(coord, 1.0f);
  return align_corners ? fmul(fmul(c1, 0.5f), (float)(size - 1)) : fmul(ffma(c1, (float)size, -1.0f), 0.5f);
}

__device__ __forceinline__ float clip_coordinates(float in, int clip_limit) {
  return fminf((float)(clip_limit - 1), fmaxf(in, 0.0f));
}

__device__ __forceinline__ float clip_coordinates_set_grad(float in, int clip_limit, float* grad_in) {
  // borders count as out of bounds for the gradient
  if (in <= 0.0f) {
    *grad_in = 0.0f;
    return 0.0f;
  }
  const float max = (float)(clip_limit - 1);
  if (in >= max) {
    *grad_in = 0.0f;
    return max;
  }
  *grad_in = 1.0f;
  return in;
}

// Reflects `in` until it falls between twice_low / 2 and twice_high / 2 (inclusive).
__device__ __forceinline__ float reflect_coordinates_set_grad(float in, int twice_low, int twice_high,
                                                              float* grad_in) {
  if (twice_low == twice_high) {
    *grad_in = 0.0f;
    return 0.0f;
  }
  const float min = (float)twice_low / 2;
  const float span = (float)(twice_high - twice_low) / 2;
  in = fsub(in, min);
  float mult = 1.0f;
  if (in < 0.0f) {
    mult = -1.0f;
    in = -in;
  }
  const float extra = fmodf(in, span);
  const int flips = (int)floorf(fdiv(in, span));
  if (flips % 2 == 0) {
    *grad_in = mult;
    return fadd(extra, min);
  }
  *grad_in = -mult;
  return fadd(fsub(span, extra), min);
}

__device__ __forceinline__ float safe_downgrade_to_int_range(float x) {
  // any value that is not within bounds; keeps the int conversions below defined
  if (x > (float)(INT_MAX - 1) || x < (float)INT_MIN || !isfinite(x)) return -100.0f;
  return x;
}

// grid_sampler_compute_source_index_set_grad: the source coordinate of a grid coordinate and d source / d grid.
// (The reflection's fabs / sign split gives the same coordinate as torch's forward-only reflect_coordinates.)
__device__ __forceinline__ float source_index(float coord, int size, int padding, bool align_corners, float* grad) {
  float g = align_corners ? (float)(size - 1) / 2 : (float)size / 2;
  coord = unnormalize(coord, size, align_corners);
  if (padding == B200R_PAD_BORDER) {
    float gc;
    coord = clip_coordinates_set_grad(coord, size, &gc);
    g = g * gc;
  } else if (padding == B200R_PAD_REFLECTION) {
    float gr, gc;
    coord = align_corners ? reflect_coordinates_set_grad(coord, 0, 2 * (size - 1), &gr)
                          : reflect_coordinates_set_grad(coord, -1, 2 * size - 1, &gr);
    coord = clip_coordinates_set_grad(coord, size, &gc);
    g = g * gr * gc;
  }
  *grad = g;
  return safe_downgrade_to_int_range(coord);
}

// The forward's coordinate: clip_coordinates (fmin / fmax, so a NaN becomes 0) where the gradient twin compares.
__device__ __forceinline__ float source_index(float coord, int size, int padding, bool align_corners) {
  coord = unnormalize(coord, size, align_corners);
  if (padding == B200R_PAD_BORDER) {
    coord = clip_coordinates(coord, size);
  } else if (padding == B200R_PAD_REFLECTION) {
    float unused;
    coord = align_corners ? reflect_coordinates_set_grad(coord, 0, 2 * (size - 1), &unused)
                          : reflect_coordinates_set_grad(coord, -1, 2 * size - 1, &unused);
    coord = clip_coordinates(coord, size);
  }
  return safe_downgrade_to_int_range(coord);
}

__device__ __forceinline__ bool in_bounds(int y, int x, int H, int W) { return y >= 0 && y < H && x >= 0 && x < W; }

struct Geometry {
  const int64_t* pix_to_face;
  const float* bary;
  const float* face_uvs;
  const float* maps;
  int64_t total, slots_per_image;
  int H_in, W_in, C, padding;
  bool align_corners;
};

// The slot's face, barycentrics and grid coordinates.
__device__ __forceinline__ void slot_grid(const Geometry& g, int64_t s, int64_t& f, float (&w)[3], float& gx,
                                          float& gy) {
  f = __ldg(g.pix_to_face + s);
  float u = 0.0f, v = 0.0f;
  w[0] = w[1] = w[2] = 0.0f;
  if (f >= 0) {
    w[0] = __ldg(g.bary + s * 3 + 0);
    w[1] = __ldg(g.bary + s * 3 + 1);
    w[2] = __ldg(g.bary + s * 3 + 2);
    interp_uv(g.face_uvs, f, w[0], w[1], w[2], u, v);
  }
  gx = torch_lerp(-1.0f, 1.0f, u);
  gy = torch_lerp(1.0f, -1.0f, v);
}

// Corners of a bilinear sample: weights nw, ne, sw, se, torch's products.
struct Bilinear {
  int ix, iy;  // the north-west corner
  float w[4];
};
__device__ __forceinline__ Bilinear bilinear(float ix, float iy) {
  Bilinear b;
  b.ix = (int)floorf(ix);
  b.iy = (int)floorf(iy);
  const float x0 = (float)b.ix, y0 = (float)b.iy, x1 = (float)(b.ix + 1), y1 = (float)(b.iy + 1);
  b.w[0] = fmul(fsub(x1, ix), fsub(y1, iy));
  b.w[1] = fmul(fsub(ix, x0), fsub(y1, iy));
  b.w[2] = fmul(fsub(x1, ix), fsub(iy, y0));
  b.w[3] = fmul(fsub(ix, x0), fsub(iy, y0));
  return b;
}

// One thread per slot.  CT channels per pass: C itself for C <= 4 (registers, one pass), 4 for larger C.
template <int MODE, int CT>
__global__ void __launch_bounds__(kThreads) texture_uv_forward_kernel(const Geometry g, float* __restrict__ texels) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; s < g.total; s += stride) {
    int64_t f;
    float w[3], gx, gy;
    slot_grid(g, s, f, w, gx, gy);
    const float ix = source_index(gx, g.W_in, g.padding, g.align_corners);
    const float iy = source_index(gy, g.H_in, g.padding, g.align_corners);
    const float* map = g.maps + (s / g.slots_per_image) * g.H_in * (int64_t)g.W_in * g.C;
    float* out = texels + s * g.C;
    if (MODE == B200R_SAMPLE_NEAREST) {
      const int x = (int)rintf(ix), y = (int)rintf(iy);
      const bool in = in_bounds(y, x, g.H_in, g.W_in);
      const float* p = map + ((int64_t)y * g.W_in + x) * g.C;
      for (int c0 = 0; c0 < g.C; c0 += CT) {
#pragma unroll
        for (int i = 0; i < CT; ++i)
          if (c0 + i < g.C) out[c0 + i] = in ? __ldg(p + c0 + i) : 0.0f;
      }
    } else {
      const Bilinear b = bilinear(ix, iy);
      bool in[4];
      const float* p[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const int x = b.ix + (k & 1), y = b.iy + (k >> 1);
        in[k] = in_bounds(y, x, g.H_in, g.W_in);
        p[k] = map + ((int64_t)y * g.W_in + x) * g.C;
      }
      for (int c0 = 0; c0 < g.C; c0 += CT) {
        float acc[CT];
#pragma unroll
        for (int i = 0; i < CT; ++i) acc[i] = 0.0f;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          if (!in[k]) continue;
#pragma unroll
          for (int i = 0; i < CT; ++i)
            if (c0 + i < g.C) acc[i] = ffma(b.w[k], __ldg(p[k] + c0 + i), acc[i]);
        }
#pragma unroll
        for (int i = 0; i < CT; ++i)
          if (c0 + i < g.C) out[c0 + i] = acc[i];
      }
    }
  }
}

__device__ __forceinline__ void red_add(float* p, float v) {
  asm volatile("red.global.add.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}

// Adds one warp's per-lane values g[0..M) at out + key * stride (M consecutive floats; entries i with mask bit i clear
// are not added).  Lanes with the same key are merged first (one MATCH, then pointer jumping), so each distinct key of
// the warp costs at most M reductions; sums that are exactly 0 are skipped (they cannot change a +0-initialised
// sum).  Every lane of the warp must call it; lanes with nothing to add pass key = -1.
template <int M>
__device__ __forceinline__ void warp_merge_add(float* __restrict__ out, int64_t key, int64_t stride, float (&g)[M],
                                               unsigned mask) {
  if (__all_sync(0xffffffffu, key < 0)) return;
  const int lane = threadIdx.x & 31;
  const unsigned grp = __match_any_sync(0xffffffffu, key);
  const unsigned above = lane == 31 ? 0u : grp & (0xffffffffu << (lane + 1));
  int next = (key >= 0 && above != 0u) ? __ffs((int)above) - 1 : -1;
  while (__any_sync(0xffffffffu, next >= 0)) {
    const int src = next >= 0 ? next : lane;
#pragma unroll
    for (int i = 0; i < M; ++i) {
      const float v = __shfl_sync(0xffffffffu, g[i], src);
      if (next >= 0) g[i] += v;
    }
    const int nn = __shfl_sync(0xffffffffu, next, src);
    next = next >= 0 ? nn : -1;
  }
  if (key >= 0 && lane == __ffs((int)grp) - 1) {
    float* o = out + key * stride;
#pragma unroll
    for (int i = 0; i < M; ++i)
      if (((mask >> i) & 1u) && g[i] != 0.0f) red_add(o + i, g[i]);
  }
}

struct BackwardOut {
  float* grad_maps;       // may be null
  float* grad_bary;       // may be null
  float* grad_face_uvs;   // may be null
};

template <int MODE, int CT>
__global__ void __launch_bounds__(kThreads)
    texture_uv_backward_kernel(const Geometry g, const float* __restrict__ grad_texels, const BackwardOut o) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  // warp-uniform trip count: every lane reaches the warp-wide scatters
  for (int64_t s0 = (int64_t)blockIdx.x * blockDim.x; s0 < g.total; s0 += stride) {
    const int64_t s = s0 + threadIdx.x;
    const bool active = s < g.total;
    int64_t f = -1;
    float w[3] = {0.0f, 0.0f, 0.0f}, gx = 0.0f, gy = 0.0f;
    if (active) slot_grid(g, s, f, w, gx, gy);
    float mx = 0.0f, my = 0.0f;
    const float ix = source_index(gx, g.W_in, g.padding, g.align_corners, &mx);
    const float iy = source_index(gy, g.H_in, g.padding, g.align_corners, &my);
    const int64_t n = active ? s / g.slots_per_image : 0;
    const int64_t texels_per_image = (int64_t)g.H_in * g.W_in;
    const float* map = g.maps + n * texels_per_image * g.C;
    const float* go = grad_texels + (active ? s : 0) * g.C;
    if (MODE == B200R_SAMPLE_NEAREST) {
      if (o.grad_maps != nullptr) {
        const int x = (int)rintf(ix), y = (int)rintf(iy);
        const bool in = active && in_bounds(y, x, g.H_in, g.W_in);
        const int64_t texel = n * texels_per_image + (int64_t)y * g.W_in + x;
        for (int c0 = 0; c0 < g.C; c0 += CT) {
          float v[CT];
          unsigned mask = 0u;
          bool any = false;
#pragma unroll
          for (int i = 0; i < CT; ++i) {
            v[i] = (in && c0 + i < g.C) ? __ldg(go + c0 + i) : 0.0f;
            if (c0 + i < g.C) mask |= 1u << i;
            any = any || v[i] != 0.0f;
          }
          warp_merge_add<CT>(o.grad_maps + c0, any ? texel : -1, g.C, v, mask);
        }
      }
      if (active && o.grad_bary != nullptr) {  // the grid gets no gradient from a nearest sample
        o.grad_bary[s * 3 + 0] = 0.0f;
        o.grad_bary[s * 3 + 1] = 0.0f;
        o.grad_bary[s * 3 + 2] = 0.0f;
      }
      continue;
    }
    const Bilinear b = bilinear(ix, iy);
    bool in[4];
    const float* p[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int x = b.ix + (k & 1), y = b.iy + (k >> 1);
      in[k] = active && in_bounds(y, x, g.H_in, g.W_in);
      p[k] = map + ((int64_t)y * g.W_in + x) * g.C;
    }
    // d texel / d (ix, iy) of each corner's value: nw (-dy1, -dx1), ne (dy1, -dx0), sw (-dy0, dx1), se (dy0, dx0)
    const float dx1 = fsub((float)(b.ix + 1), ix), dx0 = fsub(ix, (float)b.ix);
    const float dy1 = fsub((float)(b.iy + 1), iy), dy0 = fsub(iy, (float)b.iy);
    const float wx[4] = {-dy1, dy1, -dy0, dy0}, wy[4] = {-dx1, -dx0, dx1, dx0};
    const bool want_grid = f >= 0 && (o.grad_bary != nullptr || o.grad_face_uvs != nullptr);
    float gix = 0.0f, giy = 0.0f;
    for (int c0 = 0; c0 < g.C; c0 += CT) {
      float gc[CT];
      unsigned mask = 0u;
#pragma unroll
      for (int i = 0; i < CT; ++i) {
        gc[i] = (active && c0 + i < g.C) ? __ldg(go + c0 + i) : 0.0f;
        if (c0 + i < g.C) mask |= 1u << i;
      }
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if (o.grad_maps != nullptr) {
          float v[CT];
          bool any = false;
#pragma unroll
          for (int i = 0; i < CT; ++i) {
            v[i] = in[k] ? b.w[k] * gc[i] : 0.0f;
            any = any || v[i] != 0.0f;
          }
          const int64_t texel = n * texels_per_image + (int64_t)(b.iy + (k >> 1)) * g.W_in + (b.ix + (k & 1));
          warp_merge_add<CT>(o.grad_maps + c0, any ? texel : -1, g.C, v, mask);
        }
        if (want_grid && in[k]) {
#pragma unroll
          for (int i = 0; i < CT; ++i) {
            if (c0 + i >= g.C) continue;
            const float val = __ldg(p[k] + c0 + i);
            gix += val * wx[k] * gc[i];
            giy += val * wy[k] * gc[i];
          }
        }
      }
    }
    // grid gradient -> lerp (d grid / d uv = (2, -2)) -> barycentric interpolation of the corner UVs
    const float gu = mx * gix * 2.0f, gv = my * giy * -2.0f;
    if (active && o.grad_bary != nullptr) {
      float gb[3] = {0.0f, 0.0f, 0.0f};
      if (f >= 0) {
        const float* a = g.face_uvs + f * 6;
#pragma unroll
        for (int i = 0; i < 3; ++i) gb[i] = __ldg(a + 2 * i) * gu + __ldg(a + 2 * i + 1) * gv;
      }
      o.grad_bary[s * 3 + 0] = gb[0];
      o.grad_bary[s * 3 + 1] = gb[1];
      o.grad_bary[s * 3 + 2] = gb[2];
    }
    if (o.grad_face_uvs != nullptr) {
      float v[6] = {w[0] * gu, w[0] * gv, w[1] * gu, w[1] * gv, w[2] * gu, w[2] * gv};
      warp_merge_add<6>(o.grad_face_uvs, f, 6, v, 0x3fu);
    }
  }
}

template <int MODE>
void launch(bool backward, int C, const Geometry& g, dim3 grid, const float* grad_texels, const BackwardOut& o,
            float* texels, cudaStream_t stream) {
#define B200R_TEXTURE_LAUNCH(CT)                                                                    \
  if (backward)                                                                                     \
    texture_uv_backward_kernel<MODE, CT><<<grid, kThreads, 0, stream>>>(g, grad_texels, o);         \
  else                                                                                              \
    texture_uv_forward_kernel<MODE, CT><<<grid, kThreads, 0, stream>>>(g, texels);
  switch (C) {
    case 1: B200R_TEXTURE_LAUNCH(1) break;
    case 2: B200R_TEXTURE_LAUNCH(2) break;
    case 3: B200R_TEXTURE_LAUNCH(3) break;
    default: B200R_TEXTURE_LAUNCH(4) break;
  }
#undef B200R_TEXTURE_LAUNCH
}

int check_texture_args(int32_t N, int32_t H, int32_t W, int32_t K, int64_t F, int32_t H_in, int32_t W_in, int32_t C,
                       int32_t mode, int32_t padding) {
  if (N < 0 || H < 0 || W < 0 || K < 0 || F < 0) return fail(B200R_ERR_INVALID_ARGUMENT, "negative size");
  if (H_in < 1 || W_in < 1 || C < 1) return fail(B200R_ERR_INVALID_ARGUMENT, "texture maps must be non-empty");
  if (mode != B200R_SAMPLE_BILINEAR && mode != B200R_SAMPLE_NEAREST)
    return fail(B200R_ERR_INVALID_ARGUMENT, "unknown sampling mode");
  if (padding != B200R_PAD_ZEROS && padding != B200R_PAD_BORDER && padding != B200R_PAD_REFLECTION)
    return fail(B200R_ERR_INVALID_ARGUMENT, "unknown padding mode");
  return B200R_OK;
}

int run(bool backward, const int64_t* pix_to_face, const float* bary, const float* face_uvs, int64_t F,
        const float* maps, int32_t N, int32_t H, int32_t W, int32_t K, int32_t H_in, int32_t W_in, int32_t C,
        int32_t mode, int32_t padding, int32_t align_corners, const float* grad_texels, const BackwardOut& o,
        float* texels, cudaStream_t stream) {
  const int64_t spi = (int64_t)H * W * K, total = (int64_t)N * spi;
  const Geometry g{pix_to_face, bary, face_uvs, maps, total, spi, H_in, W_in, C, padding, align_corners != 0};
  const dim3 grid((unsigned)cap_grid_stride_blocks((total + kThreads - 1) / kThreads));
  if (mode == B200R_SAMPLE_NEAREST)
    launch<B200R_SAMPLE_NEAREST>(backward, C, g, grid, grad_texels, o, texels, stream);
  else
    launch<B200R_SAMPLE_BILINEAR>(backward, C, g, grid, grad_texels, o, texels, stream);
  return B200R_OK;
}

}  // namespace
}  // namespace b200r

using namespace b200r;

extern "C" int b200r_texture_uv_forward(const int64_t* pix_to_face, const float* barycentric_coords,
                                        const float* face_uvs, int64_t F, const float* maps, int32_t N, int32_t H,
                                        int32_t W, int32_t K, int32_t H_in, int32_t W_in, int32_t C, int32_t mode,
                                        int32_t padding, int32_t align_corners, float* texels, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int rc = check_texture_args(N, H, W, K, F, H_in, W_in, C, mode, padding);
  if (rc != B200R_OK) return rc;
  if ((int64_t)N * H * W * K == 0) return B200R_OK;
  run(false, pix_to_face, barycentric_coords, face_uvs, F, maps, N, H, W, K, H_in, W_in, C, mode, padding,
      align_corners, nullptr, BackwardOut{nullptr, nullptr, nullptr}, texels, stream);
  B200R_LAUNCHED("texture_uv_forward_kernel");
  return B200R_OK;
}

extern "C" int b200r_texture_uv_backward(const float* grad_texels, const int64_t* pix_to_face,
                                         const float* barycentric_coords, const float* face_uvs, int64_t F,
                                         const float* maps, int32_t N, int32_t H, int32_t W, int32_t K, int32_t H_in,
                                         int32_t W_in, int32_t C, int32_t mode, int32_t padding,
                                         int32_t align_corners, float* grad_maps, float* grad_barycentric_coords,
                                         float* grad_face_uvs, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int rc = check_texture_args(N, H, W, K, F, H_in, W_in, C, mode, padding);
  if (rc != B200R_OK) return rc;
  if (grad_maps != nullptr && N > 0)
    B200R_CUDA_OK(cudaMemsetAsync(grad_maps, 0, sizeof(float) * (size_t)N * H_in * W_in * C, stream));
  if (grad_face_uvs != nullptr && F > 0)
    B200R_CUDA_OK(cudaMemsetAsync(grad_face_uvs, 0, sizeof(float) * (size_t)F * 6, stream));
  if ((int64_t)N * H * W * K == 0) return B200R_OK;
  run(true, pix_to_face, barycentric_coords, face_uvs, F, maps, N, H, W, K, H_in, W_in, C, mode, padding,
      align_corners, grad_texels, BackwardOut{grad_maps, grad_barycentric_coords, grad_face_uvs}, nullptr, stream);
  B200R_LAUNCHED("texture_uv_backward_kernel");
  return B200R_OK;
}
