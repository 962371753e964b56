// Mesh blending: the step between the rasterizer's Fragments and the RGBA image (SURVEY.md 8f-5).
//
// 1. sigmoid_alpha_blend forward / backward: drop-in for pytorch3d._C.sigmoid_alpha_blend[_backward]
//    (SigmoidAlphaBlendForwardKernel / BackwardKernel, pytorch3d/csrc/blending/sigmoid_alpha_blend.cu), bit-identical
//    to the reference kernels built for sm_90a.  The reference mixes float and double: its literals are double, so
//      prob  = (float)(1. / (1. + (double)expf(-dist / sigma)))        (-dist / sigma: float IEEE divide)
//      alpha = (float)((double)alpha * (1.0 - (double)prob))           (per valid slot, ascending k)
//      out   = (float)(1.0 - (double)alpha)
//      grad  = (float)((((double)g * (-1.0 / (double)sigma)) * prob) * (double)(float)(1.0 - alphas[pix]))
//    and the face index is read into an int before the `< 0` test.  Restated below with explicit intrinsics.
//    The forward runs one thread per pixel (the product over the slots is sequential), the backward one thread per
//    slot; the backward writes every slot (0 for empty ones): no zero-fill, no atomics.
//
// 2. softmax_rgb_blend forward / backward (no counterpart in pytorch3d._C): the torch chain of
//    pytorch3d/renderer/blending.py softmax_rgb_blend fused into one kernel per direction on the rasterizer's layout.
//    Every elementwise step is the operation torch's CUDA kernels perform, in the same precision:
//      p~_k  = 1 / (1 + expf(-x)),  x = (-d_k) * (1.0f / sigma)      (division of a tensor by a Python scalar is a
//      p_k   = p~_k * v_k                                              product with the float reciprocal)
//      zi_k  = ((zfar - z_k) * (1.0f / (float)(zfar - znear))) * v_k   (Python scalars: the range is a double)
//            = ((zfar_n - z_k) / (zfar_n - znear_n)) * v_k             ((N,) tensors: an IEEE divide)
//      m     = max(max_k zi_k, 1e-10f)                                 (masked slots enter as zi = 0)
//      e_k   = expf((zi_k - m) * (1.0f / gamma)),  w_k = p_k * e_k
//      delta = max(expf((1e-10f - m) * (1.0f / gamma)), 1e-10f)
//      rgb_c = (sum_k w_k * c_kc + delta * bg_c) / (sum_k w_k + delta),  alpha = 1 - prod_k (1 - p_k)
//    Only the order of the sums and the product over k differs from torch's reductions.
//    Backward (G: upstream rgb gradient, Ga: alpha gradient, D = sum w + delta, q_k = G.(c_k - rgb) / D):
//      dc_k = w_k G / D;  dp_k = q_k e_k + Ga prod_{l!=k}(1 - p_l)  (exclusive prefix x suffix products, no division);
//      dd_k = -v_k p~_k (1 - p~_k) / sigma * dp_k;  dzi_k = q_k w_k / gamma (+ dm on the first slot attaining the
//      maximum, when m passed its clamp), dm = -(sum_k q_k w_k + [delta passed its clamp] delta G.(bg - rgb) / D) / gamma;
//      dzbuf_k = -v_k dzi_k / (zfar - znear).
//    Every output element belongs to one slot of one pixel and is written once by the thread owning the slot: no
//    atomics.
//    K buckets: K <= 8 runs one thread per pixel with the slots in registers (16-byte loads and stores when K = 8);
//    8 < K <= 150 runs one warp per pixel, lane k % 32 holding slot k in registers, all accesses coalesced.
//
// 3. SoftDepthShader / HardDepthShader forward / backward (no counterpart in pytorch3d._C; DESIGN.md section 19): the
//    torch chains of pytorch3d/renderer/mesh/shader.py, one kernel per direction, in the same K buckets as 2.
//      p_k = softmax_prob(d_k) * v_k (k < K), p_K = 1;  c_k = sum_{j <= k} p_j;  w_k = min(c_k, 1) - min(c_{k-1}, 1)
//      out = sum_{k <= K} w_k depth_k  (depth_K = zfar)
//    Only the order of the prefix sum and of the sum over k differs from torch's cumsum and sum.
#include "common.cuh"
#include "raster_math.cuh"

namespace b200r {

// ------------------------------------------------------------------------------------------------ sigmoid alpha
__device__ __forceinline__ float sigmoid_prob_ref(float d, float sigma) {
  const float dist = -d;  // -1.0 * d: exact in double, exact back in float
  const float x = __fdiv_rn(-dist, sigma);
  return __double2float_rn(__ddiv_rn(1.0, __dadd_rn(1.0, (double)expf(x))));
}

__global__ void __launch_bounds__(256)
    sigmoid_alpha_blend_forward_kernel(const float* __restrict__ dists, const int64_t* __restrict__ pix_to_face,
                                       int64_t P, int K, float sigma, float* __restrict__ alphas) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t pix = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; pix < P; pix += stride) {
    const float* dp = dists + pix * K;
    const int64_t* fp = pix_to_face + pix * K;
    float alpha = 1.0f;
    for (int k = 0; k < K; ++k) {
      if ((int)fp[k] < 0) continue;
      const float prob = sigmoid_prob_ref(dp[k], sigma);
      alpha = __double2float_rn(__dmul_rn((double)alpha, __dsub_rn(1.0, (double)prob)));
    }
    alphas[pix] = __double2float_rn(__dsub_rn(1.0, (double)alpha));
  }
}

// One thread per slot (like the reference's kernel): the slots of consecutive threads are consecutive in memory, so
// every load and store is coalesced; the per-pixel values are broadcast reads of neighbouring threads.
__global__ void __launch_bounds__(256)
    sigmoid_alpha_blend_backward_kernel(const float* __restrict__ grad_alphas, const float* __restrict__ alphas,
                                        const float* __restrict__ dists, const int64_t* __restrict__ pix_to_face,
                                        int64_t P, int K, float sigma, float* __restrict__ grad_dists) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t total = P * K;
  const double scale = __ddiv_rn(-1.0, (double)sigma);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
    if ((int)pix_to_face[i] < 0) {
      grad_dists[i] = 0.0f;
      continue;
    }
    const int64_t pix = i / K;
    const float alpha = __double2float_rn(__dsub_rn(1.0, (double)alphas[pix]));
    const double ga = __dmul_rn((double)grad_alphas[pix], scale);
    const float prob = sigmoid_prob_ref(dists[i], sigma);
    grad_dists[i] = __double2float_rn(__dmul_rn(__dmul_rn(ga, (double)prob), (double)alpha));
  }
}

// ------------------------------------------------------------------------------------------------ softmax rgb
constexpr float kBlendEps = 1e-10f;  // blending.py softmax_rgb_blend: eps = 1e-10

struct SoftmaxArgs {
  float inv_sigma, inv_gamma;
  const float* bg;  // device (3,) or null: then bg0..2
  float bg0, bg1, bg2;
  const float* znear;  // device (N,) or null: then zn
  const float* zfar;   // device (N,) or null: then zf
  float zn, zf, inv_range;  // inv_range = 1.0f / (float)(zfar - znear) when both are scalars
};

// z_inv = (zfar - z) / (zfar - znear) * mask, as torch evaluates it for the given kinds of znear / zfar.
struct ZMap {
  float zf, a;
  bool divide;
};

__device__ __forceinline__ ZMap zmap_of(const SoftmaxArgs& s, int64_t n) {
  if (s.znear != nullptr || s.zfar != nullptr) {
    const float zf = s.zfar ? s.zfar[n] : s.zf;
    const float zn = s.znear ? s.znear[n] : s.zn;
    return {zf, fsub(zf, zn), true};
  }
  return {s.zf, s.inv_range, false};
}

__device__ __forceinline__ float z_inv_of(const ZMap& zm, float z, float v) {
  const float t = fsub(zm.zf, z);
  return fmul(zm.divide ? fdiv(t, zm.a) : fmul(t, zm.a), v);
}

// d z_inv / d z for a valid slot
__device__ __forceinline__ float dzinv_dz(const ZMap& zm) { return zm.divide ? -fdiv(1.0f, zm.a) : -zm.a; }

__device__ __forceinline__ float softmax_prob(float d, float inv_sigma) {  // torch.sigmoid(-d / sigma)
  const float x = fmul(-d, inv_sigma);
  return fdiv(1.0f, fadd(1.0f, expf(-x)));
}

struct Slot {
  float c0, c1, c2, d, z, v;
};

__device__ __forceinline__ bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// A pixel's RGBA value: one 16-byte access where the address allows it (tensors handed in may start at any float).
__device__ __forceinline__ float4 load4(const float* p, bool vec) {
  return vec ? __ldg(reinterpret_cast<const float4*>(p)) : make_float4(p[0], p[1], p[2], p[3]);
}
__device__ __forceinline__ void store4(float* p, float4 v, bool vec) {
  if (vec) {
    *reinterpret_cast<float4*>(p) = v;
  } else {
    p[0] = v.x; p[1] = v.y; p[2] = v.z; p[3] = v.w;
  }
}

// Loads of one pixel's K slots.  Register bucket (KMAX > 0): all K <= KMAX slots at once, 16-byte loads when
// K == KMAX == 8 and the rows are 16-byte aligned.  COLORS = false leaves out the colours (depth blending).
template <int KMAX, bool COLORS = true>
struct SlotCache {
  float c[KMAX][3], d[KMAX], z[KMAX], v[KMAX];

  __device__ __forceinline__ void load(const float* cp, const int64_t* fp, const float* zp, const float* dp, int K,
                                       bool vec) {
    if constexpr (KMAX == 8) {
      if (vec) {
        load_vec8(cp, fp, zp, dp);
        return;
      }
    }
#pragma unroll
    for (int k = 0; k < KMAX; ++k) {
      if (k < K) {
        if constexpr (COLORS) {
          c[k][0] = __ldg(cp + 3 * k); c[k][1] = __ldg(cp + 3 * k + 1); c[k][2] = __ldg(cp + 3 * k + 2);
        }
        d[k] = __ldg(dp + k);
        z[k] = __ldg(zp + k);
        v[k] = __ldg(fp + k) >= 0 ? 1.0f : 0.0f;
      }
    }
  }

  // The arrays hold the pixel's gradients after the backward: stored with the same access shape as the loads.
  __device__ __forceinline__ void store(float* cp, float* dp, float* zp, int K, bool vec) {
    if constexpr (KMAX == 8) {
      if (vec) {
        if constexpr (COLORS) {
          float4* c4 = reinterpret_cast<float4*>(cp);
#pragma unroll
          for (int i = 0; i < 6; ++i)
            c4[i] = make_float4(c[(4 * i) / 3][(4 * i) % 3], c[(4 * i + 1) / 3][(4 * i + 1) % 3],
                                c[(4 * i + 2) / 3][(4 * i + 2) % 3], c[(4 * i + 3) / 3][(4 * i + 3) % 3]);
        }
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          reinterpret_cast<float4*>(dp)[i] = make_float4(d[4 * i], d[4 * i + 1], d[4 * i + 2], d[4 * i + 3]);
          reinterpret_cast<float4*>(zp)[i] = make_float4(z[4 * i], z[4 * i + 1], z[4 * i + 2], z[4 * i + 3]);
        }
        return;
      }
    }
#pragma unroll
    for (int k = 0; k < KMAX; ++k) {
      if (k < K) {
        if constexpr (COLORS) {
          cp[3 * k] = c[k][0]; cp[3 * k + 1] = c[k][1]; cp[3 * k + 2] = c[k][2];
        }
        dp[k] = d[k];
        zp[k] = z[k];
      }
    }
  }

  // K == 8: a pixel's colours are 96 bytes, its indices 64, its depths and distances 32 each -- six, four, two and
  // two 16-byte loads.
  __device__ __forceinline__ void load_vec8(const float* cp, const int64_t* fp, const float* zp, const float* dp) {
    {
      if constexpr (COLORS) {
        const float4* c4 = reinterpret_cast<const float4*>(cp);
#pragma unroll
        for (int i = 0; i < 6; ++i) {
          const float4 t = __ldg(c4 + i);
          const float tt[4] = {t.x, t.y, t.z, t.w};
#pragma unroll
          for (int j = 0; j < 4; ++j) c[(4 * i + j) / 3][(4 * i + j) % 3] = tt[j];
        }
      }
      const float4* d4 = reinterpret_cast<const float4*>(dp);
      const float4* z4 = reinterpret_cast<const float4*>(zp);
      const longlong2* f2 = reinterpret_cast<const longlong2*>(fp);
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const float4 a = __ldg(d4 + i), b = __ldg(z4 + i);
        d[4 * i] = a.x; d[4 * i + 1] = a.y; d[4 * i + 2] = a.z; d[4 * i + 3] = a.w;
        z[4 * i] = b.x; z[4 * i + 1] = b.y; z[4 * i + 2] = b.z; z[4 * i + 3] = b.w;
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const longlong2 f = __ldg(f2 + i);
        v[2 * i] = f.x >= 0 ? 1.0f : 0.0f;
        v[2 * i + 1] = f.y >= 0 ? 1.0f : 0.0f;
      }
    }
  }
};

template <int KMAX>
__device__ __forceinline__ Slot slot_at(const SlotCache<KMAX>& sc, int k) {
  return {sc.c[k][0], sc.c[k][1], sc.c[k][2], sc.d[k], sc.z[k], sc.v[k]};
}

// The slots of a pixel in ascending / descending order, unrolled with compile-time indices so that the cached arrays
// stay in registers.
template <int KMAX, typename F>
__device__ __forceinline__ void for_slots(int K, F&& body) {
#pragma unroll
  for (int k = 0; k < KMAX; ++k)
    if (k < K) body(k);
}

template <int KMAX, typename F>
__device__ __forceinline__ void for_slots_reverse(int K, F&& body) {
#pragma unroll
  for (int k = KMAX - 1; k >= 0; --k)
    if (k < K) body(k);
}

// The forward quantities of one pixel that the backward needs again.
struct PixelBlend {
  float m, delta, D, r0, r1, r2, trans;  // trans = prod_k (1 - p_k)
  int argmax;
  bool m_passed, delta_passed;
};

template <int KMAX>
__device__ __forceinline__ PixelBlend blend_pixel(const SlotCache<KMAX>& sc, int K, const ZMap& zm,
                                                  const SoftmaxArgs& s, float bg0, float bg1, float bg2) {
  PixelBlend b;
  // pass 1: max of z_inv (the first slot attaining it) and the transmittance
  float zmax = 0.0f, trans = 1.0f;
  int arg = 0;
  for_slots<KMAX>(K, [&](int k) {
    const Slot t = slot_at<KMAX>(sc, k);
    const float zi = z_inv_of(zm, t.z, t.v);
    if (k == 0 || zi > zmax) {
      zmax = zi;
      arg = k;
    }
    trans = fmul(trans, fsub(1.0f, fmul(softmax_prob(t.d, s.inv_sigma), t.v)));
  });
  b.m_passed = zmax >= kBlendEps;  // clamp(min=eps) passes the gradient where the input is >= eps
  b.m = b.m_passed ? zmax : kBlendEps;
  b.argmax = arg;
  b.trans = trans;
  const float de = expf(fmul(fsub(kBlendEps, b.m), s.inv_gamma));
  b.delta_passed = de >= kBlendEps;
  b.delta = b.delta_passed ? de : kBlendEps;
  // pass 2: weights, their sum and the weighted colours
  float S = 0.0f, a0 = 0.0f, a1 = 0.0f, a2 = 0.0f;
  for_slots<KMAX>(K, [&](int k) {
    const Slot t = slot_at<KMAX>(sc, k);
    const float p = fmul(softmax_prob(t.d, s.inv_sigma), t.v);
    const float w = fmul(p, expf(fmul(fsub(z_inv_of(zm, t.z, t.v), b.m), s.inv_gamma)));
    S = fadd(S, w);
    a0 = fadd(a0, fmul(w, t.c0));
    a1 = fadd(a1, fmul(w, t.c1));
    a2 = fadd(a2, fmul(w, t.c2));
  });
  b.D = fadd(S, b.delta);
  b.r0 = fdiv(fadd(a0, fmul(b.delta, bg0)), b.D);
  b.r1 = fdiv(fadd(a1, fmul(b.delta, bg1)), b.D);
  b.r2 = fdiv(fadd(a2, fmul(b.delta, bg2)), b.D);
  return b;
}


// ---- K <= 8: one thread per pixel, the pixel's slots in registers.  At K = 8 every access is whole 16-byte vectors
// (a pixel's colours are 96 bytes, its indices 64, its depths, distances and their gradients 32 each): full sectors.
template <int KMAX>
__global__ void __launch_bounds__(256)
    softmax_rgb_blend_forward_kernel(const float* __restrict__ colors, const int64_t* __restrict__ pix_to_face,
                                     const float* __restrict__ zbuf, const float* __restrict__ dists, int64_t P,
                                     int64_t HW, int K, SoftmaxArgs s, float* __restrict__ out) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const float bg0 = s.bg ? s.bg[0] : s.bg0, bg1 = s.bg ? s.bg[1] : s.bg1, bg2 = s.bg ? s.bg[2] : s.bg2;
  const bool vec = K == 8 && aligned16(colors) && aligned16(pix_to_face) && aligned16(zbuf) && aligned16(dists);
  const bool out4 = aligned16(out);
  for (int64_t pix = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; pix < P; pix += stride) {
    SlotCache<KMAX> sc;
    sc.load(colors + pix * K * 3, pix_to_face + pix * K, zbuf + pix * K, dists + pix * K, K, vec);
    const PixelBlend b = blend_pixel<KMAX>(sc, K, zmap_of(s, pix / HW), s, bg0, bg1, bg2);
    store4(out + 4 * pix, make_float4(b.r0, b.r1, b.r2, fsub(1.0f, b.trans)), out4);
  }
}

template <int KMAX>
__global__ void __launch_bounds__(256)
    softmax_rgb_blend_backward_kernel(const float* __restrict__ grad_out, const float* __restrict__ colors,
                                      const int64_t* __restrict__ pix_to_face, const float* __restrict__ zbuf,
                                      const float* __restrict__ dists, int64_t P, int64_t HW, int K, SoftmaxArgs s,
                                      float* __restrict__ grad_colors, float* __restrict__ grad_dists,
                                      float* __restrict__ grad_zbuf) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const float bg0 = s.bg ? s.bg[0] : s.bg0, bg1 = s.bg ? s.bg[1] : s.bg1, bg2 = s.bg ? s.bg[2] : s.bg2;
  const bool vec = K == 8 && aligned16(colors) && aligned16(pix_to_face) && aligned16(zbuf) && aligned16(dists) &&
                   aligned16(grad_colors) && aligned16(grad_dists) && aligned16(grad_zbuf);
  const bool g4 = aligned16(grad_out);
  for (int64_t pix = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; pix < P; pix += stride) {
    const ZMap zm = zmap_of(s, pix / HW);
    const float dzdz = dzinv_dz(zm);
    SlotCache<KMAX> sc;
    sc.load(colors + pix * K * 3, pix_to_face + pix * K, zbuf + pix * K, dists + pix * K, K, vec);
    const PixelBlend b = blend_pixel<KMAX>(sc, K, zm, s, bg0, bg1, bg2);
    const float4 g = load4(grad_out + 4 * pix, g4);
    const float inv_D = 1.0f / b.D;
    // exclusive prefix products of (1 - p)
    float pre[KMAX];
    float run = 1.0f;
    for_slots<KMAX>(K, [&](int k) {
      pre[k] = run;
      run *= 1.0f - softmax_prob(sc.d[k], s.inv_sigma) * sc.v[k];
    });
    // the gradients, kept in registers (sc.c / sc.d / sc.z are overwritten slot by slot) and stored together
    float suf = 1.0f, sum_qw = 0.0f, dz_arg = 0.0f;
    for_slots_reverse<KMAX>(K, [&](int k) {
      const Slot t = slot_at<KMAX>(sc, k);
      const float pt = softmax_prob(t.d, s.inv_sigma);
      const float p = pt * t.v;
      const float e = expf((z_inv_of(zm, t.z, t.v) - b.m) * s.inv_gamma);
      const float w = p * e;
      const float wD = w * inv_D;
      const float q = (g.x * (t.c0 - b.r0) + g.y * (t.c1 - b.r1) + g.z * (t.c2 - b.r2)) * inv_D;
      const float dp_k = q * e + g.w * (pre[k] * suf);
      suf *= 1.0f - p;
      sc.c[k][0] = wD * g.x;
      sc.c[k][1] = wD * g.y;
      sc.c[k][2] = wD * g.z;
      sc.d[k] = -(t.v * pt * (1.0f - pt) * s.inv_sigma) * dp_k;
      const float dzi = q * w * s.inv_gamma;
      sum_qw += q * w;
      if (k == b.argmax) dz_arg = dzi;  // completed below, with the gradient of m
      sc.z[k] = t.v * dzdz * dzi;
    });
    float dm = 0.0f;
    if (b.m_passed) {
      float t = sum_qw;
      if (b.delta_passed) t += b.delta * (g.x * (bg0 - b.r0) + g.y * (bg1 - b.r1) + g.z * (bg2 - b.r2)) * inv_D;
      dm = -t * s.inv_gamma;
    }
    for_slots<KMAX>(K, [&](int k) {
      if (k == b.argmax) sc.z[k] = sc.v[k] * dzdz * (dz_arg + dm);
    });
    sc.store(grad_colors + pix * K * 3, grad_dists + pix * K, grad_zbuf + pix * K, K, vec);
  }
}

// ---- K > 8: one warp per pixel, slot k on lane k % 32 (NS = ceil(K / 32) slots per lane, kept in registers).  Loads
// and stores of the (N,H,W,K) arrays are coalesced across the lanes; the colour rows (3 floats per slot) go through a
// per-warp shared-memory buffer so that they too move as contiguous 128-byte lines.  Max (first slot attaining it),
// sums and the product over K are butterfly reductions, which leave the same bits in every lane; the exclusive
// products prod_{l != k} (1 - p_l) come from prefix and suffix scans across the lanes.
constexpr unsigned kFullMask = 0xffffffffu;
constexpr int kWarpsPerBlock = 8;

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fadd(v, __shfl_xor_sync(kFullMask, v, o));
  return v;
}

__device__ __forceinline__ float warp_prod(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmul(v, __shfl_xor_sync(kFullMask, v, o));
  return v;
}

// Scans of x under `op` (associative and commutative, identity `id`) over a pixel's slots, x_of(j) the value of slot
// 32 j + lane:
// Hillis-Steele scans inside each row of 32 slots, the row totals carried across the rows.
//   UP:   up[j] = op over the slots <= k,  pre[j] = op over the slots < k  (id at slot 0)
//   DOWN: down[j] = op over the slots >= k, suf[j] = op over the slots > k  (id at the last slot of the last row)
// pre at slot k holds the bits of up at slot k - 1, suf at slot k those of down at slot k + 1.
template <int NS, bool UP, bool DOWN, typename X, typename Op>
__device__ __forceinline__ void warp_scans(X&& x_of, int lane, float id, Op op, float (&up)[NS],
                                           float (&pre)[NS], float (&down)[NS], float (&suf)[NS]) {
  float total[NS];
#pragma unroll
  for (int j = 0; j < NS; ++j) {
    const float x = x_of(j);
    float u = x, d = x;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      float a = id, b = id;
      if constexpr (UP) a = __shfl_up_sync(kFullMask, u, o);
      if constexpr (DOWN) b = __shfl_down_sync(kFullMask, d, o);
      if (UP && lane >= o) u = op(u, a);
      if (DOWN && lane + o < 32) d = op(d, b);
    }
    total[j] = UP ? __shfl_sync(kFullMask, u, 31) : __shfl_sync(kFullMask, d, 0);
    if constexpr (UP) pre[j] = __shfl_up_sync(kFullMask, u, 1);
    if constexpr (DOWN) suf[j] = __shfl_down_sync(kFullMask, d, 1);
    if (UP && lane == 0) pre[j] = id;
    if (DOWN && lane == 31) suf[j] = id;
    up[j] = u;
    down[j] = d;
  }
  if constexpr (UP) {
    float before = id;
#pragma unroll
    for (int j = 0; j < NS; ++j) {
      pre[j] = op(pre[j], before);
      up[j] = op(up[j], before);
      before = op(before, total[j]);
    }
  }
  if constexpr (DOWN) {
    float after = id;
#pragma unroll
    for (int j = NS - 1; j >= 0; --j) {
      suf[j] = op(suf[j], after);
      down[j] = op(down[j], after);
      after = op(after, total[j]);
    }
  }
}

template <int NS, bool BACKWARD>
__global__ void __launch_bounds__(256)
    softmax_rgb_blend_warp_kernel(const float* __restrict__ grad_out, const float* __restrict__ colors,
                                  const int64_t* __restrict__ pix_to_face, const float* __restrict__ zbuf,
                                  const float* __restrict__ dists, int64_t P, int64_t HW, int K, SoftmaxArgs s,
                                  float* __restrict__ out, float* __restrict__ grad_colors,
                                  float* __restrict__ grad_dists, float* __restrict__ grad_zbuf) {
  __shared__ float stage[kWarpsPerBlock][96];
  const int lane = threadIdx.x & 31;
  float* buf = stage[threadIdx.x >> 5];
  const int64_t warps = (int64_t)gridDim.x * kWarpsPerBlock;
  const float bg0 = s.bg ? s.bg[0] : s.bg0, bg1 = s.bg ? s.bg[1] : s.bg1, bg2 = s.bg ? s.bg[2] : s.bg2;
  const bool io4 = aligned16(BACKWARD ? grad_out : out);
  for (int64_t pix = (int64_t)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5); pix < P; pix += warps) {
    const float* cp = colors + pix * K * 3;
    const int64_t* fp = pix_to_face + pix * K;
    const ZMap zm = zmap_of(s, pix / HW);
    float c[NS][3], pt[NS], v[NS], zi[NS];
    float zmax = -INFINITY, trans = 1.0f;
    int arg = INT_MAX;
#pragma unroll
    for (int j = 0; j < NS; ++j) {
      const int k = 32 * j + lane, nr = min(32, K - 32 * j);  // nr > 0: NS = ceil(K / 32)
      for (int t = lane; t < 3 * nr; t += 32) buf[t] = __ldg(cp + 96 * j + t);
      __syncwarp();
      const bool in = lane < nr;
      c[j][0] = in ? buf[3 * lane] : 0.0f;
      c[j][1] = in ? buf[3 * lane + 1] : 0.0f;
      c[j][2] = in ? buf[3 * lane + 2] : 0.0f;
      __syncwarp();
      v[j] = in && __ldg(fp + k) >= 0 ? 1.0f : 0.0f;
      pt[j] = softmax_prob(in ? __ldg(dists + pix * K + k) : 0.0f, s.inv_sigma);
      zi[j] = z_inv_of(zm, in ? __ldg(zbuf + pix * K + k) : 0.0f, v[j]);
      if (in) {
        if (zi[j] > zmax) {  // ascending k within the lane: strictly greater keeps the first
          zmax = zi[j];
          arg = k;
        }
        trans = fmul(trans, fsub(1.0f, fmul(pt[j], v[j])));
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float oz = __shfl_xor_sync(kFullMask, zmax, o);
      const int oa = __shfl_xor_sync(kFullMask, arg, o);
      if (oz > zmax || (oz == zmax && oa < arg)) {
        zmax = oz;
        arg = oa;
      }
    }
    trans = warp_prod(trans);
    const bool m_passed = zmax >= kBlendEps;
    const float m = m_passed ? zmax : kBlendEps;
    const float de = expf(fmul(fsub(kBlendEps, m), s.inv_gamma));
    const bool delta_passed = de >= kBlendEps;
    const float delta = delta_passed ? de : kBlendEps;
    float S = 0.0f, a0 = 0.0f, a1 = 0.0f, a2 = 0.0f;
#pragma unroll
    for (int j = 0; j < NS; ++j) {
      if (32 * j + lane < K) {
        const float w = fmul(fmul(pt[j], v[j]), expf(fmul(fsub(zi[j], m), s.inv_gamma)));
        S = fadd(S, w);
        a0 = fadd(a0, fmul(w, c[j][0]));
        a1 = fadd(a1, fmul(w, c[j][1]));
        a2 = fadd(a2, fmul(w, c[j][2]));
      }
    }
    const float D = fadd(warp_sum(S), delta);
    const float r0 = fdiv(fadd(warp_sum(a0), fmul(delta, bg0)), D);
    const float r1 = fdiv(fadd(warp_sum(a1), fmul(delta, bg1)), D);
    const float r2 = fdiv(fadd(warp_sum(a2), fmul(delta, bg2)), D);
    if constexpr (!BACKWARD) {
      if (lane == 0) store4(out + 4 * pix, make_float4(r0, r1, r2, fsub(1.0f, trans)), io4);
    } else {
      const float4 g = load4(grad_out + 4 * pix, io4);
      const float inv_D = 1.0f / D;
      const float dzdz = dzinv_dz(zm);
      // exclusive prefix / suffix products of (1 - p)
      float up[NS], pre[NS], down[NS], suf[NS];
      warp_scans<NS, true, true>([&](int j) { return 32 * j + lane < K ? 1.0f - pt[j] * v[j] : 1.0f; }, lane, 1.0f,
                                 [](float a, float b) { return a * b; }, up, pre, down, suf);
      float sum_qw = 0.0f, dz_arg = 0.0f;
      float gz[NS];
#pragma unroll
      for (int j = 0; j < NS; ++j) {
        const int k = 32 * j + lane, nr = min(32, K - 32 * j);
        const bool in = lane < nr;
        const float p = pt[j] * v[j];
        const float e = expf((zi[j] - m) * s.inv_gamma);
        const float w = in ? p * e : 0.0f;
        const float wD = w * inv_D;
        const float q = (g.x * (c[j][0] - r0) + g.y * (c[j][1] - r1) + g.z * (c[j][2] - r2)) * inv_D;
        const float dp_k = q * e + g.w * (pre[j] * suf[j]);
        buf[3 * lane] = wD * g.x;
        buf[3 * lane + 1] = wD * g.y;
        buf[3 * lane + 2] = wD * g.z;
        __syncwarp();
        for (int t = lane; t < 3 * nr; t += 32) grad_colors[pix * K * 3 + 96 * j + t] = buf[t];
        __syncwarp();
        const float dzi = q * w * s.inv_gamma;
        sum_qw += q * w;
        if (k == arg) dz_arg = dzi;  // completed below, with the gradient of m
        gz[j] = v[j] * dzdz * dzi;
        if (in) grad_dists[pix * K + k] = -(v[j] * pt[j] * (1.0f - pt[j]) * s.inv_sigma) * dp_k;
      }
      sum_qw = warp_sum(sum_qw);
      float dm = 0.0f;
      if (m_passed) {
        float t = sum_qw;
        if (delta_passed) t += delta * (g.x * (bg0 - r0) + g.y * (bg1 - r1) + g.z * (bg2 - r2)) * inv_D;
        dm = -t * s.inv_gamma;
      }
#pragma unroll
      for (int j = 0; j < NS; ++j) {
        const int k = 32 * j + lane;
        if (k == arg) gz[j] = v[j] * dzdz * (dz_arg + dm);
        if (k < K) grad_zbuf[pix * K + k] = gz[j];
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ depth
// zfar of the depth shaders: a device float (a 1-element tensor, read in the kernel) or, when null, a number.
struct DepthFar {
  const float* ptr;
  float value;
};

__device__ __forceinline__ float zfar_of(const DepthFar& f) { return f.ptr ? __ldg(f.ptr) : f.value; }

// clamp(max=1), which lets a NaN through
__device__ __forceinline__ float clamp1(float c) { return c > 1.0f ? 1.0f : c; }

// ---- K <= 8: one thread per pixel, the slots in registers, the prefix sums in ascending k.  Slot K (p = 1, depth
// zfar) follows the loop.
template <int KMAX>
__global__ void __launch_bounds__(256)
    soft_depth_forward_kernel(const int64_t* __restrict__ pix_to_face, const float* __restrict__ zbuf,
                              const float* __restrict__ dists, int64_t P, int K, float inv_sigma, DepthFar far,
                              float* __restrict__ out) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const bool vec = K == 8 && aligned16(pix_to_face) && aligned16(zbuf) && aligned16(dists);
  const float zf = zfar_of(far);
  for (int64_t pix = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; pix < P; pix += stride) {
    SlotCache<KMAX, false> sc;
    sc.load(nullptr, pix_to_face + pix * K, zbuf + pix * K, dists + pix * K, K, vec);
    float c = 0.0f, prev = 0.0f, acc = 0.0f;
    for_slots<KMAX>(K, [&](int k) {
      c = fadd(c, fmul(softmax_prob(sc.d[k], inv_sigma), sc.v[k]));
      const float ct = clamp1(c);
      acc = fadd(acc, fmul(fsub(ct, prev), sc.z[k]));
      prev = ct;
    });
    out[pix] = fadd(acc, fmul(fsub(clamp1(fadd(c, 1.0f)), prev), zf));
  }
}

template <int KMAX>
__global__ void __launch_bounds__(256)
    soft_depth_backward_kernel(const float* __restrict__ grad_out, const int64_t* __restrict__ pix_to_face,
                               const float* __restrict__ zbuf, const float* __restrict__ dists, int64_t P, int K,
                               float inv_sigma, DepthFar far, float* __restrict__ grad_zbuf,
                               float* __restrict__ grad_dists) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const bool vec = K == 8 && aligned16(pix_to_face) && aligned16(zbuf) && aligned16(dists) &&
                   aligned16(grad_zbuf) && aligned16(grad_dists);
  const float zf = zfar_of(far);
  for (int64_t pix = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; pix < P; pix += stride) {
    SlotCache<KMAX, false> sc;
    sc.load(nullptr, pix_to_face + pix * K, zbuf + pix * K, dists + pix * K, K, vec);
    const float g = __ldg(grad_out + pix);
    float s[KMAX], cs[KMAX];  // sigmoids and prefix sums c_k
    float c = 0.0f;
    for_slots<KMAX>(K, [&](int k) {
      s[k] = softmax_prob(sc.d[k], inv_sigma);
      c = fadd(c, fmul(s[k], sc.v[k]));
      cs[k] = c;
    });
    // slot K: gw_K = g zfar, gc~_K = gw_K - 0; gp runs the suffix sums of gc from slot K down
    float gw_next = fmul(g, zf);
    float gp = fadd(c, 1.0f) <= 1.0f ? gw_next : 0.0f;
    for_slots_reverse<KMAX>(K, [&](int k) {
      const float gw = fmul(g, sc.z[k]);
      gp = fadd(gp, cs[k] <= 1.0f ? fsub(gw, gw_next) : 0.0f);
      gw_next = gw;
      sc.z[k] = fmul(g, fsub(clamp1(cs[k]), k > 0 ? clamp1(cs[k > 0 ? k - 1 : 0]) : 0.0f));
      sc.d[k] = -fmul(fmul(fmul(fmul(gp, sc.v[k]), fsub(1.0f, s[k])), s[k]), inv_sigma);
    });
    sc.store(nullptr, grad_dists + pix * K, grad_zbuf + pix * K, K, vec);
  }
}

// ---- 8 < K <= 150: one warp per pixel, slot k on lane k % 32 of row k / 32, slot K (p = 1, depth zfar) included:
// NS = ceil((K + 1) / 32) rows.  The prefix sums c_k and the suffix sums of the backward are warp_scans; c_{k-1}
// is the exclusive prefix, which has the bits of c_{k-1} itself.
// (4 blocks per SM: a 64-register budget, within which ptxas allocates the NS = 4 backward without the spill it
// makes when left to its own target)
template <int NS, bool BACKWARD>
__global__ void __launch_bounds__(256, 4)
    soft_depth_warp_kernel(const float* __restrict__ grad_out, const int64_t* __restrict__ pix_to_face,
                           const float* __restrict__ zbuf, const float* __restrict__ dists, int64_t P, int K,
                           float inv_sigma, DepthFar far, float* __restrict__ out, float* __restrict__ grad_zbuf,
                           float* __restrict__ grad_dists) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * kWarpsPerBlock;
  const float zf = zfar_of(far);
  const auto add = [](float a, float b) { return fadd(a, b); };
  for (int64_t pix = (int64_t)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5); pix < P; pix += warps) {
    const int64_t base = pix * K;
    float s[NS], v[NS], z[NS], p[NS];
#pragma unroll
    for (int j = 0; j < NS; ++j) {
      const int k = 32 * j + lane;
      const bool in = k < K;
      v[j] = in && __ldg(pix_to_face + base + k) >= 0 ? 1.0f : 0.0f;
      s[j] = softmax_prob(in ? __ldg(dists + base + k) : 0.0f, inv_sigma);
      z[j] = in ? __ldg(zbuf + base + k) : (k == K ? zf : 0.0f);
      p[j] = in ? fmul(s[j], v[j]) : (k == K ? 1.0f : 0.0f);
    }
    float c[NS], cprev[NS], down_unused[NS], suf_unused[NS];
    warp_scans<NS, true, false>([&](int j) { return p[j]; }, lane, 0.0f, add, c, cprev, down_unused, suf_unused);
    if constexpr (!BACKWARD) {
      float acc = 0.0f;
#pragma unroll
      for (int j = 0; j < NS; ++j)
        if (32 * j + lane <= K) acc = fadd(acc, fmul(fsub(clamp1(c[j]), clamp1(cprev[j])), z[j]));
      acc = warp_sum(acc);
      if (lane == 0) out[pix] = acc;
    } else {
      const float g = __ldg(grad_out + pix);
      float gw[NS];
#pragma unroll
      for (int j = 0; j < NS; ++j) gw[j] = 32 * j + lane <= K ? fmul(g, z[j]) : 0.0f;
      float gc[NS];
#pragma unroll
      for (int j = 0; j < NS; ++j) {  // gc_k = [c_k <= 1] (gw_k - gw_{k+1})
        const float below = __shfl_down_sync(kFullMask, gw[j], 1);
        const float next_row = __shfl_sync(kFullMask, gw[j + 1 < NS ? j + 1 : j], 0);
        const float next = lane < 31 ? below : (j + 1 < NS ? next_row : 0.0f);
        gc[j] = c[j] <= 1.0f ? fsub(gw[j], next) : 0.0f;
      }
      float up_unused[NS], pre_unused[NS], gp[NS];  // gp_k = sum of gc over the slots >= k
      warp_scans<NS, false, true>([&](int j) { return gc[j]; }, lane, 0.0f, add, up_unused, pre_unused, gp,
                                  suf_unused);
#pragma unroll
      for (int j = 0; j < NS; ++j) {
        const int k = 32 * j + lane;
        if (k < K) {
          grad_zbuf[base + k] = fmul(g, fsub(clamp1(c[j]), clamp1(cprev[j])));
          grad_dists[base + k] = -fmul(fmul(fmul(fmul(gp[j], v[j]), fsub(1.0f, s[j])), s[j]), inv_sigma);
        }
      }
    }
  }
}

// HardDepthShader: slot 0's depth on covered pixels, zfar elsewhere.  One thread per pixel.
__global__ void __launch_bounds__(256)
    hard_depth_forward_kernel(const int64_t* __restrict__ pix_to_face, const float* __restrict__ zbuf, int64_t P,
                              int K, DepthFar far, float* __restrict__ out) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const float zf = zfar_of(far);
  for (int64_t pix = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; pix < P; pix += stride)
    out[pix] = __ldg(pix_to_face + pix * K) >= 0 ? __ldg(zbuf + pix * K) : zf;
}

// The gradient of slot 0's depth on covered pixels; every other slot gets 0, written here (no zero-fill pass).  One
// thread per slot, so that the stores of a warp are contiguous: a thread per pixel writing its K slots is several times
// slower at large K (DESIGN.md section 19).
__global__ void __launch_bounds__(256)
    hard_depth_backward_kernel(const float* __restrict__ grad_out, const int64_t* __restrict__ pix_to_face, int64_t P,
                               int K, float* __restrict__ grad_zbuf) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t total = P * K;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
    const int64_t pix = i / K;
    grad_zbuf[i] = i == pix * K && __ldg(pix_to_face + i) >= 0 ? __ldg(grad_out + pix) : 0.0f;
  }
}

}  // namespace b200r

using namespace b200r;

// Grid of a kernel that walks each pixel's row of K slots with one thread.  For long rows the number of resident
// threads is capped so that the rows being walked stay in L1 (each thread touches a line per input array):
// `threads_per_sm` for K > 8, full occupancy otherwise (and for threads_per_sm = 0).
static int64_t blend_blocks(int64_t threads, int K, int threads_per_sm) {
  const int64_t blocks = cap_grid_stride_blocks((threads + 255) / 256);
  if (K <= 8 || threads_per_sm == 0) return blocks;
  const int64_t cap = cap_grid_stride_blocks(1 << 30) / 32 * (threads_per_sm / 256);  // SMs x blocks per SM
  return blocks < cap ? blocks : cap;
}

extern "C" int b200r_sigmoid_alpha_blend_forward(const float* dists, const int64_t* pix_to_face, int32_t N, int32_t H,
                                                 int32_t W, int32_t K, float sigma, float* alphas, void* stream_) {
  if (N < 0 || H < 0 || W < 0 || K < 0) return fail(B200R_ERR_INVALID_ARGUMENT, "negative size");
  const int64_t P = (int64_t)N * H * W;
  if (P == 0) return B200R_OK;
  sigmoid_alpha_blend_forward_kernel<<<(unsigned)blend_blocks(P, K, 1024), 256, 0, static_cast<cudaStream_t>(stream_)>>>(
      dists, pix_to_face, P, K, sigma, alphas);
  B200R_LAUNCHED("sigmoid_alpha_blend_forward_kernel");
  return B200R_OK;
}

extern "C" int b200r_sigmoid_alpha_blend_backward(const float* grad_alphas, const float* alphas, const float* dists,
                                                  const int64_t* pix_to_face, int32_t N, int32_t H, int32_t W,
                                                  int32_t K, float sigma, float* grad_dists, void* stream_) {
  if (N < 0 || H < 0 || W < 0 || K < 0) return fail(B200R_ERR_INVALID_ARGUMENT, "negative size");
  const int64_t P = (int64_t)N * H * W;
  if (P == 0 || K == 0) return B200R_OK;
  sigmoid_alpha_blend_backward_kernel<<<(unsigned)blend_blocks(P * K, 0, 0), 256, 0, static_cast<cudaStream_t>(stream_)>>>(
      grad_alphas, alphas, dists, pix_to_face, P, K, sigma, grad_dists);
  B200R_LAUNCHED("sigmoid_alpha_blend_backward_kernel");
  return B200R_OK;
}

// K > 8: one warp per pixel, NS = ceil(K / 32) slots per lane.
template <bool BACKWARD>
static int launch_warp_kernel(const float* grad_out, const float* colors, const int64_t* pix_to_face,
                              const float* zbuf, const float* dists, int64_t P, int64_t HW, int K,
                              const SoftmaxArgs& s, float* out, float* grad_colors, float* grad_dists,
                              float* grad_zbuf, cudaStream_t stream) {
  const unsigned blocks = (unsigned)cap_grid_stride_blocks((P + kWarpsPerBlock - 1) / kWarpsPerBlock);
#define B200R_WARP(NS)                                                                                             \
  softmax_rgb_blend_warp_kernel<NS, BACKWARD><<<blocks, 32 * kWarpsPerBlock, 0, stream>>>(                        \
      grad_out, colors, pix_to_face, zbuf, dists, P, HW, K, s, out, grad_colors, grad_dists, grad_zbuf)
  switch ((K + 31) / 32) {
    case 1: B200R_WARP(1); break;
    case 2: B200R_WARP(2); break;
    case 3: B200R_WARP(3); break;
    case 4: B200R_WARP(4); break;
    default: B200R_WARP(5); break;  // K <= 150 (checked by the caller)
  }
#undef B200R_WARP
  B200R_LAUNCHED(BACKWARD ? "softmax_rgb_blend_warp_kernel<backward>" : "softmax_rgb_blend_warp_kernel<forward>");
  return B200R_OK;
}

static int softmax_args(int32_t N, int32_t H, int32_t W, int32_t K, float sigma, float gamma, const float* background,
                        const float* background_value, const float* znear, const float* zfar, double znear_value,
                        double zfar_value, SoftmaxArgs* s) {
  if (N < 0 || H < 0 || W < 0 || K < 0) return fail(B200R_ERR_INVALID_ARGUMENT, "negative size");
  if (K > B200R_MAX_K) return fail(B200R_ERR_INVALID_ARGUMENT, "Must have faces_per_pixel <= 150");
  if (background == nullptr && background_value == nullptr)
    return fail(B200R_ERR_INVALID_ARGUMENT, "a background colour is required");
  s->inv_sigma = 1.0f / sigma;
  s->inv_gamma = 1.0f / gamma;
  s->bg = background;
  s->bg0 = background ? 0.0f : background_value[0];
  s->bg1 = background ? 0.0f : background_value[1];
  s->bg2 = background ? 0.0f : background_value[2];
  s->znear = znear;
  s->zfar = zfar;
  s->zn = (float)znear_value;
  s->zf = (float)zfar_value;
  s->inv_range = 1.0f / (float)(zfar_value - znear_value);
  return B200R_OK;
}

extern "C" int b200r_softmax_rgb_blend_forward(const float* colors, const int64_t* pix_to_face, const float* zbuf,
                                               const float* dists, int32_t N, int32_t H, int32_t W, int32_t K,
                                               float sigma, float gamma, const float* background,
                                               const float* background_value, const float* znear, const float* zfar,
                                               double znear_value, double zfar_value, float* out, void* stream_) {
  SoftmaxArgs s;
  int rc = softmax_args(N, H, W, K, sigma, gamma, background, background_value, znear, zfar, znear_value, zfar_value,
                        &s);
  if (rc != B200R_OK) return rc;
  const int64_t P = (int64_t)N * H * W;
  if (P == 0) return B200R_OK;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (K <= 8) {
    softmax_rgb_blend_forward_kernel<8><<<(unsigned)blend_blocks(P, K, 0), 256, 0, stream>>>(
        colors, pix_to_face, zbuf, dists, P, (int64_t)H * W, K, s, out);
    B200R_LAUNCHED("softmax_rgb_blend_forward_kernel");
    return B200R_OK;
  }
  return launch_warp_kernel<false>(nullptr, colors, pix_to_face, zbuf, dists, P, (int64_t)H * W, K, s, out, nullptr,
                                   nullptr, nullptr, stream);
}

extern "C" int b200r_softmax_rgb_blend_backward(const float* grad_out, const float* colors, const int64_t* pix_to_face,
                                                const float* zbuf, const float* dists, int32_t N, int32_t H, int32_t W,
                                                int32_t K, float sigma, float gamma, const float* background,
                                                const float* background_value, const float* znear, const float* zfar,
                                                double znear_value, double zfar_value, float* grad_colors,
                                                float* grad_dists, float* grad_zbuf, void* stream_) {
  SoftmaxArgs s;
  int rc = softmax_args(N, H, W, K, sigma, gamma, background, background_value, znear, zfar, znear_value, zfar_value,
                        &s);
  if (rc != B200R_OK) return rc;
  const int64_t P = (int64_t)N * H * W;
  if (P == 0 || K == 0) return B200R_OK;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (K <= 8) {
    softmax_rgb_blend_backward_kernel<8><<<(unsigned)blend_blocks(P, K, 0), 256, 0, stream>>>(
        grad_out, colors, pix_to_face, zbuf, dists, P, (int64_t)H * W, K, s, grad_colors, grad_dists, grad_zbuf);
    B200R_LAUNCHED("softmax_rgb_blend_backward_kernel");
    return B200R_OK;
  }
  return launch_warp_kernel<true>(grad_out, colors, pix_to_face, zbuf, dists, P, (int64_t)H * W, K, s, nullptr,
                                  grad_colors, grad_dists, grad_zbuf, stream);
}

static int depth_args(int32_t N, int32_t H, int32_t W, int32_t K) {
  if (N < 0 || H < 0 || W < 0) return fail(B200R_ERR_INVALID_ARGUMENT, "negative size");
  if (K < 1 || K > B200R_MAX_K) return fail(B200R_ERR_INVALID_ARGUMENT, "Must have 1 <= faces_per_pixel <= 150");
  return B200R_OK;
}

// K > 8: one warp per pixel, NS = ceil((K + 1) / 32) rows of slots.
template <bool BACKWARD>
static int launch_depth_warp_kernel(const float* grad_out, const int64_t* pix_to_face, const float* zbuf,
                                    const float* dists, int64_t P, int K, float inv_sigma, DepthFar far, float* out,
                                    float* grad_zbuf, float* grad_dists, cudaStream_t stream) {
  const unsigned blocks = (unsigned)cap_grid_stride_blocks((P + kWarpsPerBlock - 1) / kWarpsPerBlock);
#define B200R_DEPTH_WARP(NS)                                                                                       \
  soft_depth_warp_kernel<NS, BACKWARD><<<blocks, 32 * kWarpsPerBlock, 0, stream>>>(                               \
      grad_out, pix_to_face, zbuf, dists, P, K, inv_sigma, far, out, grad_zbuf, grad_dists)
  switch ((K + 32) / 32) {
    case 1: B200R_DEPTH_WARP(1); break;
    case 2: B200R_DEPTH_WARP(2); break;
    case 3: B200R_DEPTH_WARP(3); break;
    case 4: B200R_DEPTH_WARP(4); break;
    default: B200R_DEPTH_WARP(5); break;  // K + 1 <= 151 (checked by the caller)
  }
#undef B200R_DEPTH_WARP
  B200R_LAUNCHED(BACKWARD ? "soft_depth_warp_kernel<backward>" : "soft_depth_warp_kernel<forward>");
  return B200R_OK;
}

extern "C" int b200r_soft_depth_blend_forward(const int64_t* pix_to_face, const float* zbuf, const float* dists,
                                              int32_t N, int32_t H, int32_t W, int32_t K, float sigma,
                                              const float* zfar, float zfar_value, float* out, void* stream_) {
  const int rc = depth_args(N, H, W, K);
  if (rc != B200R_OK) return rc;
  const int64_t P = (int64_t)N * H * W;
  if (P == 0) return B200R_OK;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const DepthFar far{zfar, zfar_value};
  if (K <= 8) {
    soft_depth_forward_kernel<8><<<(unsigned)blend_blocks(P, K, 0), 256, 0, stream>>>(pix_to_face, zbuf, dists, P,
                                                                                      K, 1.0f / sigma, far, out);
    B200R_LAUNCHED("soft_depth_forward_kernel");
    return B200R_OK;
  }
  return launch_depth_warp_kernel<false>(nullptr, pix_to_face, zbuf, dists, P, K, 1.0f / sigma, far, out, nullptr,
                                         nullptr, stream);
}

extern "C" int b200r_soft_depth_blend_backward(const float* grad_out, const int64_t* pix_to_face, const float* zbuf,
                                               const float* dists, int32_t N, int32_t H, int32_t W, int32_t K,
                                               float sigma, const float* zfar, float zfar_value, float* grad_zbuf,
                                               float* grad_dists, void* stream_) {
  const int rc = depth_args(N, H, W, K);
  if (rc != B200R_OK) return rc;
  const int64_t P = (int64_t)N * H * W;
  if (P == 0) return B200R_OK;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const DepthFar far{zfar, zfar_value};
  if (K <= 8) {
    soft_depth_backward_kernel<8><<<(unsigned)blend_blocks(P, K, 0), 256, 0, stream>>>(
        grad_out, pix_to_face, zbuf, dists, P, K, 1.0f / sigma, far, grad_zbuf, grad_dists);
    B200R_LAUNCHED("soft_depth_backward_kernel");
    return B200R_OK;
  }
  return launch_depth_warp_kernel<true>(grad_out, pix_to_face, zbuf, dists, P, K, 1.0f / sigma, far, nullptr,
                                        grad_zbuf, grad_dists, stream);
}

extern "C" int b200r_hard_depth_forward(const int64_t* pix_to_face, const float* zbuf, int32_t N, int32_t H, int32_t W,
                                        int32_t K, const float* zfar, float zfar_value, float* out, void* stream_) {
  const int rc = depth_args(N, H, W, K);
  if (rc != B200R_OK) return rc;
  const int64_t P = (int64_t)N * H * W;
  if (P == 0) return B200R_OK;
  hard_depth_forward_kernel<<<(unsigned)blend_blocks(P, 0, 0), 256, 0, static_cast<cudaStream_t>(stream_)>>>(
      pix_to_face, zbuf, P, K, DepthFar{zfar, zfar_value}, out);
  B200R_LAUNCHED("hard_depth_forward_kernel");
  return B200R_OK;
}

extern "C" int b200r_hard_depth_backward(const float* grad_out, const int64_t* pix_to_face, int32_t N, int32_t H,
                                         int32_t W, int32_t K, float* grad_zbuf, void* stream_) {
  const int rc = depth_args(N, H, W, K);
  if (rc != B200R_OK) return rc;
  const int64_t P = (int64_t)N * H * W;
  if (P == 0) return B200R_OK;
  hard_depth_backward_kernel<<<(unsigned)blend_blocks(P * K, 0, 0), 256, 0, static_cast<cudaStream_t>(stream_)>>>(
      grad_out, pix_to_face, P, K, grad_zbuf);
  B200R_LAUNCHED("hard_depth_backward_kernel");
  return B200R_OK;
}
