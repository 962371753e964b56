// Splatter blending: the blend of SplatterPhongShader (pytorch3d/renderer/splatter_blend.py SplatterBlender; Cole et
// al., "Differentiable Surface Rendering via Non-Differentiable Sampling"), fused into one kernel for the forward and
// two for the backward.  The reference builds (N,H,W,K,9,5) splat tensors and reduces them with a bmm; here every
// pixel gathers its 3 x 3 neighbourhood from shared memory and no intermediate has a K or a 9 dimension.
//
// Inputs after the reference's projection step: colors (N,H,W,K,3), pixel_coords_screen (N,H,W,K,3), background_mask
// (N,H,W,K).  A background slot takes the coordinates (1, 1, 1) and RGBA 0 (_prepare_pixels_and_colors).
//
// 1. Occlusion (_compute_occlusion_layers).  Depths are unfolded with zero padding, so a neighbour outside the image
//    has depth 0 in every layer.  For pixel q and direction d, p is the neighbour at (dh, dw) = (d/3 - 1, d%3 - 1):
//      A = argmin_k |p_k - q_0|,  B = argmin_k |p_0 - q_k|   (ties: the first slot, as torch's min(dim))
//      occ_d = -B if min_k |p_0 - q_k| < min_k |p_k - q_0|, else A.
// 2. Splats (_compute_splatting_colors_and_weights, _offset_splats).  The splat that pixel q receives in direction d
//    comes from the source pixel at (dh, dw) = (d%3 - 1, d/3 - 1): the TRANSPOSE of the neighbour the occlusion test
//    of direction d looked at (the reference's unfold and its gather index the directions differently; reproduced on
//    purpose, DESIGN.md section 11).  With c = floor(xy) - xy + 0.5 of the source slot and o_d = (d/3 - 1, d%3 - 1):
//      w = expf(-((c0 + o0)^2 + (c1 + o1)^2) * inv),  inv = 1.0f / (float)(2 sigma^2)  (a tensor divided by a Python
//      scalar is a product with the float reciprocal);  sw = (alpha * norm) * w,  norm = 1.05f / sum_d expf(-|o_d|^2 inv)
//    and the splat adds (sw * rgb, sw) to layer 0 if occ_d > k, layer 1 if occ_d == k, layer 2 if occ_d < k.
// 3. Compose (_normalize_and_compose_all_layers): N_l = S_l * (1 / max(W_l, 1)); out = (bg, 0), then for l = 2, 1, 0:
//    out = N_l + (1 - N_l.a) * out.  (The alpha channel of S_l is W_l: alpha is 1 wherever sw is not 0.)
// Only the order of the sums over the 9 K splats differs from the reference's bmm.
//
// Backward (gradients as autograd takes them through that chain; floor passes none, so d c / d xy = -1, and z gets 0):
//   record kernel, one thread per pixel q: recomputes the forward and writes a record of 24 floats (96 bytes):
//     E_l = (dS_l.rgb, dS_l.a + dW_l) for l = 0..2 -- the gradient of a splat's colour and weight in layer l --
//     and occ_d for the 9 directions.  dW_l passes torch.maximum: all of it above 1, half at 1, none below.
//   gather kernel, one thread per slot of source pixel s: for each direction d it reads the record of its target
//     q = s - (d%3 - 1, d/3 - 1), and with E = E_{bucket}:  dsw = E.rgb . rgb + E.a,  d rgb += E.rgb * sw,
//     d xy -= (-(dsw * norm * w) * inv) * 2 (c + o).  Every output is written once by the thread owning its slot:
//     no atomics, no zero-fill.
//
// Tiles: a CTA owns 32 x 8 pixels and stages the tile plus a one-pixel halo in shared memory, structure of arrays.
// The forward and record kernels stage up to 8 slots per pixel at once (z, c0, c1, r, g, b, alpha * norm): for K <= 8
// every input is read once and both sweeps (depth minima, then splat sums) run on the staged slots.  Larger K (up to
// 150) runs in chunks of 8 slots, first the depth minima over all chunks, then the splat sums over all chunks.
#include "common.cuh"
#include "raster_math.cuh"

namespace b200r {

constexpr int kSplatTileW = 32, kSplatTileH = 8;
constexpr int kSplatThreads = kSplatTileW * kSplatTileH;  // 256: one warp per tile row
constexpr int kSplatHaloW = kSplatTileW + 2, kSplatHaloH = kSplatTileH + 2;
constexpr int kSplatHalo = kSplatHaloW * kSplatHaloH;  // 340 staged pixels
constexpr int kSplatChunk = 8;                          // slots staged at once
enum SplatField { kZ, kC0, kC1, kR, kG, kB, kAlpha, kSplatFields };
constexpr int kRecord = 24;       // floats per pixel record (96 bytes): E_0, E_1, E_2 (4 each), occ_0..8, 3 unused
constexpr int kRecordOcc = 12;    // first occ field
constexpr int kRecordFields = 21;  // fields the gather kernel stages

struct SplatArgs {
  float inv;        // 1.0f / (float)(2 sigma^2)
  const float* bg;  // device (3,) or null: then bg0..2
  float bg0, bg1, bg2;
};

// 1.05 / sum_d exp(-|o_d|^2 / (2 sigma^2)) in the reference's float operations, summed in direction order.
__device__ __forceinline__ float splat_norm(float inv) {
  float s = 0.0f;
#pragma unroll
  for (int d = 0; d < 9; ++d) {
    const int m = (d / 3 - 1) * (d / 3 - 1) + (d % 3 - 1) * (d % 3 - 1);
    s = fadd(s, expf(fmul(-(float)m, inv)));
  }
  return fdiv(1.05f, s);
}

// floor(x) - x + 0.5: the offset of a coordinate from its pixel centre.
__device__ __forceinline__ float centre_offset(float x) { return fadd(fsub(floorf(x), x), 0.5f); }

// exp(-((c0 + o0)^2 + (c1 + o1)^2) * inv); e0 / e1 return c + o.
__device__ __forceinline__ float splat_kernel(float c0, float c1, int d, float inv, float& e0, float& e1) {
  e0 = fadd(c0, (float)(d / 3 - 1));
  e1 = fadd(c1, (float)(d % 3 - 1));
  const float dist2 = fadd(fmul(e0, e0), fmul(e1, e1));
  return expf(fmul(-dist2, inv));
}

// Bucket of slot k under occlusion id occ: 0 above the matched slot (occ > k), 1 at it, 2 below.
__device__ __forceinline__ int bucket_of(int occ, int k) { return occ > k ? 0 : (occ == k ? 1 : 2); }

// Stage slots [k0, k0 + kc) of the tile's halo: field f of slot kk of halo pixel pos at sm[(f * kcs + kk) * 340 + pos].
// Pixels outside the image stage depth 0 (the reference's zero padding) and alpha 0 (no splat); background slots stage
// depth 1, c = floor(1) - 1 + 0.5 = 0.5 and alpha 0.  `full` = false stages the depths alone.
__device__ __forceinline__ void stage_slots(float* sm, int kcs, const float* __restrict__ colors,
                                            const float* __restrict__ coords, const uint8_t* __restrict__ mask,
                                            int64_t n, int H, int W, int K, int y0, int x0, int k0, int kc, bool full,
                                            float norm) {
  for (int i = threadIdx.x; i < kSplatHalo * kc; i += kSplatThreads) {
    const int pos = i / kc, kk = i - pos * kc;
    const int gy = y0 + pos / kSplatHaloW - 1, gx = x0 + pos % kSplatHaloW - 1;
    float z = 0.0f, c0 = 0.0f, c1 = 0.0f, r = 0.0f, g = 0.0f, b = 0.0f, a = 0.0f;
    if (gy >= 0 && gy < H && gx >= 0 && gx < W) {
      const int64_t slot = ((n * H + gy) * W + gx) * K + k0 + kk;
      if (__ldg(mask + slot)) {
        z = 1.0f;
        c0 = c1 = 0.5f;
      } else {
        z = __ldg(coords + 3 * slot + 2);
        if (full) {
          c0 = centre_offset(__ldg(coords + 3 * slot));
          c1 = centre_offset(__ldg(coords + 3 * slot + 1));
          r = __ldg(colors + 3 * slot);
          g = __ldg(colors + 3 * slot + 1);
          b = __ldg(colors + 3 * slot + 2);
          a = norm;  // alpha (1) * norm
        }
      }
    }
    float* p = sm + kk * kSplatHalo + pos;
    p[kZ * kcs * kSplatHalo] = z;
    if (full) {
      p[kC0 * kcs * kSplatHalo] = c0;
      p[kC1 * kcs * kSplatHalo] = c1;
      p[kR * kcs * kSplatHalo] = r;
      p[kG * kcs * kSplatHalo] = g;
      p[kB * kcs * kSplatHalo] = b;
      p[kAlpha * kcs * kSplatHalo] = a;
    }
  }
}

// Forward (RECORD = false: writes out) and the backward's record kernel (RECORD = true: reads grad_out, writes the
// record).  One thread per pixel of a 32 x 8 tile; image n0 + blockIdx.z, tile row ty0 + blockIdx.y.
template <bool RECORD>
__global__ void __launch_bounds__(kSplatThreads)
    splatter_blend_pixel_kernel(const float* __restrict__ colors, const float* __restrict__ coords,
                                const uint8_t* __restrict__ mask, int n0, int ty0, int H, int W, int K, SplatArgs s,
                                const float* __restrict__ grad_out, float* __restrict__ out) {
  extern __shared__ float sm[];
  const int kcs = K < kSplatChunk ? K : kSplatChunk;  // slots per staged chunk
  const int nchunk = (K + kSplatChunk - 1) / kSplatChunk;
  const int64_t n = n0 + blockIdx.z;  // unsigned: n >= 0 is known to the compiler
  const int y0 = (ty0 + blockIdx.y) * kSplatTileH, x0 = blockIdx.x * kSplatTileW;
  const int tx = threadIdx.x % kSplatTileW, ty = threadIdx.x / kSplatTileW;
  const float norm = splat_norm(s.inv);
  const int self = (ty + 1) * kSplatHaloW + tx + 1;
  auto Z = [&](int kk, int pos) { return sm[(kZ * kcs + kk) * kSplatHalo + pos]; };

  // sweep 1: the depth minima of the 9 directions over all K slots
  float q0 = 0.0f, p0[9], minA[9], minB[9];
  int argA[9], argB[9];
  for (int c = 0; c < nchunk; ++c) {
    const int k0 = c * kSplatChunk, kc = min(kSplatChunk, K - k0);
    if (c > 0) __syncthreads();
    stage_slots(sm, kcs, colors, coords, mask, n, H, W, K, y0, x0, k0, kc, nchunk == 1, norm);
    __syncthreads();
    for (int kk = 0; kk < kc; ++kk) {
      const int k = k0 + kk;
      const float qk = Z(kk, self);
      if (k == 0) {
        q0 = qk;
#pragma unroll
        for (int d = 0; d < 9; ++d) p0[d] = Z(0, self + (d / 3 - 1) * kSplatHaloW + (d % 3 - 1));
      }
#pragma unroll
      for (int d = 0; d < 9; ++d) {
        const float pk = Z(kk, self + (d / 3 - 1) * kSplatHaloW + (d % 3 - 1));
        const float a = fabsf(fsub(pk, q0)), b = fabsf(fsub(p0[d], qk));
        if (k == 0 || a < minA[d]) {  // strictly smaller: ties keep the first slot
          minA[d] = a;
          argA[d] = k;
        }
        if (k == 0 || b < minB[d]) {
          minB[d] = b;
          argB[d] = k;
        }
      }
    }
  }
  int occ[9];
#pragma unroll
  for (int d = 0; d < 9; ++d) occ[d] = minB[d] < minA[d] ? -argB[d] : argA[d];

  // sweep 2: the splats received from the 9 source pixels, summed per layer: rgb and weight
  float S[3][4];
#pragma unroll
  for (int l = 0; l < 3; ++l) S[l][0] = S[l][1] = S[l][2] = S[l][3] = 0.0f;
  for (int c = 0; c < nchunk; ++c) {
    const int k0 = c * kSplatChunk, kc = min(kSplatChunk, K - k0);
    if (nchunk > 1) {
      __syncthreads();
      stage_slots(sm, kcs, colors, coords, mask, n, H, W, K, y0, x0, k0, kc, true, norm);
      __syncthreads();
    }
    for (int kk = 0; kk < kc; ++kk) {
      const int k = k0 + kk;
      const float* f = sm + kk * kSplatHalo;
#pragma unroll
      for (int d = 0; d < 9; ++d) {
        const int src = self + (d % 3 - 1) * kSplatHaloW + (d / 3 - 1);
        const float A = f[kAlpha * kcs * kSplatHalo + src];
        // A source slot without a face splats exactly 0; where the whole warp's sources are such slots (most of the
        // deeper layers of a typical frame) the adds are skipped, which changes no bit of the sums.
        if (!__any_sync(0xffffffffu, A != 0.0f)) continue;
        float e0, e1;
        const float w = splat_kernel(f[kC0 * kcs * kSplatHalo + src], f[kC1 * kcs * kSplatHalo + src], d, s.inv,
                                     e0, e1);
        const float sw = fmul(A, w);
        const float sr = fmul(sw, f[kR * kcs * kSplatHalo + src]);
        const float sg = fmul(sw, f[kG * kcs * kSplatHalo + src]);
        const float sb = fmul(sw, f[kB * kcs * kSplatHalo + src]);
        const int l = bucket_of(occ[d], k);
        if (l == 0) {
          S[0][0] = fadd(S[0][0], sr); S[0][1] = fadd(S[0][1], sg); S[0][2] = fadd(S[0][2], sb);
          S[0][3] = fadd(S[0][3], sw);
        } else if (l == 1) {
          S[1][0] = fadd(S[1][0], sr); S[1][1] = fadd(S[1][1], sg); S[1][2] = fadd(S[1][2], sb);
          S[1][3] = fadd(S[1][3], sw);
        } else {
          S[2][0] = fadd(S[2][0], sr); S[2][1] = fadd(S[2][1], sg); S[2][2] = fadd(S[2][2], sb);
          S[2][3] = fadd(S[2][3], sw);
        }
      }
    }
  }

  const int y = y0 + ty, x = x0 + tx;
  if (y >= H || x >= W) return;
  const int64_t pix = (n * H + y) * W + x;
  const float bg0 = s.bg ? s.bg[0] : s.bg0, bg1 = s.bg ? s.bg[1] : s.bg1, bg2 = s.bg ? s.bg[2] : s.bg2;
  // normalise and compose: o[0] = (bg, 0), o[i + 1] = N_{2 - i} + (1 - N_{2 - i}.a) o[i]
  float inv_l[3], Nl[3][4], o[4][4] = {{bg0, bg1, bg2, 0.0f}};
#pragma unroll
  for (int l = 0; l < 3; ++l) {
    inv_l[l] = fdiv(1.0f, fmaxf(S[l][3], 1.0f));
#pragma unroll
    for (int j = 0; j < 4; ++j) Nl[l][j] = fmul(S[l][j], inv_l[l]);
  }
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const int l = 2 - i;
    const float t = fsub(1.0f, Nl[l][3]);
#pragma unroll
    for (int j = 0; j < 4; ++j) o[i + 1][j] = fadd(Nl[l][j], fmul(t, o[i][j]));
  }
  if constexpr (!RECORD) {
    float* op = out + 4 * pix;
    const float4 v = make_float4(o[3][0], o[3][1], o[3][2], o[3][3]);
    if ((reinterpret_cast<uintptr_t>(op) & 15u) == 0) {
      *reinterpret_cast<float4*>(op) = v;
    } else {
      op[0] = v.x; op[1] = v.y; op[2] = v.z; op[3] = v.w;
    }
  } else {
    float g[4] = {grad_out[4 * pix], grad_out[4 * pix + 1], grad_out[4 * pix + 2], grad_out[4 * pix + 3]};
    float rec[kRecord];
#pragma unroll
    for (int l = 0; l < 3; ++l) {  // l = 0 is composed last: its gradient is the first to come back
      // out_l = N_l + (1 - N_l.a) o_below, o_below = o[2 - l]
      float ea = 0.0f;
#pragma unroll
      for (int j = 0; j < 4; ++j) ea -= g[j] * o[2 - l][j];
      const float dNa = g[3] + ea;
      const float dinv = g[0] * S[l][0] + g[1] * S[l][1] + g[2] * S[l][2] + dNa * S[l][3];
      const float W = S[l][3];
      const float dmax = -dinv * inv_l[l] * inv_l[l];  // d (1 / m) / dm = -1 / m^2
      const float dW = W > 1.0f ? dmax : (W == 1.0f ? 0.5f * dmax : 0.0f);
      rec[4 * l] = g[0] * inv_l[l];
      rec[4 * l + 1] = g[1] * inv_l[l];
      rec[4 * l + 2] = g[2] * inv_l[l];
      rec[4 * l + 3] = dNa * inv_l[l] + dW;
      const float t = 1.0f - Nl[l][3];
#pragma unroll
      for (int j = 0; j < 4; ++j) g[j] *= t;
    }
#pragma unroll
    for (int d = 0; d < 9; ++d) rec[kRecordOcc + d] = (float)occ[d];
    rec[21] = rec[22] = rec[23] = 0.0f;
    float4* rp = reinterpret_cast<float4*>(out + kRecord * pix);  // the workspace: 16-byte aligned
#pragma unroll
    for (int i = 0; i < kRecord / 4; ++i) rp[i] = make_float4(rec[4 * i], rec[4 * i + 1], rec[4 * i + 2], rec[4 * i + 3]);
  }
}

// Backward gather: one thread per slot of a 32 x 8 tile (k fastest, so consecutive threads touch consecutive memory);
// the records of the tile and its halo are staged in shared memory (records outside the image stage as 0: their
// splats were dropped by the reference's padding).
__global__ void __launch_bounds__(kSplatThreads)
    splatter_blend_gather_kernel(const float* __restrict__ colors, const float* __restrict__ coords,
                                 const uint8_t* __restrict__ mask, int n0, int ty0, int H, int W, int K, SplatArgs s,
                                 const float* __restrict__ record, float* __restrict__ grad_colors,
                                 float* __restrict__ grad_coords) {
  __shared__ float rs[kRecordFields * kSplatHalo];
  const int64_t n = n0 + blockIdx.z;  // unsigned: n >= 0 is known to the compiler
  const int y0 = (ty0 + blockIdx.y) * kSplatTileH, x0 = blockIdx.x * kSplatTileW;
  const float norm = splat_norm(s.inv);
  for (int i = threadIdx.x; i < kSplatHalo * kRecordFields; i += kSplatThreads) {
    const int pos = i / kRecordFields, f = i - pos * kRecordFields;
    const int gy = y0 + pos / kSplatHaloW - 1, gx = x0 + pos % kSplatHaloW - 1;
    rs[f * kSplatHalo + pos] =
        gy >= 0 && gy < H && gx >= 0 && gx < W ? __ldg(record + ((n * H + gy) * W + gx) * kRecord + f) : 0.0f;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < kSplatThreads * K; i += kSplatThreads) {
    const int p = i / K, k = i - p * K;
    const int ty = p / kSplatTileW, tx = p % kSplatTileW;
    const int y = y0 + ty, x = x0 + tx;
    if (y >= H || x >= W) continue;
    const int64_t slot = ((n * H + y) * W + x) * K + k;
    float gr = 0.0f, gg = 0.0f, gb = 0.0f, gx0 = 0.0f, gx1 = 0.0f;
    if (!__ldg(mask + slot)) {
      const float c0 = centre_offset(__ldg(coords + 3 * slot)), c1 = centre_offset(__ldg(coords + 3 * slot + 1));
      const float r = __ldg(colors + 3 * slot), g = __ldg(colors + 3 * slot + 1), b = __ldg(colors + 3 * slot + 2);
      const int self = (ty + 1) * kSplatHaloW + tx + 1;
#pragma unroll
      for (int d = 0; d < 9; ++d) {
        const int q = self - (d % 3 - 1) * kSplatHaloW - (d / 3 - 1);  // the pixel this splat lands on
        const int l = bucket_of((int)rs[(kRecordOcc + d) * kSplatHalo + q], k);
        const float* E = rs + 4 * l * kSplatHalo + q;
        const float Er = E[0], Eg = E[kSplatHalo], Eb = E[2 * kSplatHalo], Ea = E[3 * kSplatHalo];
        float e0, e1;
        const float w = splat_kernel(c0, c1, d, s.inv, e0, e1);
        const float sw = fmul(norm, w);
        const float dsw = Er * r + Eg * g + Eb * b + Ea;
        gr += Er * sw;
        gg += Eg * sw;
        gb += Eb * sw;
        const float ddist2 = -((dsw * norm) * w * s.inv);
        gx0 -= ddist2 * 2.0f * e0;
        gx1 -= ddist2 * 2.0f * e1;
      }
    }
    grad_colors[3 * slot] = gr;
    grad_colors[3 * slot + 1] = gg;
    grad_colors[3 * slot + 2] = gb;
    grad_coords[3 * slot] = gx0;
    grad_coords[3 * slot + 1] = gx1;
    grad_coords[3 * slot + 2] = 0.0f;
  }
}

}  // namespace b200r

using namespace b200r;

static int splatter_args(int32_t N, int32_t H, int32_t W, int32_t K, double sigma, const float* background,
                         const float* background_value, SplatArgs* s) {
  if (N < 0 || H < 0 || W < 0 || K < 0) return fail(B200R_ERR_INVALID_ARGUMENT, "negative size");
  if (K > B200R_MAX_K) return fail(B200R_ERR_INVALID_ARGUMENT, "Must have faces_per_pixel <= 150");
  if (!(sigma > 0.0)) return fail(B200R_ERR_INVALID_ARGUMENT, "Only positive standard deviations make sense.");
  if (background == nullptr && background_value == nullptr)
    return fail(B200R_ERR_INVALID_ARGUMENT, "a background colour is required");
  s->inv = 1.0f / (float)(2.0 * sigma * sigma);
  s->bg = background;
  s->bg0 = background ? 0.0f : background_value[0];
  s->bg1 = background ? 0.0f : background_value[1];
  s->bg2 = background ? 0.0f : background_value[2];
  return B200R_OK;
}

// Both kernels are launched over the images and tile rows in chunks of at most 65535, the limit of grid.y and grid.z;
// each launch gets its first image n0 and first tile row ty0.  f(grid, n0, ty0) launches one chunk and returns its
// status; the first failure stops the launches.
template <typename Launch>
static int for_each_splatter_chunk(int32_t N, int32_t H, int32_t W, Launch f) {
  constexpr int kMaxGridYZ = 65535;
  const int TX = (W + kSplatTileW - 1) / kSplatTileW, TY = (H + kSplatTileH - 1) / kSplatTileH;
  for (int n0 = 0; n0 < N; n0 += kMaxGridYZ)
    for (int ty0 = 0; ty0 < TY; ty0 += kMaxGridYZ) {
      const int rc = f(dim3((unsigned)TX, (unsigned)min(TY - ty0, kMaxGridYZ), (unsigned)min(N - n0, kMaxGridYZ)),
                       n0, ty0);
      if (rc != B200R_OK) return rc;
    }
  return B200R_OK;
}

template <bool RECORD>
static int launch_pixel_kernel(const float* colors, const float* coords, const uint8_t* mask, int32_t N, int32_t H,
                               int32_t W, int32_t K, const SplatArgs& s, const float* grad_out, float* out,
                               cudaStream_t stream) {
  const int kcs = K < kSplatChunk ? K : kSplatChunk;
  const size_t smem = (size_t)kSplatFields * kcs * kSplatHalo * sizeof(float);  // 76,160 bytes at K >= 8
  B200R_CUDA_OK(cudaFuncSetAttribute(splatter_blend_pixel_kernel<RECORD>,
                                     cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  return for_each_splatter_chunk(N, H, W, [&](dim3 grid, int n0, int ty0) {
    splatter_blend_pixel_kernel<RECORD><<<grid, kSplatThreads, smem, stream>>>(colors, coords, mask, n0, ty0, H, W, K,
                                                                               s, grad_out, out);
    B200R_LAUNCHED(RECORD ? "splatter_blend_pixel_kernel<record>" : "splatter_blend_pixel_kernel<forward>");
    return B200R_OK;
  });
}

extern "C" int b200r_splatter_blend_forward(const float* colors, const float* pixel_coords_screen,
                                            const uint8_t* background_mask, int32_t N, int32_t H, int32_t W,
                                            int32_t K, double sigma, const float* background,
                                            const float* background_value, float* out, void* stream_) {
  SplatArgs s;
  int rc = splatter_args(N, H, W, K, sigma, background, background_value, &s);
  if (rc != B200R_OK) return rc;
  if (K == 0) return fail(B200R_ERR_INVALID_ARGUMENT, "faces_per_pixel must be at least 1");
  if ((int64_t)N * H * W == 0) return B200R_OK;
  return launch_pixel_kernel<false>(colors, pixel_coords_screen, background_mask, N, H, W, K, s, nullptr, out,
                                    static_cast<cudaStream_t>(stream_));
}

extern "C" size_t b200r_splatter_blend_workspace_bytes(int32_t N, int32_t H, int32_t W) {
  if (N <= 0 || H <= 0 || W <= 0) return 0;
  return (size_t)N * H * W * kRecord * sizeof(float);
}

extern "C" int b200r_splatter_blend_backward(const float* grad_out, const float* colors,
                                             const float* pixel_coords_screen, const uint8_t* background_mask,
                                             int32_t N, int32_t H, int32_t W, int32_t K, double sigma,
                                             const float* background, const float* background_value, void* workspace,
                                             size_t workspace_bytes, float* grad_colors,
                                             float* grad_pixel_coords_screen, void* stream_) {
  SplatArgs s;
  int rc = splatter_args(N, H, W, K, sigma, background, background_value, &s);
  if (rc != B200R_OK) return rc;
  if (K == 0) return fail(B200R_ERR_INVALID_ARGUMENT, "faces_per_pixel must be at least 1");
  if ((int64_t)N * H * W == 0) return B200R_OK;
  if (workspace == nullptr || workspace_bytes < b200r_splatter_blend_workspace_bytes(N, H, W) ||
      (reinterpret_cast<uintptr_t>(workspace) & 15u) != 0)
    return fail(B200R_ERR_INVALID_ARGUMENT, "splatter_blend_backward: workspace too small or not 16-byte aligned");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  float* record = static_cast<float*>(workspace);
  rc = launch_pixel_kernel<true>(colors, pixel_coords_screen, background_mask, N, H, W, K, s, grad_out, record, stream);
  if (rc != B200R_OK) return rc;
  return for_each_splatter_chunk(N, H, W, [&](dim3 grid, int n0, int ty0) {
    splatter_blend_gather_kernel<<<grid, kSplatThreads, 0, stream>>>(colors, pixel_coords_screen, background_mask, n0,
                                                                     ty0, H, W, K, s, record, grad_colors,
                                                                     grad_pixel_coords_screen);
    B200R_LAUNCHED("splatter_blend_gather_kernel");
    return B200R_OK;
  });
}
