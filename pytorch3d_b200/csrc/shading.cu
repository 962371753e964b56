// Phong and flat shading, forward and backward (DESIGN.md section 12), and Gouraud shading (section 16, below).
//
// What pytorch3d/renderer/mesh/shading.py (_phong_shading_with_pixels, phong_shading, flat_shading) computes with the
// light models of renderer/lighting.py (PointLights, DirectionalLights, AmbientLights), per rasterized slot:
//
//   p, n   = barycentric interpolation of the face's corner positions / normals   (phong)
//            the face's centroid / normal                                          (flat)
//            0 where pix_to_face < 0
//   L      = location - p (point) | direction (directional)
//   cos    = <normalize(n), normalize(L)>,  normalize(x) = x / max(|x|, 1e-6)
//   diffuse  = md * (ld * relu(cos))
//   R      = -normalize(L) + 2 * (cos * normalize(n))
//   alpha  = relu(<normalize(cam - p), R>) * (cos > 0)
//   specular = ms * (ls * alpha^shininess)
//   colour = (ambient + diffuse) * texel + specular
//
// The chain of the reference writes about two dozen (N,H,W,K[,3]) tensors; here the forward is one kernel that reads
// the slot's face index, barycentrics and texel and writes the colour (and on request the interpolated position), and
// the backward is one kernel plus, when a light, material or camera tensor requires grad, a small kernel that sums the
// per-CTA partial sums of the per-batch parameter gradients in a fixed order.  The per-batch constants arrive as one
// float32 row of B200R_SHADING_PARAMS values per image (include/b200_raster.h).  Nothing synchronises the host.
//
// Positions use the FMA chain of interp_face_attrs_forward_kernel, so they are bit-identical to
// interpolate_face_attributes.  The final colour is composed with explicitly rounded products and sums, in the
// reference's order, so that slots whose lighting terms are exact (background slots, shininess 0) give torch's bits.
// The non-differentiable points follow torch's backward formulas: relu and the (cos > 0) mask pass no gradient at 0,
// clamp_min passes it where |x| >= eps, the norm's gradient is 0 at a zero vector, pow gives 0 to the base where the
// exponent is 0 and 0 to the exponent where the base is 0 and the exponent >= 0.
#include "common.cuh"
#include "raster_math.cuh"

namespace b200r {
namespace {

constexpr int kP = B200R_SHADING_PARAMS;
enum : int { AMB = 0, LD = 3, LS = 6, MD = 9, MS = 12, LOC = 15, CAM = 18, SHIN = 21 };
constexpr float kNormEps = 1e-6f;  // F.normalize(..., eps=1e-6) in lighting.py
constexpr int kThreads = 256;

struct V3 {
  float x, y, z;
};
__device__ __forceinline__ V3 ld3(const float* p) { return {__ldg(p), __ldg(p + 1), __ldg(p + 2)}; }
__device__ __forceinline__ float dot3(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ V3 sub3(V3 a, V3 b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }

// fma(w2,a2, fma(w1,a1, fma(w0,a0,0))) per component, corners 3 floats apart: interp_face_attrs_forward_kernel's chain
__device__ __forceinline__ V3 interp3(const float* a, float w0, float w1, float w2) {
  V3 r;
  r.x = ffma(w2, __ldg(a + 6), ffma(w1, __ldg(a + 3), ffma(w0, __ldg(a + 0), 0.0f)));
  r.y = ffma(w2, __ldg(a + 7), ffma(w1, __ldg(a + 4), ffma(w0, __ldg(a + 1), 0.0f)));
  r.z = ffma(w2, __ldg(a + 8), ffma(w1, __ldg(a + 5), ffma(w0, __ldg(a + 2), 0.0f)));
  return r;
}

struct Unit {  // u = x / c with r = |x|, c = max(r, eps)
  V3 u;
  float r, c;
};
__device__ __forceinline__ Unit normalize3(V3 x) {
  const float r = sqrtf(x.x * x.x + x.y * x.y + x.z * x.z);
  const float c = fmaxf(r, kNormEps);
  return {{x.x / c, x.y / c, x.z / c}, r, c};
}
// Gradient of x / max(|x|, eps) for the upstream g.
__device__ __forceinline__ V3 normalize3_backward(V3 x, const Unit& n, V3 g) {
  V3 gx = {g.x / n.c, g.y / n.c, g.z / n.c};
  if (n.r >= kNormEps) {  // clamp_min passes the gradient; r > 0 here, so the norm's gradient is x / r
    const float s = (-(g.x * x.x + g.y * x.y + g.z * x.z) / (n.c * n.c)) / n.r;
    gx.x += x.x * s;
    gx.y += x.y * s;
    gx.z += x.z * s;
  }
  return gx;
}

// Every intermediate of one slot's lighting that the backward needs.
struct Lit {
  V3 L, V;
  Unit nn, ln, vn;
  V3 R;
  float cos, angle, dot_vr, alpha, pw, shin;
};

template <int LIGHT>
__device__ __forceinline__ void light_slot(V3 p, V3 n, const float* __restrict__ prm, Lit& t) {
  t.shin = __ldg(prm + SHIN);
  if (LIGHT == B200R_LIGHT_AMBIENT) {
    t.angle = 0.0f;
    t.pw = 0.0f;
    return;
  }
  const V3 loc = ld3(prm + LOC);
  t.L = LIGHT == B200R_LIGHT_POINT ? sub3(loc, p) : loc;
  t.nn = normalize3(n);
  t.ln = normalize3(t.L);
  t.cos = dot3(t.nn.u, t.ln.u);
  t.angle = t.cos > 0.0f ? t.cos : 0.0f;
  t.V = sub3(ld3(prm + CAM), p);
  t.vn = normalize3(t.V);
  const float c2 = 2.0f;
  t.R = {-t.ln.u.x + c2 * (t.cos * t.nn.u.x), -t.ln.u.y + c2 * (t.cos * t.nn.u.y),
         -t.ln.u.z + c2 * (t.cos * t.nn.u.z)};
  t.dot_vr = dot3(t.vn.u, t.R);
  const float rel = t.dot_vr > 0.0f ? t.dot_vr : 0.0f;
  t.alpha = rel * (t.cos > 0.0f ? 1.0f : 0.0f);
  t.pw = powf(t.alpha, t.shin);
}

// (ambient + md * (ld * angle)) * texel + ms * (ls * pw), every product and sum rounded, in the reference's order
__device__ __forceinline__ float compose(const float* __restrict__ prm, int c, float angle, float pw, float texel) {
  const float diffuse = fmul(__ldg(prm + MD + c), fmul(__ldg(prm + LD + c), angle));
  const float specular = fmul(__ldg(prm + MS + c), fmul(__ldg(prm + LS + c), pw));
  return fadd(fmul(fadd(__ldg(prm + AMB + c), diffuse), texel), specular);
}

template <bool FLAT, int LIGHT>
__device__ __forceinline__ void slot_geometry(int64_t f, int64_t s, const float* __restrict__ bary,
                                              const float* __restrict__ face_pos, const float* __restrict__ face_nrm,
                                              bool want_pos, V3& p, V3& n, float (&w)[3]) {
  p = {0.0f, 0.0f, 0.0f};
  n = {0.0f, 0.0f, 0.0f};
  w[0] = w[1] = w[2] = 0.0f;
  if (f < 0) return;
  const bool need_pos = want_pos || LIGHT != B200R_LIGHT_AMBIENT;
  const bool need_nrm = LIGHT != B200R_LIGHT_AMBIENT;
  if (FLAT) {
    if (need_pos) p = ld3(face_pos + f * 3);
    if (need_nrm) n = ld3(face_nrm + f * 3);
  } else {
    w[0] = __ldg(bary + s * 3 + 0);
    w[1] = __ldg(bary + s * 3 + 1);
    w[2] = __ldg(bary + s * 3 + 2);
    if (need_pos) p = interp3(face_pos + f * 9, w[0], w[1], w[2]);
    if (need_nrm) n = interp3(face_nrm + f * 9, w[0], w[1], w[2]);
  }
}

template <bool FLAT, int LIGHT>
__global__ void __launch_bounds__(kThreads)
    shading_forward_kernel(const int64_t* __restrict__ pix_to_face, const float* __restrict__ bary,
                           const float* __restrict__ face_pos, const float* __restrict__ face_nrm,
                           const float* __restrict__ texels, const float* __restrict__ params, int64_t total,
                           int64_t slots_per_image, float* __restrict__ colors, float* __restrict__ positions) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; s < total; s += stride) {
    const int64_t f = __ldg(pix_to_face + s);
    const float* prm = params + (s / slots_per_image) * kP;
    V3 p, n;
    float w[3];
    slot_geometry<FLAT, LIGHT>(f, s, bary, face_pos, face_nrm, positions != nullptr, p, n, w);
    if (positions != nullptr) {
      positions[s * 3 + 0] = p.x;
      positions[s * 3 + 1] = p.y;
      positions[s * 3 + 2] = p.z;
    }
    Lit t;
    light_slot<LIGHT>(p, n, prm, t);
    const V3 tx = ld3(texels + s * 3);
    colors[s * 3 + 0] = compose(prm, 0, t.angle, t.pw, tx.x);
    colors[s * 3 + 1] = compose(prm, 1, t.angle, t.pw, tx.y);
    colors[s * 3 + 2] = compose(prm, 2, t.angle, t.pw, tx.z);
  }
}

// Gradient of one point's colour (ambient + diffuse) * texel + specular (light_slot, compose) for the upstream g: the
// texel gradient goes to row i of gtex (i * 3 + c; gtex may be null), the position and normal gradients are added into gp and gn
// (left as they are for ambient light), and with PARAMS every parameter gradient is added into acc.
template <int LIGHT, bool PARAMS>
__device__ __forceinline__ void lighting_backward(const float* prm, const Lit& t, V3 n, V3 g, V3 tx, float* gtex,
                                                  int64_t i, V3& gp, V3& gn, float (&acc)[kP]) {
  const float gc[3] = {g.x, g.y, g.z}, tc[3] = {tx.x, tx.y, tx.z};
  float g_angle = 0.0f, g_pw = 0.0f;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float md = __ldg(prm + MD + c), ld = __ldg(prm + LD + c);
    const float ms = __ldg(prm + MS + c), ls = __ldg(prm + LS + c);
    const float ldang = fmul(ld, t.angle), lspow = fmul(ls, t.pw);
    if (gtex != nullptr) gtex[i * 3 + c] = fmul(gc[c], fadd(__ldg(prm + AMB + c), fmul(md, ldang)));
    const float gd = gc[c] * tc[c];  // gradient of the diffuse colour
    const float g_ldang = gd * md, g_lspow = gc[c] * ms;
    if (PARAMS) {
      acc[AMB + c] += gd;
      acc[MD + c] += gd * ldang;
      acc[LD + c] += g_ldang * t.angle;
      acc[MS + c] += gc[c] * lspow;
      acc[LS + c] += g_lspow * t.pw;
    }
    g_angle += g_ldang * ld;
    g_pw += g_lspow * ls;
  }
  if (LIGHT != B200R_LIGHT_AMBIENT) {
    // pow: no gradient to the base where the exponent is 0, none to the exponent where the base is 0 (exponent >= 0)
    const float g_alpha = t.shin == 0.0f ? 0.0f : g_pw * (t.shin * powf(t.alpha, t.shin - 1.0f));
    if (PARAMS && !(t.alpha == 0.0f && t.shin >= 0.0f)) acc[SHIN] += g_pw * (t.pw * logf(t.alpha));
    // alpha = relu(<vn, R>) * (cos > 0): relu and the mask pass nothing at 0
    const float g_dot = (t.cos > 0.0f && t.dot_vr > 0.0f) ? g_alpha : 0.0f;
    const V3 g_vn = {g_dot * t.R.x, g_dot * t.R.y, g_dot * t.R.z};
    const V3 g_R = {g_dot * t.vn.u.x, g_dot * t.vn.u.y, g_dot * t.vn.u.z};
    // R = -ln + 2 * (cos * nn); angle = relu(cos); cos = <nn, ln>
    const float g_cos = 2.0f * dot3(g_R, t.nn.u) + (t.angle > 0.0f ? g_angle : 0.0f);
    const V3 g_nn = {2.0f * g_R.x * t.cos + g_cos * t.ln.u.x, 2.0f * g_R.y * t.cos + g_cos * t.ln.u.y,
                     2.0f * g_R.z * t.cos + g_cos * t.ln.u.z};
    const V3 g_ln = {g_cos * t.nn.u.x - g_R.x, g_cos * t.nn.u.y - g_R.y, g_cos * t.nn.u.z - g_R.z};
    gn = normalize3_backward(n, t.nn, g_nn);
    const V3 g_L = normalize3_backward(t.L, t.ln, g_ln);
    const V3 g_V = normalize3_backward(t.V, t.vn, g_vn);
    gp = {-g_V.x, -g_V.y, -g_V.z};
    if (LIGHT == B200R_LIGHT_POINT) {
      gp = {gp.x - g_L.x, gp.y - g_L.y, gp.z - g_L.z};
    }
    if (PARAMS) {
      acc[LOC + 0] += g_L.x;
      acc[LOC + 1] += g_L.y;
      acc[LOC + 2] += g_L.z;
      acc[CAM + 0] += g_V.x;
      acc[CAM + 1] += g_V.y;
      acc[CAM + 2] += g_V.z;
    }
  }
}

// Merges one warp's per-lane gradients (M floats each) over the lanes that hold the same key: one MATCH, then pointer
// jumping as in the rasterizer's backward (DESIGN.md section 6).  Returns true on the one lane per distinct key >= 0
// that holds its key's sum.  Every lane of the warp must call it; lanes without a key pass key = -1.
template <int M>
__device__ __forceinline__ bool warp_merge(int64_t key, float (&g)[M]) {
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
  return key >= 0 && lane == __ffs((int)grp) - 1;
}

// Adds one warp's per-slot face gradients into `out` (M floats per face), so every distinct face of the warp costs one
// set of M atomics.  Every lane of the warp must call it; lanes without a face pass face = -1.
template <int M>
__device__ __forceinline__ void warp_scatter(float* __restrict__ out, int64_t face, float (&g)[M]) {
  if (warp_merge<M>(face, g)) {
    float* o = out + face * M;
#pragma unroll
    for (int i = 0; i < M; ++i) atomicAdd(o + i, g[i]);
  }
}

struct BackwardArgs {
  const float* grad_colors;
  const float* grad_positions;  // may be null
  const int64_t* pix_to_face;
  const float* bary;
  const float* face_pos;
  const float* face_nrm;
  const float* texels;
  const float* params;
  int64_t slots_per_image;
  float* grad_texels;    // may be null
  float* grad_bary;      // may be null (and is, in flat mode)
  float* grad_face_pos;  // may be null
  float* grad_face_nrm;  // may be null
  float* partials;       // (N, gridDim.x, kP) when PARAMS
};

// The CTA's sum of every thread's acc, written to row[0:kP]: a fixed-order reduction, butterfly within warps, then
// warps 0..7 in order.  Every thread of the CTA must call it.
__device__ __forceinline__ void store_partial_row(const float (&acc)[kP], float* row) {
  __shared__ float red[kThreads / 32][kP];
#pragma unroll
  for (int i = 0; i < kP; ++i) {
    float v = acc[i];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5][i] = v;
  }
  __syncthreads();
  if (threadIdx.x < kP) {
    float v = 0.0f;
#pragma unroll
    for (int wi = 0; wi < kThreads / 32; ++wi) v += red[wi][threadIdx.x];
    row[threadIdx.x] = v;
  }
}

// grid (blocks per image, N): a CTA only sees the slots of one image, so its parameter gradients are one partial row.
template <bool FLAT, int LIGHT, bool PARAMS>
__global__ void __launch_bounds__(kThreads) shading_backward_kernel(const BackwardArgs a) {
  constexpr int CORNERS = FLAT ? 1 : 3;
  const int64_t img = blockIdx.y;
  const float* prm = a.params + img * kP;
  float acc[kP];
#pragma unroll
  for (int i = 0; i < kP; ++i) acc[i] = 0.0f;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  // warp-uniform trip count: every lane reaches the warp-wide scatter
  for (int64_t s0 = (int64_t)blockIdx.x * blockDim.x; s0 < a.slots_per_image; s0 += stride) {
    const int64_t local = s0 + threadIdx.x;
    const bool active = local < a.slots_per_image;
    const int64_t s = img * a.slots_per_image + (active ? local : 0);
    const int64_t f = active ? __ldg(a.pix_to_face + s) : -1;
    V3 p, n;
    float w[3];
    slot_geometry<FLAT, LIGHT>(f, s, a.bary, a.face_pos, a.face_nrm, false, p, n, w);
    V3 gp = {0.0f, 0.0f, 0.0f}, gn = {0.0f, 0.0f, 0.0f};
    if (active) {
      Lit t;
      light_slot<LIGHT>(p, n, prm, t);
      lighting_backward<LIGHT, PARAMS>(prm, t, n, ld3(a.grad_colors + s * 3), ld3(a.texels + s * 3),
                                       a.grad_texels, s, gp, gn, acc);
      if (a.grad_positions != nullptr) {
        const V3 u = ld3(a.grad_positions + s * 3);
        gp = {gp.x + u.x, gp.y + u.y, gp.z + u.z};
      }
      if (a.grad_bary != nullptr) {  // phong only: <corner position, gp> + <corner normal, gn>, 0 in background slots
        float gb[3] = {0.0f, 0.0f, 0.0f};
        if (f >= 0) {
#pragma unroll
          for (int i = 0; i < 3; ++i) {
            gb[i] = dot3(ld3(a.face_pos + f * 9 + i * 3), gp);
            if (LIGHT != B200R_LIGHT_AMBIENT) gb[i] += dot3(ld3(a.face_nrm + f * 9 + i * 3), gn);
          }
        }
        a.grad_bary[s * 3 + 0] = gb[0];
        a.grad_bary[s * 3 + 1] = gb[1];
        a.grad_bary[s * 3 + 2] = gb[2];
      }
    }
    const float wc[3] = {FLAT ? 1.0f : w[0], w[1], w[2]};
    if (a.grad_face_pos != nullptr) {
      float g[3 * CORNERS];
#pragma unroll
      for (int i = 0; i < CORNERS; ++i) {
        g[3 * i + 0] = wc[i] * gp.x;
        g[3 * i + 1] = wc[i] * gp.y;
        g[3 * i + 2] = wc[i] * gp.z;
      }
      warp_scatter<3 * CORNERS>(a.grad_face_pos, f, g);
    }
    if (LIGHT != B200R_LIGHT_AMBIENT && a.grad_face_nrm != nullptr) {
      float g[3 * CORNERS];
#pragma unroll
      for (int i = 0; i < CORNERS; ++i) {
        g[3 * i + 0] = wc[i] * gn.x;
        g[3 * i + 1] = wc[i] * gn.y;
        g[3 * i + 2] = wc[i] * gn.z;
      }
      warp_scatter<3 * CORNERS>(a.grad_face_nrm, f, g);
    }
  }
  if (PARAMS) store_partial_row(acc, a.partials + (img * gridDim.x + blockIdx.x) * kP);
}

// grad_params[n, j] = sum over the CTAs b of image n, in order, of partials[n, b, j]
__global__ void __launch_bounds__(kThreads)
    shading_params_sum_kernel(const float* __restrict__ partials, int blocks_per_image, int64_t rows,
                              float* __restrict__ grad_params) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * kP) return;
  const int64_t n = i / kP, j = i - n * kP;
  float v = 0.0f;
  for (int b = 0; b < blocks_per_image; ++b) v += __ldg(partials + (n * blocks_per_image + b) * kP + j);
  grad_params[i] = v;
}

// CTAs per image of the backward.  A function of the shape only (not of the device), so that the parameter gradients
// are summed in the same order on every GPU.
int backward_blocks_per_image(int32_t N, int64_t slots_per_image) {
  const int64_t want = (slots_per_image + kThreads - 1) / kThreads;
  const int64_t cap = N > 0 ? (int64_t)4224 / N : 4224;  // 32 CTAs per SM of a 132-SM H100 in all
  int64_t b = want < cap ? want : cap;
  return (int)(b < 1 ? 1 : b);
}

template <bool FLAT, int LIGHT>
void launch_forward(const int64_t* p2f, const float* bary, const float* fp, const float* fn, const float* texels,
                    const float* params, int64_t total, int64_t spi, float* colors, float* positions,
                    cudaStream_t stream) {
  const int64_t blocks = cap_grid_stride_blocks((total + kThreads - 1) / kThreads);
  shading_forward_kernel<FLAT, LIGHT>
      <<<(unsigned)blocks, kThreads, 0, stream>>>(p2f, bary, fp, fn, texels, params, total, spi, colors, positions);
}

template <bool FLAT, int LIGHT>
void launch_backward(const BackwardArgs& a, dim3 grid, bool params, cudaStream_t stream) {
  if (params)
    shading_backward_kernel<FLAT, LIGHT, true><<<grid, kThreads, 0, stream>>>(a);
  else
    shading_backward_kernel<FLAT, LIGHT, false><<<grid, kThreads, 0, stream>>>(a);
}

template <int LIGHT>
void launch_forward_mode(bool flat, const int64_t* p2f, const float* bary, const float* fp, const float* fn,
                         const float* texels, const float* params, int64_t total, int64_t spi, float* colors,
                         float* positions, cudaStream_t stream) {
  if (flat)
    launch_forward<true, LIGHT>(p2f, bary, fp, fn, texels, params, total, spi, colors, positions, stream);
  else
    launch_forward<false, LIGHT>(p2f, bary, fp, fn, texels, params, total, spi, colors, positions, stream);
}

template <int LIGHT>
void launch_backward_mode(bool flat, const BackwardArgs& a, dim3 grid, bool params, cudaStream_t stream) {
  if (flat)
    launch_backward<true, LIGHT>(a, grid, params, stream);
  else
    launch_backward<false, LIGHT>(a, grid, params, stream);
}

// ---- Gouraud shading (DESIGN.md section 16) ----
// The vertex stage lights every vertex with its mesh's parameter row (light_slot, compose); the slot stage interpolates
// the shaded vertex colours with interp_face_attrs_forward_kernel's FMA chain.  Vertex-stage grids are
// (blocks per mesh, meshes); a CTA strides over its mesh's vertex range [first[m], first[m] + num[m]).

template <int LIGHT>
__global__ void __launch_bounds__(kThreads)
    gouraud_vertex_forward_kernel(const float* __restrict__ verts, const float* __restrict__ normals,
                                  const float* __restrict__ verts_colors, const int64_t* __restrict__ first,
                                  const int64_t* __restrict__ num, const float* __restrict__ params,
                                  float* __restrict__ verts_shaded) {
  const int64_t m = blockIdx.y;
  const float* prm = params + m * kP;
  const int64_t v0 = __ldg(first + m), v1 = v0 + __ldg(num + m);
  for (int64_t v = v0 + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < v1; v += (int64_t)gridDim.x * blockDim.x) {
    V3 p = {0.0f, 0.0f, 0.0f}, n = {0.0f, 0.0f, 0.0f};
    if (LIGHT != B200R_LIGHT_AMBIENT) {
      p = ld3(verts + v * 3);
      n = ld3(normals + v * 3);
    }
    Lit t;
    light_slot<LIGHT>(p, n, prm, t);
    const V3 c = ld3(verts_colors + v * 3);
    verts_shaded[v * 3 + 0] = compose(prm, 0, t.angle, t.pw, c.x);
    verts_shaded[v * 3 + 1] = compose(prm, 1, t.angle, t.pw, c.y);
    verts_shaded[v * 3 + 2] = compose(prm, 2, t.angle, t.pw, c.z);
  }
}

__global__ void __launch_bounds__(kThreads)
    gouraud_slot_forward_kernel(const int64_t* __restrict__ pix_to_face, const float* __restrict__ bary,
                                const int64_t* __restrict__ faces, const float* __restrict__ verts_shaded, int64_t P,
                                float* __restrict__ colors) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; s < P; s += stride) {
    const int64_t f = __ldg(pix_to_face + s);
    float c[3] = {0.0f, 0.0f, 0.0f};
    if (f >= 0) {
      const float w0 = __ldg(bary + s * 3 + 0), w1 = __ldg(bary + s * 3 + 1), w2 = __ldg(bary + s * 3 + 2);
      const float* a0 = verts_shaded + __ldg(faces + f * 3 + 0) * 3;
      const float* a1 = verts_shaded + __ldg(faces + f * 3 + 1) * 3;
      const float* a2 = verts_shaded + __ldg(faces + f * 3 + 2) * 3;
#pragma unroll
      for (int d = 0; d < 3; ++d) c[d] = ffma(w2, __ldg(a2 + d), ffma(w1, __ldg(a1 + d), ffma(w0, __ldg(a0 + d), 0.0f)));
    }
    colors[s * 3 + 0] = c[0];
    colors[s * 3 + 1] = c[1];
    colors[s * 3 + 2] = c[2];
  }
}

// grad_bary[s, i] = <verts_shaded[v_i], g> as interp_face_attrs_backward_kernel rounds it (one FMA per channel, from
// 0); w_i * g is merged over the warp's lanes of the same face, then added to the face's three rows of grad_shaded.
__global__ void __launch_bounds__(kThreads)
    gouraud_slot_backward_kernel(const float* __restrict__ grad_colors, const int64_t* __restrict__ pix_to_face,
                                 const float* __restrict__ bary, const int64_t* __restrict__ faces,
                                 const float* __restrict__ verts_shaded, int64_t P, float* __restrict__ grad_bary,
                                 float* __restrict__ grad_shaded) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  // warp-uniform trip count: every lane reaches the warp-wide merge
  for (int64_t s0 = (int64_t)blockIdx.x * blockDim.x; s0 < P; s0 += stride) {
    const int64_t s = s0 + threadIdx.x;
    const bool active = s < P;
    const int64_t f = active ? __ldg(pix_to_face + s) : -1;
    float g[9] = {0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f};
    int64_t vi[3] = {0, 0, 0};
    if (f >= 0) {
      const V3 u = ld3(grad_colors + s * 3);
      const float w[3] = {__ldg(bary + s * 3 + 0), __ldg(bary + s * 3 + 1), __ldg(bary + s * 3 + 2)};
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        vi[i] = __ldg(faces + f * 3 + i);
        g[3 * i + 0] = w[i] * u.x;
        g[3 * i + 1] = w[i] * u.y;
        g[3 * i + 2] = w[i] * u.z;
      }
      if (grad_bary != nullptr) {
#pragma unroll
        for (int i = 0; i < 3; ++i) {
          const V3 a = ld3(verts_shaded + vi[i] * 3);
          grad_bary[s * 3 + i] = ffma(a.z, u.z, ffma(a.y, u.y, ffma(a.x, u.x, 0.0f)));
        }
      }
    } else if (active && grad_bary != nullptr) {
      grad_bary[s * 3 + 0] = 0.0f;
      grad_bary[s * 3 + 1] = 0.0f;
      grad_bary[s * 3 + 2] = 0.0f;
    }
    if (grad_shaded != nullptr && warp_merge<9>(f, g)) {
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        float* o = grad_shaded + vi[i] * 3;
        atomicAdd(o + 0, g[3 * i + 0]);
        atomicAdd(o + 1, g[3 * i + 1]);
        atomicAdd(o + 2, g[3 * i + 2]);
      }
    }
  }
}

struct GouraudBackwardArgs {
  const float* grad_shaded;
  const float* verts;
  const float* normals;
  const float* verts_colors;
  const int64_t* first;
  const int64_t* num;
  const float* params;
  float* grad_verts;         // may be null
  float* grad_normals;       // may be null
  float* grad_verts_colors;  // may be null
  float* partials;           // (meshes, gridDim.x, kP) when PARAMS
};

// Same grid as the vertex forward; every vertex's gradients are written once, the parameter gradients go to one
// partial row per CTA.
template <int LIGHT, bool PARAMS>
__global__ void __launch_bounds__(kThreads) gouraud_vertex_backward_kernel(const GouraudBackwardArgs a) {
  const int64_t m = blockIdx.y;
  const float* prm = a.params + m * kP;
  float acc[kP];
#pragma unroll
  for (int i = 0; i < kP; ++i) acc[i] = 0.0f;
  const int64_t v0 = __ldg(a.first + m), v1 = v0 + __ldg(a.num + m);
  for (int64_t v = v0 + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < v1; v += (int64_t)gridDim.x * blockDim.x) {
    V3 p = {0.0f, 0.0f, 0.0f}, n = {0.0f, 0.0f, 0.0f};
    if (LIGHT != B200R_LIGHT_AMBIENT) {
      p = ld3(a.verts + v * 3);
      n = ld3(a.normals + v * 3);
    }
    Lit t;
    light_slot<LIGHT>(p, n, prm, t);
    V3 gp = {0.0f, 0.0f, 0.0f}, gn = {0.0f, 0.0f, 0.0f};
    lighting_backward<LIGHT, PARAMS>(prm, t, n, ld3(a.grad_shaded + v * 3), ld3(a.verts_colors + v * 3),
                                     a.grad_verts_colors, v, gp, gn, acc);
    if (a.grad_verts != nullptr) {
      a.grad_verts[v * 3 + 0] = gp.x;
      a.grad_verts[v * 3 + 1] = gp.y;
      a.grad_verts[v * 3 + 2] = gp.z;
    }
    if (a.grad_normals != nullptr) {
      a.grad_normals[v * 3 + 0] = gn.x;
      a.grad_normals[v * 3 + 1] = gn.y;
      a.grad_normals[v * 3 + 2] = gn.z;
    }
  }
  if (PARAMS) store_partial_row(acc, a.partials + (m * gridDim.x + blockIdx.x) * kP);
}

// CTAs per mesh of the vertex stage: enough for the mean mesh size, capped like the slot backward's.  A function of
// (V, meshes) only, so that the parameter gradients are summed in the same order on every GPU.
int gouraud_blocks_per_mesh(int32_t meshes, int64_t V) {
  if (meshes <= 0) return 1;
  const int64_t want = (V + (int64_t)meshes * kThreads - 1) / ((int64_t)meshes * kThreads);
  const int64_t cap = (int64_t)4224 / meshes;
  int64_t b = want < cap ? want : cap;
  return (int)(b < 1 ? 1 : b);
}

size_t align256(size_t n) { return (n + 255) & ~(size_t)255; }

template <int LIGHT>
void launch_gouraud_vertex_backward(const GouraudBackwardArgs& a, dim3 grid, bool params, cudaStream_t stream) {
  if (params)
    gouraud_vertex_backward_kernel<LIGHT, true><<<grid, kThreads, 0, stream>>>(a);
  else
    gouraud_vertex_backward_kernel<LIGHT, false><<<grid, kThreads, 0, stream>>>(a);
}

int check_gouraud_args(int64_t V, int32_t meshes, int64_t F, int64_t P, int32_t light, const float* normals) {
  if (V < 0 || meshes < 0 || F < 0 || P < 0) return fail(B200R_ERR_INVALID_ARGUMENT, "negative size");
  if (light != B200R_LIGHT_POINT && light != B200R_LIGHT_DIRECTIONAL && light != B200R_LIGHT_AMBIENT)
    return fail(B200R_ERR_INVALID_ARGUMENT, "unknown light kind");
  if (light != B200R_LIGHT_AMBIENT && normals == nullptr && V > 0)
    return fail(B200R_ERR_INVALID_ARGUMENT, "gouraud shading needs vertex normals for a point or directional light");
  if (meshes > 65535) return fail(B200R_ERR_INVALID_ARGUMENT, "gouraud shading: at most 65535 meshes per call");
  if (meshes == 0 && V > 0) return fail(B200R_ERR_INVALID_ARGUMENT, "gouraud shading: vertices but no meshes");
  return B200R_OK;
}

int check_shading_args(int32_t N, int32_t H, int32_t W, int32_t K, int64_t F, int32_t flat, int32_t light,
                       const float* bary) {
  if (N < 0 || H < 0 || W < 0 || K < 0 || F < 0) return fail(B200R_ERR_INVALID_ARGUMENT, "negative size");
  if (light != B200R_LIGHT_POINT && light != B200R_LIGHT_DIRECTIONAL && light != B200R_LIGHT_AMBIENT)
    return fail(B200R_ERR_INVALID_ARGUMENT, "unknown light kind");
  if (!flat && bary == nullptr && (int64_t)N * H * W * K > 0)
    return fail(B200R_ERR_INVALID_ARGUMENT, "phong shading needs barycentric coordinates");
  return B200R_OK;
}

}  // namespace
}  // namespace b200r

using namespace b200r;

extern "C" int b200r_shading_forward(const int64_t* pix_to_face, const float* barycentric_coords,
                                     const float* face_positions, const float* face_normals, int64_t F,
                                     const float* texels, const float* params, int32_t N, int32_t H, int32_t W,
                                     int32_t K, int32_t flat, int32_t light, float* colors, float* positions,
                                     void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int rc = check_shading_args(N, H, W, K, F, flat, light, barycentric_coords);
  if (rc != B200R_OK) return rc;
  const int64_t spi = (int64_t)H * W * K, total = (int64_t)N * spi;
  if (total == 0) return B200R_OK;
  if (light == B200R_LIGHT_POINT)
    launch_forward_mode<B200R_LIGHT_POINT>(flat != 0, pix_to_face, barycentric_coords, face_positions, face_normals,
                                           texels, params, total, spi, colors, positions, stream);
  else if (light == B200R_LIGHT_DIRECTIONAL)
    launch_forward_mode<B200R_LIGHT_DIRECTIONAL>(flat != 0, pix_to_face, barycentric_coords, face_positions,
                                                 face_normals, texels, params, total, spi, colors, positions, stream);
  else
    launch_forward_mode<B200R_LIGHT_AMBIENT>(flat != 0, pix_to_face, barycentric_coords, face_positions, face_normals,
                                             texels, params, total, spi, colors, positions, stream);
  B200R_LAUNCHED("shading_forward_kernel");
  return B200R_OK;
}

extern "C" size_t b200r_shading_workspace_bytes(int32_t N, int32_t H, int32_t W, int32_t K) {
  if (N <= 0 || H < 0 || W < 0 || K < 0) return 0;
  const int64_t spi = (int64_t)H * W * K;
  return sizeof(float) * (size_t)N * (size_t)backward_blocks_per_image(N, spi) * kP;
}

extern "C" int b200r_shading_backward(const float* grad_colors, const float* grad_positions,
                                      const int64_t* pix_to_face, const float* barycentric_coords,
                                      const float* face_positions, const float* face_normals, int64_t F,
                                      const float* texels, const float* params, int32_t N, int32_t H, int32_t W,
                                      int32_t K, int32_t flat, int32_t light, void* workspace,
                                      size_t workspace_bytes, float* grad_texels, float* grad_barycentric_coords,
                                      float* grad_face_positions, float* grad_face_normals, float* grad_params,
                                      void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int rc = check_shading_args(N, H, W, K, F, flat, light, barycentric_coords);
  if (rc != B200R_OK) return rc;
  const int64_t corners = flat ? 1 : 3;
  if (grad_face_positions != nullptr && F > 0)
    B200R_CUDA_OK(cudaMemsetAsync(grad_face_positions, 0, sizeof(float) * (size_t)(F * corners * 3), stream));
  if (grad_face_normals != nullptr && F > 0)
    B200R_CUDA_OK(cudaMemsetAsync(grad_face_normals, 0, sizeof(float) * (size_t)(F * corners * 3), stream));
  const int64_t spi = (int64_t)H * W * K;
  if (N == 0) return B200R_OK;
  if (spi == 0) {
    if (grad_params != nullptr) B200R_CUDA_OK(cudaMemsetAsync(grad_params, 0, sizeof(float) * (size_t)N * kP, stream));
    return B200R_OK;
  }
  if (N > 65535) return fail(B200R_ERR_INVALID_ARGUMENT, "shading backward: at most 65535 images per call");
  const bool want_params = grad_params != nullptr;
  const int bpi = backward_blocks_per_image(N, spi);
  if (want_params && (workspace == nullptr || workspace_bytes < b200r_shading_workspace_bytes(N, H, W, K)))
    return fail(B200R_ERR_INVALID_ARGUMENT, "shading backward: workspace too small");
  BackwardArgs a{grad_colors,   grad_positions, pix_to_face,   barycentric_coords, face_positions,
                 face_normals,  texels,         params,        spi,                grad_texels,
                 flat ? nullptr : grad_barycentric_coords,     grad_face_positions, grad_face_normals,
                 static_cast<float*>(workspace)};
  const dim3 grid((unsigned)bpi, (unsigned)N);
  if (light == B200R_LIGHT_POINT)
    launch_backward_mode<B200R_LIGHT_POINT>(flat != 0, a, grid, want_params, stream);
  else if (light == B200R_LIGHT_DIRECTIONAL)
    launch_backward_mode<B200R_LIGHT_DIRECTIONAL>(flat != 0, a, grid, want_params, stream);
  else
    launch_backward_mode<B200R_LIGHT_AMBIENT>(flat != 0, a, grid, want_params, stream);
  B200R_LAUNCHED("shading_backward_kernel");
  if (want_params) {
    const int64_t n = (int64_t)N * kP;
    shading_params_sum_kernel<<<(unsigned)((n + kThreads - 1) / kThreads), kThreads, 0, stream>>>(
        static_cast<const float*>(workspace), bpi, N, grad_params);
    B200R_LAUNCHED("shading_params_sum_kernel");
  }
  return B200R_OK;
}

extern "C" int b200r_gouraud_forward(const float* verts, const float* normals, const float* verts_colors, int64_t V,
                                     const int64_t* mesh_first_vert, const int64_t* mesh_num_verts, int32_t meshes,
                                     const float* params, const int64_t* faces, int64_t F, const int64_t* pix_to_face,
                                     const float* barycentric_coords, int64_t P, int32_t light, float* verts_shaded,
                                     float* colors, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int rc = check_gouraud_args(V, meshes, F, P, light, normals);
  if (rc != B200R_OK) return rc;
  if (V > 0 && meshes > 0) {
    const dim3 grid((unsigned)gouraud_blocks_per_mesh(meshes, V), (unsigned)meshes);
    if (light == B200R_LIGHT_POINT)
      gouraud_vertex_forward_kernel<B200R_LIGHT_POINT><<<grid, kThreads, 0, stream>>>(
          verts, normals, verts_colors, mesh_first_vert, mesh_num_verts, params, verts_shaded);
    else if (light == B200R_LIGHT_DIRECTIONAL)
      gouraud_vertex_forward_kernel<B200R_LIGHT_DIRECTIONAL><<<grid, kThreads, 0, stream>>>(
          verts, normals, verts_colors, mesh_first_vert, mesh_num_verts, params, verts_shaded);
    else
      gouraud_vertex_forward_kernel<B200R_LIGHT_AMBIENT><<<grid, kThreads, 0, stream>>>(
          verts, normals, verts_colors, mesh_first_vert, mesh_num_verts, params, verts_shaded);
    B200R_LAUNCHED("gouraud_vertex_forward_kernel");
  }
  if (P > 0) {
    const int64_t blocks = cap_grid_stride_blocks((P + kThreads - 1) / kThreads);
    gouraud_slot_forward_kernel<<<(unsigned)blocks, kThreads, 0, stream>>>(pix_to_face, barycentric_coords, faces,
                                                                          verts_shaded, P, colors);
    B200R_LAUNCHED("gouraud_slot_forward_kernel");
  }
  return B200R_OK;
}

extern "C" size_t b200r_gouraud_workspace_bytes(int32_t meshes, int64_t V) {
  if (meshes < 0 || V < 0) return 0;
  return align256(sizeof(float) * (size_t)V * 3) +
         sizeof(float) * (size_t)meshes * (size_t)gouraud_blocks_per_mesh(meshes, V) * kP;
}

extern "C" int b200r_gouraud_backward(const float* grad_colors, const float* verts, const float* normals,
                                      const float* verts_colors, int64_t V, const int64_t* mesh_first_vert,
                                      const int64_t* mesh_num_verts, int32_t meshes, const float* params,
                                      const int64_t* faces, int64_t F, const int64_t* pix_to_face,
                                      const float* barycentric_coords, int64_t P, int32_t light,
                                      const float* verts_shaded, void* workspace, size_t workspace_bytes,
                                      float* grad_verts, float* grad_normals, float* grad_verts_colors,
                                      float* grad_barycentric_coords, float* grad_params, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int rc = check_gouraud_args(V, meshes, F, P, light, normals);
  if (rc != B200R_OK) return rc;
  const bool want_vertex = grad_verts != nullptr || grad_normals != nullptr || grad_verts_colors != nullptr ||
                           grad_params != nullptr;
  if (want_vertex && (workspace == nullptr || workspace_bytes < b200r_gouraud_workspace_bytes(meshes, V)))
    return fail(B200R_ERR_INVALID_ARGUMENT, "gouraud backward: workspace too small");
  float* grad_shaded = want_vertex ? static_cast<float*>(workspace) : nullptr;
  float* partials = want_vertex ? reinterpret_cast<float*>(static_cast<char*>(workspace) +
                                                           align256(sizeof(float) * (size_t)V * 3))
                                : nullptr;
  if (grad_shaded != nullptr && V > 0)
    B200R_CUDA_OK(cudaMemsetAsync(grad_shaded, 0, sizeof(float) * (size_t)V * 3, stream));
  if (P > 0 && (grad_shaded != nullptr || grad_barycentric_coords != nullptr)) {
    const int64_t blocks = cap_grid_stride_blocks((P + kThreads - 1) / kThreads);
    gouraud_slot_backward_kernel<<<(unsigned)blocks, kThreads, 0, stream>>>(
        grad_colors, pix_to_face, barycentric_coords, faces, verts_shaded, P, grad_barycentric_coords, grad_shaded);
    B200R_LAUNCHED("gouraud_slot_backward_kernel");
  }
  if (!want_vertex || meshes == 0) return B200R_OK;
  if (V == 0) {
    if (grad_params != nullptr)
      B200R_CUDA_OK(cudaMemsetAsync(grad_params, 0, sizeof(float) * (size_t)meshes * kP, stream));
    return B200R_OK;
  }
  const int bpm = gouraud_blocks_per_mesh(meshes, V);
  const GouraudBackwardArgs a{grad_shaded, verts,      normals,           verts_colors,
                              mesh_first_vert, mesh_num_verts, params, grad_verts,
                              light == B200R_LIGHT_AMBIENT ? nullptr : grad_normals, grad_verts_colors, partials};
  const dim3 grid((unsigned)bpm, (unsigned)meshes);
  const bool want_params = grad_params != nullptr;
  if (light == B200R_LIGHT_POINT)
    launch_gouraud_vertex_backward<B200R_LIGHT_POINT>(a, grid, want_params, stream);
  else if (light == B200R_LIGHT_DIRECTIONAL)
    launch_gouraud_vertex_backward<B200R_LIGHT_DIRECTIONAL>(a, grid, want_params, stream);
  else
    launch_gouraud_vertex_backward<B200R_LIGHT_AMBIENT>(a, grid, want_params, stream);
  B200R_LAUNCHED("gouraud_vertex_backward_kernel");
  if (light == B200R_LIGHT_AMBIENT && grad_normals != nullptr)
    B200R_CUDA_OK(cudaMemsetAsync(grad_normals, 0, sizeof(float) * (size_t)V * 3, stream));
  if (want_params) {
    const int64_t n = (int64_t)meshes * kP;
    shading_params_sum_kernel<<<(unsigned)((n + kThreads - 1) / kThreads), kThreads, 0, stream>>>(partials, bpm,
                                                                                                  meshes, grad_params);
    B200R_LAUNCHED("shading_params_sum_kernel");
  }
  return B200R_OK;
}
