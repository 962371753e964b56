// Frustum culling and z-clipping of faces, and the conversion of a rasterization of the clipped faces back to the
// unclipped ones, forward and backward (DESIGN.md section 14).
//
// What pytorch3d/renderer/mesh/clip.py clip_faces and convert_clipped_rasterization_to_original_faces compute, in the
// reference's output layout.  Every face falls in one case (clip.py:392-423 of the reference):
//   1  in front of z_clip and not culled -> one output face, itself
//   2  culled, or all three vertices behind -> nothing
//   3  two vertices behind -> (p4, p5, p1), one barycentric conversion row
//   4  one vertex behind   -> (p4, p2, p5) and (p5, p2, p3), two rows; the two halves name each other as neighbours
// Output faces keep the order of their source faces.  Conversion rows: case-3 faces, then case-4 first halves, then
// case-4 second halves, each in face order.
//
// Count pass: one thread per face classifies it and every CTA writes its totals; one CTA scans the CTA totals and writes
// the four-word record {F_clipped, n_case3, n_case4, faces not in case 1}, which the host reads once to size the
// outputs.  Fill and backward passes: one thread per face classifies it again, a block scan plus the CTA's offset
// gives its output face and conversion rows.  The clip backward writes each face's gradient once (no atomics).
//
// All arithmetic reproduces torch's separately rounded elementwise ops (__f*_rn, no contraction); the perspective
// divide by the Python float z_clip is a multiply by (float)(1.0 / z_clip), as torch's CUDA division by a scalar does.
#include "common.cuh"
#include "raster_math.cuh"

namespace b200r {
namespace {

constexpr int kThreads = 256;
constexpr int kScanThreads = 1024;
constexpr int kWords = 4;  // per-CTA counters in the workspace: output faces, case 3, case 4, faces not in case 1

struct ClipParams {
  const float* face_verts;  // (F,3,3), or null: the faces are verts[faces] (count pass of the identity check)
  const float* verts;
  const int64_t* faces;
  int64_t F;
  float plane[6];  // left, right, top, bottom, znear, zfar
  int cull_mask;   // bit i: plane i is used
  bool has_z, perspective;
  float z, inv_z;  // z_clip as float32, and 1 / z_clip taken in double and rounded to float32
};

__device__ __forceinline__ void load_face(const ClipParams& p, int64_t f, float (&v)[9]) {
  if (p.face_verts != nullptr) {
    const float* a = p.face_verts + f * 9;
#pragma unroll
    for (int i = 0; i < 9; ++i) v[i] = __ldg(a + i);
  } else {
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      const float* a = p.verts + __ldg(p.faces + f * 3 + j) * 3;
#pragma unroll
      for (int i = 0; i < 3; ++i) v[j * 3 + i] = __ldg(a + i);
    }
  }
}

// Case 1..4 of a face, and (through p1) the index of the vertex that is alone on its side of the plane.
// Culling keeps the reference's indexing: plane `axis` tests the three coordinates of VERTEX number `axis`
// (face_verts[:, axis] on an (F,3,3) tensor, clip.py:189-195).
__device__ __forceinline__ int classify(const ClipParams& p, const float (&v)[9], int& p1) {
  bool culled = false;
#pragma unroll
  for (int i = 0; i < 6; ++i) {
    if (!((p.cull_mask >> i) & 1)) continue;
    const int axis = i >> 1;
    const float c = p.plane[i];
    const bool less = (i & 1) == 0;
    bool all = true;
#pragma unroll
    for (int k = 0; k < 3; ++k) all = all && (less ? v[axis * 3 + k] < c : v[axis * 3 + k] > c);
    culled = culled || all;
  }
  p1 = 0;
  if (culled) return 2;
  if (!p.has_z) return 1;
  const bool b0 = v[2] < p.z, b1 = v[5] < p.z, b2 = v[8] < p.z;
  const int nb = (int)b0 + (int)b1 + (int)b2;
  if (nb == 0) return 1;
  if (nb == 3) return 2;
  const bool lone = nb == 2 ? false : true;  // case 3: the vertex in front; case 4: the one behind
  p1 = b0 == lone ? 0 : (b1 == lone ? 1 : 2);
  return nb == 2 ? 3 : 4;
}

__device__ __forceinline__ int out_count(int c) { return c == 1 || c == 3 ? 1 : (c == 4 ? 2 : 0); }

// Per-CTA counters of the faces [blockIdx.x * 256, +256): output faces, case 3, case 4, not case 1.
__global__ void __launch_bounds__(kThreads) clip_count_kernel(const ClipParams p, int64_t* __restrict__ cta_counts) {
  const int64_t f = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  int c = 1, p1;
  if (f < p.F) {
    float v[9];
    load_face(p, f, v);
    c = classify(p, v, p1);
  }
  int cnt[kWords] = {f < p.F ? out_count(c) : 0, c == 3, c == 4, c != 1};
  __shared__ int part[kThreads / 32][kWords];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int j = 0; j < kWords; ++j) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) cnt[j] += __shfl_xor_sync(0xffffffffu, cnt[j], o);
    if (lane == 0) part[wid][j] = cnt[j];
  }
  __syncthreads();
  if (threadIdx.x < kWords) {
    int s = 0;
#pragma unroll
    for (int w = 0; w < kThreads / 32; ++w) s += part[w][threadIdx.x];
    cta_counts[(int64_t)blockIdx.x * kWords + threadIdx.x] = s;
  }
}

// One CTA: exclusive scan of the nb CTA counters in place (64-bit), then the totals record.
__global__ void __launch_bounds__(kScanThreads) clip_scan_kernel(int64_t* __restrict__ record,
                                                                 int64_t* __restrict__ cta_counts, int64_t nb) {
  __shared__ long long warp_sums[kScanThreads / 32][kWords];
  __shared__ long long carry[kWords];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (tid < kWords) carry[tid] = 0;
  __syncthreads();
  for (int64_t base = 0; base < nb; base += kScanThreads) {
    const int64_t b = base + tid;
    long long x[kWords], incl[kWords];
#pragma unroll
    for (int j = 0; j < kWords; ++j) {
      x[j] = b < nb ? cta_counts[b * kWords + j] : 0;
      incl[j] = x[j];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const long long y = __shfl_up_sync(0xffffffffu, incl[j], o);
        if (lane >= o) incl[j] += y;
      }
      if (lane == 31) warp_sums[wid][j] = incl[j];
    }
    __syncthreads();
    if (wid == 0) {
#pragma unroll
      for (int j = 0; j < kWords; ++j) {
        long long s = warp_sums[lane][j];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const long long y = __shfl_up_sync(0xffffffffu, s, o);
          if (lane >= o) s += y;
        }
        warp_sums[lane][j] = s;  // inclusive over warps
      }
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < kWords; ++j) {
      const long long before = carry[j] + (wid > 0 ? warp_sums[wid - 1][j] : 0) + incl[j] - x[j];
      if (b < nb) cta_counts[b * kWords + j] = before;
    }
    __syncthreads();
    if (tid < kWords) carry[tid] += warp_sums[kScanThreads / 32 - 1][tid];
    __syncthreads();
  }
  if (tid < kWords) record[tid] = carry[tid];
}

// This thread's face: its case, p1, vertices, and the offsets of its output face and conversion row counters
// (exclusive over all faces before it).  Every thread of the CTA must call it (block scan).
struct FaceSlot {
  int c, p1;
  int64_t out, r3, r4;
  float v[9];
};
__device__ __forceinline__ FaceSlot face_slot(const ClipParams& p, const int64_t* __restrict__ cta_offsets) {
  FaceSlot s;
  const int64_t f = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  s.c = 2;
  s.p1 = 0;
  if (f < p.F) {
    load_face(p, f, s.v);
    s.c = classify(p, s.v, s.p1);
  }
  // packed counters: output faces in bits 0-10, case 3 in 11-20, case 4 in 21-30 (a CTA has <= 512 / 256 / 256)
  const int mine = out_count(s.c) | ((int)(s.c == 3) << 11) | ((int)(s.c == 4) << 21);
  __shared__ int warp_tot[kThreads / 32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int incl = mine;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += y;
  }
  if (lane == 31) warp_tot[wid] = incl;
  __syncthreads();
  int before = incl - mine;
  for (int w = 0; w < wid; ++w) before += warp_tot[w];
  const int64_t* o = cta_offsets + (int64_t)blockIdx.x * kWords;
  s.out = o[0] + (before & 0x7ff);
  s.r3 = o[1] + ((before >> 11) & 0x3ff);
  s.r4 = o[2] + ((before >> 21) & 0x3ff);
  return s;
}

// p1..p5 and the weights of clip.py:253-318: w2 = (p1.z - z) / (p1.z - p2.z), p4 = p1 (1 - w2) + p2 w2, and for a
// perspective camera p4.xy = (p1.xy p1.z (1 - w2) + p2.xy p2.z w2) / z; the same with w3 and p3 for p5.
// v[3 i + c] without a dynamically indexed (local-memory) array
__device__ __forceinline__ float pick(const float (&v)[9], int i, int c) {
  return i == 0 ? v[c] : (i == 1 ? v[3 + c] : v[6 + c]);
}

struct Intersections {
  float p[5][3];
  float w2, w3;
  int i[3];
};
__device__ __forceinline__ Intersections intersect(const ClipParams& prm, const float (&v)[9], int p1) {
  Intersections r;
  r.i[0] = p1;
  r.i[1] = p1 == 2 ? 0 : p1 + 1;
  r.i[2] = p1 == 0 ? 2 : p1 - 1;
#pragma unroll
  for (int k = 0; k < 3; ++k)
#pragma unroll
    for (int c = 0; c < 3; ++c) r.p[k][c] = pick(v, r.i[k], c);
  const float n = fsub(r.p[0][2], prm.z);
  r.w2 = fdiv(n, fsub(r.p[0][2], r.p[1][2]));
  r.w3 = fdiv(n, fsub(r.p[0][2], r.p[2][2]));
  const float w[2] = {r.w2, r.w3};
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    const float* q = r.p[1 + e];
    const float t = fsub(1.0f, w[e]);
#pragma unroll
    for (int c = 0; c < 3; ++c) r.p[3 + e][c] = fadd(fmul(r.p[0][c], t), fmul(q[c], w[e]));
    if (prm.perspective) {
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const float a = fmul(r.p[0][c], r.p[0][2]), b = fmul(q[c], q[2]);
        r.p[3 + e][c] = fmul(fadd(fmul(a, t), fmul(b, w[e])), prm.inv_z);
      }
    }
  }
  return r;
}

__device__ __forceinline__ void store_face(float* __restrict__ out, const float* a, const float* b, const float* c) {
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    out[k] = a[k];
    out[3 + k] = b[k];
    out[6 + k] = c[k];
  }
}

// conversion row (3,3): column k holds the barycentric weights of the clipped face's vertex k w.r.t. the original
// face; bary[j] = {vertex index -> weight} of up to two entries
struct Bary {
  int a, b;
  float wa, wb;
};
__device__ __forceinline__ void store_row(float* __restrict__ row, const Bary (&cols)[3]) {
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int k = 0; k < 3; ++k) row[i * 3 + k] = cols[k].a == i ? cols[k].wa : (cols[k].b == i ? cols[k].wb : 0.0f);
}

struct FillOut {
  float* face_verts;
  int64_t* c2u;
  float* conversion;  // null when no face is in case 3 or 4 (then so are the next two)
  int64_t* conv_idx;
  int64_t* neighbor;
  int64_t n3, n4;
};

__global__ void __launch_bounds__(kThreads)
    clip_fill_kernel(const ClipParams p, const int64_t* __restrict__ cta_offsets, const FillOut o) {
  const FaceSlot s = face_slot(p, cta_offsets);
  const int64_t f = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (s.c == 2) return;
  const int64_t d = s.out;
  if (s.c == 1) {
    store_face(o.face_verts + d * 9, s.v, s.v + 3, s.v + 6);
    o.c2u[d] = f;
    if (o.conversion != nullptr) {
      o.conv_idx[d] = -1;
      o.neighbor[d] = -1;
    }
    return;
  }
  const Intersections r = intersect(p, s.v, s.p1);
  const float t2 = fsub(1.0f, r.w2), t3 = fsub(1.0f, r.w3);
  const Bary b1{r.i[0], -1, 1.0f, 0.0f}, b2{r.i[1], -1, 1.0f, 0.0f}, b3{r.i[2], -1, 1.0f, 0.0f};
  const Bary b4{r.i[0], r.i[1], t2, r.w2}, b5{r.i[0], r.i[2], t3, r.w3};
  if (s.c == 3) {
    store_face(o.face_verts + d * 9, r.p[3], r.p[4], r.p[0]);
    o.c2u[d] = f;
    o.conv_idx[d] = s.r3;
    o.neighbor[d] = -1;
    const Bary cols[3] = {b4, b5, b1};
    store_row(o.conversion + s.r3 * 9, cols);
    return;
  }
  const int64_t ra = o.n3 + s.r4, rb = o.n3 + o.n4 + s.r4;
  store_face(o.face_verts + d * 9, r.p[3], r.p[1], r.p[4]);
  store_face(o.face_verts + (d + 1) * 9, r.p[4], r.p[1], r.p[2]);
  o.c2u[d] = f;
  o.c2u[d + 1] = f;
  o.conv_idx[d] = ra;
  o.conv_idx[d + 1] = rb;
  o.neighbor[d] = d + 1;
  o.neighbor[d + 1] = d;
  const Bary ca[3] = {b4, b2, b5}, cb[3] = {b5, b2, b3};
  store_row(o.conversion + ra * 9, ca);
  store_row(o.conversion + rb * 9, cb);
}

// first_clipped[m] = number of output faces of the faces before first[m] (a lower bound in the ascending c2u; F_clipped
// for a first index at or past F, the clamp of an empty last mesh); num_clipped[m] = first_clipped[m + 1] -
// first_clipped[m], the last mesh running to F_clipped (clip.py:448-453).
__device__ __forceinline__ int64_t lower_bound(const int64_t* __restrict__ a, int64_t n, int64_t x) {
  int64_t lo = 0, hi = n;
  while (lo < hi) {
    const int64_t mid = lo + ((hi - lo) >> 1);
    if (__ldg(a + mid) < x)
      lo = mid + 1;
    else
      hi = mid;
  }
  return lo;
}
__global__ void __launch_bounds__(kThreads)
    clip_meshes_kernel(const int64_t* __restrict__ first, int32_t N, const int64_t* __restrict__ c2u,
                       int64_t F_clipped, int64_t* __restrict__ first_clipped, int64_t* __restrict__ num_clipped) {
  const int m = blockIdx.x * kThreads + threadIdx.x;
  if (m >= N) return;
  const int64_t a = lower_bound(c2u, F_clipped, __ldg(first + m));
  const int64_t b = m + 1 < N ? lower_bound(c2u, F_clipped, __ldg(first + m + 1)) : F_clipped;
  first_clipped[m] = a;
  num_clipped[m] = b - a;
}

// d loss / d face_verts_unclipped, one thread per original face.  Follows autograd through clip.py:253-318: w3 is
// detached (in p5 and in p5's conversion column), the perspective xy of p4 / p5 overwrite the linear ones in place
// (their gradient flows through the world-space formula only), w2 collects the gradient of p4 and of p4's conversion
// column.  Case-1 faces copy their output's gradient; culled and case-2 faces get 0.
__global__ void __launch_bounds__(kThreads)
    clip_backward_kernel(const ClipParams p, const int64_t* __restrict__ cta_offsets, int64_t n3, int64_t n4,
                         const float* __restrict__ grad_out, const float* __restrict__ grad_conv,
                         float* __restrict__ grad_in) {
  const FaceSlot s = face_slot(p, cta_offsets);
  const int64_t f = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (f >= p.F) return;
  float* gi = grad_in + f * 9;
  if (s.c == 2 || (s.c == 1 && grad_out == nullptr)) {
#pragma unroll
    for (int i = 0; i < 9; ++i) gi[i] = 0.0f;
    return;
  }
  if (s.c == 1) {
#pragma unroll
    for (int i = 0; i < 9; ++i) gi[i] = __ldg(grad_out + s.out * 9 + i);
    return;
  }
  const Intersections r = intersect(p, s.v, s.p1);
  float G[5][3] = {};  // gradients of p1..p5 as output vertices
  auto add = [&](int k, const float* g) {
#pragma unroll
    for (int c = 0; c < 3; ++c) G[k][c] += __ldg(g + c);
  };
  float gw2 = 0.0f;
  int64_t row_w2;  // the conversion row whose column 0 is p4's
  if (s.c == 3) {
    if (grad_out != nullptr) {
      const float* g = grad_out + s.out * 9;
      add(3, g);
      add(4, g + 3);
      add(0, g + 6);
    }
    row_w2 = s.r3;
  } else {
    if (grad_out != nullptr) {
      const float* g = grad_out + s.out * 9;
      add(3, g);
      add(1, g + 3);
      add(4, g + 6);
      add(4, g + 9);
      add(1, g + 12);
      add(2, g + 15);
    }
    row_w2 = n3 + s.r4;
  }
  if (grad_conv != nullptr) {  // column 0 of the row: (1 - w2) at p1's index, w2 at p2's
    const float* g = grad_conv + row_w2 * 9;
    gw2 = __ldg(g + r.i[1] * 3) - __ldg(g + r.i[0] * 3);
  }
  float d[3][3];
#pragma unroll
  for (int k = 0; k < 3; ++k)
#pragma unroll
    for (int c = 0; c < 3; ++c) d[k][c] = G[k][c];
  const float* P1 = r.p[0];
  const float w[2] = {r.w2, r.w3};
#pragma unroll
  for (int e = 0; e < 2; ++e) {  // p4 (with p2, w2) and p5 (with p3, w3 detached)
    const float* Q = r.p[1 + e];
    const float* Ge = G[3 + e];
    const float t = 1.0f - w[e];
    float gw = 0.0f;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      if (c < 2 && p.perspective) {
        const float h = Ge[c] * p.inv_z;
        const float a = P1[c] * P1[2], b = Q[c] * Q[2];
        const float ga = h * t, gb = h * w[e];
        gw += h * (b - a);
        d[0][c] += ga * P1[2];
        d[0][2] += ga * P1[c];
        d[1 + e][c] += gb * Q[2];
        d[1 + e][2] += gb * Q[c];
      } else {
        d[0][c] += Ge[c] * t;
        d[1 + e][c] += Ge[c] * w[e];
        gw += Ge[c] * (Q[c] - P1[c]);
      }
    }
    if (e == 0) gw2 += gw;
  }
  // w2 = (p1.z - z) / (p1.z - p2.z)
  const float den = P1[2] - r.p[1][2];
  const float gden = -gw2 * r.w2 / den;
  d[0][2] += gw2 / den + gden;
  d[1][2] -= gden;
#pragma unroll
  for (int j = 0; j < 3; ++j)  // original vertex j is p1, p2 or p3
#pragma unroll
    for (int c = 0; c < 3; ++c) gi[j * 3 + c] = r.i[0] == j ? d[0][c] : (r.i[1] == j ? d[1][c] : d[2][c]);
}

// ------------------------------------------------------------------------------------------------- conversion

// One thread per slot: pix_to_face -> c2u[f] (-1 stays -1); slots whose face has a conversion row get
// bary = conv[row] @ bary as fma(c2, b2, fma(c1, b1, c0 * b0)) per component, the others are copied.
__global__ void __launch_bounds__(kThreads)
    clip_convert_forward_kernel(const int64_t* __restrict__ pix_to_face, const float* __restrict__ bary, int64_t S,
                                const int64_t* __restrict__ c2u, const float* __restrict__ conversion,
                                const int64_t* __restrict__ conv_idx, int64_t* __restrict__ p2f_out,
                                float* __restrict__ bary_out) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; s < S; s += stride) {
    const int64_t f = __ldg(pix_to_face + s);
    p2f_out[s] = f >= 0 ? __ldg(c2u + f) : -1;
    if (bary_out == nullptr) continue;
    float b[3] = {__ldg(bary + s * 3), __ldg(bary + s * 3 + 1), __ldg(bary + s * 3 + 2)};
    const int64_t row = f >= 0 ? __ldg(conv_idx + f) : -1;
    if (row >= 0) {
      const float* m = conversion + row * 9;
      float o[3];
#pragma unroll
      for (int i = 0; i < 3; ++i)
        o[i] = ffma(__ldg(m + i * 3 + 2), b[2], ffma(__ldg(m + i * 3 + 1), b[1], fmul(__ldg(m + i * 3), b[0])));
#pragma unroll
      for (int i = 0; i < 3; ++i) b[i] = o[i];
    }
#pragma unroll
    for (int i = 0; i < 3; ++i) bary_out[s * 3 + i] = b[i];
  }
}

__device__ __forceinline__ void red_add(float* p, float v) {
  asm volatile("red.global.add.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}

// Adds one warp's per-lane 9-vectors at out + key * 9; lanes with the same key are merged first (one MATCH, then pointer
// jumping) and sums that are exactly 0 are skipped.  Every lane must call it; lanes with nothing to add pass key = -1.
__device__ __forceinline__ void warp_merge_add9(float* __restrict__ out, int64_t key, float (&g)[9]) {
  if (__all_sync(0xffffffffu, key < 0)) return;
  const int lane = threadIdx.x & 31;
  const unsigned grp = __match_any_sync(0xffffffffu, key);
  const unsigned above = lane == 31 ? 0u : grp & (0xffffffffu << (lane + 1));
  int next = (key >= 0 && above != 0u) ? __ffs((int)above) - 1 : -1;
  while (__any_sync(0xffffffffu, next >= 0)) {
    const int src = next >= 0 ? next : lane;
#pragma unroll
    for (int i = 0; i < 9; ++i) {
      const float v = __shfl_sync(0xffffffffu, g[i], src);
      if (next >= 0) g[i] += v;
    }
    const int nn = __shfl_sync(0xffffffffu, next, src);
    next = next >= 0 ? nn : -1;
  }
  if (key >= 0 && lane == __ffs((int)grp) - 1) {
    float* o = out + key * 9;
#pragma unroll
    for (int i = 0; i < 9; ++i)
      if (g[i] != 0.0f) red_add(o + i, g[i]);
  }
}

// grad_bary = conv[row]^T g on converted slots and g elsewhere (written once); grad_conversion[row] += g b^T.
__global__ void __launch_bounds__(kThreads)
    clip_convert_backward_kernel(const float* __restrict__ grad_bary_out, const int64_t* __restrict__ pix_to_face,
                                 const float* __restrict__ bary, int64_t S, const float* __restrict__ conversion,
                                 const int64_t* __restrict__ conv_idx, float* __restrict__ grad_bary,
                                 float* __restrict__ grad_conversion) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t s0 = (int64_t)blockIdx.x * blockDim.x; s0 < S; s0 += stride) {  // warp-uniform trip count
    const int64_t s = s0 + threadIdx.x;
    const bool active = s < S;
    const int64_t f = active ? __ldg(pix_to_face + s) : -1;
    const int64_t row = f >= 0 ? __ldg(conv_idx + f) : -1;
    float g[3] = {0.0f, 0.0f, 0.0f};
    if (active) {
#pragma unroll
      for (int i = 0; i < 3; ++i) g[i] = __ldg(grad_bary_out + s * 3 + i);
    }
    if (active && grad_bary != nullptr) {
      float o[3] = {g[0], g[1], g[2]};
      if (row >= 0) {
        const float* m = conversion + row * 9;
#pragma unroll
        for (int k = 0; k < 3; ++k)
          o[k] = __ldg(m + 0 * 3 + k) * g[0] + __ldg(m + 1 * 3 + k) * g[1] + __ldg(m + 2 * 3 + k) * g[2];
      }
#pragma unroll
      for (int k = 0; k < 3; ++k) grad_bary[s * 3 + k] = o[k];
    }
    if (grad_conversion != nullptr) {
      float v[9];
      bool any = false;
      float b[3] = {0.0f, 0.0f, 0.0f};
      if (row >= 0) {
#pragma unroll
        for (int k = 0; k < 3; ++k) b[k] = __ldg(bary + s * 3 + k);
      }
#pragma unroll
      for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          v[i * 3 + k] = g[i] * b[k];
          any = any || v[i * 3 + k] != 0.0f;
        }
      warp_merge_add9(grad_conversion, row >= 0 && any ? row : -1, v);
    }
  }
}

int make_params(const float* face_verts, const float* verts, const int64_t* faces, int64_t F, const float* planes,
                int32_t cull_mask, int32_t has_z_clip, double z_clip, int32_t perspective_correct, ClipParams& p) {
  if (F < 0) return fail(B200R_ERR_INVALID_ARGUMENT, "negative number of faces");
  if (F > INT32_MAX) return fail(B200R_ERR_INVALID_ARGUMENT, "more than 2^31-1 packed faces are not supported");
  if (cull_mask != 0 && planes == nullptr) return fail(B200R_ERR_INVALID_ARGUMENT, "planes is required");
  p.face_verts = face_verts;
  p.verts = verts;
  p.faces = faces;
  p.F = F;
  for (int i = 0; i < 6; ++i) p.plane[i] = ((cull_mask >> i) & 1) ? planes[i] : 0.0f;
  p.cull_mask = cull_mask & 0x3f;
  p.has_z = has_z_clip != 0;
  p.perspective = perspective_correct != 0;
  // torch compares with and subtracts the scalar as float32, and its CUDA kernel divides by it as a multiply by the
  // reciprocal taken in double and rounded once to float32 (x / 1.05 on the H100 equals x * (float)(1.0 / 1.05), which
  // differs from x * (1.0f / 1.05f))
  p.z = (float)z_clip;
  p.inv_z = (float)(1.0 / z_clip);
  return B200R_OK;
}

inline int64_t num_ctas(int64_t F) { return (F + kThreads - 1) / kThreads; }

}  // namespace
}  // namespace b200r

using namespace b200r;

extern "C" int64_t b200r_clip_faces_workspace_words(int64_t F) { return kWords + kWords * num_ctas(F < 0 ? 0 : F); }

extern "C" int b200r_clip_faces_count(const float* face_verts, const float* verts, const int64_t* faces, int64_t F,
                                      const float* planes, int32_t cull_mask, int32_t has_z_clip, double z_clip,
                                      int64_t* workspace, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  ClipParams p;
  int rc = make_params(face_verts, verts, faces, F, planes, cull_mask, has_z_clip, z_clip, 0, p);
  if (rc != B200R_OK) return rc;
  if (face_verts == nullptr && F > 0 && (verts == nullptr || faces == nullptr))
    return fail(B200R_ERR_INVALID_ARGUMENT, "face_verts or (verts, faces) is required");
  const int64_t nb = num_ctas(F);
  if (nb > 0) {
    clip_count_kernel<<<(unsigned)nb, kThreads, 0, stream>>>(p, workspace + kWords);
    B200R_LAUNCHED("clip_count_kernel");
  }
  clip_scan_kernel<<<1, kScanThreads, 0, stream>>>(workspace, workspace + kWords, nb);
  B200R_LAUNCHED("clip_scan_kernel");
  return B200R_OK;
}

extern "C" int b200r_clip_faces_fill(const float* face_verts, int64_t F, const int64_t* mesh_to_face_first_idx,
                                     int32_t N, const float* planes, int32_t cull_mask, int32_t has_z_clip,
                                     double z_clip, int32_t perspective_correct, const int64_t* workspace,
                                     int64_t F_clipped, int64_t n_case3, int64_t n_case4, float* face_verts_clipped,
                                     int64_t* first_clipped, int64_t* num_clipped, int64_t* clipped_to_unclipped,
                                     float* barycentric_conversion, int64_t* clipped_to_conversion,
                                     int64_t* neighbor_idx, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  ClipParams p;
  int rc = make_params(face_verts, nullptr, nullptr, F, planes, cull_mask, has_z_clip, z_clip, perspective_correct, p);
  if (rc != B200R_OK) return rc;
  if (N < 0 || F_clipped < 0 || n_case3 < 0 || n_case4 < 0) return fail(B200R_ERR_INVALID_ARGUMENT, "negative size");
  const bool convert = n_case3 + n_case4 > 0;
  if (convert && (barycentric_conversion == nullptr || clipped_to_conversion == nullptr || neighbor_idx == nullptr))
    return fail(B200R_ERR_INVALID_ARGUMENT, "clipped faces need the conversion and neighbour outputs");
  const int64_t nb = num_ctas(F);
  if (nb > 0) {
    const FillOut o{face_verts_clipped, clipped_to_unclipped, convert ? barycentric_conversion : nullptr,
                    clipped_to_conversion, neighbor_idx, n_case3, n_case4};
    clip_fill_kernel<<<(unsigned)nb, kThreads, 0, stream>>>(p, workspace + kWords, o);
    B200R_LAUNCHED("clip_fill_kernel");
  }
  if (N > 0) {
    clip_meshes_kernel<<<(unsigned)div_up(N, kThreads), kThreads, 0, stream>>>(
        mesh_to_face_first_idx, N, clipped_to_unclipped, F_clipped, first_clipped, num_clipped);
    B200R_LAUNCHED("clip_meshes_kernel");
  }
  return B200R_OK;
}

extern "C" int b200r_clip_faces_backward(const float* face_verts, int64_t F, const float* planes, int32_t cull_mask,
                                         int32_t has_z_clip, double z_clip, int32_t perspective_correct,
                                         const int64_t* workspace, int64_t n_case3, int64_t n_case4,
                                         const float* grad_face_verts_clipped, const float* grad_conversion,
                                         float* grad_face_verts, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  ClipParams p;
  int rc = make_params(face_verts, nullptr, nullptr, F, planes, cull_mask, has_z_clip, z_clip, perspective_correct, p);
  if (rc != B200R_OK) return rc;
  const int64_t nb = num_ctas(F);
  if (nb == 0) return B200R_OK;
  clip_backward_kernel<<<(unsigned)nb, kThreads, 0, stream>>>(p, workspace + kWords, n_case3, n_case4,
                                                               grad_face_verts_clipped, grad_conversion,
                                                               grad_face_verts);
  B200R_LAUNCHED("clip_backward_kernel");
  return B200R_OK;
}

extern "C" int b200r_clip_convert_forward(const int64_t* pix_to_face, const float* barycentric_coords, int64_t S,
                                          const int64_t* clipped_to_unclipped, const float* barycentric_conversion,
                                          const int64_t* clipped_to_conversion, int64_t* pix_to_face_unclipped,
                                          float* barycentric_coords_unclipped, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (S < 0) return fail(B200R_ERR_INVALID_ARGUMENT, "negative size");
  if (barycentric_coords_unclipped != nullptr && (barycentric_conversion == nullptr || clipped_to_conversion == nullptr))
    return fail(B200R_ERR_INVALID_ARGUMENT, "converting barycentrics needs the conversion rows and their index");
  if (S == 0) return B200R_OK;
  const dim3 grid((unsigned)cap_grid_stride_blocks((S + kThreads - 1) / kThreads));
  clip_convert_forward_kernel<<<grid, kThreads, 0, stream>>>(pix_to_face, barycentric_coords, S, clipped_to_unclipped,
                                                            barycentric_conversion, clipped_to_conversion,
                                                            pix_to_face_unclipped, barycentric_coords_unclipped);
  B200R_LAUNCHED("clip_convert_forward_kernel");
  return B200R_OK;
}

extern "C" int b200r_clip_convert_backward(const float* grad_barycentric_coords_unclipped, const int64_t* pix_to_face,
                                           const float* barycentric_coords, int64_t S,
                                           const float* barycentric_conversion, const int64_t* clipped_to_conversion,
                                           int64_t T, float* grad_barycentric_coords, float* grad_conversion,
                                           void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (S < 0 || T < 0) return fail(B200R_ERR_INVALID_ARGUMENT, "negative size");
  if (grad_conversion != nullptr && T > 0)
    B200R_CUDA_OK(cudaMemsetAsync(grad_conversion, 0, sizeof(float) * (size_t)T * 9, stream));
  if (S == 0 || (grad_barycentric_coords == nullptr && grad_conversion == nullptr)) return B200R_OK;
  const dim3 grid((unsigned)cap_grid_stride_blocks((S + kThreads - 1) / kThreads));
  clip_convert_backward_kernel<<<grid, kThreads, 0, stream>>>(grad_barycentric_coords_unclipped, pix_to_face,
                                                             barycentric_coords, S, barycentric_conversion,
                                                             clipped_to_conversion, grad_barycentric_coords,
                                                             grad_conversion);
  B200R_LAUNCHED("clip_convert_backward_kernel");
  return B200R_OK;
}
