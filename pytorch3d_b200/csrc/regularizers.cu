// Mesh regularisers: edge loss, Laplacian smoothing and normal consistency, forward and deterministic backward
// (DESIGN.md section 18).  The results are those of pytorch3d/loss/mesh_edge_loss.py, mesh_laplacian_smoothing.py and
// mesh_normal_consistency.py.
//
// The edge table.  Face-edge j of face f has the id c = j * F + f and the endpoints (f1, f2), (f2, f0), (f0, f1) for
// j = 0, 1, 2 (the order of Meshes._compute_edges_packed), keyed by min << b | max over b = key_bits(V) bits (64-bit
// keys once 2b > 32).  A stable radix sort of the 3F (key, id) pairs puts the face-edges of one undirected edge into one
// run; the runs, in ascending (min, max) order, are the reference's edges_packed, and an inclusive scan of the run heads
// numbers them (faces_packed_to_edges_packed).  Meshes own contiguous ascending vertex ranges, so each mesh's edges are
// the contiguous runs whose min lies in its range, found by binary search.  The edge count E stays on the device: the
// kernels are sized by the bound 3F and threads past E exit.  A face index outside [0, V) gives a key past every edge
// and belongs to no edge.
//
// The adjacency.  The directed copies 2e + side of the E edges, keyed by their source vertex and put into runs per
// vertex (sort_into_runs of keyed_runs.cuh), list each vertex's incident edges in edge order, which is also ascending
// neighbour order; a self-loop (i, i) appears twice, as in the coalesced adjacency of laplacian().
//
// cot and cotcurv walk the vertex -> corner table of mesh_tables.cuh: a corner's row of L is the cotangents of its
// face's two other angles against the two other corners.
//
// Every per-vertex, per-edge and per-mesh sum is one thread in a fixed order; the scalar is a fixed-shape tree (per
// block partials over a grid that depends on the length only, then one block).  There are no float atomics, nothing
// synchronises the host, and the workspace depends only on (V, F, N).  The forward leaves its tables in the workspace,
// and the backward reads them without sorting again; each backward writes each vertex's gradient once.
#include <cub/device/device_scan.cuh>

#include "mesh_tables.cuh"

namespace b200r {
namespace {

constexpr int kReduceBlocksMax = 1024;
constexpr float kCosEps = 1e-8f;       // torch.cosine_similarity's default eps
constexpr float kAreaClamp = 1e-12f;   // cot_laplacian's eps

// Separately rounded vector arithmetic: no product is contracted into an FMA with a sum.  The cotangent rows cancel
// terms near 1e6 (clamped areas), where an FMA's unrounded product leaves a residue that the reference's torch ops,
// rounding each step, do not have; a vertex whose faces are all clamped scales that residue by 0.25 / 1e-6.
__device__ __forceinline__ float3 sub3(float3 a, float3 b) {
  return make_float3(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y), __fsub_rn(a.z, b.z));
}
__device__ __forceinline__ float3 add3(float3 a, float3 b) {
  return make_float3(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y), __fadd_rn(a.z, b.z));
}
__device__ __forceinline__ float3 scale3(float3 a, float s) {
  return make_float3(__fmul_rn(a.x, s), __fmul_rn(a.y, s), __fmul_rn(a.z, s));
}
__device__ __forceinline__ float dot3(float3 a, float3 b) {
  return __fadd_rn(__fadd_rn(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)), __fmul_rn(a.z, b.z));
}
__device__ __forceinline__ float3 cross3(float3 a, float3 b) {
  return make_float3(__fsub_rn(__fmul_rn(a.y, b.z), __fmul_rn(a.z, b.y)),
                     __fsub_rn(__fmul_rn(a.z, b.x), __fmul_rn(a.x, b.z)),
                     __fsub_rn(__fmul_rn(a.x, b.y), __fmul_rn(a.y, b.x)));
}
__device__ __forceinline__ float3 vert3(const float* __restrict__ verts, int64_t v) { return load3(verts, v); }

// The corners (a, b) of face-edge j: (1, 2), (2, 0), (0, 1).
__device__ __forceinline__ int edge_corner_a(int j) { return j == 0 ? 1 : (j == 1 ? 2 : 0); }
__device__ __forceinline__ int edge_corner_b(int j) { return j == 0 ? 2 : (j == 1 ? 0 : 1); }

__device__ __forceinline__ float mesh_weight(const int64_t* __restrict__ first, const int64_t* __restrict__ num, int N,
                                             int64_t v) {
  const int m = find_owner(first, num, N, v);
  return m < 0 ? 0.0f : 1.0f / (float)__ldg(num + m);
}

// ---- the edge table -----------------------------------------------------------------------------------------------

template <typename Key>
__global__ void __launch_bounds__(kThreads)
    edge_keys_kernel(const int64_t* __restrict__ faces, int64_t F, int64_t V, int bits, Key* __restrict__ keys,
                     int32_t* __restrict__ ids) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const Key invalid = ((Key)V << bits) | (Key)V;
  for (int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; f < F; f += stride) {
    int64_t v[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) v[k] = __ldg(faces + 3 * f + k);
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      const int64_t a = v[edge_corner_a(j)], b = v[edge_corner_b(j)];
      const bool ok = a >= 0 && a < V && b >= 0 && b < V;
      const int64_t lo = a < b ? a : b, hi = a < b ? b : a;
      keys[j * F + f] = ok ? (((Key)lo << bits) | (Key)hi) : invalid;
      ids[j * F + f] = (int32_t)(j * F + f);
    }
  }
}

template <typename Key>
__device__ __forceinline__ bool key_valid(Key k, int bits, int64_t V) {
  return (int64_t)(k >> bits) < V;
}

template <typename Key>
__global__ void __launch_bounds__(kThreads)
    edge_heads_kernel(const Key* __restrict__ keys, int64_t n, int64_t V, int bits, int64_t* __restrict__ heads) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const Key k = keys[i];
    heads[i] = (key_valid(k, bits, V) && (i == 0 || keys[i - 1] != k)) ? 1 : 0;
  }
}

// run[i] = the inclusive scan of the heads at i, narrowed; for each run head: edge_start[e] and the endpoints; the
// last valid position writes edge_start[E] and E.  (E = 0 and edge_start[0] = 0 are set before the launch, for the
// case of no valid face-edge.)
template <typename Key>
__global__ void __launch_bounds__(kThreads)
    edge_runs_kernel(const Key* __restrict__ keys, const int64_t* __restrict__ scan, int64_t n, int64_t V, int bits,
                     int32_t* __restrict__ run, int32_t* __restrict__ edge_start, int32_t* __restrict__ edge_v,
                     int32_t* __restrict__ num_edges) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const Key k = keys[i];
    const int32_t r = (int32_t)scan[i];
    run[i] = r;
    const int64_t lo = (int64_t)(k >> bits);
    if (lo >= V) continue;
    const int32_t e = r - 1;
    const Key prev = i > 0 ? keys[i - 1] : ~k;
    const Key next = i + 1 < n ? keys[i + 1] : ~(Key)0;  // all ones: past every vertex
    if (prev != k) {
      edge_start[e] = (int32_t)i;
      edge_v[2 * e] = (int32_t)lo;
      edge_v[2 * e + 1] = (int32_t)(k - ((Key)lo << bits));
    }
    if ((int64_t)(next >> bits) >= V) {
      edge_start[e + 1] = (int32_t)(i + 1);
      *num_edges = e + 1;
    }
  }
}

// rank[i] = the position of sorted face-edge i within its run: the number of pairs it closes with earlier ones.
__global__ void __launch_bounds__(kThreads)
    pair_ranks_kernel(const int32_t* __restrict__ run, const int32_t* __restrict__ edge_start,
                      const int32_t* __restrict__ num_edges, int64_t n, int64_t* __restrict__ rank) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int32_t E = *num_edges;
  const int32_t valid = E > 0 ? edge_start[E] : 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
    rank[i] = i < valid ? i - edge_start[run[i] - 1] : 0;
}

// The first edge whose min is >= v (edges [0, E) in ascending order).
__device__ __forceinline__ int32_t edge_lower_bound(const int32_t* __restrict__ edge_v, int32_t E, int64_t v) {
  int32_t lo = 0, hi = E;
  while (lo < hi) {
    const int32_t mid = (lo + hi) >> 1;
    if ((int64_t)edge_v[2 * mid] < v)
      lo = mid + 1;
    else
      hi = mid;
  }
  return lo;
}

// Per mesh: its edges [edge_begin, edge_begin + edge_count) and, when pair_prefix is given, its number of face pairs.
__global__ void __launch_bounds__(kThreads)
    mesh_ranges_kernel(const int64_t* __restrict__ first, const int64_t* __restrict__ num, int N,
                       const int32_t* __restrict__ edge_v, const int32_t* __restrict__ edge_start,
                       const int32_t* __restrict__ num_edges, const int64_t* __restrict__ pair_prefix,
                       int32_t* __restrict__ edge_begin, int32_t* __restrict__ edge_count,
                       int64_t* __restrict__ pairs) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= N) return;
  const int32_t E = *num_edges;
  const int64_t f = __ldg(first + m);
  const int32_t lo = edge_lower_bound(edge_v, E, f), hi = edge_lower_bound(edge_v, E, f + __ldg(num + m));
  edge_begin[m] = lo;
  edge_count[m] = hi - lo;
  if (pair_prefix != nullptr) pairs[m] = hi > lo ? pair_prefix[edge_start[hi]] - pair_prefix[edge_start[lo]] : 0;
}

// ---- the adjacency ------------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(kThreads)
    adjacency_keys_kernel(const int32_t* __restrict__ edge_v, const int32_t* __restrict__ num_edges, int64_t n,
                          int64_t V, uint32_t* __restrict__ keys, int32_t* __restrict__ ids) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t E = *num_edges;
  for (int64_t d = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; d < n; d += stride) {
    keys[d] = (d >> 1) < E ? (uint32_t)edge_v[d] : (uint32_t)V;
    ids[d] = (int32_t)d;
  }
}

// ---- the scalar ---------------------------------------------------------------------------------------------------

int reduce_blocks(int64_t n) {
  const int64_t b = (n + 4 * kThreads - 1) / (4 * kThreads);
  return (int)(b < 1 ? 1 : (b > kReduceBlocksMax ? kReduceBlocksMax : b));
}

__device__ __forceinline__ float block_sum(float v) {
  __shared__ float s[kThreads];
  s[threadIdx.x] = v;
  __syncthreads();
#pragma unroll
  for (int w = kThreads / 2; w > 0; w >>= 1) {
    if ((int)threadIdx.x < w) s[threadIdx.x] = s[threadIdx.x] + s[threadIdx.x + w];
    __syncthreads();
  }
  return s[0];
}

// Block b sums terms [b * chunk, (b + 1) * chunk): each thread a strided run in order, then a fixed tree.
__global__ void __launch_bounds__(kThreads)
    reduce_partials_kernel(const float* __restrict__ terms, int64_t n, float* __restrict__ partials) {
  const int64_t chunk = (n + gridDim.x - 1) / gridDim.x;
  const int64_t begin = (int64_t)blockIdx.x * chunk;
  const int64_t end = begin + chunk < n ? begin + chunk : n;
  float acc = 0.0f;
  for (int64_t i = begin + threadIdx.x; i < end; i += kThreads) acc += terms[i];
  const float total = block_sum(acc);
  if (threadIdx.x == 0) partials[blockIdx.x] = total;
}

__global__ void __launch_bounds__(kThreads)
    reduce_final_kernel(const float* __restrict__ partials, int blocks, int N, float* __restrict__ out) {
  float acc = 0.0f;
  for (int i = threadIdx.x; i < blocks; i += kThreads) acc += partials[i];
  const float total = block_sum(acc);
  if (threadIdx.x == 0) *out = total / (float)N;
}

// ---- edge loss ----------------------------------------------------------------------------------------------------

__device__ __forceinline__ float edge_weight(const int64_t* __restrict__ first, const int64_t* __restrict__ num, int N,
                                             const int32_t* __restrict__ edge_count, int64_t v0) {
  const int m = find_owner(first, num, N, v0);
  return m < 0 ? 0.0f : 1.0f / (float)edge_count[m];
}

__global__ void __launch_bounds__(kThreads)
    edge_terms_kernel(const float* __restrict__ verts, const int32_t* __restrict__ edge_v,
                      const int32_t* __restrict__ num_edges, int64_t n, const int64_t* __restrict__ first,
                      const int64_t* __restrict__ num, int N, const int32_t* __restrict__ edge_count, float target,
                      float* __restrict__ terms) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t E = *num_edges;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += stride) {
    float t = 0.0f;
    if (e < E) {
      const int64_t a = edge_v[2 * e], b = edge_v[2 * e + 1];
      const float l = norm3(sub3(vert3(verts, a), vert3(verts, b))) - target;
      t = l * l * edge_weight(first, num, N, edge_count, a);
    }
    terms[e] = t;
  }
}

// rows[e] = d loss / d v0 of edge e (v1 gets its negative); 0 for a zero-length edge, as torch's norm backward.
__global__ void __launch_bounds__(kThreads)
    edge_grad_rows_kernel(const float* __restrict__ grad_loss, const float* __restrict__ verts,
                          const int32_t* __restrict__ edge_v, const int32_t* __restrict__ num_edges, int64_t n,
                          const int64_t* __restrict__ first, const int64_t* __restrict__ num, int N,
                          const int32_t* __restrict__ edge_count, float target, float* __restrict__ rows) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t E = *num_edges;
  const float g = __ldg(grad_loss) / (float)N;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n && e < E; e += stride) {
    const int64_t a = edge_v[2 * e], b = edge_v[2 * e + 1];
    const float3 d = sub3(vert3(verts, a), vert3(verts, b));
    const float len = norm3(d);
    const float coef = g * edge_weight(first, num, N, edge_count, a) * 2.0f * (len - target);
    store3(rows, e, len == 0.0f ? make_float3(0.0f, 0.0f, 0.0f) : scale3(d, coef / len));
  }
}

// The row of directed copy d = 2e + side in the adjacency of v: rows[e], added where v is the edge's min (side 0) and
// subtracted where it is the max.
struct EdgeRows : AddedRows {
  const float* rows;
  __device__ float3 operator()(int64_t, int32_t d) const { return load3(rows, d >> 1); }
  __device__ static bool negated(int32_t d) { return d & 1; }
};

// ---- Laplacian smoothing ------------------------------------------------------------------------------------------

// y_i = sum over the adjacency of v_j / deg_i - v_i (-v_i for an isolated vertex).
__device__ __forceinline__ float3 uniform_row(const float* __restrict__ verts, const int32_t* __restrict__ offsets,
                                              const int32_t* __restrict__ adjacency,
                                              const int32_t* __restrict__ edge_v, int64_t v, int32_t& deg) {
  const int32_t b = offsets[v], e = offsets[v + 1];
  deg = e - b;
  float3 acc = make_float3(0.0f, 0.0f, 0.0f);
  const float r = deg > 0 ? 1.0f / (float)deg : 0.0f;
  for (int32_t i = b; i < e; ++i) {
    const int32_t d = adjacency[i];
    const float3 p = vert3(verts, edge_v[d ^ 1]);  // the other endpoint of directed copy d
    acc = make_float3(fmaf(r, p.x, acc.x), fmaf(r, p.y, acc.y), fmaf(r, p.z, acc.z));
  }
  return sub3(acc, vert3(verts, v));
}

struct CotRow {
  float3 y;     // the row of the loss before its norm
  float w;      // norm_w
  float lsum;   // the row sum of L
};

// The row of L.v, its row sum and the vertex's area sum, over its corners; then y for cot or cotcurv.
__device__ __forceinline__ CotRow cot_row(const float* __restrict__ verts, const int64_t* __restrict__ faces,
                                          const int32_t* __restrict__ offsets, const int32_t* __restrict__ corners,
                                          const float* __restrict__ cotarea, int64_t V, int64_t F, int64_t v,
                                          bool curv) {
  float3 lv = make_float3(0.0f, 0.0f, 0.0f);
  float ls = 0.0f, as = 0.0f;
  for (int32_t i = offsets[v]; i < offsets[v + 1]; ++i) {
    const int64_t c = corners[i];
    const int j = c >= 2 * F ? 2 : (c >= F ? 1 : 0);
    const int64_t f = c - j * F;
    const int j1 = j == 2 ? 0 : j + 1, j2 = j == 0 ? 2 : j - 1;
    const float c1 = cotarea[4 * f + j1], c2 = cotarea[4 * f + j2];
    const int64_t a = __ldg(faces + 3 * f + j1), b = __ldg(faces + 3 * f + j2);
    const float nan = __int_as_float(0x7fc00000);
    const float3 pa = (a >= 0 && a < V) ? vert3(verts, a) : make_float3(nan, nan, nan);
    const float3 pb = (b >= 0 && b < V) ? vert3(verts, b) : make_float3(nan, nan, nan);
    // corner j's row: the next corner weighted by the cotangent at the one after, and vice versa
    lv = add3(lv, add3(scale3(pa, c2), scale3(pb, c1)));
    ls = __fadd_rn(ls, __fadd_rn(c1, c2));
    as = __fadd_rn(as, cotarea[4 * f + 3]);
  }
  const float3 p = vert3(verts, v);
  CotRow r;
  r.lsum = ls;
  if (!curv) {
    r.w = ls > 0.0f ? 1.0f / ls : ls;  // the reference leaves non-positive row sums as they are
    r.y = sub3(scale3(lv, r.w), p);
  } else {
    r.w = 0.25f * (as > 0.0f ? 1.0f / as : 0.0f);
    r.y = scale3(sub3(lv, scale3(p, ls)), r.w);
  }
  return r;
}

// Per face: the three cotangents / 4 (of the angles at corners 0, 1, 2) and Heron's area, clamped as the reference.
__global__ void __launch_bounds__(kThreads)
    cot_faces_kernel(const float* __restrict__ verts, const int64_t* __restrict__ faces, int64_t V, int64_t F,
                     float* __restrict__ cotarea) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; f < F; f += stride) {
    float3 p[3];
    face_corners(verts, faces, V, f, p);
    const float A = norm3(sub3(p[1], p[2])), B = norm3(sub3(p[0], p[2])), C = norm3(sub3(p[0], p[1]));
    const float s = __fmul_rn(0.5f, __fadd_rn(__fadd_rn(A, B), C));
    const float prod = __fmul_rn(__fmul_rn(__fmul_rn(s, __fsub_rn(s, A)), __fsub_rn(s, B)), __fsub_rn(s, C));
    const float area = __fsqrt_rn(prod < kAreaClamp ? kAreaClamp : prod);  // clamp(min=eps): NaN stays NaN
    const float A2 = __fmul_rn(A, A), B2 = __fmul_rn(B, B), C2 = __fmul_rn(C, C);
    cotarea[4 * f + 0] = __fmul_rn(__fdiv_rn(__fsub_rn(__fadd_rn(B2, C2), A2), area), 0.25f);
    cotarea[4 * f + 1] = __fmul_rn(__fdiv_rn(__fsub_rn(__fadd_rn(A2, C2), B2), area), 0.25f);
    cotarea[4 * f + 2] = __fmul_rn(__fdiv_rn(__fsub_rn(__fadd_rn(A2, B2), C2), area), 0.25f);
    cotarea[4 * f + 3] = area;
  }
}

// METHOD 0 uniform, 1 cot, 2 cotcurv: terms[v] = |y_v| / V_mesh(v).
template <int METHOD>
__global__ void __launch_bounds__(kThreads)
    laplacian_terms_kernel(const float* __restrict__ verts, const int64_t* __restrict__ faces, int64_t V, int64_t F,
                           const int32_t* __restrict__ offsets, const int32_t* __restrict__ entries,
                           const int32_t* __restrict__ edge_v, const float* __restrict__ cotarea,
                           const int64_t* __restrict__ first, const int64_t* __restrict__ num, int N,
                           float* __restrict__ terms) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < V; v += stride) {
    float3 y;
    if (METHOD == 0) {
      int32_t deg;
      y = uniform_row(verts, offsets, entries, edge_v, v, deg);
    } else {
      y = cot_row(verts, faces, offsets, entries, cotarea, V, F, v, METHOD == 2).y;
    }
    terms[v] = norm3(y) * mesh_weight(first, num, N, v);
  }
}

// Backward, first pass.  G_v = d loss / d y_v (0 where |y_v| = 0); h[v] = G_v scaled by the row's constant (1 / deg
// for uniform, norm_w for cot and cotcurv) and grad_verts[v] = the diagonal part: G_v (uniform, cot) or lsum * h[v]
// (cotcurv).  The second pass adds (L^T h)_v, with L symmetric for cot.
template <int METHOD>
__global__ void __launch_bounds__(kThreads)
    laplacian_backward_rows_kernel(const float* __restrict__ grad_loss, const float* __restrict__ verts,
                                   const int64_t* __restrict__ faces, int64_t V, int64_t F,
                                   const int32_t* __restrict__ offsets, const int32_t* __restrict__ entries,
                                   const int32_t* __restrict__ edge_v, const float* __restrict__ cotarea,
                                   const int64_t* __restrict__ first, const int64_t* __restrict__ num, int N,
                                   float* __restrict__ h, float* __restrict__ grad_verts) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const float g = __ldg(grad_loss) / (float)N;
  for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < V; v += stride) {
    float3 y;
    float scale, lsum = 0.0f;
    if (METHOD == 0) {
      int32_t deg;
      y = uniform_row(verts, offsets, entries, edge_v, v, deg);
      scale = deg > 0 ? 1.0f / (float)deg : 0.0f;
    } else {
      const CotRow r = cot_row(verts, faces, offsets, entries, cotarea, V, F, v, METHOD == 2);
      y = r.y;
      scale = r.w;
      lsum = r.lsum;
    }
    const float n = norm3(y);
    const float k = n == 0.0f ? 0.0f : g * mesh_weight(first, num, N, v) / n;
    const float3 G = scale3(y, k);
    const float3 H = scale3(G, scale);
    store3(h, v, H);
    store3(grad_verts, v, METHOD == 2 ? scale3(H, lsum) : G);
  }
}

template <int METHOD>
__global__ void __launch_bounds__(kThreads)
    laplacian_backward_verts_kernel(const int64_t* __restrict__ faces, int64_t V, int64_t F,
                                    const int32_t* __restrict__ offsets, const int32_t* __restrict__ entries,
                                    const int32_t* __restrict__ edge_v, const float* __restrict__ cotarea,
                                    const float* __restrict__ h, float* __restrict__ grad_verts) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < V; v += stride) {
    float3 acc = make_float3(0.0f, 0.0f, 0.0f);
    for (int32_t i = offsets[v]; i < offsets[v + 1]; ++i) {
      if (METHOD == 0) {
        acc = add3(acc, load3(h, edge_v[entries[i] ^ 1]));
      } else {
        const int64_t c = entries[i];
        const int j = c >= 2 * F ? 2 : (c >= F ? 1 : 0);
        const int64_t f = c - j * F;
        const int j1 = j == 2 ? 0 : j + 1, j2 = j == 0 ? 2 : j - 1;
        const int64_t a = __ldg(faces + 3 * f + j1), b = __ldg(faces + 3 * f + j2);
        if (a >= 0 && a < V) acc = add3(acc, scale3(load3(h, a), cotarea[4 * f + j2]));
        if (b >= 0 && b < V) acc = add3(acc, scale3(load3(h, b), cotarea[4 * f + j1]));
      }
    }
    store3(grad_verts, v, sub3(acc, load3(grad_verts, v)));
  }
}

// ---- normal consistency -------------------------------------------------------------------------------------------

__device__ __forceinline__ int face_edge_of(int64_t c, int64_t F, int64_t& f) {
  const int j = c >= 2 * F ? 2 : (c >= F ? 1 : 0);
  f = c - j * F;
  return j;
}

// n of sorted face-edge i: sum_k (v1 - v0) x (f_k - v0), v0 and v1 the edge's min and max vertex.
__global__ void __launch_bounds__(kThreads)
    nc_normals_kernel(const float* __restrict__ verts, const int64_t* __restrict__ faces, int64_t V, int64_t F,
                      const int32_t* __restrict__ sorted_ids, const int32_t* __restrict__ run,
                      const int32_t* __restrict__ edge_v, const int32_t* __restrict__ edge_start,
                      const int32_t* __restrict__ num_edges, float* __restrict__ normals) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int32_t E = *num_edges;
  const int64_t valid = E > 0 ? edge_start[E] : 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < valid; i += stride) {
    int64_t f;
    face_edge_of(sorted_ids[i], F, f);
    const int32_t e = run[i] - 1;
    const float3 v0 = vert3(verts, edge_v[2 * e]), v1 = vert3(verts, edge_v[2 * e + 1]);
    float3 p[3];
    face_corners(verts, faces, V, f, p);
    const float3 d = sub3(v1, v0);
    // each cross product as torch.cross rounds it on the CPU, so that d x d of a face with a repeated vertex leaves the
    // same rounding residue as the reference's
    float3 n = cross_fma(d, sub3(p[0], v0));
    n = add3(n, cross_fma(d, sub3(p[1], v0)));
    store3(normals, i, add3(n, cross_fma(d, sub3(p[2], v0))));
  }
}

__device__ __forceinline__ float nc_clamped_norm(float3 n, float& raw) {
  raw = norm3(n);
  return raw < kCosEps ? kCosEps : raw;
}

__device__ __forceinline__ float pair_weight(const int64_t* __restrict__ first, const int64_t* __restrict__ num, int N,
                                             const int64_t* __restrict__ pairs, int64_t v0) {
  const int m = find_owner(first, num, N, v0);
  return m < 0 ? 0.0f : 1.0f / (float)pairs[m];
}

// terms[i] = the sum over the earlier face-edges i' of i's run of 1 - cos(n_i', -n_i), weighted by 1 / the pairs of
// the mesh.  cos is torch's: (a / max(|a|, eps)) . (b / max(|b|, eps)).
__global__ void __launch_bounds__(kThreads)
    nc_terms_kernel(const float* __restrict__ normals, const int32_t* __restrict__ run,
                    const int32_t* __restrict__ edge_v, const int32_t* __restrict__ edge_start,
                    const int32_t* __restrict__ num_edges, int64_t n, const int64_t* __restrict__ first,
                    const int64_t* __restrict__ num, int N, const int64_t* __restrict__ pairs,
                    float* __restrict__ terms) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int32_t E = *num_edges;
  const int64_t valid = E > 0 ? edge_start[E] : 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    float t = 0.0f;
    const int32_t e = i < valid ? run[i] - 1 : 0;
    if (i < valid && edge_start[e] < i) {
      float raw;
      const float3 b = load3(normals, i);
      const float3 ub = scale3(b, -1.0f / nc_clamped_norm(b, raw));
      for (int64_t k = edge_start[e]; k < i; ++k) {
        const float3 a = load3(normals, k);
        const float na = nc_clamped_norm(a, raw);
        const float3 ua = make_float3(a.x / na, a.y / na, a.z / na);
        t += 1.0f - dot3(ua, ub);
      }
      t *= pair_weight(first, num, N, pairs, edge_v[2 * e]);
    }
    terms[i] = t;
  }
}

// grad_n[c] for face-edge id c (sorted position i): the sum over the other face-edges of its run of the gradient of
// their pair's term with respect to n_i, as autograd forms it through cosine_similarity (the clamp under no_grad, the
// norm's gradient 0 where |n| = 0).  Face-edges in no edge get 0.
__global__ void __launch_bounds__(kThreads)
    nc_grad_normals_kernel(const float* __restrict__ grad_loss, const float* __restrict__ normals,
                           const int32_t* __restrict__ sorted_ids, const int32_t* __restrict__ run,
                           const int32_t* __restrict__ edge_v, const int32_t* __restrict__ edge_start,
                           const int32_t* __restrict__ num_edges, int64_t n, const int64_t* __restrict__ first,
                           const int64_t* __restrict__ num, int N, const int64_t* __restrict__ pairs,
                           float* __restrict__ grad_n) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int32_t E = *num_edges;
  const int64_t valid = E > 0 ? edge_start[E] : 0;
  const float g = __ldg(grad_loss) / (float)N;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    float3 acc = make_float3(0.0f, 0.0f, 0.0f);
    const int32_t e = i < valid ? run[i] - 1 : 0;
    if (i < valid && edge_start[e + 1] - edge_start[e] > 1) {  // in at least one pair, so the mesh's count is > 0
      float raw_i;
      const float3 ni = load3(normals, i);
      const float Ai = nc_clamped_norm(ni, raw_i);
      const float3 ui = make_float3(ni.x / Ai, ni.y / Ai, ni.z / Ai);
      const float3 dir = raw_i == 0.0f ? make_float3(0.0f, 0.0f, 0.0f) : scale3(ni, 1.0f / raw_i);
      for (int64_t k = edge_start[e]; k < edge_start[e + 1]; ++k) {
        if (k == i) continue;
        float raw;
        const float3 p = load3(normals, k);
        const float Ap = nc_clamped_norm(p, raw);
        const float3 up = make_float3(p.x / Ap, p.y / Ap, p.z / Ap);
        const float s = dot3(up, ui);
        acc = add3(acc, scale3(sub3(up, scale3(dir, s)), 1.0f / Ai));
      }
      acc = scale3(acc, g * pair_weight(first, num, N, pairs, edge_v[2 * e]));
    }
    store3(grad_n, sorted_ids[i], acc);
  }
}

// Per face: the gradients of its three face-edges' n to its corners, rows (f, k) = d loss / d corner k.
//   n = d x U, d = v1 - v0, U = sum_k (f_k - v0): v1 gets U x g, v0 gets -(U x g) - 3 (g x d), every corner g x d.
// An edge's endpoints are two of its face's corners: (1, 2), (2, 0), (0, 1), ordered by vertex id.
__global__ void __launch_bounds__(kThreads)
    nc_corner_rows_kernel(const float* __restrict__ verts, const int64_t* __restrict__ faces, int64_t V, int64_t F,
                          const float* __restrict__ grad_n, float* __restrict__ rows) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; f < F; f += stride) {
    float3 p[3];
    face_corners(verts, faces, V, f, p);
    int64_t idx[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) idx[k] = __ldg(faces + 3 * f + k);
    float3 r[3] = {make_float3(0.0f, 0.0f, 0.0f), make_float3(0.0f, 0.0f, 0.0f), make_float3(0.0f, 0.0f, 0.0f)};
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      const float3 g = load3(grad_n, j * F + f);
      if (g.x == 0.0f && g.y == 0.0f && g.z == 0.0f) continue;
      const int a = edge_corner_a(j), b = edge_corner_b(j);
      const int c0 = idx[b] < idx[a] ? b : a, c1 = idx[b] < idx[a] ? a : b;
      const float3 d = sub3(p[c1], p[c0]);
      const float3 U = add3(add3(sub3(p[0], p[c0]), sub3(p[1], p[c0])), sub3(p[2], p[c0]));
      const float3 gu = cross3(g, d), gd = cross3(U, g);
#pragma unroll
      for (int k = 0; k < 3; ++k) r[k] = add3(r[k], gu);
      r[c1] = add3(r[c1], gd);
      r[c0] = sub3(r[c0], add3(gd, scale3(gu, 3.0f)));
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) store3(rows, 3 * f + k, r[k]);
  }
}

// ---- the edge-table hook's outputs --------------------------------------------------------------------------------

__global__ void __launch_bounds__(kThreads)
    edge_table_outputs_kernel(const int32_t* __restrict__ sorted_ids, const int32_t* __restrict__ run,
                              const int32_t* __restrict__ edge_v, const int32_t* __restrict__ edge_start,
                              const int32_t* __restrict__ num_edges, int64_t n, int64_t F,
                              int64_t* __restrict__ edges, int64_t* __restrict__ face_to_edge,
                              int64_t* __restrict__ E_out) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int32_t E = *num_edges;
  const int64_t valid = E > 0 ? edge_start[E] : 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    if (i == 0) *E_out = E;
    if (i < E) {
      edges[2 * i] = edge_v[2 * i];
      edges[2 * i + 1] = edge_v[2 * i + 1];
    }
    int64_t f;
    const int j = face_edge_of(sorted_ids[i], F, f);
    face_to_edge[3 * f + j] = i < valid ? run[i] - 1 : -1;
  }
}

// ---- host side ----------------------------------------------------------------------------------------------------

bool wide_keys(int64_t V) { return 2 * key_bits(V) > 32; }

// The workspace: every region is a function of (V, F, N).  `tab` holds the vertex offsets and the corner ids or the
// adjacency; `sorted`, `run`, `estart`, `edge_v`, `ecount`, `ebegin`, `pairs`, `prefix` the edge table; `fpos` the
// normals of the sorted face-edges (normal consistency) or the edge gradient rows; `ftmp` the terms of the scalar,
// then the backward's per-vertex or per-face-edge gradients; `fface` the cotangents and areas, or the corner rows.
struct Layout {
  size_t tab, sorted, run, estart, edge_v, nedges, ebegin, ecount, pairs, prefix, keys_in, keys_out, ids_in, fpos, ftmp,
      fface, partials, cub, cub_bytes, total;
};

bool layout(int64_t V, int64_t F, int N, Layout& L) {
  const size_t n3 = 3 * (size_t)F, n6 = 6 * (size_t)F, v = (size_t)V, nm = (size_t)(N > 0 ? N : 1);
  Carver c;
  L.tab = c.take(sizeof(int32_t) * (v + 1 + n6));
  L.sorted = c.take(sizeof(int32_t) * n3);
  L.run = c.take(sizeof(int32_t) * n3);
  L.estart = c.take(sizeof(int32_t) * (n3 + 1));
  L.edge_v = c.take(sizeof(int32_t) * 2 * n3);
  L.nedges = c.take(sizeof(int32_t));
  L.ebegin = c.take(sizeof(int32_t) * nm);
  L.ecount = c.take(sizeof(int32_t) * nm);
  L.pairs = c.take(sizeof(int64_t) * nm);
  L.prefix = c.take(sizeof(int64_t) * (n3 + 1));
  L.keys_in = c.take(sizeof(uint32_t) * n6);   // 3F 64-bit or 6F 32-bit keys
  L.keys_out = c.take(sizeof(uint32_t) * n6);
  L.ids_in = c.take(sizeof(int32_t) * n6);
  L.fpos = c.take(sizeof(float) * 3 * n3);
  L.ftmp = c.take(sizeof(float) * (3 * v > 3 * n3 ? 3 * v : 3 * n3));
  L.fface = c.take(sizeof(float) * 9 * (size_t)F);
  L.partials = c.take(sizeof(float) * kReduceBlocksMax);
  size_t need = 0, b = 0;
  const int bits = key_bits(V);
  if (n3 > 0) {
    const bool sized = wide_keys(V) ? sort_bytes<uint64_t, int32_t>((int)n3, 2 * bits, b)
                                    : sort_bytes<uint32_t, int32_t>((int)n3, 2 * bits, b);
    if (!sized) return false;
    need = b > need ? b : need;
    if (!run_sort_bytes(V, (int64_t)n6, b)) return false;  // the adjacency; covers the corner table's 3F
    need = b > need ? b : need;
    if (cub::DeviceScan::InclusiveSum(nullptr, b, (const int64_t*)nullptr, (int64_t*)nullptr, (int)n3) != cudaSuccess)
      return false;
    need = b > need ? b : need;
  }
  L.cub_bytes = need;
  L.cub = c.take(need);
  L.total = c.used;
  return true;
}

int check_sizes(const char* op, int64_t V, int64_t F, int N) {
  if (V < 0 || F < 0 || N < 0) return fail(B200R_ERR_INVALID_ARGUMENT, std::string(op) + ": negative size");
  if (N == 0) return fail(B200R_ERR_INVALID_ARGUMENT, std::string(op) + ": needs at least one mesh");
  if (V >= ((int64_t)1 << 31) - 1)
    return fail(B200R_ERR_INVALID_ARGUMENT, std::string(op) + ": at most 2^31 - 2 vertices");
  if (6 * F >= ((int64_t)1 << 31))
    return fail(B200R_ERR_INVALID_ARGUMENT, std::string(op) + ": at most (2^31 - 1) / 6 faces (6F < 2^31)");
  return B200R_OK;
}

int checked_layout(const char* op, int64_t V, int64_t F, int N, size_t workspace_bytes, const void* workspace,
                   Layout& L) {
  int rc = check_sizes(op, V, F, N);
  if (rc != B200R_OK) return rc;
  const bool sized = layout(V, F, N, L);
  return check_workspace(op, "b200r_regularizers_workspace_bytes", sized, L.total, workspace, workspace_bytes);
}

struct Ws {
  char* base;
  const Layout& L;
  template <typename T>
  T* at(size_t off) const { return reinterpret_cast<T*>(base + off); }
  int32_t* tab() const { return at<int32_t>(L.tab); }
  int32_t* sorted() const { return at<int32_t>(L.sorted); }
  int32_t* run() const { return at<int32_t>(L.run); }
  int32_t* estart() const { return at<int32_t>(L.estart); }
  int32_t* edge_v() const { return at<int32_t>(L.edge_v); }
  int32_t* nedges() const { return at<int32_t>(L.nedges); }
  int32_t* ebegin() const { return at<int32_t>(L.ebegin); }
  int32_t* ecount() const { return at<int32_t>(L.ecount); }
  int64_t* pairs() const { return at<int64_t>(L.pairs); }
  int64_t* prefix() const { return at<int64_t>(L.prefix); }
  float* fpos() const { return at<float>(L.fpos); }
  float* ftmp() const { return at<float>(L.ftmp); }
  float* fface() const { return at<float>(L.fface); }
  float* partials() const { return at<float>(L.partials); }
  void* cub() const { return base + L.cub; }
};

template <typename Key>
int sort_edges(const int64_t* faces, int64_t V, int64_t F, const Ws& w, cudaStream_t stream) {
  const int64_t n = 3 * F;
  const int bits = key_bits(V);
  Key* keys_in = w.at<Key>(w.L.keys_in);
  Key* keys_out = w.at<Key>(w.L.keys_out);
  int32_t* ids_in = w.at<int32_t>(w.L.ids_in);
  edge_keys_kernel<Key><<<grid_for(F), kThreads, 0, stream>>>(faces, F, V, bits, keys_in, ids_in);
  B200R_LAUNCHED("edge_keys_kernel");
  size_t cub_bytes = w.L.cub_bytes;
  B200R_CUDA_OK(cub::DeviceRadixSort::SortPairs(w.cub(), cub_bytes, keys_in, keys_out, ids_in, w.sorted(), (int)n, 0,
                                                2 * bits, stream));
  // the scan is 64-bit (cub's 32-bit scan kernel spills on sm_90a); heads and scan use the sort's free input buffers
  int64_t* heads = w.at<int64_t>(w.L.ids_in);
  int64_t* scan = w.at<int64_t>(w.L.keys_in);
  edge_heads_kernel<Key><<<grid_for(n), kThreads, 0, stream>>>(keys_out, n, V, bits, heads);
  B200R_LAUNCHED("edge_heads_kernel");
  cub_bytes = w.L.cub_bytes;
  B200R_CUDA_OK(cub::DeviceScan::InclusiveSum(w.cub(), cub_bytes, heads, scan, (int)n, stream));
  edge_runs_kernel<Key><<<grid_for(n), kThreads, 0, stream>>>(keys_out, scan, n, V, bits, w.run(), w.estart(),
                                                             w.edge_v(), w.nedges());
  B200R_LAUNCHED("edge_runs_kernel");
  return B200R_OK;
}

// The edge table, each mesh's edge range and (with_pairs) its number of face pairs.
int build_edges(const int64_t* faces, int64_t V, int64_t F, const int64_t* first, const int64_t* num, int N,
                bool with_pairs, const Ws& w, cudaStream_t stream) {
  const int64_t n = 3 * F;
  B200R_CUDA_OK(cudaMemsetAsync(w.nedges(), 0, sizeof(int32_t), stream));
  B200R_CUDA_OK(cudaMemsetAsync(w.estart(), 0, sizeof(int32_t), stream));
  if (n > 0) {
    const int rc = wide_keys(V) ? sort_edges<uint64_t>(faces, V, F, w, stream) : sort_edges<uint32_t>(faces, V, F, w,
                                                                                                      stream);
    if (rc != B200R_OK) return rc;
  }
  if (with_pairs) {
    B200R_CUDA_OK(cudaMemsetAsync(w.prefix(), 0, sizeof(int64_t), stream));
    if (n > 0) {
      int64_t* rank = w.at<int64_t>(w.L.keys_in);  // free once sorted
      pair_ranks_kernel<<<grid_for(n), kThreads, 0, stream>>>(w.run(), w.estart(), w.nedges(), n, rank);
      B200R_LAUNCHED("pair_ranks_kernel");
      size_t cub_bytes = w.L.cub_bytes;
      B200R_CUDA_OK(cub::DeviceScan::InclusiveSum(w.cub(), cub_bytes, rank, w.prefix() + 1, (int)n, stream));
    }
  }
  mesh_ranges_kernel<<<div_up(N, kThreads), kThreads, 0, stream>>>(first, num, N, w.edge_v(), w.estart(), w.nedges(),
                                                                    with_pairs ? w.prefix() : nullptr, w.ebegin(),
                                                                    w.ecount(), w.pairs());
  B200R_LAUNCHED("mesh_ranges_kernel");
  return B200R_OK;
}

// The adjacency (offsets[V + 1], then the directed copies of the edges by source vertex) at tab, from the edge table.
int build_adjacency(int64_t V, int64_t F, const Ws& w, cudaStream_t stream) {
  const int64_t n = 6 * F;
  uint32_t* keys_in = w.at<uint32_t>(w.L.keys_in);
  int32_t* ids_in = w.at<int32_t>(w.L.ids_in);
  if (n > 0) {
    adjacency_keys_kernel<<<grid_for(n), kThreads, 0, stream>>>(w.edge_v(), w.nedges(), n, V, keys_in, ids_in);
    B200R_LAUNCHED("adjacency_keys_kernel");
  }
  return sort_into_runs(keys_in, w.at<uint32_t>(w.L.keys_out), ids_in, w.tab() + V + 1, n, V, w.cub(), w.L.cub_bytes,
                        w.tab(), stream);
}

int build_corners(const int64_t* faces, int64_t V, int64_t F, const Ws& w, cudaStream_t stream) {
  return build_table(faces, V, F, w.at<uint32_t>(w.L.keys_in), w.at<uint32_t>(w.L.keys_out),
                     w.at<int32_t>(w.L.ids_in), w.cub(), w.L.cub_bytes, w.tab(), stream);
}

int reduce(const float* terms, int64_t n, int N, const Ws& w, float* out, cudaStream_t stream) {
  const int blocks = reduce_blocks(n);
  reduce_partials_kernel<<<blocks, kThreads, 0, stream>>>(terms, n, w.partials());
  B200R_LAUNCHED("reduce_partials_kernel");
  reduce_final_kernel<<<1, kThreads, 0, stream>>>(w.partials(), blocks, N, out);
  B200R_LAUNCHED("reduce_final_kernel");
  return B200R_OK;
}

}  // namespace
}  // namespace b200r

using namespace b200r;

extern "C" size_t b200r_regularizers_workspace_bytes(int64_t V, int64_t F, int32_t N) {
  if (V < 0 || F < 0 || N < 0) return 0;
  Layout L{};
  const bool sized = layout(V, F, N, L);
  return workspace_size(sized, L.total);
}

#define B200R_REG_PROLOGUE(op)                                                             \
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);                               \
  Layout L{};                                                                              \
  int rc = checked_layout(op, V, F, N, workspace_bytes, workspace, L);                     \
  if (rc != B200R_OK) return rc;                                                           \
  const Ws w{static_cast<char*>(workspace), L};

extern "C" int b200r_mesh_edge_table(const int64_t* faces, int64_t V, int64_t F, const int64_t* mesh_first_vert,
                                     const int64_t* mesh_num_verts, int32_t N, void* workspace,
                                     size_t workspace_bytes, int64_t* edges, int64_t* face_to_edge,
                                     int64_t* num_edges_per_mesh, int64_t* num_edges, void* stream_) {
  B200R_REG_PROLOGUE("mesh_edge_table");
  rc = build_edges(faces, V, F, mesh_first_vert, mesh_num_verts, N, false, w, stream);
  if (rc != B200R_OK) return rc;
  const int64_t n = 3 * F;
  if (n > 0) {
    edge_table_outputs_kernel<<<grid_for(n), kThreads, 0, stream>>>(w.sorted(), w.run(), w.edge_v(), w.estart(),
                                                                    w.nedges(), n, F, edges, face_to_edge, num_edges);
    B200R_LAUNCHED("edge_table_outputs_kernel");
  } else {
    B200R_CUDA_OK(cudaMemsetAsync(num_edges, 0, sizeof(int64_t), stream));
  }
  // the per-mesh counts, widened
  B200R_CUDA_OK(cudaMemsetAsync(num_edges_per_mesh, 0, sizeof(int64_t) * N, stream));
  B200R_CUDA_OK(cudaMemcpy2DAsync(num_edges_per_mesh, sizeof(int64_t), w.ecount(), sizeof(int32_t), sizeof(int32_t), N,
                                  cudaMemcpyDeviceToDevice, stream));
  return B200R_OK;
}

extern "C" int b200r_mesh_edge_loss_forward(const float* verts, int64_t V, const int64_t* faces, int64_t F,
                                            const int64_t* mesh_first_vert, const int64_t* mesh_num_verts, int32_t N,
                                            float target_length, void* workspace, size_t workspace_bytes, float* loss,
                                            void* stream_) {
  B200R_REG_PROLOGUE("mesh_edge_loss_forward");
  rc = build_edges(faces, V, F, mesh_first_vert, mesh_num_verts, N, false, w, stream);
  if (rc != B200R_OK) return rc;
  rc = build_adjacency(V, F, w, stream);
  if (rc != B200R_OK) return rc;
  const int64_t n = 3 * F;
  if (n > 0) {
    edge_terms_kernel<<<grid_for(n), kThreads, 0, stream>>>(verts, w.edge_v(), w.nedges(), n, mesh_first_vert,
                                                            mesh_num_verts, N, w.ecount(), target_length, w.ftmp());
    B200R_LAUNCHED("edge_terms_kernel");
  }
  return reduce(w.ftmp(), n, N, w, loss, stream);
}

extern "C" int b200r_mesh_edge_loss_backward(const float* grad_loss, const float* verts, int64_t V,
                                             const int64_t* faces, int64_t F, const int64_t* mesh_first_vert,
                                             const int64_t* mesh_num_verts, int32_t N, float target_length,
                                             void* workspace, size_t workspace_bytes, float* grad_verts,
                                             void* stream_) {
  B200R_REG_PROLOGUE("mesh_edge_loss_backward");
  (void)faces;
  if (V == 0) return B200R_OK;
  const int64_t n = 3 * F;
  if (n > 0) {
    edge_grad_rows_kernel<<<grid_for(n), kThreads, 0, stream>>>(grad_loss, verts, w.edge_v(), w.nedges(), n,
                                                                mesh_first_vert, mesh_num_verts, N, w.ecount(),
                                                                target_length, w.fpos());
    B200R_LAUNCHED("edge_grad_rows_kernel");
  }
  segmented_sum_kernel<Mode::kSum>
      <<<grid_for(V), kThreads, 0, stream>>>(w.tab(), w.tab() + V + 1, V, EdgeRows{{}, w.fpos()}, nullptr, grad_verts);
  B200R_LAUNCHED("segmented_sum_kernel");
  return B200R_OK;
}

template <int METHOD>
static int laplacian_forward(const float* verts, int64_t V, const int64_t* faces, int64_t F, const int64_t* first,
                             const int64_t* num, int N, const Ws& w, float* loss, cudaStream_t stream) {
  int rc;
  if (METHOD == 0) {
    rc = build_edges(faces, V, F, first, num, N, false, w, stream);
    if (rc != B200R_OK) return rc;
    rc = build_adjacency(V, F, w, stream);
  } else {
    rc = build_corners(faces, V, F, w, stream);
    if (rc == B200R_OK && F > 0) {
      cot_faces_kernel<<<grid_for(F), kThreads, 0, stream>>>(verts, faces, V, F, w.fface());
      B200R_LAUNCHED("cot_faces_kernel");
    }
  }
  if (rc != B200R_OK) return rc;
  if (V > 0) {
    laplacian_terms_kernel<METHOD><<<grid_for(V), kThreads, 0, stream>>>(
        verts, faces, V, F, w.tab(), w.tab() + V + 1, w.edge_v(), w.fface(), first, num, N, w.ftmp());
    B200R_LAUNCHED("laplacian_terms_kernel");
  }
  return reduce(w.ftmp(), V, N, w, loss, stream);
}

template <int METHOD>
static int laplacian_backward(const float* grad_loss, const float* verts, int64_t V, const int64_t* faces, int64_t F,
                              const int64_t* first, const int64_t* num, int N, const Ws& w, float* grad_verts,
                              cudaStream_t stream) {
  if (V == 0) return B200R_OK;
  laplacian_backward_rows_kernel<METHOD><<<grid_for(V), kThreads, 0, stream>>>(
      grad_loss, verts, faces, V, F, w.tab(), w.tab() + V + 1, w.edge_v(), w.fface(), first, num, N, w.ftmp(),
      grad_verts);
  B200R_LAUNCHED("laplacian_backward_rows_kernel");
  laplacian_backward_verts_kernel<METHOD><<<grid_for(V), kThreads, 0, stream>>>(
      faces, V, F, w.tab(), w.tab() + V + 1, w.edge_v(), w.fface(), w.ftmp(), grad_verts);
  B200R_LAUNCHED("laplacian_backward_verts_kernel");
  return B200R_OK;
}

extern "C" int b200r_mesh_laplacian_smoothing_forward(const float* verts, int64_t V, const int64_t* faces, int64_t F,
                                                      const int64_t* mesh_first_vert, const int64_t* mesh_num_verts,
                                                      int32_t N, int32_t method, void* workspace,
                                                      size_t workspace_bytes, float* loss, void* stream_) {
  B200R_REG_PROLOGUE("mesh_laplacian_smoothing_forward");
  switch (method) {
    case B200R_LAPLACIAN_UNIFORM:
      return laplacian_forward<0>(verts, V, faces, F, mesh_first_vert, mesh_num_verts, N, w, loss, stream);
    case B200R_LAPLACIAN_COT:
      return laplacian_forward<1>(verts, V, faces, F, mesh_first_vert, mesh_num_verts, N, w, loss, stream);
    case B200R_LAPLACIAN_COTCURV:
      return laplacian_forward<2>(verts, V, faces, F, mesh_first_vert, mesh_num_verts, N, w, loss, stream);
  }
  return fail(B200R_ERR_INVALID_ARGUMENT, "mesh_laplacian_smoothing_forward: Method should be one of {uniform, cot, "
                                          "cotcurv}");
}

extern "C" int b200r_mesh_laplacian_smoothing_backward(const float* grad_loss, const float* verts, int64_t V,
                                                       const int64_t* faces, int64_t F,
                                                       const int64_t* mesh_first_vert, const int64_t* mesh_num_verts,
                                                       int32_t N, int32_t method, void* workspace,
                                                       size_t workspace_bytes, float* grad_verts, void* stream_) {
  B200R_REG_PROLOGUE("mesh_laplacian_smoothing_backward");
  switch (method) {
    case B200R_LAPLACIAN_UNIFORM:
      return laplacian_backward<0>(grad_loss, verts, V, faces, F, mesh_first_vert, mesh_num_verts, N, w, grad_verts,
                                   stream);
    case B200R_LAPLACIAN_COT:
      return laplacian_backward<1>(grad_loss, verts, V, faces, F, mesh_first_vert, mesh_num_verts, N, w, grad_verts,
                                   stream);
    case B200R_LAPLACIAN_COTCURV:
      return laplacian_backward<2>(grad_loss, verts, V, faces, F, mesh_first_vert, mesh_num_verts, N, w, grad_verts,
                                   stream);
  }
  return fail(B200R_ERR_INVALID_ARGUMENT, "mesh_laplacian_smoothing_backward: Method should be one of {uniform, cot, "
                                          "cotcurv}");
}

extern "C" int b200r_mesh_normal_consistency_forward(const float* verts, int64_t V, const int64_t* faces, int64_t F,
                                                     const int64_t* mesh_first_vert, const int64_t* mesh_num_verts,
                                                     int32_t N, void* workspace, size_t workspace_bytes, float* loss,
                                                     void* stream_) {
  B200R_REG_PROLOGUE("mesh_normal_consistency_forward");
  rc = build_edges(faces, V, F, mesh_first_vert, mesh_num_verts, N, true, w, stream);
  if (rc != B200R_OK) return rc;
  rc = build_corners(faces, V, F, w, stream);
  if (rc != B200R_OK) return rc;
  const int64_t n = 3 * F;
  if (n > 0) {
    nc_normals_kernel<<<grid_for(n), kThreads, 0, stream>>>(verts, faces, V, F, w.sorted(), w.run(), w.edge_v(),
                                                            w.estart(), w.nedges(), w.fpos());
    B200R_LAUNCHED("nc_normals_kernel");
    nc_terms_kernel<<<grid_for(n), kThreads, 0, stream>>>(w.fpos(), w.run(), w.edge_v(), w.estart(), w.nedges(), n,
                                                          mesh_first_vert, mesh_num_verts, N, w.pairs(), w.ftmp());
    B200R_LAUNCHED("nc_terms_kernel");
  }
  return reduce(w.ftmp(), n, N, w, loss, stream);
}

extern "C" int b200r_mesh_normal_consistency_backward(const float* grad_loss, const float* verts, int64_t V,
                                                      const int64_t* faces, int64_t F,
                                                      const int64_t* mesh_first_vert, const int64_t* mesh_num_verts,
                                                      int32_t N, void* workspace, size_t workspace_bytes,
                                                      float* grad_verts, void* stream_) {
  B200R_REG_PROLOGUE("mesh_normal_consistency_backward");
  if (V == 0) return B200R_OK;
  const int64_t n = 3 * F;
  if (n > 0) {
    nc_grad_normals_kernel<<<grid_for(n), kThreads, 0, stream>>>(grad_loss, w.fpos(), w.sorted(), w.run(), w.edge_v(),
                                                                 w.estart(), w.nedges(), n, mesh_first_vert,
                                                                 mesh_num_verts, N, w.pairs(), w.ftmp());
    B200R_LAUNCHED("nc_grad_normals_kernel");
    nc_corner_rows_kernel<<<grid_for(F), kThreads, 0, stream>>>(verts, faces, V, F, w.ftmp(), w.fface());
    B200R_LAUNCHED("nc_corner_rows_kernel");
  }
  segmented_sum_kernel<Mode::kSum>
      <<<grid_for(V), kThreads, 0, stream>>>(w.tab(), w.tab() + V + 1, V, CornerRows<true>{{}, w.fface(), F}, nullptr,
                                             grad_verts);
  B200R_LAUNCHED("segmented_sum_kernel");
  return B200R_OK;
}
