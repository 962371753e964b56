/*
 * b200_raster.h -- C ABI of the H100-native differentiable rasterizer (libb200raster.so).
 *
 * This is the drop-in boundary for PyTorch3D's native rasterizer ops.  The reference reaches its
 * kernels through the pybind11 module pytorch3d._C (pytorch3d/csrc/ext.cpp:53-56); the four entry
 * points below take exactly the arguments of those ops, flattened to plain pointers and sizes
 * (no torch types), so any host language can bind them.  INTEGRATION.md shows the binding a
 * PyTorch3D maintainer would add; pytorch3d_b200/_C.py is that binding for this repo.
 *
 * Conventions
 *  - all pointers are DEVICE pointers on the current CUDA device unless the function name ends in
 *    `_host` (then they are host pointers and the call performs the H2D/D2H copies itself);
 *  - `stream` is a cudaStream_t passed as void* (NULL = default stream); calls are asynchronous and
 *    never synchronise the host (the reference ops do not either, rasterize_meshes.cu:383-384);
 *  - tensors are dense/contiguous in the layouts documented per argument (the reference ops call
 *    .contiguous() themselves, rasterize_meshes.cu:802-804; the Python host does it here);
 *  - outputs are fully written by the kernels, including the -1 padding of empty slots
 *    (the reference pre-fills with at::full, rasterize_meshes.cu:788-791);
 *  - return value: 0 = ok, otherwise an error code; b200r_last_error() gives the message.  Messages
 *    for argument errors match the reference's TORCH_CHECK / AT_ERROR texts.
 */
#ifndef B200_RASTER_H_
#define B200_RASTER_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200R_OK 0
#define B200R_ERR_INVALID_ARGUMENT 1
#define B200R_ERR_CUDA 2
#define B200R_ERR_WORKSPACE 3

/* kMaxPointsPerPixel, pytorch3d/csrc/rasterize_points/rasterization_utils.cuh:48 */
#define B200R_MAX_K 150

/* Library / build identification ("b200raster <version> sm_90a"). */
const char* b200r_version(void);

/* Message of the last failing call on the calling thread ("" if none). */
const char* b200r_last_error(void);

/* ------------------------------------------------------------------ meshes ------------------ */

/*
 * Scratch bytes needed by b200r_rasterize_meshes_forward for F packed faces, N meshes and an
 * H x W image.  pair_capacity = number of (tile, face) pairs the bin lists can hold; pass <= 0
 * for the default (min(F * tiles_per_image, 32*F + 64*N*tiles_per_image)).  If the real number of
 * pairs exceeds the capacity the affected tiles transparently fall back to testing every face of
 * their mesh, so results never depend on it (the reference drops faces and prints a warning
 * instead, rasterize_coarse.cu:186-201).
 */
size_t b200r_rasterize_meshes_workspace_bytes(int64_t F, int32_t N, int32_t H, int32_t W, int64_t pair_capacity);

/*
 * Replaces pytorch3d._C.rasterize_meshes
 *   (RasterizeMeshes, pytorch3d/csrc/rasterize_meshes/rasterize_meshes.h:513-562;
 *    call site pytorch3d/renderer/mesh/rasterize_meshes.py:297-310).
 *
 *  face_verts                 float32 (F,3,3)   packed faces in NDC (+X left, +Y up, z = depth)
 *  (mesh_to_face_first_idx / num_faces_per_mesh must describe ASCENDING, NON-OVERLAPPING ranges of the packed array --
 *   what Meshes produces: every face belongs to exactly one image.  The reference's kernels loop over each image's
 *   range and so also accept overlapping ranges; here images other than a face's owner would not see it.)
 *  mesh_to_face_first_idx     int64   (N,)      first packed face of each mesh (ascending)
 *  num_faces_per_mesh         int64   (N,)
 *  clipped_faces_neighbor_idx int64   (F,)      -1 or index of the other half of a clipped face
 *                                               (may be NULL = all -1)
 *  blur_radius, faces_per_pixel (K <= 150), perspective_correct, clip_barycentric_coords,
 *  cull_backfaces             as in the reference.
 *  bin_size, max_faces_per_bin  accepted for signature compatibility; they are performance hints
 *                             in the reference ("should not affect the output",
 *                             rasterize_meshes.py:73-80) and are ignored here: tiling is internal
 *                             and exact.
 * Outputs (all fully written):
 *  pix_to_face int64 (N,H,W,K); zbuf float32 (N,H,W,K); bary float32 (N,H,W,K,3);
 *  dists float32 (N,H,W,K); empty slots = -1.  For every pixel the K nearest faces are returned
 *  in increasing (z, face index) order.
 *  workspace: >= b200r_rasterize_meshes_workspace_bytes(...) bytes of device memory, 16B aligned.
 */
int b200r_rasterize_meshes_forward(const float* face_verts, int64_t F, const int64_t* mesh_to_face_first_idx,
                                   const int64_t* num_faces_per_mesh, const int64_t* clipped_faces_neighbor_idx,
                                   int32_t N, int32_t H, int32_t W, float blur_radius, int32_t faces_per_pixel,
                                   int32_t bin_size, int32_t max_faces_per_bin, int32_t perspective_correct,
                                   int32_t clip_barycentric_coords, int32_t cull_backfaces, int64_t* pix_to_face,
                                   float* zbuf, float* bary, float* dists, void* workspace, size_t workspace_bytes,
                                   int64_t pair_capacity, void* stream);

/*
 * Replaces pytorch3d._C.rasterize_meshes_backward
 *   (RasterizeMeshesBackward, rasterize_meshes.h:211-218; call site rasterize_meshes.py:334-342).
 *  grad_face_verts float32 (F,3,3) is zeroed and accumulated by the call.
 */
int b200r_rasterize_meshes_backward(const float* face_verts, int64_t F, const int64_t* pix_to_face,
                                    const float* grad_zbuf, const float* grad_bary, const float* grad_dists,
                                    int32_t N, int32_t H, int32_t W, int32_t K, int32_t perspective_correct,
                                    int32_t clip_barycentric_coords, float* grad_face_verts, void* stream);

/*
 * Fused gather entry points (SURVEY.md 8 f-4): the same rasterization, but taking the packed mesh itself.
 * Replace the `face_verts = verts_packed[faces_packed]` autograd node of the reference's wrapper
 * (pytorch3d/renderer/mesh/rasterize_meshes.py:144-148) together with the op it feeds: the setup pass gathers
 * the vertices of each face, and the backward adds the per-face gradient straight into the vertices.
 *
 *  verts  float32 (V,3) packed vertices;  faces int64 (F,3) packed vertex indices (0 <= index < V; a face with
 *         an out-of-range index is rasterized as NaN, i.e. never hit -- the reference raises a device assert)
 *  face_verts_out  float32 (F,3,3), written by the forward call: the gathered faces, to be passed to the
 *         backward call (what the reference's autograd saves)
 *  grad_verts      float32 (V,3), zeroed and accumulated by the backward call
 * All other arguments as in b200r_rasterize_meshes_forward / _backward (same workspace size).
 */
int b200r_rasterize_meshes_forward_indexed(const float* verts, int64_t V, const int64_t* faces, int64_t F,
                                           const int64_t* mesh_to_face_first_idx, const int64_t* num_faces_per_mesh,
                                           const int64_t* clipped_faces_neighbor_idx, int32_t N, int32_t H,
                                           int32_t W, float blur_radius, int32_t faces_per_pixel,
                                           int32_t perspective_correct, int32_t clip_barycentric_coords,
                                           int32_t cull_backfaces, int64_t* pix_to_face, float* zbuf, float* bary,
                                           float* dists, float* face_verts_out, void* workspace,
                                           size_t workspace_bytes, int64_t pair_capacity, void* stream);

int b200r_rasterize_meshes_backward_indexed(const float* face_verts, const int64_t* faces, int64_t F, int64_t V,
                                            const int64_t* pix_to_face, const float* grad_zbuf,
                                            const float* grad_bary, const float* grad_dists, int32_t N, int32_t H,
                                            int32_t W, int32_t K, int32_t perspective_correct,
                                            int32_t clip_barycentric_coords, float* grad_verts, void* stream);

/* ------------------------------------------------------------------ points ------------------ */

size_t b200r_rasterize_points_workspace_bytes(int64_t P, int32_t N, int32_t H, int32_t W, int64_t pair_capacity);

/*
 * Replaces pytorch3d._C.rasterize_points
 *   (RasterizePoints, pytorch3d/csrc/rasterize_points/rasterize_points.h:343-374;
 *    call site pytorch3d/renderer/points/rasterize_points.py:200-212).
 *  points float32 (P,3); cloud_to_packed_first_idx / num_points_per_cloud int64 (N,);
 *  radius float32 (P,) in NDC units; points_per_pixel K <= 150.
 * Outputs: idx int32 (N,H,W,K); zbuf float32 (N,H,W,K); dists float32 (N,H,W,K) (squared xy distance).
 */
int b200r_rasterize_points_forward(const float* points, int64_t P, const int64_t* cloud_to_packed_first_idx,
                                   const int64_t* num_points_per_cloud, const float* radius, int32_t N, int32_t H,
                                   int32_t W, int32_t points_per_pixel, int32_t bin_size,
                                   int32_t max_points_per_bin, int32_t* idx, float* zbuf, float* dists,
                                   void* workspace, size_t workspace_bytes, int64_t pair_capacity, void* stream);

/*
 * Replaces pytorch3d._C.rasterize_points_backward
 *   (RasterizePointsBackward, rasterize_points.h:281-285; call site rasterize_points.py:229-231).
 */
int b200r_rasterize_points_backward(const float* points, int64_t P, const int32_t* idxs, const float* grad_zbuf,
                                    const float* grad_dists, int32_t N, int32_t H, int32_t W, int32_t K,
                                    float* grad_points, void* stream);

/* ------------------------------------------------------------------ compositing ------------- */

/*
 * Replaces pytorch3d._C.accum_alphacomposite
 *   (alphaCompositeForward, pytorch3d/csrc/compositing/alpha_composite.h:59-82;
 *    call site pytorch3d/renderer/compositing.py:47-49).
 *  features float32, logical shape (C,P), addressed through element strides: feature (c, p) at
 *  features[c * feature_stride_c + p * feature_stride_p] (the renderer passes `features_packed().permute(1, 0)`, a (C,P)
 *  view of point-major memory; contiguous (C,P) is stride_c = P, stride_p = 1); alphas float32 and points_idx int64,
 *  logical shape (N,K,H,W), addressed through the four ELEMENT strides given (the renderer passes permuted views of
 *  (N,H,W,K) tensors); result float32 (N,C,H,W) contiguous, fully written.
 */
int b200r_alpha_composite_forward_strided(const float* features, int64_t C, int64_t P, int64_t feature_stride_c,
                                          int64_t feature_stride_p, const float* alphas, const int64_t* alpha_strides,
                                          const int64_t* points_idx, const int64_t* idx_strides, int32_t N, int32_t K,
                                          int32_t H, int32_t W, float* result, void* stream);

/*
 * Replaces pytorch3d._C.accum_alphacomposite_backward
 *   (alphaCompositeBackward, alpha_composite.h:84-116; call site compositing.py:58-60).
 *  grad_out (N,C,H,W) contiguous; grad_features (C,P), with the strides of features, is zeroed and accumulated;
 *  grad_alphas (N,K,H,W) contiguous, fully written.
 */
int b200r_alpha_composite_backward_strided(const float* grad_out, const float* features, int64_t C, int64_t P,
                                           int64_t feature_stride_c, int64_t feature_stride_p, const float* alphas,
                                           const int64_t* alpha_strides, const int64_t* points_idx,
                                           const int64_t* idx_strides, int32_t N, int32_t K, int32_t H, int32_t W,
                                           float* grad_features, float* grad_alphas, void* stream);

/*
 * Replace pytorch3d._C.accum_weightedsum / accum_weightedsum_backward
 *   (weightedSumForward / Backward, pytorch3d/csrc/compositing/weighted_sum.h:57-78, 80-110) and
 * pytorch3d._C.accum_weightedsumnorm / accum_weightedsumnorm_backward
 *   (weightedSumNormForward / Backward, compositing/norm_weighted_sum.h:57-79, 81-112):
 *   result[n,c,y,x] = sum_k alpha[n,k,y,x] * features[c, idx[n,k,y,x]]   (norm: / max(sum_k alpha, 1e-4)),
 * slots with idx < 0 skipped.  Arguments and layouts as b200r_alpha_composite_forward_strided / _backward_strided
 * without the two feature strides: features (and grad_features) are (C,P) contiguous.
 */
int b200r_weighted_sum_forward(const float* features, int64_t C, int64_t P, const float* alphas,
                               const int64_t* alpha_strides, const int64_t* points_idx, const int64_t* idx_strides,
                               int32_t N, int32_t K, int32_t H, int32_t W, float* result, void* stream);
int b200r_weighted_sum_backward(const float* grad_outputs, const float* features, int64_t C, int64_t P,
                                const float* alphas, const int64_t* alpha_strides, const int64_t* points_idx,
                                const int64_t* idx_strides, int32_t N, int32_t K, int32_t H, int32_t W,
                                float* grad_features, float* grad_alphas, void* stream);
int b200r_norm_weighted_sum_forward(const float* features, int64_t C, int64_t P, const float* alphas,
                                    const int64_t* alpha_strides, const int64_t* points_idx,
                                    const int64_t* idx_strides, int32_t N, int32_t K, int32_t H, int32_t W,
                                    float* result, void* stream);
int b200r_norm_weighted_sum_backward(const float* grad_outputs, const float* features, int64_t C, int64_t P,
                                     const float* alphas, const int64_t* alpha_strides, const int64_t* points_idx,
                                     const int64_t* idx_strides, int32_t N, int32_t K, int32_t H, int32_t W,
                                     float* grad_features, float* grad_alphas, void* stream);

/* ------------------------------------------------------------------ face attribute interpolation */

/*
 * Replaces pytorch3d._C.interp_face_attrs_forward
 *   (InterpFaceAttrsForward, pytorch3d/csrc/interp_face_attrs/interp_face_attrs.h:45-66;
 *    call site pytorch3d/ops/interp_face_attrs.py:66).
 *  pix_to_face int64 (P,); barycentric_coords float32 (P,3); face_attrs float32 (F,3,D); pix_attrs float32 (P,D),
 *  fully written (0 where pix_to_face < 0).
 */
int b200r_interp_face_attrs_forward(const int64_t* pix_to_face, const float* barycentric_coords,
                                    const float* face_attrs, int64_t P, int64_t F, int64_t D, float* pix_attrs,
                                    void* stream);

/*
 * Replaces pytorch3d._C.interp_face_attrs_backward
 *   (InterpFaceAttrsBackward, interp_face_attrs.h:88-118; call site interp_face_attrs.py:74).
 *  grad_barycentric_coords (P,3) fully written; grad_face_attrs (F,3,D) zeroed and accumulated.
 */
int b200r_interp_face_attrs_backward(const int64_t* pix_to_face, const float* barycentric_coords,
                                     const float* face_attrs, const float* grad_pix_attrs, int64_t P, int64_t F,
                                     int64_t D, float* grad_barycentric_coords, float* grad_face_attrs, void* stream);

/* ------------------------------------------------------------------ mesh blending ------------------------ */

/*
 * Replace pytorch3d._C.sigmoid_alpha_blend / sigmoid_alpha_blend_backward
 *   (SigmoidAlphaBlend / SigmoidAlphaBlendBackward, pytorch3d/csrc/blending/sigmoid_alpha_blend.h;
 *    call site pytorch3d/renderer/blending.py _SigmoidAlphaBlend).  Bit-identical to the reference's CUDA kernels.
 *  dists float32 (N,H,W,K); pix_to_face int64 (N,H,W,K) (a slot is empty when the index, read as a 32-bit int, is < 0);
 *  alphas float32 (N,H,W), fully written: 1 - prod over valid slots of (1 - sigmoid(-dist / sigma)).
 *  Backward: grad_alphas and alphas (the forward's output) float32 (N,H,W); grad_dists float32 (N,H,W,K), fully
 *  written (0 in empty slots).
 */
int b200r_sigmoid_alpha_blend_forward(const float* dists, const int64_t* pix_to_face, int32_t N, int32_t H, int32_t W,
                                      int32_t K, float sigma, float* alphas, void* stream);
int b200r_sigmoid_alpha_blend_backward(const float* grad_alphas, const float* alphas, const float* dists,
                                       const int64_t* pix_to_face, int32_t N, int32_t H, int32_t W, int32_t K,
                                       float sigma, float* grad_dists, void* stream);

/*
 * Fused softmax_rgb_blend (additional entry points, no counterpart in pytorch3d._C): the torch chain of
 * pytorch3d/renderer/blending.py softmax_rgb_blend in one kernel per direction, on the rasterizer's layout.
 *  colors float32 (N,H,W,K,3); pix_to_face int64 (N,H,W,K) (valid where >= 0); zbuf, dists float32 (N,H,W,K);
 *  K <= 150.  sigma, gamma as in BlendParams.
 *  background: device float32 (3,), or NULL and then background_value: HOST float[3].
 *  znear / zfar: device float32 (N,) per image, or NULL and then the scalar znear_value / zfar_value (a double, as a
 *  Python float: the range zfar - znear is formed in double precision, like the Python expression).
 *  out float32 (N,H,W,4) RGBA, fully written.
 * Backward: grad_out float32 (N,H,W,4); grad_colors (N,H,W,K,3), grad_dists and grad_zbuf (N,H,W,K) float32, fully
 * written.  The gradient through the per-pixel maximum of the inverse depth goes to the first slot attaining it.
 */
int b200r_softmax_rgb_blend_forward(const float* colors, const int64_t* pix_to_face, const float* zbuf,
                                    const float* dists, int32_t N, int32_t H, int32_t W, int32_t K, float sigma,
                                    float gamma, const float* background, const float* background_value,
                                    const float* znear, const float* zfar, double znear_value, double zfar_value,
                                    float* out, void* stream);
int b200r_softmax_rgb_blend_backward(const float* grad_out, const float* colors, const int64_t* pix_to_face,
                                     const float* zbuf, const float* dists, int32_t N, int32_t H, int32_t W, int32_t K,
                                     float sigma, float gamma, const float* background, const float* background_value,
                                     const float* znear, const float* zfar, double znear_value, double zfar_value,
                                     float* grad_colors, float* grad_dists, float* grad_zbuf, void* stream);

/*
 * Fused depth shading (additional entry points, no counterpart in pytorch3d._C): the torch chains of
 * pytorch3d/renderer/mesh/shader.py SoftDepthShader.forward and HardDepthShader.forward, one kernel per direction, on
 * the rasterizer's layout (DESIGN.md section 19).
 *  pix_to_face int64 (N,H,W,K) (valid where >= 0); zbuf, dists float32 (N,H,W,K); 1 <= K <= 150.
 *  zfar: device float32, one value, or NULL and then the number zfar_value.
 *  Soft: out float32 (N,H,W,1), fully written: sum_k w_k depth_k over the K slots and a last one of probability 1 at
 *  depth zfar, w_k the differences of the prefix sums of sigmoid(-dists / sigma) * [valid] clamped to 1.
 *  Backward: grad_out float32 (N,H,W,1); grad_zbuf and grad_dists float32 (N,H,W,K), fully written, no atomics.
 *  Hard: out float32 (N,H,W,1), fully written: zbuf of slot 0 where pix_to_face of slot 0 is valid, zfar elsewhere.
 *  Backward: grad_out float32 (N,H,W,1); grad_zbuf float32 (N,H,W,K), fully written (0 outside valid slots 0).
 */
int b200r_soft_depth_blend_forward(const int64_t* pix_to_face, const float* zbuf, const float* dists, int32_t N,
                                   int32_t H, int32_t W, int32_t K, float sigma, const float* zfar, float zfar_value,
                                   float* out, void* stream);
int b200r_soft_depth_blend_backward(const float* grad_out, const int64_t* pix_to_face, const float* zbuf,
                                    const float* dists, int32_t N, int32_t H, int32_t W, int32_t K, float sigma,
                                    const float* zfar, float zfar_value, float* grad_zbuf, float* grad_dists,
                                    void* stream);
int b200r_hard_depth_forward(const int64_t* pix_to_face, const float* zbuf, int32_t N, int32_t H, int32_t W, int32_t K,
                             const float* zfar, float zfar_value, float* out, void* stream);
int b200r_hard_depth_backward(const float* grad_out, const int64_t* pix_to_face, int32_t N, int32_t H, int32_t W,
                              int32_t K, float* grad_zbuf, void* stream);

/*
 * Fused splatter blending (additional entry points, no counterpart in pytorch3d._C): what
 * pytorch3d/renderer/splatter_blend.py SplatterBlender.forward computes after its projection step, in one kernel for
 * the forward and two for the backward (DESIGN.md section 11).
 *  colors float32 (N,H,W,K,3); pixel_coords_screen float32 (N,H,W,K,3) (x, y in pixels, z the depth);
 *  background_mask bool / uint8 (N,H,W,K) (nonzero: background slot); 1 <= K <= 150; sigma > 0 in pixels.
 *  background: device float32 (3,), or NULL and then background_value: HOST float[3].
 *  out float32 (N,H,W,4) RGBA, fully written.
 * Backward: grad_out float32 (N,H,W,4); workspace of b200r_splatter_blend_workspace_bytes(N, H, W) bytes, 16-byte
 * aligned (a 96-byte record per pixel); grad_colors and grad_pixel_coords_screen float32 (N,H,W,K,3), fully written
 * (0 in background slots and in the z channel).  No atomics: the results are deterministic.
 */
int b200r_splatter_blend_forward(const float* colors, const float* pixel_coords_screen, const uint8_t* background_mask,
                                 int32_t N, int32_t H, int32_t W, int32_t K, double sigma, const float* background,
                                 const float* background_value, float* out, void* stream);
size_t b200r_splatter_blend_workspace_bytes(int32_t N, int32_t H, int32_t W);
int b200r_splatter_blend_backward(const float* grad_out, const float* colors, const float* pixel_coords_screen,
                                  const uint8_t* background_mask, int32_t N, int32_t H, int32_t W, int32_t K,
                                  double sigma, const float* background, const float* background_value,
                                  void* workspace, size_t workspace_bytes, float* grad_colors,
                                  float* grad_pixel_coords_screen, void* stream);

/*
 * Fused Phong / flat shading (additional entry points, no counterpart in pytorch3d._C): what
 * pytorch3d/renderer/mesh/shading.py phong_shading, _phong_shading_with_pixels and flat_shading compute with the
 * PointLights, DirectionalLights and AmbientLights of renderer/lighting.py, one thread per slot (DESIGN.md section 12).
 *  pix_to_face int64 (N,H,W,K); barycentric_coords float32 (N,H,W,K,3) (phong; may be NULL when flat);
 *  face_positions, face_normals float32 (F,3,3) (phong: corners of each face) or (F,3) (flat: centroid and normal);
 *  face_normals may be NULL for ambient light; texels float32 (N,H,W,K,3);
 *  params float32 (N, B200R_SHADING_PARAMS), one row per image:
 *    [0:3] ambient (material ambient * light ambient), [3:6] light diffuse, [6:9] light specular,
 *    [9:12] material diffuse, [12:15] material specular, [15:18] light location (point) or direction (directional),
 *    [18:21] camera centre, [21] shininess;
 *  light: B200R_LIGHT_POINT / _DIRECTIONAL / _AMBIENT; flat: 0 phong, 1 flat.
 *  colors float32 (N,H,W,K,3), fully written; positions float32 (N,H,W,K,3) or NULL: the interpolated positions
 *  (bit-identical to b200r_interp_face_attrs_forward), 0 in background slots.
 * Backward: grad_colors float32 (N,H,W,K,3); grad_positions the same shape or NULL.  Every output may be NULL
 *  (not computed): grad_texels, grad_barycentric_coords (N,H,W,K,3) (phong), grad_face_positions, grad_face_normals
 *  (shapes of the face inputs; zero-filled here, then accumulated with atomics), grad_params (N, B200R_SHADING_PARAMS).
 *  grad_params needs a workspace of b200r_shading_workspace_bytes(N, H, W, K) bytes; it and every other output except
 *  the two face gradients are deterministic.  N <= 65535.
 */
#define B200R_SHADING_PARAMS 22
#define B200R_LIGHT_POINT 0
#define B200R_LIGHT_DIRECTIONAL 1
#define B200R_LIGHT_AMBIENT 2
int b200r_shading_forward(const int64_t* pix_to_face, const float* barycentric_coords, const float* face_positions,
                          const float* face_normals, int64_t F, const float* texels, const float* params, int32_t N,
                          int32_t H, int32_t W, int32_t K, int32_t flat, int32_t light, float* colors,
                          float* positions, void* stream);
size_t b200r_shading_workspace_bytes(int32_t N, int32_t H, int32_t W, int32_t K);
int b200r_shading_backward(const float* grad_colors, const float* grad_positions, const int64_t* pix_to_face,
                           const float* barycentric_coords, const float* face_positions, const float* face_normals,
                           int64_t F, const float* texels, const float* params, int32_t N, int32_t H, int32_t W,
                           int32_t K, int32_t flat, int32_t light, void* workspace, size_t workspace_bytes,
                           float* grad_texels, float* grad_barycentric_coords, float* grad_face_positions,
                           float* grad_face_normals, float* grad_params, void* stream);

/*
 * Fused Gouraud shading (additional entry points, no counterpart in pytorch3d._C): what
 * pytorch3d/renderer/mesh/shading.py gouraud_shading computes -- every vertex lit with its mesh's parameter row, the
 * shaded vertex colours then interpolated at the rasterized slots (DESIGN.md section 16).
 *  verts, normals, verts_colors float32 (V,3) packed; normals may be NULL for ambient light;
 *  mesh_first_vert, mesh_num_verts int64 (meshes,) device arrays: mesh m owns vertices [first[m], first[m] + num[m]);
 *  the ranges must cover every vertex once (the packed layout; the vertex outputs are written over the ranges only),
 *  and V > 0 needs meshes > 0;
 *  params float32 (meshes, B200R_SHADING_PARAMS), one row per mesh in the layout above; faces int64 (F,3) packed;
 *  pix_to_face int64 (P,) and barycentric_coords float32 (P,3) with P = N*H*W*K; light: B200R_LIGHT_*.
 *  verts_shaded float32 (V,3) and colors float32 (P,3), fully written; colors are bit-identical to
 *  b200r_interp_face_attrs_forward fed verts_shaded[faces].  meshes <= 65535.
 * Backward: grad_colors float32 (P,3); verts_shaded as returned by the forward.  Every output may be NULL: grad_verts,
 *  grad_normals, grad_verts_colors (V,3), grad_barycentric_coords (P,3), grad_params (meshes, B200R_SHADING_PARAMS).
 *  Any of the vertex-side outputs (all but grad_barycentric_coords) needs a workspace of
 *  b200r_gouraud_workspace_bytes(meshes, V) bytes.  grad_barycentric_coords is bit-identical to
 *  b200r_interp_face_attrs_backward's; the vertex-side gradients start from a sum accumulated with atomics.
 */
int b200r_gouraud_forward(const float* verts, const float* normals, const float* verts_colors, int64_t V,
                          const int64_t* mesh_first_vert, const int64_t* mesh_num_verts, int32_t meshes,
                          const float* params, const int64_t* faces, int64_t F, const int64_t* pix_to_face,
                          const float* barycentric_coords, int64_t P, int32_t light, float* verts_shaded,
                          float* colors, void* stream);
size_t b200r_gouraud_workspace_bytes(int32_t meshes, int64_t V);
int b200r_gouraud_backward(const float* grad_colors, const float* verts, const float* normals,
                           const float* verts_colors, int64_t V, const int64_t* mesh_first_vert,
                           const int64_t* mesh_num_verts, int32_t meshes, const float* params, const int64_t* faces,
                           int64_t F, const int64_t* pix_to_face, const float* barycentric_coords, int64_t P,
                           int32_t light, const float* verts_shaded, void* workspace, size_t workspace_bytes,
                           float* grad_verts, float* grad_normals, float* grad_verts_colors,
                           float* grad_barycentric_coords, float* grad_params, void* stream);

/*
 * Fused UV texture sampling (additional entry points, no counterpart in pytorch3d._C): what
 * pytorch3d/renderer/mesh/textures.py TexturesUV.sample_textures computes for a texture with one map per mesh -- the
 * slot's UV interpolated from its face's corner UVs ((0, 0) where pix_to_face < 0), mapped to grid coordinates with
 * torch.lerp and the y flip, then F.grid_sample of map n, the slot's image -- one thread per slot (DESIGN.md section 13).
 *  pix_to_face int64 (N,H,W,K); barycentric_coords float32 (N,H,W,K,3); face_uvs float32 (F,3,2);
 *  maps float32 (N,H_in,W_in,C), channel last, read in place (64-bit offsets); H_in, W_in, C >= 1;
 *  mode: B200R_SAMPLE_BILINEAR / _NEAREST; padding: B200R_PAD_ZEROS / _BORDER / _REFLECTION (torch's enum values).
 *  texels float32 (N,H,W,K,C), fully written.
 * Backward: grad_texels float32 (N,H,W,K,C).  Every output may be NULL (not computed): grad_maps (N,H_in,W_in,C) and
 *  grad_face_uvs (F,3,2) are zero-filled here, then accumulated with atomics; grad_barycentric_coords (N,H,W,K,3) is
 *  written once per slot (0 in background slots and for "nearest") and is deterministic.
 */
#define B200R_SAMPLE_BILINEAR 0
#define B200R_SAMPLE_NEAREST 1
#define B200R_PAD_ZEROS 0
#define B200R_PAD_BORDER 1
#define B200R_PAD_REFLECTION 2
int b200r_texture_uv_forward(const int64_t* pix_to_face, const float* barycentric_coords, const float* face_uvs,
                             int64_t F, const float* maps, int32_t N, int32_t H, int32_t W, int32_t K, int32_t H_in,
                             int32_t W_in, int32_t C, int32_t mode, int32_t padding, int32_t align_corners,
                             float* texels, void* stream);
int b200r_texture_uv_backward(const float* grad_texels, const int64_t* pix_to_face, const float* barycentric_coords,
                              const float* face_uvs, int64_t F, const float* maps, int32_t N, int32_t H, int32_t W,
                              int32_t K, int32_t H_in, int32_t W_in, int32_t C, int32_t mode, int32_t padding,
                              int32_t align_corners, float* grad_maps, float* grad_barycentric_coords,
                              float* grad_face_uvs, void* stream);

/*
 * Fused texture atlas sampling (additional entry points, no counterpart in pytorch3d._C): what
 * pytorch3d/renderer/mesh/textures.py TexturesAtlas.sample_textures computes -- the slot's cell of its face's R x R
 * patch from (b0, b1) with the reference's truncation, clamp and diagonal flip, read with torch's negative-index wrap
 * and multiplied by float(pix_to_face >= 0) -- one thread per slot (DESIGN.md section 15).
 *  pix_to_face int64 (N,H,W,K); barycentric_coords float32 (N,H,W,K,3); atlas float32 (F,R,R,C), contiguous, read in
 *  place (64-bit offsets); R, C >= 1.  texels float32 (N,H,W,K,C), fully written.  A slot whose cell the reference
 *  cannot index (it raises) gets texel 0.
 * Backward: grad_texels float32 (N,H,W,K,C) -> grad_atlas float32 (F,R,R,C), zero-filled here, then every cell that
 *  receives a contribution is written once: the sum of its slots' grad_texels * float(pix_to_face >= 0) in ascending
 *  slot order from +0.  Deterministic, no atomics (a stable radix sort of (cell, slot) pairs).  N*H*W*K < 2^31.
 *  workspace: b200r_texture_atlas_workspace_bytes(N, H, W, K, F, R) bytes, a function of the shapes only (0 when there
 *  is nothing to sort or no device to size the sort for).
 */
size_t b200r_texture_atlas_workspace_bytes(int32_t N, int32_t H, int32_t W, int32_t K, int64_t F, int32_t R);
int b200r_texture_atlas_forward(const int64_t* pix_to_face, const float* barycentric_coords, const float* atlas,
                                int64_t F, int32_t R, int32_t C, int32_t N, int32_t H, int32_t W, int32_t K,
                                float* texels, void* stream);
int b200r_texture_atlas_backward(const float* grad_texels, const int64_t* pix_to_face,
                                 const float* barycentric_coords, int64_t F, int32_t R, int32_t C, int32_t N,
                                 int32_t H, int32_t W, int32_t K, void* workspace, size_t workspace_bytes,
                                 float* grad_atlas, void* stream);

/*
 * Mesh normals (DESIGN.md section 17).  verts float32 (V,3) and faces int64 (F,3), contiguous, read in place (64-bit
 * offsets); V < 2^31 - 1 and 3F < 2^31, larger sizes return B200R_ERR_INVALID_ARGUMENT.  A face index outside [0, V)
 * (the reference does not check them) gives NaN for that face and belongs to no vertex.  All entry points are
 * asynchronous, use no float atomics and are deterministic.
 *
 * The vertex -> corner table: int32, V + 1 offsets followed by the 3F corner ids j * F + f sorted by their vertex
 * faces[f, j] (stable, so in (j, f) order within a vertex).  Vertex v's corners are ids[offsets[v] .. offsets[v+1]).
 *
 * face_areas_normals_forward / _backward: pytorch3d._C's ops of these names (face_areas_normals.h), for float32.  The
 *  forward writes areas (F,) and normals (F,3), bit-identical to the reference's CUDA kernel built for sm_90a.  The
 *  backward takes grad_areas (F,) and grad_normals (F,3) float32, contiguous, and writes grad_verts (V,3): the
 *  reference's per-corner terms summed per vertex in the table's order (the table is built in the call).
 * verts_normals_forward: what pytorch3d.structures.Meshes._compute_vertex_normals computes, bit-identical to it on the
 *  CPU: normals (V,3) = s / max(|s|, 1e-6), s the sum of (v2 - v1) x (v0 - v1) over the vertex's corners.  Also writes
 *  the table (V + 1 + 3F ints) and s (V,3) float32, which the backward reads.
 * verts_normals_backward: grad_normals float32 (V,3), contiguous -> grad_verts (V,3), autograd's gradient of that chain.
 * workspace: b200r_normals_workspace_bytes(V, F) bytes for any of the three entry points that take one, a function of
 *  the shapes only; it allocates and launches nothing (0 when there is no device to size the sort for).
 */
size_t b200r_normals_workspace_bytes(int64_t V, int64_t F);
int b200r_face_areas_normals_forward(const float* verts, int64_t V, const int64_t* faces, int64_t F, float* areas,
                                     float* normals, void* stream);
int b200r_face_areas_normals_backward(const float* grad_areas, const float* grad_normals, const float* verts,
                                      int64_t V, const int64_t* faces, int64_t F, void* workspace,
                                      size_t workspace_bytes, float* grad_verts, void* stream);
int b200r_verts_normals_forward(const float* verts, int64_t V, const int64_t* faces, int64_t F, void* workspace,
                                size_t workspace_bytes, int32_t* table, float* sums, float* normals, void* stream);
int b200r_verts_normals_backward(const float* grad_normals, const float* verts, int64_t V, const int64_t* faces,
                                 int64_t F, const int32_t* table, const float* sums, void* workspace,
                                 size_t workspace_bytes, float* grad_verts, void* stream);

/*
 * Mesh surface sampling (DESIGN.md section 20): what pytorch3d.ops.sample_points_from_meshes computes, with draws from
 * a counter-based generator.  verts float32 (V,3), faces int64 (F,3) packed, mesh_first_face / mesh_num_faces int64
 * (N,), all contiguous device arrays read in place (64-bit offsets).  N >= 1, S >= 1, V < 2^31 - 1, N * S <= 2^40; the
 * backward also needs 3 N S < 2^31.  All entry points are asynchronous, use no float atomics and are deterministic.
 *
 * forward: S samples per mesh, each face drawn with probability proportional to its face_areas_normals area (a face of
 *  zero area never), barycentrics w0 = 1 - sqrt(u), w1 = sqrt(u) (1 - v), w2 = sqrt(u) v.  Writes samples (N,S,3),
 *  normals (N,S,3) if not NULL ((v1 - v0) x (v2 - v1) normalised), face_idx (N,S) int64 (the packed face, -1 for a
 *  mesh without faces, whose samples, normals and bary are zeros) and bary (N,S,3).  The draws come from one
 *  Philox4x32-10 evaluation per sample, keyed by seed (2 int64 on the device, their low 32 bits) with the sample's
 *  index n * S + s as counter; or, when draw_face, draw_u and draw_v ((N,S) int64 packed faces, float32 u and v) are
 *  given, from those (seed may then be NULL).  *status (device int32) is set to the B200R_SAMPLE_* bits below.
 * backward: grad_samples (N,S,3), grad_normals (N,S,3) or NULL, contiguous float32, with the forward's face_idx and
 *  bary -> grad_verts (V,3).
 * workspace: b200r_sample_points_workspace_bytes(V, F, N, S, pass) bytes, pass 0 for the forward and 1 for the
 *  backward, a function of the shapes only (0 for bad sizes, or when there is no device to size the sort for).
 */
#define B200R_SAMPLE_HAS_VALID 1  /* some mesh has a face */
#define B200R_SAMPLE_NONFINITE 2  /* some vertex coordinate is NaN or infinite */
#define B200R_SAMPLE_BAD_TOTAL 4  /* a mesh with faces has a total area that is not positive and finite */
#define B200R_SAMPLE_HAS_EMPTY 8  /* some mesh has no face */
size_t b200r_sample_points_workspace_bytes(int64_t V, int64_t F, int64_t N, int64_t S, int32_t pass);
int b200r_sample_points_forward(const float* verts, int64_t V, const int64_t* faces, int64_t F,
                                const int64_t* mesh_first_face, const int64_t* mesh_num_faces, int64_t N, int64_t S,
                                const int64_t* seed, const int64_t* draw_face, const float* draw_u,
                                const float* draw_v, void* workspace, size_t workspace_bytes, float* samples,
                                float* normals, int64_t* face_idx, float* bary, int32_t* status, void* stream);
int b200r_sample_points_backward(const float* grad_samples, const float* grad_normals, const float* verts, int64_t V,
                                 const int64_t* faces, int64_t F, int64_t N, int64_t S, const int64_t* face_idx,
                                 const float* bary, void* workspace, size_t workspace_bytes, float* grad_verts,
                                 void* stream);

/*
 * Chamfer distance (DESIGN.md section 21): what pytorch3d/loss/chamfer.py's chamfer_distance computes for D = 3, with
 * the nearest neighbours of the reference's KNearestNeighborKernelV3<float, 3, 1> bit for bit.  x (N,P1,3) and y
 * (N,P2,3) float32, x_lengths / y_lengths int64 (N,) or NULL (all P), x_normals (N,P1,3) and y_normals (N,P2,3) float32
 * or both NULL, weights float32 (N,) or NULL, all contiguous device arrays.  N, P1, P2 >= 1 and 2 (N P1 + N P2) < 2^31.
 * All entry points are asynchronous, use no float atomics and are deterministic.
 *
 * forward: dist_x / idx_x (N,P1) and, unless single_directional, dist_y / idx_y (N,P2): each point's nearest-neighbour
 *  distance and index in the other cloud (0 and 0 for padding and for an empty other cloud).  cloud (4N + 1 floats)
 *  and argmax (2N int32) keep the per-cloud state the backward reads.  Outputs: with point_reduction NONE, the distance
 *  terms out_x (N,P1) and out_y (N,P2) and the normal terms out_nx / out_ny; otherwise the loss in out_x and the normal
 *  loss in out_nx ((N,) for batch_reduction NONE, else one float).  *status (device int32) gets the B200R_CHAMFER_*
 *  bits of the data-dependent checks below.
 * backward: grad_x / grad_y (and grad_nx / grad_ny) are the upstream gradients of the outputs in the same layout
 *  (grad_y and grad_ny only for point_reduction NONE) -> grad_points (N P1 + N P2, 3): x's rows, then y's; and
 *  grad_normals likewise.  Either may be NULL.
 * workspace: b200r_chamfer_workspace_bytes(N, P1, P2, pass) bytes, pass 0 for the forward and 1 for the backward.
 */
#define B200R_CHAMFER_POINT_NONE 0
#define B200R_CHAMFER_POINT_SUM 1
#define B200R_CHAMFER_POINT_MEAN 2
#define B200R_CHAMFER_POINT_MAX 3
#define B200R_CHAMFER_BATCH_NONE 0
#define B200R_CHAMFER_BATCH_SUM 1
#define B200R_CHAMFER_BATCH_MEAN 2
#define B200R_CHAMFER_X_LENGTH 1      /* some x_lengths[n] > P1 */
#define B200R_CHAMFER_Y_LENGTH 2      /* some y_lengths[n] > P2 */
#define B200R_CHAMFER_W_NEGATIVE 4    /* some weight is not >= 0 */
#define B200R_CHAMFER_W_ZERO_SUM 8    /* the weights sum to 0 */
size_t b200r_chamfer_workspace_bytes(int64_t N, int64_t P1, int64_t P2, int32_t pass);
int b200r_chamfer_forward(const float* x, const float* y, int64_t N, int64_t P1, int64_t P2, const int64_t* x_lengths,
                          const int64_t* y_lengths, const float* x_normals, const float* y_normals,
                          const float* weights, int32_t norm, int32_t point_reduction, int32_t batch_reduction,
                          int32_t single_directional, int32_t abs_cosine, void* workspace, size_t workspace_bytes,
                          float* dist_x, int32_t* idx_x, float* dist_y, int32_t* idx_y, float* cloud, int32_t* argmax,
                          float* out_x, float* out_y, float* out_nx, float* out_ny, int32_t* status, void* stream);
int b200r_chamfer_backward(const float* x, const float* y, int64_t N, int64_t P1, int64_t P2,
                           const int64_t* x_lengths, const int64_t* y_lengths, const float* x_normals,
                           const float* y_normals, const float* weights, int32_t norm, int32_t point_reduction,
                           int32_t batch_reduction, int32_t single_directional, int32_t abs_cosine,
                           const int32_t* idx_x, const int32_t* idx_y, const float* cloud, const int32_t* argmax,
                           const float* grad_x, const float* grad_y, const float* grad_nx, const float* grad_ny,
                           void* workspace, size_t workspace_bytes, float* grad_points, float* grad_normals,
                           void* stream);

/*
 * Mesh regularisers (DESIGN.md section 18): what pytorch3d/loss/mesh_edge_loss.py, mesh_laplacian_smoothing.py and
 * mesh_normal_consistency.py compute, as a float32 scalar `loss` (a device pointer), and its gradient to the verts.
 *  verts float32 (V,3) and faces int64 (F,3), contiguous, read in place (64-bit offsets); V < 2^31 - 1 and 6F < 2^31,
 *  larger sizes return B200R_ERR_INVALID_ARGUMENT.  mesh_first_vert, mesh_num_verts int64 (N,) device arrays, as
 *  b200r_gouraud_* takes them: mesh m owns vertices [first[m], first[m] + num[m]), the ranges ascending and covering
 *  every vertex; N >= 1 (the loss is divided by N, empty meshes included).  A face index outside [0, V) belongs to no
 *  edge and no vertex.  All entry points are asynchronous, use no float atomics and are deterministic.
 *  Edges are the distinct (min, max) vertex pairs of the face-edges in ascending order, as Meshes.edges_packed();
 *  self-loops included.
 * edge loss: sum over edges of (|v0 - v1| - target_length)^2 / (edges of the mesh), over N.
 * Laplacian smoothing: sum over vertices of |y_v| / (vertices of the mesh), over N, with y = L v for method
 *  B200R_LAPLACIAN_UNIFORM, the cotangent rows of cot_laplacian() for _COT and _COTCURV; L and its weights are
 *  constants of the backward.  Another method returns B200R_ERR_INVALID_ARGUMENT.
 * normal consistency: over every pair of face-edges on one edge, 1 - cos(n_a, -n_b), n = sum_k (v1 - v0) x (f_k - v0),
 *  weighted by 1 / (pairs of the mesh), over N.  With no pair at all the loss is 0 and its gradient 0.
 * workspace: b200r_regularizers_workspace_bytes(V, F, N) bytes, a function of the shapes only (0 when there is no
 *  device to size the sorts for).  The forward leaves its tables there; the backward takes the same buffer, as the
 *  forward of the same loss (and method) on the same faces left it, and the same arguments, and does not sort again.
 *  grad_loss is a float32 device scalar; grad_verts (V,3) is fully written.
 * mesh_edge_table: the edge table alone, for tests: edges int64 (3F,2) (the first E rows written), face_to_edge int64
 *  (F,3) (faces_packed_to_edges_packed; -1 for a face-edge with a vertex out of range), num_edges_per_mesh int64 (N,)
 *  and E int64 (1,), all device arrays.
 */
#define B200R_LAPLACIAN_UNIFORM 0
#define B200R_LAPLACIAN_COT 1
#define B200R_LAPLACIAN_COTCURV 2
size_t b200r_regularizers_workspace_bytes(int64_t V, int64_t F, int32_t N);
int b200r_mesh_edge_table(const int64_t* faces, int64_t V, int64_t F, const int64_t* mesh_first_vert,
                          const int64_t* mesh_num_verts, int32_t N, void* workspace, size_t workspace_bytes,
                          int64_t* edges, int64_t* face_to_edge, int64_t* num_edges_per_mesh, int64_t* num_edges,
                          void* stream);
int b200r_mesh_edge_loss_forward(const float* verts, int64_t V, const int64_t* faces, int64_t F,
                                 const int64_t* mesh_first_vert, const int64_t* mesh_num_verts, int32_t N,
                                 float target_length, void* workspace, size_t workspace_bytes, float* loss,
                                 void* stream);
int b200r_mesh_edge_loss_backward(const float* grad_loss, const float* verts, int64_t V, const int64_t* faces,
                                  int64_t F, const int64_t* mesh_first_vert, const int64_t* mesh_num_verts, int32_t N,
                                  float target_length, void* workspace, size_t workspace_bytes, float* grad_verts,
                                  void* stream);
int b200r_mesh_laplacian_smoothing_forward(const float* verts, int64_t V, const int64_t* faces, int64_t F,
                                           const int64_t* mesh_first_vert, const int64_t* mesh_num_verts, int32_t N,
                                           int32_t method, void* workspace, size_t workspace_bytes, float* loss,
                                           void* stream);
int b200r_mesh_laplacian_smoothing_backward(const float* grad_loss, const float* verts, int64_t V,
                                            const int64_t* faces, int64_t F, const int64_t* mesh_first_vert,
                                            const int64_t* mesh_num_verts, int32_t N, int32_t method, void* workspace,
                                            size_t workspace_bytes, float* grad_verts, void* stream);
int b200r_mesh_normal_consistency_forward(const float* verts, int64_t V, const int64_t* faces, int64_t F,
                                          const int64_t* mesh_first_vert, const int64_t* mesh_num_verts, int32_t N,
                                          void* workspace, size_t workspace_bytes, float* loss, void* stream);
int b200r_mesh_normal_consistency_backward(const float* grad_loss, const float* verts, int64_t V,
                                           const int64_t* faces, int64_t F, const int64_t* mesh_first_vert,
                                           const int64_t* mesh_num_verts, int32_t N, void* workspace,
                                           size_t workspace_bytes, float* grad_verts, void* stream);

/*
 * Fused frustum culling and z-clipping (additional entry points, no counterpart in pytorch3d._C): what
 * pytorch3d/renderer/mesh/clip.py clip_faces and convert_clipped_rasterization_to_original_faces compute, with the
 * reference's output layout (DESIGN.md section 14).  All entry points are asynchronous.
 *  Frustum: planes[6] = left, right, top, bottom, znear, zfar (host array, float32); bit i of cull_mask says plane i is
 *  used (0 when the frustum does not cull).  has_z_clip / z_clip: the clipping plane (compared and subtracted as
 *  float32, divided by as a multiply by (float)(1.0 / z_clip), as torch's CUDA kernels do).
 *  Count: face_verts float32 (F,3,3), or (face_verts NULL) verts float32 (V,3) with faces int64 (F,3) read in place.
 *  workspace: b200r_clip_faces_workspace_words(F) int64 words; words 0..3 become the record {F_clipped, n_case3,
 *  n_case4, number of faces culled or clipped}, which the caller reads to size the outputs of the fill.
 *  Fill: the same face_verts and frustum as the count, and its workspace.  Outputs face_verts_clipped (F_clipped,3,3),
 *  first_clipped / num_clipped (N,), clipped_to_unclipped (F_clipped,); when n_case3 + n_case4 > 0 also
 *  barycentric_conversion (n_case3 + 2 n_case4,3,3), clipped_to_conversion and neighbor_idx (F_clipped,).
 *  Backward: grad_face_verts (F,3,3) written once per face from grad_face_verts_clipped and grad_conversion (each may be
 *  NULL: no gradient); deterministic.
 *  Convert: pix_to_face int64 and barycentric_coords float32 of S slots; barycentric_coords_unclipped may be NULL (then
 *  only pix_to_face is mapped).  Convert backward: grad_conversion (T,3,3) is zero-filled here and accumulated with
 *  atomics; grad_barycentric_coords is written once per slot; either may be NULL.
 */
int64_t b200r_clip_faces_workspace_words(int64_t F);
int b200r_clip_faces_count(const float* face_verts, const float* verts, const int64_t* faces, int64_t F,
                           const float* planes, int32_t cull_mask, int32_t has_z_clip, double z_clip,
                           int64_t* workspace, void* stream);
int b200r_clip_faces_fill(const float* face_verts, int64_t F, const int64_t* mesh_to_face_first_idx, int32_t N,
                          const float* planes, int32_t cull_mask, int32_t has_z_clip, double z_clip,
                          int32_t perspective_correct, const int64_t* workspace, int64_t F_clipped, int64_t n_case3,
                          int64_t n_case4, float* face_verts_clipped, int64_t* first_clipped, int64_t* num_clipped,
                          int64_t* clipped_to_unclipped, float* barycentric_conversion,
                          int64_t* clipped_to_conversion, int64_t* neighbor_idx, void* stream);
int b200r_clip_faces_backward(const float* face_verts, int64_t F, const float* planes, int32_t cull_mask,
                              int32_t has_z_clip, double z_clip, int32_t perspective_correct,
                              const int64_t* workspace, int64_t n_case3, int64_t n_case4,
                              const float* grad_face_verts_clipped, const float* grad_conversion,
                              float* grad_face_verts, void* stream);
int b200r_clip_convert_forward(const int64_t* pix_to_face, const float* barycentric_coords, int64_t S,
                               const int64_t* clipped_to_unclipped, const float* barycentric_conversion,
                               const int64_t* clipped_to_conversion, int64_t* pix_to_face_unclipped,
                               float* barycentric_coords_unclipped, void* stream);
int b200r_clip_convert_backward(const float* grad_barycentric_coords_unclipped, const int64_t* pix_to_face,
                                const float* barycentric_coords, int64_t S, const float* barycentric_conversion,
                                const int64_t* clipped_to_conversion, int64_t T, float* grad_barycentric_coords,
                                float* grad_conversion, void* stream);

/* ------------------------------------------------------------------ frame exchange between GPUs ---------- */

/*
 * The path's only collective (BASELINE.json north_star: "NCCL over NVLink only to gather rendered frames"; the
 * reference has no counterpart, tests/test_render_multigpu.py:120-185 only moves modules between devices).
 * Fragments are exchanged in a packed, lossless form -- 1 byte per pixel (number of valid slots) + 24 bytes per
 * VALID slot -- that one kernel writes straight into the memory of every peer over NVLink.
 *
 * Peer memory: b200r_peer_alloc cudaMallocs `bytes` on the current device and returns a 64-byte CUDA IPC handle
 * that another process of the same node turns into a device pointer with b200r_peer_open (peer access is enabled
 * on first use).  b200r_peer_close / b200r_peer_free undo them.
 */
int b200r_peer_alloc(size_t bytes, void** ptr, unsigned char* handle64);
int b200r_peer_open(const unsigned char* handle64, void** ptr);
int b200r_peer_close(void* ptr);
int b200r_peer_free(void* ptr);

/* Bytes of one packed-stream region sized for `n_images` frames of H x W x K slots (worst case: every slot valid). */
size_t b200r_packed_frames_bytes(int64_t n_images, int32_t H, int32_t W, int32_t K);

/*
 * Pack the Fragments of `n_images` local frames (the four outputs of b200r_rasterize_meshes_forward; valid slots
 * first in every pixel, as the rasterizer writes them) and store the stream into each of the `n_dst` regions
 * (HOST array of device pointers: local memory or b200r_peer_open'ed peer memory; each region laid out for
 * `n_images_layout` >= n_images frames).  `cursor`: one device int32 of scratch.  K <= 32, n_dst <= 16.
 * Completion of the kernel on `stream` + any cross-rank synchronisation (e.g. an NCCL barrier enqueued behind it)
 * makes the stream readable on the destination.
 */
int b200r_fragments_pack_push(const int64_t* pix_to_face, const float* zbuf, const float* bary, const float* dists,
                              int32_t n_images, int32_t H, int32_t W, int32_t K, int64_t n_images_layout,
                              void* const* dst_regions, int32_t n_dst, int32_t* cursor, void* stream);

/*
 * Expand a packed stream (device pointer `region`, written by b200r_fragments_pack_push with the same H, W, K and
 * n_images_layout) into dense full-batch buffers: frame j of the stream lands at batch position image_index[j]
 * (device int32 (n_images,)), its face ids shifted by face_shift[j] (device int64 (n_images,): first global packed face
 * of the mesh minus its first face in the sender's local packing); empty slots are written as -1.
 */
int b200r_fragments_unpack(const void* region, int32_t n_images, int32_t H, int32_t W, int32_t K,
                           int64_t n_images_layout, const int32_t* image_index, const int64_t* face_shift,
                           int64_t* pix_to_face, float* zbuf, float* bary, float* dists, void* stream);

/*
 * Exchange context: one per process, holding the arenas of all ranks (own memory + b200r_peer_open'ed peers; each
 * arena = 2 halves x `world` regions of b200r_packed_frames_bytes(n_images_layout, H, W, K) bytes), the batch geometry
 * (HOST arrays: images per rank; for every image of every rank, in rank order, its position in the full batch and its
 * face-id shift) and the events that order one step:
 *   b200r_exchange_push    on compute_stream: pack this rank's frames, push them into every arena; side_stream then
 *                          waits for the pack.  (`consumer_stream`: the stream that reads the results.)
 *   <cross-rank barrier>   the caller's, enqueued on side_stream: e.g. a 4-byte NCCL all-reduce
 *   b200r_exchange_expand  on side_stream: expand all ranks' streams into the dense full-batch buffers
 *   b200r_exchange_wait    make a stream wait for that expansion
 * Arena halves and result buffers alternate with the step's parity; a half is rewritten only behind the NEXT step's
 * barrier, which every rank enqueues behind its own expansion of this step.
 */
int b200r_exchange_create(int32_t world, int32_t rank, int32_t H, int32_t W, int32_t K, int64_t n_images_layout,
                          const int32_t* n_images_per_rank, const int32_t* image_index, const int64_t* face_shift,
                          void* const* arenas, void** handle);
int b200r_exchange_destroy(void* handle);
int b200r_exchange_push(void* handle, const int64_t* pix_to_face, const float* zbuf, const float* bary,
                        const float* dists, void* compute_stream, void* side_stream, void* consumer_stream);
int b200r_exchange_expand(void* handle, int64_t* pix_to_face, float* zbuf, float* bary, float* dists,
                          void* side_stream, int32_t* parity_out);
int b200r_exchange_wait(void* handle, int32_t parity, void* stream);

/* ------------------------------------------------------------------ host-buffer entry points - */

/*
 * Same operators with HOST buffers: the call stages inputs to the device (pinned staging is the
 * caller's choice), runs the kernels and copies the results back, synchronising before returning.
 * This is what a non-PyTorch host (cgo / JNI / ctypes) would bind, and what bench.py times as the
 * end-to-end number.
 */
int b200r_rasterize_meshes_forward_host(const float* face_verts, int64_t F, const int64_t* mesh_to_face_first_idx,
                                        const int64_t* num_faces_per_mesh,
                                        const int64_t* clipped_faces_neighbor_idx, int32_t N, int32_t H, int32_t W,
                                        float blur_radius, int32_t faces_per_pixel, int32_t perspective_correct,
                                        int32_t clip_barycentric_coords, int32_t cull_backfaces,
                                        int64_t* pix_to_face, float* zbuf, float* bary, float* dists);

int b200r_rasterize_meshes_backward_host(const float* face_verts, int64_t F, const int64_t* pix_to_face,
                                         const float* grad_zbuf, const float* grad_bary, const float* grad_dists,
                                         int32_t N, int32_t H, int32_t W, int32_t K, int32_t perspective_correct,
                                         int32_t clip_barycentric_coords, float* grad_face_verts);

int b200r_rasterize_points_forward_host(const float* points, int64_t P, const int64_t* cloud_to_packed_first_idx,
                                        const int64_t* num_points_per_cloud, const float* radius, int32_t N,
                                        int32_t H, int32_t W, int32_t points_per_pixel, int32_t* idx, float* zbuf,
                                        float* dists);

int b200r_rasterize_points_backward_host(const float* points, int64_t P, const int32_t* idxs,
                                         const float* grad_zbuf, const float* grad_dists, int32_t N, int32_t H,
                                         int32_t W, int32_t K, float* grad_points);

/* Number of kernels this library has launched in this process (for bench.py's gpu_launches). */
int64_t b200r_kernel_launch_count(void);

/*
 * Phase timing for bench.py's roofline line.  When enabled, the forward / backward entry points record
 * CUDA events on the caller's stream around their phases; b200r_last_phase_ms synchronises on those
 * events and returns the durations of the most recent call on this thread:
 *   out[0] = binning (setup+count, scan, fill, sort)   out[1] = fine kernel   out[2] = backward kernel
 * (entries of phases that did not run are 0).  Disabled by default; adds no work when disabled.
 */
void b200r_set_profiling(int32_t enabled);
int b200r_last_phase_ms(float out[3]);

/*
 * Fused point rendering (additional entry points, no counterpart in pytorch3d._C): weights = 1 - dists / radius2 and
 * alpha compositing of the point features in one kernel per direction -- what PointsRenderer.forward does between the
 * rasterizer and the image (pytorch3d/renderer/points/renderer.py:63-73) -- reading the rasterizer's outputs as they
 * are: idx int32 (N,H,W,K), dists float32 (N,H,W,K); images float32 (N,C,H,W); feature (c, p) at
 * features[c * feature_stride_c + p * feature_stride_p] (the renderer's `features_packed().permute(1, 0)` is a view of
 * point-major memory: strides (1, C); grad_features uses the same strides).
 * Forward values are bit-identical to the unfused chain; the backward zero-fills grad_features (C,P), accumulates it
 * with atomics and writes grad_dists (N,H,W,K) = d loss / d dists.
 */
int b200r_points_alpha_render_forward(const float* features, int64_t C, int64_t P, int64_t feature_stride_c,
                                      int64_t feature_stride_p, const int32_t* idx, const float* dists,
                                      float radius2, int32_t N, int32_t K, int32_t H, int32_t W, float* images,
                                      void* stream);
int b200r_points_alpha_render_backward(const float* grad_images, const float* features, int64_t C, int64_t P,
                                       int64_t feature_stride_c, int64_t feature_stride_p, const int32_t* idx,
                                       const float* dists, float radius2, int32_t N, int32_t K, int32_t H, int32_t W,
                                       float* grad_features, float* grad_dists, void* stream);

/*
 * Test hooks of the reference's coarse stage (pytorch3d._C._rasterize_meshes_coarse / _rasterize_points_coarse,
 * pytorch3d/csrc/ext.cpp:69-73; RasterizeMeshesCoarse rasterize_meshes.h:292-318, RasterizePointsCoarse
 * rasterize_points.h:140-166): the dense table bin_faces / bin_points int32 (N, BH, BW, M), BH = 1 + (H-1)/bin_size,
 * -1 padded, elements of a bin in arbitrary order (sort for a canonical form).  bin_counts int32 (N, BH, BW) scratch;
 * *overflow (device int32) is set to 1 if a bin received more than M elements (the reference prints a warning,
 * rasterize_coarse.cu:186-201).  Not used by the rasterizer itself, whose tile lists are compact and exact.
 */
int b200r_rasterize_meshes_coarse(const float* face_verts, int64_t F, const int64_t* mesh_to_face_first_idx,
                                  const int64_t* num_faces_per_mesh, int32_t N, int32_t H, int32_t W,
                                  float blur_radius, int32_t bin_size, int32_t max_faces_per_bin, int32_t* bin_faces,
                                  int32_t* bin_counts, int32_t* overflow, void* stream);
int b200r_rasterize_points_coarse(const float* points, int64_t P, const int64_t* cloud_to_packed_first_idx,
                                  const int64_t* num_points_per_cloud, const float* radius, int32_t N, int32_t H,
                                  int32_t W, int32_t bin_size, int32_t max_points_per_bin, int32_t* bin_points,
                                  int32_t* bin_counts, int32_t* overflow, void* stream);

/*
 * Farthest point sampling and ball query (DESIGN.md section 22): pytorch3d.ops.sample_farthest_points and
 * pytorch3d.ops.ball_query for D = 3, bit for bit what the reference's CUDA kernels compute.  Points are contiguous
 * float32 (N, P, 3) device arrays, lengths int64 (N,) or NULL (all P), clamped to [0, P].  All entry points are
 * asynchronous, use no float atomics and are deterministic.
 *
 * sample_farthest_points: idx (N, max_K) int64.  Row n is start_idxs[n], then min(K[n], lengths[n]) - 1 selections,
 *  then -1; a start index outside [0, lengths[n]) of a non-empty cloud gives a row of -1.  K[n] > max_K is read as
 *  max_K.  cluster_size 0 lets the library choose the CTAs per cloud (1 to 16), else forces it.  scratch: N P floats,
 *  or NULL when the clouds fit on chip (the call fails otherwise).  P < 2^31.
 * ball_query_forward: idx (N, P1, K) int64, dists (N, P1, K) float32 and, unless NULL, nn (N, P1, K, 3) float32: the
 *  first K targets j in ascending order with dist2 < radius * radius (float32), padded with -1, 0 and 0.  With
 *  skip_points_outside_cube and radius < 0 nothing is found.  N P1 K < 2^31 and N P2 < 2^31.
 * ball_query_backward: grad_dists (N, P1, K) and grad_nn (N, P1, K, 3), either NULL -> grad_p1 (N, P1, 3) and
 *  grad_p2 (N, P2, 3), either NULL.  workspace: b200r_ball_query_workspace_bytes(N, P1, P2, K) bytes.
 */
int b200r_sample_farthest_points(const float* points, int64_t N, int64_t P, const int64_t* lengths, const int64_t* K,
                                 const int64_t* start_idxs, int64_t max_K, int32_t cluster_size, float* scratch,
                                 int64_t* idx, void* stream);
size_t b200r_ball_query_workspace_bytes(int64_t N, int64_t P1, int64_t P2, int64_t K);
int b200r_ball_query_forward(const float* p1, const float* p2, int64_t N, int64_t P1, int64_t P2,
                             const int64_t* lengths1, const int64_t* lengths2, int64_t K, float radius,
                             int32_t skip_points_outside_cube, int64_t* idx, float* dists, float* nn, void* stream);
int b200r_ball_query_backward(const float* p1, const float* p2, int64_t N, int64_t P1, int64_t P2,
                              const int64_t* lengths1, const int64_t* lengths2, int64_t K, const int64_t* idx,
                              const float* grad_dists, const float* grad_nn, void* workspace, size_t workspace_bytes,
                              float* grad_p1, float* grad_p2, void* stream);

/*
 * Programmatic dependent launch between the kernels of one call (setup -> scan -> fill -> fine; backward -> scatter):
 * the next kernel is made resident while its predecessor drains.  On by default; results never depend on it.
 */
void b200r_set_pdl(int32_t enabled);

#ifdef __cplusplus
}
#endif
#endif /* B200_RASTER_H_ */
