"""ctypes loader of libb200raster.so -- the C-ABI boundary (include/b200_raster.h).

There is no CPU or PyTorch fallback: if the CUDA library is missing the import of the ops
fails loudly with the build command to run.
"""
import ctypes
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "lib", "libb200raster.so")

_c_f = ctypes.POINTER(ctypes.c_float)
_vp = ctypes.c_void_p
_i32, _i64, _f32, _f64, _sz = ctypes.c_int32, ctypes.c_int64, ctypes.c_float, ctypes.c_double, ctypes.c_size_t

# name -> (restype, argtypes); mirrors include/b200_raster.h one to one.
SIGNATURES = {
    "b200r_version": (ctypes.c_char_p, []),
    "b200r_last_error": (ctypes.c_char_p, []),
    "b200r_kernel_launch_count": (_i64, []),
    "b200r_set_profiling": (None, [_i32]),
    "b200r_set_pdl": (None, [_i32]),
    "b200r_last_phase_ms": (ctypes.c_int, [ctypes.POINTER(ctypes.c_float)]),
    "b200r_rasterize_meshes_workspace_bytes": (_sz, [_i64, _i32, _i32, _i32, _i64]),
    "b200r_rasterize_meshes_forward": (
        ctypes.c_int,
        [_vp, _i64, _vp, _vp, _vp, _i32, _i32, _i32, _f32, _i32, _i32, _i32, _i32, _i32, _i32,
         _vp, _vp, _vp, _vp, _vp, _sz, _i64, _vp]),
    "b200r_rasterize_meshes_backward": (
        ctypes.c_int, [_vp, _i64, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _vp, _vp]),
    "b200r_rasterize_meshes_forward_indexed": (
        ctypes.c_int,
        [_vp, _i64, _vp, _i64, _vp, _vp, _vp, _i32, _i32, _i32, _f32, _i32, _i32, _i32, _i32,
         _vp, _vp, _vp, _vp, _vp, _vp, _sz, _i64, _vp]),
    "b200r_rasterize_meshes_backward_indexed": (
        ctypes.c_int, [_vp, _vp, _i64, _i64, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _vp, _vp]),
    "b200r_rasterize_points_workspace_bytes": (_sz, [_i64, _i32, _i32, _i32, _i64]),
    "b200r_rasterize_points_forward": (
        ctypes.c_int,
        [_vp, _i64, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _sz, _i64, _vp]),
    "b200r_rasterize_points_backward": (
        ctypes.c_int, [_vp, _i64, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _vp, _vp]),
    "b200r_alpha_composite_forward_strided": (
        ctypes.c_int, [_vp, _i64, _i64, _i64, _i64, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _vp, _vp]),
    "b200r_alpha_composite_backward_strided": (
        ctypes.c_int, [_vp, _vp, _i64, _i64, _i64, _i64, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _vp, _vp, _vp]),
    "b200r_weighted_sum_forward": (
        ctypes.c_int, [_vp, _i64, _i64, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _vp, _vp]),
    "b200r_weighted_sum_backward": (
        ctypes.c_int, [_vp, _vp, _i64, _i64, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _vp, _vp, _vp]),
    "b200r_norm_weighted_sum_forward": (
        ctypes.c_int, [_vp, _i64, _i64, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _vp, _vp]),
    "b200r_norm_weighted_sum_backward": (
        ctypes.c_int, [_vp, _vp, _i64, _i64, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _vp, _vp, _vp]),
    "b200r_points_alpha_render_forward": (
        ctypes.c_int, [_vp, _i64, _i64, _i64, _i64, _vp, _vp, _f32, _i32, _i32, _i32, _i32, _vp, _vp]),
    "b200r_points_alpha_render_backward": (
        ctypes.c_int, [_vp, _vp, _i64, _i64, _i64, _i64, _vp, _vp, _f32, _i32, _i32, _i32, _i32, _vp, _vp, _vp]),
    "b200r_sigmoid_alpha_blend_forward": (ctypes.c_int, [_vp, _vp, _i32, _i32, _i32, _i32, _f32, _vp, _vp]),
    "b200r_sigmoid_alpha_blend_backward": (
        ctypes.c_int, [_vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _f32, _vp, _vp]),
    "b200r_softmax_rgb_blend_forward": (
        ctypes.c_int, [_vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _f32, _f32, _vp, _vp, _vp, _vp, _f64, _f64, _vp, _vp]),
    "b200r_softmax_rgb_blend_backward": (
        ctypes.c_int,
        [_vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _f32, _f32, _vp, _vp, _vp, _vp, _f64, _f64, _vp, _vp, _vp, _vp]),
    "b200r_soft_depth_blend_forward": (
        ctypes.c_int, [_vp, _vp, _vp, _i32, _i32, _i32, _i32, _f32, _vp, _f32, _vp, _vp]),
    "b200r_soft_depth_blend_backward": (
        ctypes.c_int, [_vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _f32, _vp, _f32, _vp, _vp, _vp]),
    "b200r_hard_depth_forward": (ctypes.c_int, [_vp, _vp, _i32, _i32, _i32, _i32, _vp, _f32, _vp, _vp]),
    "b200r_hard_depth_backward": (ctypes.c_int, [_vp, _vp, _i32, _i32, _i32, _i32, _vp, _vp]),
    "b200r_splatter_blend_forward": (
        ctypes.c_int, [_vp, _vp, _vp, _i32, _i32, _i32, _i32, _f64, _vp, _vp, _vp, _vp]),
    "b200r_splatter_blend_workspace_bytes": (_sz, [_i32, _i32, _i32]),
    "b200r_splatter_blend_backward": (
        ctypes.c_int, [_vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _f64, _vp, _vp, _vp, _sz, _vp, _vp, _vp]),
    "b200r_shading_forward": (
        ctypes.c_int, [_vp, _vp, _vp, _vp, _i64, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _vp]),
    "b200r_shading_workspace_bytes": (_sz, [_i32, _i32, _i32, _i32]),
    "b200r_shading_backward": (
        ctypes.c_int,
        [_vp, _vp, _vp, _vp, _vp, _vp, _i64, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _vp, _sz, _vp, _vp, _vp,
         _vp, _vp, _vp]),
    "b200r_gouraud_forward": (
        ctypes.c_int, [_vp, _vp, _vp, _i64, _vp, _vp, _i32, _vp, _vp, _i64, _vp, _vp, _i64, _i32, _vp, _vp, _vp]),
    "b200r_gouraud_workspace_bytes": (_sz, [_i32, _i64]),
    "b200r_gouraud_backward": (
        ctypes.c_int,
        [_vp, _vp, _vp, _vp, _i64, _vp, _vp, _i32, _vp, _vp, _i64, _vp, _vp, _i64, _i32, _vp, _vp, _sz, _vp, _vp, _vp,
         _vp, _vp, _vp]),
    "b200r_texture_uv_forward": (
        ctypes.c_int, [_vp, _vp, _vp, _i64, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _vp, _vp]),
    "b200r_texture_uv_backward": (
        ctypes.c_int,
        [_vp, _vp, _vp, _vp, _i64, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _vp,
         _vp]),
    "b200r_texture_atlas_workspace_bytes": (_sz, [_i32, _i32, _i32, _i32, _i64, _i32]),
    "b200r_texture_atlas_forward": (
        ctypes.c_int, [_vp, _vp, _vp, _i64, _i32, _i32, _i32, _i32, _i32, _i32, _vp, _vp]),
    "b200r_texture_atlas_backward": (
        ctypes.c_int, [_vp, _vp, _vp, _i64, _i32, _i32, _i32, _i32, _i32, _i32, _vp, _sz, _vp, _vp]),
    "b200r_normals_workspace_bytes": (_sz, [_i64, _i64]),
    "b200r_face_areas_normals_forward": (ctypes.c_int, [_vp, _i64, _vp, _i64, _vp, _vp, _vp]),
    "b200r_face_areas_normals_backward": (ctypes.c_int, [_vp, _vp, _vp, _i64, _vp, _i64, _vp, _sz, _vp, _vp]),
    "b200r_verts_normals_forward": (ctypes.c_int, [_vp, _i64, _vp, _i64, _vp, _sz, _vp, _vp, _vp, _vp]),
    "b200r_verts_normals_backward": (ctypes.c_int, [_vp, _vp, _i64, _vp, _i64, _vp, _vp, _vp, _sz, _vp, _vp]),
    "b200r_sample_points_workspace_bytes": (_sz, [_i64, _i64, _i64, _i64, _i32]),
    "b200r_sample_points_forward": (
        ctypes.c_int,
        [_vp, _i64, _vp, _i64, _vp, _vp, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _sz, _vp, _vp, _vp, _vp, _vp, _vp]),
    "b200r_sample_points_backward": (
        ctypes.c_int, [_vp, _vp, _vp, _i64, _vp, _i64, _i64, _i64, _vp, _vp, _vp, _sz, _vp, _vp]),
    "b200r_chamfer_workspace_bytes": (_sz, [_i64, _i64, _i64, _i32]),
    "b200r_chamfer_forward": (
        ctypes.c_int,
        [_vp, _vp, _i64, _i64, _i64] + [_vp] * 5 + [_i32] * 5 + [_vp, _sz] + [_vp] * 11 + [_vp]),
    "b200r_chamfer_backward": (
        ctypes.c_int,
        [_vp, _vp, _i64, _i64, _i64] + [_vp] * 5 + [_i32] * 5 + [_vp] * 8 + [_vp, _sz] + [_vp] * 3),
    "b200r_sample_farthest_points": (ctypes.c_int, [_vp, _i64, _i64, _vp, _vp, _vp, _i64, _i32, _vp, _vp, _vp]),
    "b200r_ball_query_workspace_bytes": (_sz, [_i64, _i64, _i64, _i64]),
    "b200r_ball_query_forward": (
        ctypes.c_int, [_vp, _vp, _i64, _i64, _i64, _vp, _vp, _i64, _f32, _i32, _vp, _vp, _vp, _vp]),
    "b200r_ball_query_backward": (
        ctypes.c_int, [_vp, _vp, _i64, _i64, _i64, _vp, _vp, _i64, _vp, _vp, _vp, _vp, _sz, _vp, _vp, _vp]),
    "b200r_regularizers_workspace_bytes": (_sz, [_i64, _i64, _i32]),
    "b200r_mesh_edge_table": (ctypes.c_int, [_vp, _i64, _i64, _vp, _vp, _i32, _vp, _sz, _vp, _vp, _vp, _vp, _vp]),
    "b200r_mesh_edge_loss_forward": (ctypes.c_int, [_vp, _i64, _vp, _i64, _vp, _vp, _i32, _f32, _vp, _sz, _vp, _vp]),
    "b200r_mesh_edge_loss_backward": (
        ctypes.c_int, [_vp, _vp, _i64, _vp, _i64, _vp, _vp, _i32, _f32, _vp, _sz, _vp, _vp]),
    "b200r_mesh_laplacian_smoothing_forward": (
        ctypes.c_int, [_vp, _i64, _vp, _i64, _vp, _vp, _i32, _i32, _vp, _sz, _vp, _vp]),
    "b200r_mesh_laplacian_smoothing_backward": (
        ctypes.c_int, [_vp, _vp, _i64, _vp, _i64, _vp, _vp, _i32, _i32, _vp, _sz, _vp, _vp]),
    "b200r_mesh_normal_consistency_forward": (ctypes.c_int, [_vp, _i64, _vp, _i64, _vp, _vp, _i32, _vp, _sz, _vp, _vp]),
    "b200r_mesh_normal_consistency_backward": (
        ctypes.c_int, [_vp, _vp, _i64, _vp, _i64, _vp, _vp, _i32, _vp, _sz, _vp, _vp]),
    "b200r_clip_faces_workspace_words": (_i64, [_i64]),
    "b200r_clip_faces_count": (ctypes.c_int, [_vp, _vp, _vp, _i64, _vp, _i32, _i32, _f64, _vp, _vp]),
    "b200r_clip_faces_fill": (
        ctypes.c_int,
        [_vp, _i64, _vp, _i32, _vp, _i32, _i32, _f64, _i32, _vp, _i64, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
         _vp]),
    "b200r_clip_faces_backward": (
        ctypes.c_int, [_vp, _i64, _vp, _i32, _i32, _f64, _i32, _vp, _i64, _i64, _vp, _vp, _vp, _vp]),
    "b200r_clip_convert_forward": (ctypes.c_int, [_vp, _vp, _i64, _vp, _vp, _vp, _vp, _vp, _vp]),
    "b200r_clip_convert_backward": (ctypes.c_int, [_vp, _vp, _vp, _i64, _vp, _vp, _i64, _vp, _vp, _vp]),
    "b200r_interp_face_attrs_forward":(ctypes.c_int, [_vp, _vp, _vp, _i64, _i64, _i64, _vp, _vp]),
    "b200r_interp_face_attrs_backward": (ctypes.c_int, [_vp, _vp, _vp, _vp, _i64, _i64, _i64, _vp, _vp, _vp]),
    "b200r_rasterize_meshes_coarse": (
        ctypes.c_int, [_vp, _i64, _vp, _vp, _i32, _i32, _i32, _f32, _i32, _i32, _vp, _vp, _vp, _vp]),
    "b200r_rasterize_points_coarse": (
        ctypes.c_int, [_vp, _i64, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp]),
    "b200r_peer_alloc": (ctypes.c_int, [_sz, ctypes.POINTER(_vp), ctypes.c_char_p]),
    "b200r_peer_open": (ctypes.c_int, [ctypes.c_char_p, ctypes.POINTER(_vp)]),
    "b200r_peer_close": (ctypes.c_int, [_vp]),
    "b200r_peer_free": (ctypes.c_int, [_vp]),
    "b200r_packed_frames_bytes": (_sz, [_i64, _i32, _i32, _i32]),
    "b200r_fragments_pack_push": (
        ctypes.c_int, [_vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _i64, ctypes.POINTER(_vp), _i32, _vp, _vp]),
    "b200r_fragments_unpack": (
        ctypes.c_int, [_vp, _i32, _i32, _i32, _i32, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "b200r_exchange_create": (
        ctypes.c_int, [_i32, _i32, _i32, _i32, _i32, _i64, _vp, _vp, _vp, ctypes.POINTER(_vp), ctypes.POINTER(_vp)]),
    "b200r_exchange_destroy": (ctypes.c_int, [_vp]),
    "b200r_exchange_push": (ctypes.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "b200r_exchange_expand": (ctypes.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, ctypes.POINTER(_i32)]),
    "b200r_exchange_wait": (ctypes.c_int, [_vp, _i32, _vp]),
    "b200r_rasterize_meshes_forward_host": (
        ctypes.c_int,
        [_vp, _i64, _vp, _vp, _vp, _i32, _i32, _i32, _f32, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp]),
    "b200r_rasterize_meshes_backward_host": (
        ctypes.c_int, [_vp, _i64, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _vp]),
    "b200r_rasterize_points_forward_host": (
        ctypes.c_int, [_vp, _i64, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _vp, _vp, _vp]),
    "b200r_rasterize_points_backward_host": (
        ctypes.c_int, [_vp, _i64, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _vp]),
}

_lib = None


def load():
    """Load (once) and return the ctypes handle with typed prototypes."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            "pytorch3d_b200: %s is missing. Build it with `python -m pytorch3d_b200.build` "
            "(nvcc, sm_90a). There is no CPU fallback." % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the .so does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def last_error():
    return load().b200r_last_error().decode()


def check(rc):
    """Turn a C-ABI status into the exception the reference op would raise (RuntimeError)."""
    if rc != 0:
        raise RuntimeError(last_error() or ("libb200raster error %d" % rc))
