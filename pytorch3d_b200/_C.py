"""Operator-level drop-in for the rasterizer part of `pytorch3d._C`.

Same names, positional arguments, return values and error behaviour as the pybind11 ops registered
in pytorch3d/csrc/ext.cpp:53-56:

    rasterize_meshes, rasterize_meshes_backward, rasterize_points, rasterize_points_backward

implemented by calling the C ABI of libb200raster.so (include/b200_raster.h) on the tensors' device
pointers and the current CUDA stream.  These four ops and the fused indexed pair are bound by the torch C++ extension
csrc/torch_ext.cpp (the kind of binding the reference uses), which checks their arguments; every other op calls the C
ABI through ctypes.  PyTorch is used only for device memory and streams.
There is no CPU path: CPU tensors raise RuntimeError, like a CUDA-less build of the reference does
for CUDA tensors (rasterize_meshes.h:137-139, mirrored).
"""
import ctypes
import importlib.util
import os
from typing import Tuple

import torch

from . import _lib

kMaxPointsPerPixel = 150  # rasterization_utils.cuh:48

# Capacity (in (tile, element) pairs) of the bin lists; 0 = library default.  Results never depend on it:
# tiles whose list does not fit fall back to testing every element of their mesh / cloud.  Tests lower it
# to exercise that path.
PAIR_CAPACITY = 0

_EXT = None


def _ext():
    """The torch C++ extension over the C ABI (csrc/torch_ext.cpp), loaded once.  It is built by
    `python -m pytorch3d_b200.build` next to libb200raster.so; without it the rasterizer ops fail loudly."""
    global _EXT
    if _EXT is None:
        from . import build as _build
        path = _build.ext_path()
        if not os.path.exists(path):
            raise ImportError(
                "pytorch3d_b200: %s is missing. Build it with `python -m pytorch3d_b200.build` "
                "(nvcc, sm_90a; g++ for the torch extension). There is no CPU fallback." % path)
        _lib.load()  # fails loudly if libb200raster.so itself is missing
        spec = importlib.util.spec_from_file_location(_build.EXT_NAME, path)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        _EXT = mod
    return _EXT


def _ptr(t):
    return t.data_ptr() if t is not None and t.numel() > 0 else None


def _require_cuda(*named):
    dev = None
    for name, t in named:
        if not t.is_cuda:
            raise RuntimeError(
                "%s must be a CUDA tensor: pytorch3d_b200 is an H100-native (sm_90a) rasterizer and has "
                "no CPU implementation." % name)
        if dev is None:
            dev = t.device
        elif t.device != dev:
            raise RuntimeError(
                "Expected all tensors to be on the same device (%s is on %s, expected %s)" % (name, t.device, dev))
    return dev


def _stream_ptr(device):
    return torch.cuda.current_stream(device).cuda_stream


def rasterize_meshes(
    face_verts: torch.Tensor,
    mesh_to_face_first_idx: torch.Tensor,
    num_faces_per_mesh: torch.Tensor,
    clipped_faces_neighbor_idx: torch.Tensor,
    image_size: Tuple[int, int],
    blur_radius: float,
    faces_per_pixel: int,
    bin_size: int,
    max_faces_per_bin: int,
    perspective_correct: bool,
    clip_barycentric_coords: bool,
    cull_backfaces: bool,
):
    """pytorch3d._C.rasterize_meshes (RasterizeMeshes, rasterize_meshes.h:513-562).

    Clipped-face neighbours are only produced by clip_faces: the kernel variant with the neighbour logic is used unless
    the caller tagged the tensor `_b200_all_minus_one` (our own wrapper does when nothing was clipped); no host sync
    either way.
    """
    return _ext().rasterize_meshes(
        face_verts, mesh_to_face_first_idx, num_faces_per_mesh, clipped_faces_neighbor_idx,
        (int(image_size[0]), int(image_size[1])), float(blur_radius), int(faces_per_pixel), int(bin_size),
        int(max_faces_per_bin), bool(perspective_correct), bool(clip_barycentric_coords), bool(cull_backfaces),
        int(PAIR_CAPACITY), bool(getattr(clipped_faces_neighbor_idx, "_b200_all_minus_one", False)))


def rasterize_meshes_backward(
    face_verts: torch.Tensor,
    pix_to_face: torch.Tensor,
    grad_zbuf: torch.Tensor,
    grad_bary: torch.Tensor,
    grad_dists: torch.Tensor,
    perspective_correct: bool,
    clip_barycentric_coords: bool,
):
    """pytorch3d._C.rasterize_meshes_backward (RasterizeMeshesBackward, rasterize_meshes.h:211-218)."""
    return _ext().rasterize_meshes_backward(face_verts, pix_to_face, grad_zbuf, grad_bary, grad_dists,
                                            bool(perspective_correct), bool(clip_barycentric_coords))


def rasterize_meshes_indexed(
    verts_packed: torch.Tensor,
    faces_packed: torch.Tensor,
    mesh_to_face_first_idx: torch.Tensor,
    num_faces_per_mesh: torch.Tensor,
    image_size: Tuple[int, int],
    blur_radius: float,
    faces_per_pixel: int,
    perspective_correct: bool,
    clip_barycentric_coords: bool,
    cull_backfaces: bool,
):
    """Fused `rasterize_meshes(verts_packed[faces_packed], ...)` (no counterpart in pytorch3d._C; SURVEY.md 8 f-4).

    Returns (pix_to_face, zbuf, bary, dists, face_verts): the four Fragments buffers and the gathered (F,3,3)
    faces that `rasterize_meshes_backward_indexed` needs.
    """
    return _ext().rasterize_meshes_indexed(verts_packed, faces_packed, mesh_to_face_first_idx, num_faces_per_mesh,
                                           (int(image_size[0]), int(image_size[1])), float(blur_radius),
                                           int(faces_per_pixel), bool(perspective_correct),
                                           bool(clip_barycentric_coords), bool(cull_backfaces), int(PAIR_CAPACITY))


def rasterize_meshes_backward_indexed(
    face_verts: torch.Tensor,
    faces_packed: torch.Tensor,
    num_verts: int,
    pix_to_face: torch.Tensor,
    grad_zbuf: torch.Tensor,
    grad_bary: torch.Tensor,
    grad_dists: torch.Tensor,
    perspective_correct: bool,
    clip_barycentric_coords: bool,
):
    """Backward of `rasterize_meshes_indexed`: the gradient w.r.t. verts_packed, (V, 3)."""
    return _ext().rasterize_meshes_backward_indexed(face_verts, faces_packed, int(num_verts), pix_to_face, grad_zbuf,
                                                    grad_bary, grad_dists, bool(perspective_correct),
                                                    bool(clip_barycentric_coords))


def rasterize_points(
    points: torch.Tensor,
    cloud_to_packed_first_idx: torch.Tensor,
    num_points_per_cloud: torch.Tensor,
    image_size: Tuple[int, int],
    radius: torch.Tensor,
    points_per_pixel: int,
    bin_size: int,
    max_points_per_bin: int,
):
    """pytorch3d._C.rasterize_points (RasterizePoints, rasterize_points.h:343-374)."""
    return _ext().rasterize_points(points, cloud_to_packed_first_idx, num_points_per_cloud,
                                   (int(image_size[0]), int(image_size[1])), radius, int(points_per_pixel),
                                   int(bin_size), int(max_points_per_bin), int(PAIR_CAPACITY))


def rasterize_points_backward(points: torch.Tensor, idxs: torch.Tensor, grad_zbuf: torch.Tensor,
                              grad_dists: torch.Tensor):
    """pytorch3d._C.rasterize_points_backward (RasterizePointsBackward, rasterize_points.h:281-285)."""
    return _ext().rasterize_points_backward(points, idxs, grad_zbuf, grad_dists)



# ------------------------------------------------------------------------------------------------ the ctypes ops
# Every op below checks each tensor it hands the library by pointer (device, then dtype and shape, then the kernels'
# size limits) and calls the library through `_launch`.

F32, I32, I64 = torch.float32, torch.int32, torch.int64
_TYPE_NAMES = {F32: "Float", I32: "Int", I64: "Long", torch.bool: "Bool"}


def _launch(dev, name, *args):
    """b200r_<name>(*args, current stream of dev) on the device `dev`; a failed status raises RuntimeError."""
    lib = _lib.load()
    with torch.cuda.device(dev):
        _lib.check(getattr(lib, "b200r_" + name)(*args, _stream_ptr(dev)))


def _workspace_size(name, *sizes):
    return int(getattr(_lib.load(), "b200r_%s_workspace_bytes" % name)(*sizes))


def _workspace(dev, name, *sizes, required=False):
    """(uint8 workspace on dev, its bytes) as b200r_<name>_workspace_bytes(*sizes) sizes it; (None, 0) when it needs
    none, unless `required`: then a size of 0 raises.  The caching allocator's blocks are 512-byte aligned."""
    ws_bytes = _workspace_size(name, *sizes)
    if ws_bytes == 0 and required:
        raise RuntimeError("%s: could not size the workspace for sizes %s" % (name, sizes))
    return (torch.empty((ws_bytes,), dtype=torch.uint8, device=dev) if ws_bytes else None), ws_bytes


# The two dtype errors of ATen, which the reference's ops raise: data_ptr<T>()'s, here with the argument named at the
# end, and checkScalarType's, which the blending, shading and texture ops use for their float inputs.
_DATA_PTR_TEXT = "expected scalar type {want} but found {got} for {name}"
_SCALAR_TYPE_TEXT = "Expected tensor for {name} to have scalar type {want}; but got {got}"


def _check_tensor(name, t, dtype, shape=None, dims=None, op=None, text=_DATA_PTR_TEXT):
    """Raises RuntimeError unless `t` has `dtype` and `shape`, each when given (None in `shape` leaves a dimension
    free).  The message names the op when given, the argument, and the expected dtype (in `text`) or shape (`dims`,
    default the sizes)."""
    if dtype is not None and t.dtype != dtype:
        raise RuntimeError((op + ": " if op else "") + text.format(want=_TYPE_NAMES[dtype], got=t.dtype, name=name))
    if shape is not None and not _fits(t.shape, shape):
        if dims is None:
            dims = ", ".join("*" if s is None else str(s) for s in shape) + ("," if len(shape) == 1 else "")
        raise RuntimeError("%s%s must be (%s), got %s" % (op + ": " if op else "", name, dims, tuple(t.shape)))


def _check_float(name, t, shape=None, dims=None):
    """_check_tensor for a float32 input of the blending, shading and texture ops, with checkScalarType's text."""
    _check_tensor(name, t, F32, shape, dims, text=_SCALAR_TYPE_TEXT)


def _fits(size, shape):
    """Whether `size` is `shape`, where None leaves a dimension free."""
    if len(size) != len(shape):
        return False
    for n, s in zip(size, shape):
        if s is not None and s != n:
            return False
    return True


def _check_verts_faces(op, verts, faces, *named):
    """(V, F, device) of float32 verts (V, 3) and int64 faces (F, 3) on one CUDA device with the (name, tensor) pairs
    `named`; the caller checks its own size limit."""
    dev = _require_cuda(("verts", verts), ("faces", faces), *named)
    _check_tensor("verts", verts, F32, (None, 3), "V, 3", op)
    _check_tensor("faces", faces, I64, (None, 3), "F, 3", op)
    return int(verts.shape[0]), int(faces.shape[0]), dev


def _check_ranges(op, first_name, first, num_name, num):
    """N of the int64 (N,) per-mesh ranges `first` and `num`."""
    _check_tensor(first_name, first, I64, (None,), "N,", op)
    N = int(first.shape[0])
    _check_tensor(num_name, num, I64, (N,), "N,", op)
    return N


def _refuse_nondeterministic(op, why):
    if torch.are_deterministic_algorithms_enabled() and not torch.is_deterministic_algorithms_warn_only_enabled():
        raise RuntimeError("%s does not have a deterministic implementation (%s), but you set "
                           "'torch.use_deterministic_algorithms(True)'." % (op, why))


def _c(t):
    return t.contiguous() if t is not None else None


def _strides4(t):
    return (ctypes.c_int64 * 4)(*[int(v) for v in t.stride()])


def _check_composite_inputs(features, weights, index, index_dtype, dims, grad=None):
    """(C, P, device) of features (C, P) f32 and of the float32 per-slot weights (name, tensor) and `index_dtype`
    per-slot indices (name, tensor), both of the 4-d shape `dims`; the upstream gradient (name, tensor), when given, is
    only checked for its device here."""
    dev = _require_cuda(*([grad] if grad is not None else []), ("features", features), weights, index)
    _check_tensor("features", features, F32, (None, None), "C, P")
    _check_tensor(*index, index_dtype, (None,) * 4, dims)
    _check_tensor(*weights, F32, tuple(index[1].shape), dims)
    return int(features.shape[0]), int(features.shape[1]), dev


def _feature_layout(features):
    """(tensor to read, stride_c, stride_p): a (C, P) view of point-major memory (`features_packed().permute(1, 0)`,
    what the renderer passes) is read in place; anything else as a contiguous (C, P) array."""
    C, P = (int(v) for v in features.shape)
    if features.stride(0) == 1 and features.stride(1) == C and P > 0:
        return features, 1, C
    f = features.contiguous()
    return f, P, 1


def _grad_features(layout, C, P, dev):
    """grad_features (C, P) with the memory layout `features` was read in: point-major when it was read in place."""
    if layout and layout[0] == 1 and C > 1:
        return torch.empty((P, C), dtype=F32, device=dev).permute(1, 0)
    return torch.empty((C, P), dtype=F32, device=dev)


def _composite(name, features, alphas, points_idx, strided):
    """The compositing forwards: alphas (N,K,H,W) f32, points_idx (N,K,H,W) i64 (any strides) -> (N,C,H,W) f32.  With
    `strided` b200r_<name> takes the features' strides (see _feature_layout), else a contiguous (C, P) array."""
    C, P, dev = _check_composite_inputs(features, ("alphas", alphas), ("points_idx", points_idx), I64, "N, K, H, W")
    N, K, H, W = (int(v) for v in points_idx.shape)
    feat, *layout = _feature_layout(features) if strided else (features.contiguous(),)
    result = torch.empty((N, C, H, W), dtype=F32, device=dev)
    if result.numel() == 0:
        return result
    if K == 0:
        return result.zero_()
    _launch(dev, name, _ptr(feat), C, P, *layout, alphas.data_ptr(), _strides4(alphas), points_idx.data_ptr(),
            _strides4(points_idx), N, K, H, W, _ptr(result))
    return result


def _composite_grad(name, grad_outputs, features, alphas, points_idx, strided):
    """The compositing backwards -> (grad_features (C,P) with the memory layout `features` is read in, grad_alphas)."""
    C, P, dev = _check_composite_inputs(features, ("alphas", alphas), ("points_idx", points_idx), I64, "N, K, H, W",
                                        ("grad_outputs", grad_outputs))
    N, K, H, W = (int(v) for v in points_idx.shape)
    _check_tensor("grad_outputs", grad_outputs, F32, (N, C, H, W), "N, C, H, W")
    feat, *layout = _feature_layout(features) if strided else (features.contiguous(),)
    go = grad_outputs.contiguous()
    grad_features = _grad_features(layout, C, P, dev)
    grad_alphas = torch.empty((N, K, H, W), dtype=F32, device=dev)
    if C * P == 0 or grad_alphas.numel() == 0:
        return grad_features.zero_(), grad_alphas.zero_()
    _launch(dev, name, _ptr(go), _ptr(feat), C, P, *layout, alphas.data_ptr(), _strides4(alphas), points_idx.data_ptr(),
            _strides4(points_idx), N, K, H, W, grad_features.data_ptr(), _ptr(grad_alphas))
    return grad_features, grad_alphas


def accum_alphacomposite(features: torch.Tensor, alphas: torch.Tensor, points_idx: torch.Tensor):
    """pytorch3d._C.accum_alphacomposite (alphaCompositeForward, csrc/compositing/alpha_composite.h:59-82).

    features (C,P) f32 (a (C,P) view of point-major memory -- what the renderer passes -- is read in place), alphas
    (N,K,H,W) f32, points_idx (N,K,H,W) i64 (any strides) -> (N,C,H,W) f32."""
    return _composite("alpha_composite_forward_strided", features, alphas, points_idx, True)


def accum_alphacomposite_backward(grad_outputs: torch.Tensor, features: torch.Tensor, alphas: torch.Tensor,
                                  points_idx: torch.Tensor):
    """pytorch3d._C.accum_alphacomposite_backward (alpha_composite.h:84-116) -> (grad_features, grad_alphas);
    grad_features (C,P) has the memory layout of `features`."""
    return _composite_grad("alpha_composite_backward_strided", grad_outputs, features, alphas, points_idx, True)


def points_alpha_render(features: torch.Tensor, idx: torch.Tensor, dists: torch.Tensor, radius: float):
    """Fused `accum_alphacomposite(features, 1 - dists / radius**2, idx)` on the rasterizer's own layout (no counterpart
    in pytorch3d._C; SURVEY.md 8f-2): features (C,P) f32, idx (N,H,W,K) i32, dists (N,H,W,K) f32 -> (N,C,H,W) f32."""
    C, P, dev = _check_composite_inputs(features, ("dists", dists), ("idx", idx), I32, "N, H, W, K")
    N, H, W, K = (int(v) for v in idx.shape)
    feat, fs_c, fs_p = _feature_layout(features)
    ii, dd = idx.contiguous(), dists.contiguous()
    images = torch.empty((N, C, H, W), dtype=F32, device=dev)
    if images.numel() == 0:
        return images
    _launch(dev, "points_alpha_render_forward", _ptr(feat), C, P, fs_c, fs_p, _ptr(ii), _ptr(dd),
            float(radius) * float(radius), N, K, H, W, _ptr(images))
    return images


def points_alpha_render_backward(grad_images: torch.Tensor, features: torch.Tensor, idx: torch.Tensor,
                                 dists: torch.Tensor, radius: float):
    """Backward of `points_alpha_render` -> (grad_features (C,P) with the memory layout of `features`, grad_dists
    (N,H,W,K))."""
    C, P, dev = _check_composite_inputs(features, ("dists", dists), ("idx", idx), I32, "N, H, W, K",
                                        ("grad_images", grad_images))
    N, H, W, K = (int(v) for v in idx.shape)
    _check_tensor("grad_images", grad_images, F32, (N, C, H, W), "N, C, H, W")
    feat, *layout = _feature_layout(features)
    go, ii, dd = grad_images.contiguous(), idx.contiguous(), dists.contiguous()
    grad_features = _grad_features(layout, C, P, dev)
    grad_dists = torch.empty((N, H, W, K), dtype=F32, device=dev)
    if C * P == 0 or grad_dists.numel() == 0:
        return grad_features.zero_(), grad_dists.zero_()
    _launch(dev, "points_alpha_render_backward", _ptr(go), _ptr(feat), C, P, *layout, _ptr(ii), _ptr(dd),
            float(radius) * float(radius), N, K, H, W, grad_features.data_ptr(), _ptr(grad_dists))
    return grad_features, grad_dists


def accum_weightedsum(features: torch.Tensor, alphas: torch.Tensor, points_idx: torch.Tensor):
    """pytorch3d._C.accum_weightedsum (weightedSumForward, csrc/compositing/weighted_sum.h:57-78)."""
    return _composite("weighted_sum_forward", features, alphas, points_idx, False)


def accum_weightedsum_backward(grad_outputs: torch.Tensor, features: torch.Tensor, alphas: torch.Tensor,
                               points_idx: torch.Tensor):
    """pytorch3d._C.accum_weightedsum_backward (weighted_sum.h:80-110) -> (grad_features, grad_alphas)."""
    return _composite_grad("weighted_sum_backward", grad_outputs, features, alphas, points_idx, False)


def accum_weightedsumnorm(features: torch.Tensor, alphas: torch.Tensor, points_idx: torch.Tensor):
    """pytorch3d._C.accum_weightedsumnorm (weightedSumNormForward, csrc/compositing/norm_weighted_sum.h:57-79)."""
    return _composite("norm_weighted_sum_forward", features, alphas, points_idx, False)


def accum_weightedsumnorm_backward(grad_outputs: torch.Tensor, features: torch.Tensor, alphas: torch.Tensor,
                                   points_idx: torch.Tensor):
    """pytorch3d._C.accum_weightedsumnorm_backward (norm_weighted_sum.h:81-112) -> (grad_features, grad_alphas)."""
    return _composite_grad("norm_weighted_sum_backward", grad_outputs, features, alphas, points_idx, False)


def _check_interp_inputs(pix_to_face, barycentric_coords, face_attrs, grad_pix_attrs=None):
    """(P, F, D, device), with the reference's shape errors (interp_face_attrs.cu)."""
    dev = _require_cuda(("pix_to_face", pix_to_face), ("barycentric_coords", barycentric_coords),
                        ("face_attributes", face_attrs),
                        *([("pix_attrs", grad_pix_attrs)] if grad_pix_attrs is not None else []))
    _check_tensor("pix_to_face", pix_to_face, I64, (None,), "P,")
    _check_tensor("barycentric_coords", barycentric_coords, F32)
    _check_tensor("face_attrs", face_attrs, F32)
    P = int(pix_to_face.shape[0])
    if tuple(barycentric_coords.shape) != (P, 3):
        raise RuntimeError("barycentric_coords must have size (P, 3)")
    if face_attrs.dim() != 3 or face_attrs.shape[1] != 3:
        raise RuntimeError("face_attrs must have size (F, 3, D)")
    F, D = int(face_attrs.shape[0]), int(face_attrs.shape[2])
    if grad_pix_attrs is not None:
        _check_tensor("grad_pix_attrs", grad_pix_attrs, F32)
        if tuple(grad_pix_attrs.shape) != (P, D):
            raise RuntimeError("grad_pix_attrs must have size (P, D)")
    return P, F, D, dev


def interp_face_attrs_forward(pix_to_face: torch.Tensor, barycentric_coords: torch.Tensor, face_attrs: torch.Tensor):
    """pytorch3d._C.interp_face_attrs_forward (csrc/interp_face_attrs/interp_face_attrs.h:45-66):
    pix_to_face (P,) i64, barycentric_coords (P,3) f32, face_attrs (F,3,D) f32 -> (P,D) f32."""
    P, F, D, dev = _check_interp_inputs(pix_to_face, barycentric_coords, face_attrs)
    p2f, bary, attrs = pix_to_face.contiguous(), barycentric_coords.contiguous(), face_attrs.contiguous()
    out = torch.empty((P, D), dtype=F32, device=dev)
    if out.numel() == 0:
        return out
    _launch(dev, "interp_face_attrs_forward", _ptr(p2f), _ptr(bary), _ptr(attrs), P, F, D, _ptr(out))
    return out


def interp_face_attrs_backward(pix_to_face: torch.Tensor, barycentric_coords: torch.Tensor, face_attrs: torch.Tensor,
                               grad_pix_attrs: torch.Tensor):
    """pytorch3d._C.interp_face_attrs_backward (interp_face_attrs.h:88-118) -> (grad_bary (P,3), grad_attrs (F,3,D))."""
    P, F, D, dev = _check_interp_inputs(pix_to_face, barycentric_coords, face_attrs, grad_pix_attrs)
    p2f, bary, attrs = pix_to_face.contiguous(), barycentric_coords.contiguous(), face_attrs.contiguous()
    gp = grad_pix_attrs.contiguous()
    grad_bary = torch.empty((P, 3), dtype=F32, device=dev)
    grad_attrs = torch.empty((F, 3, D), dtype=F32, device=dev)
    if grad_attrs.numel() == 0 or P == 0:
        return grad_bary.zero_(), grad_attrs.zero_()
    _launch(dev, "interp_face_attrs_backward", _ptr(p2f), _ptr(bary), _ptr(attrs), _ptr(gp), P, F, D, _ptr(grad_bary),
            _ptr(grad_attrs))
    return grad_bary, grad_attrs


def _check_index(pix_to_face, name="pix_to_face", dtype=I64):
    """The (N, H, W, K) of the per-slot tensor `name` of `dtype` (the face indices, or the splatter blend's background
    mask); dtype None checks the shape alone."""
    _check_tensor(name, pix_to_face, dtype)
    if pix_to_face.dim() != 4:
        raise RuntimeError("%s must have dimensions (N, H, W, K), got %s" % (name, tuple(pix_to_face.shape)))
    return tuple(pix_to_face.shape)


def sigmoid_alpha_blend(dists: torch.Tensor, pix_to_face: torch.Tensor, sigma: float):
    """pytorch3d._C.sigmoid_alpha_blend (SigmoidAlphaBlend, csrc/blending/sigmoid_alpha_blend.h): dists (N,H,W,K) f32,
    pix_to_face (N,H,W,K) i64 -> alphas (N,H,W) f32, bit-identical to the reference's CUDA kernel."""
    dev = _require_cuda(("distances", dists), ("pix_to_face", pix_to_face))
    N, H, W, K = _check_index(pix_to_face)
    _check_float("distances", dists, (N, H, W, K), "N, H, W, K")
    dd, p2f = dists.contiguous(), pix_to_face.contiguous()
    alphas = torch.empty((N, H, W), dtype=F32, device=dev)
    if alphas.numel() == 0:
        return alphas
    _launch(dev, "sigmoid_alpha_blend_forward", _ptr(dd), _ptr(p2f), N, H, W, K, float(sigma), _ptr(alphas))
    return alphas


def sigmoid_alpha_blend_backward(grad_alphas: torch.Tensor, alphas: torch.Tensor, dists: torch.Tensor,
                                 pix_to_face: torch.Tensor, sigma: float):
    """pytorch3d._C.sigmoid_alpha_blend_backward (SigmoidAlphaBlendBackward) -> grad_dists (N,H,W,K) f32."""
    dev = _require_cuda(("grad_alphas", grad_alphas), ("alphas", alphas), ("distances", dists),
                        ("pix_to_face", pix_to_face))
    N, H, W, K = _check_index(pix_to_face)
    _check_float("distances", dists, (N, H, W, K), "N, H, W, K")
    _check_float("alphas", alphas, (N, H, W), "N, H, W")
    _check_float("grad_alphas", grad_alphas, (N, H, W), "N, H, W")
    if alphas.numel() == 0:
        return grad_alphas  # what the reference returns for an empty image (sigmoid_alpha_blend.cu)
    ga, al, dd, p2f = grad_alphas.contiguous(), alphas.contiguous(), dists.contiguous(), pix_to_face.contiguous()
    grad_dists = torch.empty((N, H, W, K), dtype=F32, device=dev)
    if grad_dists.numel() == 0:
        return grad_dists
    _launch(dev, "sigmoid_alpha_blend_backward", _ptr(ga), _ptr(al), _ptr(dd), _ptr(p2f), N, H, W, K, float(sigma),
            _ptr(grad_dists))
    return grad_dists


def _softmax_side_args(dev, N, background_color, znear, zfar):
    """(background ptr, host background value, znear ptr, zfar ptr, znear value, zfar value, tensors to keep alive).
    Tensors are read on the device; Python numbers go to the kernel as numbers."""
    keep = []
    if torch.is_tensor(background_color):
        bg = background_color
        if bg.device != dev or bg.dtype != F32 or bg.numel() != 3:
            raise RuntimeError("background_color must be a float32 tensor of 3 values on %s" % dev)
        bg = bg.reshape(3).contiguous()
        keep.append(bg)
        bg_ptr, bg_val = bg.data_ptr(), None
    else:
        vals = [float(v) for v in background_color]
        if len(vals) != 3:
            raise RuntimeError("background_color must have 3 values")
        bg_ptr, bg_val = None, (ctypes.c_float * 3)(*vals)
    ptrs, values = [], []
    for name, z in (("znear", znear), ("zfar", zfar)):
        if torch.is_tensor(z):
            if z.device != dev or z.dtype != F32 or z.dim() != 1 or z.shape[0] not in (1, N):
                raise RuntimeError("%s must be a number or a float32 tensor of shape (N,) on %s" % (name, dev))
            z = z.expand(N).contiguous()
            keep.append(z)
            ptrs.append(z.data_ptr())
            values.append(0.0)
        else:
            ptrs.append(None)
            values.append(float(z))
    return bg_ptr, bg_val, ptrs[0], ptrs[1], values[0], values[1], keep


def _check_softmax_inputs(colors, pix_to_face, zbuf, dists, grad_out=None):
    dev = _require_cuda(*([("grad_out", grad_out)] if grad_out is not None else []), ("colors", colors),
                        ("zbuf", zbuf), ("dists", dists), ("pix_to_face", pix_to_face))
    shape = _check_index(pix_to_face)
    _check_float("colors", colors, shape + (3,), "N, H, W, K, 3")
    _check_float("zbuf", zbuf, shape, "N, H, W, K")
    _check_float("dists", dists, shape, "N, H, W, K")
    if grad_out is not None:
        _check_float("grad_out", grad_out, shape[:3] + (4,), "N, H, W, 4")
    if shape[3] > kMaxPointsPerPixel:
        raise RuntimeError("Must have faces_per_pixel <= %d" % kMaxPointsPerPixel)
    return shape + (dev,)


def softmax_rgb_blend(colors: torch.Tensor, pix_to_face: torch.Tensor, zbuf: torch.Tensor, dists: torch.Tensor,
                      sigma: float, gamma: float, background_color, znear=1.0, zfar=100.0):
    """Fused pytorch3d.renderer.blending.softmax_rgb_blend on the rasterizer's layout (no counterpart in pytorch3d._C;
    SURVEY.md 8f-5): colors (N,H,W,K,3) f32, pix_to_face (N,H,W,K) i64, zbuf / dists (N,H,W,K) f32; background_color a
    float32 CUDA tensor of 3 values or 3 numbers; znear / zfar numbers or float32 (N,) CUDA tensors -> (N,H,W,4) f32."""
    N, H, W, K, dev = _check_softmax_inputs(colors, pix_to_face, zbuf, dists)
    bg_ptr, bg_val, zn_ptr, zf_ptr, zn, zf, keep = _softmax_side_args(dev, N, background_color, znear, zfar)
    c, p2f, zb, dd = colors.contiguous(), pix_to_face.contiguous(), zbuf.contiguous(), dists.contiguous()
    out = torch.empty((N, H, W, 4), dtype=F32, device=dev)
    if out.numel() == 0:
        return out
    _launch(dev, "softmax_rgb_blend_forward", _ptr(c), _ptr(p2f), _ptr(zb), _ptr(dd), N, H, W, K, float(sigma),
            float(gamma), bg_ptr, bg_val, zn_ptr, zf_ptr, zn, zf, _ptr(out))
    del keep
    return out


def softmax_rgb_blend_backward(grad_out: torch.Tensor, colors: torch.Tensor, pix_to_face: torch.Tensor,
                               zbuf: torch.Tensor, dists: torch.Tensor, sigma: float, gamma: float, background_color,
                               znear=1.0, zfar=100.0):
    """Backward of `softmax_rgb_blend` -> (grad_colors (N,H,W,K,3), grad_dists (N,H,W,K), grad_zbuf (N,H,W,K))."""
    N, H, W, K, dev = _check_softmax_inputs(colors, pix_to_face, zbuf, dists, grad_out)
    bg_ptr, bg_val, zn_ptr, zf_ptr, zn, zf, keep = _softmax_side_args(dev, N, background_color, znear, zfar)
    go = grad_out.contiguous()
    c, p2f, zb, dd = colors.contiguous(), pix_to_face.contiguous(), zbuf.contiguous(), dists.contiguous()
    grad_colors = torch.empty((N, H, W, K, 3), dtype=F32, device=dev)
    grad_dists = torch.empty((N, H, W, K), dtype=F32, device=dev)
    grad_zbuf = torch.empty((N, H, W, K), dtype=F32, device=dev)
    if grad_dists.numel() == 0:
        return grad_colors, grad_dists, grad_zbuf
    _launch(dev, "softmax_rgb_blend_backward", _ptr(go), _ptr(c), _ptr(p2f), _ptr(zb), _ptr(dd), N, H, W, K,
            float(sigma), float(gamma), bg_ptr, bg_val, zn_ptr, zf_ptr, zn, zf, _ptr(grad_colors), _ptr(grad_dists),
            _ptr(grad_zbuf))
    del keep
    return grad_colors, grad_dists, grad_zbuf


def _depth_zfar_arg(dev, zfar):
    """(zfar ptr, zfar value, tensor to keep alive).  A 1-element float32 tensor on `dev` is read on the device; a
    Python number goes to the kernel as a number."""
    if torch.is_tensor(zfar):
        if zfar.device != dev or zfar.dtype != F32 or zfar.numel() != 1:
            raise RuntimeError("zfar must be a number or a 1-element float32 tensor on %s" % dev)
        z = zfar.reshape(1).contiguous()
        return z.data_ptr(), 0.0, z
    return None, float(zfar), None


def _check_depth_inputs(pix_to_face, named_floats, grad_out=None):
    """(N, H, W, K, device) of pix_to_face and the float32 (N, H, W, K) tensors `named_floats`, and of the float32
    (N, H, W, 1) grad_out when given."""
    dev = _require_cuda(*([("grad_out", grad_out)] if grad_out is not None else []), *named_floats,
                        ("pix_to_face", pix_to_face))
    shape = _check_index(pix_to_face)
    for name, t in named_floats:
        _check_float(name, t, shape, "N, H, W, K")
    if grad_out is not None:
        _check_float("grad_out", grad_out, shape[:3] + (1,), "N, H, W, 1")
    if not 1 <= shape[3] <= kMaxPointsPerPixel:
        raise RuntimeError("Must have 1 <= faces_per_pixel <= %d" % kMaxPointsPerPixel)
    return shape + (dev,)


def soft_depth_blend(pix_to_face: torch.Tensor, zbuf: torch.Tensor, dists: torch.Tensor, sigma: float, zfar):
    """Fused SoftDepthShader of pytorch3d/renderer/mesh/shader.py on the rasterizer's layout (no counterpart in
    pytorch3d._C): pix_to_face (N,H,W,K) i64, zbuf / dists (N,H,W,K) f32, 1 <= K <= 150; zfar a number or a 1-element
    float32 tensor on the same device -> (N,H,W,1) f32."""
    N, H, W, K, dev = _check_depth_inputs(pix_to_face, [("zbuf", zbuf), ("dists", dists)])
    zf_ptr, zf, keep = _depth_zfar_arg(dev, zfar)
    p2f, zb, dd = pix_to_face.contiguous(), zbuf.contiguous(), dists.contiguous()
    out = torch.empty((N, H, W, 1), dtype=F32, device=dev)
    if out.numel() == 0:
        return out
    _launch(dev, "soft_depth_blend_forward", _ptr(p2f), _ptr(zb), _ptr(dd), N, H, W, K, float(sigma), zf_ptr, zf,
            _ptr(out))
    del keep
    return out


def soft_depth_blend_backward(grad_out: torch.Tensor, pix_to_face: torch.Tensor, zbuf: torch.Tensor,
                              dists: torch.Tensor, sigma: float, zfar):
    """Backward of `soft_depth_blend` -> (grad_zbuf (N,H,W,K), grad_dists (N,H,W,K))."""
    N, H, W, K, dev = _check_depth_inputs(pix_to_face, [("zbuf", zbuf), ("dists", dists)], grad_out)
    zf_ptr, zf, keep = _depth_zfar_arg(dev, zfar)
    go, p2f, zb, dd = grad_out.contiguous(), pix_to_face.contiguous(), zbuf.contiguous(), dists.contiguous()
    grad_zbuf = torch.empty((N, H, W, K), dtype=F32, device=dev)
    grad_dists = torch.empty((N, H, W, K), dtype=F32, device=dev)
    if grad_zbuf.numel() == 0:
        return grad_zbuf, grad_dists
    _launch(dev, "soft_depth_blend_backward", _ptr(go), _ptr(p2f), _ptr(zb), _ptr(dd), N, H, W, K, float(sigma), zf_ptr,
            zf, _ptr(grad_zbuf), _ptr(grad_dists))
    del keep
    return grad_zbuf, grad_dists


def hard_depth(pix_to_face: torch.Tensor, zbuf: torch.Tensor, zfar):
    """Fused HardDepthShader of pytorch3d/renderer/mesh/shader.py: zbuf of slot 0 where pix_to_face of slot 0 is valid,
    zfar elsewhere.  pix_to_face (N,H,W,K) i64, zbuf (N,H,W,K) f32; zfar as for `soft_depth_blend` -> (N,H,W,1) f32."""
    N, H, W, K, dev = _check_depth_inputs(pix_to_face, [("zbuf", zbuf)])
    zf_ptr, zf, keep = _depth_zfar_arg(dev, zfar)
    p2f, zb = pix_to_face.contiguous(), zbuf.contiguous()
    out = torch.empty((N, H, W, 1), dtype=F32, device=dev)
    if out.numel() == 0:
        return out
    _launch(dev, "hard_depth_forward", _ptr(p2f), _ptr(zb), N, H, W, K, zf_ptr, zf, _ptr(out))
    del keep
    return out


def hard_depth_backward(grad_out: torch.Tensor, pix_to_face: torch.Tensor):
    """Backward of `hard_depth` -> grad_zbuf (N,H,W,K): grad_out on slot 0 of valid pixels, 0 everywhere else."""
    N, H, W, K, dev = _check_depth_inputs(pix_to_face, [], grad_out)
    go, p2f = grad_out.contiguous(), pix_to_face.contiguous()
    grad_zbuf = torch.empty((N, H, W, K), dtype=F32, device=dev)
    if grad_zbuf.numel() == 0:
        return grad_zbuf
    _launch(dev, "hard_depth_backward", _ptr(go), _ptr(p2f), N, H, W, K, _ptr(grad_zbuf))
    return grad_zbuf


def _check_splatter_inputs(colors, pixel_coords_screen, background_mask, sigma, grad_out=None):
    dev = _require_cuda(*([("grad_out", grad_out)] if grad_out is not None else []), ("colors", colors),
                        ("pixel_coords_screen", pixel_coords_screen), ("background_mask", background_mask))
    shape = _check_index(background_mask, "background_mask", torch.bool)
    _check_float("colors", colors, shape + (3,), "N, H, W, K, 3")
    _check_float("pixel_coords_screen", pixel_coords_screen, shape + (3,), "N, H, W, K, 3")
    if grad_out is not None:
        _check_float("grad_out", grad_out, shape[:3] + (4,), "N, H, W, 4")
    if shape[3] > kMaxPointsPerPixel:
        raise RuntimeError("Must have faces_per_pixel <= %d" % kMaxPointsPerPixel)
    if shape[3] < 1:
        raise RuntimeError("faces_per_pixel must be at least 1")
    if not float(sigma) > 0.0:
        raise RuntimeError("Only positive standard deviations make sense.")
    return shape + (dev,)


def splatter_blend(colors: torch.Tensor, pixel_coords_screen: torch.Tensor, background_mask: torch.Tensor,
                   sigma: float, background_color):
    """Fused splatter blend (the blend of pytorch3d.renderer.splatter_blend.SplatterBlender after its projection step;
    no counterpart in pytorch3d._C): colors and pixel_coords_screen (N,H,W,K,3) f32, background_mask (N,H,W,K) bool,
    sigma > 0 in pixels; background_color a float32 CUDA tensor of 3 values or 3 numbers -> (N,H,W,4) f32 RGBA."""
    N, H, W, K, dev = _check_splatter_inputs(colors, pixel_coords_screen, background_mask, sigma)
    bg_ptr, bg_val, _, _, _, _, keep = _softmax_side_args(dev, N, background_color, 1.0, 100.0)
    c, xyz, m = colors.contiguous(), pixel_coords_screen.contiguous(), background_mask.contiguous()
    out = torch.empty((N, H, W, 4), dtype=F32, device=dev)
    if out.numel() == 0:
        return out
    _launch(dev, "splatter_blend_forward", _ptr(c), _ptr(xyz), _ptr(m), N, H, W, K, float(sigma), bg_ptr, bg_val,
            _ptr(out))
    del keep
    return out


def splatter_blend_backward(grad_out: torch.Tensor, colors: torch.Tensor, pixel_coords_screen: torch.Tensor,
                            background_mask: torch.Tensor, sigma: float, background_color):
    """Backward of `splatter_blend` -> (grad_colors (N,H,W,K,3), grad_pixel_coords_screen (N,H,W,K,3)); both are 0 in
    background slots, and the z channel of grad_pixel_coords_screen is 0."""
    N, H, W, K, dev = _check_splatter_inputs(colors, pixel_coords_screen, background_mask, sigma, grad_out)
    bg_ptr, bg_val, _, _, _, _, keep = _softmax_side_args(dev, N, background_color, 1.0, 100.0)
    go = grad_out.contiguous()
    c, xyz, m = colors.contiguous(), pixel_coords_screen.contiguous(), background_mask.contiguous()
    grad_colors = torch.empty((N, H, W, K, 3), dtype=F32, device=dev)
    grad_xyz = torch.empty((N, H, W, K, 3), dtype=F32, device=dev)
    if grad_colors.numel() == 0:
        return grad_colors, grad_xyz
    ws, ws_bytes = _workspace(dev, "splatter_blend", N, H, W)
    _launch(dev, "splatter_blend_backward", _ptr(go), _ptr(c), _ptr(xyz), _ptr(m), N, H, W, K, float(sigma), bg_ptr,
            bg_val, _ptr(ws), ws_bytes, _ptr(grad_colors), _ptr(grad_xyz))
    del keep
    return grad_colors, grad_xyz


SHADING_PARAMS = 22  # B200R_SHADING_PARAMS: the per-image parameter row of the shading ops
LIGHT_KINDS = {"point": 0, "directional": 1, "ambient": 2}  # B200R_LIGHT_*


def _check_shading_inputs(pix_to_face, barycentric_coords, face_positions, face_normals, texels, params, flat, light,
                          grads=()):
    """(N, H, W, K, F, device); raises RuntimeError naming the argument for anything the kernels cannot take.  `grads`
    are the (name, tensor) upstream gradients, float32 (N, H, W, K, 3) or None."""
    if light not in LIGHT_KINDS:
        raise RuntimeError("light must be one of %s, got %r" % (sorted(LIGHT_KINDS), light))
    if light != "ambient" and face_normals is None:
        raise RuntimeError("face_normals are required for %s light" % light)
    if not flat and barycentric_coords is None:
        raise RuntimeError("barycentric_coords are required for phong shading")
    grads = [(name, t) for name, t in grads if t is not None]
    floats = [("texels", texels), ("params", params), ("face_positions", face_positions)]
    if not flat:
        floats.append(("barycentric_coords", barycentric_coords))
    if light != "ambient":
        floats.append(("face_normals", face_normals))
    dev = _require_cuda(*grads, *floats, ("pix_to_face", pix_to_face))
    shape = _check_index(pix_to_face)
    _check_float("texels", texels, shape + (3,), "N, H, W, K, 3")
    if not flat:
        _check_float("barycentric_coords", barycentric_coords, shape + (3,), "N, H, W, K, 3")
    face_shape = (3,) if flat else (3, 3)
    face_dims = "F, 3" if flat else "F, 3, 3"
    _check_float("face_positions", face_positions, (None,) + face_shape, face_dims)
    F = int(face_positions.shape[0])
    if light != "ambient":
        _check_float("face_normals", face_normals, (F,) + face_shape, face_dims)
    _check_float("params", params, (shape[0], SHADING_PARAMS), "N, %d" % SHADING_PARAMS)
    for name, t in grads:
        _check_float(name, t, shape + (3,), "N, H, W, K, 3")
    return shape + (F, dev)


def shading_forward(pix_to_face: torch.Tensor, barycentric_coords, face_positions: torch.Tensor, face_normals,
                    texels: torch.Tensor, params: torch.Tensor, flat: bool, light: str, return_positions: bool = False):
    """Fused Phong (flat=False) or flat shading (no counterpart in pytorch3d._C; DESIGN.md section 12): pix_to_face
    (N,H,W,K) i64; barycentric_coords (N,H,W,K,3) f32 (phong only); face_positions / face_normals (F,3,3) f32 (phong)
    or (F,3) (flat), face_normals unused (may be None) for ambient light; texels (N,H,W,K,3) f32; params (N,22) f32 (the
    row of include/b200_raster.h); light "point", "directional" or "ambient".
    -> (colors (N,H,W,K,3), positions (N,H,W,K,3) or None)."""
    N, H, W, K, F, dev = _check_shading_inputs(pix_to_face, barycentric_coords, face_positions, face_normals, texels,
                                               params, flat, light)
    p2f, tx, prm, fp = pix_to_face.contiguous(), texels.contiguous(), params.contiguous(), face_positions.contiguous()
    bary = None if flat else barycentric_coords.contiguous()
    fn = None if light == "ambient" else face_normals.contiguous()
    colors = torch.empty((N, H, W, K, 3), dtype=F32, device=dev)
    positions = torch.empty((N, H, W, K, 3), dtype=F32, device=dev) if return_positions else None
    if colors.numel() == 0:
        return colors, positions
    _launch(dev, "shading_forward", _ptr(p2f), _ptr(bary), _ptr(fp), _ptr(fn), F, _ptr(tx), _ptr(prm), N, H, W, K,
            int(bool(flat)), LIGHT_KINDS[light], _ptr(colors), _ptr(positions))
    return colors, positions


def _outputs(dev, *wanted):
    """float32 tensors of the (flag, shape) pairs `wanted`, None where the flag is false."""
    return [torch.empty(shape, dtype=F32, device=dev) if flag else None for flag, shape in wanted]


def shading_backward(grad_colors: torch.Tensor, grad_positions, pix_to_face: torch.Tensor, barycentric_coords,
                     face_positions: torch.Tensor, face_normals, texels: torch.Tensor, params: torch.Tensor, flat: bool,
                     light: str, needs_input_grad=(True, True, True, True, True)):
    """Backward of `shading_forward` -> (grad_texels, grad_barycentric_coords, grad_face_positions, grad_face_normals,
    grad_params); an entry is None where `needs_input_grad` (same order) is false, and grad_barycentric_coords is None
    in flat mode.  grad_params is deterministic; the two face gradients are accumulated with atomics."""
    N, H, W, K, F, dev = _check_shading_inputs(pix_to_face, barycentric_coords, face_positions, face_normals, texels,
                                               params, flat, light,
                                               (("grad_colors", grad_colors), ("grad_positions", grad_positions)))
    shape = (N, H, W, K, 3)
    need_tx, need_bary, need_fp, need_fn, need_prm = (bool(v) for v in needs_input_grad)
    need_bary = need_bary and not flat
    need_fn = need_fn and face_normals is not None
    gc, p2f, tx, prm = grad_colors.contiguous(), pix_to_face.contiguous(), texels.contiguous(), params.contiguous()
    gp, fp = _c(grad_positions), face_positions.contiguous()
    bary = None if flat else barycentric_coords.contiguous()
    fn = None if light == "ambient" else face_normals.contiguous()
    g_tx, g_bary, g_fp, g_fn, g_prm = _outputs(
        dev, (need_tx, shape), (need_bary, shape), (need_fp, tuple(face_positions.shape)),
        (need_fn, tuple(face_normals.shape) if need_fn else None), (need_prm, (N, SHADING_PARAMS)))
    ws, ws_bytes = _workspace(dev, "shading", N, H, W, K) if need_prm else (None, 0)
    _launch(dev, "shading_backward", _ptr(gc), _ptr(gp), _ptr(p2f), _ptr(bary), _ptr(fp), _ptr(fn), F, _ptr(tx),
            _ptr(prm), N, H, W, K, int(bool(flat)), LIGHT_KINDS[light], _ptr(ws), ws_bytes, _ptr(g_tx), _ptr(g_bary),
            _ptr(g_fp), _ptr(g_fn), _ptr(g_prm))
    if N * H * W * K == 0:  # nothing was launched: the outputs the kernels would have written
        for t in (g_tx, g_bary):
            if t is not None:
                t.zero_()
    return g_tx, g_bary, g_fp, g_fn, g_prm


def _check_gouraud_inputs(verts, normals, verts_colors, mesh_first_vert, mesh_num_verts, params, faces, pix_to_face,
                          barycentric_coords, light, grads=()):
    """(V, F, meshes, device); raises RuntimeError naming the argument for anything the kernels cannot take.  `grads`
    are the backward's (name, tensor, shape, dims) extra float32 inputs."""
    if light not in LIGHT_KINDS:
        raise RuntimeError("light must be one of %s, got %r" % (sorted(LIGHT_KINDS), light))
    if light != "ambient" and normals is None:
        raise RuntimeError("normals are required for %s light" % light)
    floats = [("verts", verts), ("verts_colors", verts_colors), ("params", params),
              ("barycentric_coords", barycentric_coords)] + ([("normals", normals)] if normals is not None else [])
    V, F, dev = _check_verts_faces(None, verts, faces, *[g[:2] for g in grads], *floats[1:],
                                   ("mesh_first_vert", mesh_first_vert), ("mesh_num_verts", mesh_num_verts),
                                   ("pix_to_face", pix_to_face))
    for name, t in (("verts_colors", verts_colors), ("normals", normals)):
        if t is not None:
            _check_float(name, t, (V, 3), "V, 3")
    meshes = _check_ranges(None, "mesh_first_vert", mesh_first_vert, "mesh_num_verts", mesh_num_verts)
    if meshes > 65535:
        raise RuntimeError("at most 65535 meshes per call, got %d" % meshes)
    _check_float("params", params, (meshes, SHADING_PARAMS), "meshes, %d" % SHADING_PARAMS)
    shape = _check_index(pix_to_face)
    _check_float("barycentric_coords", barycentric_coords, shape + (3,), "N, H, W, K, 3")
    for name, t, g_shape, dims in grads:
        _check_float(name, t, g_shape, dims)
    return V, F, meshes, dev


def gouraud_forward(verts: torch.Tensor, normals, verts_colors: torch.Tensor, mesh_first_vert: torch.Tensor,
                    mesh_num_verts: torch.Tensor, params: torch.Tensor, faces: torch.Tensor, pix_to_face: torch.Tensor,
                    barycentric_coords: torch.Tensor, light: str):
    """Fused Gouraud shading (no counterpart in pytorch3d._C; DESIGN.md section 16): verts, normals (None for ambient
    light), verts_colors (V,3) f32 packed; mesh_first_vert, mesh_num_verts (meshes,) i64; params (meshes,22) f32, one
    row per mesh; faces (F,3) i64 packed; pix_to_face (N,H,W,K) i64; barycentric_coords (N,H,W,K,3) f32; light
    "point", "directional" or "ambient".  -> (colors (N,H,W,K,3), verts_shaded (V,3))."""
    V, F, meshes, dev = _check_gouraud_inputs(verts, normals, verts_colors, mesh_first_vert, mesh_num_verts, params,
                                              faces, pix_to_face, barycentric_coords, light)
    P = pix_to_face.numel()
    v, vc, prm, fc = verts.contiguous(), verts_colors.contiguous(), params.contiguous(), faces.contiguous()
    nrm = None if light == "ambient" else normals.contiguous()
    first, num = mesh_first_vert.contiguous(), mesh_num_verts.contiguous()
    p2f, bary = pix_to_face.contiguous(), barycentric_coords.contiguous()
    shaded = torch.empty((V, 3), dtype=F32, device=dev)
    colors = torch.empty(tuple(pix_to_face.shape) + (3,), dtype=F32, device=dev)
    _launch(dev, "gouraud_forward", _ptr(v), _ptr(nrm), _ptr(vc), V, _ptr(first), _ptr(num), meshes, _ptr(prm),
            _ptr(fc), F, _ptr(p2f), _ptr(bary), P, LIGHT_KINDS[light], _ptr(shaded), _ptr(colors))
    return colors, shaded


def gouraud_backward(grad_colors: torch.Tensor, verts: torch.Tensor, normals, verts_colors: torch.Tensor,
                     mesh_first_vert: torch.Tensor, mesh_num_verts: torch.Tensor, params: torch.Tensor,
                     faces: torch.Tensor, pix_to_face: torch.Tensor, barycentric_coords: torch.Tensor, light: str,
                     verts_shaded: torch.Tensor, needs_input_grad=(True, True, True, True, True)):
    """Backward of `gouraud_forward` -> (grad_verts, grad_normals, grad_verts_colors, grad_barycentric_coords,
    grad_params); an entry is None where `needs_input_grad` (same order) is false.  grad_barycentric_coords is
    deterministic; the other four start from a per-vertex sum accumulated with atomics, so requesting them under
    torch.use_deterministic_algorithms(True) raises, as the reference's interpolation backward does."""
    grads = (("grad_colors", grad_colors, tuple(pix_to_face.shape) + (3,), "N, H, W, K, 3"),
             ("verts_shaded", verts_shaded, tuple(verts.shape), "V, 3"))
    V, F, meshes, dev = _check_gouraud_inputs(verts, normals, verts_colors, mesh_first_vert, mesh_num_verts, params,
                                              faces, pix_to_face, barycentric_coords, light, grads)
    need_v, need_n, need_vc, need_bary, need_prm = (bool(x) for x in needs_input_grad)
    need_n = need_n and normals is not None
    need_vertex = need_v or need_n or need_vc or need_prm
    if need_vertex:
        _refuse_nondeterministic("gouraud_backward",
                                 "the gradient of the shaded vertex colours is accumulated with atomics")
    P = pix_to_face.numel()
    gc, v, vc, prm = grad_colors.contiguous(), verts.contiguous(), verts_colors.contiguous(), params.contiguous()
    nrm = None if light == "ambient" else normals.contiguous()
    first, num, fc = mesh_first_vert.contiguous(), mesh_num_verts.contiguous(), faces.contiguous()
    p2f, bary, shaded = pix_to_face.contiguous(), barycentric_coords.contiguous(), verts_shaded.contiguous()
    g_v, g_n, g_vc, g_bary, g_prm = _outputs(dev, (need_v, (V, 3)), (need_n, (V, 3)), (need_vc, (V, 3)),
                                             (need_bary, tuple(barycentric_coords.shape)),
                                             (need_prm, (meshes, SHADING_PARAMS)))
    ws, ws_bytes = _workspace(dev, "gouraud", meshes, V) if need_vertex else (None, 0)
    _launch(dev, "gouraud_backward", _ptr(gc), _ptr(v), _ptr(nrm), _ptr(vc), V, _ptr(first), _ptr(num), meshes,
            _ptr(prm), _ptr(fc), F, _ptr(p2f), _ptr(bary), P, LIGHT_KINDS[light], _ptr(shaded), _ptr(ws), ws_bytes,
            _ptr(g_v), _ptr(g_n), _ptr(g_vc), _ptr(g_bary), _ptr(g_prm))
    return g_v, g_n, g_vc, g_bary, g_prm


SAMPLING_MODES = {"bilinear": 0, "nearest": 1}  # B200R_SAMPLE_*: torch's GridSamplerInterpolation
PADDING_MODES = {"zeros": 0, "border": 1, "reflection": 2}  # B200R_PAD_*: torch's GridSamplerPadding


def _check_texture_inputs(pix_to_face, barycentric_coords, face_uvs, maps, sampling_mode, padding_mode,
                          grad_texels=None):
    """(N, H, W, K, H_in, W_in, C, device); raises RuntimeError naming the argument for anything the kernels cannot
    take, and ValueError when the maps' batch is not the Fragments' N.  Shapes are checked before devices and dtypes,
    so that a CPU caller learns about a wrong shape first."""
    if sampling_mode not in SAMPLING_MODES:
        raise RuntimeError("sampling_mode must be one of %s, got %r" % (sorted(SAMPLING_MODES), sampling_mode))
    if padding_mode not in PADDING_MODES:
        raise RuntimeError("padding_mode must be one of %s, got %r" % (sorted(PADDING_MODES), padding_mode))
    shape = _check_index(pix_to_face, dtype=None)
    _check_tensor("barycentric_coords", barycentric_coords, None, shape + (3,), "N, H, W, K, 3")
    _check_tensor("face_uvs", face_uvs, None, (None, 3, 2), "F, 3, 2")
    _check_tensor("maps", maps, None, (None,) * 4, "N, H_in, W_in, C")
    if min(maps.shape[1:]) < 1:
        raise RuntimeError("maps must be (N, H_in, W_in, C) with H_in, W_in, C >= 1, got %s" % (tuple(maps.shape),))
    if maps.shape[0] != shape[0]:
        raise ValueError("maps must have one map per image: maps has batch %d, the Fragments have N = %d"
                         % (maps.shape[0], shape[0]))
    H_in, W_in, C = (int(v) for v in maps.shape[1:])
    floats = [("barycentric_coords", barycentric_coords), ("face_uvs", face_uvs), ("maps", maps)]
    if grad_texels is not None:
        _check_tensor("grad_texels", grad_texels, None, shape + (C,), "N, H, W, K, C")
        floats.insert(0, ("grad_texels", grad_texels))
    return shape + (H_in, W_in, C, _check_texture_devices(pix_to_face, floats))


def _check_texture_devices(pix_to_face, floats):
    """The device of pix_to_face and the (name, tensor) `floats`, after their shapes: then their dtypes."""
    dev = _require_cuda(*floats, ("pix_to_face", pix_to_face))
    _check_tensor("pix_to_face", pix_to_face, I64)
    for name, t in floats:
        _check_float(name, t)
    return dev


def texture_uv_forward(pix_to_face: torch.Tensor, barycentric_coords: torch.Tensor, face_uvs: torch.Tensor,
                       maps: torch.Tensor, sampling_mode: str = "bilinear", padding_mode: str = "border",
                       align_corners: bool = True):
    """Fused TexturesUV.sample_textures for one map per image (no counterpart in pytorch3d._C; DESIGN.md section 13):
    pix_to_face (N,H,W,K) i64, barycentric_coords (N,H,W,K,3) f32, face_uvs (F,3,2) f32, maps (N,H_in,W_in,C) f32
    (channel last, read in place when contiguous) -> texels (N,H,W,K,C) f32, contiguous."""
    N, H, W, K, H_in, W_in, C, dev = _check_texture_inputs(pix_to_face, barycentric_coords, face_uvs, maps,
                                                           sampling_mode, padding_mode)
    F = int(face_uvs.shape[0])
    p2f, bary, fuv, m = pix_to_face.contiguous(), barycentric_coords.contiguous(), face_uvs.contiguous(), maps.contiguous()
    texels = torch.empty((N, H, W, K, C), dtype=F32, device=dev)
    if texels.numel() == 0:
        return texels
    _launch(dev, "texture_uv_forward", _ptr(p2f), _ptr(bary), _ptr(fuv), F, _ptr(m), N, H, W, K, H_in, W_in, C,
            SAMPLING_MODES[sampling_mode], PADDING_MODES[padding_mode], int(bool(align_corners)), _ptr(texels))
    return texels


def texture_uv_backward(grad_texels: torch.Tensor, pix_to_face: torch.Tensor, barycentric_coords: torch.Tensor,
                        face_uvs: torch.Tensor, maps: torch.Tensor, sampling_mode: str = "bilinear",
                        padding_mode: str = "border", align_corners: bool = True, needs_input_grad=(True, True, True)):
    """Backward of `texture_uv_forward` -> (grad_maps (N,H_in,W_in,C), grad_barycentric_coords (N,H,W,K,3),
    grad_face_uvs (F,3,2)); an entry is None where `needs_input_grad` (same order) is false.  grad_barycentric_coords is
    deterministic; the other two are accumulated with atomics, so requesting them under
    torch.use_deterministic_algorithms(True) raises, as torch's grid sampler backward does."""
    N, H, W, K, H_in, W_in, C, dev = _check_texture_inputs(pix_to_face, barycentric_coords, face_uvs, maps,
                                                           sampling_mode, padding_mode, grad_texels)
    need_maps, need_bary, need_fuv = (bool(v) for v in needs_input_grad)
    if need_maps or need_fuv:
        _refuse_nondeterministic("texture_uv_backward", "grad_maps and grad_face_uvs are accumulated with atomics")
    F = int(face_uvs.shape[0])
    go = grad_texels.contiguous()
    p2f, bary, fuv, m = pix_to_face.contiguous(), barycentric_coords.contiguous(), face_uvs.contiguous(), maps.contiguous()
    g_maps, g_bary, g_fuv = _outputs(dev, (need_maps, (N, H_in, W_in, C)), (need_bary, (N, H, W, K, 3)),
                                     (need_fuv, (F, 3, 2)))
    _launch(dev, "texture_uv_backward", _ptr(go), _ptr(p2f), _ptr(bary), _ptr(fuv), F, _ptr(m), N, H, W, K, H_in, W_in,
            C, SAMPLING_MODES[sampling_mode], PADDING_MODES[padding_mode], int(bool(align_corners)), _ptr(g_maps),
            _ptr(g_bary), _ptr(g_fuv))
    return g_maps, g_bary, g_fuv


def texture_atlas_key_bits(F: int, R: int):
    """(key bits, key bytes) of the backward's sort for an (F, R, R, C) atlas: the cells and the sentinel F·R² need
    ceil(log2(F·R² + 1)) bits; keys are 32-bit below 2³² cells and 64-bit from there (b200r_texture_atlas_backward)."""
    bits = max(1, (int(F) * int(R) * int(R)).bit_length())
    return bits, 4 if bits <= 32 else 8


def _check_atlas_inputs(pix_to_face, barycentric_coords, atlas, grad_texels=None):
    """(N, H, W, K, F, R, C, device); raises RuntimeError naming the argument for anything the kernels cannot take.
    Shapes are checked before devices and dtypes, as for the UV textures."""
    shape = _check_index(pix_to_face, dtype=None)
    _check_tensor("barycentric_coords", barycentric_coords, None, shape + (3,), "N, H, W, K, 3")
    _check_tensor("atlas", atlas, None, (None,) * 4, "F, R, R, C")
    if atlas.shape[1] != atlas.shape[2] or atlas.shape[1] < 1 or atlas.shape[3] < 1:
        raise RuntimeError("atlas must be (F, R, R, C) with R, C >= 1, got %s" % (tuple(atlas.shape),))
    F, R, _, C = (int(v) for v in atlas.shape)
    floats = [("barycentric_coords", barycentric_coords), ("atlas", atlas)]
    if grad_texels is not None:
        _check_tensor("grad_texels", grad_texels, None, shape + (C,), "N, H, W, K, C")
        floats.insert(0, ("grad_texels", grad_texels))
    return shape + (F, R, C, _check_texture_devices(pix_to_face, floats))


def texture_atlas_forward(pix_to_face: torch.Tensor, barycentric_coords: torch.Tensor, atlas: torch.Tensor):
    """Fused TexturesAtlas.sample_textures (no counterpart in pytorch3d._C; DESIGN.md section 15): pix_to_face
    (N,H,W,K) i64, barycentric_coords (N,H,W,K,3) f32, atlas (F,R,R,C) f32, the packed atlas (read in place when
    contiguous) -> texels (N,H,W,K,C) f32, contiguous.  Slots whose cell the reference cannot index (it raises) get 0."""
    N, H, W, K, F, R, C, dev = _check_atlas_inputs(pix_to_face, barycentric_coords, atlas)
    p2f, bary, a = pix_to_face.contiguous(), barycentric_coords.contiguous(), atlas.contiguous()
    texels = torch.empty((N, H, W, K, C), dtype=F32, device=dev)
    if texels.numel() == 0:
        return texels
    _launch(dev, "texture_atlas_forward", _ptr(p2f), _ptr(bary), _ptr(a), F, R, C, N, H, W, K, _ptr(texels))
    return texels


def texture_atlas_backward(grad_texels: torch.Tensor, pix_to_face: torch.Tensor, barycentric_coords: torch.Tensor,
                           atlas: torch.Tensor):
    """Backward of `texture_atlas_forward` -> grad_atlas (F,R,R,C) f32: each cell's sum of grad_texels ·
    float(pix_to_face >= 0) over the slots that read it, in ascending slot order.  Deterministic (a stable sort, no
    atomics), so it runs under torch.use_deterministic_algorithms(True); nothing synchronises the host."""
    N, H, W, K, F, R, C, dev = _check_atlas_inputs(pix_to_face, barycentric_coords, atlas, grad_texels)
    go, p2f, bary = grad_texels.contiguous(), pix_to_face.contiguous(), barycentric_coords.contiguous()
    grad_atlas = torch.empty((F, R, R, C), dtype=F32, device=dev)
    ws, ws_bytes = _workspace(dev, "texture_atlas", N, H, W, K, F, R)
    _launch(dev, "texture_atlas_backward", _ptr(go), _ptr(p2f), _ptr(bary), F, R, C, N, H, W, K, _ptr(ws), ws_bytes,
            _ptr(grad_atlas))
    return grad_atlas


def normals_key_bits(V: int):
    """The key bits of the vertex -> corner table's sort: vertex ids and the key V (faces out of range) need
    ceil(log2(V + 1)) bits, at least 1 (b200r_normals_workspace_bytes)."""
    return max(1, int(V).bit_length())


def normals_table_size(V: int, F: int):
    """Entries (int32) of the vertex -> corner table: V + 1 offsets, then the 3F corner ids."""
    return int(V) + 1 + 3 * int(F)


def normals_sizes_ok(V: int, F: int):
    """Whether the normal kernels take these sizes (b200r_normals_workspace_bytes)."""
    return V < (1 << 31) - 1 and 3 * F < (1 << 31)


def _check_normals_inputs(op, verts, faces, *named):
    """(V, F, device) of verts / faces on one CUDA device with the (name, tensor) pairs `named`, within the kernels'
    size limits."""
    V, F, dev = _check_verts_faces(op, verts, faces, *named)
    if not normals_sizes_ok(V, F):
        raise RuntimeError("%s: at most 2^31 - 2 vertices and (2^31 - 1) / 3 faces, got V = %d, F = %d" % (op, V, F))
    return V, F, dev


def face_areas_normals_forward(verts: torch.Tensor, faces: torch.Tensor):
    """pytorch3d._C.face_areas_normals_forward (FaceAreasNormalsForward, csrc/face_areas_normals/face_areas_normals.h)
    for float32: verts (V,3) f32, faces (F,3) i64 -> (areas (F,) f32, normals (F,3) f32), bit-identical to the
    reference's CUDA kernel."""
    V, F, dev = _check_normals_inputs("face_areas_normals_forward", verts, faces)
    v, f = verts.contiguous(), faces.contiguous()
    areas = torch.empty((F,), dtype=F32, device=dev)
    normals = torch.empty((F, 3), dtype=F32, device=dev)
    _launch(dev, "face_areas_normals_forward", _ptr(v), V, _ptr(f), F, _ptr(areas), _ptr(normals))
    return areas, normals


def face_areas_normals_backward(grad_areas: torch.Tensor, grad_normals: torch.Tensor, verts: torch.Tensor,
                                faces: torch.Tensor):
    """pytorch3d._C.face_areas_normals_backward (FaceAreasNormalsBackward) for float32 -> grad_verts (V,3) f32: the
    reference's per-corner gradients, summed per vertex in a fixed order.  Deterministic (no atomics), so unlike the
    reference it runs under torch.use_deterministic_algorithms(True)."""
    op = "face_areas_normals_backward"
    V, F, dev = _check_normals_inputs(op, verts, faces, ("grad_areas", grad_areas), ("grad_normals", grad_normals))
    _check_tensor("grad_areas", grad_areas, F32, (F,), "F,", op)
    _check_tensor("grad_normals", grad_normals, F32, (F, 3), "F, 3", op)
    ga, gn, v, f = grad_areas.contiguous(), grad_normals.contiguous(), verts.contiguous(), faces.contiguous()
    grad_verts = torch.empty((V, 3), dtype=F32, device=dev)
    ws, ws_bytes = _workspace(dev, "normals", V, F)
    _launch(dev, "face_areas_normals_backward", _ptr(ga), _ptr(gn), _ptr(v), V, _ptr(f), F, _ptr(ws), ws_bytes,
            _ptr(grad_verts))
    return grad_verts


def verts_normals_forward(verts: torch.Tensor, faces: torch.Tensor):
    """Fused Meshes._compute_vertex_normals (no counterpart in pytorch3d._C; DESIGN.md section 17): verts (V,3) f32,
    faces (F,3) i64 -> (normals (V,3) f32, table (V + 1 + 3F,) i32, sums (V,3) f32).  The normals are bit-identical to
    the reference's torch chain on the CPU; the table and the unnormalised sums are what `verts_normals_backward`
    reads."""
    V, F, dev = _check_normals_inputs("verts_normals_forward", verts, faces)
    v, f = verts.contiguous(), faces.contiguous()
    normals = torch.empty((V, 3), dtype=F32, device=dev)
    table = torch.empty((normals_table_size(V, F),), dtype=I32, device=dev)
    sums = torch.empty((V, 3), dtype=F32, device=dev)
    ws, ws_bytes = _workspace(dev, "normals", V, F)
    _launch(dev, "verts_normals_forward", _ptr(v), V, _ptr(f), F, _ptr(ws), ws_bytes, _ptr(table), _ptr(sums),
            _ptr(normals))
    return normals, table, sums


def verts_normals_backward(grad_normals: torch.Tensor, verts: torch.Tensor, faces: torch.Tensor, table: torch.Tensor,
                           sums: torch.Tensor):
    """Backward of `verts_normals_forward` -> grad_verts (V,3) f32, from the forward's table and sums (no sort).
    Deterministic, no atomics; nothing synchronises the host."""
    op = "verts_normals_backward"
    V, F, dev = _check_normals_inputs(op, verts, faces, ("grad_normals", grad_normals), ("sums", sums),
                                      ("table", table))
    _check_tensor("grad_normals", grad_normals, F32, (V, 3), "V, 3", op)
    _check_tensor("sums", sums, F32, (V, 3), "V, 3", op)
    _check_tensor("table", table, I32, (normals_table_size(V, F),), "V + 1 + 3F,", op)
    gn, v, f, t, s = (x.contiguous() for x in (grad_normals, verts, faces, table, sums))
    grad_verts = torch.empty((V, 3), dtype=F32, device=dev)
    ws, ws_bytes = _workspace(dev, "normals", V, F)
    _launch(dev, "verts_normals_backward", _ptr(gn), _ptr(v), V, _ptr(f), F, _ptr(t), _ptr(s), _ptr(ws), ws_bytes,
            _ptr(grad_verts))
    return grad_verts


# Bits of the status word of sample_points_forward (B200R_SAMPLE_*).
SAMPLE_HAS_VALID, SAMPLE_NONFINITE, SAMPLE_BAD_TOTAL, SAMPLE_HAS_EMPTY = 1, 2, 4, 8


def sampling_sizes_ok(V: int, F: int, N: int, S: int):
    """Whether the sampling kernels take these sizes (b200r_sample_points_forward)."""
    return V < (1 << 31) - 1 and 1 <= N < (1 << 31) and F // 4096 + N + 1 < (1 << 31) and 1 <= S <= (1 << 40) // N


def sample_points_forward(verts: torch.Tensor, faces: torch.Tensor, mesh_first_face: torch.Tensor,
                          mesh_num_faces: torch.Tensor, num_samples: int, return_normals: bool, seed: torch.Tensor):
    """Fused pytorch3d.ops.sample_points_from_meshes (DESIGN.md section 20): verts (V,3) f32, faces (F,3) i64 packed,
    the per-mesh face ranges (N,) i64 and a seed, two int64 on the device (their low 32 bits key the generator) ->
    (samples (N,S,3) f32, normals (N,S,3) f32 or None, face_idx (N,S) i64, bary (N,S,3) f32, status (1,) i32).  The
    status bits (SAMPLE_*) are on the device; nothing here synchronises the host."""
    return _sample_points(verts, faces, mesh_first_face, mesh_num_faces, num_samples, return_normals, seed, None)


def _sample_points_from_draws(verts: torch.Tensor, faces: torch.Tensor, mesh_first_face: torch.Tensor,
                              mesh_num_faces: torch.Tensor, return_normals: bool, face_idx: torch.Tensor,
                              u: torch.Tensor, v: torch.Tensor):
    """Test hook: `sample_points_forward` with the draws given -- face_idx (N,S) i64 packed faces, u and v (N,S) f32 --
    instead of drawn, so that the outputs can be compared bit for bit with the reference's for the same draws."""
    _check_tensor("face_idx", face_idx, I64, (None, None), "N, S")
    return _sample_points(verts, faces, mesh_first_face, mesh_num_faces, int(face_idx.shape[1]), return_normals, None,
                          (face_idx, u, v))


def _sample_points(verts, faces, mesh_first_face, mesh_num_faces, num_samples, return_normals, seed, draws):
    op = "sample_points_forward"
    extra = [("seed", seed)] if draws is None else list(zip(("face_idx", "u", "v"), draws))
    V, F, dev = _check_verts_faces(op, verts, faces, ("mesh_first_face", mesh_first_face),
                                   ("mesh_num_faces", mesh_num_faces), *extra)
    N = _check_ranges(op, "mesh_first_face", mesh_first_face, "mesh_num_faces", mesh_num_faces)
    S = int(num_samples)
    if draws is None:
        _check_tensor("seed", seed.reshape(-1), I64, (2,), "2,", op)
    else:
        for name, t, dtype in zip(("face_idx", "u", "v"), draws, (I64, F32, F32)):
            _check_tensor(name, t, dtype, (N, S), "N, S", op)
    if S < 1:
        raise RuntimeError("%s: num_samples must be at least 1, got %d" % (op, S))
    if not sampling_sizes_ok(V, F, N, S):
        raise RuntimeError("%s: at most 2^31 - 2 vertices, 1 to 2^31 - 1 meshes and 2^40 samples, got V = %d, F = %d, "
                           "N = %d, S = %d" % (op, V, F, N, S))
    v, f, first, num = verts.contiguous(), faces.contiguous(), mesh_first_face.contiguous(), mesh_num_faces.contiguous()
    sd = _c(seed)
    d_face, d_u, d_v = (t.contiguous() for t in draws) if draws is not None else (None, None, None)
    samples = torch.empty((N, S, 3), dtype=F32, device=dev)
    normals = torch.empty((N, S, 3), dtype=F32, device=dev) if return_normals else None
    face_idx = torch.empty((N, S), dtype=I64, device=dev)
    bary = torch.empty((N, S, 3), dtype=F32, device=dev)
    status = torch.empty((1,), dtype=I32, device=dev)
    ws, ws_bytes = _workspace(dev, "sample_points", V, F, N, S, 0, required=True)
    _launch(dev, "sample_points_forward", _ptr(v), V, _ptr(f), F, _ptr(first), _ptr(num), N, S, _ptr(sd), _ptr(d_face),
            _ptr(d_u), _ptr(d_v), _ptr(ws), ws_bytes, samples.data_ptr(), _ptr(normals), face_idx.data_ptr(),
            bary.data_ptr(), status.data_ptr())
    return samples, normals, face_idx, bary, status


def sample_points_backward(grad_samples: torch.Tensor, grad_normals, verts: torch.Tensor, faces: torch.Tensor,
                           face_idx: torch.Tensor, bary: torch.Tensor):
    """Backward of `sample_points_forward` -> grad_verts (V,3) f32, from the forward's face_idx and bary; grad_normals
    may be None.  Deterministic, no float atomics, no host synchronisation."""
    op = "sample_points_backward"
    grads = [("grad_samples", grad_samples)] + ([("grad_normals", grad_normals)] if grad_normals is not None else [])
    V, F, dev = _check_verts_faces(op, verts, faces, ("face_idx", face_idx), ("bary", bary), *grads)
    _check_tensor("face_idx", face_idx, I64, (None, None), "N, S", op)
    N, S = int(face_idx.shape[0]), int(face_idx.shape[1])
    for name, t in [("bary", bary)] + grads:
        _check_tensor(name, t, F32, (N, S, 3), "N, S, 3", op)
    if V >= (1 << 31) - 1 or 3 * N * S >= (1 << 31):
        raise RuntimeError("%s: at most 2^31 - 2 vertices and 3 N S < 2^31 sample corners, got V = %d, N = %d, S = %d"
                           % (op, V, N, S))
    gs, gn, v, f, fi, b = (_c(t) for t in (grad_samples, grad_normals, verts, faces, face_idx, bary))
    grad_verts = torch.empty((V, 3), dtype=F32, device=dev)
    ws, ws_bytes = _workspace(dev, "sample_points", V, F, N, S, 1, required=True)
    _launch(dev, "sample_points_backward", _ptr(gs), _ptr(gn), _ptr(v), V, _ptr(f), F, N, S, _ptr(fi), _ptr(b),
            _ptr(ws), ws_bytes, _ptr(grad_verts))
    return grad_verts


# Reductions and status bits of chamfer_forward (B200R_CHAMFER_*).
CHAMFER_POINT = {None: 0, "sum": 1, "mean": 2, "max": 3}
CHAMFER_BATCH = {None: 0, "sum": 1, "mean": 2}
CHAMFER_X_LENGTH, CHAMFER_Y_LENGTH, CHAMFER_W_NEGATIVE, CHAMFER_W_ZERO_SUM = 1, 2, 4, 8


def chamfer_sizes_ok(N: int, P1: int, P2: int):
    """Whether the chamfer kernels take these sizes (b200r_chamfer_forward): the backward's sort ids are int32."""
    return N >= 1 and P1 >= 1 and P2 >= 1 and 2 * (N * P1 + N * P2) < (1 << 31)


def _check_chamfer_inputs(op, x, y, x_lengths, y_lengths, x_normals, y_normals, weights):
    """(N, P1, P2, device): float32 x (N, P1, 3) and y (N, P2, 3), int64 (N,) lengths, float32 normals of the clouds'
    shapes and float32 (N,) weights, all on one CUDA device; raises RuntimeError otherwise."""
    dev = _require_cuda(*[(k, t) for k, t in (("x", x), ("y", y), ("x_lengths", x_lengths), ("y_lengths", y_lengths),
                                              ("x_normals", x_normals), ("y_normals", y_normals), ("weights", weights))
                          if t is not None])
    _check_tensor("x", x, F32, (None, None, 3), "N, P1, 3", op)
    N, P1 = int(x.shape[0]), int(x.shape[1])
    _check_tensor("y", y, F32, (N, None, 3), "N, P2, 3", op)
    P2 = int(y.shape[1])
    if (x_normals is None) != (y_normals is None):
        raise RuntimeError("%s: give both normals or neither" % op)
    for name, t, dtype, shape, dims in (("x_lengths", x_lengths, I64, (N,), "N,"),
                                        ("y_lengths", y_lengths, I64, (N,), "N,"),
                                        ("x_normals", x_normals, F32, (N, P1, 3), "N, P1, 3"),
                                        ("y_normals", y_normals, F32, (N, P2, 3), "N, P2, 3"),
                                        ("weights", weights, F32, (N,), "N,")):
        if t is not None:
            _check_tensor(name, t, dtype, shape, dims, op)
    if not chamfer_sizes_ok(N, P1, P2):
        raise RuntimeError("%s: takes N, P1, P2 >= 1 and 2 (N P1 + N P2) < 2^31, got N = %d, P1 = %d, P2 = %d"
                           % (op, N, P1, P2))
    return N, P1, P2, dev


def chamfer_forward(x, y, x_lengths, y_lengths, x_normals, y_normals, weights, norm: int, point_reduction,
                    batch_reduction, single_directional: bool, abs_cosine: bool):
    """Fused pytorch3d.loss.chamfer_distance for D = 3 (DESIGN.md section 21).  Returns (outputs, state, status):
    outputs (loss_x, loss_y, normals_x, normals_y) -- per-point terms for point_reduction None, else the loss and the
    normal loss in the first and third (None where absent); state (dist_x, idx_x, dist_y, idx_y, cloud, argmax) for
    the backward; status (1,) i32 with the CHAMFER_* bits on the device.  Nothing here synchronises the host."""
    N, P1, P2, dev = _check_chamfer_inputs("chamfer_forward", x, y, x_lengths, y_lengths, x_normals, y_normals,
                                           weights)
    if norm not in (1, 2):
        raise RuntimeError("chamfer_forward: norm must be 1 or 2")
    pr, br = CHAMFER_POINT[point_reduction], CHAMFER_BATCH[batch_reduction]
    if pr == 0 and br != 0:
        raise RuntimeError("chamfer_forward: batch_reduction must be None when point_reduction is None")
    x, y, xl, yl, xn, yn, w = (_c(t) for t in (x, y, x_lengths, y_lengths, x_normals, y_normals, weights))
    nrm = xn is not None
    f32 = dict(dtype=F32, device=dev)
    dist_x = torch.empty((N, P1), **f32)
    idx_x = torch.empty((N, P1), dtype=I32, device=dev)
    dist_y = torch.empty((N, P2), **f32) if not single_directional else None
    idx_y = torch.empty((N, P2), dtype=I32, device=dev) if not single_directional else None
    cloud = torch.empty((4 * N + 1,), **f32)
    argmax = torch.empty((2 * N,), dtype=I32, device=dev)
    status = torch.empty((1,), dtype=I32, device=dev)
    if pr == 0:
        out_x = torch.empty((N, P1), **f32)
        out_y = torch.empty((N, P2), **f32) if not single_directional else None
        out_nx = torch.empty((N, P1), **f32) if nrm else None
        out_ny = torch.empty((N, P2), **f32) if nrm and not single_directional else None
    else:
        shape = (N,) if br == 0 else ()
        out_x, out_y = torch.empty(shape, **f32), None
        out_nx, out_ny = (torch.empty(shape, **f32) if nrm else None), None
    ws, ws_bytes = _workspace(dev, "chamfer", N, P1, P2, 0, required=True)
    _launch(dev, "chamfer_forward", _ptr(x), _ptr(y), N, P1, P2, _ptr(xl), _ptr(yl), _ptr(xn), _ptr(yn), _ptr(w),
            int(norm), pr, br, int(bool(single_directional)), int(bool(abs_cosine)), _ptr(ws), ws_bytes, _ptr(dist_x),
            _ptr(idx_x), _ptr(dist_y), _ptr(idx_y), _ptr(cloud), _ptr(argmax), _ptr(out_x), _ptr(out_y),
            _ptr(out_nx), _ptr(out_ny), _ptr(status))
    return (out_x, out_y, out_nx, out_ny), (dist_x, idx_x, dist_y, idx_y, cloud, argmax), status


def chamfer_backward(x, y, x_lengths, y_lengths, x_normals, y_normals, weights, norm: int, point_reduction,
                     batch_reduction, single_directional: bool, abs_cosine: bool, state, grads, need_points: bool,
                     need_normals: bool):
    """Backward of `chamfer_forward`: grads (g_x, g_y, g_nx, g_ny) are the upstream gradients of its outputs (None
    for an output without one: zeros) -> (grad_x, grad_y, grad_x_normals, grad_y_normals), the pairs asked for by
    need_points / need_normals (None otherwise).  Deterministic, no float atomics, no host synchronisation."""
    op = "chamfer_backward"
    N, P1, P2, dev = _check_chamfer_inputs(op, x, y, x_lengths, y_lengths, x_normals, y_normals, weights)
    pr, br = CHAMFER_POINT[point_reduction], CHAMFER_BATCH[batch_reduction]
    _, idx_x, _, idx_y, cloud, argmax = state
    nrm = x_normals is not None
    need_normals = need_normals and nrm
    if not (need_points or need_normals):
        return None, None, None, None
    shapes = ((N, P1), (N, P2)) if pr == 0 else ((((N,) if br == 0 else ())),) * 2
    named = [("idx_x", idx_x, I32, (N, P1)), ("cloud", cloud, F32, (4 * N + 1,)), ("argmax", argmax, I32, (2 * N,))]
    if not single_directional:
        named.append(("idx_y", idx_y, I32, (N, P2)))
    g = []
    for k, (name, t) in enumerate(zip(("grad_loss_x", "grad_loss_y", "grad_normals_x", "grad_normals_y"), grads)):
        present = (k % 2 == 0 or pr == 0) and (k < 2 or nrm) and not (k % 2 == 1 and single_directional)
        if not present:
            g.append(None)
        elif t is None:
            g.append(torch.zeros(shapes[k % 2], dtype=F32, device=dev))
        else:
            g.append(t.to(F32).contiguous())
            named.append((name, g[-1], F32, shapes[k % 2]))
    _require_cuda(("x", x), *[n[:2] for n in named])
    for name, t, dtype, shape in named:
        _check_tensor(name, t, dtype, shape, None, op)
    x, y, xl, yl, xn, yn, w = (_c(t) for t in (x, y, x_lengths, y_lengths, x_normals, y_normals, weights))
    V = N * P1 + N * P2
    gp, gn = _outputs(dev, (need_points, (V, 3)), (need_normals, (V, 3)))
    ws, ws_bytes = _workspace(dev, "chamfer", N, P1, P2, 1, required=True)
    _launch(dev, "chamfer_backward", _ptr(x), _ptr(y), N, P1, P2, _ptr(xl), _ptr(yl), _ptr(xn), _ptr(yn), _ptr(w),
            int(norm), pr, br, int(bool(single_directional)), int(bool(abs_cosine)), _ptr(idx_x), _ptr(idx_y),
            _ptr(cloud), _ptr(argmax), _ptr(g[0]), _ptr(g[1]), _ptr(g[2]), _ptr(g[3]), _ptr(ws), ws_bytes, _ptr(gp),
            _ptr(gn))
    gx, gy = (gp[:N * P1].view(N, P1, 3), gp[N * P1:].view(N, P2, 3)) if gp is not None else (None, None)
    gnx, gny = (gn[:N * P1].view(N, P1, 3), gn[N * P1:].view(N, P2, 3)) if gn is not None else (None, None)
    return gx, gy, gnx, gny


def _chamfer_nn(x, y, x_lengths=None, y_lengths=None, norm: int = 2):
    """Test hook: the fused search alone -- (dist_x (N,P1) f32, idx_x (N,P1) i64, dist_y (N,P2) f32, idx_y (N,P2)
    i64), each point's nearest neighbour in the other cloud as the reference's knn_points(K=1) finds it."""
    _, state, _ = chamfer_forward(x, y, x_lengths, y_lengths, None, None, None, norm, None, None, False, True)
    return state[0], state[1].long(), state[2], state[3].long()


# ------------------------------------------- farthest point sampling and ball query (DESIGN.md section 22)

def fps_sizes_ok(P: int):
    """Whether the farthest-point-sampling kernel takes clouds of P points: its keys hold the index in 32 bits."""
    return 0 <= P < (1 << 31)


def ball_query_sizes_ok(N: int, P1: int, P2: int, K: int):
    """Whether the ball query kernels take these sizes: the backward's sort ids and keys are int32."""
    return min(N, P1, P2, K) >= 0 and N * P1 * K < (1 << 31) and N * P2 < (1 << 31)


def sample_farthest_points(points: torch.Tensor, lengths: torch.Tensor, K: torch.Tensor, start_idxs: torch.Tensor,
                           max_K_known: int = -1, cluster_size: int = 0):
    """pytorch3d._C.sample_farthest_points for D = 3: idx (N, max_K) int64 (DESIGN.md section 22).  max_K is
    max_K_known when it is positive, else max(K), which synchronises the host once.  cluster_size 0 lets the library
    choose the CTAs per cloud; 1 to 16 forces it (a test and timing hook)."""
    op = "sample_farthest_points"
    dev = _require_cuda(("points", points), ("lengths", lengths), ("K", K), ("start_idxs", start_idxs))
    _check_tensor("points", points, F32, (None, None, 3), "N, P, 3", op)
    N, P = int(points.shape[0]), int(points.shape[1])
    if lengths.dim() != 1 or lengths.shape[0] != N:
        raise RuntimeError("Point and lengths must have the same batch dimension")
    if K.dim() != 1 or K.shape[0] != N:
        raise RuntimeError("Points and K must have the same batch dimension")
    for name, t in (("lengths", lengths), ("K", K), ("start_idxs", start_idxs)):
        _check_tensor(name, t, I64, (N,), "N,", op)
    if not fps_sizes_ok(P):
        raise RuntimeError("%s: takes P < 2^31, got P = %d" % (op, P))
    if not 0 <= int(cluster_size) <= 16:
        raise RuntimeError("%s: cluster_size must be 0 to 16" % op)
    max_K = int(max_K_known) if max_K_known > 0 else int(K.max())
    idx = torch.empty((N, max_K), dtype=I64, device=dev)
    if idx.numel() == 0:
        return idx
    if P == 0:  # FarthestPointSamplingCuda returns its -1 fill before any launch
        return idx.fill_(-1)
    points, lengths, K, start_idxs = (t.contiguous() for t in (points, lengths, K, start_idxs))
    scratch = torch.empty((N, P), dtype=F32, device=dev)
    _launch(dev, "sample_farthest_points", _ptr(points), N, P, _ptr(lengths), _ptr(K), _ptr(start_idxs), max_K,
            int(cluster_size), _ptr(scratch), _ptr(idx))
    return idx


def _check_ball_inputs(op, p1, p2, lengths1, lengths2, *named):
    """(N, P1, P2, device): float32 p1 (N, P1, 3) and p2 (N, P2, 3), int64 (N,) lengths (or None), and the (name,
    tensor, dtype, shape) entries of `named` with None standing for N, P1, all on one CUDA device."""
    dev = _require_cuda(*[(k, t) for k, t in (("p1", p1), ("p2", p2), ("lengths1", lengths1), ("lengths2", lengths2))
                          if t is not None], *[(k, t) for k, t, _, _ in named if t is not None])
    _check_tensor("p1", p1, F32, (None, None, 3), "N, P1, 3", op)
    N, P1 = int(p1.shape[0]), int(p1.shape[1])
    _check_tensor("p2", p2, F32, (N, None, 3), "N, P2, 3", op)
    for name, t in (("lengths1", lengths1), ("lengths2", lengths2)):
        if t is not None:
            _check_tensor(name, t, I64, (N,), "N,", op)
    for name, t, dtype, shape in named:
        if t is not None:
            _check_tensor(name, t, dtype, shape, None, op)
    return N, P1, int(p2.shape[1]), dev


def ball_query_forward(p1, p2, lengths1, lengths2, K: int, radius: float, skip_points_outside_cube: bool,
                       return_nn: bool):
    """Ball query for D = 3 (DESIGN.md section 22): (idx (N, P1, K) int64, dists (N, P1, K) float32, nn (N, P1, K, 3)
    float32 or None), idx and dists bit for bit the reference's BallQueryCuda, nn what masked_gather(p2, idx) gives.
    Lengths may be None (all P).  No host synchronisation."""
    op = "ball_query_forward"
    N, P1, P2, dev = _check_ball_inputs(op, p1, p2, lengths1, lengths2)
    K = int(K)
    if K < 0:
        raise RuntimeError("Trying to create tensor with negative dimension %d: [%d, %d, %d]" % (K, N, P1, K))
    if not ball_query_sizes_ok(N, P1, P2, K):
        raise RuntimeError("%s: takes N P1 K < 2^31 and N P2 < 2^31, got N = %d, P1 = %d, P2 = %d, K = %d"
                           % (op, N, P1, P2, K))
    p1, p2, l1, l2 = (_c(t) for t in (p1, p2, lengths1, lengths2))
    idx = torch.empty((N, P1, K), dtype=I64, device=dev)
    dists = torch.empty((N, P1, K), dtype=F32, device=dev)
    nn = torch.empty((N, P1, K, 3), dtype=F32, device=dev) if return_nn else None
    if idx.numel() > 0:
        _launch(dev, "ball_query_forward", _ptr(p1), _ptr(p2), N, P1, P2, _ptr(l1), _ptr(l2), K, float(radius),
                int(bool(skip_points_outside_cube)), _ptr(idx), _ptr(dists), _ptr(nn))
    return idx, dists, nn


def ball_query(p1, p2, lengths1, lengths2, K: int, radius: float, skip_points_outside_cube: bool):
    """pytorch3d._C.ball_query for D = 3: (idx, dists)."""
    idx, dists, _ = ball_query_forward(p1, p2, lengths1, lengths2, K, radius, skip_points_outside_cube, False)
    return idx, dists


def ball_query_backward(p1, p2, lengths1, lengths2, idx, grad_dists, grad_nn, need_p1: bool = True,
                        need_p2: bool = True):
    """Backward of `ball_query_forward` -> (grad_p1 (N, P1, 3), grad_p2 (N, P2, 3)), each None unless asked for.
    grad_dists (N, P1, K) and grad_nn (N, P1, K, 3) are the upstream gradients of dists and nn, either None.
    Deterministic, no float atomics, no host synchronisation."""
    op = "ball_query_backward"
    _check_tensor("idx", idx, I64, (None, None, None), "N, P1, K", op)
    N, P1, K = (int(v) for v in idx.shape)
    grad_dists = grad_dists.to(F32).contiguous() if grad_dists is not None else None
    grad_nn = grad_nn.to(F32).contiguous() if grad_nn is not None else None
    N, P1, P2, dev = _check_ball_inputs(op, p1, p2, lengths1, lengths2, ("idx", idx, I64, (N, P1, K)),
                                        ("grad_dists", grad_dists, F32, (N, P1, K)),
                                        ("grad_nn", grad_nn, F32, (N, P1, K, 3)))
    if not ball_query_sizes_ok(N, P1, P2, K):
        raise RuntimeError("%s: takes N P1 K < 2^31 and N P2 < 2^31, got N = %d, P1 = %d, P2 = %d, K = %d"
                           % (op, N, P1, P2, K))
    gp1, gp2 = _outputs(dev, (need_p1, (N, P1, 3)), (need_p2, (N, P2, 3)))
    if gp1 is None and gp2 is None:
        return None, None
    p1, p2, l1, l2, idx = (_c(t) for t in (p1, p2, lengths1, lengths2, idx))
    ws, ws_bytes = _workspace(dev, "ball_query", N, P1, P2, K) if gp2 is not None else (None, 0)
    _launch(dev, "ball_query_backward", _ptr(p1), _ptr(p2), N, P1, P2, _ptr(l1), _ptr(l2), K, _ptr(idx),
            _ptr(grad_dists), _ptr(grad_nn), _ptr(ws), ws_bytes, _ptr(gp1), _ptr(gp2))
    return gp1, gp2


LAPLACIAN_METHODS = {"uniform": 0, "cot": 1, "cotcurv": 2}  # B200R_LAPLACIAN_*


def regularizer_sizes_ok(V: int, F: int, N: int):
    """Whether the regulariser kernels take these sizes (b200r_regularizers_workspace_bytes)."""
    return V < (1 << 31) - 1 and 6 * F < (1 << 31) and 1 <= N < (1 << 31)


def _check_regularizer_inputs(op, verts, faces, mesh_first_vert, mesh_num_verts, *named):
    """(V, F, N, device) of verts / faces and the int64 (N,) per-mesh vertex ranges on one CUDA device with the (name,
    tensor) pairs `named`, within the kernels' size limits."""
    V, F, dev = _check_verts_faces(op, verts, faces, ("mesh_first_vert", mesh_first_vert),
                                   ("mesh_num_verts", mesh_num_verts), *named)
    N = _check_ranges(op, "mesh_first_vert", mesh_first_vert, "mesh_num_verts", mesh_num_verts)
    if not regularizer_sizes_ok(V, F, N):
        raise RuntimeError("%s: at most 2^31 - 2 vertices, (2^31 - 1) / 6 faces and 1 to 2^31 - 1 meshes, got V = %d, "
                           "F = %d, N = %d" % (op, V, F, N))
    return V, F, N, dev


def _check_regularizer_workspace(workspace, V, F, N, dev):
    """The bytes of the forward's workspace, which a backward hands back: uint8, contiguous, on dev, large enough."""
    ws_bytes = _workspace_size("regularizers", V, F, N)
    if not (workspace is None and ws_bytes == 0) and (
            workspace is None or not workspace.is_cuda or workspace.device != dev or workspace.dtype != torch.uint8
            or workspace.numel() < ws_bytes or not workspace.is_contiguous()):
        raise RuntimeError("workspace must be the uint8 workspace of the matching forward on %s" % dev)
    return ws_bytes


def mesh_edge_table(faces: torch.Tensor, V: int, mesh_first_vert: torch.Tensor, mesh_num_verts: torch.Tensor):
    """The edge table of the regularisers, for tests: faces (F,3) i64 with vertices in [0, V), the per-mesh vertex
    ranges -> (edges (E,2) i64, face_to_edge (F,3) i64, num_edges_per_mesh (N,) i64), PyTorch3D's edges_packed(),
    faces_packed_to_edges_packed() and num_edges_per_mesh().  Reads E on the host."""
    verts = torch.empty((int(V), 3), dtype=F32, device=faces.device) if faces.is_cuda else torch.empty((int(V), 3))
    V, F, N, dev = _check_regularizer_inputs("mesh_edge_table", verts, faces, mesh_first_vert, mesh_num_verts)
    f, first, num = faces.contiguous(), mesh_first_vert.contiguous(), mesh_num_verts.contiguous()
    edges = torch.empty((3 * F, 2), dtype=I64, device=dev)
    face_to_edge = torch.empty((F, 3), dtype=I64, device=dev)
    counts = torch.empty((N,), dtype=I64, device=dev)
    E = torch.empty((1,), dtype=I64, device=dev)
    ws, ws_bytes = _workspace(dev, "regularizers", V, F, N)
    _launch(dev, "mesh_edge_table", _ptr(f), V, F, _ptr(first), _ptr(num), N, _ptr(ws), ws_bytes, _ptr(edges),
            _ptr(face_to_edge), _ptr(counts), _ptr(E))
    return edges[:int(E.item())], face_to_edge, counts


def _regularizer_forward(name, verts, faces, mesh_first_vert, mesh_num_verts, *params):
    """(loss () f32, workspace) of the fused regulariser b200r_<name>."""
    V, F, N, dev = _check_regularizer_inputs(name, verts, faces, mesh_first_vert, mesh_num_verts)
    v, f, first, num = (t.contiguous() for t in (verts, faces, mesh_first_vert, mesh_num_verts))
    loss = torch.empty((), dtype=F32, device=dev)
    ws, ws_bytes = _workspace(dev, "regularizers", V, F, N)
    _launch(dev, name, _ptr(v), V, _ptr(f), F, _ptr(first), _ptr(num), N, *params, _ptr(ws), ws_bytes,
            loss.data_ptr())
    return loss, ws


def _regularizer_backward(name, grad_loss, verts, faces, mesh_first_vert, mesh_num_verts, workspace, *params):
    """grad_verts (V,3) f32 of the fused regulariser b200r_<name>, from the forward's workspace."""
    V, F, N, dev = _check_regularizer_inputs(name, verts, faces, mesh_first_vert, mesh_num_verts,
                                             ("grad_loss", grad_loss))
    _check_tensor("grad_loss", grad_loss.reshape(()) if grad_loss.numel() == 1 else grad_loss, F32, (), None, name)
    ws_bytes = _check_regularizer_workspace(workspace, V, F, N, dev)
    g, v, f, first, num = (t.contiguous() for t in (grad_loss, verts, faces, mesh_first_vert, mesh_num_verts))
    grad_verts = torch.empty((V, 3), dtype=F32, device=dev)
    _launch(dev, name, g.data_ptr(), _ptr(v), V, _ptr(f), F, _ptr(first), _ptr(num), N, *params, _ptr(workspace),
            ws_bytes, _ptr(grad_verts))
    return grad_verts


def mesh_edge_loss_forward(verts, faces, mesh_first_vert, mesh_num_verts, target_length: float):
    """Fused pytorch3d.loss.mesh_edge_loss (DESIGN.md section 18) -> (loss () f32, workspace): the workspace holds the
    tables `mesh_edge_loss_backward` reads."""
    return _regularizer_forward("mesh_edge_loss_forward", verts, faces, mesh_first_vert, mesh_num_verts,
                                float(target_length))


def mesh_edge_loss_backward(grad_loss, verts, faces, mesh_first_vert, mesh_num_verts, target_length: float,
                            workspace):
    """Backward of `mesh_edge_loss_forward` -> grad_verts (V,3) f32, from the forward's workspace (no sort).
    Deterministic, no atomics; grad_loss stays on the device."""
    return _regularizer_backward("mesh_edge_loss_backward", grad_loss, verts, faces, mesh_first_vert, mesh_num_verts,
                                 workspace, float(target_length))


def _laplacian_method(method):
    if method not in LAPLACIAN_METHODS:
        raise ValueError("Method should be one of {uniform, cot, cotcurv}")
    return LAPLACIAN_METHODS[method]


def mesh_laplacian_smoothing_forward(verts, faces, mesh_first_vert, mesh_num_verts, method: str):
    """Fused pytorch3d.loss.mesh_laplacian_smoothing for method "uniform", "cot" or "cotcurv" (DESIGN.md section 18)
    -> (loss () f32, workspace)."""
    m = _laplacian_method(method)
    return _regularizer_forward("mesh_laplacian_smoothing_forward", verts, faces, mesh_first_vert, mesh_num_verts, m)


def mesh_laplacian_smoothing_backward(grad_loss, verts, faces, mesh_first_vert, mesh_num_verts, method: str,
                                      workspace):
    """Backward of `mesh_laplacian_smoothing_forward` -> grad_verts (V,3) f32, with L and its weights constant (no
    sort).  Deterministic, no atomics."""
    m = _laplacian_method(method)
    return _regularizer_backward("mesh_laplacian_smoothing_backward", grad_loss, verts, faces, mesh_first_vert,
                                 mesh_num_verts, workspace, m)


def mesh_normal_consistency_forward(verts, faces, mesh_first_vert, mesh_num_verts):
    """Fused pytorch3d.loss.mesh_normal_consistency (DESIGN.md section 18) -> (loss () f32, workspace).  The face pairs
    are enumerated on the device: nothing reads the edge counts on the host."""
    return _regularizer_forward("mesh_normal_consistency_forward", verts, faces, mesh_first_vert, mesh_num_verts)


def mesh_normal_consistency_backward(grad_loss, verts, faces, mesh_first_vert, mesh_num_verts, workspace):
    """Backward of `mesh_normal_consistency_forward` -> grad_verts (V,3) f32 (no sort, no scatter).  Deterministic,
    no atomics."""
    return _regularizer_backward("mesh_normal_consistency_backward", grad_loss, verts, faces, mesh_first_vert,
                                 mesh_num_verts, workspace)


# the name the test hook is known by
_mesh_edge_table = mesh_edge_table


def _clip_frustum_args(frustum):
    """(planes (6,) float32 host array, cull_mask, has_z_clip, z_clip, perspective_correct) of a ClipFrustum-like
    object for the b200r_clip_* entry points."""
    values = (frustum.left, frustum.right, frustum.top, frustum.bottom, frustum.znear, frustum.zfar)
    mask = 0
    if frustum.cull:
        for i, v in enumerate(values):
            if v is not None:
                mask |= 1 << i
    planes = (ctypes.c_float * 6)(*[0.0 if v is None else float(v) for v in values])
    z = frustum.z_clip_value
    return planes, mask, int(z is not None), 0.0 if z is None else float(z), int(bool(frustum.perspective_correct))


def _check_clip_workspace(workspace, F):
    """The int64 workspace of `clip_faces_count` for F faces."""
    words = int(_lib.load().b200r_clip_faces_workspace_words(F))
    _check_tensor("workspace", workspace, I64, (words,), "workspace words of clip_faces_count,")


def clip_faces_count(frustum, face_verts=None, verts=None, faces=None):
    """Count pass of the fused clip_faces (DESIGN.md section 14): classifies every face of face_verts (F,3,3) -- or of
    verts[faces], read in place -- against `frustum` and returns the int64 workspace whose first four words are the
    record (F_clipped, n_case3, n_case4, number of faces culled or clipped).  Asynchronous: the caller reads the record."""
    if face_verts is not None:
        dev = _require_cuda(("face_verts", face_verts))
        _check_tensor("face_verts", face_verts, F32, (None, 3, 3), "F, 3, 3")
        F = int(face_verts.shape[0])
        fv, v, f = face_verts.contiguous(), None, None
    else:
        _, F, dev = _check_verts_faces(None, verts, faces)
        fv, v, f = None, verts.contiguous(), faces.contiguous()
    planes, mask, has_z, z, _ = _clip_frustum_args(frustum)
    ws = torch.empty((int(_lib.load().b200r_clip_faces_workspace_words(F)),), dtype=I64, device=dev)
    _launch(dev, "clip_faces_count", _ptr(fv), _ptr(v), _ptr(f), F, planes, mask, has_z, z, _ptr(ws))
    return ws


def clip_faces_fill(face_verts, mesh_to_face_first_idx, num_faces_per_mesh, frustum, workspace, record):
    """Fill pass of the fused clip_faces: the seven ClippedFaces fields in the reference's layout, from the workspace of
    `clip_faces_count(frustum, face_verts)` and its record (a 4-sequence read by the caller).  The last three are empty
    tensors when no face was clipped (only culled)."""
    dev = _require_cuda(("face_verts", face_verts), ("mesh_to_face_first_idx", mesh_to_face_first_idx),
                        ("num_faces_per_mesh", num_faces_per_mesh), ("workspace", workspace))
    _check_tensor("face_verts", face_verts, F32, (None, 3, 3), "F, 3, 3")
    F = int(face_verts.shape[0])
    N = _check_ranges(None, "mesh_to_face_first_idx", mesh_to_face_first_idx, "num_faces_per_mesh", num_faces_per_mesh)
    _check_clip_workspace(workspace, F)
    F_clipped, n3, n4 = (int(v) for v in record[:3])
    T = n3 + 2 * n4
    planes, mask, has_z, z, persp = _clip_frustum_args(frustum)
    fv, first = face_verts.contiguous(), mesh_to_face_first_idx.contiguous()
    out_fv = torch.empty((F_clipped, 3, 3), dtype=F32, device=dev)
    out_first = torch.empty((N,), dtype=I64, device=dev)
    out_num = torch.empty((N,), dtype=I64, device=dev)
    c2u = torch.empty((F_clipped,), dtype=I64, device=dev)
    conv = torch.empty((T, 3, 3), dtype=F32, device=dev)
    conv_idx = torch.empty((F_clipped if T > 0 else 0,), dtype=I64, device=dev)
    neighbor = torch.empty((F_clipped if T > 0 else 0,), dtype=I64, device=dev)
    _launch(dev, "clip_faces_fill", _ptr(fv), F, _ptr(first), N, planes, mask, has_z, z, persp, _ptr(workspace),
            F_clipped, n3, n4, _ptr(out_fv), _ptr(out_first), _ptr(out_num), _ptr(c2u), _ptr(conv), _ptr(conv_idx),
            _ptr(neighbor))
    return out_fv, out_first, out_num, c2u, conv, conv_idx, neighbor


def clip_faces_backward(face_verts, frustum, workspace, record, grad_face_verts_clipped, grad_conversion):
    """d loss / d face_verts (F,3,3) of the fused clip_faces from the gradients of its clipped face_verts and of its
    barycentric_conversion (either may be None); deterministic, no host synchronisation."""
    grads = [(name, g, shape) for name, g, shape in (
        ("grad_face_verts_clipped", grad_face_verts_clipped, (int(record[0]), 3, 3)),
        ("grad_conversion", grad_conversion, (int(record[1]) + 2 * int(record[2]), 3, 3))) if g is not None]
    dev = _require_cuda(("face_verts", face_verts), ("workspace", workspace), *[g[:2] for g in grads])
    _check_tensor("face_verts", face_verts, F32, (None, 3, 3), "F, 3, 3")
    F = int(face_verts.shape[0])
    _check_clip_workspace(workspace, F)
    for name, g, shape in grads:
        _check_tensor(name, g, F32, shape)
    n3, n4 = int(record[1]), int(record[2])
    planes, mask, has_z, z, persp = _clip_frustum_args(frustum)
    fv, gfv, gc = (_c(t) for t in (face_verts, grad_face_verts_clipped, grad_conversion))
    grad = torch.empty((F, 3, 3), dtype=F32, device=dev)
    _launch(dev, "clip_faces_backward", _ptr(fv), F, planes, mask, has_z, z, persp, _ptr(workspace), n3, n4, _ptr(gfv),
            _ptr(gc), _ptr(grad))
    return grad


def _check_clip_convert_inputs(pix_to_face, barycentric_coords, conversion, grad=None):
    """The device of pix_to_face (any shape) i64 with its float32 barycentric_coords (pix_to_face.shape + (3,)), of the
    (name, tensor) clipped-face maps `conversion` -- int64 (F_clipped,) indices and the float32 (T, 3, 3)
    barycentric_conversion -- and of the float32 upstream gradient (name, tensor) of barycentric_coords when given."""
    dev = _require_cuda(*([grad] if grad is not None else []), ("pix_to_face", pix_to_face),
                        ("barycentric_coords", barycentric_coords), *conversion)
    _check_tensor("pix_to_face", pix_to_face, I64)
    bary_shape = tuple(pix_to_face.shape) + (3,)
    _check_tensor("barycentric_coords", barycentric_coords, F32, bary_shape, "pix_to_face.shape + (3,)")
    for name, t in conversion:
        if name == "barycentric_conversion":
            _check_tensor(name, t, F32, (None, 3, 3), "T, 3, 3")
        else:
            _check_tensor(name, t, I64, (None,), "F_clipped,")
    if grad is not None:
        _check_tensor(*grad, F32, bary_shape, "pix_to_face.shape + (3,)")
    return dev


def clip_convert_forward(pix_to_face, barycentric_coords, faces_clipped_to_unclipped_idx, barycentric_conversion=None,
                         faces_clipped_to_conversion_idx=None):
    """Fused convert_clipped_rasterization_to_original_faces: (pix_to_face_unclipped, bary_unclipped).  Without a
    conversion only pix_to_face is mapped and bary_unclipped is None."""
    conversion = [("faces_clipped_to_unclipped_idx", faces_clipped_to_unclipped_idx)]
    if barycentric_conversion is not None:
        conversion += [("barycentric_conversion", barycentric_conversion),
                       ("faces_clipped_to_conversion_idx", faces_clipped_to_conversion_idx)]
    dev = _check_clip_convert_inputs(pix_to_face, barycentric_coords, conversion)
    p2f, bary = pix_to_face.contiguous(), barycentric_coords.contiguous()
    c2u = faces_clipped_to_unclipped_idx.contiguous()
    conv = barycentric_conversion.contiguous() if barycentric_conversion is not None else None
    cidx = faces_clipped_to_conversion_idx.contiguous() if barycentric_conversion is not None else None
    p2f_out = torch.empty_like(p2f)
    bary_out = torch.empty_like(bary) if conv is not None else None
    _launch(dev, "clip_convert_forward", _ptr(p2f), _ptr(bary), p2f.numel(), _ptr(c2u), _ptr(conv), _ptr(cidx),
            _ptr(p2f_out), _ptr(bary_out))
    return p2f_out, bary_out


def clip_convert_backward(grad_bary_unclipped, pix_to_face, barycentric_coords, barycentric_conversion,
                          faces_clipped_to_conversion_idx, needs_input_grad=(True, True)):
    """Backward of `clip_convert_forward` -> (grad_barycentric_coords, grad_conversion); an entry is None where
    `needs_input_grad` (same order) is false.  grad_conversion is accumulated with atomics, so requesting it under
    torch.use_deterministic_algorithms(True) raises, like the rasterizer backward in the same graph."""
    dev = _check_clip_convert_inputs(pix_to_face, barycentric_coords,
                                     [("barycentric_conversion", barycentric_conversion),
                                      ("faces_clipped_to_conversion_idx", faces_clipped_to_conversion_idx)],
                                     ("grad_bary_unclipped", grad_bary_unclipped))
    need_bary, need_conv = (bool(v) for v in needs_input_grad)
    if need_conv:
        _refuse_nondeterministic("clip_convert_backward", "grad_conversion is accumulated with atomics")
    g, p2f, bary = grad_bary_unclipped.contiguous(), pix_to_face.contiguous(), barycentric_coords.contiguous()
    conv, cidx = barycentric_conversion.contiguous(), faces_clipped_to_conversion_idx.contiguous()
    T = int(conv.shape[0])
    g_bary = torch.empty_like(bary) if need_bary else None
    g_conv = torch.empty_like(conv) if need_conv else None
    _launch(dev, "clip_convert_backward", _ptr(g), _ptr(p2f), _ptr(bary), p2f.numel(), _ptr(conv), _ptr(cidx), T,
            _ptr(g_bary), _ptr(g_conv))
    return g_bary, g_conv


# ------------------------------------------------------------------------------------------------ test hooks
# pytorch3d/csrc/ext.cpp:69-73: "These are only visible for testing; users should not call them directly".  Provided so
# that the reference's own tests of these entry points can run against this build; none of them is on the product path.

def _coarse(kind, elems, first, num, image_size, bin_size, max_per_bin, blur_radius=None, radius=None):
    dev = _require_cuda(("elements", elems), ("first_idx", first), ("num_per_batch", num),
                        *([("radius", radius)] if radius is not None else []))
    H, W = int(image_size[0]), int(image_size[1])
    N, E = int(num.shape[0]), int(elems.shape[0])
    el = elems.contiguous()
    f64, n64 = first.contiguous().to(I64), num.contiguous().to(I64)
    _check_tensor("elements", el, F32)
    _check_tensor("num_per_batch", n64, I64, (N,), "N,")
    _check_tensor("first_idx", f64, I64, (N,), "N,")
    if radius is not None:
        _check_tensor("radius", radius, F32, (E,), "num_points,")
    bin_size, M = int(bin_size), int(max_per_bin)
    if bin_size <= 0:
        raise RuntimeError("bin_size must be positive for the coarse stage")
    BH, BW = 1 + (H - 1) // bin_size, 1 + (W - 1) // bin_size
    if BH >= 22 or BW >= 22:  # kMaxItemsPerBin (rasterize_coarse.cu:244-249)
        raise RuntimeError("In RasterizeCoarseCuda got num_bins_y: %d, num_bins_x: %d, too many bins" % (BH, BW))
    bins = torch.empty((N, BH, BW, M), dtype=I32, device=dev)
    counts = torch.empty((N, BH, BW), dtype=I32, device=dev)
    overflow = torch.zeros((1,), dtype=I32, device=dev)
    if blur_radius is not None:
        args = (_ptr(el), E, _ptr(f64), _ptr(n64), N, H, W, float(blur_radius))
    else:
        args = (_ptr(el), E, _ptr(f64), _ptr(n64), _ptr(radius.contiguous()), N, H, W)
    _launch(dev, "rasterize_%s_coarse" % kind, *args, bin_size, M, bins.data_ptr(), counts.data_ptr(),
            overflow.data_ptr())
    if int(overflow.item()) != 0:
        import warnings
        warnings.warn("Bin size was too small in the coarse rasterization phase. This caused an overflow, meaning "
                      "output may be incomplete. To solve, try increasing max_faces_per_bin / max_points_per_bin, "
                      "decreasing bin_size, or setting bin_size to 0 to use the naive rasterization.")
    # canonical form: ascending element index inside every bin, -1 padding last
    big = torch.iinfo(torch.int32).max
    bins = torch.where(bins < 0, torch.full_like(bins, big), bins).sort(dim=-1).values
    return torch.where(bins == big, torch.full_like(bins, -1), bins)


def _rasterize_meshes_coarse(face_verts, mesh_to_face_first_idx, num_faces_per_mesh, image_size, blur_radius, bin_size,
                             max_faces_per_bin):
    """pytorch3d._C._rasterize_meshes_coarse (RasterizeMeshesCoarse, rasterize_meshes.h:292-318) -> bin_faces
    (N, BH, BW, M) int32, -1 padded, ascending inside every bin."""
    if face_verts.dim() != 3 or face_verts.shape[1] != 3 or face_verts.shape[2] != 3:
        raise RuntimeError("face_verts must have dimensions (num_faces, 3, 3)")
    return _coarse("meshes", face_verts, mesh_to_face_first_idx, num_faces_per_mesh, image_size, bin_size,
                   max_faces_per_bin, blur_radius=blur_radius)


def _rasterize_points_coarse(points, cloud_to_packed_first_idx, num_points_per_cloud, image_size, radius, bin_size,
                             max_points_per_bin):
    """pytorch3d._C._rasterize_points_coarse (RasterizePointsCoarse, rasterize_points.h:140-166)."""
    if points.dim() != 2 or points.shape[1] != 3:
        raise RuntimeError("points must have dimensions (num_points, 3)")
    return _coarse("points", points, cloud_to_packed_first_idx, num_points_per_cloud, image_size, bin_size,
                   max_points_per_bin, radius=radius)


def _rasterize_meshes_naive(face_verts, mesh_to_face_first_idx, num_faces_per_mesh, clipped_faces_neighbor_idx,
                            image_size, blur_radius, faces_per_pixel, perspective_correct, clip_barycentric_coords,
                            cull_backfaces):
    """pytorch3d._C._rasterize_meshes_naive (RasterizeMeshesNaive, rasterize_meshes.h:109-145): this build has one path;
    it returns the naive kernel's result for every bin_size."""
    return rasterize_meshes(face_verts, mesh_to_face_first_idx, num_faces_per_mesh, clipped_faces_neighbor_idx,
                            image_size, blur_radius, faces_per_pixel, 0, 0, perspective_correct,
                            clip_barycentric_coords, cull_backfaces)


def _rasterize_points_naive(points, cloud_to_packed_first_idx, num_points_per_cloud, image_size, radius,
                            points_per_pixel):
    """pytorch3d._C._rasterize_points_naive (RasterizePointsNaive, rasterize_points.h:65-95)."""
    return rasterize_points(points, cloud_to_packed_first_idx, num_points_per_cloud, image_size, radius,
                            points_per_pixel, 0, 0)


def _rasterize_meshes_fine(face_verts, bin_faces, clipped_faces_neighbor_idx, image_size, blur_radius, bin_size,
                           faces_per_pixel, perspective_correct, clip_barycentric_coords, cull_backfaces):
    """pytorch3d._C._rasterize_meshes_fine (RasterizeMeshesFine, rasterize_meshes.h:407-452).  The reference's fine stage
    looks only at the faces listed in a pixel's bin; this build bins exactly by itself, so `bin_faces` only tells which
    image a face belongs to (the index range of the faces listed for image n) -- for a table produced by the coarse stage
    (every face in every bin it can touch) the result is the same."""
    if bin_faces.dim() != 4:
        raise RuntimeError("bin_faces must have 4 dimensions")
    N = int(bin_faces.shape[0])
    flat = bin_faces.reshape(N, -1).to(torch.int64)
    big = torch.iinfo(torch.int64).max
    lo = torch.where(flat >= 0, flat, torch.full_like(flat, big)).min(dim=1).values.tolist()  # (host sync: test hook)
    hi = flat.max(dim=1).values.tolist()
    first_l, num_l, at = [], [], 0
    for a, b in zip(lo, hi):  # ascending ranges; an image without listed faces gets an empty range
        if b >= 0:
            first_l.append(int(a))
            num_l.append(int(b - a + 1))
            at = int(b) + 1
        else:
            first_l.append(at)
            num_l.append(0)
    first = torch.tensor(first_l, dtype=torch.int64, device=face_verts.device)
    num = torch.tensor(num_l, dtype=torch.int64, device=face_verts.device)
    return rasterize_meshes(face_verts, first, num, clipped_faces_neighbor_idx, image_size, blur_radius,
                            faces_per_pixel, bin_size, int(bin_faces.shape[3]), perspective_correct,
                            clip_barycentric_coords, cull_backfaces)
