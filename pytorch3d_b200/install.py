"""Rebind an installed PyTorch3D onto the H100-native rasterizer ops.

PyTorch3D reaches its native rasterizer through module attributes:
    pytorch3d/renderer/mesh/rasterize_meshes.py:14      from pytorch3d import _C
    pytorch3d/renderer/points/rasterize_points.py:13    from pytorch3d import _C
    pytorch3d/renderer/compositing.py:10                from pytorch3d import _C
    pytorch3d/ops/interp_face_attrs.py:10               from pytorch3d import _C
and calls `_C.rasterize_meshes[_backward]`, `_C.rasterize_points[_backward]`, `_C.accum_alphacomposite[_backward]`,
`_C.accum_weightedsum[_backward]`, `_C.accum_weightedsumnorm[_backward]`, `_C.interp_face_attrs_forward/_backward`.
`install()` replaces that `_C` name *in those modules only* with a proxy that serves these ops from
`pytorch3d_b200._C` for CUDA tensors and forwards everything else (including CPU tensors) to the original module,
so `MeshRasterizer` / `PointsRasterizer` / `MeshRenderer` / `PointsRenderer` work unchanged.
`uninstall()` restores the originals.

`install_blending()` (separate, so that `install()` keeps its four modules) serves the mesh blending step:
    pytorch3d/renderer/blending.py          from pytorch3d import _C   (sigmoid_alpha_blend[_backward])
                                            softmax_rgb_blend, hard_rgb_blend (pure torch)
    pytorch3d/renderer/mesh/shader.py       from ..blending import hard_rgb_blend, softmax_rgb_blend, ...
It proxies `_C` of the blending module for the two sigmoid ops and replaces the two torch blends, in both modules, by
functions that send float32 CUDA inputs to `pytorch3d_b200.blending` and everything else (CPU tensors, other dtypes; a
background colour, znear or zfar that requires grad) to the originals.

`install_splatter()` (separate again) serves SplatterPhongShader's blend:
    pytorch3d/renderer/splatter_blend.py    class SplatterBlender (pure torch)
    pytorch3d/renderer/mesh/shader.py       from ..splatter_blend import SplatterBlender
It replaces the class name in both modules by one whose instances send float32 CUDA inputs with K <= 150 and a
constant background colour to `pytorch3d_b200.splatter_blend`, and everything else to an instance of the original.

`install_shading()` (separate again) serves the per-pixel lighting of SoftPhongShader, HardPhongShader,
SplatterPhongShader and HardFlatShader:
    pytorch3d/renderer/mesh/shading.py      phong_shading, _phong_shading_with_pixels, flat_shading (pure torch)
    pytorch3d/renderer/mesh/shader.py       from .shading import _phong_shading_with_pixels, flat_shading, ...
It replaces the three functions in both modules by functions that send float32 CUDA inputs lit by PyTorch3D's own
PointLights / DirectionalLights / AmbientLights and Materials to `pytorch3d_b200.shading`, and everything else to the
originals.

`install_gouraud()` (separate again, so that `install_shading()` keeps its three functions) serves the per-vertex
lighting of SoftGouraudShader and HardGouraudShader:
    pytorch3d/renderer/mesh/shading.py      gouraud_shading (pure torch: per-vertex lighting, a gather, interpolation)
    pytorch3d/renderer/mesh/shader.py       from .shading import gouraud_shading, ...
It replaces the function in both modules by one that sends float32 CUDA vertices, vertex colours and barycentrics
with int64 CUDA pix_to_face, all on one device, a 3-channel `TexturesVertex`, PyTorch3D's own PointLights /
DirectionalLights / AmbientLights and Materials, cameras with R and T, and properties and cameras of batch 1 or
len(meshes) to `pytorch3d_b200.shading`,
and everything else (1-channel vertex features, other textures, subclasses, CPU tensors) to the original.

`install_textures()` (separate again) serves the texture sampling of every mesh shader for `TexturesUV`:
    pytorch3d/renderer/mesh/textures.py     TexturesUV.sample_textures (pure torch: interpolation, grid_sample)
It replaces the method on the class itself, so every import path sees it.  Textures with one map per mesh (no
`maps_ids`), float32 CUDA maps and barycentrics and int64 CUDA pix_to_face on one device, one of the two sampling modes
"bilinear" / "nearest" and one of the three padding modes go to `pytorch3d_b200.textures`; everything else (CPU
tensors, tensors on different devices, other dtypes, multi-map textures, "bicubic", empty textures) to the original
method.

`install_texture_atlas()` (separate again) serves the texture sampling of every mesh shader for `TexturesAtlas`:
    pytorch3d/renderer/mesh/textures.py     TexturesAtlas.sample_textures (pure torch: a dozen elementwise ops, a gather)
It replaces the method on the class itself, as `install_textures()` does.  It packs the atlas once; a non-empty float32
CUDA atlas (F, R, R, C) with R >= 1, int64 CUDA pix_to_face and float32 barycentrics on one device go to
`pytorch3d_b200.texture_atlas`; everything else (CPU tensors, tensors on different devices, other dtypes, empty
textures) to the original method.

`install_clipping()` (separate again) serves the frustum culling and z-clipping that `MeshRasterizer` turns on for
perspective cameras:
    pytorch3d/renderer/mesh/rasterize_meshes.py   from .clip import clip_faces, convert_clipped_rasterization_to_...
It replaces the two names in that module by functions that send float32 CUDA face_verts (and the Fragments of such a
call) to `pytorch3d_b200.clip`'s fused pair, returning the reference's own `ClippedFaces`; everything else (CPU
tensors, other dtypes) goes to the originals.

`install_normals()` (separate again) serves the mesh normals that every lit shader, `sample_points_from_meshes` and
the face-area users read:
    pytorch3d/ops/mesh_face_areas_normals.py   from pytorch3d import _C   (face_areas_normals_forward/_backward)
    pytorch3d/structures/meshes.py             Meshes._compute_vertex_normals (pure torch: a gather, torch.cross,
                                               three index_add calls, F.normalize)
It proxies `_C` of the first module for the two face ops: float32 CUDA verts with int64 CUDA faces on one device go to
`pytorch3d_b200._C`, everything else (CPU tensors, float64 verts) to the original.  So `faces_normals_packed()`,
`faces_areas_packed()`, HardFlatShader and `sample_points_from_meshes` run the new kernels.  It replaces the method
`_compute_vertex_normals` on the class `Meshes`, as `install_textures()` does, keeping its `refresh` and caching
semantics (including the `refresh=True` recomputation of `offset_verts_`): a non-empty mesh whose `verts_packed()` is
float32 CUDA and `faces_packed()` int64 CUDA on the same device goes to `pytorch3d_b200.normals.verts_normals`;
everything else, empty meshes included (the original stores an int64 (N, 3) zero tensor), to the original method.

`install_regularizers()` (separate again) serves the three shape priors of a mesh-fitting loop:
    pytorch3d/loss/__init__.py                      from .mesh_edge_loss import mesh_edge_loss, ... (by name)
    pytorch3d/loss/mesh_edge_loss.py                mesh_edge_loss (torch: edges_packed(), a gather, a norm)
    pytorch3d/loss/mesh_laplacian_smoothing.py      mesh_laplacian_smoothing (sparse matrices, cuSPARSE)
    pytorch3d/loss/mesh_normal_consistency.py       mesh_normal_consistency (a host copy, a CPU pair enumeration)
It replaces the three names in `pytorch3d.loss` and in their defining modules by functions that send meshes whose
`verts_packed()` is float32 CUDA and `faces_packed()` int64 CUDA on the same device, within the kernels' size limits
(V < 2^31 - 1, 6F < 2^31), to `pytorch3d_b200.regularizers`; everything else (CPU tensors, float64 verts, oversized
meshes, an unknown Laplacian method, for which the original raises) goes to the originals.

`install_depth_shading()` (separate again) serves the depth shaders of depth-supervised fitting:
    pytorch3d/renderer/mesh/shader.py       SoftDepthShader.forward, HardDepthShader.forward (pure torch)
It replaces the method `forward` on both classes, as `install_textures()` does.  A call goes to
`pytorch3d_b200.blending.soft_depth` / `hard_depth` when pix_to_face is int64 CUDA, zbuf (and dists for
SoftDepthShader) float32 of the same 4-D shape on its device, 1 <= K <= 150, `blend_params.sigma` a real number, and
zfar -- `kwargs.get("zfar", getattr(cameras, "zfar", 100.0))`, as the shaders resolve it -- a real number or a
1-element float32 tensor on that device that does not require grad.  Everything else goes to the original method:
CPU tensors, other dtypes, K = 0 or K > 150, `dists` None (for which SoftDepthShader raises), a per-image zfar of N > 1
values (for which both raise), and a zfar that requires grad.

`install_sampling()` (separate again) serves the surface sampling of the mesh-to-mesh fitting loop:
    pytorch3d/ops/__init__.py                       from .sample_points_from_meshes import sample_points_from_meshes
    pytorch3d/ops/sample_points_from_meshes.py      sample_points_from_meshes (torch: multinomial, rand, gathers)
It replaces the function in its defining module and the name in `pytorch3d.ops` (where the import makes the package
attribute the function, not the submodule) by one that sends meshes whose `verts_packed()` is float32 CUDA and
`faces_packed()` int64 CUDA on the same device, with an integer num_samples >= 1, within the kernels' size limits, to
`pytorch3d_b200.sampling`; everything else (CPU tensors, float64 verts, oversized inputs, and `return_textures=True`
on a batch containing a mesh without faces, for which the original raises) goes to the original.

`install_chamfer()` (separate again) serves the loss of both fitting loops:
    pytorch3d/loss/__init__.py                      from .chamfer import chamfer_distance
    pytorch3d/loss/chamfer.py                       chamfer_distance (knn_points, knn_gather, torch reductions)
It replaces the function in its defining module and the name in `pytorch3d.loss` by one that sends float32 CUDA
clouds with D = 3 on one device (tensors or Pointclouds), with int64 (N,) lengths, float32 (N, P, 3) normals and
float32 (N,) weights that do not require grad on that device, within the kernels' size limits, to
`pytorch3d_b200.chamfer`; everything else (CPU tensors, float64, D != 3, mixed devices, weights that require grad,
oversized inputs, and calls the reference rejects) goes to the original.

`install_point_ops()` (separate again) serves PointNet++'s sample-and-group:
    pytorch3d/ops/__init__.py                       from .sample_farthest_points import sample_farthest_points
                                                    from .ball_query import ball_query
    pytorch3d/ops/sample_farthest_points.py         sample_farthest_points (FarthestPointSampling, masked_gather)
    pytorch3d/ops/ball_query.py                     ball_query (BallQuery, knn_points_backward, masked_gather)
It replaces each function in its defining module and the name in `pytorch3d.ops` by one that sends float32 CUDA
clouds with D = 3 and int64 (N,) lengths (or None) on their device, within the kernels' size limits, to
`pytorch3d_b200.point_ops`; everything else (CPU tensors, float64, D != 3, mixed devices, a K the reference would
reject, oversized inputs) goes to the original.
"""
import importlib
import numbers
import types

import torch

from . import _C as _b200_C

_OPS = ("rasterize_meshes", "rasterize_meshes_backward", "rasterize_points", "rasterize_points_backward",
        "accum_alphacomposite", "accum_alphacomposite_backward", "accum_weightedsum", "accum_weightedsum_backward",
        "accum_weightedsumnorm", "accum_weightedsumnorm_backward", "interp_face_attrs_forward",
        "interp_face_attrs_backward")
_MODULES = ("pytorch3d.renderer.mesh.rasterize_meshes", "pytorch3d.renderer.points.rasterize_points",
            "pytorch3d.renderer.compositing", "pytorch3d.ops.interp_face_attrs")
_BLEND_OPS = ("sigmoid_alpha_blend", "sigmoid_alpha_blend_backward")
_BLEND_MODULE = "pytorch3d.renderer.blending"
_BLEND_FUNCTIONS = ("softmax_rgb_blend", "hard_rgb_blend")
_BLEND_FUNCTION_MODULES = ("pytorch3d.renderer.blending", "pytorch3d.renderer.mesh.shader")
_SPLATTER_MODULES = ("pytorch3d.renderer.splatter_blend", "pytorch3d.renderer.mesh.shader")
_SHADING_MODULES = ("pytorch3d.renderer.mesh.shading", "pytorch3d.renderer.mesh.shader")
_SHADING_FUNCTIONS = ("phong_shading", "_phong_shading_with_pixels", "flat_shading")
_TEXTURES_MODULE = "pytorch3d.renderer.mesh.textures"
_CLIP_MODULE = "pytorch3d.renderer.mesh.rasterize_meshes"
_CLIP_FUNCTIONS = ("clip_faces", "convert_clipped_rasterization_to_original_faces")
_NORMALS_MODULE = "pytorch3d.ops.mesh_face_areas_normals"
_NORMALS_OPS = ("face_areas_normals_forward", "face_areas_normals_backward")
_MESHES_MODULE = "pytorch3d.structures.meshes"
_LOSS_PACKAGE = "pytorch3d.loss"
_LOSS_FUNCTIONS = ("mesh_edge_loss", "mesh_laplacian_smoothing", "mesh_normal_consistency")
_OPS_PACKAGE = "pytorch3d.ops"
_SAMPLING_MODULE = "pytorch3d.ops.sample_points_from_meshes"
_SHADER_MODULE = "pytorch3d.renderer.mesh.shader"
_DEPTH_SHADERS = ("SoftDepthShader", "HardDepthShader")
_saved = {}
# (module name, attribute) -> original (install_blending, install_splatter, install_shading, install_gouraud,
# install_clipping, install_normals, install_regularizers, install_sampling, install_chamfer and install_point_ops)
_saved_blend = {}
# (module name, class name, method name) -> original (install_textures, install_texture_atlas, install_normals,
# install_depth_shading)
_saved_methods = {}


def _first_is_cuda(name, args):
    first = args[0] if args else None
    return first is None or getattr(first, "is_cuda", False)


class _Proxy(types.ModuleType):
    """`ops` are served by `pytorch3d_b200._C` when `fused(name, args)` holds (by default: the first argument is a CUDA
    tensor) and by the original module otherwise; every other name is the original's."""

    def __init__(self, original, ops=_OPS, fused=_first_is_cuda):
        super().__init__("pytorch3d_b200._C_proxy")
        self.__dict__["_original"] = original
        self.__dict__["_ops"] = ops
        self.__dict__["_fused"] = fused

    def __getattr__(self, name):
        original = self.__dict__["_original"]
        if name in self.__dict__["_ops"]:
            ours = getattr(_b200_C, name)
            theirs = getattr(original, name, None)
            fused = self.__dict__["_fused"]

            def dispatch(*args, **kwargs):
                if theirs is not None and not fused(name, args):
                    return theirs(*args, **kwargs)  # e.g. CPU tensors keep the reference's CPU path
                return ours(*args, **kwargs)

            return dispatch
        return getattr(original, name)


def install():
    """Patch pytorch3d (must be importable).  Returns the list of patched module names."""
    import importlib
    patched = []
    for modname in _MODULES:
        mod = importlib.import_module(modname)
        if modname not in _saved:
            _saved[modname] = mod._C
            mod._C = _Proxy(mod._C)
        patched.append(modname)
    return patched


def _requires_grad(x):
    return torch.is_tensor(x) and x.requires_grad


def _float32(colors, fragments):
    """The fused blend takes float32 colours, depths and distances; other dtypes keep the original torch code."""
    return all(getattr(t, "dtype", None) == torch.float32
               for t in (colors, getattr(fragments, "zbuf", None), getattr(fragments, "dists", None)))


def _blend_dispatch(name, original):
    from . import blending as ours
    if name == "softmax_rgb_blend":
        def softmax_rgb_blend(colors, fragments, blend_params, znear=1.0, zfar=100):
            if (not colors.is_cuda or not _float32(colors, fragments)
                    or _requires_grad(getattr(blend_params, "background_color", None))
                    or _requires_grad(znear) or _requires_grad(zfar)):
                return original(colors, fragments, blend_params, znear, zfar)
            return ours.softmax_rgb_blend(colors, fragments, blend_params, znear, zfar)
        return softmax_rgb_blend

    def hard_rgb_blend(colors, fragments, blend_params):
        if not colors.is_cuda or colors.dtype != torch.float32:
            return original(colors, fragments, blend_params)
        return ours.hard_rgb_blend(colors, fragments, blend_params)
    return hard_rgb_blend


def install_blending():
    """Patch PyTorch3D's mesh blending (must be importable).  Returns the list of patched module names."""
    import importlib
    mod = importlib.import_module(_BLEND_MODULE)
    if (_BLEND_MODULE, "_C") not in _saved_blend:
        _saved_blend[(_BLEND_MODULE, "_C")] = mod._C
        mod._C = _Proxy(mod._C, _BLEND_OPS)
    for modname in _BLEND_FUNCTION_MODULES:
        m = importlib.import_module(modname)
        for name in _BLEND_FUNCTIONS:
            if (modname, name) not in _saved_blend:
                _saved_blend[(modname, name)] = getattr(m, name)
                setattr(m, name, _blend_dispatch(name, getattr(m, name)))
    return list(_BLEND_FUNCTION_MODULES)


def _splatter_dispatch(original):
    """A stand-in for the class `SplatterBlender` that sends float32 CUDA inputs with K <= 150 and a constant background
    to the fused op, and everything else to an instance of the original class, built on first use."""
    from . import splatter_blend as ours

    class SplatterBlender(torch.nn.Module):
        def __init__(self, input_shape, device):
            super().__init__()
            self._input_shape, self._device = input_shape, device
            self._ours = ours.SplatterBlender(input_shape, device)
            self._original = None

        def to(self, device):
            self._device = device
            if self._original is not None:
                self._original.to(device)
            return super().to(device)

        def forward(self, colors, pixel_coords_cameras, cameras, background_mask, blend_params):
            if (colors.is_cuda and colors.dtype == torch.float32 and pixel_coords_cameras.dtype == torch.float32
                    and colors.dim() == 5 and colors.shape[3] <= _b200_C.kMaxPointsPerPixel
                    and not _requires_grad(getattr(blend_params, "background_color", None))):
                return self._ours(colors, pixel_coords_cameras, cameras, background_mask, blend_params)
            if self._original is None:
                self._original = original(self._input_shape, self._device)
            return self._original(colors, pixel_coords_cameras, cameras, background_mask, blend_params)

    SplatterBlender.__qualname__ = "SplatterBlender"
    SplatterBlender.__module__ = __name__
    return SplatterBlender


def install_splatter():
    """Patch PyTorch3D's splatter blending (must be importable): the name `SplatterBlender` in
    pytorch3d.renderer.splatter_blend and in pytorch3d.renderer.mesh.shader, where `SplatterPhongShader` builds its
    blender.  Blenders built before the call, and names imported from those modules before it, keep the original.
    Returns the list of patched module names."""
    import importlib
    for modname in _SPLATTER_MODULES:
        m = importlib.import_module(modname)
        if (modname, "SplatterBlender") not in _saved_blend:
            _saved_blend[(modname, "SplatterBlender")] = m.SplatterBlender
            m.SplatterBlender = _splatter_dispatch(m.SplatterBlender)
    return list(_SPLATTER_MODULES)


def _shading_fused(fragments, lights, materials, texels):
    """Whether the fused shading takes these inputs: float32 CUDA texels and Fragments, 3 texel channels, lights exactly
    PyTorch3D's PointLights / DirectionalLights / AmbientLights and materials exactly its Materials, all with 3
    channels, and material diffuse / specular colours of batch 1 (other batches do not broadcast in the reference)."""
    import importlib
    try:
        lighting = importlib.import_module("pytorch3d.renderer.lighting")
        materials_mod = importlib.import_module("pytorch3d.renderer.materials")
    except ImportError:
        return False
    light_types = tuple(getattr(lighting, n) for n in ("PointLights", "DirectionalLights", "AmbientLights")
                        if hasattr(lighting, n))
    if type(lights) not in light_types or type(materials) is not getattr(materials_mod, "Materials", None):
        return False
    bary = getattr(fragments, "bary_coords", None)
    if not (getattr(texels, "is_cuda", False) and texels.dtype == torch.float32 and texels.dim() == 5
            and texels.shape[-1] == 3 and getattr(bary, "dtype", None) == torch.float32 and bary.is_cuda
            and getattr(fragments.pix_to_face, "is_cuda", False) and fragments.pix_to_face.dtype == torch.int64):
        return False
    for owner, names in ((lights, ("ambient_color", "diffuse_color", "specular_color")),
                         (materials, ("ambient_color", "diffuse_color", "specular_color"))):
        for name in names:
            t = getattr(owner, name, None)
            if t is None and owner is lights and name != "ambient_color":
                continue  # AmbientLights
            if not torch.is_tensor(t) or t.dim() != 2 or t.shape[-1] != 3:
                return False
    return materials.diffuse_color.shape[0] == 1 and materials.specular_color.shape[0] == 1


def _shading_dispatch(name, original):
    from . import shading as ours

    def shade(meshes, fragments, lights, cameras, materials, texels):
        if _shading_fused(fragments, lights, materials, texels):
            return getattr(ours, name)(meshes, fragments, lights, cameras, materials, texels)
        return original(meshes, fragments, lights, cameras, materials, texels)

    shade.__name__ = shade.__qualname__ = name
    return shade


def install_shading():
    """Patch PyTorch3D's Phong and flat shading (must be importable): `phong_shading`, `_phong_shading_with_pixels` and
    `flat_shading` in pytorch3d.renderer.mesh.shading and in pytorch3d.renderer.mesh.shader, which imports them by name.
    Float32 CUDA inputs lit by PyTorch3D's own light and material classes go to `pytorch3d_b200.shading`; everything
    else (CPU tensors, other dtypes, light or material subclasses with their own models) to the originals.  Returns the
    list of patched module names."""
    import importlib
    for modname in _SHADING_MODULES:
        m = importlib.import_module(modname)
        for name in _SHADING_FUNCTIONS:
            if (modname, name) not in _saved_blend and hasattr(m, name):
                _saved_blend[(modname, name)] = getattr(m, name)
                setattr(m, name, _shading_dispatch(name, getattr(m, name)))
    return list(_SHADING_MODULES)


def _gouraud_fused(meshes, fragments, lights, cameras, materials):
    """Whether the fused Gouraud shading takes this call (see the module docstring)."""
    try:
        lighting = importlib.import_module("pytorch3d.renderer.lighting")
        materials_mod = importlib.import_module("pytorch3d.renderer.materials")
        textures_mod = importlib.import_module(_TEXTURES_MODULE)
    except ImportError:
        return False
    light_types = tuple(getattr(lighting, n) for n in ("PointLights", "DirectionalLights", "AmbientLights")
                        if hasattr(lighting, n))
    if type(lights) not in light_types or type(materials) is not getattr(materials_mod, "Materials", None):
        return False
    if type(getattr(meshes, "textures", None)) is not getattr(textures_mod, "TexturesVertex", None):
        return False
    verts, feats = meshes.verts_packed(), meshes.textures.verts_features_packed()
    bary, p2f = getattr(fragments, "bary_coords", None), fragments.pix_to_face
    if not all(getattr(t, "is_cuda", False) for t in (verts, feats, bary, p2f)):
        return False
    if verts.device != p2f.device or feats.device != p2f.device or bary.device != p2f.device:
        return False
    if verts.dtype != torch.float32 or feats.dtype != torch.float32 or bary.dtype != torch.float32 \
            or p2f.dtype != torch.int64:
        return False
    if feats.dim() != 2 or feats.shape[1] != 3:
        return False  # 1-channel features broadcast in the reference
    n = len(meshes)
    for owner, names in ((lights, ("ambient_color", "diffuse_color", "specular_color", "location", "direction")),
                         (materials, ("ambient_color", "diffuse_color", "specular_color", "shininess"))):
        for name in names:
            t = getattr(owner, name, None)
            if t is None:
                continue
            if not torch.is_tensor(t) or t.dim() < 1 or t.shape[0] not in (1, n):
                return False
            if name != "shininess" and (t.dim() != 2 or t.shape[-1] != 3):
                return False
    for name in ("R", "T"):  # the camera batch: the fused op forms one camera centre per mesh
        t = getattr(cameras, name, None)
        if not torch.is_tensor(t) or t.dim() < 1 or t.shape[0] not in (1, n):
            return False
    return True


def _gouraud_dispatch(original):
    from . import shading as ours

    def gouraud_shading(meshes, fragments, lights, cameras, materials):
        if _gouraud_fused(meshes, fragments, lights, cameras, materials):
            return ours.gouraud_shading(meshes, fragments, lights, cameras, materials)
        return original(meshes, fragments, lights, cameras, materials)

    gouraud_shading.__doc__ = original.__doc__
    return gouraud_shading


def install_gouraud():
    """Patch PyTorch3D's Gouraud shading (must be importable): `gouraud_shading` in pytorch3d.renderer.mesh.shading and
    in pytorch3d.renderer.mesh.shader, which imports it by name.  Returns the list of patched module names."""
    for modname in _SHADING_MODULES:
        m = importlib.import_module(modname)
        if (modname, "gouraud_shading") not in _saved_blend and hasattr(m, "gouraud_shading"):
            _saved_blend[(modname, "gouraud_shading")] = m.gouraud_shading
            m.gouraud_shading = _gouraud_dispatch(m.gouraud_shading)
    return list(_SHADING_MODULES)


def _textures_fused(textures, fragments):
    """Whether the fused texture sampling takes this call: one map per mesh, a non-empty texture, float32 CUDA maps and
    barycentrics and int64 CUDA pix_to_face on one device, a sampling and padding mode the kernels implement, one map per
    image."""
    if textures.maps_ids_padded() is not None or textures.isempty():
        return False
    if textures.sampling_mode not in _b200_C.SAMPLING_MODES or textures.padding_mode not in _b200_C.PADDING_MODES:
        return False
    maps, bary, p2f = textures.maps_padded(), getattr(fragments, "bary_coords", None), fragments.pix_to_face
    if not all(getattr(t, "is_cuda", False) for t in (maps, bary, p2f)):
        return False
    if maps.device != p2f.device or bary.device != p2f.device:
        return False  # the reference moves the maps to the Fragments' device
    if maps.dtype != torch.float32 or bary.dtype != torch.float32 or p2f.dtype != torch.int64:
        return False
    return maps.dim() == 4 and p2f.dim() == 4 and maps.shape[0] == p2f.shape[0]


def _textures_dispatch(original):
    from . import textures as ours

    def sample_textures(self, fragments, **kwargs):
        if _textures_fused(self, fragments):
            return ours.sample_textures(self, fragments, **kwargs)
        return original(self, fragments, **kwargs)

    sample_textures.__name__ = "sample_textures"
    sample_textures.__qualname__ = "TexturesUV.sample_textures"
    sample_textures.__doc__ = original.__doc__
    return sample_textures


def install_textures():
    """Patch PyTorch3D's UV texture sampling (must be importable): the method `sample_textures` of the class
    `TexturesUV` in pytorch3d.renderer.mesh.textures, so that existing objects and every import path see it.  Returns
    the list of patched module names."""
    import importlib
    m = importlib.import_module(_TEXTURES_MODULE)
    key = (_TEXTURES_MODULE, "TexturesUV", "sample_textures")
    if key not in _saved_methods:
        cls = m.TexturesUV
        _saved_methods[key] = cls.__dict__["sample_textures"]
        cls.sample_textures = _textures_dispatch(cls.__dict__["sample_textures"])
    return [_TEXTURES_MODULE]


def _atlas_fused(atlas, fragments):
    """Whether the fused atlas sampling takes this call: a float32 CUDA atlas (F, R, R, C) with R >= 1 (an empty texture
    packs to R = 0), float32 barycentrics and int64 CUDA pix_to_face, all on one device."""
    bary, p2f = getattr(fragments, "bary_coords", None), fragments.pix_to_face
    if not all(getattr(t, "is_cuda", False) for t in (atlas, bary, p2f)):
        return False
    if atlas.device != p2f.device or bary.device != p2f.device:
        return False
    if atlas.dtype != torch.float32 or bary.dtype != torch.float32 or p2f.dtype != torch.int64:
        return False
    return atlas.dim() == 4 and atlas.shape[1] >= 1 and p2f.dim() == 4


def _atlas_dispatch(original):
    from . import texture_atlas as ours

    def sample_textures(self, fragments, **kwargs):
        atlas = self.atlas_packed()  # once: the fused path samples this very tensor
        if _atlas_fused(atlas, fragments):
            return ours.sample_textures_atlas(fragments, atlas)
        return original(self, fragments, **kwargs)

    sample_textures.__name__ = "sample_textures"
    sample_textures.__qualname__ = "TexturesAtlas.sample_textures"
    sample_textures.__doc__ = original.__doc__
    return sample_textures


def install_texture_atlas():
    """Patch PyTorch3D's texture atlas sampling (must be importable): the method `sample_textures` of the class
    `TexturesAtlas` in pytorch3d.renderer.mesh.textures, so that existing objects and every import path see it.
    Returns the list of patched module names."""
    m = importlib.import_module(_TEXTURES_MODULE)
    key = (_TEXTURES_MODULE, "TexturesAtlas", "sample_textures")
    if key not in _saved_methods:
        cls = m.TexturesAtlas
        _saved_methods[key] = cls.__dict__["sample_textures"]
        cls.sample_textures = _atlas_dispatch(cls.__dict__["sample_textures"])
    return [_TEXTURES_MODULE]


def _clip_dispatch(name, original):
    from . import clip as ours

    if name == "clip_faces":
        def clip_faces(face_verts_unclipped, mesh_to_face_first_idx, num_faces_per_mesh, frustum):
            if not (getattr(face_verts_unclipped, "is_cuda", False) and face_verts_unclipped.dtype == torch.float32):
                return original(face_verts_unclipped, mesh_to_face_first_idx, num_faces_per_mesh, frustum)
            out = ours.clip_faces_fused(face_verts_unclipped, mesh_to_face_first_idx, num_faces_per_mesh, frustum)
            cls = importlib.import_module("pytorch3d.renderer.mesh.clip").ClippedFaces
            return cls(**{f: getattr(out, f) for f in ours.ClippedFaces.__slots__})

        return clip_faces

    def convert_clipped_rasterization_to_original_faces(pix_to_face_clipped, bary_coords_clipped, clipped_faces):
        conv = getattr(clipped_faces, "barycentric_conversion", None)
        if not (getattr(pix_to_face_clipped, "is_cuda", False) and pix_to_face_clipped.dtype == torch.int64
                and getattr(bary_coords_clipped, "dtype", None) == torch.float32
                and (conv is None or conv.dtype == torch.float32)):
            return original(pix_to_face_clipped, bary_coords_clipped, clipped_faces)
        return ours.convert_clipped_fused(pix_to_face_clipped, bary_coords_clipped, clipped_faces)

    return convert_clipped_rasterization_to_original_faces


def install_clipping():
    """Patch PyTorch3D's frustum culling and z-clipping (must be importable): `clip_faces` and
    `convert_clipped_rasterization_to_original_faces` in pytorch3d.renderer.mesh.rasterize_meshes, which imports them
    by name.  Float32 CUDA inputs go to the fused functions of `pytorch3d_b200.clip`; everything else to the originals.
    Returns the list of patched module names."""
    m = importlib.import_module(_CLIP_MODULE)
    for name in _CLIP_FUNCTIONS:
        if (_CLIP_MODULE, name) not in _saved_blend:
            _saved_blend[(_CLIP_MODULE, name)] = getattr(m, name)
            setattr(m, name, _clip_dispatch(name, getattr(m, name)))
    return [_CLIP_MODULE]


def _mesh_fused(verts, faces):
    """Whether the fused normal ops take these packed tensors: float32 CUDA verts (V, 3) and int64 CUDA faces (F, 3) on
    one device, within the kernels' size limits."""
    if not (getattr(verts, "is_cuda", False) and getattr(faces, "is_cuda", False) and verts.device == faces.device):
        return False
    if verts.dtype != torch.float32 or faces.dtype != torch.int64:
        return False
    if verts.dim() != 2 or verts.shape[1] != 3 or faces.dim() != 2 or faces.shape[1] != 3:
        return False
    return _b200_C.normals_sizes_ok(int(verts.shape[0]), int(faces.shape[0]))


def _face_normals_fused(name, args):
    """The proxied face ops: verts is argument 0 of the forward and 2 of the backward."""
    verts_at = 0 if name == "face_areas_normals_forward" else 2
    if len(args) <= verts_at + 1:
        return False
    return _mesh_fused(args[verts_at], args[verts_at + 1])


def _vertex_normals_dispatch(original):
    from . import normals as ours

    def _compute_vertex_normals(self, refresh: bool = False):
        if not (refresh or any(v is None for v in [self._verts_normals_packed])):
            return
        if not self.isempty():
            verts, faces = self.verts_packed(), self.faces_packed()
            if _mesh_fused(verts, faces):
                self._verts_normals_packed = ours.verts_normals(verts, faces)
                return
        return original(self, refresh=refresh)

    _compute_vertex_normals.__qualname__ = "Meshes._compute_vertex_normals"
    _compute_vertex_normals.__doc__ = original.__doc__
    return _compute_vertex_normals


def install_normals():
    """Patch PyTorch3D's mesh normals (must be importable): `_C` in pytorch3d.ops.mesh_face_areas_normals for the two
    face ops, and the method `_compute_vertex_normals` of the class `Meshes` in pytorch3d.structures.meshes.  Returns
    the list of patched module names."""
    mod = importlib.import_module(_NORMALS_MODULE)
    if (_NORMALS_MODULE, "_C") not in _saved_blend:
        _saved_blend[(_NORMALS_MODULE, "_C")] = mod._C
        mod._C = _Proxy(mod._C, _NORMALS_OPS, _face_normals_fused)
    m = importlib.import_module(_MESHES_MODULE)
    key = (_MESHES_MODULE, "Meshes", "_compute_vertex_normals")
    if key not in _saved_methods:
        cls = m.Meshes
        _saved_methods[key] = cls.__dict__["_compute_vertex_normals"]
        cls._compute_vertex_normals = _vertex_normals_dispatch(cls.__dict__["_compute_vertex_normals"])
    return [_NORMALS_MODULE, _MESHES_MODULE]


def _regularizer_fused(meshes):
    """Whether the fused regularisers take this batch: at least one mesh, float32 CUDA verts and int64 CUDA faces on
    one device, within the kernels' size limits."""
    if len(meshes) == 0:
        return False
    verts, faces = meshes.verts_packed(), meshes.faces_packed()
    return _mesh_fused(verts, faces) and _b200_C.regularizer_sizes_ok(int(verts.shape[0]), int(faces.shape[0]),
                                                                      len(meshes))


def _regularizer_dispatch(name, original):
    from . import regularizers as ours

    if name == "mesh_edge_loss":
        def mesh_edge_loss(meshes, target_length: float = 0.0):
            if _regularizer_fused(meshes):
                return ours.mesh_edge_loss(meshes, target_length)
            return original(meshes, target_length)
        fn = mesh_edge_loss
    elif name == "mesh_laplacian_smoothing":
        def mesh_laplacian_smoothing(meshes, method: str = "uniform"):
            if method in _b200_C.LAPLACIAN_METHODS and _regularizer_fused(meshes):
                return ours.mesh_laplacian_smoothing(meshes, method)
            return original(meshes, method)
        fn = mesh_laplacian_smoothing
    else:
        def mesh_normal_consistency(meshes):
            if _regularizer_fused(meshes):
                return ours.mesh_normal_consistency(meshes)
            return original(meshes)
        fn = mesh_normal_consistency
    fn.__doc__ = original.__doc__
    return fn


def install_regularizers():
    """Patch PyTorch3D's mesh regularisers (must be importable): `mesh_edge_loss`, `mesh_laplacian_smoothing` and
    `mesh_normal_consistency` in pytorch3d.loss and in their defining modules pytorch3d.loss.<name>.  Returns the list
    of patched module names."""
    patched = [_LOSS_PACKAGE]
    package = importlib.import_module(_LOSS_PACKAGE)
    for name in _LOSS_FUNCTIONS:
        modname = _LOSS_PACKAGE + "." + name
        module = importlib.import_module(modname)
        original = module.__dict__[name]
        for owner, key in ((module, modname), (package, _LOSS_PACKAGE)):
            if (key, name) not in _saved_blend:
                _saved_blend[(key, name)] = owner.__dict__[name]
                setattr(owner, name, _regularizer_dispatch(name, original))
        patched.append(modname)
    return patched


def _sampling_fused(meshes, num_samples):
    """Whether the fused sampler takes this call: at least one mesh, float32 CUDA verts and int64 CUDA faces on one
    device, an integer num_samples >= 1, within the kernels' size limits."""
    if len(meshes) == 0 or not isinstance(num_samples, numbers.Integral) or isinstance(num_samples, bool):
        return False
    verts, faces = meshes.verts_packed(), meshes.faces_packed()
    return _mesh_fused(verts, faces) and _b200_C.sampling_sizes_ok(int(verts.shape[0]), int(faces.shape[0]),
                                                                   len(meshes), int(num_samples))


def _sampling_dispatch(original):
    from . import sampling as ours

    def sample_points_from_meshes(meshes, num_samples: int = 10000, return_normals: bool = False,
                                  return_textures: bool = False):
        if _sampling_fused(meshes, num_samples):
            try:
                return ours.sample_points_from_meshes(meshes, num_samples, return_normals, return_textures)
            except ours.EmptyMeshWithTextures:
                pass
        return original(meshes, num_samples, return_normals, return_textures)

    sample_points_from_meshes.__doc__ = original.__doc__
    return sample_points_from_meshes


def install_sampling():
    """Patch PyTorch3D's surface sampling (must be importable): `sample_points_from_meshes` in
    pytorch3d.ops.sample_points_from_meshes and in pytorch3d.ops.  Returns the list of patched module names."""
    package = importlib.import_module(_OPS_PACKAGE)
    module = importlib.import_module(_SAMPLING_MODULE)
    name = "sample_points_from_meshes"
    original = module.__dict__[name]
    for owner, key in ((module, _SAMPLING_MODULE), (package, _OPS_PACKAGE)):
        if (key, name) not in _saved_blend:
            _saved_blend[(key, name)] = owner.__dict__[name]
            setattr(owner, name, _sampling_dispatch(original))
    return [_OPS_PACKAGE, _SAMPLING_MODULE]


_CHAMFER_MODULE = "pytorch3d.loss.chamfer"


def _chamfer_cloud(points, lengths, normals):
    """(points, lengths, normals) as chamfer.py reads them from a tensor or a Pointclouds-like object."""
    if torch.is_tensor(points):
        return points, lengths, normals
    if hasattr(points, "points_padded") and hasattr(points, "num_points_per_cloud"):
        return points.points_padded(), points.num_points_per_cloud(), points.normals_padded()
    return None, None, None


def _chamfer_fused(x, y, x_lengths, y_lengths, x_normals, y_normals, weights, norm, point_reduction):
    """Whether the fused chamfer_distance takes this call: float32 CUDA (N, P, 3) clouds with D = 3 on one device,
    int64 (N,) lengths and float32 (N, P, 3) normals there, float32 (N,) weights that do not require grad, within the
    kernels' size limits.  Calls the reference rejects go to it too, so that it raises."""
    x, x_lengths, x_normals = _chamfer_cloud(x, x_lengths, x_normals)
    y, y_lengths, y_normals = _chamfer_cloud(y, y_lengths, y_normals)
    if x is None or y is None or norm not in (1, 2) or isinstance(norm, bool):
        return False
    if point_reduction == "max" and (x_normals is not None or y_normals is not None):
        return False
    if not (x.is_cuda and x.dtype == torch.float32 and x.dim() == 3 and x.shape[2] == 3):
        return False
    dev = x.device
    if not (y.is_cuda and y.device == dev and y.dtype == torch.float32 and y.dim() == 3 and y.shape[2] == 3
            and y.shape[0] == x.shape[0]):
        return False
    N, P1, P2 = int(x.shape[0]), int(x.shape[1]), int(y.shape[1])
    for t in (x_lengths, y_lengths):
        if t is not None and not (torch.is_tensor(t) and t.is_cuda and t.device == dev and t.dtype == torch.int64
                                  and tuple(t.shape) == (N,)):
            return False
    if x_normals is not None and y_normals is not None:
        for t, P in ((x_normals, P1), (y_normals, P2)):
            if not (torch.is_tensor(t) and t.is_cuda and t.device == dev and t.dtype == torch.float32
                    and tuple(t.shape) == (N, P, 3)):
                return False
    if weights is not None and not (torch.is_tensor(weights) and weights.is_cuda and weights.device == dev
                                    and weights.dtype == torch.float32 and tuple(weights.shape) == (N,)
                                    and not weights.requires_grad):
        return False
    return _b200_C.chamfer_sizes_ok(N, P1, P2)


def _chamfer_dispatch(original):
    from . import chamfer as ours

    def chamfer_distance(x, y, x_lengths=None, y_lengths=None, x_normals=None, y_normals=None, weights=None,
                         batch_reduction="mean", point_reduction="mean", norm: int = 2,
                         single_directional: bool = False, abs_cosine: bool = True):
        args = (x, y, x_lengths, y_lengths, x_normals, y_normals, weights, batch_reduction, point_reduction, norm,
                single_directional, abs_cosine)
        if _chamfer_fused(x, y, x_lengths, y_lengths, x_normals, y_normals, weights, norm, point_reduction):
            return ours.chamfer_distance(*args)
        return original(*args)

    chamfer_distance.__doc__ = original.__doc__
    return chamfer_distance


def install_chamfer():
    """Patch PyTorch3D's chamfer loss (must be importable): `chamfer_distance` in pytorch3d.loss.chamfer and in
    pytorch3d.loss.  Returns the list of patched module names."""
    package = importlib.import_module(_LOSS_PACKAGE)
    module = importlib.import_module(_CHAMFER_MODULE)
    name = "chamfer_distance"
    original = module.__dict__[name]
    for owner, key in ((module, _CHAMFER_MODULE), (package, _LOSS_PACKAGE)):
        if (key, name) not in _saved_blend:
            _saved_blend[(key, name)] = owner.__dict__[name]
            setattr(owner, name, _chamfer_dispatch(original))
    return [_LOSS_PACKAGE, _CHAMFER_MODULE]


_FPS_MODULE = "pytorch3d.ops.sample_farthest_points"
_BALL_MODULE = "pytorch3d.ops.ball_query"


def _cloud_fused(points):
    return (torch.is_tensor(points) and points.is_cuda and points.dtype == torch.float32 and points.dim() == 3
            and points.shape[2] == 3)


def _lengths_fused(lengths, points):
    return lengths is None or (torch.is_tensor(lengths) and lengths.is_cuda and lengths.device == points.device
                               and lengths.dtype == torch.int64 and tuple(lengths.shape) == (points.shape[0],))


def _fps_fused(points, lengths, K):
    """Whether the fused sampler takes this call: float32 CUDA (N, P, 3) points, int64 (N,) lengths (or None) on their
    device, K an int, a list or a tensor on that device, P < 2^31."""
    if not (_cloud_fused(points) and _lengths_fused(lengths, points)):
        return False
    if torch.is_tensor(K):
        if not (K.is_cuda and K.device == points.device):
            return False
    elif not isinstance(K, (int, list)) or isinstance(K, bool):
        return False
    return _b200_C.fps_sizes_ok(int(points.shape[1]))


def _ball_fused(p1, p2, lengths1, lengths2, K):
    """Whether the fused ball query takes this call: float32 CUDA (N, P1, 3) and (N, P2, 3) clouds on one device,
    int64 (N,) lengths (or None) there, an integer K >= 0, within the kernels' size limits."""
    if not (_cloud_fused(p1) and _cloud_fused(p2) and p2.device == p1.device and p2.shape[0] == p1.shape[0]):
        return False
    if not (_lengths_fused(lengths1, p1) and _lengths_fused(lengths2, p1)):
        return False
    if not isinstance(K, numbers.Integral) or isinstance(K, bool):
        return False
    return _b200_C.ball_query_sizes_ok(int(p1.shape[0]), int(p1.shape[1]), int(p2.shape[1]), int(K))


def _fps_dispatch(original):
    from . import point_ops as ours

    def sample_farthest_points(points, lengths=None, K=50, random_start_point: bool = False):
        if _fps_fused(points, lengths, K):
            return ours.sample_farthest_points(points, lengths, K, random_start_point)
        return original(points, lengths, K, random_start_point)

    sample_farthest_points.__doc__ = original.__doc__
    return sample_farthest_points


def _ball_dispatch(original):
    from . import point_ops as ours

    def ball_query(p1, p2, lengths1=None, lengths2=None, K: int = 500, radius: float = 0.2, return_nn: bool = True,
                   skip_points_outside_cube: bool = False):
        args = (p1, p2, lengths1, lengths2, K, radius, return_nn, skip_points_outside_cube)
        if _ball_fused(p1, p2, lengths1, lengths2, K):
            return ours.ball_query(*args)
        return original(*args)

    ball_query.__doc__ = original.__doc__
    return ball_query


def install_point_ops():
    """Patch PyTorch3D's point sampling and grouping (must be importable): `sample_farthest_points` in
    pytorch3d.ops.sample_farthest_points and in pytorch3d.ops, and `ball_query` in pytorch3d.ops.ball_query and in
    pytorch3d.ops.  Returns the list of patched module names."""
    package = importlib.import_module(_OPS_PACKAGE)
    for modname, name, dispatch in ((_FPS_MODULE, "sample_farthest_points", _fps_dispatch),
                                    (_BALL_MODULE, "ball_query", _ball_dispatch)):
        module = importlib.import_module(modname)  # the package's attribute of this name is the function
        original = module.__dict__[name]
        for owner, key in ((module, modname), (package, _OPS_PACKAGE)):
            if (key, name) not in _saved_blend:
                _saved_blend[(key, name)] = owner.__dict__[name]
                setattr(owner, name, dispatch(original))
    return [_OPS_PACKAGE, _FPS_MODULE, _BALL_MODULE]


def _depth_fragments_fused(fragments, soft):
    """int64 CUDA pix_to_face (N, H, W, K) with 1 <= K <= 150, and float32 zbuf (and dists) of its shape on its device."""
    p2f = getattr(fragments, "pix_to_face", None)
    if not (getattr(p2f, "is_cuda", False) and p2f.dtype == torch.int64 and p2f.dim() == 4
            and 1 <= p2f.shape[3] <= _b200_C.kMaxPointsPerPixel):
        return False
    for name in ("zbuf", "dists") if soft else ("zbuf",):
        t = getattr(fragments, name, None)
        if not (getattr(t, "dtype", None) == torch.float32 and t.device == p2f.device and t.shape == p2f.shape):
            return False
    return True


def _real(x):
    return isinstance(x, numbers.Real) and not torch.is_tensor(x)


def _zfar_fused(zfar, device):
    """A real number, or a 1-element float32 tensor (0-d or (1,)) on `device` that does not require grad."""
    if torch.is_tensor(zfar):
        return (zfar.dtype == torch.float32 and zfar.numel() == 1 and zfar.dim() <= 1 and zfar.device == device
                and not zfar.requires_grad)
    return _real(zfar)


def _depth_shader_dispatch(cls, original):
    from . import blending as ours
    soft = cls.__name__ == "SoftDepthShader"

    def forward(self, fragments, meshes, **kwargs):
        if _depth_fragments_fused(fragments, soft):
            cameras = super(cls, self)._get_cameras(**kwargs)  # the reference's error when there are none
            zfar = kwargs.get("zfar", getattr(cameras, "zfar", 100.0))
            if _zfar_fused(zfar, fragments.pix_to_face.device):
                if not soft:
                    return ours.hard_depth(fragments, zfar)
                sigma = self.blend_params.sigma
                if _real(sigma):
                    return ours.soft_depth(fragments, sigma, zfar)
        return original(self, fragments, meshes, **kwargs)

    forward.__qualname__ = cls.__name__ + ".forward"
    forward.__doc__ = original.__doc__
    return forward


def install_depth_shading():
    """Patch PyTorch3D's depth shaders (must be importable): the method `forward` of the classes `SoftDepthShader` and
    `HardDepthShader` in pytorch3d.renderer.mesh.shader, so that existing shaders and every import path see it.
    Returns the list of patched module names."""
    m = importlib.import_module(_SHADER_MODULE)
    for clsname in _DEPTH_SHADERS:
        key = (_SHADER_MODULE, clsname, "forward")
        if key not in _saved_methods:
            cls = getattr(m, clsname)
            _saved_methods[key] = cls.__dict__["forward"]
            cls.forward = _depth_shader_dispatch(cls, cls.__dict__["forward"])
    return [_SHADER_MODULE]


def uninstall():
    """Undo `install()`, `install_blending()`, `install_splatter()`, `install_shading()`, `install_gouraud()`,
    `install_textures()`, `install_texture_atlas()`, `install_clipping()`, `install_normals()`,
    `install_regularizers()`, `install_depth_shading()`, `install_sampling()`, `install_chamfer()` and
    `install_point_ops()`."""
    import importlib
    for modname, original in list(_saved.items()):
        importlib.import_module(modname)._C = original
        del _saved[modname]
    for (modname, name), original in list(_saved_blend.items()):
        setattr(importlib.import_module(modname), name, original)
        del _saved_blend[(modname, name)]
    for (modname, clsname, name), original in list(_saved_methods.items()):
        setattr(getattr(importlib.import_module(modname), clsname), name, original)
        del _saved_methods[(modname, clsname, name)]
