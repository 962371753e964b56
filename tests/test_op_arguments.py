"""Argument checks of the ctypes ops: one row per op.  For every row a small valid call succeeds, and for every tensor
argument a wrong dtype and a wrong shape each raise RuntimeError naming the argument, before anything is launched.

Every bad argument starts with the good one's bytes: a wrong dtype is the same memory viewed as another dtype of the
same width, and a wrong shape is the good tensor stacked twice along a new leading dimension.  A build that forgot a
check therefore reads the valid inputs, and no memory past a buffer."""
import re

import pytest
import torch

DEV = "cuda"
N, H, W, K = 1, 4, 4, 2
SAME_WIDTH = {torch.float32: torch.int32, torch.int32: torch.float32, torch.int64: torch.float64,
              torch.bool: torch.uint8, torch.uint8: torch.int8}


def _g(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _rand(*shape, seed=0):
    return torch.rand(*shape, generator=_g(seed), device=DEV)


def _idx(lo, hi, *shape, dtype=torch.int64, seed=0):
    return torch.randint(lo, hi, shape, generator=_g(seed), device=DEV, dtype=dtype)


def _slots(F, seed=1):
    return _idx(-1, F, N, H, W, K, seed=seed)


def _compositing(name):
    def build():
        from pytorch3d_b200 import _C
        t = dict(grad_outputs=_rand(N, 3, H, W), features=_rand(3, 10), alphas=_rand(N, K, H, W),
                 points_idx=_idx(-1, 10, N, K, H, W))
        return t, lambda t: getattr(_C, name)(t["grad_outputs"], t["features"], t["alphas"], t["points_idx"])
    return build


def _alphacomposite():
    from pytorch3d_b200 import _C
    t = dict(features=_rand(3, 10), alphas=_rand(N, K, H, W), points_idx=_idx(-1, 10, N, K, H, W))
    return t, lambda t: _C.accum_alphacomposite(t["features"], t["alphas"], t["points_idx"])


def _points_alpha_render_backward():
    from pytorch3d_b200 import _C
    t = dict(grad_images=_rand(N, 3, H, W), features=_rand(3, 10), idx=_idx(-1, 10, N, H, W, K, dtype=torch.int32),
             dists=_rand(N, H, W, K))
    return t, lambda t: _C.points_alpha_render_backward(t["grad_images"], t["features"], t["idx"], t["dists"], 0.5)


def _interp(backward):
    def build():
        from pytorch3d_b200 import _C
        t = dict(pix_to_face=_idx(-1, 5, 8), barycentric_coords=_rand(8, 3), face_attrs=_rand(5, 3, 2))
        if not backward:
            return t, lambda t: _C.interp_face_attrs_forward(t["pix_to_face"], t["barycentric_coords"],
                                                             t["face_attrs"])
        t["grad_pix_attrs"] = _rand(8, 2)
        return t, lambda t: _C.interp_face_attrs_backward(t["pix_to_face"], t["barycentric_coords"], t["face_attrs"],
                                                          t["grad_pix_attrs"])
    return build


def _clip_scene():
    from pytorch3d_b200 import _C
    from pytorch3d_b200.clip import ClipFrustum
    fv = _rand(10, 3, 3) * 3.0 - 1.5
    fv[..., 2] = _rand(10, 3, seed=1) * 2.0 - 0.4
    fr = ClipFrustum(z_clip_value=0.3)
    ws = _C.clip_faces_count(fr, face_verts=fv)
    return fv, fr, ws, ws[:4].tolist()


def _clip_faces_fill():
    from pytorch3d_b200 import _C
    fv, fr, ws, rec = _clip_scene()
    t = dict(face_verts=fv, mesh_to_face_first_idx=torch.tensor([0, 4], device=DEV),
             num_faces_per_mesh=torch.tensor([4, 6], device=DEV), workspace=ws)
    return t, lambda t: _C.clip_faces_fill(t["face_verts"], t["mesh_to_face_first_idx"], t["num_faces_per_mesh"], fr,
                                           t["workspace"], rec)


def _clip_faces_backward():
    from pytorch3d_b200 import _C
    fv, fr, ws, rec = _clip_scene()
    assert rec[1] + rec[2] > 0, rec
    t = dict(face_verts=fv, workspace=ws, grad_face_verts_clipped=_rand(rec[0], 3, 3),
             grad_conversion=_rand(rec[1] + 2 * rec[2], 3, 3))
    return t, lambda t: _C.clip_faces_backward(t["face_verts"], fr, t["workspace"], rec, t["grad_face_verts_clipped"],
                                               t["grad_conversion"])


def _clip_convert(backward):
    def build():
        from pytorch3d_b200 import _C
        t = dict(pix_to_face=_slots(3), barycentric_coords=_rand(N, H, W, K, 3),
                 barycentric_conversion=_rand(2, 3, 3),
                 faces_clipped_to_conversion_idx=torch.tensor([0, -1, 1], device=DEV))
        if not backward:
            t["faces_clipped_to_unclipped_idx"] = torch.tensor([0, 2, 4], device=DEV)
            return t, lambda t: _C.clip_convert_forward(t["pix_to_face"], t["barycentric_coords"],
                                                        t["faces_clipped_to_unclipped_idx"],
                                                        t["barycentric_conversion"],
                                                        t["faces_clipped_to_conversion_idx"])
        t["grad_bary_unclipped"] = _rand(N, H, W, K, 3, seed=2)
        return t, lambda t: _C.clip_convert_backward(t["grad_bary_unclipped"], t["pix_to_face"],
                                                     t["barycentric_coords"], t["barycentric_conversion"],
                                                     t["faces_clipped_to_conversion_idx"])
    return build


def _chamfer_inputs():
    return dict(x=_rand(2, 5, 3), y=_rand(2, 6, 3, seed=1), x_lengths=torch.tensor([5, 4], device=DEV),
                y_lengths=torch.tensor([6, 6], device=DEV), x_normals=_rand(2, 5, 3, seed=2),
                y_normals=_rand(2, 6, 3, seed=3), weights=_rand(2, seed=4))


_CHAMFER_OPTS = (2, "mean", "mean", False, False)


def _chamfer_forward():
    from pytorch3d_b200 import _C
    return _chamfer_inputs(), lambda t: _C.chamfer_forward(*list(t.values())[:7], *_CHAMFER_OPTS)


def _chamfer_backward():
    from pytorch3d_b200 import _C
    t = _chamfer_inputs()
    _, state, _ = _C.chamfer_forward(*t.values(), *_CHAMFER_OPTS)
    names = ("x", "y", "x_lengths", "y_lengths", "x_normals", "y_normals", "weights")
    t.update(idx_x=state[1], idx_y=state[3], cloud=state[4], argmax=state[5],
             grad_loss_x=_rand((), seed=5), grad_normals_x=_rand((), seed=6))

    def call(t):
        state = (None, t["idx_x"], None, t["idx_y"], t["cloud"], t["argmax"])
        return _C.chamfer_backward(*(t[k] for k in names), *_CHAMFER_OPTS, state,
                                   (t["grad_loss_x"], None, t["grad_normals_x"], None), True, True)
    return t, call


def _sigmoid_alpha_blend_backward():
    from pytorch3d_b200 import _C
    t = dict(grad_alphas=_rand(N, H, W), alphas=_rand(N, H, W, seed=1), distances=_rand(N, H, W, K, seed=2),
             pix_to_face=_slots(5))
    return t, lambda t: _C.sigmoid_alpha_blend_backward(t["grad_alphas"], t["alphas"], t["distances"],
                                                        t["pix_to_face"], 1e-4)


def _softmax_rgb_blend_backward():
    from pytorch3d_b200 import _C
    t = dict(grad_out=_rand(N, H, W, 4), colors=_rand(N, H, W, K, 3), pix_to_face=_slots(5),
             zbuf=_rand(N, H, W, K, seed=2), dists=_rand(N, H, W, K, seed=3))
    return t, lambda t: _C.softmax_rgb_blend_backward(t["grad_out"], t["colors"], t["pix_to_face"], t["zbuf"],
                                                      t["dists"], 1e-4, 1e-4, (1.0, 1.0, 1.0))


def _soft_depth_blend_backward():
    from pytorch3d_b200 import _C
    t = dict(grad_out=_rand(N, H, W, 1), pix_to_face=_slots(5), zbuf=_rand(N, H, W, K, seed=2),
             dists=_rand(N, H, W, K, seed=3))
    return t, lambda t: _C.soft_depth_blend_backward(t["grad_out"], t["pix_to_face"], t["zbuf"], t["dists"], 1e-4,
                                                     100.0)


def _splatter_blend_backward():
    from pytorch3d_b200 import _C
    t = dict(grad_out=_rand(N, H, W, 4), colors=_rand(N, H, W, K, 3), pixel_coords_screen=_rand(N, H, W, K, 3) * 4,
             background_mask=_rand(N, H, W, K, seed=3) < 0.3)
    return t, lambda t: _C.splatter_blend_backward(t["grad_out"], t["colors"], t["pixel_coords_screen"],
                                                   t["background_mask"], 0.5, (1.0, 1.0, 1.0))


def _shading_forward():
    from pytorch3d_b200 import _C
    t = dict(pix_to_face=_slots(5), barycentric_coords=_rand(N, H, W, K, 3), face_positions=_rand(5, 3, 3),
             face_normals=_rand(5, 3, 3, seed=2), texels=_rand(N, H, W, K, 3, seed=3),
             params=torch.zeros(N, _C.SHADING_PARAMS, device=DEV))
    return t, lambda t: _C.shading_forward(*t.values(), False, "point")


def _gouraud_backward():
    from pytorch3d_b200 import _C
    t = dict(grad_colors=_rand(N, H, W, K, 3), verts=_rand(6, 3), normals=_rand(6, 3, seed=1),
             verts_colors=_rand(6, 3, seed=2), mesh_first_vert=torch.tensor([0], device=DEV),
             mesh_num_verts=torch.tensor([6], device=DEV), params=torch.zeros(1, _C.SHADING_PARAMS, device=DEV),
             faces=_idx(0, 6, 5, 3), pix_to_face=_slots(5), barycentric_coords=_rand(N, H, W, K, 3, seed=3),
             verts_shaded=_rand(6, 3, seed=4))
    args = ("grad_colors", "verts", "normals", "verts_colors", "mesh_first_vert", "mesh_num_verts", "params", "faces",
            "pix_to_face", "barycentric_coords")
    return t, lambda t: _C.gouraud_backward(*(t[k] for k in args), "point", t["verts_shaded"])


def _texture_uv_backward():
    from pytorch3d_b200 import _C
    t = dict(grad_texels=_rand(N, H, W, K, 3), pix_to_face=_slots(5), barycentric_coords=_rand(N, H, W, K, 3, seed=1),
             face_uvs=_rand(5, 3, 2, seed=2), maps=_rand(N, 6, 7, 3, seed=3))
    return t, lambda t: _C.texture_uv_backward(*t.values())


def _texture_atlas_backward():
    from pytorch3d_b200 import _C
    t = dict(grad_texels=_rand(N, H, W, K, 3), pix_to_face=_slots(5), barycentric_coords=_rand(N, H, W, K, 3, seed=1),
             atlas=_rand(5, 4, 4, 3, seed=2))
    return t, lambda t: _C.texture_atlas_backward(*t.values())


def _verts_normals_backward():
    from pytorch3d_b200 import _C
    verts, faces = _rand(6, 3), _idx(0, 6, 5, 3)
    _, table, sums = _C.verts_normals_forward(verts, faces)
    t = dict(grad_normals=_rand(6, 3, seed=1), verts=verts, faces=faces, table=table, sums=sums)
    return t, lambda t: _C.verts_normals_backward(*t.values())


def _sample_points_backward():
    from pytorch3d_b200 import _C
    t = dict(grad_samples=_rand(2, 7, 3), grad_normals=_rand(2, 7, 3, seed=1), verts=_rand(6, 3, seed=2),
             faces=_idx(0, 6, 5, 3), face_idx=_idx(0, 5, 2, 7), bary=_rand(2, 7, 3, seed=3))
    return t, lambda t: _C.sample_points_backward(*t.values())


def _mesh_edge_loss_backward():
    from pytorch3d_b200 import _C
    t = dict(verts=_rand(6, 3), faces=_idx(0, 6, 5, 3), mesh_first_vert=torch.tensor([0], device=DEV),
             mesh_num_verts=torch.tensor([6], device=DEV))
    _, ws = _C.mesh_edge_loss_forward(*t.values(), 0.5)
    t.update(grad_loss=torch.ones((), device=DEV), workspace=ws)
    return t, lambda t: _C.mesh_edge_loss_backward(t["grad_loss"], t["verts"], t["faces"], t["mesh_first_vert"],
                                                   t["mesh_num_verts"], 0.5, t["workspace"])


# (row, builder, arguments without a wrong-dtype case, arguments without a wrong-shape case): chamfer_backward casts its
# upstream gradients to float32; any contiguous uint8 workspace at least as large as the forward's is accepted; and
# clip_convert_backward takes pix_to_face of any shape, barycentric_coords (checked) giving its size, so a larger
# pix_to_face is no wrong shape there but would make a build without that check read past barycentric_coords.
ROWS = [
    ("accum_alphacomposite", _alphacomposite, (), ()),
    ("accum_alphacomposite_backward", _compositing("accum_alphacomposite_backward"), (), ()),
    ("accum_weightedsum_backward", _compositing("accum_weightedsum_backward"), (), ()),
    ("accum_weightedsumnorm_backward", _compositing("accum_weightedsumnorm_backward"), (), ()),
    ("points_alpha_render_backward", _points_alpha_render_backward, (), ()),
    ("interp_face_attrs_forward", _interp(False), (), ()),
    ("interp_face_attrs_backward", _interp(True), (), ()),
    ("clip_faces_fill", _clip_faces_fill, (), ()),
    ("clip_faces_backward", _clip_faces_backward, (), ()),
    ("clip_convert_forward", _clip_convert(False), (), ()),
    ("clip_convert_backward", _clip_convert(True), (), ("pix_to_face",)),
    ("chamfer_forward", _chamfer_forward, (), ()),
    ("chamfer_backward", _chamfer_backward, ("grad_loss_x", "grad_normals_x"), ()),
    ("sigmoid_alpha_blend_backward", _sigmoid_alpha_blend_backward, (), ()),
    ("softmax_rgb_blend_backward", _softmax_rgb_blend_backward, (), ()),
    ("soft_depth_blend_backward", _soft_depth_blend_backward, (), ()),
    ("splatter_blend_backward", _splatter_blend_backward, (), ()),
    ("shading_forward", _shading_forward, (), ()),
    ("gouraud_backward", _gouraud_backward, (), ()),
    ("texture_uv_backward", _texture_uv_backward, (), ()),
    ("texture_atlas_backward", _texture_atlas_backward, (), ()),
    ("verts_normals_backward", _verts_normals_backward, (), ()),
    ("sample_points_backward", _sample_points_backward, (), ()),
    ("mesh_edge_loss_backward", _mesh_edge_loss_backward, (), ("workspace",)),
]


def _wrong_dtype(t):
    return t.view(SAME_WIDTH[t.dtype])


def _wrong_shape(t):
    return t.unsqueeze(0).expand(2, *t.shape).contiguous()


@pytest.mark.gpu
@pytest.mark.parametrize("row", ROWS, ids=[r[0] for r in ROWS])
def test_arguments_are_checked(built_lib, row):
    _, build, no_dtype, no_shape = row
    tensors, call = build()
    call(tensors)
    torch.cuda.synchronize()
    for name in tensors:
        for kind, bad in (("dtype", _wrong_dtype), ("shape", _wrong_shape)):
            if name in (no_dtype if kind == "dtype" else no_shape):
                continue
            with pytest.raises(RuntimeError, match=r"\b%s\b" % re.escape(name)) as err:
                call(dict(tensors, **{name: bad(tensors[name])}))
            assert type(err.value) is RuntimeError, (name, kind)
    torch.cuda.synchronize()


# Exact dtype errors of the drop-ins for pytorch3d._C and of the per-slot index tensors: ATen's texts, which the
# reference raises, with the argument named at the end of data_ptr<T>()'s.
DTYPE_TEXTS = [
    ("accum_alphacomposite", "features", "expected scalar type Float but found torch.int32 for features"),
    ("accum_alphacomposite", "points_idx", "expected scalar type Long but found torch.float64 for points_idx"),
    ("accum_weightedsum_backward", "alphas", "expected scalar type Float but found torch.int32 for alphas"),
    ("points_alpha_render_backward", "idx", "expected scalar type Int but found torch.float32 for idx"),
    ("interp_face_attrs_forward", "pix_to_face", "expected scalar type Long but found torch.float64 for pix_to_face"),
    ("interp_face_attrs_backward", "face_attrs", "expected scalar type Float but found torch.int32 for face_attrs"),
    ("sigmoid_alpha_blend_backward", "distances",
     "Expected tensor for distances to have scalar type Float; but got torch.int32"),
    ("sigmoid_alpha_blend_backward", "pix_to_face", "expected scalar type Long but found torch.float64 for pix_to_face"),
    ("splatter_blend_backward", "background_mask",
     "expected scalar type Bool but found torch.uint8 for background_mask"),
    ("texture_uv_backward", "maps", "Expected tensor for maps to have scalar type Float; but got torch.int32"),
    ("gouraud_backward", "faces", "expected scalar type Long but found torch.float64 for faces"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("row, name, text", DTYPE_TEXTS, ids=["%s-%s" % r[:2] for r in DTYPE_TEXTS])
def test_dtype_error_texts(built_lib, row, name, text):
    tensors, call = dict((r[0], r[1]) for r in ROWS)[row]()
    with pytest.raises(RuntimeError) as err:
        call(dict(tensors, **{name: _wrong_dtype(tensors[name])}))
    assert str(err.value) == text
