"""Writes tests/golden/reference_golden_sampling.npz: the reference's own sample_points_from_meshes
(pytorch3d/ops/sample_points_from_meshes.py, with ops/mesh_face_areas_normals.py, ops/packed_to_padded.py,
structures/meshes.py and renderer/mesh/textures.py) on the CPU, on the seeded scenes of tests/test_sampling.py
(SCENES), in the record format of make_reference_golden.py (tests/helpers.py: reference_record) with every row kept.

The reference modules are imported with stand-ins only for the packages around them, as make_regularizers_golden.py
does; `pytorch3d._C` is the reference's own CPU face-area and packed-to-padded ops, built by
oracle/build_ref_normals.py and oracle/build_ref_sampling.py.  Each scene runs under
torch.manual_seed(test_sampling.SEED); the draws that produced the outputs are recovered by re-seeding and replaying
the reference's multinomial, then rand, calls with the same shapes and in the same order.  Each output is its own case:
  sampling/<scene>/face, u, v          the draws: packed face ids (N, S) (0 in rows of meshes without faces), u, v
  sampling/<scene>/samples, normals    the outputs with return_normals=True
  sampling/<scene>/grad_samples        d/d verts of (samples * gs).sum(), gs of test_sampling.upstream
  sampling/<scene>/grad_normals        d/d verts of (samples * gs + normals * gn).sum()
  sampling/<scene>/textures_vertex, textures_uv   return_textures=True with a TexturesVertex / TexturesUV (scenes of
                                                  TEXTURED only)
  sampling/zero_total/error            the CPU reference's error on a mesh whose faces all have zero area (bytes)

    python tests/golden/make_sampling_golden.py [OUT_DIR]
"""
import importlib.util
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.dirname(HERE)]

from helpers import reference_record  # noqa: E402
from oracle import build_ref, build_ref_normals, build_ref_sampling  # noqa: E402


def put(store, case, array):
    for field, v in reference_record([array], 1, 1 << 20)[0].items():
        store["%s/0/%s" % (case, field)] = v


def _load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod
    spec.loader.exec_module(mod)
    return mod


def reference_modules():
    ref = os.path.join(build_ref.REF, "pytorch3d")
    p2p_op, fan_op = build_ref_sampling.load(), build_ref_normals.load()
    assert p2p_op is not None, "build oracle/_ref/ref_sampling_cpu.so first (python oracle/build_ref_sampling.py)"
    assert fan_op is not None, "build oracle/_ref/ref_normals_cpu.so first (python oracle/build_ref_normals.py)"
    op = types.SimpleNamespace(packed_to_padded=p2p_op.packed_to_padded, padded_to_packed=p2p_op.padded_to_packed,
                               face_areas_normals_forward=fan_op.face_areas_normals_forward,
                               face_areas_normals_backward=fan_op.face_areas_normals_backward)
    stub_names = ("pytorch3d", "pytorch3d.ops", "pytorch3d.structures", "pytorch3d.renderer", "pytorch3d.renderer.mesh")
    stubs = {n: types.ModuleType(n) for n in stub_names}
    for m in stubs.values():
        m.__path__ = []
    stubs["pytorch3d"].__path__ = [ref]  # pytorch3d.common imports as the reference's own
    stubs["pytorch3d"]._C = op
    sys.modules.update(stubs)
    interp = _load("pytorch3d.ops.interp_face_attrs", os.path.join(ref, "ops", "interp_face_attrs.py"))
    stubs["pytorch3d.ops"].interpolate_face_attributes = interp.interpolate_face_attributes
    _load("pytorch3d.structures.utils", os.path.join(ref, "structures", "utils.py"))
    _load("pytorch3d.renderer.mesh.utils", os.path.join(ref, "renderer", "mesh", "utils.py"))
    fan = _load("pytorch3d.ops.mesh_face_areas_normals", os.path.join(ref, "ops", "mesh_face_areas_normals.py"))
    p2p = _load("pytorch3d.ops.packed_to_padded", os.path.join(ref, "ops", "packed_to_padded.py"))
    textures = _load("pytorch3d.renderer.mesh.textures", os.path.join(ref, "renderer", "mesh", "textures.py"))
    # renderer/mesh/rasterizer.py imports the cameras and the rasterizer; the sampler only builds its Fragments
    rast = types.ModuleType("pytorch3d.renderer.mesh.rasterizer")
    from pytorch3d_b200.rasterizer import Fragments
    rast.Fragments = Fragments
    sys.modules[rast.__name__] = rast
    meshes = _load("pytorch3d.structures.meshes", os.path.join(ref, "structures", "meshes.py"))
    sampler = _load("pytorch3d.ops.sample_points_from_meshes",
                    os.path.join(ref, "ops", "sample_points_from_meshes.py"))
    return types.SimpleNamespace(meshes=meshes, textures=textures, sampler=sampler, fan=fan, p2p=p2p)


def replay_draws(ref, m, S):
    """The reference's draws for `m`, replayed from the current seed: multinomial over the padded areas, then rand."""
    verts, faces = m.verts_packed(), m.faces_packed()
    mesh_to_face = m.mesh_to_faces_packed_first_idx()
    areas, _ = ref.fan.mesh_face_areas_normals(verts.detach(), faces)
    max_faces = m.num_faces_per_mesh().max().item()
    areas_padded = ref.p2p.packed_to_padded(areas, mesh_to_face[m.valid], max_faces)
    idx = areas_padded.multinomial(S, replacement=True) + mesh_to_face[m.valid].view(-1, 1)
    uv = torch.rand(2, idx.shape[0], S, dtype=verts.dtype)
    N = len(m)
    face = torch.zeros((N, S), dtype=torch.int64)
    u = torch.zeros((N, S))
    v = torch.zeros((N, S))
    face[m.valid], u[m.valid], v[m.valid] = idx, uv[0], uv[1]
    return face, u, v


def record(ts):
    saved = {n: m for n, m in sys.modules.items() if n == "pytorch3d" or n.startswith("pytorch3d.")}
    store = {}
    try:
        ref = reference_modules()
        for name in ts.SCENES:
            s = ts.scene(name)
            S = ts.NUM_SAMPLES
            gs, gn = ts.upstream(name, (len(s["faces_list"]), S))
            leaf = s["verts"].clone().requires_grad_(True)
            m = ref.meshes.Meshes(verts=list(torch.split(leaf, s["nverts"])), faces=s["faces_list"])
            torch.manual_seed(ts.SEED)
            samples, normals = ref.sampler.sample_points_from_meshes(m, S, return_normals=True)
            torch.manual_seed(ts.SEED)
            face, u, v = replay_draws(ref, m, S)
            for field, t in (("face", face), ("u", u), ("v", v), ("samples", samples), ("normals", normals)):
                put(store, "sampling/%s/%s" % (name, field), t.detach())
            (samples * gs).sum().backward(retain_graph=True)
            put(store, "sampling/%s/grad_samples" % name, leaf.grad.clone())
            leaf.grad = None
            ((samples * gs).sum() + (normals * gn).sum()).backward()
            put(store, "sampling/%s/grad_normals" % name, leaf.grad.clone())
            if name in ts.TEXTURED:
                tex = ts.textures(s)
                tv = ref.textures.TexturesVertex(verts_features=list(torch.split(tex["colors"], s["nverts"])))
                tu = ref.textures.TexturesUV(maps=tex["maps"], faces_uvs=tex["faces_uvs"], verts_uvs=tex["verts_uvs"])
                for field, t in (("textures_vertex", tv), ("textures_uv", tu)):
                    mt = ref.meshes.Meshes(verts=list(torch.split(s["verts"], s["nverts"])), faces=s["faces_list"],
                                           textures=t)
                    torch.manual_seed(ts.SEED)
                    _, out = ref.sampler.sample_points_from_meshes(mt, S, return_textures=True)
                    torch.manual_seed(ts.SEED)
                    assert torch.equal(replay_draws(ref, mt, S)[0], face)
                    put(store, "sampling/%s/%s" % (name, field), out)
        s = ts.scene("zero_total")
        m = ref.meshes.Meshes(verts=list(torch.split(s["verts"], s["nverts"])), faces=s["faces_list"])
        try:
            ref.sampler.sample_points_from_meshes(m, 10)
            raise AssertionError("the reference sampled a mesh of zero total area")
        except RuntimeError as e:
            msg = str(e)
        store["sampling/zero_total/error/0/message"] = np.frombuffer(msg.encode(), np.uint8)
    finally:
        for n in [n for n in sys.modules if n == "pytorch3d" or n.startswith("pytorch3d.")]:
            del sys.modules[n]
        sys.modules.update(saved)
    return store


def main():
    import test_sampling as ts
    out_dir = sys.argv[1] if len(sys.argv) > 1 else HERE
    torch.set_grad_enabled(True)
    store = record(ts)
    out = os.path.join(out_dir, "reference_golden_sampling.npz")
    np.savez_compressed(out, **store)
    print("wrote %s: %d arrays, %d bytes" % (out, len(store), os.path.getsize(out)))
    assert os.path.getsize(out) < 1 << 20, "%s is larger than 1 MB: store fewer samples" % out


if __name__ == "__main__":
    main()
