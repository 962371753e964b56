"""Times the fused Gouraud shading on the GPU against the torch chain of the reference's
pytorch3d/renderer/mesh/shading.py gouraud_shading (tests/test_gouraud.py: chain_gouraud).  CUDA events after warm-up,
peak memory of forward + backward; the card's name and power limit are read in the same run.

    python tools/time_gouraud.py OUT_DIR        -> OUT_DIR/time_gouraud.json

Workloads: the north-star Fragments (8 tori of 187 x 187, 512 x 512, K = 8, no blur) from the rasterizer, and
8 x 256 x 256 at K = 50 with random faces of the same tori and random barycentrics (tools/time_shading.py).  One point
light, shininess 64, random per-vertex colours; the vertices and colours require grad, the light, material and camera
tensors do not.  The chain forms the camera centre once per mesh and gathers it per vertex; the reference builds V
world-to-view transforms for it, so the chain understates the reference's cost.
Stage times: `*_vertex_stage_us` is the `_C` call with no slots (the vertex kernel alone, plus in the backward the
zeroing of the per-vertex workspace); `*_slot_stage_us` is the full `_C` call minus it.  `fused_backward_us` /
`chain_backward_us` are autograd's backward (fresh .grad fields); `fused_backward_kernel_us` the `_C` backward alone.
Bandwidth: algorithmic bytes over time, as a fraction of the H100 SXM's 3.35 TB/s -- forward 32 B per slot
(pix_to_face 8, barycentrics 12, colours 12) + 24 B per face (its vertex indices) + 48 B per vertex (position, normal,
colour read, shaded colour written); backward 32 B per slot (pix_to_face, barycentrics, upstream gradient; the timed
call requests no barycentric gradient) + 24 B per face + 120 B per vertex (shaded colour read, workspace read-modify-written, position, normal,
colour and workspace read again, three gradients written).
"""
import json
import os
import subprocess
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]

from time_blend import _events_ms, _peak_bytes, _time_backward_ms  # noqa: E402
from time_shading import north_star_scene, random_scene  # noqa: E402

PEAK_BYTES_PER_S = 3.35e12


class _Mesh:
    """The packed-mesh accessors gouraud_shading reads, over fixed tensors (equal-sized tori)."""

    def __init__(self, verts, faces, normals, colors, first, num):
        self._t = (verts, faces, normals, first, num)
        self.textures = types.SimpleNamespace(verts_features_packed=lambda: colors)

    def __len__(self):
        return int(self._t[3].shape[0])

    def verts_packed(self):
        return self._t[0]

    def faces_packed(self):
        return self._t[1]

    def verts_normals_packed(self):
        return self._t[2]

    def mesh_to_verts_packed_first_idx(self):
        return self._t[3]

    def num_verts_per_mesh(self):
        return self._t[4]


def measure(name, m, p2f, bary, dev, iters):
    import test_gouraud as tg
    from pytorch3d_b200 import _C
    from pytorch3d_b200.shading import _params, gouraud_shading
    N, H, W, K = (int(v) for v in p2f.shape)
    F, V = int(m.faces_packed().shape[0]), int(m.verts_packed().shape[0])
    g = torch.Generator(device=dev).manual_seed(2)
    grad = torch.randn(N, H, W, K, 3, generator=g, device=dev)
    lights = types.SimpleNamespace(ambient_color=torch.tensor([[0.3, 0.3, 0.3]], device=dev),
                                   diffuse_color=torch.tensor([[0.6, 0.5, 0.4]], device=dev),
                                   specular_color=torch.tensor([[0.3, 0.3, 0.3]], device=dev),
                                   location=torch.tensor([[0.5, 1.0, -1.0]], device=dev))
    cameras = types.SimpleNamespace(get_camera_center=lambda: torch.zeros(1, 3, device=dev))
    materials = types.SimpleNamespace(ambient_color=torch.ones(1, 3, device=dev),
                                      diffuse_color=torch.ones(1, 3, device=dev),
                                      specular_color=torch.ones(1, 3, device=dev),
                                      shininess=torch.tensor([64.0], device=dev))
    verts = m.verts_packed().detach().clone().requires_grad_(True)
    colors = torch.rand(V, 3, generator=g, device=dev).requires_grad_(True)
    faces = m.faces_packed()
    normals = m.verts_normals_packed().detach()
    first = torch.zeros(N, dtype=torch.int64, device=dev)
    num = torch.full((N,), V // N, dtype=torch.int64, device=dev)
    first[1:] = torch.cumsum(num, 0)[:-1]
    mesh = _Mesh(verts, faces, normals, colors, first, num)
    frags = types.SimpleNamespace(pix_to_face=p2f, bary_coords=bary)
    leaves = [verts, colors]
    slots = N * H * W * K
    bytes_fwd, bytes_bwd = 32 * slots + 24 * F + 48 * V, 32 * slots + 24 * F + 120 * V
    params = _params(N, lights, cameras, materials, "point", dev)
    v, c = verts.detach(), colors.detach()
    none_p2f, none_bary = p2f[:0], bary[:0]

    def fwd(pf, br):
        return _C.gouraud_forward(v, normals, c, first, num, params, faces, pf, br, "point")

    shaded = fwd(p2f, bary)[1]
    needs = (True, False, True, False, False)

    def bwd(pf, br, gr):
        return _C.gouraud_backward(gr, v, normals, c, first, num, params, faces, pf, br, "point", shaded, needs)

    def fused():
        return gouraud_shading(mesh, frags, lights, cameras, materials)

    def chain():
        return tg.chain_gouraud(mesh, frags, lights, cameras, materials)

    res = {"N": N, "H": H, "W": W, "K": K, "F": F, "V": V, "slots": slots,
           "background_fraction": float((p2f < 0).float().mean())}
    with torch.no_grad():
        for _ in range(3):
            fwd(p2f, bary)
        res["fused_forward_us"] = 1e3 * _events_ms(lambda: fwd(p2f, bary), iters)
        res["fused_forward_vertex_stage_us"] = 1e3 * _events_ms(lambda: fwd(none_p2f, none_bary), iters)
        res["fused_forward_slot_stage_us"] = res["fused_forward_us"] - res["fused_forward_vertex_stage_us"]
        for _ in range(2):
            bwd(p2f, bary, grad)
        res["fused_backward_kernel_us"] = 1e3 * _events_ms(lambda: bwd(p2f, bary, grad), iters)
        res["fused_backward_vertex_stage_us"] = 1e3 * _events_ms(lambda: bwd(none_p2f, none_bary, grad[:0]), iters)
        res["fused_backward_slot_stage_us"] = res["fused_backward_kernel_us"] - res["fused_backward_vertex_stage_us"]
    for _ in range(2):
        fused().backward(grad)
    res["fused_backward_us"] = 1e3 * _time_backward_ms(fused, grad, leaves, iters)
    for leaf in leaves:
        leaf.grad = None
    res["fused_peak_bytes_fwd_bwd"] = _peak_bytes(lambda: fused().backward(grad))
    res["fused_forward_bandwidth_fraction"] = bytes_fwd / (res["fused_forward_us"] * 1e-6) / PEAK_BYTES_PER_S
    res["fused_backward_bandwidth_fraction"] = bytes_bwd / (res["fused_backward_kernel_us"] * 1e-6) / PEAK_BYTES_PER_S
    try:
        for leaf in leaves:
            leaf.grad = None
        with torch.no_grad():
            want = chain()
            got = fused()
            res["max_abs_diff_forward"] = float((got - want).abs().max())
            del want, got
            for _ in range(2):
                chain()
            res["chain_forward_us"] = 1e3 * _events_ms(chain, max(3, iters // 4))
        chain().backward(grad)
        res["chain_backward_us"] = 1e3 * _time_backward_ms(chain, grad, leaves, max(3, iters // 4))
        for leaf in leaves:
            leaf.grad = None
        res["chain_peak_bytes_fwd_bwd"] = _peak_bytes(lambda: chain().backward(grad))
        res["forward_speedup"] = res["chain_forward_us"] / res["fused_forward_us"]
        res["backward_speedup"] = res["chain_backward_us"] / res["fused_backward_us"]
    except torch.cuda.OutOfMemoryError:
        res["chain"] = "out of memory"
    for leaf in leaves:
        leaf.grad = None
    torch.cuda.empty_cache()
    print(name, json.dumps(res), flush=True)
    return res


def main():
    out_dir = sys.argv[1] if len(sys.argv) > 1 else "."
    assert torch.cuda.is_available(), "time_gouraud.py measures on a CUDA device"
    dev = torch.device("cuda:0")
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               stdout=subprocess.PIPE, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = "not measured"
    report = {"device": torch.cuda.get_device_name(dev), "power_limit": power, "workloads": {}}
    report["workloads"]["north_star_8x512x512_K8"] = measure("north_star", *north_star_scene(dev), dev, 20)
    report["workloads"]["random_8x256x256_K50"] = measure("random_K50", *random_scene(8, 256, 256, 50, dev), dev, 20)
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "time_gouraud.json"), "w") as fh:
        json.dump(report, fh, indent=1)
    print(json.dumps({"device": report["device"], "power_limit": power}))


if __name__ == "__main__":
    main()
