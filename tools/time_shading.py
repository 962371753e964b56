"""Times the fused Phong shading on the GPU against the torch chain of the reference's
pytorch3d/renderer/mesh/shading.py and renderer/lighting.py (tests/test_shading.py: chain_phong).  CUDA events after
warm-up, peak memory of forward + backward; the card's name and power limit are read in the same run.

    python tools/time_shading.py OUT_DIR        -> OUT_DIR/time_shading.json

Workloads: the north-star Fragments (8 tori of 187 x 187, 512 x 512, K = 8, no blur) from the rasterizer, and
8 x 256 x 256 at K = 50 with random faces of the same tori and random barycentrics.  One point light, shininess 64,
random texels; the vertices and texels require grad, the light, material and camera tensors do not.
Backward times: `fused_backward_us` / `chain_backward_us` are autograd's backward (with fresh .grad fields; for the
fused op this includes torch's scatter of the face gradients to the vertices); `fused_backward_kernel_us` is the `_C`
backward call alone, which the backward bandwidth fraction uses.
Bandwidth: algorithmic bytes over time, as a fraction of the H100 SXM's 3.35 TB/s -- forward 44 B per slot
(pix_to_face 8, barycentrics 12, texels 12, colours 12) + 72 B per face (corner positions and normals); backward 68 B
per slot (the forward's reads, the upstream gradient 12, grad texels 12, grad barycentrics 12) + 144 B per face (the
corners read, their gradients written).
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

PEAK_BYTES_PER_S = 3.35e12


def _torus(dev):
    from pytorch3d_b200 import synthetic
    return synthetic.torus_batch(8, 187, 187, seed=0, device=dev)


def north_star_scene(dev):
    from pytorch3d_b200 import _C
    m = _torus(dev)
    p2f, _, bary, _, _ = _C.rasterize_meshes_indexed(m.verts_packed(), m.faces_packed(),
                                                     m.mesh_to_faces_packed_first_idx(), m.num_faces_per_mesh(),
                                                     (512, 512), 0.0, 8, False, False, False)
    return m, p2f, bary


def random_scene(N, H, W, K, dev):
    m = _torus(dev)
    g = torch.Generator(device=dev).manual_seed(1)
    F = int(m.faces_packed().shape[0])
    p2f = torch.randint(0, F, (N, H, W, K), generator=g, device=dev)
    p2f = torch.where(torch.rand(N, H, W, K, generator=g, device=dev) < 0.3, -1, p2f)
    bary = torch.rand(N, H, W, K, 3, generator=g, device=dev) + 0.05
    return m, p2f, bary / bary.sum(-1, keepdim=True)


def measure(name, m, p2f, bary, dev, iters):
    import test_shading as ts
    from pytorch3d_b200 import _C
    from pytorch3d_b200.shading import _params, phong_shading
    N, H, W, K = (int(v) for v in p2f.shape)
    F = int(m.faces_packed().shape[0])
    g = torch.Generator(device=dev).manual_seed(2)
    texels = torch.rand(N, H, W, K, 3, generator=g, device=dev)
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
    faces = m.faces_packed()
    normals = m.verts_normals_packed().detach()
    mesh = types.SimpleNamespace(verts_packed=lambda: verts, faces_packed=lambda: faces,
                                 verts_normals_packed=lambda: normals)
    frags = types.SimpleNamespace(pix_to_face=p2f, bary_coords=bary)
    tx = texels.clone().requires_grad_(True)
    leaves = [verts, tx]
    slots = N * H * W * K
    bytes_fwd, bytes_bwd = 44 * slots + 72 * F, 68 * slots + 144 * F
    fv, fn = verts.detach()[faces], normals[faces]
    params = _params(N, lights, cameras, materials, "point", dev)

    def fused():
        return phong_shading(mesh, frags, lights, cameras, materials, tx)

    def chain():
        return ts.chain_phong(mesh, frags, lights, cameras, materials, tx)

    res = {"N": N, "H": H, "W": W, "K": K, "F": F, "slots": slots,
           "background_fraction": float((p2f < 0).float().mean())}
    with torch.no_grad():
        for _ in range(3):
            _C.shading_forward(p2f, bary, fv, fn, texels, params, False, "point")
        res["fused_forward_us"] = 1e3 * _events_ms(
            lambda: _C.shading_forward(p2f, bary, fv, fn, texels, params, False, "point"), iters)
    for _ in range(2):
        fused().backward(grad)
    res["fused_backward_us"] = 1e3 * _time_backward_ms(fused, grad, leaves, iters)
    needs = (True, True, True, False, False)
    for _ in range(2):
        _C.shading_backward(grad, None, p2f, bary, fv, fn, texels, params, False, "point", needs)
    res["fused_backward_kernel_us"] = 1e3 * _events_ms(
        lambda: _C.shading_backward(grad, None, p2f, bary, fv, fn, texels, params, False, "point", needs), iters)
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
    assert torch.cuda.is_available(), "time_shading.py measures on a CUDA device"
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
    with open(os.path.join(out_dir, "time_shading.json"), "w") as fh:
        json.dump(report, fh, indent=1)
    print(json.dumps({"device": report["device"], "power_limit": power}))


if __name__ == "__main__":
    main()
