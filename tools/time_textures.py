"""Times the fused UV texture sampling on the GPU against the torch chain of the reference's
TexturesUV.sample_textures (tests/test_textures.py: chain_sample).  CUDA events after warm-up, peak memory of forward +
backward; the card's name and power limit are read in the same run.

    python tools/time_textures.py OUT_DIR        -> OUT_DIR/time_textures.json

Workloads: the north-star Fragments (8 tori of 187 x 187, 512 x 512, K = 8, no blur) from the rasterizer with one
1024 x 1024 RGB map per mesh, and 8 x 256 x 256 at K = 50 with random faces of the same tori, random barycentrics and
one 512 x 512 RGB map per image.  Both use the TexturesUV defaults: bilinear, border padding, align_corners=True.  The
maps, the vertex UVs and the barycentrics require grad.
Backward times: `fused_backward_us` / `chain_backward_us` are autograd's backward (with fresh .grad fields);
`fused_backward_kernel_us` is the `_C` backward call alone (zero fills included), which the backward bandwidth
fraction uses.  The upstream gradient is nonzero on every slot, background slots included, so on the north-star
Fragments 88 % of the slots add into one texel per image (the worst case for that texel); the `..._background_zero`
times repeat the fused backward with the upstream gradient zeroed where pix_to_face < 0, as it arrives from the blend.
Bandwidth: algorithmic bytes over time, as a fraction of the H100 SXM's 3.35 TB/s -- forward 20 B per slot read
(pix_to_face 8, barycentrics 12) and 4 C B written, + 24 B per face (corner UVs); backward the forward's reads, the
upstream gradient 4 C B and grad_bary 12 B per slot, the grad_maps zero fill and write (2 x 4 C B per texel), and the
face UVs' gradient (24 B per face).  The texels the samples touch are not counted.
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


def _torus(dev, map_size):
    from pytorch3d_b200 import synthetic
    return synthetic.textured_torus_batch(8, 187, 187, map_size=map_size, seed=0, device=dev)


def north_star_scene(dev):
    from pytorch3d_b200 import _C
    m, verts_uvs, faces_uvs, maps = _torus(dev, (1024, 1024))
    p2f, _, bary, _, _ = _C.rasterize_meshes_indexed(m.verts_packed(), m.faces_packed(),
                                                     m.mesh_to_faces_packed_first_idx(), m.num_faces_per_mesh(),
                                                     (512, 512), 0.0, 8, False, False, False)
    return verts_uvs, faces_uvs, maps, p2f, bary


def random_scene(N, H, W, K, dev):
    m, verts_uvs, faces_uvs, maps = _torus(dev, (512, 512))
    g = torch.Generator(device=dev).manual_seed(1)
    F = int(m.faces_packed().shape[0])
    p2f = torch.randint(0, F, (N, H, W, K), generator=g, device=dev)
    p2f = torch.where(torch.rand(N, H, W, K, generator=g, device=dev) < 0.3, -1, p2f)
    bary = torch.rand(N, H, W, K, 3, generator=g, device=dev) + 0.05
    return verts_uvs, faces_uvs, maps, p2f, bary / bary.sum(-1, keepdim=True)


def measure(name, verts_uvs, faces_uvs, maps, p2f, bary, dev, iters):
    import test_textures as tt
    from pytorch3d_b200 import _C
    N, H, W, K = (int(v) for v in p2f.shape)
    _, H_in, W_in, C = (int(v) for v in maps.shape)
    g = torch.Generator(device=dev).manual_seed(2)
    grad = torch.randn(N, H, W, K, C, generator=g, device=dev)
    mp = maps.detach().clone().requires_grad_(True)
    vuv = [v.detach().clone().requires_grad_(True) for v in verts_uvs]
    by = bary.detach().clone().requires_grad_(True)
    frags = types.SimpleNamespace(pix_to_face=p2f, bary_coords=by)
    leaves = [mp, by] + vuv
    fuv = tt.packed_face_uvs([v.detach() for v in verts_uvs], faces_uvs)
    F = int(fuv.shape[0])
    slots = N * H * W * K
    bytes_fwd = (20 + 4 * C) * slots + 24 * F
    bytes_bwd = (20 + 8 * C + 12) * slots + 2 * 4 * C * N * H_in * W_in + 48 * F

    def fused():
        return tt.fused_sample(frags, mp, tt.packed_face_uvs(vuv, faces_uvs))

    def chain():
        return tt.chain_sample(frags, mp, tt.packed_face_uvs(vuv, faces_uvs))

    res = {"N": N, "H": H, "W": W, "K": K, "F": F, "map": [H_in, W_in, C], "slots": slots,
           "background_fraction": float((p2f < 0).float().mean())}
    with torch.no_grad():
        for _ in range(3):
            _C.texture_uv_forward(p2f, bary, fuv, maps)
        res["fused_forward_us"] = 1e3 * _events_ms(lambda: _C.texture_uv_forward(p2f, bary, fuv, maps), iters)
    for _ in range(2):
        fused().backward(grad)
    res["fused_backward_us"] = 1e3 * _time_backward_ms(fused, grad, leaves, iters)
    for _ in range(2):
        _C.texture_uv_backward(grad, p2f, bary, fuv, maps)
    res["fused_backward_kernel_us"] = 1e3 * _events_ms(lambda: _C.texture_uv_backward(grad, p2f, bary, fuv, maps),
                                                       iters)
    grad_bg0 = grad * (p2f >= 0).unsqueeze(-1).to(grad.dtype)
    res["fused_backward_us_background_zero"] = 1e3 * _time_backward_ms(fused, grad_bg0, leaves, iters)
    for _ in range(2):
        _C.texture_uv_backward(grad_bg0, p2f, bary, fuv, maps)
    res["fused_backward_kernel_us_background_zero"] = 1e3 * _events_ms(
        lambda: _C.texture_uv_backward(grad_bg0, p2f, bary, fuv, maps), iters)
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
    assert torch.cuda.is_available(), "time_textures.py measures on a CUDA device"
    dev = torch.device("cuda:0")
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               stdout=subprocess.PIPE, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = "not measured"
    report = {"device": torch.cuda.get_device_name(dev), "power_limit": power, "workloads": {}}
    report["workloads"]["north_star_8x512x512_K8_1024map"] = measure("north_star", *north_star_scene(dev), dev, 20)
    report["workloads"]["random_8x256x256_K50_512map"] = measure("random_K50", *random_scene(8, 256, 256, 50, dev),
                                                                 dev, 20)
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "time_textures.json"), "w") as fh:
        json.dump(report, fh, indent=1)
    print(json.dumps({"device": report["device"], "power_limit": power}))


if __name__ == "__main__":
    main()
