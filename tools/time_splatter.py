"""Times the fused splatter blend on the GPU against the torch chain of the reference's
pytorch3d/renderer/splatter_blend.py (tests/test_splatter_blend.py: splatter_chain).  CUDA events after warm-up, peak
memory of forward + backward; the card's name and power limit are read in the same run.

    python tools/time_splatter.py OUT_DIR        -> OUT_DIR/time_splatter.json

Workloads: the north-star Fragments (8 tori of 187 x 187, 512 x 512, K = 8, no blur) with the background mask from
pix_to_face < 0, the rasterizer's depths and random colours and sub-pixel positions; and 8 x 256 x 256 at K in {2, 50}
on random scenes.  A chain that runs out of memory is reported as such.
Backward times: `fused_backward_us` / `chain_backward_us` are autograd's backward (with fresh .grad fields);
`fused_backward_kernel_us` is the `_C` backward call alone, which the backward bandwidth fraction uses.
Bandwidth: algorithmic bytes over time, as a fraction of the H100 SXM's 3.35 TB/s -- forward 25 B read per slot
(colours 12, positions 12, mask 1) + 16 B written per pixel; backward 25 B read + 24 B written per slot (grad colours
12, grad positions 12) + 16 B read per pixel (upstream gradient).
"""
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]

from time_blend import _events_ms, _peak_bytes, _time_backward_ms  # noqa: E402

PEAK_BYTES_PER_S = 3.35e12
SIGMA = 0.5
BG = (1.0, 1.0, 1.0)


def north_star_scene(dev):
    from pytorch3d_b200 import _C, synthetic
    m = synthetic.torus_batch(8, 187, 187, seed=0)
    p2f, zbuf = _C.rasterize_meshes_indexed(m.verts_packed().to(dev), m.faces_packed().to(dev),
                                            m.mesh_to_faces_packed_first_idx().to(dev), m.num_faces_per_mesh().to(dev),
                                            (512, 512), 0.0, 8, False, False, False)[:2]
    N, H, W, K = (int(v) for v in p2f.shape)
    g = torch.Generator(device=dev).manual_seed(0)
    hh, ww = torch.meshgrid(torch.arange(H, device=dev) + 0.5, torch.arange(W, device=dev) + 0.5, indexing="ij")
    xy = torch.stack([hh, ww], -1)[None, :, :, None].expand(N, H, W, K, 2)
    xy = xy + 0.2 * (torch.rand(N, H, W, K, 2, generator=g, device=dev) - 0.5)
    coords = torch.cat([xy, zbuf[..., None]], -1).contiguous()
    colors = torch.rand(N, H, W, K, 3, generator=g, device=dev)
    return colors, coords, p2f < 0


def random_scene(N, H, W, K, dev):
    import test_splatter_blend as ts
    colors, coords, mask, _ = ts.splatter_scene(N, H, W, K, SIGMA, "far", device=dev)
    return colors, coords, mask


def measure(name, colors, coords, mask, dev, iters):
    import test_splatter_blend as ts
    from pytorch3d_b200 import _C
    from pytorch3d_b200.blending import BlendParams
    from pytorch3d_b200.splatter_blend import splatter_blend
    N, H, W, K = (int(v) for v in mask.shape)
    grad = torch.randn((N, H, W, 4), device=dev)
    params = BlendParams(sigma=SIGMA, background_color=BG)
    slots, pixels = N * H * W * K, N * H * W
    bytes_fwd, bytes_bwd = 25 * slots + 16 * pixels, 49 * slots + 16 * pixels
    leaves = [t.clone().requires_grad_(True) for t in (colors, coords)]

    def fused():
        return splatter_blend(leaves[0], leaves[1], mask, params)

    def chain():
        return ts.splatter_chain(leaves[0], leaves[1], mask, SIGMA, BG)

    res = {"N": N, "H": H, "W": W, "K": K, "slots": slots, "background_fraction": float(mask.float().mean())}
    with torch.no_grad():
        for _ in range(3):
            _C.splatter_blend(colors, coords, mask, SIGMA, BG)
        res["fused_forward_us"] = 1e3 * _events_ms(lambda: _C.splatter_blend(colors, coords, mask, SIGMA, BG), iters)
    for _ in range(2):
        fused().backward(grad)
    res["fused_backward_us"] = 1e3 * _time_backward_ms(fused, grad, leaves, iters)
    res["fused_backward_kernel_us"] = 1e3 * _events_ms(
        lambda: _C.splatter_blend_backward(grad, colors, coords, mask, SIGMA, BG), iters)
    for leaf in leaves:
        leaf.grad = None
    res["fused_peak_bytes_fwd_bwd"] = _peak_bytes(lambda: fused().backward(grad))
    res["fused_forward_bandwidth_fraction"] = bytes_fwd / (res["fused_forward_us"] * 1e-6) / PEAK_BYTES_PER_S
    res["fused_backward_bandwidth_fraction"] = bytes_bwd / (res["fused_backward_kernel_us"] * 1e-6) / PEAK_BYTES_PER_S
    # the chain, with outputs compared to the fused op's on the same inputs
    try:
        for leaf in leaves:
            leaf.grad = None
        with torch.no_grad():
            want = ts.splatter_chain(colors, coords, mask, SIGMA, BG)
            got = _C.splatter_blend(colors, coords, mask, SIGMA, BG)
            res["max_abs_diff_forward"] = float((got - want).abs().max())
            del want, got
            for _ in range(2):
                ts.splatter_chain(colors, coords, mask, SIGMA, BG)
            res["chain_forward_us"] = 1e3 * _events_ms(lambda: ts.splatter_chain(colors, coords, mask, SIGMA, BG),
                                                       max(3, iters // 4))
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
    assert torch.cuda.is_available(), "time_splatter.py measures on a CUDA device"
    assert not torch.backends.cuda.matmul.allow_tf32, "the chain's bmm must run in full float32"
    dev = torch.device("cuda:0")
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               stdout=subprocess.PIPE, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = "not measured"
    report = {"device": torch.cuda.get_device_name(dev), "power_limit": power, "workloads": {}}
    report["workloads"]["north_star_8x512x512_K8"] = measure("north_star", *north_star_scene(dev), dev, 20)
    for K in (2, 50):
        report["workloads"]["random_8x256x256_K%d" % K] = measure("random_K%d" % K, *random_scene(8, 256, 256, K, dev),
                                                                  dev, 20)
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "time_splatter.json"), "w") as fh:
        json.dump(report, fh, indent=1)
    print(json.dumps({"device": report["device"], "power_limit": power}))


if __name__ == "__main__":
    main()
