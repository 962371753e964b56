"""Times the depth shaders on the GPU: the fused soft_depth / hard_depth against the torch chains of the reference's
SoftDepthShader / HardDepthShader (restated in tests/test_depth_shading.py).  CUDA events after warm-up; the card's
name and power limit are read in the same run.

    python tools/time_depth.py OUT_DIR        -> OUT_DIR/time_depth.json

Workloads: the ns_blur Fragments of bench.py (8 tori of 187 x 187, 512 x 512, K = 8, blur 1e-4), and random Fragments
of 8 x 256 x 256 at K = 50 and K = 100.  zfar is a 1-element CUDA tensor, as FoVPerspectiveCameras hold it.
Backward times: `*_backward_us` are autograd's backward (with fresh .grad fields); `fused_backward_kernel_us` is the
`_C` backward call alone, which the backward bandwidth fraction uses.
Bandwidth: algorithmic bytes over time, as a fraction of the H100 SXM's 3.35 TB/s.  SoftDepth forward: 16 B per slot
(index 8, zbuf 4, dists 4) + 4 B per pixel (depth); backward: 16 B read + 8 B written per slot (grad zbuf, grad
dists) + 4 B per pixel (upstream gradient).  HardDepth forward: 12 B (slot 0's index and depth) + 4 B per pixel;
backward: 8 B (slot 0's index) + 4 B read per pixel + 4 B written per slot.
"""
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]

from time_blend import (PEAK_BYTES_PER_S, _events_ms, _peak_bytes, _time_backward_ms,  # noqa: E402
                        ns_blur_fragments, random_fragments)

SIGMA = 1e-4


def _leaves(*ts):
    return [t.clone().requires_grad_(True) for t in ts]


def _clear(leaves):
    for leaf in leaves:
        leaf.grad = None


def measure_soft(p2f, zbuf, dists, zfar, iters):
    import test_depth_shading as td
    from pytorch3d_b200 import _C, blending
    N, H, W, K = (int(v) for v in p2f.shape)
    grad = torch.randn((N, H, W, 1), device=p2f.device)
    slots, pixels = N * H * W * K, N * H * W
    leaves = _leaves(zbuf, dists)
    fused = lambda: blending.soft_depth(td.frags(p2f, *leaves), SIGMA, zfar)  # noqa: E731
    chain = lambda: td.soft_depth_chain(p2f, leaves[0], leaves[1], SIGMA, zfar)  # noqa: E731
    res = {}
    with torch.no_grad():
        for _ in range(3):
            fused()
            chain()
        res["fused_forward_us"] = 1e3 * _events_ms(fused, iters)
        res["chain_forward_us"] = 1e3 * _events_ms(chain, iters)
    for _ in range(2):
        fused().backward(grad)
        chain().backward(grad)
    res["fused_backward_us"] = 1e3 * _time_backward_ms(fused, grad, leaves, iters)
    res["chain_backward_us"] = 1e3 * _time_backward_ms(chain, grad, leaves, iters)
    res["fused_backward_kernel_us"] = 1e3 * _events_ms(
        lambda: _C.soft_depth_blend_backward(grad, p2f, zbuf, dists, SIGMA, zfar), iters)
    _clear(leaves)
    res["fused_peak_bytes_fwd_bwd"] = _peak_bytes(lambda: fused().backward(grad))
    _clear(leaves)
    res["chain_peak_bytes_fwd_bwd"] = _peak_bytes(lambda: chain().backward(grad))
    _clear(leaves)
    res["fused_forward_bandwidth_fraction"] = (16 * slots + 4 * pixels) / (res["fused_forward_us"] * 1e-6) \
        / PEAK_BYTES_PER_S
    res["fused_backward_bandwidth_fraction"] = (24 * slots + 4 * pixels) / (res["fused_backward_kernel_us"] * 1e-6) \
        / PEAK_BYTES_PER_S
    res["forward_speedup"] = res["chain_forward_us"] / res["fused_forward_us"]
    res["backward_speedup"] = res["chain_backward_us"] / res["fused_backward_us"]
    return res


def measure_hard(p2f, zbuf, zfar, iters):
    import test_depth_shading as td
    from pytorch3d_b200 import _C, blending
    N, H, W, K = (int(v) for v in p2f.shape)
    grad = torch.randn((N, H, W, 1), device=p2f.device)
    slots, pixels = N * H * W * K, N * H * W
    leaves = _leaves(zbuf)
    fused = lambda: blending.hard_depth(td.frags(p2f, leaves[0], None), zfar)  # noqa: E731
    chain = lambda: td.hard_depth_chain(p2f, leaves[0], zfar)  # noqa: E731
    res = {}
    with torch.no_grad():
        for _ in range(3):
            fused()
            chain()
        res["fused_forward_us"] = 1e3 * _events_ms(fused, iters)
        res["chain_forward_us"] = 1e3 * _events_ms(chain, iters)
    for _ in range(2):
        fused().backward(grad)
        chain().backward(grad)
    res["fused_backward_us"] = 1e3 * _time_backward_ms(fused, grad, leaves, iters)
    res["chain_backward_us"] = 1e3 * _time_backward_ms(chain, grad, leaves, iters)
    res["fused_backward_kernel_us"] = 1e3 * _events_ms(lambda: _C.hard_depth_backward(grad, p2f), iters)
    _clear(leaves)
    res["fused_peak_bytes_fwd_bwd"] = _peak_bytes(lambda: fused().backward(grad))
    _clear(leaves)
    res["chain_peak_bytes_fwd_bwd"] = _peak_bytes(lambda: chain().backward(grad))
    _clear(leaves)
    res["fused_forward_bandwidth_fraction"] = 16 * pixels / (res["fused_forward_us"] * 1e-6) / PEAK_BYTES_PER_S
    res["fused_backward_bandwidth_fraction"] = (12 * pixels + 4 * slots) / (res["fused_backward_kernel_us"] * 1e-6) \
        / PEAK_BYTES_PER_S
    res["forward_speedup"] = res["chain_forward_us"] / res["fused_forward_us"]
    res["backward_speedup"] = res["chain_backward_us"] / res["fused_backward_us"]
    return res


def main():
    out_dir = sys.argv[1] if len(sys.argv) > 1 else "."
    assert torch.cuda.is_available(), "time_depth.py measures on a CUDA device"
    dev = torch.device("cuda:0")
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               stdout=subprocess.PIPE, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = "not measured"
    zfar = torch.tensor([100.0], device=dev)
    report = {"device": torch.cuda.get_device_name(dev), "power_limit": power, "workloads": {}}
    workloads = [("ns_blur_8x512x512_K8", lambda: ns_blur_fragments(dev))] + [
        ("random_8x256x256_K%d" % K, lambda K=K: random_fragments(8, 256, 256, K, dev)) for K in (50, 100)]
    for name, make in workloads:
        p2f, zbuf, dists = make()
        N, H, W, K = (int(v) for v in p2f.shape)
        row = {"N": N, "H": H, "W": W, "K": K, "slots": N * H * W * K,
               "soft": measure_soft(p2f, zbuf, dists, zfar, 20), "hard": measure_hard(p2f, zbuf, zfar, 20)}
        report["workloads"][name] = row
        print(name, json.dumps(row), flush=True)
        del p2f, zbuf, dists
        torch.cuda.empty_cache()
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "time_depth.json"), "w") as fh:
        json.dump(report, fh, indent=1)
    print(json.dumps({"device": report["device"], "power_limit": power}))


if __name__ == "__main__":
    main()
