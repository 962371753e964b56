"""Times the mesh blending ops on the GPU: the fused softmax_rgb_blend against the torch chain of the reference's
pytorch3d/renderer/blending.py, and sigmoid_alpha_blend against the reference's CUDA kernels (when
oracle/_ref/ref_blend_cuda.so was built).  CUDA events after warm-up; the card's name and power limit are read in the
same run.

    python tools/time_blend.py OUT_DIR        -> OUT_DIR/time_blend.json

Workloads: the ns_blur Fragments of bench.py (8 tori of 187 x 187, 512 x 512, K = 8, blur 1e-4) with random colours,
and the reference's blending benchmark shape (N = 8, 256 x 256, K in {2, 50, 100}) on random Fragments.
Backward times: `fused_backward_us` / `chain_backward_us` are autograd's backward (with fresh .grad fields);
`fused_backward_kernel_us` is the `_C` backward call alone, which the backward bandwidth fraction uses.
Bandwidth: algorithmic bytes over time, as a fraction of the H100 SXM's 3.35 TB/s -- forward 28 B per slot
(colours 12, index 8, zbuf 4, dists 4) + 16 B per pixel (RGBA); backward 28 B per slot read + 20 B per slot written
(grad colours 12, grad dists 4, grad zbuf 4) + 16 B per pixel (upstream gradient).
"""
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

PEAK_BYTES_PER_S = 3.35e12


def _events_ms(fn, iters):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / iters


def _time_backward_ms(make_out, grad, leaves, iters):
    """Mean time of out.backward(grad) alone: each iteration runs the forward outside the timed window and starts
    from empty .grad fields (no accumulation into earlier gradients)."""
    total = 0.0
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(iters):
        for leaf in leaves:
            leaf.grad = None
        out = make_out()
        start.record()
        out.backward(grad)
        end.record()
        end.synchronize()
        total += start.elapsed_time(end)
    return total / iters


def _peak_bytes(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def random_fragments(N, H, W, K, dev, seed=0):
    g = torch.Generator(device=dev).manual_seed(seed)
    n_valid = (torch.rand(N, H, W, 1, generator=g, device=dev) * (K + 1)).long().clamp(max=K)
    valid = torch.arange(K, device=dev).view(1, 1, 1, K) < n_valid
    p2f = torch.where(valid, torch.randint(0, 100000, (N, H, W, K), generator=g, device=dev), -1)
    zbuf = torch.where(valid, 1.0 + 9.0 * torch.rand(N, H, W, K, generator=g, device=dev), -1.0)
    dists = torch.where(valid, torch.randn(N, H, W, K, generator=g, device=dev) * 1e-3, -1.0)
    return p2f, zbuf, dists


def ns_blur_fragments(dev):
    from pytorch3d_b200 import _C, synthetic
    m = synthetic.torus_batch(8, 187, 187, seed=0)
    out = _C.rasterize_meshes_indexed(m.verts_packed().to(dev), m.faces_packed().to(dev),
                                      m.mesh_to_faces_packed_first_idx().to(dev), m.num_faces_per_mesh().to(dev),
                                      (512, 512), 1e-4, 8, False, False, False)
    return out[0], out[1], out[3]


def measure(name, p2f, zbuf, dists, dev, iters, ref_sigmoid):
    import test_blending as tb
    from pytorch3d_b200 import _C, blending
    N, H, W, K = (int(v) for v in p2f.shape)
    colors = torch.rand((N, H, W, K, 3), device=dev)
    grad = torch.randn((N, H, W, 4), device=dev)
    params = blending.BlendParams(sigma=1e-4, gamma=1e-4)
    slots, pixels = N * H * W * K, N * H * W
    bytes_fwd, bytes_bwd = 28 * slots + 16 * pixels, 48 * slots + 16 * pixels

    leaves = [t.clone().requires_grad_(True) for t in (colors, zbuf, dists)]

    def fused():
        c, z, d = leaves
        return blending.softmax_rgb_blend(c, tb.frags(p2f, z, d), params)

    def chain():
        c, z, d = leaves
        return tb.softmax_chain(c, p2f, z, d, 1e-4, 1e-4, (1.0, 1.0, 1.0))

    res = {"N": N, "H": H, "W": W, "K": K, "slots": slots}
    with torch.no_grad():
        for _ in range(3):
            _C.softmax_rgb_blend(colors, p2f, zbuf, dists, 1e-4, 1e-4, (1.0, 1.0, 1.0))
            tb.softmax_chain(colors, p2f, zbuf, dists, 1e-4, 1e-4, (1.0, 1.0, 1.0))
        res["fused_forward_us"] = 1e3 * _events_ms(
            lambda: _C.softmax_rgb_blend(colors, p2f, zbuf, dists, 1e-4, 1e-4, (1.0, 1.0, 1.0)), iters)
        res["chain_forward_us"] = 1e3 * _events_ms(
            lambda: tb.softmax_chain(colors, p2f, zbuf, dists, 1e-4, 1e-4, (1.0, 1.0, 1.0)), iters)
    for _ in range(2):
        fused().backward(grad)
        chain().backward(grad)
    res["fused_backward_us"] = 1e3 * _time_backward_ms(fused, grad, leaves, iters)
    res["chain_backward_us"] = 1e3 * _time_backward_ms(chain, grad, leaves, iters)
    res["fused_backward_kernel_us"] = 1e3 * _events_ms(lambda: _C.softmax_rgb_blend_backward(
        grad, colors, p2f, zbuf, dists, 1e-4, 1e-4, (1.0, 1.0, 1.0)), iters)
    for leaf in leaves:
        leaf.grad = None
    res["fused_peak_bytes_fwd_bwd"] = _peak_bytes(lambda: fused().backward(grad))
    for leaf in leaves:
        leaf.grad = None
    res["chain_peak_bytes_fwd_bwd"] = _peak_bytes(lambda: chain().backward(grad))
    for leaf in leaves:
        leaf.grad = None
    res["fused_forward_bandwidth_fraction"] = bytes_fwd / (res["fused_forward_us"] * 1e-6) / PEAK_BYTES_PER_S
    res["fused_backward_bandwidth_fraction"] = bytes_bwd / (res["fused_backward_kernel_us"] * 1e-6) / PEAK_BYTES_PER_S
    res["forward_speedup"] = res["chain_forward_us"] / res["fused_forward_us"]
    res["backward_speedup"] = res["chain_backward_us"] / res["fused_backward_us"]
    # sigmoid_alpha_blend: ours against the reference's kernels
    alphas = _C.sigmoid_alpha_blend(dists, p2f, 1e-4)
    ga = torch.randn((N, H, W), device=dev)
    res["sigmoid_forward_us"] = 1e3 * _events_ms(lambda: _C.sigmoid_alpha_blend(dists, p2f, 1e-4), iters)
    res["sigmoid_backward_us"] = 1e3 * _events_ms(
        lambda: _C.sigmoid_alpha_blend_backward(ga, alphas, dists, p2f, 1e-4), iters)
    if ref_sigmoid is not None:
        ref_sigmoid.sigmoid_alpha_blend(dists, p2f, 1e-4)
        res["reference_sigmoid_forward_us"] = 1e3 * _events_ms(
            lambda: ref_sigmoid.sigmoid_alpha_blend(dists, p2f, 1e-4), iters)
        res["reference_sigmoid_backward_us"] = 1e3 * _events_ms(
            lambda: ref_sigmoid.sigmoid_alpha_blend_backward(ga, alphas, dists, p2f, 1e-4), iters)
    else:
        res["reference_sigmoid_forward_us"] = res["reference_sigmoid_backward_us"] = "not measured"
    print(name, json.dumps(res), flush=True)
    return res


def main():
    out_dir = sys.argv[1] if len(sys.argv) > 1 else "."
    assert torch.cuda.is_available(), "time_blend.py measures on a CUDA device"
    from oracle import build_ref_blend
    dev = torch.device("cuda:0")
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               stdout=subprocess.PIPE, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = "not measured"
    ref_sigmoid = build_ref_blend.load(cuda=True)
    report = {"device": torch.cuda.get_device_name(dev), "power_limit": power, "workloads": {}}
    report["workloads"]["ns_blur_8x512x512_K8"] = measure("ns_blur", *ns_blur_fragments(dev), dev, 20, ref_sigmoid)
    for K in (2, 50, 100):
        report["workloads"]["reference_bm_8x256x256_K%d" % K] = measure(
            "bm_K%d" % K, *random_fragments(8, 256, 256, K, dev), dev, 20, ref_sigmoid)
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "time_blend.json"), "w") as fh:
        json.dump(report, fh, indent=1)
    print(json.dumps({"device": report["device"], "power_limit": power}))


if __name__ == "__main__":
    main()
