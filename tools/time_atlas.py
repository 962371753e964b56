"""Times the fused texture atlas sampling on the GPU against the torch chain of the reference's
TexturesAtlas.sample_textures (tests/test_texture_atlas.py: chain_sample).  CUDA events after warm-up, peak memory of
forward + backward; the card's name and power limit are read in the same run.

    python tools/time_atlas.py OUT_DIR        -> OUT_DIR/time_atlas.json

Workloads: the north-star Fragments (8 tori of 187 x 187 = 559,504 faces, 512 x 512, K = 8, no blur) from the
rasterizer with a seeded R = 4 RGB atlas (107 MB), and 8 x 256 x 256 at K = 50 with random faces of the same tori, 30 %
background slots, random barycentrics and an R = 8 RGB atlas.  The atlas requires grad.
Backward times: `fused_backward_us` / `chain_backward_us` are autograd's backward (with a fresh .grad field);
`fused_backward_kernel_us` is the `_C` backward call alone (workspace allocation, zero fill, key pass, sort and
segmented sum).  The upstream gradient is nonzero on every slot, background slots included (their contribution g * 0
is dropped by the key pass); the `..._background_zero` times repeat the fused backward with it zeroed where
pix_to_face < 0, as it arrives from the blend.
Bandwidth: algorithmic bytes from shapes over time, as a fraction of the H100 SXM's 3.35 TB/s.  Forward: 20 B per slot
read (pix_to_face 8, barycentrics 12) and 4 C B written; the atlas cells the samples touch are not counted.  Backward:
the key pass reads 20 + 4 C B and writes key + 4 B per slot; the radix sort reads the keys once to count digits, then
per 8-bit digit pass reads and writes key + 4 B per slot; the segmented pass reads key + 4 B and the upstream gradient
(4 C B) per slot (an upper bound: sentinel slots read no gradient); the atlas gradient is zero-filled and written
(2 x 4 C B per cell).
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


def _atlas(F, R, dev):
    return torch.rand(F, R, R, 3, generator=torch.Generator(device=dev).manual_seed(3), device=dev)


def north_star_scene(dev):
    from pytorch3d_b200 import _C
    m = _torus(dev)
    p2f, _, bary, _, _ = _C.rasterize_meshes_indexed(m.verts_packed(), m.faces_packed(),
                                                     m.mesh_to_faces_packed_first_idx(), m.num_faces_per_mesh(),
                                                     (512, 512), 0.0, 8, False, False, False)
    return _atlas(int(m.faces_packed().shape[0]), 4, dev), p2f, bary


def random_scene(N, H, W, K, R, dev):
    F = int(_torus(dev).faces_packed().shape[0])
    g = torch.Generator(device=dev).manual_seed(1)
    p2f = torch.randint(0, F, (N, H, W, K), generator=g, device=dev)
    p2f = torch.where(torch.rand(N, H, W, K, generator=g, device=dev) < 0.3, -1, p2f)
    bary = torch.rand(N, H, W, K, 3, generator=g, device=dev) + 0.05
    return _atlas(F, R, dev), p2f, bary / bary.sum(-1, keepdim=True)


def algorithmic_bytes(N, H, W, K, F, R, C):
    """(forward, backward) bytes, as the module docstring counts them."""
    from pytorch3d_b200._C import texture_atlas_key_bits
    slots, cells = N * H * W * K, F * R * R
    bits, kb = texture_atlas_key_bits(F, R)
    passes = (bits + 7) // 8
    fwd = (20 + 4 * C) * slots
    bwd = ((20 + 4 * C) + (kb + 4) + kb + passes * 2 * (kb + 4) + (kb + 4 + 4 * C)) * slots + 2 * 4 * C * cells
    return fwd, bwd


def measure(name, atlas, p2f, bary, dev, iters):
    import test_texture_atlas as ta
    from pytorch3d_b200 import _C
    N, H, W, K = (int(v) for v in p2f.shape)
    F, R, _, C = (int(v) for v in atlas.shape)
    g = torch.Generator(device=dev).manual_seed(2)
    grad = torch.randn(N, H, W, K, C, generator=g, device=dev)
    leaf = atlas.detach().clone().requires_grad_(True)
    frags = types.SimpleNamespace(pix_to_face=p2f, bary_coords=bary)
    bytes_fwd, bytes_bwd = algorithmic_bytes(N, H, W, K, F, R, C)

    def fused():
        return ta.fused_sample(frags, leaf)

    def chain():
        return ta.chain_sample(frags, leaf)

    res = {"N": N, "H": H, "W": W, "K": K, "F": F, "R": R, "C": C, "slots": N * H * W * K,
           "atlas_bytes": 4 * F * R * R * C, "background_fraction": float((p2f < 0).float().mean()),
           "key_bits": _C.texture_atlas_key_bits(F, R)[0]}
    with torch.no_grad():
        for _ in range(3):
            _C.texture_atlas_forward(p2f, bary, atlas)
        res["fused_forward_us"] = 1e3 * _events_ms(lambda: _C.texture_atlas_forward(p2f, bary, atlas), iters)
    for _ in range(2):
        fused().backward(grad)
    res["fused_backward_us"] = 1e3 * _time_backward_ms(fused, grad, [leaf], iters)
    for _ in range(2):
        _C.texture_atlas_backward(grad, p2f, bary, atlas)
    res["fused_backward_kernel_us"] = 1e3 * _events_ms(lambda: _C.texture_atlas_backward(grad, p2f, bary, atlas),
                                                       iters)
    grad_bg0 = grad * (p2f >= 0).unsqueeze(-1).to(grad.dtype)
    res["fused_backward_us_background_zero"] = 1e3 * _time_backward_ms(fused, grad_bg0, [leaf], iters)
    for _ in range(2):
        _C.texture_atlas_backward(grad_bg0, p2f, bary, atlas)
    res["fused_backward_kernel_us_background_zero"] = 1e3 * _events_ms(
        lambda: _C.texture_atlas_backward(grad_bg0, p2f, bary, atlas), iters)
    leaf.grad = None
    res["fused_peak_bytes_fwd_bwd"] = _peak_bytes(lambda: fused().backward(grad))
    res["fused_forward_bandwidth_fraction"] = bytes_fwd / (res["fused_forward_us"] * 1e-6) / PEAK_BYTES_PER_S
    res["fused_backward_bandwidth_fraction"] = bytes_bwd / (res["fused_backward_kernel_us"] * 1e-6) / PEAK_BYTES_PER_S
    leaf.grad = None
    with torch.no_grad():
        want, got = chain(), fused()
        res["forward_bit_identical"] = bool(torch.equal(want, got))
        del want, got
        for _ in range(2):
            chain()
        res["chain_forward_us"] = 1e3 * _events_ms(chain, max(3, iters // 4))
    chain().backward(grad)
    want_grad = leaf.grad
    leaf.grad = None
    fused().backward(grad)
    res["backward_max_abs_diff"] = float((leaf.grad - want_grad).abs().max())
    res["backward_max_abs"] = float(want_grad.abs().max())
    del want_grad
    res["chain_backward_us"] = 1e3 * _time_backward_ms(chain, grad, [leaf], max(3, iters // 4))
    leaf.grad = None
    res["chain_peak_bytes_fwd_bwd"] = _peak_bytes(lambda: chain().backward(grad))
    res["forward_speedup"] = res["chain_forward_us"] / res["fused_forward_us"]
    res["backward_speedup"] = res["chain_backward_us"] / res["fused_backward_us"]
    leaf.grad = None
    torch.cuda.empty_cache()
    print(name, json.dumps(res), flush=True)
    return res


def main():
    out_dir = sys.argv[1] if len(sys.argv) > 1 else "."
    assert torch.cuda.is_available(), "time_atlas.py measures on a CUDA device"
    dev = torch.device("cuda:0")
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               stdout=subprocess.PIPE, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = "not measured"
    report = {"device": torch.cuda.get_device_name(dev), "power_limit": power, "workloads": {}}
    report["workloads"]["north_star_8x512x512_K8_R4"] = measure("north_star", *north_star_scene(dev), dev, 20)
    report["workloads"]["random_8x256x256_K50_R8"] = measure("random_K50", *random_scene(8, 256, 256, 50, 8, dev),
                                                             dev, 20)
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "time_atlas.json"), "w") as fh:
        json.dump(report, fh, indent=1)
    print(json.dumps({"device": report["device"], "power_limit": power}))


if __name__ == "__main__":
    main()
