"""Times the fused mesh normals on the GPU against the torch chain of the reference's Meshes._compute_vertex_normals
(PackedMeshes.verts_normals_packed restates it) and, when oracle/_ref/ref_normals_cuda.so is present, the reference's
own CUDA face_areas_normals op.  CUDA events after warm-up; peak memory of forward + backward; the card's name and power
limit are read in the same run.

    python tools/time_normals.py OUT_DIR        -> OUT_DIR/time_normals.json

Workloads: the north-star tori (8 tori of 187 x 187: V = 279,752, F = 559,504) and the config-5 torus (707 x 707:
V = 499,849, F = 999,698), random-rotated as synthetic.torus_batch makes them; the vertices require grad.
Fields:
  vn_fused_forward_us / vn_fused_backward_us   autograd's forward / backward of normals.verts_normals (fresh .grad)
  vn_kernel_forward_us / vn_kernel_backward_us the `_C` calls alone
  vn_chain_forward_us / vn_chain_backward_us   the torch chain
  fan_fused_forward_us / fan_fused_backward_us `_C.face_areas_normals_forward/_backward`
  fan_reference_forward_us / _backward_us      the reference's CUDA op built for sm_90a ("not measured" when absent)
  stage_us                                     per-kernel times of one vertex-normal forward and backward and one face
                                               backward from torch.profiler, in a phase of their own after the timings;
                                               "table" is the vertex -> corner table (key pass, cub's radix sort,
                                               offsets), which the face backward builds again and the vertex backward
                                               reads from the forward
Bandwidth: algorithmic bytes over the `_C` time, as a fraction of the H100 SXM's 3.35 TB/s.  Counted: each array the
op must touch once -- vertex-normal forward 24 B per face (indices) + 36 B per face (the three corners' positions) +
24 B per vertex (normals written); backward the same plus 24 B per vertex (upstream gradient) and 24 B per vertex
(gradient written) in place of the normals; face forward 24 + 36 B per face read and 16 B per face written; face
backward 24 + 36 + 16 B per face read and 12 B per vertex written.  The table, the sort's passes and the per-face
workspace rows are not counted: they are what the fused ops add over that floor.
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
TABLE_KERNELS = ("corner_keys_kernel", "run_offsets_kernel", "RadixSort")


def _stages(fn):
    """{kernel group: µs} of one call of fn from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        if e.device_type.name != "CUDA" or getattr(e, "device_time_total", 0) <= 0:
            continue
        name = "table" if any(k in e.key for k in TABLE_KERNELS) else e.key.split("(")[0].split("<")[0][-60:]
        out[name] = out.get(name, 0.0) + float(e.device_time_total)
    return out


def measure(name, m, dev, iters):
    from pytorch3d_b200 import _C, normals
    from pytorch3d_b200.structures import PackedMeshes
    from oracle import build_ref_normals
    verts = m.verts_packed().to(dev).contiguous()
    faces = m.faces_packed().to(dev).contiguous()
    V, F = int(verts.shape[0]), int(faces.shape[0])
    g = torch.Generator(device=dev).manual_seed(3)
    grad = torch.randn(V, 3, generator=g, device=dev)
    ga, gn = torch.randn(F, generator=g, device=dev), torch.randn(F, 3, generator=g, device=dev)
    leaf = verts.clone().requires_grad_(True)
    res = {"V": V, "F": F}

    def fused():
        return normals.verts_normals(leaf, faces)

    def chain():
        return PackedMeshes([leaf], [faces]).verts_normals_packed()

    with torch.no_grad():
        for _ in range(3):
            fused()
        res["vn_fused_forward_us"] = 1e3 * _events_ms(fused, iters)
        out, table, sums = _C.verts_normals_forward(verts, faces)
        res["vn_kernel_forward_us"] = 1e3 * _events_ms(lambda: _C.verts_normals_forward(verts, faces), iters)
        for _ in range(2):
            _C.verts_normals_backward(grad, verts, faces, table, sums)
        res["vn_kernel_backward_us"] = 1e3 * _events_ms(
            lambda: _C.verts_normals_backward(grad, verts, faces, table, sums), iters)
        want = chain()
        res["vn_max_abs_diff_forward"] = float((out - want).abs().max())
        del want
        for _ in range(2):
            chain()
        res["vn_chain_forward_us"] = 1e3 * _events_ms(chain, iters)
    for _ in range(2):
        fused().backward(grad)
    res["vn_fused_backward_us"] = 1e3 * _time_backward_ms(fused, grad, [leaf], iters)
    leaf.grad = None
    res["vn_fused_peak_bytes_fwd_bwd"] = _peak_bytes(lambda: fused().backward(grad))
    fused_grad = leaf.grad.clone()
    leaf.grad = None
    chain().backward(grad)
    res["vn_max_abs_diff_backward"] = float((leaf.grad - fused_grad).abs().max())
    res["vn_chain_backward_us"] = 1e3 * _time_backward_ms(chain, grad, [leaf], iters)
    leaf.grad = None
    res["vn_chain_peak_bytes_fwd_bwd"] = _peak_bytes(lambda: chain().backward(grad))
    leaf.grad = None
    res["vn_forward_speedup"] = res["vn_chain_forward_us"] / res["vn_fused_forward_us"]
    res["vn_backward_speedup"] = res["vn_chain_backward_us"] / res["vn_fused_backward_us"]

    with torch.no_grad():
        for _ in range(3):
            _C.face_areas_normals_forward(verts, faces)
            _C.face_areas_normals_backward(ga, gn, verts, faces)
        res["fan_fused_forward_us"] = 1e3 * _events_ms(lambda: _C.face_areas_normals_forward(verts, faces), iters)
        res["fan_fused_backward_us"] = 1e3 * _events_ms(
            lambda: _C.face_areas_normals_backward(ga, gn, verts, faces), iters)
        ref = build_ref_normals.load(cuda=True)
        if ref is not None and getattr(ref, "with_cuda", False):
            fa, fn = _C.face_areas_normals_forward(verts, faces)
            ra, rn = ref.face_areas_normals_forward(verts, faces)
            res["fan_forward_bit_identical_to_reference"] = bool(torch.equal(fa, ra) and torch.equal(fn, rn))
            for _ in range(3):
                ref.face_areas_normals_forward(verts, faces)
                ref.face_areas_normals_backward(ga, gn, verts, faces)
            res["fan_reference_forward_us"] = 1e3 * _events_ms(lambda: ref.face_areas_normals_forward(verts, faces),
                                                               iters)
            res["fan_reference_backward_us"] = 1e3 * _events_ms(
                lambda: ref.face_areas_normals_backward(ga, gn, verts, faces), iters)
        else:
            res["fan_reference_forward_us"] = res["fan_reference_backward_us"] = "not measured"

    vn_fwd_bytes = 60 * F + 24 * V
    vn_bwd_bytes = 60 * F + 48 * V + 12 * V
    res["vn_forward_bandwidth_fraction"] = vn_fwd_bytes / (res["vn_kernel_forward_us"] * 1e-6) / PEAK_BYTES_PER_S
    res["vn_backward_bandwidth_fraction"] = vn_bwd_bytes / (res["vn_kernel_backward_us"] * 1e-6) / PEAK_BYTES_PER_S
    res["fan_forward_bandwidth_fraction"] = 76 * F / (res["fan_fused_forward_us"] * 1e-6) / PEAK_BYTES_PER_S
    res["fan_backward_bandwidth_fraction"] = (76 * F + 12 * V) / (res["fan_fused_backward_us"] * 1e-6) \
        / PEAK_BYTES_PER_S

    with torch.no_grad():
        res["stage_us"] = {
            "vn_forward": _stages(lambda: _C.verts_normals_forward(verts, faces)),
            "vn_backward": _stages(lambda: _C.verts_normals_backward(grad, verts, faces, table, sums)),
            "fan_backward": _stages(lambda: _C.face_areas_normals_backward(ga, gn, verts, faces)),
        }
    fwd = res["stage_us"]["vn_forward"]
    res["vn_forward_table_share"] = fwd.get("table", 0.0) / max(sum(fwd.values()), 1e-9)
    torch.cuda.empty_cache()
    print(name, json.dumps(res), flush=True)
    return res


def main():
    from pytorch3d_b200 import synthetic
    out_dir = sys.argv[1] if len(sys.argv) > 1 else "."
    assert torch.cuda.is_available(), "time_normals.py measures on a CUDA device"
    dev = torch.device("cuda:0")
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               stdout=subprocess.PIPE, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = "not measured"
    report = {"device": torch.cuda.get_device_name(dev), "power_limit": power, "workloads": {}}
    report["workloads"]["north_star_8x187x187"] = measure("north_star", synthetic.torus_batch(8, 187, 187, seed=0),
                                                          dev, 50)
    report["workloads"]["config5_707x707"] = measure("config5", synthetic.torus_batch(1, 707, 707, seed=0), dev, 50)
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "time_normals.json"), "w") as fh:
        json.dump(report, fh, indent=1)
    print(json.dumps({"device": report["device"], "power_limit": power}))


if __name__ == "__main__":
    main()
