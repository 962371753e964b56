"""Times the fused sample_points_from_meshes (pytorch3d_b200.sampling) against the reference's chain, restated here from
torch ops (pytorch3d/ops/sample_points_from_meshes.py: the emptiness and finiteness checks, the face areas under
no_grad, the padding, multinomial, rand, the gathers and the masked writes).

Per workload: forward and backward (through autograd) times from CUDA events, peak memory, host synchronisations per
forward (counted under torch.cuda.set_sync_debug_mode("warn")), and the fused forward's share of 3.35 TB/s (H100 SXM
HBM3) for the bytes it must move: faces (24 B) and their corners (36 B) and the float64 prefix (8 B, written and read
once) per face; per sample, the drawn face's row and corners (60 B) and the outputs (samples 12 B, normals 12 B, face id
8 B, barycentrics 12 B).  The card's name and power limit are printed with the table.

    python tools/time_sampling.py [--reps 20]
"""
import argparse
import json
import os
import subprocess
import sys
import warnings

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from pytorch3d_b200 import PackedMeshes, sampling, synthetic  # noqa: E402

HBM = 3.35e12


def chain(verts, faces, first, num, S, return_normals):
    """The reference's sample_points_from_meshes in torch ops, with its host reads."""
    valid = num > 0
    if not bool(valid.any()):
        raise ValueError("Meshes are empty.")
    if not torch.isfinite(verts).all():
        raise ValueError("Meshes contain nan or inf.")
    N = num.shape[0]
    n_valid = torch.sum(valid)
    samples = torch.zeros((N, S, 3), device=verts.device)
    with torch.no_grad():
        p = verts[faces]
        areas = torch.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0], dim=1).norm(dim=1) / 2
        max_faces = num.max().item()
        vf = first[valid]
        rows = torch.repeat_interleave(torch.arange(vf.shape[0], device=verts.device), num[valid])
        cols = torch.arange(faces.shape[0], device=verts.device) - first[valid][rows]
        padded = torch.zeros((vf.shape[0], max_faces), device=verts.device)
        padded[rows, cols] = areas
        idx = padded.multinomial(S, replacement=True)
        idx += vf.view(n_valid, 1)
    fv = verts[faces]
    v0, v1, v2 = fv[:, 0], fv[:, 1], fv[:, 2]
    uv = torch.rand(2, vf.shape[0], S, device=verts.device)
    s = uv[0].sqrt()
    w0, w1, w2 = 1.0 - s, s * (1.0 - uv[1]), s * uv[1]
    samples[valid] = w0[:, :, None] * v0[idx] + w1[:, :, None] * v1[idx] + w2[:, :, None] * v2[idx]
    if not return_normals:
        return samples
    normals = torch.zeros((N, S, 3), device=verts.device)
    n = (v1 - v0).cross(v2 - v1, dim=1)
    n = n / n.norm(dim=1, p=2, keepdim=True).clamp(min=sys.float_info.epsilon)
    normals[valid] = n[idx]
    return samples, normals


def fused(verts, faces, first, num, S, return_normals, m):
    m._verts_packed = verts
    return sampling.sample_points_from_meshes(m, S, return_normals=return_normals)


def measure(fn, args, reps):
    def fwd():
        return fn(*args)

    def loss(out):
        out = out if isinstance(out, tuple) else (out,)
        return sum(o.sum() for o in out)

    for _ in range(3):
        loss(fwd()).backward()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("warn")
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        out = fwd()
    torch.cuda.set_sync_debug_mode(0)
    syncs = sum("synchroniz" in str(x.message) for x in w)
    del out
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    tf = tb = 0.0
    for _ in range(reps):
        e[0].record()
        out = fwd()
        e[1].record()
        loss(out).backward()
        e[2].record()
        torch.cuda.synchronize()
        tf += e[0].elapsed_time(e[1])
        tb += e[1].elapsed_time(e[2])
    peak = torch.cuda.max_memory_allocated() - base
    return tf / reps, tb / reps, peak / 2 ** 20, syncs


def workloads():
    v, f = synthetic.ico_sphere(4)
    yield "tutorial ico_sphere(4), S=5k, normals", [v.float()], [f], 5000, True
    m = synthetic.torus_batch(8, 187, 187, seed=0)
    nv, nf = m.num_verts_per_mesh().tolist(), m.num_faces_per_mesh().tolist()
    vl = list(torch.split(m.verts_packed(), nv))
    fl = [x - o for x, o in zip(torch.split(m.faces_packed(), nf), m.mesh_to_verts_packed_first_idx().tolist())]
    yield "north-star 8 x 187^2 tori, S=100k, normals", vl, fl, 100_000, True
    v, f = synthetic.torus(707, 707)
    yield "config-5 torus 707^2, S=1M, normals", [v.float()], [f], 1_000_000, True
    F = (1 << 24) + 4096
    g = torch.Generator().manual_seed(0)
    i = torch.arange(F)
    yield "strip of 2^24 + 4096 faces, S=1M, normals", [torch.rand(F + 2, 3, generator=g)], \
        [torch.stack([i, i + 1, i + 2], 1)], 1_000_000, True


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         stdout=subprocess.PIPE, text=True).stdout.strip()
    print("card: %s" % smi)
    rows = []
    for name, vl, fl, S, normals in workloads():
        m = PackedMeshes([x.cuda() for x in vl], [x.cuda() for x in fl])
        verts = m.verts_packed().clone().requires_grad_(True)
        faces, first, num = m.faces_packed(), m.mesh_to_faces_packed_first_idx(), m.num_faces_per_mesh()
        V, F, N = verts.shape[0], faces.shape[0], len(vl)
        res = {"workload": name, "V": V, "F": F, "N": N, "S": S}
        ff, fb, fm, fs = measure(fused, (verts, faces, first, num, S, normals, m), a.reps)
        res.update(fused_fwd_ms=ff, fused_bwd_ms=fb, fused_peak_mb=fm, fused_syncs=fs)
        nbytes = F * (24 + 36 + 16) + N * S * (60 + 12 + (12 if normals else 0) + 8 + 12)
        res["fused_fwd_hbm_fraction"] = nbytes / (ff * 1e-3) / HBM
        if F < (1 << 24):
            cf, cb, cm, cs = measure(chain, (verts, faces, first, num, S, normals), a.reps)
            res.update(chain_fwd_ms=cf, chain_bwd_ms=cb, chain_peak_mb=cm, chain_syncs=cs)
        rows.append(res)
        print(json.dumps(res), flush=True)
        del m, verts
        torch.cuda.empty_cache()
    print("\n| workload | fwd fused / chain (ms) | bwd fused / chain (ms) | peak MB fused / chain | syncs | HBM share |")
    print("|---|---|---|---|---|---|")
    for r in rows:
        c = "chain_fwd_ms" in r
        print("| %s | %.3f / %s | %.3f / %s | %.0f / %s | %d / %s | %.2f |" % (
            r["workload"], r["fused_fwd_ms"], "%.3f" % r["chain_fwd_ms"] if c else "refused",
            r["fused_bwd_ms"], "%.3f" % r["chain_bwd_ms"] if c else "-", r["fused_peak_mb"],
            "%.0f" % r["chain_peak_mb"] if c else "-", r["fused_syncs"], str(r["chain_syncs"]) if c else "-",
            r["fused_fwd_hbm_fraction"]))
    print("card: %s" % smi)


if __name__ == "__main__":
    main()
