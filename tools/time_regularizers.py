"""Times the fused mesh regularisers on the GPU against the torch chain of the reference's losses, forward and backward
through autograd.  CUDA events, 50 iterations after warm-up; peak memory of forward + backward; the card's name and
power limit are read in the same run.

    python tools/time_regularizers.py OUT_DIR        -> OUT_DIR/time_regularizers.json

The chain restates pytorch3d/loss/mesh_edge_loss.py, mesh_laplacian_smoothing.py, mesh_normal_consistency.py and
ops/laplacian_matrices.py on a mesh without cached topology (each iteration of a fitting loop has a fresh mesh from
offset_verts): Meshes._compute_edges_packed (torch.unique and a sort of the 3F hashes), the sparse Laplacians with
torch.sparse and mm, and normal consistency's sort, host copy of the edge counts and pair enumeration.  The pair
enumeration is the reference's CPU op built by oracle/build_ref_regularizers.py when oracle/_ref has it; otherwise a
torch stand-in (pairs of the runs of length 2 vectorised, longer runs in Python, also on the host after the same copy),
and the report names which one ran ("pairs_op").

Workloads: the tutorials' scale, ico_sphere(4) (V = 2,562, F = 5,120), where launches and the host round trip dominate;
the north-star tori (8 x 187 x 187: V = 279,752, F = 559,504); the 707 x 707 torus (V = 499,849, F = 999,698).
Fields per workload and loss: fused_forward_us, fused_backward_us, chain_forward_us, chain_backward_us,
fused_peak_bytes, chain_peak_bytes, and the loss of each (fused_loss, chain_loss).
"""
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools")]

from time_blend import _events_ms, _peak_bytes, _time_backward_ms  # noqa: E402

LOSSES = (("edge", None), ("laplacian_uniform", "uniform"), ("laplacian_cot", "cot"),
          ("laplacian_cotcurv", "cotcurv"), ("normal_consistency", None))


class ChainMesh:
    """What the reference's losses read from a Meshes with no cached topology, computed as Meshes computes it."""

    def __init__(self, verts, faces, nverts, nfaces):
        self.verts, self.faces = verts, faces
        dev = verts.device
        self.N = len(nverts)
        self.num_verts = torch.tensor(nverts, device=dev)
        self.verts_to_mesh = torch.repeat_interleave(torch.arange(self.N, device=dev), self.num_verts)
        self.faces_to_mesh = torch.repeat_interleave(torch.arange(self.N, device=dev), torch.tensor(nfaces, device=dev))

    def edges(self):
        faces, V, F = self.faces, self.verts.shape[0], self.faces.shape[0]
        v0, v1, v2 = faces.chunk(3, dim=1)
        edges = torch.cat([torch.cat([v1, v2], 1), torch.cat([v2, v0], 1), torch.cat([v0, v1], 1)], 0)
        edge_to_mesh = torch.cat([self.faces_to_mesh] * 3)
        edges, _ = edges.sort(dim=1)
        h = V * edges[:, 0] + edges[:, 1]
        u, inverse = torch.unique(h, return_inverse=True)
        sorted_hash, sort_idx = torch.sort(h, dim=0)
        mask = torch.ones(h.shape[0], dtype=torch.bool, device=h.device)
        mask[1:] = sorted_hash[1:] != sorted_hash[:-1]
        e2m = edge_to_mesh[sort_idx[mask]]
        counts = torch.zeros(self.N, dtype=torch.int32, device=h.device).scatter_add_(
            0, e2m, torch.ones(1, dtype=torch.int32, device=h.device).expand(e2m.shape))
        return torch.stack([u // V, u % V], 1), e2m, counts, inverse.reshape(3, F).t()


def chain_edge_loss(m):
    edges, e2m, counts, _ = m.edges()
    w = 1.0 / counts.gather(0, e2m).float()
    v0, v1 = m.verts[edges].unbind(1)
    return (((v0 - v1).norm(dim=1, p=2) - 0.0) ** 2.0 * w).sum() / m.N


def _uniform_L(verts, edges):
    V = verts.shape[0]
    e0, e1 = edges.unbind(1)
    idx = torch.cat([torch.stack([e0, e1], 1), torch.stack([e1, e0], 1)], 0).t()
    A = torch.sparse_coo_tensor(idx, torch.ones(idx.shape[1], device=verts.device), (V, V))
    deg = torch.sparse.sum(A, dim=1).to_dense()
    d0, d1 = deg[e0], deg[e1]
    val = torch.cat([torch.where(d0 > 0, 1.0 / d0, d0), torch.where(d1 > 0, 1.0 / d1, d1)])
    L = torch.sparse_coo_tensor(idx, val, (V, V))
    i = torch.arange(V, device=verts.device)
    return L - torch.sparse_coo_tensor(torch.stack([i, i]), torch.ones(V, device=verts.device), (V, V))


def _cot_L(verts, faces):
    V, F = verts.shape[0], faces.shape[0]
    fv = verts[faces]
    a, b, c = fv[:, 0], fv[:, 1], fv[:, 2]
    A, B, C = (b - c).norm(dim=1), (a - c).norm(dim=1), (a - b).norm(dim=1)
    s = 0.5 * (A + B + C)
    area = (s * (s - A) * (s - B) * (s - C)).clamp(min=1e-12).sqrt()
    A2, B2, C2 = A * A, B * B, C * C
    cot = torch.stack([(B2 + C2 - A2) / area, (A2 + C2 - B2) / area, (A2 + B2 - C2) / area], 1) / 4.0
    idx = torch.stack([faces[:, [1, 2, 0]], faces[:, [2, 0, 1]]], 0).view(2, F * 3)
    L = torch.sparse_coo_tensor(idx, cot.view(-1), (V, V))
    L = L + L.t()
    inv = torch.zeros(V, device=verts.device).scatter_add_(0, faces.view(-1), torch.stack([area] * 3, 1).view(-1))
    pos = inv > 0
    inv[pos] = torch.reciprocal(inv[pos])
    return L, inv.view(-1, 1)


def chain_laplacian(m, method):
    verts = m.verts
    w = 1.0 / m.num_verts.gather(0, m.verts_to_mesh).float()
    with torch.no_grad():
        if method == "uniform":
            L = _uniform_L(verts, m.edges()[0])
        else:
            L, inv_areas = _cot_L(verts, m.faces)
            norm_w = torch.sparse.sum(L, dim=1).to_dense().view(-1, 1)
            if method == "cot":
                pos = norm_w > 0
                norm_w[pos] = torch.reciprocal(norm_w[pos])
            else:
                L_sum = norm_w
                norm_w = 0.25 * inv_areas
    if method == "uniform":
        loss = L.mm(verts)
    elif method == "cot":
        loss = L.mm(verts) * norm_w - verts
    else:
        loss = (L.mm(verts) - L_sum * verts) * norm_w
    return (loss.norm(dim=1) * w).sum() / m.N


def _pairs_stand_in(edge_num):
    """(P, 2) pairs of positions on one edge, as the reference's op lists them, from host counts."""
    ends = torch.cumsum(edge_num, 0)
    starts = ends - edge_num
    two = starts[edge_num == 2]
    out = [torch.stack([two, two + 1], 1)]
    for s, k in zip(starts[edge_num > 2].tolist(), edge_num[edge_num > 2].tolist()):
        out.append(torch.tensor([[s + i, s + j] for j in range(k) for i in range(j)], dtype=torch.int64))
    pairs = torch.cat(out)
    return pairs[torch.argsort(pairs[:, 0] * (int(ends[-1]) + 1) + pairs[:, 1])] if len(pairs) else pairs


def chain_normal_consistency(m, pairs_op):
    verts, faces = m.verts, m.faces
    F = faces.shape[0]
    edges, _, _, f2e = m.edges()
    with torch.no_grad():
        edge_idx = f2e.reshape(F * 3)
        vert_idx = faces.view(1, F, 3).expand(3, F, 3).transpose(0, 1).reshape(3 * F, 3)
        edge_idx, order = edge_idx.sort()
        vert_idx = vert_idx[order]
        edge_num = edge_idx.bincount(minlength=edges.shape[0])
        pairs = (pairs_op(edge_num.cpu()) if pairs_op is not None else _pairs_stand_in(edge_num.cpu())).to(verts.device)
    v0, v1 = verts[edges[edge_idx, 0]], verts[edges[edge_idx, 1]]
    n = sum((v1 - v0).cross(verts[vert_idx[:, k]] - v0, dim=1) for k in range(3))
    loss = 1 - torch.cosine_similarity(n[pairs[:, 0]], -n[pairs[:, 1]], dim=1)
    pm = m.verts_to_mesh[vert_idx[:, 0]][pairs[:, 0]]
    w = 1.0 / pm.bincount(minlength=m.N)[pm].float()
    return (loss * w).sum() / m.N


def measure(name, verts, faces, nverts, nfaces, dev, iters, pairs_op):
    from pytorch3d_b200 import regularizers
    from pytorch3d_b200.structures import PackedMeshes
    res = {"V": int(verts.shape[0]), "F": int(faces.shape[0])}
    leaf = verts.clone().requires_grad_(True)
    pm = PackedMeshes([leaf], [faces])
    pm._num_verts_per_mesh = torch.tensor(nverts, device=dev)
    pm._mesh_to_verts_packed_first_idx = torch.cumsum(pm._num_verts_per_mesh, 0) - pm._num_verts_per_mesh
    pm._N = len(nverts)
    pm._verts_packed = leaf
    cm = ChainMesh(leaf, faces, nverts, nfaces)
    g = torch.tensor(1.0, device=dev)
    for loss, arg in LOSSES:
        if loss == "edge":
            fused, chain = (lambda: regularizers.mesh_edge_loss(pm)), (lambda: chain_edge_loss(cm))
        elif loss == "normal_consistency":
            fused = lambda: regularizers.mesh_normal_consistency(pm)  # noqa: E731
            chain = lambda: chain_normal_consistency(cm, pairs_op)  # noqa: E731
        else:
            fused = lambda a=arg: regularizers.mesh_laplacian_smoothing(pm, method=a)  # noqa: E731
            chain = lambda a=arg: chain_laplacian(cm, a)  # noqa: E731
        r = {}
        for kind, fn in (("fused", fused), ("chain", chain)):
            for _ in range(3):
                fn().backward(g)
            r[kind + "_loss"] = float(fn().detach())
            r[kind + "_forward_us"] = 1e3 * _events_ms(fn, iters)
            r[kind + "_backward_us"] = 1e3 * _time_backward_ms(fn, g, [leaf], iters)
            leaf.grad = None
            r[kind + "_peak_bytes"] = _peak_bytes(lambda: fn().backward(g))
            leaf.grad = None
        r["forward_speedup"] = r["chain_forward_us"] / r["fused_forward_us"]
        r["backward_speedup"] = r["chain_backward_us"] / r["fused_backward_us"]
        res[loss] = r
        print(name, loss, json.dumps(r), flush=True)
    torch.cuda.empty_cache()
    return res


def main():
    from pytorch3d_b200 import synthetic
    from oracle import build_ref_regularizers
    out_dir = sys.argv[1] if len(sys.argv) > 1 else "."
    assert torch.cuda.is_available(), "time_regularizers.py measures on a CUDA device"
    dev = torch.device("cuda:0")
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               stdout=subprocess.PIPE, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = "not measured"
    ref = build_ref_regularizers.load()
    pairs_op = ref.mesh_normal_consistency_find_verts if ref is not None else None
    report = {"device": torch.cuda.get_device_name(dev), "power_limit": power,
              "pairs_op": "reference CPU op (oracle/_ref)" if ref is not None else "torch stand-in", "workloads": {}}
    print("pairs op:", report["pairs_op"], flush=True)
    v, f = synthetic.ico_sphere(4)
    report["workloads"]["ico_sphere4"] = measure("ico_sphere4", v.float().to(dev), f.to(dev), [v.shape[0]],
                                                 [f.shape[0]], dev, 50, pairs_op)
    for name, m in (("north_star_8x187x187", synthetic.torus_batch(8, 187, 187, seed=0)),
                    ("config5_707x707", synthetic.torus_batch(1, 707, 707, seed=0))):
        report["workloads"][name] = measure(name, m.verts_packed().to(dev), m.faces_packed().to(dev),
                                            m.num_verts_per_mesh().tolist(), m.num_faces_per_mesh().tolist(), dev,
                                            50, pairs_op)
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "time_regularizers.json"), "w") as fh:
        json.dump(report, fh, indent=1)
    print(json.dumps({"device": report["device"], "power_limit": power, "pairs_op": report["pairs_op"]}))


if __name__ == "__main__":
    main()
