"""Times the fused chamfer_distance (forward + backward) against the reference chain -- the reference's knn ops
recompiled for sm_90a (oracle/_ref/ref_knn_cuda.so) plus a torch restatement of pytorch3d/loss/chamfer.py -- on four
workloads, with CUDA events, and reports peak memory, host synchronisations per call and the search's pairs per second.
Prints the card's name and power limit with the results.

    python tools/time_chamfer.py [--iters 20]
"""
import argparse
import json
import os
import subprocess
import sys
import warnings

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import build_ref_knn  # noqa: E402
from pytorch3d_b200.chamfer import chamfer_distance  # noqa: E402


def ref_chain(ref):
    class _Knn(torch.autograd.Function):
        @staticmethod
        def forward(ctx, p1, p2, l1, l2):
            idx, d = ref.knn_points_idx(p1, p2, l1, l2, 2, 1, -1)
            ctx.save_for_backward(p1, p2, l1, l2, idx)
            return d, idx

        @staticmethod
        def backward(ctx, gd, _):
            p1, p2, l1, l2, idx = ctx.saved_tensors
            g1, g2 = ref.knn_points_backward(p1, p2, l1, l2, idx, 2, gd.contiguous())
            return g1, g2, None, None

    def one(x, y, xl, yl, xn, yn):
        N, P1, _ = x.shape
        het = (xl != P1).any()
        mask = torch.arange(P1, device=x.device)[None] >= xl[:, None]
        d, idx = _Knn.apply(x, y, xl, yl)
        cx = d[..., 0]
        if het:
            cx = cx.masked_fill(mask, 0.0)
        cn = None
        if xn is not None:
            near = yn.gather(1, idx.expand(-1, -1, 3))
            if yl.min() < 1:
                near = near.masked_fill((yl < 1)[:, None, None], 0.0)
            cn = 1 - torch.abs(F.cosine_similarity(xn, near, dim=2, eps=1e-6))
            if het:
                cn = cn.masked_fill(mask, 0.0)
            cn = cn.sum(1) / xl.clamp(min=1)
        return cx.sum(1) / xl.clamp(min=1), cn

    def cd(x, y, x_lengths, y_lengths, x_normals=None, y_normals=None):
        cx, nx = one(x, y, x_lengths, y_lengths, x_normals, y_normals)
        cy, ny = one(y, x, y_lengths, x_lengths, y_normals, x_normals)
        N = x.shape[0]
        loss = (cx + cy).sum() / N
        return loss, ((nx + ny).sum() / N if nx is not None else None)

    return cd


def workloads():
    g = torch.Generator().manual_seed(0)
    out = []
    for normals in (False, True):
        out.append(("tutorial 1 x 5000 vs 5000" + (" + normals" if normals else ""), 1, 5000, 5000, None, normals))
    out.append(("8 x 100k vs 100k", 8, 100000, 100000, None, False))
    lens = torch.randint(1000, 50001, (2, 16), generator=g)
    out.append(("16 ragged 1k-50k", 16, 50000, 50000, lens, False))
    out.append(("1 x 2^18 vs 2^18", 1, 1 << 18, 1 << 18, None, False))
    return out


def time_call(fn, iters):
    fn()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / iters, torch.cuda.max_memory_allocated() / 2**20


def count_syncs(fn):
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("warn")
    try:
        with warnings.catch_warnings(record=True) as rec:
            warnings.simplefilter("always")
            fn()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    return len([w for w in rec if "synchroniz" in str(w.message)])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    ref = build_ref_knn.load(cuda=True)
    chain = ref_chain(ref) if ref is not None else None
    dev = "cuda"
    res = {"gpu": q, "workloads": []}
    for name, N, P1, P2, lens, normals in workloads():
        g = torch.Generator().manual_seed(1)
        x = torch.rand(N, P1, 3, generator=g).to(dev).requires_grad_()
        y = torch.rand(N, P2, 3, generator=g).to(dev).requires_grad_()
        xl = (lens[0] if lens is not None else torch.full((N,), P1)).to(dev)
        yl = (lens[1] if lens is not None else torch.full((N,), P2)).to(dev)
        xn = torch.randn(N, P1, 3, generator=g).to(dev) if normals else None
        yn = torch.randn(N, P2, 3, generator=g).to(dev) if normals else None
        pairs = 2 * float((xl * yl).sum())
        row = {"workload": name}

        def step(cd):
            loss, ln = cd(x, y, x_lengths=xl if lens is not None else None,
                          y_lengths=yl if lens is not None else None, x_normals=xn, y_normals=yn)
            (loss + (ln if ln is not None else 0.0)).backward()

        def step_ref():
            loss, ln = chain(x, y, xl, yl, xn, yn)
            (loss + (ln if ln is not None else 0.0)).backward()

        ms, mem = time_call(lambda: step(chamfer_distance), a.iters)
        row.update(fused_ms=ms, fused_peak_mib=mem, fused_syncs=count_syncs(lambda: step(chamfer_distance)),
                   pairs_per_s=pairs / (ms * 1e-3))
        if chain is not None:
            ms_r, mem_r = time_call(step_ref, a.iters)
            row.update(ref_ms=ms_r, ref_peak_mib=mem_r, ref_syncs=count_syncs(step_ref), speedup=ms_r / ms)
        res["workloads"].append(row)
        print(json.dumps(row), flush=True)
    print(json.dumps({"gpu": q}))


if __name__ == "__main__":
    main()
