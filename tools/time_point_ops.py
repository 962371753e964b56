"""Times the fused farthest point sampling and ball query (pytorch3d_b200.point_ops) against the reference chain -- the
reference's ops recompiled for sm_90a (oracle/_ref/ref_point_ops_cuda.so, and ref_knn_cuda.so for ball query's
backward) behind a torch restatement of the reference's wrappers (pytorch3d/ops/sample_farthest_points.py,
ball_query.py and utils.masked_gather) -- with CUDA events, forward and backward, and reports peak memory and host
synchronisations per call.  Prints the card's name and power limit with the results.  `--sweep` also times the FPS
workloads at every forced cluster size, the evidence behind the launch policy.

    python tools/time_point_ops.py [--iters 10] [--sweep]
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

from oracle import build_ref_knn, build_ref_point_ops  # noqa: E402
from pytorch3d_b200 import _C, point_ops  # noqa: E402

DEV = "cuda"
FPS_WORKLOADS = [("fps 32x1024 K512", 32, 1024, 512), ("fps 8x8192 K1024", 8, 8192, 1024),
                 ("fps 1x100k K4096", 1, 100_000, 4096), ("fps 1x1M K1024", 1, 1_000_000, 1024)]
BALL_WORKLOADS = [("ball 16x512 in 1024 K32 r0.2", 16, 512, 1024, 32, 0.2),
                  ("ball 8x1024 in 8192 K32 r0.1", 8, 1024, 8192, 32, 0.1),
                  ("ball 4x4096 in 4096 K500 r0.2", 4, 4096, 4096, 500, 0.2),
                  ("ball 4x32k in 32k K16 r0.01", 4, 32768, 32768, 16, 0.01)]


def _gather_nn(points, idx):
    """The reference's masked_gather as torch operations (expand, gather, zero the padding in place)."""
    D = points.shape[2]
    if idx.ndim == 3:
        index = idx[..., None].expand(-1, -1, -1, D)
        points = points[:, :, None, :].expand(-1, -1, idx.shape[2], -1)
    else:
        index = idx[..., None].expand(-1, -1, D)
    mask = index.eq(-1)
    index = index.clone()
    index[mask] = 0
    out = points.gather(dim=1, index=index)
    out[mask] = 0.0
    return out


def ref_fps(ref):
    def fps(points, K):
        N, P, _ = points.shape
        lengths = torch.full((N,), P, dtype=torch.int64, device=points.device)
        Kt = torch.full((N,), K, dtype=torch.int64, device=points.device)
        with torch.no_grad():
            idx = ref.sample_farthest_points(points, lengths, Kt, torch.zeros_like(lengths), K)
        return _gather_nn(points, idx), idx
    return fps


def ref_ball(ref, knn):
    class _Ball(torch.autograd.Function):
        @staticmethod
        def forward(ctx, p1, p2, l1, l2, K, radius):
            idx, dists = ref.ball_query(p1, p2, l1, l2, K, radius, False)
            ctx.save_for_backward(p1, p2, l1, l2, idx)
            ctx.mark_non_differentiable(idx)
            return dists, idx

        @staticmethod
        def backward(ctx, gd, _):
            p1, p2, l1, l2, idx = ctx.saved_tensors
            g1, g2 = knn.knn_points_backward(p1, p2, l1, l2, idx, 2, gd.contiguous())
            return g1, g2, None, None, None, None

    def ball(p1, p2, K, radius):
        N, P1, P2 = p1.shape[0], p1.shape[1], p2.shape[1]
        l1 = torch.full((N,), P1, dtype=torch.int64, device=p1.device)
        l2 = torch.full((N,), P2, dtype=torch.int64, device=p1.device)
        dists, idx = _Ball.apply(p1, p2, l1, l2, K, radius)
        return dists, idx, _gather_nn(p2, idx)
    return ball


def _time(fn, iters):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def _peak_mib(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def _syncs(fn):
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
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--sweep", action="store_true")
    args = ap.parse_args()
    ref, knn = build_ref_point_ops.load(cuda=True), build_ref_knn.load(cuda=True)
    if ref is None or knn is None:
        raise SystemExit("oracle/_ref/ref_point_ops_cuda.so and ref_knn_cuda.so are needed (build() makes them)")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          stdout=subprocess.PIPE, text=True).stdout.strip()
    print(json.dumps({"card": card}))
    g = torch.Generator(device=DEV).manual_seed(0)
    rfps, rball = ref_fps(ref), ref_ball(ref, knn)
    for name, N, P, K in FPS_WORKLOADS:
        pts = torch.rand(N, P, 3, device=DEV, generator=g)
        ours = lambda: point_ops.sample_farthest_points(pts, K=K)  # noqa: E731
        theirs = lambda: rfps(pts, K)  # noqa: E731
        same = torch.equal(ours()[1], theirs()[1])
        iters = max(2, args.iters // (4 if P >= 100_000 else 1))
        row = {"workload": name, "same_idx": same}
        for tag, fn in (("fused", ours), ("ref", theirs)):
            row[tag + "_ms"] = round(_time(fn, iters), 3)
            row[tag + "_peak_mib"] = round(_peak_mib(fn), 1)
            row[tag + "_syncs"] = _syncs(fn)
        row["speedup"] = round(row["ref_ms"] / row["fused_ms"], 2)
        if args.sweep:
            lengths = torch.full((N,), P, dtype=torch.int64, device=DEV)
            Kt = torch.full((N,), K, dtype=torch.int64, device=DEV)
            start = torch.zeros_like(lengths)
            row["cluster_ms"] = {c: round(_time(lambda: _C.sample_farthest_points(pts, lengths, Kt, start, K, c),
                                                iters), 3) for c in (1, 2, 4, 6, 8, 12, 16)}
        print(json.dumps(row), flush=True)
    for name, N, P1, P2, K, r in BALL_WORKLOADS:
        p1 = torch.rand(N, P1, 3, device=DEV, generator=g)
        p2 = torch.rand(N, P2, 3, device=DEV, generator=g)
        gd = torch.randn(N, P1, K, device=DEV, generator=g)
        gnn = torch.randn(N, P1, K, 3, device=DEV, generator=g)
        a, b = p1.clone().requires_grad_(), p2.clone().requires_grad_()

        def fused_fwd():
            return point_ops.ball_query(a, b, K=K, radius=r)

        def ref_fwd():
            return rball(a, b, K, r)

        def fused_both():
            out = fused_fwd()
            torch.autograd.backward([out.dists, out.knn], [gd, gnn])

        def ref_both():
            d, _, nn = ref_fwd()
            torch.autograd.backward([d, nn], [gd, gnn])

        o, t = fused_fwd(), ref_fwd()
        row = {"workload": name, "same_idx": torch.equal(o.idx, t[1]),
               "same_dists": torch.equal(o.dists, t[0]), "hits_per_query": round(float((o.idx >= 0).sum()) / (N * P1), 2)}
        del o, t
        for tag, fwd, both in (("fused", fused_fwd, fused_both), ("ref", ref_fwd, ref_both)):
            with torch.no_grad():
                row[tag + "_fwd_ms"] = round(_time(fwd, args.iters), 3)
            row[tag + "_fwd_bwd_ms"] = round(_time(both, args.iters), 3)
            row[tag + "_peak_mib"] = round(_peak_mib(both), 1)
            row[tag + "_syncs"] = _syncs(both)
        row["speedup_fwd"] = round(row["ref_fwd_ms"] / row["fused_fwd_ms"], 2)
        row["speedup_fwd_bwd"] = round(row["ref_fwd_bwd_ms"] / row["fused_fwd_bwd_ms"], 2)
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
