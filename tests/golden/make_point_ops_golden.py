"""Writes tests/golden/reference_golden_point_ops.npz: the reference's own CPU farthest point sampling and ball query
ops (oracle/_ref/ref_point_ops_cpu.so, built by oracle/build_ref_point_ops.py) on the scenes of
tests/test_point_ops.py, with the ball query's gradients from the reference's CPU knn_points_backward
(oracle/_ref/ref_knn_cpu.so) plus torch's gather backward, as pytorch3d/ops/ball_query.py chains them.  The scenes use
small-integer coordinates, where the CPU build (no FMA) and the CUDA build (FMA) agree bit for bit.  Keys:
  fps/<scene>/0/idx, fps/<scene>/0/start
  ball/<case>/0/idx, ball/<case>/0/dists, ball/<case>/0/grad_p1, ball/<case>/0/grad_p2
(the name/index/field layout of the other records, so tests/helpers.py: reference reads them).

    python tests/golden/make_point_ops_golden.py [OUT_DIR]
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.dirname(HERE)]

from oracle import build_ref_knn, build_ref_point_ops  # noqa: E402
import test_point_ops as T  # noqa: E402


def _lengths(v, N, P):
    return torch.full((N,), P, dtype=torch.int64) if v is None else torch.tensor(v, dtype=torch.int64)


def _gather_nn(points, idx):
    """pytorch3d/ops/utils.py's masked_gather for (N, P1, K) idx, as torch operations: expand, gather, zero the
    padding in place."""
    D, K = points.shape[2], idx.shape[2]
    index = idx[..., None].expand(-1, -1, -1, D)
    mask = index.eq(-1)
    index = index.clone()
    index[mask] = 0
    out = points[:, :, None, :].expand(-1, -1, K, -1).gather(dim=1, index=index)
    out[mask] = 0.0
    return out


def main(out_dir):
    ref, knn = build_ref_point_ops.load(cuda=False), build_ref_knn.load(cuda=False)
    if ref is None or knn is None:
        raise SystemExit("build oracle/_ref/ref_point_ops_cpu.so and ref_knn_cpu.so first (oracle/build_ref_*.py)")
    rec = {}
    for name, sc in T.fps_scenes().items():
        pts = sc["points"]
        N, P = pts.shape[:2]
        idx = ref.sample_farthest_points(pts, _lengths(sc["lengths"], N, P), torch.tensor(sc["K"]),
                                         torch.tensor(sc["start"], dtype=torch.int64), sc["max_K"])
        rec["fps/%s/0/idx" % name] = idx.numpy()
        rec["fps/%s/0/start" % name] = np.asarray(sc["start"], np.int64)
    scenes = T.ball_scenes()
    for case, (scene, K, radius, skip) in T.BALL_CASES.items():
        sc = scenes[scene]
        p1, p2 = sc["p1"], sc["p2"]
        N, P1, P2 = p1.shape[0], p1.shape[1], p2.shape[1]
        l1, l2 = _lengths(sc["lengths1"], N, P1), _lengths(sc["lengths2"], N, P2)
        idx, dists = ref.ball_query(p1, p2, l1, l2, K, radius, skip)
        rec["ball/%s/0/idx" % case] = idx.numpy()
        rec["ball/%s/0/dists" % case] = dists.numpy()
        gd, gnn = T.ball_upstream(case, tuple(idx.shape))
        g1, g2 = knn.knn_points_backward(p1, p2, l1, l2, idx, 2, gd)
        b = p2.clone().requires_grad_()
        (_gather_nn(b, idx) * gnn).sum().backward()
        rec["ball/%s/0/grad_p1" % case] = g1.numpy()
        rec["ball/%s/0/grad_p2" % case] = (g2 + b.grad).numpy()
    path = os.path.join(out_dir, "reference_golden_point_ops.npz")
    np.savez_compressed(path, **rec)
    print("wrote", path, len(rec), "arrays")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else HERE)
