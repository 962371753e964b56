"""Farthest point sampling and ball query on the GPU (DESIGN.md section 22): PointNet++'s "sample and group".

Drop-ins for `pytorch3d.ops.sample_farthest_points`, `pytorch3d.ops.ball_query` and `pytorch3d.ops.utils.
masked_gather` with the reference's signatures, defaults, return values, dtype conversions and error messages, for
CUDA point clouds with D = 3 (other D raise ValueError).  The sampled indices and the ball query's idx and dists are bit
for bit what the reference's CUDA kernels give; the ball query's backward is deterministic (no float atomics, no
(N, P2, K, 3) buffer) and neither op synchronises the host beyond what is stated on each function.
"""
from collections import namedtuple
from typing import List, Optional, Tuple, Union

import torch
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from . import _C

_KNN = namedtuple("KNN", "dists idx knn")


def masked_gather(points: torch.Tensor, idx: torch.Tensor) -> torch.Tensor:
    """points[n, idx[n, ...]] along dim 1 with zeros where idx is -1: (N, K) idx gives (N, K, D), (N, P', K) idx gives
    (N, P', K, D).  pytorch3d.ops.utils.masked_gather's values and gradients, through torch.gather, whose backward is
    deterministic."""
    if len(idx) != len(points):
        raise ValueError("points and idx must have the same batch dimension")
    D = points.shape[2]
    if idx.ndim == 3:
        index = idx[..., None].expand(-1, -1, -1, D)
        source = points[:, :, None, :].expand(-1, -1, idx.shape[2], -1)
    elif idx.ndim == 2:
        index = idx[..., None].expand(-1, -1, D)
        source = points
    else:
        raise ValueError("idx format is not supported %s" % repr(idx.shape))
    pad = index.eq(-1)
    return source.gather(1, index.masked_fill(pad, 0)).masked_fill(pad, 0.0)


def _require_3d(op, D):
    if D != 3:
        raise ValueError("pytorch3d_b200.%s takes points with D = 3, got D = %d" % (op, D))


def sample_farthest_points(
    points: torch.Tensor,
    lengths: Optional[torch.Tensor] = None,
    K: Union[int, List, torch.Tensor] = 50,
    random_start_point: bool = False,
) -> Tuple[torch.Tensor, torch.Tensor]:
    """Iterative farthest point sampling of K points from each cloud of points (N, P, 3): (selected_points (N, K, 3),
    selected_indices (N, K)), padded with 0.0 and -1 to max(K) when K varies.  The indices are the reference's CUDA
    kernel's bit for bit; `random_start_point` makes the reference's torch RNG calls in its order, so one seed gives
    the reference's start points.

    The host is not synchronised when `lengths` is None and K is an int or a list; otherwise once, for the check
    lengths.max() <= P and, when K is a tensor, for max(K), read together."""
    N, P, D = points.shape
    _require_3d("sample_farthest_points", D)
    device = points.device
    constant_length = lengths is None
    host = {}
    if lengths is None:
        lengths = torch.full((N,), P, dtype=torch.int64, device=device)
    elif lengths.shape != (N,):
        raise ValueError("points and lengths must have same batch dimension.")
    else:
        host["lengths"] = lengths.max()
    max_K = -1
    if isinstance(K, int):
        max_K = K
        K = torch.full((N,), K, dtype=torch.int64, device=device)
    elif isinstance(K, list):
        if len(K) > 0:
            max_K = max(int(k) for k in K)
        K = torch.tensor(K, dtype=torch.int64)
        # from pinned memory, so that the copy does not synchronise the host
        K = K.pin_memory().to(device, non_blocking=True) if device.type == "cuda" else K.to(device)
    elif K.dim() == 1 and K.shape[0] == N and N > 0:
        host["K"] = K.max()
    if host:  # one synchronisation for both values
        values = dict(zip(host, torch.stack([v.to(torch.float64) for v in host.values()]).tolist()))
        if values.get("lengths", 0) > P:
            raise ValueError("A value in lengths was too large.")
        if "K" in values:
            max_K = int(values["K"])
    if K.shape[0] != N:
        raise ValueError("K and points must have the same batch dimension")
    if not (points.dtype == torch.float32):
        points = points.to(torch.float32)
    if not (lengths.dtype == torch.int64):
        lengths = lengths.to(torch.int64)
    if not (K.dtype == torch.int64):
        K = K.to(torch.int64)
    if random_start_point:
        if constant_length:
            start_idxs = torch.randint(high=P, size=(N,), device=device)
        else:
            start_idxs = (lengths * torch.rand(lengths.size(), device=device)).to(torch.int64)
    else:
        start_idxs = torch.zeros_like(lengths)
    with torch.no_grad():
        if max_K <= 0:
            idx = torch.full((N, max_K), -1, dtype=torch.int64, device=device)  # (N, 0), or the negative-size error
        else:
            idx = _C.sample_farthest_points(points, lengths, K, start_idxs, max_K)
    return masked_gather(points, idx), idx


class _BallQuery(Function):
    """dists and nn of the ball query with the deterministic backward of `_C.ball_query_backward`."""

    @staticmethod
    def forward(ctx, p1, p2, lengths1, lengths2, K, radius, skip_points_outside_cube, return_nn):
        idx, dists, nn = _C.ball_query_forward(p1, p2, lengths1, lengths2, K, radius, skip_points_outside_cube,
                                               return_nn)
        ctx.save_for_backward(p1, p2, lengths1, lengths2, idx)
        ctx.mark_non_differentiable(idx)
        ctx.set_materialize_grads(False)
        return dists, idx, nn

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_dists, grad_idx, grad_nn):
        p1, p2, lengths1, lengths2, idx = ctx.saved_tensors
        grad_p1, grad_p2 = None, None
        if grad_dists is not None or grad_nn is not None:
            grad_p1, grad_p2 = _C.ball_query_backward(p1, p2, lengths1, lengths2, idx, grad_dists, grad_nn,
                                                      ctx.needs_input_grad[0], ctx.needs_input_grad[1])
        return grad_p1, grad_p2, None, None, None, None, None, None


def ball_query(
    p1: torch.Tensor,
    p2: torch.Tensor,
    lengths1: Union[torch.Tensor, None] = None,
    lengths2: Union[torch.Tensor, None] = None,
    K: int = 500,
    radius: float = 0.2,
    return_nn: bool = True,
    skip_points_outside_cube: bool = False,
):
    """The first K points of p2 (N, P2, 3) within `radius` of each point of p1 (N, P1, 3), in index order: a
    (dists, idx, knn) named tuple as pytorch3d.ops.ball_query returns, idx and dists bit for bit the reference's CUDA
    kernel's, knn (N, P1, K, 3) what masked_gather(p2, idx) gives (None unless return_nn).  Gradients flow to p1 and p2
    from dists and knn, deterministically.  No host synchronisation."""
    if p1.shape[0] != p2.shape[0]:
        raise ValueError("pts1 and pts2 must have the same batch dimension.")
    if p1.shape[2] != p2.shape[2]:
        raise ValueError("pts1 and pts2 must have the same point dimension.")
    _require_3d("ball_query", p1.shape[2])
    p1 = p1.contiguous()
    p2 = p2.contiguous()
    dists, idx, nn = _BallQuery.apply(p1, p2, lengths1, lengths2, K, radius, skip_points_outside_cube, return_nn)
    return _KNN(dists=dists, idx=idx, knn=nn)
