"""Chamfer distance on the GPU: `chamfer_distance`, with the signature, defaults, return values, shapes, dtypes and
errors of pytorch3d/loss/chamfer.py, for float32 3-D point clouds on one CUDA device.

The nearest-neighbour search is a fused sm_90a kernel (DESIGN.md section 21) that finds, bit for bit, the neighbours
and distances of the reference's KNearestNeighborKernelV3<float, 3, 1>: the same float32 expression, ascending target
order, the lowest index on exact ties, and a NaN distance to target 0 kept.  The masks, weights, cosine term and
reductions run in an epilogue kernel with a fixed association, so repeated calls are bitwise equal.  The backward sums
every point's gradient rows in a fixed order, with no float atomics, so it runs under
`torch.use_deterministic_algorithms(True)`.

The host is synchronised only where the reference checks data values: when `x_lengths` or `y_lengths` is a tensor
(too long) or `weights` is given (negative, or summing to zero), one status word written by the kernels is read once.
Otherwise neither the forward nor the backward synchronises.

`x` and `y` are tensors (N, P, 3) or Pointclouds-like objects (`points_padded()`, `num_points_per_cloud()`,
`normals_padded()`).  Gradients reach x, y and both normals; `weights` must not require grad.
"""
import torch
from torch.autograd.function import once_differentiable

from . import _C

__all__ = ["chamfer_distance"]


class _Chamfer(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, y, x_normals, y_normals, x_lengths, y_lengths, weights, opts):
        outs, state, status = _C.chamfer_forward(x, y, x_lengths, y_lengths, x_normals, y_normals, weights, *opts)
        ctx.save_for_backward(x, y, x_normals, y_normals, x_lengths, y_lengths, weights, *state)
        ctx.opts = opts
        ctx.mark_non_differentiable(status)
        return tuple(outs) + (status,)

    @staticmethod
    @once_differentiable
    def backward(ctx, gx, gy, gnx, gny, _status):
        x, y, xn, yn, xl, yl, w, *state = ctx.saved_tensors
        need = ctx.needs_input_grad
        grads = _C.chamfer_backward(x, y, xl, yl, xn, yn, w, *ctx.opts, state, (gx, gy, gnx, gny),
                                    need[0] or need[1], need[2] or need[3])
        return tuple(g if need[k] else None for k, g in enumerate(grads)) + (None,) * 4


def _is_pointclouds(points):
    return (not torch.is_tensor(points)) and hasattr(points, "points_padded") and \
        hasattr(points, "num_points_per_cloud")


def _reference_error(msg):
    return ValueError(msg)


def _validate(batch_reduction, point_reduction, norm, x_normals, y_normals):
    if batch_reduction is not None and batch_reduction not in ["mean", "sum"]:
        raise ValueError('batch_reduction must be one of ["mean", "sum"] or None')
    if point_reduction is not None and point_reduction not in ["mean", "sum", "max"]:
        raise ValueError('point_reduction must be one of ["mean", "sum", "max"] or None')
    if point_reduction is None and batch_reduction is not None:
        raise ValueError("Batch reduction must be None if point_reduction is None")
    if not ((norm == 1) or (norm == 2)):
        raise ValueError("Support for 1 or 2 norm.")
    if point_reduction == "max" and (x_normals is not None or y_normals is not None):
        raise ValueError('Normals must be None if point_reduction is "max"')


class _Checks:
    """The reference's checks in its order.  The ones on data values ("A length value was too long") are deferred to
    the status word on the normal path; a host-decided error raised after them evaluates them first, as the
    reference would have."""

    def __init__(self):
        self.pending = []  # (tensor lengths, P) whose "too long" check precedes what follows

    def fail(self, msg):
        for lengths, P in self.pending:
            if lengths.max() > P:
                raise ValueError("A length value was too long")
        raise ValueError(msg)

    def cloud(self, points, lengths, normals):
        if _is_pointclouds(points):
            return points.points_padded(), points.num_points_per_cloud(), points.normals_padded(), False
        if not torch.is_tensor(points):
            self.fail("The input pointclouds should be either Pointclouds objects or torch.Tensor of shape "
                      "(minibatch, num_points, 3).")
        if points.ndim != 3:
            self.fail("Expected points to be of shape (N, P, D)")
        checked = False
        if lengths is not None:
            if lengths.ndim != 1 or lengths.shape[0] != points.shape[0]:
                self.fail("Expected lengths to be of shape (N,)")
            self.pending.append((lengths, points.shape[1]))
            checked = True
        if normals is not None and normals.ndim != 3:
            self.fail("Expected normals to be of shape (N, P, 3")
        return points, lengths, normals, checked


def _zero_weight_result(x, y, weights, point_reduction, batch_reduction, single_directional):
    """chamfer.py's result when weights.sum() == 0: (x.sum((1, 2)) * weights.view(N, 1)) * 0.0 for each term."""
    N = x.shape[0]
    wv = weights.view(N, 1)
    cx = (x.sum((1, 2)) * wv) * 0.0
    if single_directional:
        loss, loss_n = cx, cx
    else:
        cy = (y.sum((1, 2)) * wv) * 0.0
        if point_reduction == "max":
            loss, loss_n = torch.maximum(cx, cy), None
        elif point_reduction is not None:
            loss, loss_n = cx + cy, cx + cy
        else:
            loss, loss_n = (cx, cy), (cx, cy)
    if batch_reduction is None:
        return loss, loss_n
    loss = loss.sum()
    if loss_n is not None:
        loss_n = loss_n.sum()
    return loss, loss_n  # batch mean divides by 1 when the weights sum to zero


def chamfer_distance(x, y, x_lengths=None, y_lengths=None, x_normals=None, y_normals=None, weights=None,
                     batch_reduction="mean", point_reduction="mean", norm: int = 2, single_directional: bool = False,
                     abs_cosine: bool = True):
    """Chamfer distance between the point clouds x and y, as pytorch3d.loss.chamfer_distance: returns (loss,
    loss_normals), with the reference's shapes for every point_reduction ("mean", "sum", "max", None) and
    batch_reduction ("mean", "sum", None)."""
    _validate(batch_reduction, point_reduction, norm, x_normals, y_normals)
    chk = _Checks()
    x, x_lengths, x_normals, x_checked = chk.cloud(x, x_lengths, x_normals)
    y, y_lengths, y_normals, y_checked = chk.cloud(y, y_lengths, y_normals)
    N, P1, D = x.shape
    if y.shape[0] != N or y.shape[2] != D:
        chk.fail("y does not have the correct shape.")
    if weights is not None and weights.size(0) != N:
        chk.fail("weights must be of shape (N,).")
    if D != 3:
        raise ValueError("pytorch3d_b200.chamfer_distance takes 3-D points, got D = %d" % D)
    if x_normals is None or y_normals is None:  # the normal term needs both
        x_normals = y_normals = None
    opts = (int(norm), point_reduction, batch_reduction, bool(single_directional), bool(abs_cosine))
    out = _Chamfer.apply(x, y, x_normals, y_normals, x_lengths, y_lengths, weights, opts)
    lx, ly, nx, ny, status = out
    if x_checked or y_checked or weights is not None:
        s = int(status.item())
        if s & _C.CHAMFER_X_LENGTH and x_checked:
            raise ValueError("A length value was too long")
        if s & _C.CHAMFER_Y_LENGTH and y_checked:
            raise ValueError("A length value was too long")
        if s & _C.CHAMFER_W_NEGATIVE:
            raise ValueError("weights cannot be negative.")
        if s & _C.CHAMFER_W_ZERO_SUM:
            return _zero_weight_result(x, y, weights, point_reduction, batch_reduction, single_directional)
    if point_reduction is None and not single_directional:
        return (lx, ly), ((nx, ny) if nx is not None else None)
    return lx, nx
