"""``ScatterConnection`` with the constructor and methods of ding/torch_utils/network/scatter_connection.py:30-121 --
csrc/scatter.cu.

The map is what the reference computes on the CPU, bit for bit: each cell is +0.0 plus the entities whose flat index falls
in it, added in ascending entity order ('add'), or the entity of the largest index m ('cover'); an empty cell is +0.0.  On
CUDA the reference's 'cover' picks an arbitrary entity and its 'add' sums in an arbitrary order; these kernels give the
same bits on every run.  d x[b, m] is the map's gradient at the entity's cell, covered entities included.
"""
from typing import Tuple

import torch
import torch.nn as nn

from .. import ops, torch_ops


def _index(t, shape, name):
    if not isinstance(t, torch.Tensor) or t.dtype != torch.int64:
        raise TypeError("di_engine_b200: ScatterConnection's %s must be an int64 tensor (got %s)" %
                        (name, getattr(t, 'dtype', type(t).__name__)))
    if tuple(t.shape) != shape:
        raise ValueError("di_engine_b200: ScatterConnection's %s has shape %s, expected %s" % (name, tuple(t.shape), shape))


def _scatter(x, spatial_size, row, col, scatter_type):
    """the map (B, N, H, W) of x (B, M, N) at the flat indices col + row * W of the (B, M) int64 tensors row and col"""
    B, M, N = x.shape
    H, W = (int(s) for s in spatial_size)
    dev = ops.compute_device(x, row, col)
    host_out = not x.is_cuda
    x, row, col = (ops.to_device(t, dev) for t in (x, row, col))
    if ops.CHECK_INDICES and B * M:
        lo, hi = torch.aminmax(col + row * W)
        lo, hi = int(lo), int(hi)
        if lo < 0 or hi >= H * W:
            raise IndexError("di_engine_b200: ScatterConnection index %d is out of range for a %d x %d map" %
                             (lo if lo < 0 else hi, H, W))
    mode = ops.SCATTER_MODES[scatter_type]
    out = torch_ops.scatter(x, row, col, H, W, mode)
    return out.cpu() if host_out else out


def _check_x(x):
    if x.dtype != torch.float32:
        raise TypeError("di_engine_b200: ScatterConnection's x must be float32 (got %s); the CUDA path computes in fp32" %
                        x.dtype)
    if x.dim() != 3:
        raise ValueError("di_engine_b200: ScatterConnection's x must be (B, M, N), got %s" % (tuple(x.shape), ))


def scatter_location(x: torch.Tensor, spatial_size: Tuple[int, int], location: torch.Tensor,
                     scatter_type: str) -> torch.Tensor:
    """``forward``'s map: location (B, M, 2) int64 holds (y, x); the flat index is x + y * W"""
    _check_x(x)
    _index(location, tuple(x.shape[:2]) + (2, ), 'location')
    return _scatter(x, spatial_size, location[..., 0], location[..., 1], scatter_type)


def scatter_xy(x: torch.Tensor, spatial_size: Tuple[int, int], coord_x: torch.Tensor, coord_y: torch.Tensor,
               scatter_type: str) -> torch.Tensor:
    """``xy_forward``'s map: coord_x, coord_y (B, M) int64; the flat index is coord_x * W + coord_y"""
    _check_x(x)
    _index(coord_x, tuple(x.shape[:2]), 'coord_x')
    _index(coord_y, tuple(x.shape[:2]), 'coord_y')
    return _scatter(x, spatial_size, coord_x, coord_y, scatter_type)


def scatter_forward(self, x: torch.Tensor, spatial_size: Tuple[int, int], location: torch.Tensor) -> torch.Tensor:
    """ScatterConnection.forward (scatter_connection.py:59-88): x (B, M, N) fp32, location (B, M, 2) int64 (y, x) ->
    (B, N, H, W).  ``install()`` also sets it on the reference class."""
    return scatter_location(x, spatial_size, location, self.scatter_type)


def scatter_xy_forward(self, x: torch.Tensor, spatial_size: Tuple[int, int], coord_x: torch.Tensor,
                       coord_y) -> torch.Tensor:
    """ScatterConnection.xy_forward (scatter_connection.py:90-121): int64 coord_x, coord_y (B, M) -> (B, N, H, W)"""
    return scatter_xy(x, spatial_size, coord_x, coord_y, self.scatter_type)


class ScatterConnection(nn.Module):
    """Scatter entity features into a spatial map, drop-in for ding.torch_utils.ScatterConnection.  ``scatter_type``
    decides what a cell holding several entities gets: 'add' their sum, 'cover' the last one."""

    def __init__(self, scatter_type: str) -> None:
        super(ScatterConnection, self).__init__()
        self.scatter_type = scatter_type
        assert self.scatter_type in ['cover', 'add']

    forward = scatter_forward
    xy_forward = scatter_xy_forward
