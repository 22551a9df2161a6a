"""See package docstring."""

from __future__ import annotations

from typing import Iterable, NamedTuple, Optional

import numpy as np
import torch

from .. import _src as ops
from .._src.collective_ops.alltoallv import alltoallv_reverse
from .._src.comm import SUM, Comm
from .._src.native import codes
from .._src.utils import get_default_comm


def broadcast_parameters(params: Iterable[torch.Tensor], root: int = 0, comm: Optional[Comm] = None):
    """In-place parameter sync from ``root`` (data-parallel initialisation)."""
    comm = comm or get_default_comm()
    with torch.no_grad():
        for p in params:
            p.copy_(ops.bcast(p.detach(), root, comm=comm))


def average_gradients(params: Iterable[torch.Tensor], comm: Optional[Comm] = None) -> None:
    """All-reduce ``p.grad`` over the ranks and divide by the world size."""
    comm = comm or get_default_comm()
    n = comm.Get_size()
    for p in params:
        if p.grad is not None:
            p.grad = ops.allreduce(p.grad, SUM, comm=comm) / n


def column_parallel_matvec(a_cols: torch.Tensor, x_shard: torch.Tensor, comm: Optional[Comm] = None):
    """``A @ x`` with A column-sharded and x row-sharded: local product + allreduce."""
    return ops.allreduce(a_cols @ x_shard, SUM, comm=comm or get_default_comm())


def row_parallel_matvec(a_cols: torch.Tensor, y: torch.Tensor):
    """``A.T @ y`` for the same sharding: purely local (the transpose of the allreduce is the
    identity, cf. allreduce's VJP)."""
    return a_cols.transpose(-1, -2) @ y


def ring_shift(x: torch.Tensor, shift: int = 1, comm: Optional[Comm] = None) -> torch.Tensor:
    """Send ``x`` to rank+shift, receive from rank-shift (differentiable)."""
    comm = comm or get_default_comm()
    r, n = comm.Get_rank(), comm.Get_size()
    return ops.sendrecv(x, x, source=(r - shift) % n, dest=(r + shift) % n, comm=comm)


def alltoall_reshard(x: torch.Tensor, scatter_dim: int, gather_dim: int,
                     comm: Optional[Comm] = None) -> torch.Tensor:
    """Re-shard a tensor that is split over ranks along ``gather_dim`` so that it becomes
    split along ``scatter_dim`` (Ulysses attention: sequence-sharded <-> head-sharded)."""
    comm = comm or get_default_comm()
    n = comm.Get_size()
    if x.shape[scatter_dim] % n:
        raise ValueError("scatter_dim must be divisible by the number of ranks")
    parts = torch.stack(torch.chunk(x, n, dim=scatter_dim), dim=0)      # (n, ...)
    recv = ops.alltoall(parts, comm=comm)                               # recv[q] = peer q's chunk
    return torch.cat(list(recv.unbind(0)), dim=gather_dim)


class ExpertPlan(NamedTuple):
    """What :func:`expert_combine` needs to undo an :func:`expert_dispatch` (all on the device)."""

    order: torch.Tensor          # (N,) token index of each sorted row
    send_counts: torch.Tensor    # (nproc,) int64 tokens sent to each rank
    recv_counts: torch.Tensor    # (nproc,) int64 rows received from each rank
    comm: Comm


def expert_dispatch(x: torch.Tensor, dest_rank: torch.Tensor, capacity: Optional[int] = None,
                    comm: Optional[Comm] = None):
    """Send every token (row of ``x``) to the rank ``dest_rank`` names -- the dispatch of an
    expert-parallel mixture-of-experts layer.  Returns ``(rows, recv_counts, plan)``: the received
    tokens packed by source rank in a ``(capacity, ...)`` tensor (default capacity ``N * nproc``),
    the rows received from each rank, and the plan :func:`expert_combine` uses to bring results back.
    Tokens that do not fit the receiver's capacity are dropped, as are tokens whose destination is not
    a rank.  Differentiable; the counts never leave the device (no host synchronisation)."""
    comm = comm or get_default_comm()
    n = comm.Get_size()
    if dest_rank.shape != x.shape[:1]:
        raise ValueError(f"expert_dispatch: dest_rank must have shape ({x.shape[0]},) (got {tuple(dest_rank.shape)})")
    # invalid destinations sort last and are counted for no rank, so they are never sent
    key = torch.where((dest_rank >= 0) & (dest_rank < n), dest_rank, n).to(torch.int64)
    order = torch.argsort(key, stable=True)
    # counts from the sorted keys: torch.bincount would read its maximum back to the host
    bounds = torch.searchsorted(key[order], torch.arange(n + 1, device=key.device))
    send_counts = bounds.diff()
    # float8 tokens are gathered as their bytes: torch's index kernels do not all take float8
    picked = x.view(torch.uint8)[order].view(x.dtype) if x.dtype in codes.FP8_DTYPE_CODE else x[order]
    rows, recv_counts = ops.alltoallv(picked, send_counts, recv_capacity=capacity, comm=comm)
    return rows, recv_counts, ExpertPlan(order, send_counts, recv_counts, comm)


def expert_combine(y: torch.Tensor, plan: ExpertPlan) -> torch.Tensor:
    """Return the rows of ``y`` (laid out like :func:`expert_dispatch`'s output, e.g. the experts'
    results) to the ranks and token positions they came from.  Dropped tokens come back as zeros.
    Differentiable; no host synchronisation."""
    back = alltoallv_reverse(y, plan.recv_counts, plan.send_counts, plan.order.shape[0], plan.comm)
    return torch.zeros_like(back).index_copy(0, plan.order, back)


def pipeline_send(x: torch.Tensor, dest: int, tag: int = 0, comm: Optional[Comm] = None):
    """Stage boundary (sender side); back-propagate through the returned token."""
    return ops.send_with_grad(x, dest, tag=tag, comm=comm)


def pipeline_recv(template: torch.Tensor, source: int, tag: int = 0, comm: Optional[Comm] = None):
    """Stage boundary (receiver side); differentiable w.r.t. the sender's tensor."""
    if not template.requires_grad:
        template = template.detach().requires_grad_(True)
    return ops.recv(template, source, tag=tag, comm=comm)


def cartesian_neighbors(rank: int, nproc_y: int, nproc_x: int, periodic_x: bool = True) -> dict:
    """Neighbour ranks of ``rank`` in a (nproc_y, nproc_x) process grid (None = wall)."""
    py, px = np.unravel_index(rank, (nproc_y, nproc_x))
    flat = lambda iy, ix: int(np.ravel_multi_index((iy, ix), (nproc_y, nproc_x)))  # noqa: E731
    return {
        "south": flat(py - 1, px) if py > 0 else None,
        "north": flat(py + 1, px) if py < nproc_y - 1 else None,
        "west": flat(py, (px - 1) % nproc_x) if (px > 0 or periodic_x) else None,
        "east": flat(py, (px + 1) % nproc_x) if (px < nproc_x - 1 or periodic_x) else None,
    }
