"""reduce_scatterv -- a variable-count reduce-scatter whose counts stay on the device.

``MPI_Reduce_scatter`` (the variant with counts) for rows whose number is known only on the GPU: every
rank holds one segment of rows for each rank, and rank r receives ``op`` over the ranks' segments for r,
folded row by row.  The counts are device tensors, so the host never waits for them and the call can be
captured into a CUDA graph and replayed with other counts.  It is ``allgatherv``'s adjoint.  Extension:
the reference has no reduce-scatter.

Rules, on rank r of P (``x_r`` has shape ``(M_r, *S)``; ``M_r`` may differ between ranks, ``S`` and the
dtype may not; the capacity ``N`` must be the same on every rank):

* sent: ``s_r[p] = clamp(M_r - sum_{p'<p} s_r[p'], 0, max(send_counts_r[p], 0))`` rows, starting at row
  ``D_r(p) = sum_{p'<p} s_r[p']``, go to rank p;
* received: ``c[q] = min(s_q[r], N)`` rows from rank q.  For ``i < max_q c[q]``, ``out_r[i]`` is ``op``
  folded in rank order over the ranks q with ``i < c[q]``, applied to ``x_q[D_q(r) + i]``; rows
  ``[max_q c[q], N)`` are zero.  ``recv_counts`` = ``c`` (int64, on x's device).

Folding is reduce_scatter's: rank order, f16/bf16 accumulated in fp32 and rounded once, integers
wrapping.  An invalid count is never an error and never makes the kernel read or write out of bounds.

GPU: every rank stages, per destination, the rows it sends behind a header of its clamped counts; after
one barrier each CTA reads all headers and folds its chunks of every peer's block for this rank straight
into the output (csrc/b2_reduce.cuh: b2_k_reduce_scatterv).  Differentiable for SUM: the adjoint is the
reverse mode of allgatherv, the derivative the reduce_scatterv of the tangent.
"""

from __future__ import annotations

import numpy as np
import torch

from .. import collective_ops
from ..comm import OP_TYPES, SUM, Comm, Op, as_op
from ..utils import (NOTSET, as_tensor, check_dtype, get_default_comm, needs_autograd,
                     raise_if_token_is_set)
from ..validation import enforce_types
from . import _adjoints, _dispatch, _loc
from ._rowsv import RowsvFunction


def _require_sum(op: Op, what: str) -> None:
    if op is not SUM:
        raise NotImplementedError(f"The {what} of reduce_scatterv for {op.name} is not defined")


class _ReduceScatterv(RowsvFunction):
    vmap_error = "reduce_scatterv under vmap: the counts must not be batched (one exchange moves every batch entry)"

    @staticmethod
    def forward(x, send_counts, out_rows, op, comm):
        return _dispatch.reduce_scatterv(comm, x, send_counts, out_rows, op.code)

    @staticmethod
    def backward(ctx, g, _g_counts):
        send_counts, _, op, comm = ctx.args
        _require_sum(op, "adjoint")
        back = _adjoints.reduce_scatterv(collective_ops.eager, g, comm, ctx.in_rows, send_counts)
        return back, None, None, None, None

    @classmethod
    def jvp(cls, ctx, x_t, *_):
        _require_sum(ctx.args[2], "derivative")
        return super().jvp(ctx, x_t)


def _user_op(comm: Comm, x: torch.Tensor, send_counts: torch.Tensor, out_rows: int, op: Op):
    """``MPI.Op.Create``: the segments, clipped to ``out_rows`` and zero-padded to ``(P, out_rows, *S)``,
    are exchanged by the native all-to-all, the clipped counts with them; then each row is folded on the
    device in rank order over the ranks whose segment reaches it.  Device ops only."""
    P, M = comm.Get_size(), x.shape[0]
    s = send_counts.to(torch.int64).clamp(min=0)
    total = torch.cumsum(s, 0)
    start, end = (total - s).clamp(max=M), total.clamp(max=M)      # clamped in rank order to the M rows
    sent = torch.clamp(end - start, max=out_rows)
    i = torch.arange(out_rows, device=x.device)
    # entries past a segment read a zero row appended to x (index M)
    idx = torch.where(i < sent.view(P, 1), start.view(P, 1) + i, M)
    blocks = torch.cat([x, x.new_zeros((1, *x.shape[1:]))])[idx]
    got = _dispatch.alltoall(comm, blocks.contiguous())
    recv = _dispatch.alltoall(comm, sent.contiguous())
    out = x.new_zeros((out_rows, *x.shape[1:]))
    row = i.view(out_rows, *([1] * (x.dim() - 1)))
    covered = torch.zeros((), dtype=torch.int64, device=x.device)
    for q in range(P):
        part = got[q]
        folded = op.function(out, part)
        if not isinstance(folded, torch.Tensor) or folded.shape != out.shape:
            raise TypeError("a user-defined reduction must return a tensor of its operands' shape")
        step = torch.where(row < covered, folded.to(out.dtype), part)
        out = torch.where(row < recv[q], step, out)
        covered = torch.maximum(covered, recv[q])
    return out, recv


@enforce_types(op=OP_TYPES, recv_capacity=(type(None), np.integer), comm=(type(None), Comm))
def reduce_scatterv(x, send_counts, op, *, recv_capacity=None, comm=None, token=NOTSET):
    """Perform a variable-count reduce-scatter operation (``MPI_Reduce_scatter``) with device-resident counts.

    Arguments:
        x: input of shape ``(M, ...)``, rows grouped by destination rank; the row shape and the dtype
            must be the same on every rank, ``M`` may differ.
        send_counts: integer tensor of shape ``(nproc,)`` on ``x``'s device (or a sequence of ints):
            rows for each rank, taken in rank order from the start of ``x``.  Negative counts send
            nothing, counts past the end of ``x`` are cut at its last row.
        op: the reduction operator (e.g. ``mpi4jax_b200.MPI.SUM``).
        recv_capacity: rows of the output, ``N`` (default ``M``).  It must be the same on every rank.
            Only the first ``N`` rows of a segment take part.
        comm: the communicator (defaults to a clone of ``COMM_WORLD``).

    Returns:
        Tuple[Tensor, Tensor]: shape ``(recv_capacity, ...)``: row ``i`` is ``op`` over the ranks whose
        segment for this rank has more than ``i`` rows, folded in rank order, and rows past the longest
        segment are zero; and ``recv_counts``, int64 ``(nproc,)`` on the device: the rows folded from
        each rank.
    """
    raise_if_token_is_set(token)
    if comm is None:
        comm = get_default_comm()
    op = as_op(op)
    _loc.refuse(op, "reduce_scatterv")
    x = as_tensor(x, comm)
    check_dtype(x)
    _dispatch.check_rows("Reduce_scatterv", x)
    send_counts = _dispatch.as_counts(send_counts, x)
    cap = int(_dispatch.rowsv_capacity("Reduce_scatterv", comm, x, send_counts, recv_capacity, "send_counts", 1))
    if op.code is None:
        if needs_autograd(x):
            raise NotImplementedError(f"The derivative of reduce_scatterv for {op.name} is not defined")
        return _user_op(comm, x.contiguous(), send_counts, cap, op)
    return _ReduceScatterv.run(x, send_counts, cap, op, comm)
