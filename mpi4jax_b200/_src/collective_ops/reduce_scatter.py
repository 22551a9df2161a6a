"""reduce_scatter -- rank r receives ``op`` over ranks q of ``x_q[r]``: ``(nproc, *S) -> S``.

MPI_Reduce_scatter_block with the leading-axis convention of ``alltoall``; the exact inverse shape
of ``allgather``.  Extension: the reference has no reduce-scatter.  GPU: the LL flag-in-data kernel
for small blocks, otherwise stage all blocks -> barrier -> pull block r from every peer and reduce
it in rank order (csrc/b2_reduce.cuh).  Differentiable for SUM: the adjoint is the allgather of the
cotangent, the derivative the reduce-scatter of the tangent.
"""

from __future__ import annotations

import torch

from .. import collective_ops
from ..comm import OP_TYPES, SUM, Comm, Op, as_op
from ..utils import (NOTSET, as_tensor, check_dtype, fold, get_default_comm, needs_autograd,
                     raise_if_token_is_set)
from ..validation import enforce_types
from ..native import codes
from . import _adjoints, _dispatch, _loc


def _require_sum(op: Op, what: str) -> None:
    if op is not SUM:
        raise NotImplementedError(f"The {what} of reduce_scatter for {op.name} is not defined")


class _ReduceScatter(torch.autograd.Function):
    @staticmethod
    def forward(x, op, comm):
        return _dispatch.reduce_scatter(comm, x, op.code)

    @staticmethod
    def setup_context(ctx, inputs, output):
        _, ctx.op, ctx.comm = inputs

    @staticmethod
    def backward(ctx, g):
        _require_sum(ctx.op, "adjoint")
        return _adjoints.reduce_scatter(collective_ops.eager, g, ctx.comm), None, None

    @staticmethod
    def jvp(ctx, x_t, *_):
        _require_sum(ctx.op, "derivative")
        return _ReduceScatter.apply(x_t, ctx.op, ctx.comm)

    @staticmethod
    def vmap(info, in_dims, x, op, comm):
        # keep the (nproc, ...) axis in front: (B, P, *S) -> (P, B, *S), reduced as one message -> (B, *S)
        return _ReduceScatter.apply(x.movedim(in_dims[0], 1).contiguous(), op, comm), 0


@enforce_types(op=OP_TYPES, comm=(type(None), Comm))
def reduce_scatter(x, op, *, comm=None, token=NOTSET):
    """Perform a reduce-scatter operation (``MPI_Reduce_scatter_block``).

    Arguments:
        x: input of shape ``(nproc, ...)``; block ``q`` is this rank's contribution to rank ``q``.
        op: the reduction operator (e.g. ``mpi4jax_b200.MPI.SUM``).
        comm: the communicator (defaults to a clone of ``COMM_WORLD``).

    Returns:
        Tensor: ``op`` over all ranks of their block ``rank``, shape ``x.shape[1:]``, dtype of ``x``.  With
        ``MPI.MAXLOC`` / ``MPI.MINLOC``, ``x`` is a pair ``(values, indices)`` of shape ``(nproc, ...)`` and the
        result is the pair of this rank's blocks (see ``allreduce``).
    """
    raise_if_token_is_set(token)
    if comm is None:
        comm = get_default_comm()
    op = as_op(op)
    if _loc.is_loc(op):
        return _loc.reduce_loc("reduce_scatter", codes.OPC_REDUCE_SCATTER, x, op, comm)
    x = as_tensor(x, comm)
    check_dtype(x)
    if x.dim() == 0 or x.shape[0] != comm.Get_size():
        raise ValueError("Reduce_scatter input must have shape (nproc, ...)")
    if op.code is None:                      # MPI.Op.Create: exchange the blocks natively, fold on the device
        if needs_autograd(x):
            raise NotImplementedError(f"The derivative of reduce_scatter for {op.name} is not defined")
        return fold(list(_dispatch.alltoall(comm, x.contiguous()).unbind(0)), op)
    if not needs_autograd(x):
        return _dispatch.reduce_scatter(comm, x, op.code)
    return _ReduceScatter.apply(x, op, comm)
