"""allreduce -- reduce ``x`` over all ranks, result on every rank.

API and semantics: /root/reference/mpi4jax/_src/collective_ops/allreduce.py:41-70
(signature, returns ONE array), :132-135 (vmap = pass-through), :138-149 (JVP =
allreduce of the tangent, SUM only), :152-159 + :78-80 (transpose = identity on the
local cotangent; transposing twice gives an allreduce again).  GPU implementation:
fused LL / one-shot / two-shot / NVLS kernels (csrc/b2_reduce.cuh, b2_collectives.cu).
"""

from __future__ import annotations

import torch

from ..comm import OP_TYPES, SUM, Comm, Op, as_op
from ..native import codes
from ..utils import (NOTSET, as_tensor, check_dtype, fold, get_default_comm, needs_autograd,
                     raise_if_token_is_set)
from ..validation import enforce_types
from . import _dispatch, _loc


def _require_sum(op: Op, what: str) -> None:
    if op is not SUM:
        raise NotImplementedError(f"The {what} of allreduce for {op.name} is not defined")


class _Allreduce(torch.autograd.Function):
    """``transpose=False``: the collective.  ``transpose=True``: its linear transpose, the
    identity on the local cotangent (every rank's output depends on every rank's input with
    unit weight, and cotangents are rank-local)."""

    @staticmethod
    def forward(x, op, comm, transpose, algo):
        if transpose:
            return x.view_as(x)
        return _dispatch.allreduce(comm, x, op.code, algo)

    @staticmethod
    def setup_context(ctx, inputs, output):
        _, ctx.op, ctx.comm, ctx.transpose, ctx.algo = inputs

    @staticmethod
    def backward(ctx, g):
        _require_sum(ctx.op, "adjoint")
        return _Allreduce.apply(g, ctx.op, ctx.comm, not ctx.transpose, ctx.algo), None, None, None, None

    @staticmethod
    def jvp(ctx, x_t, *_):
        _require_sum(ctx.op, "derivative")
        return _Allreduce.apply(x_t, ctx.op, ctx.comm, ctx.transpose, ctx.algo)

    @staticmethod
    def vmap(info, in_dims, x, op, comm, transpose, algo):
        # elementwise over ranks: the batched array is reduced as one message
        return _Allreduce.apply(x, op, comm, transpose, algo), in_dims[0]


@enforce_types(op=OP_TYPES, comm=(type(None), Comm))
def allreduce(x, op, *, comm=None, token=NOTSET, algorithm="auto"):
    """Perform an allreduce operation.

    Arguments:
        x: tensor, array or scalar input; with ``MPI.MAXLOC`` / ``MPI.MINLOC`` a pair
            ``(values, indices)`` (see below).
        op: the reduction operator (e.g. ``mpi4jax_b200.MPI.SUM``).
        comm: the communicator (defaults to a clone of ``COMM_WORLD``).
        algorithm: GPU transport -- ``"auto"`` (size table), ``"ll"``, ``"oneshot"``,
            ``"twoshot"`` or ``"nvls"`` (extension; the reference has a single MPI path).

    Returns:
        Tensor: result of the allreduce (same shape and dtype as ``x``).

    With ``op=MPI.MAXLOC`` or ``MPI.MINLOC``, ``x`` is a pair ``(values, indices)`` of one shape (values
    float16, bfloat16, float32, float64, int16, int32 or int64; indices int32 or int64; elements may be
    Python scalars) and the result is the pair ``(values, indices)`` of the extreme value over the ranks and
    its index, elementwise: ties go to the smaller index, NaN wins (``collective_ops/_loc.py``).  Not
    differentiable.
    """
    raise_if_token_is_set(token)
    if comm is None:
        comm = get_default_comm()
    op = as_op(op)
    if _loc.is_loc(op):
        return _loc.reduce_loc("allreduce", codes.OPC_ALLREDUCE, x, op, comm, algorithm=algorithm)
    x = as_tensor(x, comm)
    check_dtype(x)
    algo = codes.ALGO_BY_NAME[algorithm]
    if op.code is None:                      # MPI.Op.Create: gather natively, fold on the device
        if needs_autograd(x):
            raise NotImplementedError(f"The derivative of allreduce for {op.name} is not defined")
        return fold(list(_dispatch.allgather(comm, x.contiguous()).unbind(0)), op)
    if not needs_autograd(x):
        return _dispatch.allreduce(comm, x, op.code, algo)
    return _Allreduce.apply(x, op, comm, False, algo)
