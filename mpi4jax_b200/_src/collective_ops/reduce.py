"""reduce -- the root receives the reduction of all ranks' ``x``.

Reference: /root/reference/mpi4jax/_src/collective_ops/reduce.py:45-71: non-root ranks get
their *input* back.  GPU: stage -> barrier -> root pulls P copies through the fused
reduce kernel (op + dtype cast in registers).
Extension: differentiable for SUM.  The adjoint of a reduce-to-root is a broadcast from the
root (the pair of bcast's rule); a non-root rank's result IS its input, so its own cotangent
passes through as well.  The reference defines no rule and raises.
"""

from __future__ import annotations

import numpy as np

import torch

from ..comm import OP_TYPES, SUM, Comm, Op, as_op
from ..utils import (NOTSET, as_tensor, check_dtype, fold, get_default_comm, needs_autograd,
                     raise_if_token_is_set)
from ..validation import enforce_types
from ..native import codes
from . import _dispatch, _loc
from .bcast import _check_root


class _Reduce(torch.autograd.Function):
    @staticmethod
    def forward(x, root, comm):
        res = _dispatch.reduce(comm, x, SUM.code, root)
        return res if comm.rank == root else x.view_as(x)

    @staticmethod
    def setup_context(ctx, inputs, output):
        _, ctx.root, ctx.comm = inputs

    @staticmethod
    def backward(ctx, g):
        comm, root = ctx.comm, ctx.root
        from_root = _dispatch.run_opaque(lambda t: _dispatch.bcast(comm, t, root), g.contiguous())
        return (from_root if comm.rank == root else from_root + g), None, None

    @staticmethod
    def vmap(info, in_dims, x, root, comm):
        return _Reduce.apply(x, root, comm), in_dims[0]


@enforce_types(op=OP_TYPES, root=(np.integer,), comm=(type(None), Comm))
def reduce(x, op, root, *, comm=None, token=NOTSET):
    """Perform a reduce operation.

    Returns:
        Tensor: on the root the reduced data; on every other rank the input ``x``.  With ``MPI.MAXLOC`` /
        ``MPI.MINLOC``, ``x`` and the result are ``(values, indices)`` pairs (see ``allreduce``).
    """
    raise_if_token_is_set(token)
    if comm is None:
        comm = get_default_comm()
    op = as_op(op)
    if _loc.is_loc(op):
        _check_root(root, comm, "Reduce")
        return _loc.reduce_loc("reduce", codes.OPC_REDUCE, x, op, comm, int(root))
    x = as_tensor(x, comm)
    check_dtype(x)
    _check_root(root, comm, "Reduce")
    if op.code is None:                      # MPI.Op.Create: gather natively, fold on the root
        if needs_autograd(x):
            raise NotImplementedError(f"The derivative of reduce for {op.name} is not defined")
        parts = _dispatch.gather(comm, x.contiguous(), int(root))
        return fold(list(parts.unbind(0)), op) if comm.Get_rank() == root else x
    if needs_autograd(x):
        if op is not SUM:
            raise NotImplementedError(f"The derivative of reduce for {op.name} is not defined")
        return _Reduce.apply(x, int(root), comm)
    res = _dispatch.reduce(comm, x, op.code, int(root))
    return res if comm.Get_rank() == root else x
