"""scan -- inclusive prefix reduction over ranks: rank r gets ``op(x_0, ..., x_r)``.

Reference: /root/reference/mpi4jax/_src/collective_ops/scan.py:44-60, 113-114.
GPU: stage -> barrier -> rank r pulls the staged copies of ranks 0..r through the fused
reduce kernel (P <= 8 inside an NVLink domain, so O(P) direct reads beat a log-step chain).
Extension: differentiable for SUM -- rank r's input reaches the outputs of ranks r .. P-1, so its
gradient is the SUFFIX sum of the cotangents: total - inclusive prefix + own.  The reference
defines no rule and raises.
"""

from __future__ import annotations

import torch

from ..comm import OP_TYPES, SUM, Comm, Op, as_op
from ..native import codes
from ..utils import (NOTSET, as_tensor, check_dtype, fold, get_default_comm, needs_autograd,
                     raise_if_token_is_set)
from ..validation import enforce_types
from . import _dispatch, _loc


class _Scan(torch.autograd.Function):
    @staticmethod
    def forward(x, comm):
        return _dispatch.scan(comm, x, SUM.code)

    @staticmethod
    def setup_context(ctx, inputs, output):
        _, ctx.comm = inputs

    @staticmethod
    def backward(ctx, g):
        comm = ctx.comm

        def suffix(t):
            total = _dispatch.allreduce(comm, t, SUM.code, codes.ALGO_AUTO)
            return total - _dispatch.scan(comm, t, SUM.code) + t

        return _dispatch.run_opaque(suffix, g.contiguous()), None

    @staticmethod
    def vmap(info, in_dims, x, comm):
        return _Scan.apply(x, comm), in_dims[0]


@enforce_types(op=OP_TYPES, comm=(type(None), Comm))
def scan(x, op, *, comm=None, token=NOTSET):
    """Perform a scan operation (inclusive prefix reduction over the ranks).  With ``MPI.MAXLOC`` /
    ``MPI.MINLOC``, ``x`` and the result are ``(values, indices)`` pairs (see ``allreduce``)."""
    raise_if_token_is_set(token)
    if comm is None:
        comm = get_default_comm()
    op = as_op(op)
    if _loc.is_loc(op):
        return _loc.reduce_loc("scan", codes.OPC_SCAN, x, op, comm)
    x = as_tensor(x, comm)
    check_dtype(x)
    if op.code is None:                      # MPI.Op.Create: gather natively, fold ranks 0 .. r
        if needs_autograd(x):
            raise NotImplementedError(f"The derivative of scan for {op.name} is not defined")
        parts = _dispatch.allgather(comm, x.contiguous())
        return fold(list(parts[: comm.Get_rank() + 1].unbind(0)), op)
    if needs_autograd(x):
        if op is not SUM:
            raise NotImplementedError(f"The derivative of scan for {op.name} is not defined")
        return _Scan.apply(x, comm)
    return _dispatch.scan(comm, x, op.code)
