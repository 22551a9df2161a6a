"""alltoall -- rank r sends ``x[q]`` to rank q and receives ``out[q] = x_q[r]``.

Reference: /root/reference/mpi4jax/_src/collective_ops/alltoall.py:43-67 (shape check and
its error text).  GPU: stage -> barrier -> pull, writing directly into the final layout.
Extension: differentiable (the adjoint of an all-to-all is the all-to-all of the cotangent).
"""

from __future__ import annotations

import torch

from .. import collective_ops
from ..comm import Comm
from ..utils import (NOTSET, as_tensor, check_dtype, get_default_comm, needs_autograd,
                     raise_if_token_is_set)
from ..validation import enforce_types
from . import _adjoints, _dispatch


class _Alltoall(torch.autograd.Function):
    @staticmethod
    def forward(x, comm):
        return _dispatch.alltoall(comm, x)

    @staticmethod
    def setup_context(ctx, inputs, output):
        ctx.comm = inputs[1]

    @staticmethod
    def backward(ctx, g):
        return _adjoints.alltoall(collective_ops.eager, g, ctx.comm), None

    @staticmethod
    def vmap(info, in_dims, x, comm):
        # keep the (nproc, ...) axis in front: (B, P, *S) -> (P, B, *S), exchanged as one message
        return _Alltoall.apply(x.movedim(in_dims[0], 1).contiguous(), comm), 1


@enforce_types(comm=(type(None), Comm))
def alltoall(x, *, comm=None, token=NOTSET):
    """Perform an alltoall operation.

    Arguments:
        x: input of shape ``(nproc, ...)``.

    Returns:
        Tensor: received data, same shape as ``x``.
    """
    raise_if_token_is_set(token)
    if comm is None:
        comm = get_default_comm()
    x = as_tensor(x, comm)
    check_dtype(x)
    if x.dim() == 0 or x.shape[0] != comm.Get_size():
        raise ValueError("Alltoall input must have shape (nproc, ...)")
    if not needs_autograd(x):
        return _dispatch.alltoall(comm, x)
    return _Alltoall.apply(x, comm)
