"""allgather -- every rank receives every rank's ``x``: ``S -> (nproc, *S)``.

Reference: /root/reference/mpi4jax/_src/collective_ops/allgather.py:43-60, 124-128.
GPU: stage -> barrier -> pull straight into the (nproc, *S) layout (csrc/b2_collectives.cu).
Extension: differentiable (adjoint = sum over ranks of the matching output slice, i.e. a
reduce-scatter, realised as allreduce + slice); the reference registers no AD rule.
"""

from __future__ import annotations

import torch

from .. import collective_ops
from ..comm import Comm
from ..utils import (NOTSET, as_tensor, check_dtype, get_default_comm, needs_autograd,
                     raise_if_token_is_set)
from ..validation import enforce_types
from . import _adjoints, _dispatch


class _Allgather(torch.autograd.Function):
    @staticmethod
    def forward(x, comm):
        return _dispatch.allgather(comm, x)

    @staticmethod
    def setup_context(ctx, inputs, output):
        ctx.comm = inputs[1]

    @staticmethod
    def backward(ctx, g):
        return _adjoints.allgather(collective_ops.eager, g, ctx.comm), None

    @staticmethod
    def vmap(info, in_dims, x, comm):
        # (B, *S) on every rank -> one message -> (P, B, *S): the batch axis ends up at position 1
        return _Allgather.apply(x.movedim(in_dims[0], 0).contiguous(), comm), 1


@enforce_types(comm=(type(None), Comm))
def allgather(x, *, comm=None, token=NOTSET):
    """Perform an allgather operation.

    All ranks must pass inputs of the same shape and dtype.

    Returns:
        Tensor: received data of shape ``(nproc, *x.shape)``.
    """
    raise_if_token_is_set(token)
    if comm is None:
        comm = get_default_comm()
    x = as_tensor(x, comm)
    check_dtype(x)
    if not needs_autograd(x):
        return _dispatch.allgather(comm, x)
    return _Allgather.apply(x, comm)
