"""bcast -- the root's ``x`` is delivered to every rank.

Reference: /root/reference/mpi4jax/_src/collective_ops/bcast.py:44-75: on the root the
*input itself* is returned; elsewhere ``x`` only provides shape and dtype.
Extension (BASELINE north star): differentiable.  The adjoint of a broadcast is a
reduce-to-root: the root's input gradient is the SUM of all ranks' output cotangents,
non-root inputs (templates) get zero gradient.
"""

from __future__ import annotations

import numpy as np
import torch

from .. import collective_ops
from ..comm import Comm
from ..utils import (NOTSET, as_tensor, check_dtype, get_default_comm, needs_autograd,
                     raise_if_token_is_set)
from ..validation import enforce_types
from . import _adjoints, _dispatch


class _Bcast(torch.autograd.Function):
    @staticmethod
    def forward(x, root, comm):
        out = _dispatch.bcast(comm, x, root)
        return x.view_as(x) if comm.rank == root else out

    @staticmethod
    def setup_context(ctx, inputs, output):
        _, ctx.root, ctx.comm = inputs

    @staticmethod
    def backward(ctx, g):
        return _adjoints.bcast(collective_ops.eager, g, ctx.root, ctx.comm), None, None

    @staticmethod
    def vmap(info, in_dims, x, root, comm):
        return _Bcast.apply(x, root, comm), in_dims[0]


@enforce_types(root=(np.integer,), comm=(type(None), Comm))
def bcast(x, root, *, comm=None, token=NOTSET):
    """Perform a bcast (broadcast) operation.

    Arguments:
        x: data (read on the root only; elsewhere a shape/dtype template).
        root (int): the source rank.

    Returns:
        Tensor: the root's data (on the root: ``x`` itself).
    """
    raise_if_token_is_set(token)
    if comm is None:
        comm = get_default_comm()
    x = as_tensor(x, comm)
    check_dtype(x)
    _check_root(root, comm, "Bcast")
    if not needs_autograd(x):
        out = _dispatch.bcast(comm, x, int(root))
        return x if comm.Get_rank() == root else out
    return _Bcast.apply(x, int(root), comm)


def _check_root(root, comm, opname):
    if not 0 <= int(root) < comm.Get_size():
        from ..backends.cuda import abort_or_raise

        abort_or_raise(
            f"r{comm.Get_rank()} | MPI_{opname} returned error code 4: invalid root rank "
            f"{int(root)} (communicator size {comm.Get_size()}) - aborting", 4)
