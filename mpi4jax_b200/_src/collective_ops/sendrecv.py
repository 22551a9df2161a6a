"""sendrecv -- simultaneous send to ``dest`` and receive from ``source``.

Reference: /root/reference/mpi4jax/_src/collective_ops/sendrecv.py:49-110 (signature;
``recvbuf`` is a template), :206-233 (vmap: both operands batched on the same axis),
:236-301 (reverse-mode works by swapping source and dest for the cotangent; pure
forward-mode raises, tested by tests/collective_ops/test_sendrecv.py:175-189).
GPU: ONE kernel, disjoint CTA groups push and receive concurrently, so the exchange is
deadlock-free for any message size (csrc/b2_p2p.cu).
"""

from __future__ import annotations

import numpy as np
import torch

from .. import collective_ops
from ..comm import ANY_TAG, PROC_NULL, Comm, Status
from ..utils import (NOTSET, as_tensor, carries_grad, check_dtype, check_rank, get_default_comm,
                     needs_autograd, raise_if_token_is_set)
from ..validation import enforce_types
from . import _adjoints, _dispatch


class _Sendrecv(torch.autograd.Function):
    @staticmethod
    def forward(sendbuf, recvbuf, source, dest, sendtag, recvtag, comm, status):
        return _dispatch.sendrecv(comm, sendbuf, recvbuf, source, dest, sendtag, recvtag, status)

    @staticmethod
    def setup_context(ctx, inputs, output):
        sendbuf, _, ctx.source, ctx.dest, ctx.sendtag, ctx.recvtag, ctx.comm, _ = inputs
        ctx.send_template = torch.empty_like(sendbuf)

    @staticmethod
    def backward(ctx, g):
        gs = _adjoints.sendrecv(collective_ops.eager, g, ctx.send_template, ctx.source, ctx.dest, ctx.sendtag,
                                ctx.recvtag, ctx.comm)
        return gs, None, None, None, None, None, None, None

    @staticmethod
    def jvp(ctx, *tangents):
        raise RuntimeError(
            "sendrecv cannot be used with forward-mode (vmap-of-jvp / jacfwd) differentiation: "
            "the tangent exchange would have to be transposed. Use reverse-mode (grad / jacrev)."
        )

    @staticmethod
    def vmap(info, in_dims, sendbuf, recvbuf, source, dest, sendtag, recvtag, comm, status):
        ds, dr = in_dims[0], in_dims[1]
        if ds is not None and dr is not None and ds != dr:
            raise ValueError("sendrecv under vmap needs sendbuf and recvbuf batched on the same axis")
        # an unbatched operand is broadcast along the batch axis of the other one (this is what
        # happens when the backward pass -- whose receive template is a constant -- is vmapped,
        # e.g. by jacrev); the whole batch travels as one message
        if ds is None and dr is not None:
            sendbuf = sendbuf.unsqueeze(dr).expand(
                *sendbuf.shape[:dr], info.batch_size, *sendbuf.shape[dr:]).contiguous()
            ds = dr
        elif dr is None and ds is not None:
            recvbuf = torch.empty(
                (*recvbuf.shape[:ds], info.batch_size, *recvbuf.shape[ds:]),
                dtype=recvbuf.dtype, device=recvbuf.device)
        out = _Sendrecv.apply(sendbuf, recvbuf, source, dest, sendtag, recvtag, comm, status)
        return out, ds


@enforce_types(
    source=(np.integer,), dest=(np.integer,), sendtag=(np.integer,), recvtag=(np.integer,),
    comm=(type(None), Comm), status=(type(None), Status),
)
def sendrecv(sendbuf, recvbuf, source, dest, *, sendtag=0, recvtag=ANY_TAG, comm=None,
             status=None, token=NOTSET):
    """Perform a sendrecv operation.

    Arguments:
        sendbuf: data to send to ``dest``.
        recvbuf: template (shape, dtype) of the data received from ``source``.
        source (int), dest (int): peer ranks.
        sendtag (int), recvtag (int): message tags.
        status: optional :class:`mpi4jax_b200.MPI.Status` to fill.

    Returns:
        Tensor: the received data.
    """
    raise_if_token_is_set(token)
    if comm is None:
        comm = get_default_comm()
    sendbuf = as_tensor(sendbuf, comm)
    recvbuf = as_tensor(recvbuf, comm)
    check_dtype(sendbuf)
    check_dtype(recvbuf)
    check_rank(int(dest), comm, "Sendrecv", "destination")
    check_rank(int(source), comm, "Sendrecv", "source", allow_any=True)
    if int(dest) == PROC_NULL or int(source) == PROC_NULL:
        # MPI: either half may address PROC_NULL; that half is a no-op (used at open boundaries)
        from .recv import recv as _recv
        from .send import send_with_grad as _send_grad
        from .send import send as _send

        if int(dest) != PROC_NULL:
            (_send_grad if carries_grad(sendbuf) else _send)(sendbuf, int(dest), tag=int(sendtag), comm=comm)
        if int(source) != PROC_NULL:
            return _recv(recvbuf, int(source), tag=int(recvtag), comm=comm, status=status)
        if status is not None:
            status._set_proc_null()
        return recvbuf
    if not needs_autograd(sendbuf, recvbuf):
        return _dispatch.sendrecv(comm, sendbuf, recvbuf, int(source), int(dest), int(sendtag),
                                  int(recvtag), status)
    return _Sendrecv.apply(sendbuf, recvbuf, int(source), int(dest), int(sendtag), int(recvtag),
                           comm, status)
