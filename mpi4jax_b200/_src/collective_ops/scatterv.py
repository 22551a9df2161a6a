"""scatterv -- a variable-count scatter whose counts stay on the device.

``MPI_Scatterv`` for rows whose number is known only on the GPU (work items or sequences sized on the
device): the root hands every rank a variable-length slice of one buffer, received into an output of
static capacity.  The counts are a device tensor, so the host never waits for them and the call can be
captured into a CUDA graph and replayed with other counts.  Extension: the reference has no scatterv.

Rules, on rank r of P (the root's ``x`` has shape ``(N, *S)``; on the other ranks ``x`` is a template of
the same shape and dtype whose values are not read; the capacity ``C_r`` may differ between ranks):

* the root's send counts are clamped in rank order to the ``N`` rows that exist:
  ``s'[q] = clamp(s[q], 0, N - sum_{p<q} s'[p])``; rank q's segment starts at ``d_q = sum_{p<q} s'[p]``;
* received: rows ``[0, k_r)`` of the output are root rows ``[d_r, d_r + k_r)`` with
  ``k_r = min(s'[r], C_r)``; the other rows are zero.  ``recv_count`` = ``k_r`` (int64 ``()``, on x's
  device).

An invalid count is never an error and never makes the kernel read or write out of bounds.

GPU: alltoallv's kernel in rooted mode (csrc/b2_collectives.cu: b2_k_rowsv): the root stages its rows
behind a header of its clamped counts, the other ranks stage nothing; after one barrier each CTA reads
the root's P counts and every rank pulls its chunks of its one segment straight into the output.
Differentiable: the adjoint is the reverse mode of ``gatherv`` -- each rank's first ``k_r`` cotangent rows
land on the root where they were taken from, and the templates get a zero gradient.
"""

from __future__ import annotations

import numpy as np
import torch

from .. import collective_ops
from ..comm import Comm
from ..utils import NOTSET, as_tensor, check_dtype, get_default_comm, raise_if_token_is_set
from ..validation import enforce_types
from . import _adjoints, _dispatch
from ._rowsv import RowsvFunction
from .bcast import _check_root


class _Scatterv(RowsvFunction):
    """``max_rows``: the root rows that may be sent, the same on every rank (it sizes the staging)."""

    vmap_error = "scatterv under vmap: the counts must not be batched (one exchange moves every batch entry)"

    @staticmethod
    def forward(x, send_counts, root, out_rows, max_rows, comm):
        return _dispatch.scatterv(comm, x, send_counts, root, out_rows, max_rows)

    @staticmethod
    def backward(ctx, g, _g_count):
        send_counts, root, _, max_rows, comm = ctx.args
        (recv_count,) = ctx.saved_tensors
        back = _adjoints.scatterv(collective_ops.eager, g, comm, root, ctx.in_rows, max_rows, recv_count, send_counts)
        return back, None, None, None, None, None


@enforce_types(root=(np.integer,), recv_capacity=(type(None), np.integer), comm=(type(None), Comm))
def scatterv(x, send_counts, root, *, recv_capacity=None, comm=None, token=NOTSET):
    """Perform a variable-count scatter operation (``MPI_Scatterv``) with device-resident counts.

    Arguments:
        x: on the root the rows to hand out, shape ``(N, ...)``; on every other rank a template of the same
            shape and dtype (``torch.empty`` will do: it is not read).
        send_counts: on the root an integer tensor of shape ``(nproc,)`` on ``x``'s device (or a sequence
            of ints): rows for each rank, taken in rank order from the start of ``x``.  Negative counts
            send nothing, counts past the end of ``x`` are cut at its last row.  Other ranks may pass
            None; a tensor passed there is checked but not read.
        root (int): the rank that sends.
        recv_capacity: rows of this rank's output (default ``N``, which never drops a row; may differ
            between ranks).  A segment that does not fit loses its last rows.
        comm: the communicator (defaults to a clone of ``COMM_WORLD``).

    Returns:
        Tuple[Tensor, Tensor]: this rank's rows, shape ``(recv_capacity, ...)``, zero past the segment, and
        ``recv_count``, int64 ``()`` on the device: the rows written.
    """
    raise_if_token_is_set(token)
    if comm is None:
        comm = get_default_comm()
    x = as_tensor(x, comm)
    check_dtype(x)
    _check_root(root, comm, "Scatterv")
    root = int(root)
    _dispatch.check_rows("Scatterv", x)
    if send_counts is not None:
        send_counts = _dispatch.as_counts(send_counts, x)
    cap = int(_dispatch.scatterv_capacity(comm, x, send_counts, root, recv_capacity))
    return _Scatterv.run(x, send_counts, root, cap, x.shape[0], comm)


def scatterv_bounded(x: torch.Tensor, send_counts, root: int, rows: int, max_rows: int, comm: Comm) -> torch.Tensor:
    """gatherv's adjoint: ``scatterv`` into ``rows`` rows with the staging bound ``max_rows``, which every rank
    knows even where the root's ``x`` has rows the others do not know of.  Differentiable (the adjoint is
    gatherv's reverse mode)."""
    if comm.Get_rank() == root:
        send_counts = _dispatch.as_counts(send_counts, x)
    return _Scatterv.run(x, send_counts, root, rows, max_rows, comm)[0]
