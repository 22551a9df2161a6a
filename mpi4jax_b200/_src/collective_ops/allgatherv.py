"""allgatherv -- a variable-count allgather whose counts stay on the device.

``MPI_Allgatherv`` for rows whose number is known only on the GPU (top-k gradients, tokens or particles
that survive a device-side filter): every rank contributes the first ``count`` rows of its input and
every rank receives all of them, packed in rank order into an output of static capacity.  The count
is a device tensor, so the host never waits for it and the call can be captured into a CUDA graph and
replayed with other counts.  Extension: the reference has no allgatherv.

Rules, on rank r of P (``x_r`` has shape ``(N, *S)``; ``N``, ``S`` and the dtype are the same on every
rank; capacity ``C_r``, which may differ between ranks):

* contributed: ``n_r = clamp(count_r, 0, N)`` rows, rows ``[0, n_r)`` of ``x_r``;
* received: ``c[q] = clamp(C_r - sum_{p<q} c[p], 0, n_q)`` rows from rank q land at row
  ``sum_{p<q} c[p]`` -- segments packed in source-rank order, a segment that does not fit loses its
  tail; rows past ``sum_q c[q]`` are zero.  ``recv_counts`` = ``c`` (int64, on x's device).

An invalid count is never an error and never makes the kernel read or write out of bounds.

GPU: alltoallv's kernel in gather mode (csrc/b2_collectives.cu: b2_k_rowsv).  Every rank stages its
``n_r`` rows once, behind a header holding ``n_r``; after one barrier each CTA reads the P headers,
derives the packed offsets itself and pulls its chunks of every peer's segment, each read from offset
0, straight into the output.  Differentiable: the adjoint is ``reduce_scatterv`` of the cotangent with
the received counts as send counts, so rank r gets the rank-order sum of what the receivers kept of its
rows, and only those rows travel.  The kernel's *reverse mode* (place counts) is in turn the adjoint of
``reduce_scatterv``.
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


class _Allgatherv(RowsvFunction):
    """``place_counts`` None: the forward gather into ``out_rows`` packed rows.  Otherwise the reverse mode:
    ``place_counts`` are a reduce_scatterv's send counts and ``out_rows`` its input rows; the segment from
    rank q lands where that call took rank q's rows from."""

    vmap_error = "allgatherv under vmap: the count must not be batched (one exchange moves every batch entry)"

    @staticmethod
    def forward(x, count, out_rows, place_counts, comm):
        return _dispatch.allgatherv(comm, x, count, out_rows, place_counts)

    @staticmethod
    def backward(ctx, g, _g_counts):
        _, _, place_counts, comm = ctx.args
        (recv_counts,) = ctx.saved_tensors
        counts = recv_counts if place_counts is None else place_counts
        return _adjoints.allgatherv(collective_ops.eager, g, comm, ctx.in_rows, counts), None, None, None, None


@enforce_types(recv_capacity=(type(None), np.integer), comm=(type(None), Comm))
def allgatherv(x, count, *, recv_capacity=None, comm=None, token=NOTSET):
    """Perform a variable-count allgather operation (``MPI_Allgatherv``) with a device-resident count.

    Arguments:
        x: input of shape ``(N, ...)``; ``N``, the row shape and the dtype must be the same on every rank.
        count: rows this rank contributes, taken from the start of ``x``: a Python int or an integer
            tensor of shape ``()`` on ``x``'s device.  Negative counts contribute nothing, counts past
            ``N`` are cut at ``N``.
        recv_capacity: rows of the output (default ``N * nproc``, which never drops a row; may differ
            between ranks).  A segment that does not fit loses its last rows.
        comm: the communicator (defaults to a clone of ``COMM_WORLD``).

    Returns:
        Tuple[Tensor, Tensor]: every rank's rows, shape ``(recv_capacity, ...)``, packed in rank order
        and zero past the last one, and ``recv_counts``, int64 ``(nproc,)`` on the device: the rows
        written from each rank.
    """
    raise_if_token_is_set(token)
    if comm is None:
        comm = get_default_comm()
    x = as_tensor(x, comm)
    check_dtype(x)
    _dispatch.check_rows("Allgatherv", x)
    count = _dispatch.as_counts(count, x, scalar=True)
    cap = int(_dispatch.rowsv_capacity("Allgatherv", comm, x, count, recv_capacity, "count", comm.Get_size()))
    return _Allgatherv.run(x, count, cap, None, comm)


def allgatherv_reverse(y: torch.Tensor, place_counts: torch.Tensor, rows: int, comm: Comm) -> torch.Tensor:
    """The adjoint of ``reduce_scatterv(x, place_counts, SUM)`` (``y`` laid out like its output, ``rows``
    its input rows): every rank's ``y`` travels to every rank q and lands where q took its segment for
    that rank from -- at most ``min(place_counts_q[p], len(y))`` rows from rank p, the counts clamped in
    rank order to ``rows``.  Other rows are zero.  Differentiable (the adjoint is reduce_scatterv)."""
    place_counts = _dispatch.as_counts(place_counts, y)
    count = torch.full((), y.shape[0], dtype=torch.int64, device=y.device)
    _dispatch.check_rowsv_args("Allgatherv", comm, y, place_counts, rows, "place_counts")
    return _Allgatherv.run(y, count, rows, place_counts, comm)[0]
