"""alltoallv -- a variable-count all-to-all whose counts stay on the device.

``MPI_Alltoallv`` in the shape a mixture-of-experts layer needs: rows grouped by destination rank, a
compact output of static capacity, and counts that are device tensors (e.g. computed by a router),
so the host never waits for them and the call can be captured into a CUDA graph.  Extension: the
reference has no alltoallv.

Rules, on rank r of P (``x_r`` has ``N`` rows, the same on every rank; capacity ``C_r``):

* sent: ``s'[r,q] = clamp(N - sum_{p<q} s'[r,p], 0, max(send_counts_r[q], 0))`` rows, starting at
  row ``sum_{p<q} s'[r,p]``, go to rank q;
* received: ``c[q,r] = clamp(C_r - sum_{p<q} c[p,r], 0, s'[q,r])`` rows from rank q land at row
  ``sum_{p<q} c[p,r]`` -- the first rows of q's segment, in source-rank order; rows past
  ``sum_q c[q,r]`` are zero.  ``recv_counts`` = ``c[:, r]``.

GPU: every rank stages its send rows behind a header of its clamped counts; after one barrier each
CTA reads all headers and pulls its chunks of the peers' segments straight into the output
(csrc/b2_collectives.cu: b2_k_rowsv).  Differentiable: the adjoint is the *reverse mode* of the
same kernel, which puts the rows received from rank q back where rank q sent them from.
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


class _Alltoallv(RowsvFunction):
    """``place_counts`` None: the forward exchange into ``out_rows`` packed rows.  Otherwise the reverse
    mode: ``send_counts`` are a forward's ``recv_counts``, ``place_counts`` its send counts and
    ``out_rows`` its input rows; each rank gets back the rows it sent, where it sent them from."""

    vmap_error = "alltoallv under vmap: the counts must not be batched (one exchange moves every batch entry)"

    @staticmethod
    def forward(x, send_counts, out_rows, place_counts, comm):
        return _dispatch.alltoallv(comm, x, send_counts, out_rows, place_counts)

    @staticmethod
    def backward(ctx, g, _g_counts):
        send_counts, _, place_counts, comm = ctx.args
        (recv_counts,) = ctx.saved_tensors
        back = _adjoints.alltoallv(collective_ops.eager, g, comm, ctx.in_rows, send_counts, recv_counts, place_counts)
        return back, None, None, None, None


@enforce_types(recv_capacity=(type(None), np.integer), comm=(type(None), Comm))
def alltoallv(x, send_counts, *, recv_capacity=None, comm=None, token=NOTSET):
    """Perform a variable-count alltoall operation (``MPI_Alltoallv``) with device-resident counts.

    Arguments:
        x: input of shape ``(N, ...)``, rows grouped by destination rank; ``N``, the row shape and the
            dtype must be the same on every rank.
        send_counts: integer tensor of shape ``(nproc,)`` on ``x``'s device (or a sequence of ints):
            rows for each rank, taken in rank order from the start of ``x``.  Negative counts send
            nothing, counts past the end of ``x`` are cut at its last row.
        recv_capacity: rows of the output (default ``N * nproc``, which never drops a row; may differ
            between ranks).  Segments that do not fit lose their last rows.
        comm: the communicator (defaults to a clone of ``COMM_WORLD``).

    Returns:
        Tuple[Tensor, Tensor]: the received rows, shape ``(recv_capacity, ...)``, packed in source-rank
        order and zero past the last one, and ``recv_counts``, int64 ``(nproc,)`` on the device: the rows
        written from each rank.  A sender can detect dropped rows by comparing its counts with an
        ``alltoall`` of the receivers' ``recv_counts``.
    """
    raise_if_token_is_set(token)
    if comm is None:
        comm = get_default_comm()
    x = as_tensor(x, comm)
    check_dtype(x)
    _dispatch.check_rows("Alltoallv", x)
    send_counts = _dispatch.as_counts(send_counts, x)
    cap = int(_dispatch.rowsv_capacity("Alltoallv", comm, x, send_counts, recv_capacity, "send_counts",
                                       comm.Get_size()))
    return _Alltoallv.run(x, send_counts, cap, None, comm)


def alltoallv_reverse(y: torch.Tensor, recv_counts: torch.Tensor, send_counts: torch.Tensor, rows: int,
                      comm: Comm) -> torch.Tensor:
    """The reverse of ``alltoallv(x, send_counts)`` that returned ``recv_counts``: rows of ``y`` (laid out
    like that call's output) travel back to the rank they came from and land where it sent them from,
    in an output of ``rows`` rows (that call's ``N``).  Rows that were dropped or never sent are zero.
    Differentiable (the adjoint is the forward exchange)."""
    recv_counts, send_counts = _dispatch.as_counts(recv_counts, y), _dispatch.as_counts(send_counts, y)
    _dispatch.check_rowsv_args("Alltoallv", comm, y, recv_counts, rows, "recv_counts")
    _dispatch.check_rowsv_args("Alltoallv", comm, y, send_counts, rows, "send_counts")
    return _Alltoallv.run(y, recv_counts, rows, send_counts, comm)[0]
