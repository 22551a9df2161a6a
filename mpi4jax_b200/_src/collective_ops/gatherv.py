"""gatherv -- a variable-count gather whose counts stay on the device.

``MPI_Gatherv`` for rows whose number is known only on the GPU (particles or candidates that survive a
device-side filter, per-rank results to write out): every rank contributes the first ``count`` rows of
its input and the root receives all of them, packed in rank order into an output of static capacity.
The count is a device tensor, so the host never waits for it and the call can be captured into a CUDA
graph and replayed with other counts.  Extension: the reference has no gatherv.

Rules, on rank r of P (``x_r`` has shape ``(N, *S)``; ``N``, ``S`` and the dtype are the same on every
rank; the capacity ``C`` is read on the root only):

* contributed: ``n_r = clamp(count_r, 0, N)`` rows, rows ``[0, n_r)`` of ``x_r``;
* on the root: ``c[q] = clamp(C - sum_{p<q} c[p], 0, n_q)`` rows from rank q land at row
  ``sum_{p<q} c[p]``; rows past ``sum_q c[q]`` are zero.  ``recv_counts`` = ``c`` (int64, on x's device);
* elsewhere: the result is ``x`` itself (as for ``gather``) and ``recv_counts`` is zero.

An invalid count is never an error and never makes the kernel read or write out of bounds.

GPU: allgatherv's kernel in gather mode (csrc/b2_collectives.cu: b2_k_rowsv), with output rows on the
root only: every rank stages its ``n_r`` rows behind a header holding ``n_r`` and walks the same chunks,
but only the root pulls.  Differentiable: the adjoint is ``scatterv`` of the root's cotangent with the
received counts as send counts (a non-root rank adds its own cotangent, as for ``gather``), and only
received rows travel.  The kernel's *reverse mode* (place counts) is in turn the adjoint of ``scatterv``.
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


def _result(comm, x, out, root, out_rows, reverse):
    """The root's output; elsewhere ``x`` itself (forward; under autograd, ``apply`` returns a view of it) or
    zeros of ``out_rows`` rows (reverse mode)."""
    if comm.Get_rank() == root:
        return out
    return x.new_zeros((out_rows, *x.shape[1:])) if reverse else x


class _Gatherv(RowsvFunction):
    """``reverse`` False: the forward gather into the root's ``out_rows`` packed rows.  Otherwise the reverse
    mode, the adjoint of a scatterv whose send counts were ``place_counts`` and whose input had
    ``out_rows`` rows on this rank: on the root the segment from rank q lands where that call took rank
    q's rows from; the other ranks get zeros.  ``max_rows``: the rows any rank may contribute, the same on
    every rank."""

    vmap_error = "gatherv under vmap: the count must not be batched (one exchange moves every batch entry)"

    @staticmethod
    def forward(x, count, root, out_rows, max_rows, place_counts, reverse, comm):
        out, recv_counts = _dispatch.gatherv(comm, x, count, root, out_rows, max_rows, place_counts)
        return _result(comm, x, out, root, out_rows, reverse), recv_counts

    @staticmethod
    def backward(ctx, g, _g_counts):
        _, root, _, max_rows, place_counts, reverse, comm = ctx.args
        F = collective_ops.eager
        if reverse:
            back = _adjoints.gatherv_reverse(F, g, comm, root, ctx.in_rows, max_rows, place_counts)
        else:
            (recv_counts,) = ctx.saved_tensors
            back = _adjoints.gatherv(F, g, comm, root, ctx.in_rows, max_rows, recv_counts)
        return back, None, None, None, None, None, None, None


@enforce_types(root=(np.integer,), recv_capacity=(type(None), np.integer), comm=(type(None), Comm))
def gatherv(x, count, root, *, recv_capacity=None, comm=None, token=NOTSET):
    """Perform a variable-count gather operation (``MPI_Gatherv``) with a device-resident count.

    Arguments:
        x: input of shape ``(N, ...)``; ``N``, the row shape and the dtype must be the same on every rank.
        count: rows this rank contributes, taken from the start of ``x``: a Python int or an integer
            tensor of shape ``()`` on ``x``'s device.  Negative counts contribute nothing, counts past
            ``N`` are cut at ``N``.
        root (int): the rank that receives.
        recv_capacity: rows of the root's output (default ``N * nproc``, which never drops a row); read on
            the root only.  A segment that does not fit loses its last rows.
        comm: the communicator (defaults to a clone of ``COMM_WORLD``).

    Returns:
        Tuple[Tensor, Tensor]: on the root every rank's rows, shape ``(recv_capacity, ...)``, packed in
        rank order and zero past the last one, and ``recv_counts``, int64 ``(nproc,)`` on the device: the
        rows written from each rank.  On every other rank ``x`` itself and ``(nproc,)`` zeros.
    """
    raise_if_token_is_set(token)
    if comm is None:
        comm = get_default_comm()
    x = as_tensor(x, comm)
    check_dtype(x)
    _check_root(root, comm, "Gatherv")
    root = int(root)
    _dispatch.check_rows("Gatherv", x)
    count = _dispatch.as_counts(count, x, scalar=True)
    cap = int(_dispatch.gatherv_capacity(comm, x, count, root, recv_capacity))
    return _Gatherv.run(x, count, root, cap, x.shape[0], None, False, comm)


def gatherv_reverse(y: torch.Tensor, count: torch.Tensor, place_counts, root: int, rows: int, max_rows: int,
                    comm: Comm) -> torch.Tensor:
    """The adjoint of ``scatterv`` (``y`` laid out like its output, ``count`` its recv_count, ``place_counts``
    its send counts on the root, ``rows`` its input rows on this rank, ``max_rows`` its staging bound): the
    first ``count`` rows of every rank's ``y`` land on the root where that call took them from.  Other rows
    are zero, and so is the result on every other rank.  Differentiable (the adjoint is scatterv)."""
    if comm.Get_rank() == root:
        place_counts = _dispatch.as_counts(place_counts, y)
        _dispatch.check_rowsv_args("Gatherv", comm, y, place_counts, rows, "place_counts")
    return _Gatherv.run(y, count, root, rows, max_rows, place_counts, True, comm)[0]
