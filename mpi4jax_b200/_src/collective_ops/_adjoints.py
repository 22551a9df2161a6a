"""The adjoint (VJP) of each collective that both frontends differentiate, written once.

Each function maps the output cotangent ``g`` and the state its op saved to the input cotangent, calling
collectives only through ``F``, a namespace with the public op signatures: ``collective_ops.eager`` from
the ``torch.autograd.Function`` backwards, ``compiled`` from the ``torch.library`` rules.

allreduce is not here: its eager backward is its own Function with ``transpose=True``, so that nested
transposes give the allreduce back (tests/collective_ops/test_allreduce_matvec.py); its traced rule
returns ``g``.
"""

from __future__ import annotations

import torch

from ..comm import SUM


def reduce_scatter(F, g, comm):
    """SUM: the allgather of the cotangent."""
    return F.allgather(g.contiguous(), comm=comm)


def allgather(F, g, comm):
    """The reduce-scatter of the cotangent, realised as allreduce + own slice."""
    return F.allreduce(g.contiguous(), SUM, comm=comm)[comm.Get_rank()]


def alltoall(F, g, comm):
    """The all-to-all of the cotangent."""
    return F.alltoall(g.contiguous(), comm=comm)


def alltoallv(F, g, comm, rows, send_counts, recv_counts, place_counts):
    """Forward <-> reverse mode, with the differentiated call's counts and input ``rows``: the rows travel
    back the way they came."""
    g = g.contiguous()
    if place_counts is None:
        return F._alltoallv_reverse(g, recv_counts, send_counts, rows, comm)
    return F.alltoallv(g, place_counts, recv_capacity=rows, comm=comm)[0]


def segments(g: torch.Tensor, recv_counts: torch.Tensor, rows: int) -> torch.Tensor:
    """``G`` of shape ``(P, rows, *S)`` with ``G[q, i] = g[o[q] + i]`` for ``i < recv_counts[q]`` and 0
    otherwise, where ``o`` is the exclusive prefix sum of ``recv_counts``: the segments of an allgatherv
    output, each back at the start of its source's rows.  Device ops only (no host read of the counts);
    differentiable in ``g``."""
    P = recv_counts.shape[0]
    offsets = torch.cumsum(recv_counts, 0) - recv_counts
    i = torch.arange(rows, device=g.device)
    # entries past a segment read a zero row appended to g (index g.shape[0])
    idx = torch.where(i < recv_counts.view(P, 1), offsets.view(P, 1) + i, g.shape[0])
    padded = torch.cat([g, g.new_zeros((1, *g.shape[1:]))])
    return padded[idx]


def allgatherv(F, g, comm, rows, recv_counts):
    """SUM: the received segments, zero-padded to ``(P, rows, *S)``, reduce-scattered, so rank r gets the
    rank-order sum of what the receivers kept of its rows."""
    return F.reduce_scatter(segments(g, recv_counts, rows), SUM, comm=comm)


def bcast(F, g, root, comm):
    """The sum of the cotangents on the root, zero elsewhere (the input there is only a template)."""
    total = F.reduce(g.contiguous(), SUM, root, comm=comm)
    if comm.Get_rank() == root:
        return total
    # zeros that still depend on the reduce: a second derivative then runs the reduce's backward, a bcast
    # from the root, on every rank (on the root alone it would wait for the others forever), and the
    # other ranks receive their share of it
    return total.masked_fill(total.new_ones((), dtype=torch.bool), 0)


def sendrecv(F, g, template, source, dest, sendtag, recvtag, comm):
    """The cotangent of what was received travels back to where it came from: source and dest swap,
    and each rank keeps its own tags (it sends with ``sendtag`` and receives with ``recvtag``).
    ``template`` has the shape and dtype of the differentiated call's ``sendbuf``."""
    return F.sendrecv(g.contiguous(), template, dest, source, sendtag=sendtag, recvtag=recvtag, comm=comm)
