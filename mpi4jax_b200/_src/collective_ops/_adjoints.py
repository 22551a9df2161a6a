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


def allgatherv(F, g, comm, rows, recv_counts):
    """SUM: each received segment travels back to its source, which folds them in rank order into its
    ``rows`` input rows.  ``recv_counts``: the forward call's (the segments are packed), or in the reverse
    mode its place counts (the segments lie where a reduce_scatterv took them from)."""
    return F.reduce_scatterv(g.contiguous(), recv_counts, SUM, recv_capacity=rows, comm=comm)[0]


def reduce_scatterv(F, g, comm, rows, send_counts):
    """SUM: the reverse-mode allgatherv of the cotangent -- every rank's result rows land on each rank where
    its segment for that rank came from, in an output of the differentiated call's ``rows`` input rows."""
    return F._allgatherv_reverse(g.contiguous(), send_counts, rows, comm)


def gatherv(F, g, comm, root, rows, max_rows, recv_counts):
    """The scatterv of the root's cotangent with its received counts as send counts, into the differentiated
    call's ``rows`` input rows: each rank gets back what the root kept of its rows, and only those rows
    travel.  The root's cotangent has the root's capacity in rows, which the other ranks do not know, so the
    scatterv stages with the bound ``nproc * max_rows`` that every rank knows.  On the other ranks the
    result was ``x`` itself, so their own cotangent adds (as for gather)."""
    is_root = comm.Get_rank() == root
    back = F._scatterv_bounded(g.contiguous(), recv_counts if is_root else None, root, rows,
                               max_rows * comm.Get_size(), comm)
    return back if is_root else back + g


def gatherv_reverse(F, g, comm, root, rows, max_rows, place_counts):
    """The forward scatterv that the reverse mode is the adjoint of: the root's cotangent by the place counts,
    into each rank's ``rows`` input rows of the differentiated call.  The other ranks' result was zeros, so
    their cotangent drops."""
    is_root = comm.Get_rank() == root
    return F._scatterv_bounded(g.contiguous(), place_counts if is_root else None, root, rows, max_rows, comm)


def scatterv(F, g, comm, root, rows, max_rows, recv_count, send_counts):
    """The reverse-mode gatherv of the cotangent: each rank's first ``recv_count`` rows land on the root where
    they were taken from, in an output of the differentiated call's ``rows`` input rows; the other ranks'
    inputs were templates and get zeros that are the gatherv's result, so that a second derivative runs
    its adjoint, a scatterv from the root, on every rank."""
    return F._gatherv_reverse(g.contiguous(), recv_count, send_counts, root, rows, max_rows, comm)


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
