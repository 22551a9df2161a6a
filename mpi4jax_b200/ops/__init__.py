"""Functional op namespace: the 15 primitives plus the fused ops that go beyond the
reference's one-MPI-call-per-op model (fused multi-field halo exchange)."""

from .._src import (  # noqa: F401
    allgather, allgatherv, allreduce, alltoall, alltoallv, barrier, bcast, gather, gatherv, recv, reduce,
    reduce_scatter, reduce_scatterv, scan, scatter, scatterv, send, send_with_grad, sendrecv,
)
from .halo import halo_exchange  # noqa: F401
from .linear import linear_allgather, linear_allreduce, linear_reduce_scatter  # noqa: F401
