"""Functional op namespace: the 15 primitives plus the fused ops that go beyond the
reference's one-MPI-call-per-op model (fused multi-field halo exchange, the fused linear layers and top-k
expert routing)."""

from .._src import (  # noqa: F401
    allgather, allgatherv, allreduce, alltoall, alltoallv, barrier, bcast, gather, gatherv, recv, reduce,
    reduce_scatter, reduce_scatterv, scan, scatter, scatterv, send, send_with_grad, sendrecv,
)
from .halo import halo_exchange  # noqa: F401
from .linear import linear_allgather, linear_allreduce, linear_reduce_scatter  # noqa: F401
from .moe import MoePlan, moe_combine, moe_dispatch  # noqa: F401
