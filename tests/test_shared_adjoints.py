"""One adjoint rule per collective (mpi4jax_b200/_src/collective_ops/_adjoints.py) serves the eager ops and
the ``torch.compile`` frontend: the gradient through an eager op and through the traced ``compiled`` op
must be bitwise equal, on every rank."""

from types import SimpleNamespace

import pytest
import torch

import mpi4jax_b200 as m
from mpi4jax_b200 import MPI
from mpi4jax_b200 import compiled as mc
from mpi4jax_b200._src.collective_ops.allgatherv import allgatherv_reverse
from mpi4jax_b200._src.collective_ops.alltoallv import alltoallv_reverse
from mpi4jax_b200._src.collective_ops.gatherv import gatherv_reverse

comm = MPI.COMM_WORLD
rank, size = comm.Get_rank(), comm.Get_size()

N = 5
# the two frontends; the reverse modes are public in neither
EAGER = SimpleNamespace(reduce_scatter=m.reduce_scatter, allgather=m.allgather, alltoall=m.alltoall,
                        alltoallv=m.alltoallv, _alltoallv_reverse=alltoallv_reverse, allgatherv=m.allgatherv,
                        _allgatherv_reverse=allgatherv_reverse, reduce_scatterv=m.reduce_scatterv,
                        gatherv=m.gatherv, _gatherv_reverse=gatherv_reverse, scatterv=m.scatterv,
                        bcast=m.bcast, sendrecv=m.sendrecv)


def _rand(*shape, device, seed):
    return torch.randn(shape, generator=torch.Generator().manual_seed(100 * seed + rank)).to(device)


def _a2av_counts(device):
    """Counts to clamp in rank order (negative, and past N) and a capacity that clips, different per rank."""
    return torch.tensor([[3, -1, N + 1][(q + rank) % 3] for q in range(size)], device=device), 2 + rank


def _case(op, device):
    """(loss(F, x), x) for one op."""
    if op == "reduce_scatter":
        w = _rand(3, device=device, seed=1)
        return lambda F, x: (F.reduce_scatter(x, MPI.SUM, comm=comm) * w).sum(), _rand(size, 3, device=device, seed=2)
    if op == "allgather":
        w = _rand(size, 3, device=device, seed=1)
        return lambda F, x: (F.allgather(x, comm=comm) * w).sum(), _rand(3, device=device, seed=2)
    if op == "alltoall":
        w = _rand(size, 3, device=device, seed=1)
        return lambda F, x: (F.alltoall(x, comm=comm) * w).sum(), _rand(size, 3, device=device, seed=2)
    if op == "alltoallv":
        counts, cap = _a2av_counts(device)
        w = _rand(cap, 2, device=device, seed=1)
        return (lambda F, x: (F.alltoallv(x, counts, recv_capacity=cap, comm=comm)[0] * w).sum(),
                _rand(N, 2, device=device, seed=2))
    if op == "alltoallv_reverse":
        counts, cap = _a2av_counts(device)
        recv_counts = m.alltoallv(_rand(N, 2, device=device, seed=3), counts, recv_capacity=cap, comm=comm)[1]
        w = _rand(N, 2, device=device, seed=1)
        return (lambda F, y: (F._alltoallv_reverse(y, recv_counts, counts, N, comm) * w).sum(),
                _rand(cap, 2, device=device, seed=2))
    if op == "allgatherv":
        count = torch.tensor(N - 1 - rank % 2, device=device)
        w = _rand(N * size, 2, device=device, seed=1)
        return (lambda F, x: (F.allgatherv(x, count, comm=comm)[0] * w).sum(),
                _rand(N, 2, device=device, seed=2))
    if op == "allgatherv_reverse":
        # the adjoint of a reduce_scatterv whose input had N + rank rows
        counts, _ = _a2av_counts(device)
        w = _rand(N + rank, 2, device=device, seed=1)
        return (lambda F, y: (F._allgatherv_reverse(y, counts, N + rank, comm) * w).sum(),
                _rand(3, 2, device=device, seed=2))
    if op == "reduce_scatterv":
        counts, _ = _a2av_counts(device)
        w = _rand(4, 2, device=device, seed=1)
        return (lambda F, x: (F.reduce_scatterv(x, counts, MPI.SUM, recv_capacity=4, comm=comm)[0] * w).sum(),
                _rand(N + rank, 2, device=device, seed=2))
    if op == "gatherv":
        # root: not rank 0 when there is more than one rank; its capacity clips the last segment
        root, count = size - 1, torch.tensor([N + 1, -1, 3][rank % 3], device=device)
        cap = N * size - 1 if rank == root else None
        w = _rand(N * size - 1 if rank == root else N, 2, device=device, seed=1)
        return (lambda F, x: (F.gatherv(x, count, root, recv_capacity=cap, comm=comm)[0] * w).sum(),
                _rand(N, 2, device=device, seed=2))
    if op == "gatherv_reverse":
        # the adjoint of a scatterv from the last rank into 2 + rank rows
        root, (counts, cap) = size - 1, _a2av_counts(device)
        recv_count = m.scatterv(_rand(N, 2, device=device, seed=3), counts, root, recv_capacity=cap, comm=comm)[1]
        w = _rand(N, 2, device=device, seed=1)
        return (lambda F, y: (F._gatherv_reverse(y, recv_count, counts, root, N, N, comm) * w).sum(),
                _rand(cap, 2, device=device, seed=2))
    if op == "scatterv":
        # the counts are given on the root only; the capacities clip, different per rank
        root, (counts, cap) = size - 1, _a2av_counts(device)
        counts = counts if rank == root else None
        w = _rand(cap, 2, device=device, seed=1)
        return (lambda F, x: (F.scatterv(x, counts, root, recv_capacity=cap, comm=comm)[0] * w).sum(),
                _rand(N, 2, device=device, seed=2))
    if op == "bcast":
        root = size - 1                 # not rank 0 when there is more than one rank
        w = _rand(4, device=device, seed=1)
        return lambda F, x: (F.bcast(x * 2, root, comm=comm) * w).sum(), _rand(4, device=device, seed=2)
    if op == "sendrecv":
        # a tagged send and a receive with the default recvtag (ANY_TAG): the cotangent goes back with
        # each rank's own tags, so it matches
        w = _rand(4, device=device, seed=1)
        source, dest = (rank - 1) % size, (rank + 1) % size
        return (lambda F, x: (F.sendrecv(x * 3, torch.zeros_like(x), source, dest, sendtag=4, comm=comm) * w).sum(),
                _rand(4, device=device, seed=2))
    raise AssertionError(op)


@pytest.mark.parametrize("op", ["reduce_scatter", "allgather", "alltoall", "alltoallv", "alltoallv_reverse",
                                "allgatherv", "allgatherv_reverse", "reduce_scatterv", "gatherv", "gatherv_reverse",
                                "scatterv", "bcast", "sendrecv"])
def test_eager_and_compiled_gradients_are_equal(device, op):
    loss, x = _case(op, device)
    xe = x.clone().requires_grad_(True)
    loss(EAGER, xe).backward()
    xc = x.clone().requires_grad_(True)
    torch.compile(loss, backend="aot_eager", fullgraph=True)(mc, xc).backward()
    assert torch.equal(xc.grad, xe.grad)
    m.flush()
