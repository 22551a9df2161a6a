"""sendrecv: simultaneous send and receive, Status, vmap, reverse-mode AD through one and two
exchanges, forward-mode rejection (scenario parity with
/root/reference/tests/collective_ops/test_sendrecv.py)."""

import pytest
import torch
from torch.func import grad, jacfwd, jacrev, vmap

import mpi4jax_b200 as m
from mpi4jax_b200 import MPI

from .._peer_job import needs_peers

comm = MPI.COMM_WORLD
rank = comm.Get_rank()
size = comm.Get_size()

pair = needs_peers("Runs only on rank 0 and 1", max_rank=1)
other = 1 - rank


@pair
def test_sendrecv(device):
    arr = torch.ones((3, 2), device=device) * rank
    _arr = arr.clone()
    res = m.sendrecv(arr, arr, source=other, dest=other)
    assert torch.equal(res, torch.ones_like(arr) * other)
    assert torch.equal(_arr, arr)


@pair
def test_sendrecv_status(device):
    arr = torch.ones((3, 2), device=device) * rank
    status = MPI.Status()
    res = m.sendrecv(arr, arr, source=other, dest=other, status=status)
    assert torch.equal(res, torch.ones_like(arr) * other)
    assert status.Get_source() == other


@pair
def test_sendrecv_status_jit(device):
    arr = torch.ones((3, 2), device=device) * rank
    status = MPI.Status()
    f = m.jit(lambda x, y: m.sendrecv(x, y, source=other, dest=other, status=status))
    for _ in range(3):
        res = f(arr, arr)
        assert torch.equal(res, torch.ones_like(arr) * other)
        assert status.Get_source() == other


@pair
def test_sendrecv_scalar(device):
    res = m.sendrecv(rank, rank, source=other, dest=other)
    assert res.item() == other


@pair
def test_sendrecv_jit(device):
    arr = torch.ones((3, 2), device=device) * rank
    f = m.jit(lambda x, y: m.sendrecv(x, y, source=other, dest=other))
    for _ in range(3):
        assert torch.equal(f(arr, arr), torch.ones_like(arr) * other)


@pair
def test_sendrecv_different_shapes(device):
    sendbuf = torch.ones(3 + rank, device=device) * rank
    recvbuf = torch.empty(3 + other, device=device)
    res = m.sendrecv(sendbuf, recvbuf, source=other, dest=other)
    assert torch.equal(res, torch.ones(3 + other, device=device) * other)


@pair
def test_sendrecv_vmap(device):
    arr = torch.ones((3, 2), device=device) * rank

    def fun(x, y):
        return m.sendrecv(x, y, source=other, dest=other)

    res = vmap(fun, in_dims=(0, 0))(arr, arr)
    assert torch.equal(res, torch.ones_like(arr) * other)


@pair
def test_sendrecv_grad(device):
    arr = torch.ones((3, 2), device=device) * (rank + 1)
    _arr = arr.clone()

    def f(x):
        x = m.sendrecv(x, x, source=other, dest=other)
        x = x * (rank + 1)
        return x.sum()

    res = grad(f)(arr)
    assert torch.equal(res, torch.ones_like(arr) * (other + 1))
    assert torch.equal(_arr, arr)


@pair
def test_sendrecv_grad_2(device):
    arr = torch.ones((3, 2), device=device) * (rank + 1)

    def f(x):
        x = m.sendrecv(x, x, source=other, dest=other)
        x = x * (rank + 1) * 5
        x = m.sendrecv(x, x, source=other, dest=other)
        x = x * (rank + 1) ** 2
        return x.sum()

    res = grad(f)(arr)
    solution = (rank + 1) ** 2 * (other + 1) * 5
    assert torch.equal(res, torch.ones_like(arr) * solution)


@pair
def test_sendrecv_jacfwd(device):
    arr = torch.ones((3, 2), device=device) * (rank + 1)

    def f(x):
        x = m.sendrecv(x, x, source=other, dest=other)
        return (x * (rank + 1)).sum()

    with pytest.raises(RuntimeError):
        jacfwd(f)(arr)


@pair
def test_sendrecv_jacrev(device):
    arr = torch.ones((3, 2), device=device) * (rank + 1)

    def f(x):
        x = m.sendrecv(x, x, source=other, dest=other)
        return (x * (rank + 1)).sum()

    res = jacrev(f)(arr)
    assert torch.equal(res, torch.ones_like(arr) * (other + 1))


def test_sendrecv_self(device):
    """Self-exchange (the reference's exit-time regression uses it, test_common.py:91-115)."""
    arr = torch.arange(10, dtype=torch.float32, device=device)
    f = m.jit(lambda x: m.sendrecv(x, x, source=rank, dest=rank))
    for _ in range(3):
        assert torch.equal(f(arr), arr)


def test_sendrecv_ring(device):
    """Ring shift over all ranks (building block of sequence-parallel schemes)."""
    arr = torch.ones(5, device=device) * rank
    res = m.sendrecv(arr, arr, source=(rank - 1) % size, dest=(rank + 1) % size)
    assert torch.equal(res, torch.ones(5, device=device) * ((rank - 1) % size))
