"""Scenario parity with /root/reference/tests/collective_ops/test_send_and_recv.py (+ ANY_SOURCE/ANY_TAG,
self-send and large-message cases the reference does not cover)."""

import pytest
import torch

import mpi4jax_b200 as m
from mpi4jax_b200 import MPI

from .._peer_job import needs_peers

comm = MPI.COMM_WORLD
rank = comm.Get_rank()
size = comm.Get_size()

need2 = needs_peers("need at least 2 processes to test send/recv")


@need2
def test_send_recv(device):
    arr = torch.ones((3, 2), device=device) * rank
    _arr = arr.clone()
    if rank == 0:
        for proc in range(1, size):
            res = m.recv(arr, source=proc, tag=proc)
            assert torch.equal(res, torch.ones_like(arr) * proc)
            assert torch.equal(_arr, arr)
    else:
        m.send(arr, 0, tag=rank)
        assert torch.equal(_arr, arr)


@need2
def test_send_recv_scalar(device):
    if rank == 0:
        for proc in range(1, size):
            res = m.recv(0, source=proc, tag=proc)
            assert res.item() == proc
    else:
        m.send(rank, 0, tag=rank)


@need2
def test_send_recv_jit(device):
    arr = torch.ones((3, 2), device=device) * rank

    @m.jit
    def send_jit(x):
        m.send(x, 0, tag=rank)
        return x

    for _ in range(3):
        if rank == 0:
            for proc in range(1, size):
                res = m.jit(lambda x: m.recv(x, source=proc, tag=proc))(arr)
                assert torch.equal(res, torch.ones_like(arr) * proc)
        else:
            send_jit(arr)


@needs_peers("Runs only on rank 0 and 1", max_rank=1)
def test_send_recv_deadlock(device):
    """Ops must execute in program order (reference: hangs if XLA reorders the custom calls)."""

    @m.jit
    def exchange(arr):
        if rank == 0:
            m.send(arr, 1)
            newarr = m.recv(arr, 1)
        else:
            newarr = m.recv(arr, 0)
            m.send(arr, 0)
        return newarr

    arr = torch.ones(10, device=device) * rank
    for _ in range(3):
        out = exchange(arr)
        assert torch.equal(out, torch.ones_like(arr) * (1 - rank))


@need2
def test_send_recv_status(device):
    arr = torch.ones((3, 2), device=device) * rank
    if rank == 0:
        for proc in range(1, size):
            status = MPI.Status()
            res = m.recv(arr, source=proc, tag=proc, status=status)
            assert torch.equal(res, torch.ones_like(arr) * proc)
            assert status.Get_source() == proc
            assert status.Get_tag() == proc
            assert status.Get_count() == 6
    else:
        m.send(arr, 0, tag=rank)


@need2
def test_recv_any_source_any_tag(device):
    arr = torch.ones(4, device=device) * rank
    if rank == 0:
        seen = set()
        for _ in range(1, size):
            status = MPI.Status()
            res = m.recv(arr, status=status)           # ANY_SOURCE, ANY_TAG
            src = status.Get_source()
            assert torch.equal(res, torch.ones_like(arr) * src)
            assert status.Get_tag() == 100 + src
            seen.add(src)
        assert seen == set(range(1, size))
    else:
        m.send(arr, 0, tag=100 + rank)


def test_send_recv_self(device):
    arr = torch.arange(7, dtype=torch.float32, device=device)
    m.send(arr, rank, tag=5)
    res = m.recv(torch.empty_like(arr), source=rank, tag=5)
    assert torch.equal(res, arr)


@need2
def test_send_recv_large(device):
    n = 3_000_001        # several ring fragments on the GPU path, odd size
    other = (rank + 1) % size
    prev = (rank - 1) % size
    arr = torch.arange(n, dtype=torch.float32, device=device) + rank
    if rank % 2 == 0:
        m.send(arr, other)
        res = m.recv(arr, prev)
    else:
        res = m.recv(arr, prev)
        m.send(arr, other)
    if size % 2 == 0:
        assert torch.equal(res, torch.arange(n, dtype=torch.float32, device=device) + prev)


@need2
def test_send_recv_grad(device):
    """Extension: recv is differentiable (adjoint = send back), send_with_grad closes the loop."""
    if rank == 0:
        x = torch.ones(3, device=device, requires_grad=True)
        tok = m.send_with_grad(x * 2, 1)
        tok.backward()
        assert torch.equal(x.grad, torch.ones(3, device=device) * 2 * 3)
    elif rank == 1:
        y = m.recv(torch.empty(3, device=device, requires_grad=True), source=0)
        (y * 3).sum().backward()


@need2
def test_send_recv_func_grad(device):
    """The same loop under torch.func.grad: the rules must peel the transform levels before they
    hand cotangents to the backend (raw pointers on the GPU path)."""
    if rank == 0:
        g = torch.func.grad(lambda x: m.send_with_grad(x * 2, 1))(torch.ones(3, device=device))
        assert torch.equal(g, torch.ones(3, device=device) * 2 * 3)
    elif rank == 1:
        g = torch.func.grad(lambda t: (m.recv(t, source=0) * 3).sum())(torch.empty(3, device=device))
        assert g is not None


@pytest.mark.parametrize("nelem", [5, 40_000, 300_000], ids=["tiny", "1lane", "multilane"])
@pytest.mark.parametrize("order", [(2, 0, 1), (1, 2, 0), (2, 1, 0), (0, 2, 1)])
def test_tags_matched_out_of_order_self(device, nelem, order):
    """MPI tag matching: a tagged receive takes the earliest pending message with that tag, even
    if messages with other tags were sent before it (the reference gets this from MPI itself)."""
    msgs = [torch.arange(nelem, dtype=torch.float32, device=device) + 1000 * k for k in range(3)]
    for k, x in enumerate(msgs):
        m.send(x, rank, tag=10 + k)
    for k in order:
        status = MPI.Status()
        got = m.recv(torch.empty_like(msgs[k]), source=rank, tag=10 + k, status=status)
        assert torch.equal(got, msgs[k])
        assert status.Get_tag() == 10 + k and status.Get_source() == rank
    # the queue is clean again: plain FIFO traffic with ANY_TAG still works afterwards
    for k, x in enumerate(msgs):
        m.send(x, rank, tag=20 + k)
    for k, x in enumerate(msgs):
        assert torch.equal(m.recv(torch.empty_like(x), source=rank), x)


def test_same_tag_is_not_overtaken_self(device):
    """Non-overtaking: two pending messages with the same tag are received in send order, also
    when they sit behind a message with another tag."""
    a, b, c_ = (torch.full((9,), float(v), device=device) for v in (1, 2, 3))
    m.send(a, rank, tag=1)
    m.send(b, rank, tag=7)
    m.send(c_, rank, tag=7)
    assert torch.equal(m.recv(torch.empty_like(a), source=rank, tag=7), b)
    assert torch.equal(m.recv(torch.empty_like(a), source=rank, tag=7), c_)
    assert torch.equal(m.recv(torch.empty_like(a), source=rank, tag=1), a)


@need2
def test_tags_matched_out_of_order_between_ranks(device):
    """rank r sends tags 0..3 to its right neighbour, which receives them in a different order,
    repeatedly (ring slots wrap around several times) and inside a jit-captured function."""
    dest, src = (rank + 1) % size, (rank - 1) % size
    perm = (3, 0, 2, 1)

    def round_trip(base):
        outs = []
        if rank % 2 == 0:
            for k in range(4):
                m.send(base + k, dest, tag=k)
        for k in perm:
            outs.append(m.recv(base, source=src, tag=k))
        if rank % 2 == 1:
            for k in range(4):
                m.send(base + k, dest, tag=k)
        return torch.stack(outs)

    if size % 2:
        pytest.skip("needs an even number of ranks")
    base = torch.arange(70_000, dtype=torch.float32, device=device) + 100 * rank
    want_base = torch.arange(70_000, dtype=torch.float32, device=device) + 100 * src
    want = torch.stack([want_base + k for k in perm])
    for _ in range(5):
        assert torch.equal(round_trip(base), want)
    f = m.jit(round_trip)
    for _ in range(4):
        assert torch.equal(f(base), want)
    m.flush()


def test_any_source_with_tag_matches_behind_the_head(device):
    """recv(ANY_SOURCE, tag=T) where T is not the oldest pending message of its source.  The CPU
    backend always matches it; the GPU election does so with the communicator option
    p2p_anysource_scan (default: only the oldest pending message of every source is considered)."""
    if device.type == "cuda":
        nc = comm._native_comm()         # the option belongs to this communicator: every op below uses it
        nc.set_option("p2p_anysource_scan", 1)
        try:
            _any_source_behind_the_head(device)
        finally:
            m.flush()
            nc.set_option("p2p_anysource_scan", 0)
    else:
        _any_source_behind_the_head(device)


def _any_source_behind_the_head(device):
    a = torch.full((6,), 1.0, device=device)
    b = torch.full((6,), 2.0, device=device)
    m.send(a, rank, tag=1, comm=comm)
    m.send(b, rank, tag=2, comm=comm)
    status = MPI.Status()
    got = m.recv(torch.empty_like(a), source=MPI.ANY_SOURCE, tag=2, status=status, comm=comm)
    assert torch.equal(got, b) and status.Get_source() == rank and status.Get_tag() == 2
    got = m.recv(torch.empty_like(a), source=MPI.ANY_SOURCE, tag=1, status=status, comm=comm)
    assert torch.equal(got, a) and status.Get_tag() == 1


def test_recv_size_must_match_the_message():
    """Both transports fix the message size by the receive template (the GPU kernel raises
    B2_ERR_TRUNCATE and aborts the job, so only the CPU side of the rule is exercised here)."""
    cpu = torch.device("cpu")
    m.send(torch.arange(3.0, device=cpu), rank, tag=31)
    with pytest.raises(RuntimeError, match="size mismatch"):
        m.recv(torch.empty(4, device=cpu), source=rank, tag=31)

