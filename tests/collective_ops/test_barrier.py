"""Port of /root/reference/tests/collective_ops/test_barrier.py."""

import os
import tempfile
import time

import torch

import mpi4jax_b200 as m
from mpi4jax_b200 import MPI

comm = MPI.COMM_WORLD


def test_barrier(device):
    """Ranks append lines before/after a barrier to one file; all 'start' lines must precede
    all 'done' lines."""
    rank, size = comm.Get_rank(), comm.Get_size()
    # a fresh file per run, named by rank 0: a fixed name in the shared temp directory could belong
    # to another user or to a concurrent job
    write_to = None
    if rank == 0:
        fd, write_to = tempfile.mkstemp(prefix=f"mpi4jax-b200-barrier-{device.type}-", suffix=".txt")
        os.close(fd)
    write_to = comm.bcast(write_to, root=0)
    comm.Barrier()
    time.sleep(rank * 0.2)
    with open(write_to, "a") as f:
        f.write(f"r{rank} | start\n")
    m.barrier()
    m.flush()       # the barrier is stream-ordered; flush makes it a host rendezvous
    with open(write_to, "a") as f:
        f.write(f"r{rank} | done\n")
    time.sleep(0.2)
    m.barrier()
    m.flush()
    comm.Barrier()
    with open(write_to) as f:
        outputs = f.readlines()
    comm.Barrier()
    if rank == 0:
        os.remove(write_to)
    assert len(outputs) == size * 2
    assert all(o.endswith("start\n") for o in outputs[:size])
    assert all(o.endswith("done\n") for o in outputs[size:])


def test_barrier_jit(device):
    def f(x):
        m.barrier()
        y = x + 1
        m.barrier()
        return y

    fj = m.jit(f)
    x = torch.zeros(3, device=device)
    for _ in range(3):
        assert torch.equal(fj(x), x + 1)
