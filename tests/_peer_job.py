"""Point-to-point tests need a peer rank.  In a single-process run their CPU variants skip (the
multi-rank CPU job of tests/test_multirank.py runs them), but on a GPU machine the CUDA variants
still run: the test file is run once as a two-rank job on the GPUs there are (both ranks share the
GPU when there is only one), and each test passes when it passed on both ranks of that job."""

import functools
import hashlib
import inspect
import os
import re
import tempfile

import numpy as np
import pytest
import torch
import torch.distributed as dist

from mpi4jax_b200 import MPI
from mpi4jax_b200.run import launch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
JOB_RANKS = 2
JOB_TIMEOUT_S = 900


@functools.lru_cache(maxsize=None)
def _pair_job(test_file: str):
    """(exit code, [output of every rank]).  The ranks write to log files, not pipes: a pipe that is
    not drained while the job runs would stall a rank that prints more than the pipe holds."""
    args = ["-m", "pytest", test_file, "-q", "-rp", "-m", "gpu", "-p", "no:cacheprovider"]
    cwd = os.getcwd()
    os.chdir(REPO)
    try:
        with tempfile.TemporaryDirectory(prefix="mpi4jax-b200-pair-job-") as logs:
            code, _ = launch(JOB_RANKS, args, timeout=JOB_TIMEOUT_S, output_dir=logs,
                             env_extra={"MPI4JAX_B200_NESTED": "1"})
            outs = []
            for rank in range(JOB_RANKS):
                with open(os.path.join(logs, f"rank{rank}.log")) as fh:
                    outs.append(fh.read())
        return code, outs
    finally:
        os.chdir(cwd)


def _expect_passed_in_pair_job(fn) -> None:
    test_file = os.path.relpath(inspect.getsourcefile(fn), REPO)
    test_id = f"{test_file}::{fn.__name__}[cuda]"
    code, outs = _pair_job(test_file)
    for rank, out in enumerate(outs):
        if not re.search(rf"^PASSED {re.escape(test_id)}\s*$", out, re.M):
            raise AssertionError(f"{test_id} did not pass on rank {rank} of the {JOB_RANKS}-rank job "
                                 f"(exit code {code}):\n{out[-4000:]}")


def digest(t) -> str:
    """sha1 of the bytes of a tensor or numpy array."""
    t = (torch.from_numpy(np.ascontiguousarray(t)) if isinstance(t, np.ndarray) else t.detach().cpu()).contiguous()
    return hashlib.sha1(t.view(torch.uint8).numpy().tobytes() if t.numel() else b"").hexdigest()


def _expect(ok, message):
    assert ok, message


class Checks:
    """The assertions of a multi-rank test, raised at its end.  A check that fails on one rank only must
    not leave the ranks running different sequences of collectives, so ``chk(fn, *args)`` records an
    AssertionError of ``fn(*args)`` and goes on.  ``chk.add(label, t)`` records a hash of a result that
    every rank must hold bit for bit; ``chk.add(label, t, want)`` one whose value on rank q must be
    ``want[q]``.  ``chk.finish()`` compares those over the control plane (gloo)."""

    def __init__(self):
        self.rows = []
        self.failures = []

    def __call__(self, fn, *args):
        try:
            fn(*args)
        except AssertionError as exc:
            self.failures.append(str(exc))

    def add(self, label, t, want=None):
        self.rows.append((label, digest(t), None if want is None else [digest(w) for w in want]))

    def finish(self):
        comm = MPI.COMM_WORLD
        size, rank = comm.Get_size(), comm.Get_rank()
        if size > 1:
            out = [None] * size
            dist.all_gather_object(out, [(label, h) for label, h, _ in self.rows], group=comm._group)
            for q, rows in enumerate(out):
                for (label, h), (_, h0), (_, _, want) in zip(rows, out[0], self.rows):
                    if want is None:
                        self(_expect, h == h0, f"{label}: rank {q}'s result differs from rank 0's")
                    else:
                        self(_expect, h == want[q], f"{label}: rank {q}'s result differs from rank {rank}'s "
                                                    f"expectation of it")
                self(_expect, len(rows) == len(out[0]), f"rank {q} checked {len(rows)} results, rank 0 {len(out[0])}")
        assert not self.failures, f"{len(self.failures)} checks failed on rank {rank}, the first:\n{self.failures[0]}"


def job(test_path: str, nranks: int, select: str = None, env: dict = None):
    """Run the GPU tests of ``test_path`` (``-k select``) as an ``nranks``-rank job on the GPUs there
    are; returns (exit code, [output of every rank])."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    test_file = os.path.relpath(os.path.abspath(test_path), REPO)
    args = ["-m", "pytest", test_file, "-q", "-rp", "-m", "gpu", "-p", "no:cacheprovider"]
    if select:
        args += ["-k", select]
    cwd = os.getcwd()
    os.chdir(REPO)
    try:
        with tempfile.TemporaryDirectory(prefix=f"mpi4jax-b200-job-{nranks}-") as logs:
            code, _ = launch(nranks, args, timeout=JOB_TIMEOUT_S, output_dir=logs,
                             env_extra={"MPI4JAX_B200_NESTED": "1", **(env or {})})
            outs = []
            for r in range(nranks):
                with open(os.path.join(logs, f"rank{r}.log")) as fh:
                    outs.append(fh.read())
    finally:
        os.chdir(cwd)
    return code, outs


def expect_passed(code, outs, nranks, tests) -> None:
    """Every test in ``tests`` reported PASSED (its CUDA variant) on every rank of the job."""
    for r, out in enumerate(outs):
        missing = [t for t in tests if not re.search(rf"^PASSED .*::{t}\[cuda\]", out, re.M)]
        assert code == 0 and not missing, \
            f"rank {r} of the {nranks}-rank job (exit code {code}), not passed: {missing}:\n{out[-4000:]}"


def needs_peers(reason: str, max_rank: int = None):
    """Decorator for a test that takes the ``device`` fixture and exchanges messages with other ranks.
    Inside a multi-rank job the test runs as written (ranks above ``max_rank`` skip); in a
    single-process run its CUDA variant is checked in a two-rank job and its CPU variant skips."""
    comm = MPI.COMM_WORLD
    size, rank = comm.Get_size(), comm.Get_rank()

    def deco(fn):
        if size > 1:
            if max_rank is not None and rank > max_rank:
                return pytest.mark.skip(reason=reason)(fn)
            return fn

        @functools.wraps(fn)
        def at_world_size_1(device, **fixtures):     # (other fixtures the test takes, e.g. capsys)
            if device.type != "cuda":
                pytest.skip(reason)
            _expect_passed_in_pair_job(fn)

        return at_world_size_1

    return deco
