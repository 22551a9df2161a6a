"""Point-to-point tests need a peer rank.  In a single-process run their CPU variants skip (the
multi-rank CPU job of tests/test_multirank.py runs them), but on a GPU machine the CUDA variants
still run: the test file is run once as a two-rank job on the GPUs there are (both ranks share the
GPU when there is only one), and each test passes when it passed on both ranks of that job."""

import functools
import inspect
import os
import re
import tempfile

import pytest

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
