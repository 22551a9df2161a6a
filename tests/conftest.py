"""pytest configuration.

Test strategy (mirrors the reference, SURVEY.md section 4): the same test files run
 * in-process at world size 1 (collectives degenerate to self-communication but still go
   through the full op -> backend -> transport stack), and
 * once per rank under ``python -m mpi4jax_b200.run -n 2 -m pytest ...`` (tests/test_multirank.py
   spawns that job, as the reference's CI runs ``mpirun -np 2 pytest .``).
Every test that takes the ``device`` fixture runs on CPU (gloo backend) and, marked ``gpu``,
on CUDA (native sm_90a kernels).  ``pytest -m "not gpu"`` needs no GPU.
"""

import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def pytest_report_header(config):
    import torch

    from mpi4jax_b200 import MPI, has_cuda_support

    comm = MPI.COMM_WORLD
    return (
        f"mpi4jax_b200: rank {comm.Get_rank()} of {comm.Get_size()}, torch {torch.__version__}, "
        f"cuda available: {torch.cuda.is_available()}, native ext: {has_cuda_support()}"
    )


@pytest.fixture(params=["cpu", pytest.param("cuda", marks=pytest.mark.gpu)])
def device(request):
    import torch

    if request.param == "cuda":
        if not torch.cuda.is_available():
            pytest.skip("no CUDA device")
        from mpi4jax_b200 import MPI

        return MPI.COMM_WORLD.device
    return torch.device("cpu")


@pytest.fixture(autouse=True)
def _flush_after_test():
    yield
    import mpi4jax_b200

    mpi4jax_b200.flush()
