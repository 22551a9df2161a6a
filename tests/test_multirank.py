"""Runs the distributed test files under the launcher with 2 (and 3) CPU ranks -- the
equivalent of the reference CI's ``mpirun -np 2 pytest .``
(/root/reference/.github/workflows/mpi-tests.yml:85-93).  With >= 2 GPUs the same is done
on the native path."""

import os
import sys

import pytest
import torch

from mpi4jax_b200 import MPI
from mpi4jax_b200.run import launch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SUITE = ["tests/collective_ops", "tests/test_transforms.py", "tests/test_models.py",
         "tests/test_examples.py", "tests/test_jit.py", "tests/test_common.py", "tests/test_gemm.py",
         "tests/test_compile.py", "tests/test_transport.py", "tests/test_object_api.py",
         "tests/test_more_examples.py", "tests/test_extensions.py", "tests/test_coresidency.py",
         "tests/test_shared_adjoints.py"]

inside_job = MPI.COMM_WORLD.Get_size() > 1 or "MPI4JAX_B200_NESTED" in os.environ


def _run(nprocs, marker, cpu, timeout):
    args = ["-m", "pytest", *SUITE, "-x", "-q", "-m", marker, "-p", "no:cacheprovider"]
    cwd = os.getcwd()
    os.chdir(REPO)
    try:
        code, outs = launch(nprocs, args, cpu=cpu, timeout=timeout, capture=True,
                            env_extra={"MPI4JAX_B200_NESTED": "1"})
    finally:
        os.chdir(cwd)
    assert code == 0, "\n".join(o[-3000:] for o in outs)
    for o in outs:
        assert " passed" in o


@pytest.mark.skipif(inside_job, reason="already inside a multi-rank job")
@pytest.mark.parametrize("nprocs", [2, 3])
def test_suite_multirank_cpu(nprocs):
    _run(nprocs, "not gpu", cpu=True, timeout=900)


@pytest.mark.gpu
@pytest.mark.skipif(inside_job, reason="already inside a multi-rank job")
def test_suite_multirank_gpu():
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs at least 2 GPUs")
    _run(min(n, 8) if min(n, 8) in (2, 4, 6, 8) else 2, "gpu", cpu=False, timeout=1200)
