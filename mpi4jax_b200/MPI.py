"""``mpi4jax_b200.MPI`` -- the slice of ``mpi4py.MPI`` that mpi4jax user code touches.

Reference-style programs port by changing one import::

    from mpi4py import MPI        ->   from mpi4jax_b200 import MPI
    import mpi4jax                ->   import mpi4jax_b200 as mpi4jax

``COMM_WORLD`` is created lazily on first attribute access (it initialises the
torch.distributed control plane from the launcher's RANK/WORLD_SIZE environment).
"""

from ._src.comm import (  # noqa: F401
    ANY_SOURCE,
    ANY_TAG,
    BAND,
    BOR,
    BXOR,
    BYTE,
    LAND,
    LOR,
    LXOR,
    MAX,
    MAXLOC,
    MIN,
    MINLOC,
    PROC_NULL,
    PROD,
    SUM,
    UNDEFINED,
    Comm,
    MPIError,
    Op,
    Status,
    get_world,
)

Intracomm = Comm


def __getattr__(name):
    if name == "COMM_WORLD":
        return get_world()
    raise AttributeError(f"module 'mpi4jax_b200.MPI' has no attribute {name!r}")


def Get_version():
    return (3, 1)


def Get_library_version():
    from ._src import native

    return f"mpi4jax_b200 NVLink transport ({native.NATIVE_ABI_INFO['version']})"


def Get_processor_name() -> str:
    import socket

    return socket.gethostname()


def Wtime() -> float:
    import time

    return time.perf_counter()


def Is_initialized() -> bool:
    import torch.distributed as dist

    return dist.is_initialized()


def Is_finalized() -> bool:
    return False
