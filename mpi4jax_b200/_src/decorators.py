"""Environment flags and extension guards.

Counterpart of /root/reference/mpi4jax/_src/decorators.py:1-152.  The reference
parses ``MPI4JAX_USE_CUDA_MPI`` to choose between host-staged and CUDA-aware MPI
at first lowering; there is no host-staged path here (the transport is always
peer-mapped HBM), so the flags that remain are:

=================================  ==========================================================
``MPI4JAX_B200_DEBUG``             enable the per-call debug log (also honours ``MPI4JAX_DEBUG``)
``MPI4JAX_B200_DEVICE``            ``cuda`` / ``cpu``: where scalars and numpy inputs are placed
``MPI4JAX_B200_HEAP``              ``vmm`` (default, enables NVLS) or ``ipc`` (cudaIpc fallback)
``MPI4JAX_B200_NVLS``              falsy -> do not create multicast objects
``MPI4JAX_B200_TIMEOUT``           device watchdog in seconds (default 60)
``MPI4JAX_B200_P2P_SLOT_BYTES``    bytes per p2p ring slot (default 16 MiB, ring capped at 256 MiB)
``MPI4JAX_B200_ABORT_ON_ERROR``    falsy -> raise ``MPIError`` instead of aborting the process
``MPI4JAX_USE_CUDA_MPI``           accepted for compatibility; only emits a note when falsy
=================================  ==========================================================
"""

from __future__ import annotations

import functools
import os
import warnings

_TRUTHY = ("true", "1", "on")
_FALSY = ("false", "0", "off")


def _is_truthy(val: str) -> bool:
    return val.lower() in _TRUTHY


def _is_falsy(val: str) -> bool:
    return val.lower() in _FALSY


def env_flag(name: str, default: bool) -> bool:
    """Parse a boolean environment variable; unknown spellings raise."""
    raw = os.environ.get(name)
    if raw is None or raw == "":
        return default
    if _is_truthy(raw):
        return True
    if _is_falsy(raw):
        return False
    raise RuntimeError(
        f"Invalid value for {name}: {raw!r} (use one of {_TRUTHY + _FALSY})"
    )


def env_int(name: str, default: int) -> int:
    raw = os.environ.get(name)
    return default if raw in (None, "") else int(float(raw))


def env_float(name: str, default: float) -> float:
    raw = os.environ.get(name)
    return default if raw in (None, "") else float(raw)


def ensure_cuda_ext(fn=None):
    """Raise ImportError if the native sm_90a library is unavailable.

    Usable as a plain call or as a decorator (reference: decorators.py:10-17).
    """
    from . import native

    def check():
        if not native.HAS_CUDA_EXT:
            raise ImportError(
                "The mpi4jax_b200 native CUDA library could not be loaded "
                f"({native.CUDA_EXT_ERROR}). Build it with "
                "`python -m mpi4jax_b200._src.native.build`."
            )

    if fn is None:
        check()
        return None

    @functools.wraps(fn)
    def wrapped(*args, **kwargs):
        check()
        return fn(*args, **kwargs)

    return wrapped


def ensure_xpu_ext(fn=None):
    """The reference ships an Intel XPU bridge (decorators.py:20-27); H100 has none."""

    def check():
        raise ImportError(
            "mpi4jax_b200 targets NVIDIA H100 (sm_90a) only; there is no XPU/SYCL extension."
        )

    if fn is None:
        check()
    return fn


_cuda_mpi_note_done = False


def setup_cuda_mpi() -> None:
    """One-time handling of the reference's ``MPI4JAX_USE_CUDA_MPI`` switch.

    The reference copies every GPU buffer through pageable host memory unless this
    is truthy (decorators.py:38-64).  Here device buffers travel GPU->GPU over NVLink by
    default; a falsy value selects the host-staged transport (``backends/host_staged.py``,
    see ``backends/transport.py``) and earns a warning, because on one node that is never
    what you want.
    """
    global _cuda_mpi_note_done
    if _cuda_mpi_note_done:
        return
    _cuda_mpi_note_done = True
    raw = os.environ.get("MPI4JAX_USE_CUDA_MPI")
    if raw is not None and _is_falsy(raw):
        warnings.warn(
            "MPI4JAX_USE_CUDA_MPI=0 requests host-staged transfers: CUDA tensors will be copied "
            "through host memory instead of moving directly over NVLink (unset it, or set "
            "MPI4JAX_B200_TRANSPORT=native, for the fast path)."
        )
