"""Host-framework version / capability gate.

The reference gates on the JAX version (/root/reference/mpi4jax/_src/jax_compat.py:
12-48, pinned in _latest_jax_version.txt).  The host framework here is PyTorch
(streams, CUDA graphs, autograd, ``torch.func``); this module gates on the torch
version and probes the GPU capabilities the native core needs (sm_90, VMM fd
handles, multicast).
"""

from __future__ import annotations

import os
import re
import warnings

MIN_TORCH = "2.4.0"


def _read_latest_tested() -> str:
    """Pinned in ``_latest_torch_version.txt`` (bumped by dependabot, like the reference's
    ``_latest_jax_version.txt``)."""
    here = os.path.dirname(os.path.abspath(__file__))
    try:
        with open(os.path.join(here, "_latest_torch_version.txt")) as f:
            for line in f:
                line = line.strip()
                if line.startswith("torch=="):
                    return line.split("==", 1)[1]
    except OSError:  # pragma: no cover
        pass
    return "2.11.0"


LATEST_TESTED_TORCH = _read_latest_tested()


def versiontuple(verstr: str) -> tuple:
    """``"2.11.0+cu128" -> (2, 11, 0)``; non-numeric suffixes of a component are dropped."""
    out = []
    for part in verstr.split("+")[0].split(".")[:3]:
        m = re.match(r"\d+", part)
        if not m:
            break
        out.append(int(m.group(0)))
    while len(out) < 3:
        out.append(0)
    return tuple(out)


def check_torch_version() -> None:
    import torch

    have = versiontuple(torch.__version__)
    if have < versiontuple(MIN_TORCH):
        raise RuntimeError(
            f"mpi4jax_b200 needs torch>={MIN_TORCH}, found {torch.__version__}"
        )
    if have > versiontuple(LATEST_TESTED_TORCH) and not os.environ.get(
        "MPI4JAX_B200_NO_WARN_TORCH_VERSION"
    ):
        warnings.warn(
            f"The torch version {torch.__version__} is newer than the latest version "
            f"mpi4jax_b200 was tested with ({LATEST_TESTED_TORCH}). Set "
            "MPI4JAX_B200_NO_WARN_TORCH_VERSION=1 to silence this warning."
        )


def device_capabilities(device: int = 0) -> dict:
    """Capabilities relevant to the native transport (all False without a GPU)."""
    import torch

    caps = {"cuda": False, "sm": None, "sm_90": False, "vmm": False, "multicast": False}
    if not torch.cuda.is_available():
        return caps
    major, minor = torch.cuda.get_device_capability(device)
    caps.update(cuda=True, sm=(major, minor), sm_90=((major, minor) == (9, 0)))
    try:
        from . import native

        if native.HAS_CUDA_EXT:
            native.lib.b2_init(device)
            caps["vmm"] = bool(native.lib.b2_vmm_supported(device))
            caps["multicast"] = bool(native.lib.b2_multicast_supported(device))
    except Exception:  # pragma: no cover
        pass
    return caps
