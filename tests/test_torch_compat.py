"""The host-framework version gate (`_src/torch_compat.py`): version parsing table, too-old error,
too-new warning and its silencer -- the scenarios of /root/reference/tests/test_jax_compat.py for torch."""

import importlib
import warnings

import pytest


@pytest.mark.parametrize("verstr,expected", [
    ("2.11.0", (2, 11, 0)), ("2.11.0+cu128", (2, 11, 0)), ("2.4", (2, 4, 0)),
    ("2.5.0a0+git1234", (2, 5, 0)), ("2.6.0.dev20250101", (2, 6, 0)), ("3", (3, 0, 0)),
    ("2.10.1rc2", (2, 10, 1)),
])
def test_versiontuple(verstr, expected):
    from mpi4jax_b200._src.torch_compat import versiontuple

    assert versiontuple(verstr) == expected


def test_version_warning(monkeypatch):
    import torch

    from mpi4jax_b200._src import torch_compat

    monkeypatch.setattr(torch, "__version__", "99.0.0")
    monkeypatch.delenv("MPI4JAX_B200_NO_WARN_TORCH_VERSION", raising=False)
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        torch_compat.check_torch_version()
    assert any("newer than the latest version" in str(x.message) for x in w)
    monkeypatch.setenv("MPI4JAX_B200_NO_WARN_TORCH_VERSION", "1")
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        torch_compat.check_torch_version()
    assert not w
    monkeypatch.setattr(torch, "__version__", "1.13.0")
    with pytest.raises(RuntimeError):
        torch_compat.check_torch_version()


def test_device_capabilities_keys():
    from mpi4jax_b200._src.torch_compat import device_capabilities

    caps = device_capabilities()
    assert set(caps) == {"cuda", "sm", "sm_90", "vmm", "multicast"}
