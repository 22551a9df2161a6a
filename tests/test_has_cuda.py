def test_has_cuda_support():
    from mpi4jax_b200 import has_cuda_support

    assert isinstance(has_cuda_support(), bool)
    assert has_cuda_support(), "the native sm_90a library must be built (python __graft_entry__.py)"


def test_has_sycl_support():
    from mpi4jax_b200 import has_sycl_support

    assert has_sycl_support() is False


def test_native_abi_info():
    """Counterpart of the reference's MPI_ABI_INFO test (test_common.py:170-197)."""
    from mpi4jax_b200._src.native import NATIVE_ABI_INFO

    for key in ("library", "loaded", "version", "arch", "sizeof_status_record", "sizeof_halo_desc"):
        assert key in NATIVE_ABI_INFO
    assert NATIVE_ABI_INFO["arch"] == "sm_90a"
    assert NATIVE_ABI_INFO["sizeof_status_record"] == 24
    assert NATIVE_ABI_INFO["loaded"]
    native, python = NATIVE_ABI_INFO["native"], NATIVE_ABI_INFO["python"]
    for key, val in python.items():
        assert native[key] == val, key


def test_abi_check_detects_stale_library(monkeypatch):
    """A library whose struct layout / ABI version differs from the ctypes mirrors is rejected at
    import (reference: xla_bridge/__init__.py:23-89, tests test_common.py:170-224)."""
    from mpi4jax_b200._src import native

    assert native._abi_mismatch(native.lib) == ""
    monkeypatch.setattr(native, "ABI_VERSION", native.ABI_VERSION + 1)
    msg = native._abi_mismatch(native.lib)
    assert "abi_version" in msg and "!=" in msg


def test_abi_check_raises_and_can_be_skipped(tmp_path):
    import os
    import subprocess
    import sys

    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    script = tmp_path / "abi.py"
    script.write_text(
        "import ctypes, sys\n"
        f"sys.path.insert(0, {repo!r})\n"
        "real = ctypes.CDLL\n"
        "class Fake:\n"
        "    def __new__(cls, path, *a, **k):\n"
        "        if 'libb2mpi' not in str(path): return real(path, *a, **k)\n"
        "        self = object.__new__(cls); self._h = real(path); return self\n"
        "    def __getattr__(self, name):\n"
        "        fn = getattr(self._h, name)\n"
        "        if name != 'b2_abi_info':\n"
        "            return fn\n"
        "        def lying(buf, n):\n"
        "            k = fn(buf, n); buf[2] += 8; return k\n"     # pretend B2HaloDesc grew
        "        return lying\n"
        "ctypes.CDLL = Fake\n"
        "from mpi4jax_b200._src import native\n"
        "print('loaded', native.HAS_CUDA_EXT)\n")
    env = {k: v for k, v in os.environ.items() if not k.startswith("MPI4JAX_B200_SKIP")}
    res = subprocess.run([sys.executable, str(script)], capture_output=True, text=True, env=env, timeout=120)
    assert res.returncode != 0
    assert "does not match this Python package" in res.stderr and "sizeof_halo_desc" in res.stderr
    env["MPI4JAX_B200_SKIP_ABI_CHECK"] = "1"
    res = subprocess.run([sys.executable, str(script)], capture_output=True, text=True, env=env, timeout=120)
    assert res.returncode == 0, res.stderr
    assert "loaded True" in res.stdout
