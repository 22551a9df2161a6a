"""The ring launch of the pair schedule as one launch (csrc/b2_swe_ca.cu: swe_ca_bulk_step over a table of
the four ring windows, blockIdx.y picking the window), emulated on the host with the kernels' own source
(tests/native/swe_ring_emu.cpp) inside the whole pair schedule, against the stand-alone kernels, bit for
bit."""

import ctypes
import os
import subprocess

import numpy as np
import pytest

from ._swe_emu import CUDA_INC, HAVE_TOOLCHAIN, REPO, emulate
from .test_swe_pair_emulation import _emulate_pairs

pytestmark = pytest.mark.skipif(not HAVE_TOOLCHAIN, reason="needs g++ and the CUDA headers")


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    out = tmp_path_factory.mktemp("swe_ring_emu") / "libswe_ring_emu.so"
    cmd = ["g++", "-O1", "-ffp-contract=off", "-std=c++17", "-shared", "-fPIC", "-I", os.path.join(REPO, "csrc"),
           "-I", CUDA_INC, os.path.join(REPO, "tests", "native", "swe_ring_emu.cpp"), "-o", str(out)]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    return ctypes.CDLL(str(out))


class _OneRingLaunch:
    """The emulation library with the ring launch as the device now runs it: the first of the four
    ring windows runs all four through ``emu_ca_ring`` (one launch, blockIdx.y the window), the other
    three are already done."""

    def __init__(self, lib):
        self._lib = lib

    def __getattr__(self, name):
        return getattr(self._lib, name)

    def emu_ca_window(self, p, e, w, rows, reverse):
        if w == 2:
            self._lib.emu_ca_ring(p, e, reverse)
        elif w not in (3, 4, 5):
            self._lib.emu_ca_window(p, e, w, rows, reverse)


@pytest.mark.parametrize("nsteps", [3, 4, 6])
@pytest.mark.parametrize("grid,block,rows", [
    ((1, 1), (24, 48), 5),
    ((2, 2), (24, 48), 5),
    ((1, 1), (40, 280), 7),                 # several strips per row of the north / south windows
    ((1, 2), (33, 300), 16),
    ((2, 1), (14, 48), 5),                  # ny just above the pair threshold: one inner row
    ((1, 1), (15, 140), 3),
    ((2, 2), (18, 39), 5),                  # nx % 4 == 1
])
def test_one_ring_launch_is_bit_identical_to_the_standalone_pipeline(emu, grid, block, rows, nsteps):
    """Both task orders: the warps of all four windows forwards, then backwards."""
    from mpi4jax_b200.models import ShallowWaterConfig, ShallowWaterModel

    PY, PX = grid
    model = ShallowWaterModel(ShallowWaterConfig(nx=block[1] * PX, ny=block[0] * PY), device="cpu", backend="ops")
    one = _OneRingLaunch(emu)
    a = emulate(emu, model, PY, PX, nsteps)
    b = _emulate_pairs(one, model, PY, PX, nsteps, rows)
    c = _emulate_pairs(one, model, PY, PX, nsteps, rows, reverse=1)
    for ra, rb, rc in zip(a, b, c):
        for name in ra:
            assert np.isfinite(rb[name][1:-1, 1:-1]).all(), (grid, name)
            assert np.array_equal(ra[name][1:-1, 1:-1], rb[name][1:-1, 1:-1]), (grid, name)
            assert np.array_equal(rb[name][1:-1, 1:-1], rc[name][1:-1, 1:-1]), (grid, name, "task order")
            if name in ("h", "u", "v"):
                assert np.array_equal(ra[name], rb[name]), (grid, name, "halo")
