"""The communication-avoiding shallow-water step as b2_swe_multistep_ca launches it, compiled for the
HOST (tests/native/swe_ca_bulk_emu.cpp): the one-pass bulk kernel with its lanes in lockstep, the frame
kernels with owner views and ping-pong storage, the deep exchange, on a process grid, against the
stand-alone kernels' pipeline, bit for bit."""

import ctypes
import os
import subprocess

import numpy as np
import pytest

from .test_swe_host_emulation import (  # noqa: F401  (pytestmark: needs g++ and the CUDA headers)
    CUDA_INC,
    REPO,
    _blocks,
    _ca_exchange,
    _ca_ext,
    _emulate,
    _params,
    _ptr,
    _setup,
    pytestmark,
)


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    out = tmp_path_factory.mktemp("swe_ca_bulk_emu") / "libswe_ca_bulk_emu.so"
    cmd = ["g++", "-O1", "-ffp-contract=off", "-std=c++17", "-shared", "-fPIC", "-I", os.path.join(REPO, "csrc"),
           "-I", CUDA_INC, os.path.join(REPO, "tests", "native", "swe_ca_bulk_emu.cpp"), "-o", str(out)]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    return ctypes.CDLL(str(out))


class EmuStep(ctypes.Structure):      # EmuStepPP (tests/native/swe_ca_bulk_emu.cpp): one rank's arrays for one step
    _fields_ = [(n, ctypes.c_void_p) for n in
                ("h", "u", "v", "du", "dv", "h_o", "u_o", "v_o", "du_o", "dv_o", "dh", "upf", "vpf")]


_PAIRS = ("h", "u", "v", "du", "dv")


def _emulate_ca(emu, model, PY, PX, nsteps, rows, reverse=0):
    """The launch sequence of b2_swe_multistep_ca on a process grid: per step the bulk kernel S and the
    frame chain A -> X -> D, which run concurrently.  h, u, v, du, dv are ping-pong pairs, dh is updated
    in place.  ``reverse`` walks every kernel's tasks (the bulk kernel's warps) backwards AND runs S after
    the frame chain instead of before it: the result may depend on neither.  (Messages are read before
    any rank scatters: all sends of a step come from h', u', v' frame cells, which no message writes.)"""
    from ._halo_sim import new_exchange

    ranks, ny, nx, pitch = _blocks(model, PY, PX)
    epitch = nx + 4
    for name, kind in (("h", "h"), ("u", "u"), ("v", "v")):
        new_exchange([r[name][:, :nx] for r in ranks], PY, PX, kind)
    for r in ranks:
        for n in _PAIRS:                                              # reset(): partners start as copies
            r[n + "1"] = r[n].copy()
        for n in ("hx", "upx", "vpx", "uppx", "vppx"):
            r[n] = np.full((ny + 4, epitch), np.nan, np.float32)     # NaN = never delivered / computed
        for n in ("upf", "vpf"):
            r[n] = np.full((ny, pitch), np.nan, np.float32)
    B = ctypes.byref
    _ca_exchange(emu, ranks, ("h", "u", "v"), ny, nx, pitch, epitch, PY, PX)       # b2_swe_ca_init
    for i, r in enumerate(ranks):
        p = _params(model, r, ny, nx, pitch, i // PX, PY, True)
        emu.emu_ca_init_ext(B(p), B(_ca_ext(r, epitch)), _ptr(r["u"]), _ptr(r["v"]))
    cur = ""
    for it in range(nsteps):
        nxt = "1" if cur == "" else ""
        ps = [_params(model, r, ny, nx, pitch, i // PX, PY, it == 0) for i, r in enumerate(ranks)]
        xs = [_ca_ext(r, epitch) for r in ranks]
        es = [EmuStep(**{n: r[n + cur].ctypes.data for n in _PAIRS},
                      **{n + "_o": r[n + nxt].ctypes.data for n in _PAIRS},
                      dh=r["dh"].ctypes.data, upf=r["upf"].ctypes.data, vpf=r["vpf"].ctypes.data)
              for r in ranks]
        if not reverse:
            for p, e in zip(ps, es):
                emu.emu_ca_bulk_step(B(p), B(e), rows, reverse)
        for p, x, e in zip(ps, xs, es):
            emu.emu_pp_tend_frame(B(p), B(x), B(e), reverse)
        _ca_exchange(emu, ranks, ("h" + nxt, "upf", "vpf"), ny, nx, pitch, epitch, PY, PX)
        for p, x, e in zip(ps, xs, es):
            emu.emu_pp_fric_frame(B(p), B(x), B(e), reverse)
        if reverse:
            for p, e in zip(ps, es):
                emu.emu_ca_bulk_step(B(p), B(e), rows, reverse)
        cur = nxt
    return [{k: r[k + (cur if k in _PAIRS else "")][:, :nx] for k in ("h", "u", "v", "dh", "du", "dv")}
            for r in ranks]


@pytest.mark.parametrize("grid,block,rows", [
    ((1, 1), (24, 48), 5), ((2, 1), (24, 48), 5), ((1, 2), (24, 48), 5), ((2, 2), (24, 48), 5),
    ((3, 2), (24, 48), 5), ((2, 4), (24, 48), 5),
    ((1, 1), (24, 48), 64),                 # one segment covers the bulk
    ((2, 1), (40, 280), 7),                 # several warp strips per row, a partial last strip
    ((1, 2), (33, 140), 16),                # odd bulk height: a short last segment
])
def test_emulated_one_pass_ca_pipeline_is_bit_identical_to_the_standalone_pipeline(emu, grid, block, rows):
    """One deep exchange per step + local recomputation (frame kernels with owner views, one-pass bulk
    kernel) vs the three exchanges of b2_swe_multistep, same decomposition: the same bits, walls, periodic
    wrap and the reference's stale u / v halos included, in any order of the bulk kernel's warps."""
    from mpi4jax_b200.models import ShallowWaterConfig, ShallowWaterModel

    PY, PX = grid
    model = ShallowWaterModel(ShallowWaterConfig(nx=block[1] * PX, ny=block[0] * PY), device="cpu", backend="ops")
    nsteps = 5                                                  # odd: the partners hold the result
    a = _emulate(emu, model, PY, PX, nsteps)
    b = _emulate_ca(emu, model, PY, PX, nsteps, rows)
    c = _emulate_ca(emu, model, PY, PX, nsteps, rows, reverse=1)
    for ra, rb, rc in zip(a, b, c):
        for name in ra:
            assert np.isfinite(rb[name][1:-1, 1:-1]).all(), (grid, name)
            assert np.array_equal(ra[name][1:-1, 1:-1], rb[name][1:-1, 1:-1]), (grid, name)
            assert np.array_equal(rb[name][1:-1, 1:-1], rc[name][1:-1, 1:-1]), (grid, name, "task order")
            # the main arrays' halos as well (h fresh; u, v stale by the friction step)
            if name in ("h", "u", "v"):
                assert np.array_equal(ra[name], rb[name]), (grid, name, "halo")


@pytest.mark.parametrize("shape,rows", [((16, 24), 16), ((26, 50), 5), ((17, 29), 3), ((140, 33), 16),
                                        ((31, 300), 7), ((200, 530), 64), ((200, 530), 13)])
def test_bulk_step_stores_every_bulk_cell_once(emu, shape, rows):
    """swe_ca_bulk_step's segments and warp strips cover the bulk (rows [4, ny-5], columns [4, cb1))
    exactly once, whatever the rows per segment."""
    ny, nx = shape
    p, *_ = _setup(ny, nx, False, 0, 0)
    counts = np.zeros((ny, nx), np.int32)
    emu.emu_ca_bulk_step_counts(ctypes.byref(p), rows, counts.ctypes.data_as(ctypes.POINTER(ctypes.c_int)))
    cb1 = (nx - 4) // 4 * 4
    want = np.zeros_like(counts)
    want[4:ny - 4, 4:cb1] = 1
    assert np.array_equal(counts, want)
