"""The fused halo kernel exchanges with all eight neighbours in ONE phase, the reference does
four sequential message rounds (west, north, east, south; examples/shallow_water.py:172-264).
This test simulates both schemes for every rank of several process grids and checks that
every halo cell (corners and wall rows included) ends up bit-identical -- the property the
kernel's design relies on (csrc/b2_halo.cu header).  The kernel's own message geometry and
receive rules (csrc/b2_halo_geom.h), compiled for the host, are checked against both."""

import ctypes

import numpy as np
import pytest

from ._halo_sim import neighbors, new_exchange, ref_exchange
from ._swe_emu import HAVE_TOOLCHAIN, build

GRIDS = [(1, 1), (2, 1), (2, 2), (2, 3), (2, 4), (2, 8), (3, 1), (3, 2)]
KIND_CODE = {"h": 0, "u": 1, "v": 2}


def _blocks(rng, py, px, ny, nx, periodic_x):
    """Per-rank (ny, nx) blocks; without x periodicity the wall columns hold one global column each."""
    base = [rng.standard_normal((ny, nx)) for _ in range(py * px)]
    if not periodic_x:
        west, east = rng.standard_normal((2, py * (ny - 2) + 2))
        for r, b in enumerate(base):
            iy, ix = divmod(r, px)
            if ix == 0:
                b[:, 0] = west[iy * (ny - 2): iy * (ny - 2) + ny]
            if ix == px - 1:
                b[:, -1] = east[iy * (ny - 2): iy * (ny - 2) + ny]
    return base


@pytest.mark.parametrize("periodic_x", [True, False])
@pytest.mark.parametrize("grid", GRIDS)
@pytest.mark.parametrize("kind", ["h", "u", "v"])
def test_single_phase_equals_four_rounds(grid, kind, periodic_x):
    """With walls in x the corner halo cells next to an x wall are not exchanged by the single-phase
    scheme, while the four rounds copy the y neighbour's wall-column cell there; the two agree where
    the wall columns hold one global field, as in a model cut from a global array."""
    py, px = grid
    rng = np.random.default_rng(py * 10 + px)
    base = _blocks(rng, py, px, 6, 7, periodic_x)
    a = [b.copy() for b in base]
    b = [b.copy() for b in base]
    ref_exchange(a, py, px, kind, periodic_x)
    new_exchange(b, py, px, kind, periodic_x)
    for r, (x, y) in enumerate(zip(a, b)):
        assert np.array_equal(x, y), (r, np.argwhere(x != y).tolist())


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if not HAVE_TOOLCHAIN:
        pytest.skip("needs g++ and the CUDA headers")
    return build(tmp_path_factory, "halo_emu")


def _compiled_exchange(emu, arrs, kinds, py, px, periodic_x, order):
    """b2_k_halo_ll without the transport: every message of every rank read from the senders'
    pre-exchange arrays (``arrs``: per rank, a (nfields, ny, pitch) float32 array) and received with
    the kernel's receive rule, the sides in ``order`` (the kernel's are unordered), then each rank's
    wall pass."""
    nf, ny, pitch = arrs[0].shape
    nx = pitch - 1
    kind = (ctypes.c_int * nf)(*[KIND_CODE[k] for k in kinds])
    F = ctypes.c_void_p * nf
    fields = lambda a: F(*[a[f].ctypes.data for f in range(nf)])
    snap = [a.copy() for a in arrs]
    for r, a in enumerate(arrs):
        iy, ix = divmod(r, px)
        nb, dg = neighbors(iy, ix, py, px, periodic_x)
        has = {**nb, **dg}
        uwall, vwall = int(not periodic_x and ix == px - 1), int(iy == py - 1)
        for side in order:
            key = ("west", "east", "south", "north", "sw", "se", "nw", "ne")[side]
            if has[key] is not None:
                emu.emu_halo_deliver(ny, nx, pitch, nf, kind, side, int(nb["south"] is not None),
                                     int(nb["north"] is not None), uwall, vwall, fields(snap[has[key]]), fields(a))
        emu.emu_halo_wall_pass(ny, nx, pitch, nf, kind, *[int(nb[k] is not None) for k in ("west", "east", "south",
                                                                                             "north")],
                               uwall, vwall, fields(a))


_CASES = [(grid, (k,), (6, 7)) for grid in GRIDS for k in ("h", "u", "v")] + [
    (grid, kinds, (9, 7)) for grid in ((1, 1), (2, 3), (3, 2)) for kinds in (("v", "h", "u"),
                                                                             ("u", "v", "h", "h", "v", "u", "v", "u"))]


@pytest.mark.parametrize("periodic_x", [True, False])
@pytest.mark.parametrize("grid,kinds,shape", _CASES)
def test_compiled_one_layer_exchange_equals_both_models(emu, grid, kinds, shape, periodic_x):
    """The one-layer kernel's geometry, receive rule and wall pass, compiled for the host, on every rank
    of the grid: every cell equal bit for bit (NaN payloads and -0.0 included) to the single-phase
    model and the reference's four rounds; the row padding beyond nx is never written."""
    py, px = grid
    ny, nx = shape
    rng = np.random.default_rng(py * 10 + px + 100 * len(kinds))
    per_field = [_blocks(rng, py, px, ny, nx, periodic_x) for _ in kinds]
    arrs = []
    for r in range(py * px):
        a = np.full((len(kinds), ny, nx + 1), 7.5, np.float32)          # column nx: row padding
        for f in range(len(kinds)):
            a[f, :, :nx] = per_field[f][r]
        a[:, 1, 1] = -0.0                                               # special values ride along unchanged
        a.view(np.int32)[:, ny - 2, nx - 2] = 0x7FC01234                # a NaN with a payload
        arrs.append(a)
    want = [a.copy() for a in arrs]
    backwards = [a.copy() for a in arrs]
    _compiled_exchange(emu, arrs, kinds, py, px, periodic_x, range(8))
    _compiled_exchange(emu, backwards, kinds, py, px, periodic_x, range(7, -1, -1))
    for f, kind in enumerate(kinds):
        bits = [w[f, :, :nx].view(np.int32) for w in want]
        a = [b.copy() for b in bits]
        ref_exchange(a, py, px, kind, periodic_x)
        new_exchange(bits, py, px, kind, periodic_x)
        for r in range(py * px):
            got = arrs[r][f].view(np.int32)
            assert np.array_equal(got[:, :nx], bits[r]), (r, kind, np.argwhere(got[:, :nx] != bits[r]).tolist())
            assert np.array_equal(got[:, :nx], a[r]), (r, kind)
            assert (arrs[r][f, :, nx] == 7.5).all(), (r, kind)
            assert np.array_equal(backwards[r][f].view(np.int32), got), (r, kind)
