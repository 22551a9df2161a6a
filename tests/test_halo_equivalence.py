"""The fused halo kernel exchanges with all eight neighbours in ONE phase, the reference does
four sequential message rounds (west, north, east, south; examples/shallow_water.py:172-264).
This test simulates both schemes for every rank of several process grids and checks that
every halo cell (corners and wall rows included) ends up bit-identical -- the property the
kernel's design relies on (csrc/b2_halo.cu header)."""

import numpy as np
import pytest

from ._halo_sim import new_exchange, ref_exchange


@pytest.mark.parametrize("periodic_x", [True, False])
@pytest.mark.parametrize("grid", [(1, 1), (2, 1), (2, 2), (2, 3), (2, 4), (2, 8), (3, 1), (3, 2)])
@pytest.mark.parametrize("kind", ["h", "u", "v"])
def test_single_phase_equals_four_rounds(grid, kind, periodic_x):
    """With walls in x the corner halo cells next to an x wall are not exchanged by the single-phase
    scheme, while the four rounds copy the y neighbour's wall-column cell there; the two agree where
    the wall columns hold one global field, as in a model cut from a global array."""
    py, px = grid
    rng = np.random.default_rng(py * 10 + px)
    base = [rng.standard_normal((6, 7)) for _ in range(py * px)]
    if not periodic_x:
        west, east = rng.standard_normal((2, py * 4 + 2))
        for r, b in enumerate(base):
            iy, ix = divmod(r, px)
            if ix == 0:
                b[:, 0] = west[iy * 4: iy * 4 + 6]
            if ix == px - 1:
                b[:, -1] = east[iy * 4: iy * 4 + 6]
    a = [b.copy() for b in base]
    b = [b.copy() for b in base]
    ref_exchange(a, py, px, kind, periodic_x)
    new_exchange(b, py, px, kind, periodic_x)
    for r, (x, y) in enumerate(zip(a, b)):
        assert np.array_equal(x, y), (r, np.argwhere(x != y).tolist())
