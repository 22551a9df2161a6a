"""Tile order of the persistent GEMM (csrc/b2_gemm_raster.h), compiled for the host: every order
is a bijection of the tile grid, the default is row-major, the banded order keeps the tiles in
flight inside a band of G rows."""

import ctypes
import os
import shutil
import subprocess

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++")


def _build(tmp_path, group):
    out = tmp_path / f"libraster{group}.so"
    cmd = ["g++", "-O1", "-std=c++17", "-shared", "-fPIC", f"-DB2_GEMM_RASTER_GROUP={group}", "-I",
           os.path.join(REPO, "csrc"), os.path.join(REPO, "tests", "native", "gemm_raster_emu.cpp"), "-o", str(out)]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    lib = ctypes.CDLL(str(out))
    assert lib.raster_group() == group
    return lib


def _order(lib, num_m, num_n):
    m, n = ctypes.c_int(), ctypes.c_int()
    out = []
    for t in range(num_m * num_n):
        lib.tile_coords(t, num_m, num_n, ctypes.byref(m), ctypes.byref(n))
        out.append((m.value, n.value))
    return out


@pytest.mark.parametrize("group", [0, 1, 4, 8, 16])
@pytest.mark.parametrize("grid", [(1, 1), (64, 32), (32, 16), (7, 5), (9, 32), (16, 3), (3, 64)])
def test_tile_order_is_a_bijection(tmp_path, group, grid):
    lib = _build(tmp_path, group)
    num_m, num_n = grid
    order = _order(lib, num_m, num_n)
    assert sorted(order) == [(m, n) for m in range(num_m) for n in range(num_n)]
    if group == 0:
        assert order == [(t // num_n, t % num_n) for t in range(num_m * num_n)]      # measured default
    else:
        # any `group * k` consecutive tiles stay inside one band of `group` rows (or cross one boundary)
        for start in range(0, len(order) - group, group):
            rows = {m // group for m, _ in order[start:start + group]}
            assert len(rows) <= 2
        # the 132 tiles in flight (one per H100 SM) stay within the bands they started in
        if num_m * num_n >= 132 and num_m >= group:
            bands = -(-132 // (group * num_n)) + 1
            assert len({m for m, _ in order[:132]}) <= group * bands
