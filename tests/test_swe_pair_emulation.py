"""The pair schedule of the communication-avoiding shallow-water step (csrc/b2_swe_ca.cu: swe_ca_bulk_pair
advances the bulk two steps per pass, the ring launches and the frame kernels follow) executed on the
host with the kernels' own source (tests/native/swe_pair_emu.cpp), against the stand-alone kernels, bit
for bit, and the cells each launch stores."""

import ctypes
import os
import subprocess

import numpy as np
import pytest

from ._swe_emu import CUDA_INC, HAVE_TOOLCHAIN, REPO, blocks, emulate, params
from .test_swe_host_emulation import _ca_exchange, _ca_ext

pytestmark = pytest.mark.skipif(not HAVE_TOOLCHAIN, reason="needs g++ and the CUDA headers")

_SETS = ("h", "u", "v", "du", "dv")        # three buffer sets; dh: three buffers of its own
_FIELDS = ("h", "u", "v", "dh", "du", "dv")


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    out = tmp_path_factory.mktemp("swe_pair_emu") / "libswe_pair_emu.so"
    cmd = ["g++", "-O1", "-ffp-contract=off", "-std=c++17", "-shared", "-fPIC", "-I", os.path.join(REPO, "csrc"),
           "-I", CUDA_INC, os.path.join(REPO, "tests", "native", "swe_pair_emu.cpp"), "-o", str(out)]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    return ctypes.CDLL(str(out))


class EmuIO(ctypes.Structure):      # EmuIO (tests/native/swe_pair_emu.cpp)
    _fields_ = [(n, ctypes.c_void_p) for n in
                ("h", "u", "v", "du", "dv", "h_o", "u_o", "v_o", "du_o", "dv_o", "dh_src", "dh", "upf", "vpf")]


def _key(name, k):
    return name + ("" if k == 0 else str(k))


def _io(r, i, o, di, do):
    """sets i -> o; dh from buffer di (None: in place) to buffer do"""
    return EmuIO(**{n: r[_key(n, i)].ctypes.data for n in _SETS},
                 **{n + "_o": r[_key(n, o)].ctypes.data for n in _SETS},
                 dh_src=None if di is None else r[_key("dh", di)].ctypes.data, dh=r[_key("dh", do)].ctypes.data,
                 upf=r["upf"].ctypes.data, vpf=r["vpf"].ctypes.data)


def _emulate_pairs(emu, model, PY, PX, nsteps, rows, reverse=0):
    """b2_swe_multistep_ca's launches: the Euler step and an odd step left over on the one-step schedule,
    pairs of steps as S2 next to A X D (t), then the ring launch next to A X D (t+1); three buffer sets,
    dh updated in place by a one-step launch and moved with a pair, each launch's output buffers chosen
    as b2_swe_multistep_ca does.
    ``reverse`` walks every launch's warps / tasks backwards and runs each bulk launch after the frame
    chain it runs next to."""
    from ._halo_sim import new_exchange

    ranks, ny, nx, pitch = blocks(model, PY, PX)
    epitch = nx + 4
    for name in ("h", "u", "v"):
        new_exchange([r[name][:, :nx] for r in ranks], PY, PX, name)
    for r in ranks:
        for n in _FIELDS:                                             # reset(): the other sets start as copies
            for k in (1, 2):
                r[_key(n, k)] = r[n].copy()
        for n in ("hx", "upx", "vpx", "uppx", "vppx"):
            r[n] = np.full((ny + 4, epitch), np.nan, np.float32)
        for n in ("upf", "vpf"):
            r[n] = np.full((ny, pitch), np.nan, np.float32)
    B = ctypes.byref
    _ca_exchange(emu, ranks, ("h", "u", "v"), ny, nx, pitch, epitch, PY, PX)
    for i, r in enumerate(ranks):
        p = params(model, r, ny, nx, pitch, i // PX, PY, True)
        emu.emu_ca_init_ext(B(p), B(_ca_ext(r, epitch)), r["u"].ctypes.data_as(ctypes.c_void_p),
                            r["v"].ctypes.data_as(ctypes.c_void_p))

    def frame(ps, ios, out):
        xs = [_ca_ext(r, epitch) for r in ranks]
        for p, x, e in zip(ps, xs, ios):
            emu.emu_ca_tend_frame_io(B(p), B(x), B(e), reverse)
        _ca_exchange(emu, ranks, (_key("h", out), "upf", "vpf"), ny, nx, pitch, epitch, PY, PX)
        for p, x, e in zip(ps, xs, ios):
            emu.emu_ca_fric_frame_io(B(p), B(x), B(e), reverse)

    def both(bulk, fr):
        (fr(), bulk()) if reverse else (bulk(), fr())

    pairs = emu.emu_ca_pairs(B(params(model, ranks[0], ny, nx, pitch, 0, PY, False)))
    npairs = (nsteps - 1) // 2 if pairs else 0
    moves = nsteps - npairs

    def target(mv, n, cur):           # each launch's output buffers: the last move ends in the home ones
        if mv == n - 1 and cur != 0:
            return 0
        return (2 if cur == 1 else 1) if mv == n - 2 else (cur + 1) % 3

    cur, dc, it, mv, pairs_run = 0, 0, 0, 0, 0
    while it < nsteps:
        ps = [params(model, r, ny, nx, pitch, i // PX, PY, it == 0) for i, r in enumerate(ranks)]
        pair = pairs and it > 0 and nsteps - it >= 2
        third = target(mv, moves, cur)
        nxt = 3 - cur - third if pair else third
        mv += 1
        if not pair:
            io1 = [_io(r, cur, nxt, None, dc) for r in ranks]
            both(lambda: [emu.emu_ca_window(B(p), B(e), 0, rows, reverse) for p, e in zip(ps, io1)],
                 lambda: frame(ps, io1, nxt))
            cur, it = nxt, it + 1
            continue
        dm = target(pairs_run, npairs, dc)
        dn = 3 - dc - dm
        io1 = [_io(r, cur, nxt, dc, dn) for r in ranks]
        io2 = [_io(r, nxt, third, None, dm) for r in ranks]             # (step 2 reads the ring)
        io3 = [_io(r, nxt, third, dn, dm) for r in ranks]
        both(lambda: [emu.emu_ca_pair(B(p), B(a), B(b), rows, reverse) for p, a, b in zip(ps, io1, io2)],
             lambda: frame(ps, io1, nxt))
        both(lambda: [emu.emu_ca_window(B(p), B(e), w, 2, reverse) for p, e in zip(ps, io3) for w in (2, 3, 4, 5)],
             lambda: frame(ps, io3, third))
        cur, dc, it, pairs_run = third, dm, it + 2, pairs_run + 1
    assert pairs_run == npairs and (cur == 0) == (moves > 1) and (dc == 0) == (npairs != 1)
    return [{k: r[_key(k, dc if k == "dh" else cur)][:, :nx] for k in _FIELDS} for r in ranks]


@pytest.mark.parametrize("nsteps", range(1, 8))
@pytest.mark.parametrize("grid,block,rows", [
    ((1, 1), (24, 48), 5), ((2, 1), (24, 48), 5), ((1, 2), (24, 48), 5), ((2, 2), (24, 48), 5),
    ((3, 2), (24, 48), 5), ((2, 4), (24, 48), 5),
    ((1, 1), (24, 48), 64),                 # one segment covers the inner bulk
    ((2, 1), (40, 280), 7),                 # several strips per row, a partial last strip
    ((1, 2), (33, 140), 16),                # odd inner height: a short last segment
    ((2, 2), (18, 39), 5),                  # nx % 4 == 1
    ((1, 1), (14, 48), 5),                  # the smallest block with an inner bulk: one inner row
])
def test_emulated_pair_schedule_is_bit_identical_to_the_standalone_pipeline(emu, grid, block, rows, nsteps):
    """Step counts 1-7 (Euler step, pairs, an odd step left over, every rotation of the three buffer
    sets), in both task orders: the same bits as the stand-alone kernels, halos included."""
    from mpi4jax_b200.models import ShallowWaterConfig, ShallowWaterModel

    PY, PX = grid
    model = ShallowWaterModel(ShallowWaterConfig(nx=block[1] * PX, ny=block[0] * PY), device="cpu", backend="ops")
    a = emulate(emu, model, PY, PX, nsteps)
    b = _emulate_pairs(emu, model, PY, PX, nsteps, rows)
    c = _emulate_pairs(emu, model, PY, PX, nsteps, rows, reverse=1)
    for ra, rb, rc in zip(a, b, c):
        for name in ra:
            assert np.isfinite(rb[name][1:-1, 1:-1]).all(), (grid, name)
            assert np.array_equal(ra[name][1:-1, 1:-1], rb[name][1:-1, 1:-1]), (grid, name)
            assert np.array_equal(rb[name][1:-1, 1:-1], rc[name][1:-1, 1:-1]), (grid, name, "task order")
            if name in ("h", "u", "v"):
                assert np.array_equal(ra[name], rb[name]), (grid, name, "halo")


@pytest.mark.parametrize("shape,rows", [((16, 24), 16), ((26, 50), 5), ((17, 29), 3), ((140, 33), 16),
                                        ((31, 300), 7), ((200, 530), 64), ((200, 530), 13)])
def test_pair_schedule_partitions_the_bulk(emu, shape, rows):
    """State t+2: S2's step 2 and the ring windows store every bulk cell exactly once.  State t+1: S2's
    step 1 stores each cell at most once, and every bulk cell within 6 rows of the bulk's south edge, 7
    of its north edge or 2 groups of its sides (what the ring launch and kernel A of step t+1 read)."""
    ny, nx = shape
    p = native_params(ny, nx)
    if not emu.emu_ca_pairs(ctypes.byref(p)):
        pytest.skip("no inner bulk")
    m1, m2 = np.zeros((ny, nx), np.int32), np.zeros((ny, nx), np.int32)
    P = ctypes.POINTER(ctypes.c_int)
    emu.emu_ca_pair_marks(ctypes.byref(p), rows, m1.ctypes.data_as(P), m2.ctypes.data_as(P))
    cb1 = (nx - 4) // 4 * 4
    bulk = np.zeros((ny, nx), bool)
    bulk[4:ny - 4, 4:cb1] = True
    assert set(np.unique(m2[bulk])) <= {16, 4096} and not m2[~bulk].any()
    inner = np.zeros_like(bulk)
    inner[8:ny - 7, 8:cb1 - 4] = True
    assert (m2[inner] == 16).all() and (m2[bulk & ~inner] == 4096).all()
    assert set(np.unique(m1)) <= {0, 16} and not m1[~bulk].any()
    band = bulk.copy()
    band[10:ny - 11, 12:cb1 - 8] = False
    assert (m1[band] == 16).all()


def native_params(ny, nx):
    from mpi4jax_b200._src import native

    return native.B2SweParams(ny=ny, nx=nx, pitch=(nx + 3) // 4 * 4)
