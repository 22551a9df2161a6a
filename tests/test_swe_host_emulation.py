"""The shallow-water stencil bodies compiled for the HOST (tests/native/swe_host_emu.cpp: the
CUDA source with the qualifiers defined away) -- checks, on a machine without a GPU, the launch
sequence of the stand-alone kernels against the public-ops model and the communication-avoiding
step as b2_swe_multistep_ca launches it (csrc/b2_swe_ca_body.cuh, b2_swe_ca_bulk.cuh: the one-pass
bulk kernel with its lanes in lockstep, frame kernels with owner views and ping-pong storage,
deep-halo exchange geometry, bulk / frame partition) against the stand-alone kernels, bit for bit."""

import ctypes

import numpy as np
import pytest

from mpi4jax_b200._src import native

from ._swe_emu import HAVE_TOOLCHAIN, blocks, build, emulate, params, ptr

pytestmark = pytest.mark.skipif(not HAVE_TOOLCHAIN, reason="needs g++ and the CUDA headers")


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return build(tmp_path_factory, "swe_emu")


def _close(a, b, tol):
    return np.abs(a - b).max() <= tol * (np.abs(b).max() + 1e-30)


def test_emulated_native_step_matches_the_ops_backend(emu):
    """The kernel launch sequence of b2_swe_multistep (bodies + single-phase halo exchange),
    executed on the host, vs the model written with the public ops -- the GPU suite's
    native-vs-ops comparison, on a box without a GPU."""
    import torch

    from mpi4jax_b200.models import ShallowWaterConfig, ShallowWaterModel

    cfg = ShallowWaterConfig(nx=48, ny=24)
    model = ShallowWaterModel(cfg, device="cpu", backend="ops")
    nsteps = 6
    emu_state = emulate(emu, model, 1, 1, nsteps)[0]
    model.multistep(nsteps)
    for name, t in model.state._asdict().items():
        got, want = emu_state[name], t.numpy()
        assert np.isfinite(got).all()
        tol = 2e-4 if name in ("h", "u", "v") else 2e-3
        assert _close(got[1:-1, 1:-1], want[1:-1, 1:-1], tol), name
    assert isinstance(model.h, torch.Tensor)


# ---- communication-avoiding step (csrc/b2_swe_ca_body.cuh, b2_swe_ca_bulk.cuh, b2_swe_ca.cu) ------------
_SIDES = ("w", "e", "s", "n", "sw", "se", "nw", "ne")        # HALO_W .. HALO_NE: where a message lands


def _neighbours(r, PY, PX):
    py, px = divmod(r, PX)

    def at(dy_, dx_):
        iy = py + dy_
        return None if not 0 <= iy < PY else iy * PX + (px + dx_) % PX

    return dict(w=at(0, -1), e=at(0, 1), s=at(-1, 0), n=at(1, 0), sw=at(-1, -1), se=at(-1, 1), nw=at(1, -1),
                ne=at(1, 1))


def _ca_exchange(emu, ranks, names, ny, nx, pitch, epitch, PY, PX):
    """b2_k_halo_ca without the transport: every message read from the sender's arrays as the push loop
    does and scattered as the poll loop does."""
    F3 = ctypes.c_void_p * 3
    for r, blk in enumerate(ranks):
        nb = _neighbours(r, PY, PX)
        for side, key in enumerate(_SIDES):
            q = nb[key]
            if q is None:
                continue
            send = F3(*[ranks[q][n].ctypes.data for n in names])
            recv = F3(*[blk[n].ctypes.data for n in names])
            ext = F3(blk["hx"].ctypes.data, blk["upx"].ctypes.data, blk["vpx"].ctypes.data)
            emu.emu_ca_deliver(ny, nx, pitch, epitch, side, int(nb["s"] is not None), int(nb["n"] is not None),
                               send, recv, ext)


def _ca_ext(blk, epitch):
    return native.B2SweCA(hx=blk["hx"].ctypes.data, upx=blk["upx"].ctypes.data, vpx=blk["vpx"].ctypes.data,
                          uppx=blk["uppx"].ctypes.data, vppx=blk["vppx"].ctypes.data, epitch=epitch, cb1=0)


class EmuStep(ctypes.Structure):      # EmuStep (tests/native/swe_host_emu.cpp): one rank's arrays for one step
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

    ranks, ny, nx, pitch = blocks(model, PY, PX)
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
        p = params(model, r, ny, nx, pitch, i // PX, PY, True)
        emu.emu_ca_init_ext(B(p), B(_ca_ext(r, epitch)), ptr(r["u"]), ptr(r["v"]))
    cur = ""
    for it in range(nsteps):
        nxt = "1" if cur == "" else ""
        ps = [params(model, r, ny, nx, pitch, i // PX, PY, it == 0) for i, r in enumerate(ranks)]
        xs = [_ca_ext(r, epitch) for r in ranks]
        es = [EmuStep(**{n: r[n + cur].ctypes.data for n in _PAIRS},
                      **{n + "_o": r[n + nxt].ctypes.data for n in _PAIRS},
                      dh=r["dh"].ctypes.data, upf=r["upf"].ctypes.data, vpf=r["vpf"].ctypes.data)
              for r in ranks]
        if not reverse:
            for p, e in zip(ps, es):
                emu.emu_ca_bulk_step(B(p), B(e), rows, reverse)
        for p, x, e in zip(ps, xs, es):
            emu.emu_ca_tend_frame(B(p), B(x), B(e), reverse)
        _ca_exchange(emu, ranks, ("h" + nxt, "upf", "vpf"), ny, nx, pitch, epitch, PY, PX)
        for p, x, e in zip(ps, xs, es):
            emu.emu_ca_fric_frame(B(p), B(x), B(e), reverse)
        if reverse:
            for p, e in zip(ps, es):
                emu.emu_ca_bulk_step(B(p), B(e), rows, reverse)
        cur = nxt
    return [{k: r[k + (cur if k in _PAIRS else "")][:, :nx] for k in ("h", "u", "v", "dh", "du", "dv")}
            for r in ranks]


@pytest.mark.parametrize("shape,rows", [((16, 24), 16), ((26, 50), 5), ((17, 29), 3), ((140, 33), 16),
                                        ((31, 300), 7), ((200, 530), 64), ((200, 530), 13)])
def test_ca_bulk_and_frame_partition_the_interior(emu, shape, rows):
    """The frame kernels and swe_ca_bulk_step (whatever its rows per segment) write every interior cell
    exactly once; the bulk is rows [4, ny-5] x columns [4, cb1), covered by the segments and warp strips."""
    ny, nx = shape
    p = native.B2SweParams(ny=ny, nx=nx)
    assert emu.emu_ca_supported(ctypes.byref(p)) == 1
    marks = np.zeros((ny, nx), np.int32)
    emu.emu_ca_marks(ctypes.byref(p), rows, marks.ctypes.data_as(ctypes.POINTER(ctypes.c_int)))
    owner = marks & 0xff                     # 1 = frame kernels, 16 = one store of the bulk kernel
    assert set(np.unique(owner[1:-1, 1:-1])) <= {1, 16}          # every interior cell written exactly once
    assert marks[0].sum() == marks[-1].sum() == marks[:, 0].sum() == marks[:, -1].sum() == 0
    cb1 = (nx - 4) // 4 * 4                  # east frame: 3 .. 6 columns (the bulk ends on a float4 boundary)
    bulk = np.zeros((ny, nx), bool)
    bulk[4:ny - 4, 4:cb1] = True
    assert np.array_equal(owner == 16, bulk)
    band = (marks & 256) != 0                # kernel A also computes u', v' two cells into the bulk
    want = np.zeros_like(band)
    want[1:-1, 1:-1] = True
    want[6:ny - 6, 6:cb1 - 2] = False
    assert np.array_equal(band, want)


@pytest.mark.parametrize("nsteps", [5, 6])    # both ping-pong parities: after 5 steps the partners hold the state
@pytest.mark.parametrize("grid,block,rows", [
    ((1, 1), (24, 48), 5), ((2, 1), (24, 48), 5), ((1, 2), (24, 48), 5), ((2, 2), (24, 48), 5),
    ((3, 2), (24, 48), 5), ((2, 4), (24, 48), 5),
    ((1, 1), (24, 48), 64),                 # one segment covers the bulk
    ((2, 1), (40, 280), 7),                 # several warp strips per row, a partial last strip
    ((1, 2), (33, 140), 16),                # odd bulk height: a short last segment
    ((2, 2), (18, 39), 5),                  # nx % 4 == 1: the east halo column is a float4 group of its own
])
def test_emulated_one_pass_ca_pipeline_is_bit_identical_to_the_standalone_pipeline(emu, grid, block, rows, nsteps):
    """One deep exchange per step + local recomputation (frame kernels with owner views, one-pass bulk
    kernel) vs the three exchanges of b2_swe_multistep, same decomposition: the same bits, walls, periodic
    wrap and the reference's stale u / v halos included, in any order of the bulk kernel's warps."""
    from mpi4jax_b200.models import ShallowWaterConfig, ShallowWaterModel

    PY, PX = grid
    model = ShallowWaterModel(ShallowWaterConfig(nx=block[1] * PX, ny=block[0] * PY), device="cpu", backend="ops")
    a = emulate(emu, model, PY, PX, nsteps)
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
