"""The shallow-water kernels and the halo exchange with peer ranks, bit for bit against the host emulation.

Every rank runs the native model on the GPU and also replays the whole process grid on the host with
the stencil bodies compiled by g++ (tests/_swe_emu.py).  Every rounding in the bodies is explicit, so
each rank's GPU state must equal its emulated block bit for bit, halos included: walls, periodic wrap
and diagonals that are other ranks.  ``ops.halo_exchange`` is checked the same way against the numpy
model of the eight-neighbour exchange (tests/_halo_sim.py) on process grids the test chooses, with
walls in x as well.  The emulation itself is checked against a float64 numpy step of the discrete
system at the end of the file.

At world size 1 the GPU tests run on the (1, 1) grid; launcher tests run this file as jobs of 2, 4 and
6 ranks (and 3 ranks for the halo exchange alone) whose ranks share the GPUs there are.  Failed checks
are collected and raised at the end of a test, so the ranks never diverge in the collective calls they
make, and every rank's result is hashed and compared over the control plane."""

import os
import zlib

import numpy as np
import pytest
import torch

import mpi4jax_b200 as m
from mpi4jax_b200 import MPI
from mpi4jax_b200.models import ShallowWaterConfig, ShallowWaterModel
from mpi4jax_b200.models.shallow_water import SUPPORTED_NPROC
from mpi4jax_b200.ops import halo_exchange

from ._halo_sim import neighbors, new_exchange
from ._peer_job import Checks, expect_passed, job
from ._swe_emu import FIELDS, HAVE_TOOLCHAIN, build, emulate_calls

comm = MPI.COMM_WORLD
rank = comm.Get_rank()
size = comm.Get_size()
inside_job = size > 1 or "MPI4JAX_B200_NESTED" in os.environ


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if not HAVE_TOOLCHAIN:
        pytest.skip("needs g++ and the CUDA headers")
    return build(tmp_path_factory, "swe_emu_peers")


def _same_bits(got, want, label):
    """Bitwise on int32 views: -0.0 and NaN payloads count."""
    g = got.detach().cpu().contiguous().view(torch.int32)
    w = torch.from_numpy(np.ascontiguousarray(want)).view(torch.int32)
    assert g.shape == w.shape, (label, tuple(g.shape), tuple(w.shape))
    diff = g != w
    if diff.any():
        at = diff.nonzero()[0].tolist()
        gf, wf = g.view(torch.float32), w.view(torch.float32)
        raise AssertionError(f"{label}: {int(diff.sum())} cells differ, first at {at}: "
                             f"got {gf[tuple(at)].item()!r}, want {wf[tuple(at)].item()!r}")


# ---------------------------------------------------------------------------
# the native model against the emulation, at the model's process grid
# ---------------------------------------------------------------------------
def _grid(P):
    PY = min(P, 2)
    return PY, P // PY


def _shapes():
    """Local block shapes (rows, columns), halo included."""
    shapes = [
        (12, 30), (22, 18),                     # ny < 16, nx < 24: `ca` runs the stand-alone kernels
        (20, 40), (20, 41), (20, 42), (20, 43),  # nx % 4 = 0..3: pitch padding, east frames of 3..6 columns
        (200, 72),                              # several row segments of the bulk kernel
    ]
    if size <= 2:
        shapes.append((1024, 1024))             # bulk and frame streams overlap in time
    return shapes


def _model(shape, pipeline):
    PY, PX = _grid(size)
    cfg = ShallowWaterConfig.for_resolution((shape[1] - 2) * PX, (shape[0] - 2) * PY)
    model = ShallowWaterModel(cfg, comm=comm, device=comm.device, backend="native", pipeline=pipeline)
    assert (model.ny_local, model.nx_local) == shape
    return model


def _check_state(chk, model, want, label):
    """h, u, v whole (their halos: the exchanged ones for h, stale by the friction step for u, v);
    dh, du, dv on the interior."""
    m.flush()
    for name in FIELDS:
        got = getattr(model, name)
        w = [blk[name] for blk in want]
        if name in ("dh", "du", "dv"):
            got, w = got[1:-1, 1:-1], [x[1:-1, 1:-1] for x in w]
        chk(_same_bits, got, w[rank], f"{label} {name}")
        chk.add(f"{label} {name}", got, w)


def _need_model_grid(device):
    if device.type != "cuda":
        pytest.skip("the native model needs a CUDA device")
    if size not in SUPPORTED_NPROC:
        pytest.skip(f"the model runs on {SUPPORTED_NPROC} ranks")


def test_model_matches_the_emulation(device, request):
    """reset() (the first halo exchange and, for `ca`, b2_swe_ca_init), the Euler first step, then 8 and 4
    more steps (both ping-pong parities and the odd-count copy-back), for both pipelines and every block
    shape."""
    _need_model_grid(device)
    emu = request.getfixturevalue("emu")
    PY, PX = _grid(size)
    chk = Checks()
    calls = (1, 8, 4)
    for shape in _shapes():
        want = None
        for pipeline in ("ca", "standalone"):
            model = _model(shape, pipeline)
            if want is None:
                want = emulate_calls(emu, model, PY, PX, calls)
            label = f"{pipeline} block {shape} grid {PY}x{PX}"
            _check_state(chk, model, want[0], f"{label} after reset")
            done = 0
            for k, n in enumerate(calls):
                model.multistep(n)
                done += n
                _check_state(chk, model, want[k + 1], f"{label} after {done} steps")
            del model
    chk.finish()


def test_model_under_jit_and_after_load_state(device, request):
    """m.jit(multistep(5)) replayed (eager warm-up, capture, replay) equals the emulation; a `ca` model
    restored with its frame storage continues bit-identically."""
    _need_model_grid(device)
    emu = request.getfixturevalue("emu")
    PY, PX = _grid(size)
    chk = Checks()
    shape = (36, 46)
    for pipeline in ("ca", "standalone"):
        model = _model(shape, pipeline)
        want = emulate_calls(emu, model, PY, PX, (1, 5, 5, 5, 6))
        label = f"{pipeline} block {shape} grid {PY}x{PX}"
        model.step(first_step=True)
        run = m.jit(lambda: model.multistep(5, first_step=False))
        for k in range(3):
            run()
            _check_state(chk, model, want[k + 2], f"{label} jit call {k}")
        snap = [t.clone() for t in model.state]
        ext = model.ext_state()
        model.multistep(6, first_step=False)
        _check_state(chk, model, want[5], f"{label} after 22 steps")
        if pipeline == "ca":
            model.load_state(type(model.state)(*snap), ext=ext)
            model.multistep(6, first_step=False)
            _check_state(chk, model, want[5], f"{label} restored at step 16, after 22 steps")
        del run, model
    chk.finish()


# ---------------------------------------------------------------------------
# ops.halo_exchange on process grids the test chooses
# ---------------------------------------------------------------------------
HALO_GRIDS = {1: [(1, 1)], 2: [(1, 2), (2, 1)], 3: [(3, 1), (1, 3)], 4: [(2, 2), (4, 1)], 6: [(2, 3), (3, 2)]}
KIND_SETS = (("h",), ("u",), ("v",), ("h", "u", "v"), ("u", "v", "h", "v", "u", "h", "u", "v"))
# -0.0, quiet and signalling NaNs with payload bits, +-inf, fp32 subnormals
SPECIALS = np.array([0x80000000, 0x7FC12345, 0xFFC00001, 0x7F800001, 0x7F800000, 0xFF800000, 0x00000001,
                     0x807FFFFF, 0x00400000], dtype=np.uint32).view(np.int32)


def _payload(case, q, nf, ny, nx):
    """Rank q's fields of ``case``, as int32 bits: normals with every fourth cell or so a special value."""
    g = np.random.default_rng(zlib.crc32(repr((case, q)).encode()))
    bits = g.standard_normal((nf, ny, nx)).astype(np.float32).view(np.int32)
    pick = g.random(bits.shape) < 0.25
    bits[pick] = g.choice(SPECIALS, int(pick.sum()))
    return bits


class _Halo:
    """This rank's fields for one grid and kind set: (ny, nx) views of (ny, pitch) storage whose padding
    holds a sentinel that no exchange may touch."""

    def __init__(self, device, grid, periodic_x, kinds, shape):
        self.PY, self.PX = grid
        self.periodic_x, self.kinds = periodic_x, kinds
        self.ny, self.nx = shape
        pitch = (self.nx + 3) // 4 * 4
        self.bases = [torch.full((self.ny, pitch), -7.0, dtype=torch.float32, device=device) for _ in kinds]
        self.fields = [b[:, :self.nx] for b in self.bases]
        py, px = divmod(rank, self.PX)
        nb, dg = neighbors(py, px, self.PY, self.PX, periodic_x)
        self.args = dict(**nb, **dg, periodic_x=periodic_x, at_east_wall=px == self.PX - 1,
                         at_north_wall=py == self.PY - 1)

    def fill(self, case):
        arrs = [_payload(case, q, len(self.kinds), self.ny, self.nx) for q in range(size)]
        for f, a in zip(self.fields, arrs[rank]):
            f.copy_(torch.from_numpy(a).view(torch.float32))
        return arrs

    def exchange(self, c):
        halo_exchange(self.fields, self.kinds, comm=c, **self.args)

    def check(self, chk, arrs, label):
        m.flush()
        for k, kind in enumerate(self.kinds):
            want = [a[k].copy() for a in arrs]
            new_exchange(want, self.PY, self.PX, kind, self.periodic_x)
            chk(_same_bits, self.fields[k], want[rank], f"{label} field {k} ({kind})")
            chk.add(f"{label} field {k}", self.fields[k], want)
            pad = self.bases[k][:, self.nx:]
            chk(_same_bits, pad, np.full(tuple(pad.shape), -7.0, np.float32), f"{label} field {k} row padding")


def test_halo_exchange_with_peers(device):
    """Every grid of this world size, periodic and walled x, 1 / 3 / 8 fields of mixed kinds, ny != nx
    and neither a multiple of 4, three calls with fresh data (both receive-buffer parities and the next
    message after them), the same under m.jit replay, and the halo buffer limit."""
    if device.type != "cuda":
        pytest.skip("ops.halo_exchange needs CUDA tensors")
    if size not in HALO_GRIDS:
        pytest.skip(f"no process grids listed for {size} ranks")
    chk = Checks()
    for grid in HALO_GRIDS[size]:
        for periodic_x in (True, False):
            # a communicator's halo channels count messages per side: one neighbour layout per communicator
            c = comm.Clone()
            try:
                for kinds in KIND_SETS:
                    for shape in ((19, 30), (35, 21)):
                        label = f"grid {grid} periodic_x={periodic_x} kinds {''.join(kinds)} shape {shape}"
                        h = _Halo(device, grid, periodic_x, kinds, shape)
                        for call in range(3):
                            arrs = h.fill((label, "eager", call))
                            h.exchange(c)
                            h.check(chk, arrs, f"{label} call {call}")
                        run = m.jit(lambda: h.exchange(c))
                        for call in range(3):
                            arrs = h.fill((label, "jit", call))
                            run()
                            h.check(chk, arrs, f"{label} jit call {call}")
                        del run
            finally:
                m.flush()
                c.Free()
            _halo_buffer_limit(device, chk, grid, periodic_x)
    chk.finish()


def _halo_buffer_limit(device, chk, grid, periodic_x):
    """Three fields whose longer side (341) is not a multiple of 4 on a communicator with 4 KiB halo
    buffers: the longest message (3 * 341 words of 8 bytes) just fits a side's 8192-byte buffer, as in
    test_examples.py::test_halo_exchange_at_the_halo_buffer_limit, with peers."""
    old = os.environ.get("MPI4JAX_B200_HALO_BYTES")
    os.environ["MPI4JAX_B200_HALO_BYTES"] = "4096"
    try:
        c = comm.Clone()                 # its native side is created with the small halo buffers
    finally:
        if old is None:
            del os.environ["MPI4JAX_B200_HALO_BYTES"]
        else:
            os.environ["MPI4JAX_B200_HALO_BYTES"] = old
    try:
        label = f"halo buffer limit grid {grid} periodic_x={periodic_x}"
        h = _Halo(device, grid, periodic_x, ("h", "u", "v"), (341, 99))
        for call in range(2):
            arrs = h.fill((label, call))
            h.exchange(c)
            h.check(chk, arrs, f"{label} call {call}")
    finally:
        c.Free()


# ---------------------------------------------------------------------------
# the same tests with 2, 3, 4 and 6 ranks
# ---------------------------------------------------------------------------
MODEL_TESTS = ["test_model_matches_the_emulation", "test_model_under_jit_and_after_load_state"]
HALO_TESTS = ["test_halo_exchange_with_peers"]
SMALL_SLOTS = {"MPI4JAX_B200_P2P_SLOT_BYTES": "1048576"}     # smaller p2p rings for many contexts


@pytest.mark.gpu
@pytest.mark.skipif(inside_job, reason="already inside a multi-rank job")
def test_swe_peers_two_ranks_gpu():
    """Grid 2 x 1: walls on both y sides of every rank, the diagonal is the rank below or above."""
    code, outs = job(__file__, 2, "not ranks_gpu")
    expect_passed(code, outs, 2, MODEL_TESTS + HALO_TESTS)


@pytest.mark.gpu
@pytest.mark.skipif(inside_job, reason="already inside a multi-rank job")
def test_swe_peers_three_ranks_gpu():
    """The halo exchange alone (the model has no three-rank grid): 3 x 1 has a rank with a south and a
    north neighbour."""
    code, outs = job(__file__, 3, "test_halo_exchange_with_peers")
    expect_passed(code, outs, 3, HALO_TESTS)


@pytest.mark.gpu
@pytest.mark.skipif(inside_job, reason="already inside a multi-rank job")
def test_swe_peers_four_ranks_gpu():
    """Grid 2 x 2: the diagonals are real ranks, west and east are the same peer."""
    code, outs = job(__file__, 4, "not ranks_gpu", SMALL_SLOTS)
    expect_passed(code, outs, 4, MODEL_TESTS + HALO_TESTS)


@pytest.mark.gpu
@pytest.mark.skipif(inside_job, reason="already inside a multi-rank job")
def test_swe_peers_six_ranks_gpu():
    """Grid 2 x 3: west and east are distinct peers."""
    code, outs = job(__file__, 6, "not ranks_gpu", SMALL_SLOTS)
    expect_passed(code, outs, 6, MODEL_TESTS + HALO_TESTS)


# ---------------------------------------------------------------------------
# the emulation against a float64 step of the discrete system (no GPU)
# ---------------------------------------------------------------------------
def _bc(a, kind):
    """Halo exchange + walls of the ops path on the (1, 1) grid: periodic in x, walls in y."""
    a[:, -1] = a[:, 1]
    a[:, 0] = a[:, -2]
    if kind == "v":
        a[-2, :] = 0.0


def _step64(s, cor, cfg, first):
    """ShallowWaterModel._step_ops in float64 on the (1, 1) grid; ``s``: dict of h, u, v, dh, du, dv."""
    dx, dy, dt, g, visc = cfg.dx, cfg.dy, cfg.dt, cfg.gravity, cfg.lateral_viscosity
    h, u, v = s["h"], s["u"], s["v"]
    C = (slice(1, -1), slice(1, -1))
    E = (slice(1, -1), slice(2, None))
    W = (slice(1, -1), slice(None, -2))
    N = (slice(2, None), slice(1, -1))
    S = (slice(None, -2), slice(1, -1))
    NE = (slice(2, None), slice(2, None))
    SE = (slice(None, -2), slice(2, None))
    NW = (slice(2, None), slice(None, -2))
    hc = np.pad(h[C], 1, mode="edge")
    _bc(hc, "h")
    fe, fn, q, ke = (np.zeros_like(h) for _ in range(4))
    fe[C] = 0.5 * (hc[C] + hc[E]) * u[C]
    fn[C] = 0.5 * (hc[C] + hc[N]) * v[C]
    _bc(fe, "u")
    _bc(fn, "v")
    dh_new = -(fe[C] - fe[W]) / dx - (fn[C] - fn[S]) / dy
    q[C] = (cor[1:-1, None] + ((v[E] - v[C]) / dx - (u[N] - u[C]) / dy)) * (
        1.0 / (0.25 * (hc[C] + hc[E] + hc[N] + hc[NE])))
    _bc(q, "h")
    du_new = -g * (h[E] - h[C]) / dx + 0.5 * (q[C] * 0.5 * (fn[C] + fn[E]) + q[S] * 0.5 * (fn[S] + fn[SE]))
    dv_new = -g * (h[N] - h[C]) / dy - 0.5 * (q[C] * 0.5 * (fe[C] + fe[N]) + q[W] * 0.5 * (fe[W] + fe[NW]))
    ke[C] = 0.5 * (0.5 * (u[C] ** 2 + u[W] ** 2) + 0.5 * (v[C] ** 2 + v[S] ** 2))
    _bc(ke, "h")
    du_new = du_new - (ke[E] - ke[C]) / dx
    dv_new = dv_new - (ke[N] - ke[C]) / dy
    if first:
        u[C] += dt * du_new
        v[C] += dt * dv_new
        h[C] += dt * dh_new
    else:
        u[C] += dt * (cfg.ab_a * du_new + cfg.ab_b * s["du"][C])
        v[C] += dt * (cfg.ab_a * dv_new + cfg.ab_b * s["dv"][C])
        h[C] += dt * (cfg.ab_a * dh_new + cfg.ab_b * s["dh"][C])
    s["dh"][C], s["du"][C], s["dv"][C] = dh_new, du_new, dv_new
    _bc(h, "h")
    _bc(u, "u")
    _bc(v, "v")
    fe[C] = visc * (u[E] - u[C]) / dx
    fn[C] = visc * (u[N] - u[C]) / dy
    _bc(fe, "u")
    _bc(fn, "v")
    u[C] += dt * ((fe[C] - fe[W]) / dx + (fn[C] - fn[S]) / dy)
    fe[C] = visc * (v[E] - u[C]) / dx      # sic: the reference subtracts u here
    fn[C] = visc * (v[N] - u[C]) / dy
    _bc(fe, "u")
    _bc(fn, "v")
    v[C] += dt * ((fe[C] - fe[W]) / dx + (fn[C] - fn[S]) / dy)


# Bounds on (max |e| / max |d64|, |mean e| / mean |d64|), e = emulated - float64 increment, per number
# of steps; about twice what was measured on the 48 x 24 grid (g++ -O1 -ffp-contract=off, x86-64):
#        n = 1: max, bias             n = 6: max, bias
#   h    1.2e-3, 1.6e-4               8.4e-5, 1.9e-6     (h's increment is about 1e-3 of h: fp32 rounding of h)
#   u    8.8e-5, 1.2e-6               1.0e-4, 5.4e-7
#   v    1.0e-6, 3.6e-9               2.3e-5, 1.2e-7
#   dh   1.2e-4, 6.2e-10              6.5e-5, 1.4e-9
#   du   7.0e-8, 1.6e-9               1.7e-4, 1.1e-7
#   dv   1.0e-6, 5.7e-9               4.9e-5, 1.8e-7
# The rounding of the fp32 state is noise of either sign and averages out of the bias; a wrong coefficient
# does not (1 % on the y friction of u moves u's bias after 6 steps from 5.4e-7 to 1.8e-6).
INCREMENT_BOUND = {
    1: dict(h=(3e-3, 4e-4), u=(2e-4, 3e-6), v=(3e-6, 1e-8), dh=(3e-4, 2e-9), du=(2e-7, 4e-9), dv=(3e-6, 2e-8)),
    6: dict(h=(2e-4, 4e-6), u=(2e-4, 1.2e-6), v=(5e-5, 3e-7), dh=(2e-4, 3e-9), du=(4e-4, 3e-7), dv=(1e-4, 4e-7)),
}


def _increment_errors(emu, n):
    cfg = ShallowWaterConfig(nx=48, ny=24)
    model = ShallowWaterModel(cfg, device="cpu", backend="ops")
    snaps = emulate_calls(emu, model, 1, 1, (n,))
    start, got = snaps[0][0], snaps[-1][0]
    s = {name: start[name].astype(np.float64) for name in FIELDS}
    s0 = {name: a.copy() for name, a in s.items()}
    cor = cfg.coriolis_f + np.arange(-1, cfg.ny + 1) * cfg.dy * cfg.coriolis_beta
    for it in range(n):
        _step64(s, cor, cfg, it == 0)
    err = {}
    for name in FIELDS:
        d64 = (s[name] - s0[name])[1:-1, 1:-1]
        e = (got[name].astype(np.float64) - s0[name])[1:-1, 1:-1] - d64
        err[name] = (np.abs(e).max() / np.abs(d64).max(), abs(e.mean()) / np.abs(d64).mean())
    return err


@pytest.mark.parametrize("n", [1, 6])
def test_emulated_step_increments_match_a_float64_step(emu, n):
    """The increments (state after n steps - initial state; the tendencies themselves) of the emulated
    native step against a float64 step of the same discrete system, each relative to its own scale, as a
    maximum and as a bias: unlike a comparison of absolute h (about 100 m), this sees a 1 % error in one
    flux's coefficient."""
    if size > 1:
        pytest.skip("a world-size-1 check: every rank would repeat it")
    err = _increment_errors(emu, n)
    bound = INCREMENT_BOUND[n]
    bad = {k: f"max {e[0]:.2e}, bias {e[1]:.2e} (bounds {bound[k][0]:.1e}, {bound[k][1]:.1e})"
           for k, e in err.items() if not (e[0] <= bound[k][0] and e[1] <= bound[k][1])}
    assert not bad, bad
