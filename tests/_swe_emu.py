"""The shallow-water stencil bodies compiled for the HOST (tests/native/swe_host_emu.cpp: the CUDA
source with the qualifiers defined away) and the launch sequence of b2_swe_multistep replayed with
them on a whole process grid.  Every rounding in the bodies is explicit, so this emulation computes
the bits the GPU kernels compute (used by test_swe_host_emulation.py and test_swe_peers.py)."""

import ctypes
import os
import shutil
import subprocess

import numpy as np

from mpi4jax_b200._src import native
from mpi4jax_b200.models.shallow_water import fold_constants

from ._halo_sim import new_exchange

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA_INC = next((d for d in (os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include"),
                             "/usr/local/cuda/include") if os.path.exists(os.path.join(d, "cuda_runtime.h"))), None)
HAVE_TOOLCHAIN = shutil.which("g++") is not None and CUDA_INC is not None
FIELDS = ("h", "u", "v", "dh", "du", "dv")


def build(tmp_path_factory, name):
    out = tmp_path_factory.mktemp(name) / f"lib{name}.so"
    cmd = ["g++", "-O1", "-ffp-contract=off", "-std=c++17", "-shared", "-fPIC", "-I",
           os.path.join(REPO, "csrc"), "-I", CUDA_INC, os.path.join(REPO, "tests", "native", "swe_host_emu.cpp"),
           "-o", str(out)]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    lib = ctypes.CDLL(str(out))
    # the package's ctypes mirrors of the ABI structs, against the C structs the harness is built with
    assert lib.emu_sizeof_swe_params() == ctypes.sizeof(native.B2SweParams)
    assert lib.emu_sizeof_swe_ca() == ctypes.sizeof(native.B2SweCA)
    return lib


def ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def blocks(model, PY, PX):
    """Cut the model's global initial condition into (PY x PX) blocks with one halo cell, as
    ShallowWaterModel does per rank; returns per-rank dicts of pitch-padded float32 arrays."""
    h0, u0, v0 = model.initial_conditions_global()
    NY, NX = h0.shape
    nyi, nxi = (NY - 2) // PY, (NX - 2) // PX
    pitch = (nxi + 2 + 3) // 4 * 4
    ranks = []
    for py in range(PY):
        for px in range(PX):
            blk = {}
            for name, g in (("h", h0), ("u", u0), ("v", v0)):
                a = np.zeros((nyi + 2, pitch), np.float32)
                a[:, :nxi + 2] = g[py * nyi: py * nyi + nyi + 2, px * nxi: px * nxi + nxi + 2]
                blk[name] = a
            for name in ("h1", "u1", "v1", "dh", "du", "dv", "fe", "fn", "q", "ke", "fe2", "fn2"):
                blk[name] = np.zeros((nyi + 2, pitch), np.float32)
            y_global = np.arange(-1, NY - 1) * model.cfg.dy
            cor = (model.cfg.coriolis_f + y_global[py * nyi: py * nyi + nyi + 2] * model.cfg.coriolis_beta)
            blk["cor"] = cor.astype(np.float32)
            ranks.append(blk)
    return ranks, nyi + 2, nxi + 2, pitch


def params(model, blk, ny, nx, pitch, py, PY, first):
    """The kernel parameters of the rank in process row ``py``.  A native model's own parameters are
    copied (the constants it folded), with ``coriolis`` pointed at the host array of ``blk``."""
    if getattr(model, "_params", None) is not None:
        p = native.B2SweParams.from_buffer_copy(model._params)
        assert (p.ny, p.nx, p.pitch) == (ny, nx, pitch)
        p.first_step, p.south_wall, p.north_wall = int(first), int(py == 0), int(py == PY - 1)
        p.coriolis = blk["cor"].ctypes.data
        return p
    cfg = model.cfg
    return fold_constants(native.B2SweParams(
        ny=ny, nx=nx, pitch=pitch, dx=cfg.dx, dy=cfg.dy, dt=cfg.dt, gravity=cfg.gravity,
        viscosity=cfg.lateral_viscosity, rdx=np.float32(1) / np.float32(cfg.dx),
        rdy=np.float32(1) / np.float32(cfg.dy), ab_a=cfg.ab_a, ab_b=cfg.ab_b, first_step=int(first),
        south_wall=int(py == 0), north_wall=int(py == PY - 1), coriolis=blk["cor"].ctypes.data))


def exchange(ranks, names, kinds, nx, PY, PX):
    for name, kind in zip(names, kinds):
        new_exchange([r[name][:, :nx] for r in ranks], PY, PX, kind)


def emulate_calls(emu, model, PY, PX, calls):
    """The launch sequence of b2_swe_multistep: K1 -> exchange -> K2 -> exchange -> K34 -> exchange -> K5,
    advanced by ``calls[0]``, ``calls[1]``, ... steps (the first step of all is the Euler step).  Returns
    per-rank copies of (h, u, v, dh, du, dv) after reset() and after each call."""
    ranks, ny, nx, pitch = blocks(model, PY, PX)
    # reset(): halos of the initial state, ping-pong partners start as copies
    exchange(ranks, ("h", "u", "v"), ("h", "u", "v"), nx, PY, PX)
    for r in ranks:
        r["h1"][:], r["u1"][:], r["v1"][:] = r["h"], r["u"], r["v"]
    hk, hnk = "h", "h1"

    def snapshot():
        return [{name: r[hk if name == "h" else name][:, :nx].copy() for name in FIELDS} for r in ranks]

    out = [snapshot()]
    B = ctypes.byref
    it = 0
    for n in calls:
        for _ in range(n):
            ps = [params(model, r, ny, nx, pitch, i // PX, PY, it == 0) for i, r in enumerate(ranks)]
            for r, p in zip(ranks, ps):
                emu.emu_k1_all(B(p), ptr(r[hk]), ptr(r["u"]), ptr(r["v"]), ptr(r["fe"]), ptr(r["fn"]),
                               ptr(r["q"]), ptr(r["ke"]))
            exchange(ranks, ("fe", "fn", "q", "ke"), ("u", "v", "h", "h"), nx, PY, PX)
            for r, p in zip(ranks, ps):
                emu.emu_k2_all(B(p), ptr(r[hk]), ptr(r[hnk]), ptr(r["u"]), ptr(r["v"]), ptr(r["dh"]),
                               ptr(r["du"]), ptr(r["dv"]), ptr(r["fe"]), ptr(r["fn"]), ptr(r["q"]),
                               ptr(r["ke"]))
            exchange(ranks, (hnk, "u", "v"), ("h", "u", "v"), nx, PY, PX)
            for i, (r, p) in enumerate(zip(ranks, ps)):
                emu.emu_k34(B(p), ptr(r["u"]), ptr(r["u1"]), ptr(r["v"]), ptr(r["fe2"]), ptr(r["fn2"]),
                            int(i // PX > 0))
                r["u"], r["u1"] = r["u1"], r["u"]
            exchange(ranks, ("fe2", "fn2"), ("u", "v"), nx, PY, PX)
            for r, p in zip(ranks, ps):
                emu.emu_k5(B(p), ptr(r["v"]), ptr(r["fe2"]), ptr(r["fn2"]))
            hk, hnk = hnk, hk
            it += 1
        out.append(snapshot())
    return out


def emulate(emu, model, PY, PX, nsteps):
    """Per-rank (h, u, v, dh, du, dv) after reset() and ``nsteps`` steps."""
    return emulate_calls(emu, model, PY, PX, [nsteps])[-1]
