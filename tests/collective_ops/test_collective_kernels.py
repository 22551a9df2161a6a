"""The collective kernels with peers, against an oracle that never goes through the library.

Every rank builds every rank's input itself, from a seed of (case, rank q), and computes the expected
result locally: integers in 64-bit arithmetic and then wrapped to the dtype (two's-complement
wrap-around), floats folded in rank order in the accumulate type and rounded once -- the order the
kernels document ("bitwise identical result on every rank", csrc/b2_reduce.cuh) -- and, as a second
contract, checked against an extended-precision fold within ``(P-1) u_acc sum|x_q| + ulp/2``.
That every rank holds the same bits is checked over the control plane (a hash per result).

Each transport is forced explicitly (``algorithm=``, communicator options) and the debug log line,
which names the transport a reduction launched, shows that it was taken.  In a single-process run the
CUDA tests run in a two-rank job whose ranks share the GPU; the launcher tests at the end run them with
three ranks (a non-power-of-two world, chunk unit 48 B, the two-phase scan) and the data-movement tests
with five (the widest pull-and-stage instantiations of b2_k_move)."""

import contextlib
import hashlib
import os
import re
import tempfile
import zlib

import numpy as np
import pytest
import torch
import torch.distributed as dist

import mpi4jax_b200 as m
from mpi4jax_b200 import MPI
from mpi4jax_b200._src.native import codes, set_logging

from .._peer_job import needs_peers

comm = MPI.COMM_WORLD
rank = comm.Get_rank()
size = comm.Get_size()

peers = needs_peers("collective kernels between ranks")
# (a two-rank job would report these as skipped, not passed: test_collective_kernels_three_ranks_gpu runs them)
three_or_more = pytest.mark.skipif(size < 3, reason="needs >= 3 ranks")

OPS = ("SUM", "PROD", "MIN", "MAX", "LAND", "LOR", "LXOR", "BAND", "BOR", "BXOR")
FLOATS = (torch.float16, torch.bfloat16, torch.float32, torch.float64)
SIGNED = (torch.int8, torch.int16, torch.int32, torch.int64)
UNSIGNED = (torch.uint8, torch.uint16, torch.uint32, torch.uint64)
COMPLEX = (torch.complex64, torch.complex128)
NP = {torch.float16: np.float16, torch.float32: np.float32, torch.float64: np.float64,
      torch.int8: np.int8, torch.int16: np.int16, torch.int32: np.int32, torch.int64: np.int64,
      torch.uint8: np.uint8, torch.uint16: np.uint16, torch.uint32: np.uint32, torch.uint64: np.uint64,
      torch.complex64: np.complex64, torch.complex128: np.complex128, torch.bool: np.bool_}
LL_BYTES = 64 << 10            # the LL transport carries up to half the LL buffer (128 KiB by default)


def _ops_for(dtype):
    """The ops a reduction accepts for ``dtype`` (bool maps every op to a logical one)."""
    if dtype.is_complex:
        return ("SUM", "PROD")
    if dtype.is_floating_point:
        return ("SUM", "PROD", "MIN", "MAX")
    return OPS


# ---------------------------------------------------------------------------
# inputs: the same bits on every rank for (case, q)
# ---------------------------------------------------------------------------
def _rng(case, q):
    return np.random.default_rng(zlib.crc32(repr((case, q)).encode()))


def _input(case, q, n, dtype, opname="SUM"):
    """Rank q's input of ``case`` (a CPU tensor of ``n`` elements).  Integers use every bit (sums and
    products wrap); logical ops get many zeros; float products stay near 1 and complex products are
    integer-valued (their kernel may contract ``a.re*b.re - a.im*b.im`` into an FMA)."""
    g = _rng(case, q)
    if dtype == torch.bool:
        return torch.from_numpy(g.integers(0, 2, n).astype(np.bool_))
    if dtype.is_complex:
        if opname == "PROD":
            re, im = g.integers(-2, 3, n), g.integers(-2, 3, n)
        else:
            re, im = g.standard_normal(n), g.standard_normal(n)
        return torch.from_numpy((re + 1j * im).astype(NP[dtype]))
    if dtype.is_floating_point:
        v = g.standard_normal(n)
        if opname == "PROD":
            v = 1.0 + v / 8
        return torch.from_numpy(v.astype(np.float32 if dtype != torch.float64 else np.float64)).to(dtype)
    v = np.frombuffer(g.bytes(n * dtype.itemsize), dtype=NP[dtype]).copy()
    if opname in ("LAND", "LOR", "LXOR"):
        v[g.integers(0, 2, n).astype(bool)] = 0
    return torch.from_numpy(v)


def _np(t):
    """CPU tensor -> numpy array in a type that holds it exactly (bfloat16 -> float32)."""
    return t.float().numpy() if t.dtype == torch.bfloat16 else t.numpy()


# ---------------------------------------------------------------------------
# the oracle
# ---------------------------------------------------------------------------
def _fold(xs, opname):
    """The documented result: ``xs`` (CPU tensors of ranks 0, 1, ...) folded in rank order."""
    dtype = xs[0].dtype
    if dtype == torch.bool:
        a = np.stack([x.numpy() for x in xs])
        if opname in ("SUM", "MAX", "LOR", "BOR"):
            return torch.from_numpy(a.any(0))
        if opname in ("PROD", "MIN", "LAND", "BAND"):
            return torch.from_numpy(a.all(0))
        return torch.from_numpy(a.sum(0, dtype=np.int64) % 2 == 1)
    if dtype.is_floating_point or dtype.is_complex:
        # accumulate type: float32 for f16 / bf16 / f32, the dtype itself otherwise; one rounding at the end
        acc_t = np.float32 if dtype in (torch.float16, torch.bfloat16) else NP[dtype]
        a = [_np(x).astype(acc_t) for x in xs]
        acc = a[0].copy()
        with np.errstate(all="ignore"):
            for v in a[1:]:
                if opname == "SUM":
                    acc = acc + v
                elif opname == "PROD":
                    acc = acc * v
                elif opname == "MIN":
                    acc = np.minimum(acc, v)          # NaN-propagating
                else:
                    acc = np.maximum(acc, v)
        return torch.from_numpy(acc).to(dtype)
    a = [x.numpy() for x in xs]
    wide = np.int64 if dtype.is_signed else np.uint64
    if opname in ("SUM", "PROD"):
        acc = a[0].astype(wide)
        with np.errstate(all="ignore"):
            for v in a[1:]:
                acc = acc + v.astype(wide) if opname == "SUM" else acc * v.astype(wide)
        return torch.from_numpy(acc.astype(NP[dtype]))         # wraps to the dtype
    if opname in ("LAND", "LOR", "LXOR"):
        nz = np.stack([v != 0 for v in a])
        r = nz.all(0) if opname == "LAND" else nz.any(0) if opname == "LOR" else nz.sum(0) % 2 == 1
        return torch.from_numpy(r.astype(NP[dtype]))
    fn = {"MIN": np.minimum, "MAX": np.maximum, "BAND": np.bitwise_and, "BOR": np.bitwise_or,
          "BXOR": np.bitwise_xor}[opname]
    acc = a[0].copy()
    for v in a[1:]:
        acc = fn(acc, v)
    return torch.from_numpy(acc)


def _ulp(r, dtype):
    a = np.abs(np.where(np.isfinite(r), r, 0))
    if dtype == torch.bfloat16:
        return np.spacing(a.astype(np.float32)).astype(np.float64) * 65536
    return np.spacing(a.astype(NP[dtype])).astype(np.float64)


def _check_accuracy(got, xs, opname, label):
    """Float SUM / PROD against an extended-precision fold: error <= (P-1) u_acc sum|x_q| + ulp(result)/2."""
    dtype = xs[0].dtype
    if dtype.is_complex:
        if opname != "SUM":
            return
        got, xs = torch.view_as_real(got), [torch.view_as_real(x) for x in xs]
        dtype = torch.float32 if dtype == torch.complex64 else torch.float64
    if opname not in ("SUM", "PROD"):
        return
    u = 2.0 ** -53 if dtype == torch.float64 else 2.0 ** -24
    a = [_np(x).astype(np.longdouble) for x in xs]
    with np.errstate(all="ignore"):
        return _within_bound(got, a, u, opname, dtype, label)


def _within_bound(got, a, u, opname, dtype, label):
    if opname == "SUM":
        exact, scale = sum(a[1:], a[0].copy()), sum((np.abs(v) for v in a[1:]), np.abs(a[0]))
    else:
        exact = a[0].copy()
        for v in a[1:]:
            exact = exact * v
        scale = np.abs(exact) * (1 + len(a) * u)
    r = _np(got).astype(np.longdouble)
    ok = np.isfinite(r) & np.isfinite(exact)
    bound = (len(a) - 1) * u * scale + _ulp(_np(got), dtype) / 2
    err = np.abs(r - exact)
    bad = ok & (err > bound)
    assert not bad.any(), (f"{label}: {int(bad.sum())} elements outside (P-1) u_acc sum|x| + ulp/2, e.g. "
                           f"index {int(np.argmax(bad))}: got {r[bad][0]}, exact {exact[bad][0]}, "
                           f"bound {bound[bad][0]}")


def _assert_same(got, want, label):
    """Bitwise, except that NaNs compare by position and +0.0 == -0.0."""
    got, want = got.detach().cpu(), want.detach().cpu()
    assert got.dtype == want.dtype and got.shape == want.shape, (label, got.dtype, got.shape, want.shape)
    if got.dtype.is_floating_point or got.dtype.is_complex:
        g, w = (torch.view_as_real(got), torch.view_as_real(want)) if got.dtype.is_complex else (got, want)
        gn, wn = torch.isnan(g), torch.isnan(w)
        assert torch.equal(gn, wn), f"{label}: NaN at {gn.nonzero()[:4].tolist()} vs {wn.nonzero()[:4].tolist()}"
        diff = (g != w) & ~gn
        assert not diff.any(), f"{label}: {int(diff.sum())} elements differ, first {diff.nonzero()[0].tolist()}: " \
                               f"got {g[diff][0].item()!r}, want {w[diff][0].item()!r}"
    else:
        diff = got != want
        assert not diff.any(), f"{label}: {int(diff.sum())} elements differ, first {diff.nonzero()[0].tolist()}: " \
                               f"got {got[diff][0].item()!r}, want {want[diff][0].item()!r}"


def _digest(t):
    t = t.detach().cpu().contiguous()
    return hashlib.sha1(t.view(torch.uint8).numpy().tobytes() if t.numel() else b"").hexdigest()


class _Checks:
    """The assertions of a multi-rank test, raised at its end.  A check that fails on one rank only must
    not leave the ranks running different sequences of collectives, so ``chk(fn, *args)`` records an
    AssertionError of ``fn(*args)`` and goes on; ``chk.add`` records a hash of a result that every rank
    must hold bit for bit, and ``chk.finish()`` compares those over the control plane (gloo)."""

    def __init__(self):
        self.rows = []
        self.failures = []

    def __call__(self, fn, *args):
        try:
            fn(*args)
        except AssertionError as exc:
            self.failures.append(str(exc))

    def add(self, label, t):
        self.rows.append((label, _digest(t)))

    def finish(self):
        if size > 1:
            out = [None] * size
            dist.all_gather_object(out, self.rows, group=comm._group)
            for q, rows in enumerate(out):
                for (label, h), (_, h0) in zip(rows, out[0]):
                    self(_expect, h == h0, f"{label}: rank {q}'s result differs from rank 0's")
                self(_expect, len(rows) == len(out[0]), f"rank {q} checked {len(rows)} results, rank 0 {len(out[0])}")
        assert not self.failures, f"{len(self.failures)} checks failed on rank {rank}, the first:\n{self.failures[0]}"


def _expect(ok, message):
    assert ok, message


# ---------------------------------------------------------------------------
# communicator options and the transport a call took
# ---------------------------------------------------------------------------
@contextlib.contextmanager
def _options(device, **opts):
    """Set native communicator options for the block and restore every one afterwards."""
    nc = comm._native_comm() if device.type == "cuda" else None
    old = {k: nc.get_option(k) for k in opts} if nc is not None else {}
    try:
        for k, v in opts.items():
            if nc is not None:
                nc.set_option(k, v)
        yield nc
    finally:
        m.flush()
        for k, v in old.items():
            nc.set_option(k, v)
    for k, v in old.items():
        assert nc.get_option(k) == v, k


def _logged(capsys, device, opname, fn):
    """(fn(), the transport named by the debug line of the ``MPI_<opname>`` call; None on CPU)."""
    if device.type != "cuda":
        return fn(), None
    capsys.readouterr()
    set_logging(True)
    try:
        out = fn()
    finally:
        set_logging(False)
    lines = re.findall(rf"^r{rank} \| \w{{8}} \| MPI_{opname} \(GPU\) with .* via (\w+)$", capsys.readouterr().out,
                       re.M)
    return out, lines[0] if len(lines) == 1 else f"{len(lines)} MPI_{opname} log lines {lines}"


def _auto_transport(nc, nbytes):
    """What the size table picks for an allreduce of ``nbytes`` (csrc/b2_collectives.cu: reduce_algo)."""
    if size > 1 and nbytes <= nc.get_option("ll_max") and nbytes <= LL_BYTES:
        return "ll"
    if size <= 2 or nbytes <= nc.get_option("oneshot_max"):
        return "oneshot"          # (no multicast when ranks share a GPU; nvls_min is not consulted then)
    return "twoshot"


def _n_for(nbytes, dtype):
    return max(1, nbytes // dtype.itemsize)


# ---------------------------------------------------------------------------
# allreduce
# ---------------------------------------------------------------------------
def _run_allreduce(device, capsys, chk, case, dtype, opname, n, algo, xs=None):
    xs = xs or [_input(case, q, n, dtype, opname) for q in range(size)]
    nbytes = n * dtype.itemsize
    label = f"allreduce algorithm={algo} {dtype} {opname} n={n} ({nbytes} B) P={size}"
    x = xs[rank].to(device)
    x0 = x.clone()
    res, via = _logged(capsys, device, "Allreduce",
                       lambda: m.allreduce(x, getattr(MPI, opname), comm=comm, algorithm=algo))
    if via is not None:
        want_via = _auto_transport(comm._native_comm(), nbytes) if algo == "auto" else algo
        chk(_expect, via == want_via, f"{label}: took the {via} transport, expected {want_via}")
    chk(_assert_same, res, _fold(xs, opname), label)
    if dtype.is_floating_point or dtype.is_complex:
        chk(_check_accuracy, res.cpu(), xs, opname, label)
    chk(_assert_same, x, x0, f"{label}: input changed")
    chk.add(label, res)


ALGOS = ("ll", "oneshot", "twoshot", "auto")
ALL_DTYPES = tuple(codes.DTYPE_CODE)


@peers
def test_allreduce_every_dtype_op_and_transport(device, capsys):
    """Every dtype x op x forced transport at 1 element, 17 B and 4095 B (odd vector counts, tails)."""
    chk = _Checks()
    for algo in ALGOS:
        for dtype in ALL_DTYPES:
            for opname in _ops_for(dtype) if dtype != torch.bool else OPS:
                for nbytes in (1, 17, 4095):
                    n = _n_for(nbytes, dtype)
                    _run_allreduce(device, capsys, chk, ("matrix", algo, str(dtype), opname, n),
                                   dtype, opname, n, algo)
    chk.finish()


@peers
def test_allreduce_sizes_around_vector_and_ll_limits(device, capsys):
    """15 / 16 / 17 B, 4095 B, just below and at the LL capacity, and past it (auto: one-shot or two-shot)."""
    chk = _Checks()
    cases = ((torch.float32, "SUM"), (torch.bfloat16, "SUM"), (torch.float16, "PROD"), (torch.int8, "SUM"),
             (torch.uint64, "MAX"), (torch.complex128, "SUM"), (torch.int32, "BXOR"))
    for algo in ALGOS:
        for dtype, opname in cases:
            for nbytes in (15, 16, 17, 4095, LL_BYTES - 16, LL_BYTES, LL_BYTES + 16, (LL_BYTES << 3) + 48):
                if algo == "ll" and nbytes > LL_BYTES:
                    continue
                n = _n_for(nbytes, dtype)
                _run_allreduce(device, capsys, chk, ("sizes", algo, str(dtype), opname, n), dtype, opname, n, algo)
    chk.finish()


@peers
def test_allreduce_multichunk_with_one_or_two_ctas(device, capsys):
    """max_blocks 1 and 2 with 2-4 MiB: chunks are capped at 512 KiB, so every CTA walks several chunks
    (the ``ch += gridDim.x`` loops and a barrier epoch per chunk), in the one-shot and two-shot kernels."""
    chk = _Checks()
    for blocks, nbytes in ((1, (2 << 20) + 16), (2, (3 << 20) + 4), (2, 4 << 20)):
        with _options(device, max_blocks=blocks):
            for algo in ("oneshot", "twoshot"):
                for dtype, opname in ((torch.float32, "SUM"), (torch.bfloat16, "SUM"), (torch.int16, "MAX")):
                    n = _n_for(nbytes, dtype)
                    _run_allreduce(device, capsys, chk, ("chunks", blocks, algo, str(dtype), n), dtype, opname,
                                   n, f"{algo}")
    chk.finish()


def _edge_cases():
    """(name, dtype, op, per-rank inputs) of values where kernels go wrong."""
    n = 37
    out = []
    for dtype in (torch.float16, torch.bfloat16, torch.float32, torch.float64):
        for opname in ("MIN", "MAX"):
            xs = [_input(("nan", str(dtype), opname), q, n, dtype) for q in range(size)]
            xs[size - 1][3] = float("nan")                  # NaN in one rank only
            xs[0][5] = float("nan")
            xs[size // 2][7] = float("nan")
            out.append((f"NaN {opname}", dtype, opname, xs))
        specials = torch.tensor([float("inf"), -float("inf"), 0.0, -0.0, 1.0, -1.0], dtype=torch.float64)
        xs = [specials.roll(q).to(dtype) for q in range(size)]
        for opname in ("SUM", "PROD", "MIN", "MAX"):
            out.append((f"inf/signed zero {opname}", dtype, opname, xs))
    tiny = torch.finfo(torch.float32).tiny
    sub = [torch.tensor([tiny / 8 * (q + 1), -tiny / 4, tiny / 2 ** 20, 3 * tiny / 16], dtype=torch.float32)
           for q in range(size)]
    for opname in ("SUM", "MIN", "MAX"):
        out.append((f"fp32 subnormals {opname}", torch.float32, opname, sub))
    out.append(("fp32 subnormals PROD", torch.float32, "PROD",
                [torch.tensor([tiny / 8, 1.0 + q / 8, 2.0 ** -10], dtype=torch.float32) for q in range(size)]))
    for dtype in SIGNED:
        info = torch.iinfo(dtype)
        base = torch.tensor([info.min, info.max, -1, 0, 1, info.min + 1, info.max - 1], dtype=torch.int64)
        xs = [base.roll(q).to(dtype) for q in range(size)]
        for opname in OPS:
            out.append((f"INT_MIN/INT_MAX {opname}", dtype, opname, xs))
    hi = np.array([2 ** 63, 2 ** 64 - 1, 2 ** 63 - 1, 1, 0, 2 ** 63 + 5], dtype=np.uint64)
    xs = [torch.from_numpy(np.roll(hi, q).copy()) for q in range(size)]
    for opname in ("MIN", "MAX", "SUM", "PROD"):
        out.append((f"uint64 >= 2^63 {opname}", torch.uint64, opname, xs))
    for dtype in (torch.int8, torch.uint8, torch.uint16):
        for opname in ("SUM", "PROD"):
            xs = [_input(("wrap", str(dtype), opname), q, 64, dtype, opname) for q in range(size)]
            out.append((f"wrapping {opname}", dtype, opname, xs))
    return out


@peers
def test_allreduce_edge_values(device, capsys):
    """NaN in one rank (MIN / MAX propagate it like numpy), +-inf and +-0.0, fp32 subnormals (no flush
    to zero), INT_MIN / INT_MAX, uint64 values >= 2^63 (an unsigned comparison), wrapping int8 / uint8 /
    uint16 sums and products -- through every transport."""
    chk = _Checks()
    for algo in ALGOS:
        for name, dtype, opname, xs in _edge_cases():
            _run_allreduce(device, capsys, chk, None, dtype, opname, xs[0].numel(), algo, xs=xs)
    chk.finish()


@three_or_more
def test_allreduce_nvls(device):
    """The in-switch allreduce and reduce (SUM of f32 / bf16 / f16) need a multicast object, which binds
    every device once: only on >= 3 ranks with distinct GPUs."""
    nc = comm._native_comm() if device.type == "cuda" else None
    if nc is None or size < 3 or not nc.has_nvls:
        pytest.skip("NVLS needs >= 3 ranks on distinct GPUs with multicast support")
    chk = _Checks()
    for dtype in (torch.float32, torch.bfloat16, torch.float16):
        n = (1 << 20) // dtype.itemsize + 8
        xs = [_input(("nvls", str(dtype)), q, n, dtype) for q in range(size)]
        res = m.allreduce(xs[rank].to(device), MPI.SUM, comm=comm, algorithm="nvls")
        chk(_check_accuracy, res.cpu(), xs, "SUM", f"allreduce algorithm=nvls {dtype} SUM n={n} P={size}")
        chk.add(f"nvls {dtype}", res)
    chk.finish()


# ---------------------------------------------------------------------------
# reduce and scan
# ---------------------------------------------------------------------------
@peers
def test_reduce_roots_dtypes_and_sizes(device, capsys):
    """Roots 0 and P-1; the root gets the rank-order fold, every other rank its input back (its kernel
    runs with has_out = 0)."""
    chk = _Checks()
    for root in sorted({0, size - 1}):
        for dtype in ALL_DTYPES:
            for opname in _ops_for(dtype):
                for nbytes in (1, 17, 4095, LL_BYTES + 16):
                    if nbytes > 4095 and opname not in ("SUM", "MAX"):
                        continue
                    n = _n_for(nbytes, dtype)
                    xs = [_input(("reduce", root, str(dtype), opname, n), q, n, dtype, opname) for q in range(size)]
                    label = f"reduce root={root} {dtype} {opname} n={n} ({n * dtype.itemsize} B) P={size}"
                    x = xs[rank].to(device)
                    x0 = x.clone()
                    res, via = _logged(capsys, device, "Reduce", lambda: m.reduce(x, getattr(MPI, opname), root,
                                                                               comm=comm))
                    chk(_expect, via in (None, "oneshot"), f"{label}: took the {via} transport")
                    if rank == root:
                        chk(_assert_same, res, _fold(xs, opname), label)
                        if dtype.is_floating_point:
                            chk(_check_accuracy, res.cpu(), xs, opname, label)
                    else:
                        chk(_expect, res is x, f"{label}: a non-root rank gets its input back")
                    chk(_assert_same, x, x0, f"{label}: input changed")
    chk.finish()


def _check_scan(device, capsys, chk, case, dtype, opname, n, want_via):
    xs = [_input(case, q, n, dtype, opname) for q in range(size)]
    label = f"scan {want_via} {dtype} {opname} n={n} ({n * dtype.itemsize} B) P={size}"
    x = xs[rank].to(device)
    x0 = x.clone()
    res, via = _logged(capsys, device, "Scan", lambda: m.scan(x, getattr(MPI, opname), comm=comm))
    chk(_expect, via in (None, want_via), f"{label}: took the {via} transport")
    chk(_assert_same, res, _fold(xs[: rank + 1], opname), f"{label} (prefix of rank {rank})")
    if dtype.is_floating_point:
        chk(_check_accuracy, res.cpu(), xs[: rank + 1], opname, label)
    chk(_assert_same, x, x0, f"{label}: input changed")


SCAN_CASES = ((torch.float32, "SUM"), (torch.bfloat16, "SUM"), (torch.float64, "PROD"), (torch.int32, "SUM"),
              (torch.int8, "PROD"), (torch.uint64, "MAX"), (torch.float16, "MIN"), (torch.int16, "BXOR"),
              (torch.bool, "LXOR"), (torch.complex64, "SUM"))


@peers
def test_scan_one_phase(device, capsys):
    """Rank r pulls the copies of ranks 0..r; random data, each prefix against its own rank-order fold."""
    chk = _Checks()
    for dtype, opname in SCAN_CASES:
        for nbytes in (1, 17, 4095, LL_BYTES + 48):
            n = _n_for(nbytes, dtype)
            _check_scan(device, capsys, chk, ("scan1", str(dtype), opname, n), dtype, opname, n, "oneshot")
    chk.finish()


@three_or_more
def test_scan_two_phase(device, capsys):
    """P >= 3 with oneshot_max below the message: rank s computes every prefix of sub-slice s and
    writes prefix q into rank q's staging (B2_OPC_SCAN); with one CTA, over several chunks."""
    chk = _Checks()
    for blocks, sizes in ((None, (17, 4095, 20000)), (1, ((1 << 20) + 16,))):
        opts = dict(oneshot_max=8) if blocks is None else dict(oneshot_max=8, max_blocks=blocks)
        with _options(device, **opts):
            for dtype, opname in SCAN_CASES:
                for nbytes in sizes:
                    n = _n_for(nbytes, dtype)
                    _check_scan(device, capsys, chk, ("scan2", blocks, str(dtype), opname, n), dtype, opname, n,
                                "twoshot" if n * dtype.itemsize > 8 else "oneshot")
    chk.finish()


# ---------------------------------------------------------------------------
# kernels back to back: staging parity, LL flag parity and per-CTA epochs across any mix
# ---------------------------------------------------------------------------
def _mixed_sequence(xa, xb, xc, xd):
    a = m.allreduce(xa, MPI.SUM, comm=comm, algorithm="ll")
    b = m.allreduce(xb, MPI.SUM, comm=comm, algorithm="twoshot")
    c = m.reduce(xc, MPI.MAX, size - 1, comm=comm)
    d = m.scan(xb, MPI.SUM, comm=comm)
    e = m.allgather(xd, comm=comm)
    f = m.allreduce(xc, MPI.PROD, comm=comm, algorithm="ll")
    g = m.allreduce(xa, MPI.MAX, comm=comm, algorithm="oneshot")
    h = m.allreduce(xd, MPI.BXOR, comm=comm, algorithm="ll")
    return a, b, c, d, e, f, g, h


def _mixed_inputs(call):
    shapes = ((33, torch.float32, "SUM"), (5000, torch.float32, "SUM"), (77, torch.float64, "PROD"),
              (1000, torch.int32, "SUM"))
    return [[_input(("mixed", call, k), q, n, dt, op) for q in range(size)] for k, (n, dt, op) in enumerate(shapes)]


def _mixed_oracle(ins):
    xa, xb, xc, xd = ins
    return (_fold(xa, "SUM"), _fold(xb, "SUM"), _fold(xc, "MAX") if rank == size - 1 else xc[rank],
            _fold(xb[: rank + 1], "SUM"), torch.stack(xd), _fold(xc, "PROD"), _fold(xa, "MAX"), _fold(xd, "BXOR"))


@peers
def test_mixed_call_sequences_eager_and_jit(device):
    """allreduce LL -> two-shot -> reduce -> scan -> allgather -> LL ... with different sizes, eagerly
    and as a captured CUDA graph replayed with new inputs (m.jit: warm-up, capture, replays)."""
    chk = _Checks()
    names = ("allreduce ll", "allreduce twoshot", "reduce", "scan", "allgather", "allreduce ll PROD",
             "allreduce oneshot MAX", "allreduce ll BXOR")
    f = m.jit(_mixed_sequence)
    for call in range(5):
        ins = _mixed_inputs(call)
        args = [x[rank].to(device) for x in ins]
        for mode, fn in (("eager", _mixed_sequence), ("jit", f)):
            got = fn(*args)
            for name, g, w in zip(names, got, _mixed_oracle(ins)):
                chk(_assert_same, g, w, f"mixed sequence call {call} {mode}: {name} P={size}")
                if name not in ("reduce", "scan"):             # (the others hold the same bits on every rank)
                    chk.add(f"{call} {mode} {name}", g)
    chk.finish()


@peers
def test_reduce_scatter_names_its_transport(device, capsys):
    """reduce_scatter sends a block within ll_max by LL and pulls it through the staging otherwise
    (ll_max = 0); the debug line names the transport either way."""
    chk = _Checks()
    for ll_max, want_via in ((1 << 30, "ll"), (0, "oneshot")):
        with _options(device, ll_max=ll_max):
            xs = [_input(("rs", ll_max), q, size * 33, torch.float32).reshape(size, 33) for q in range(size)]
            x = xs[rank].to(device)
            res, via = _logged(capsys, device, "Reduce_scatter_block", lambda: m.reduce_scatter(x, MPI.SUM, comm=comm))
            label = f"reduce_scatter {want_via} torch.float32 SUM 33 items per block P={size}"
            chk(_expect, via in (None, want_via), f"{label}: took the {via} transport")
            chk(_assert_same, res, _fold([xq[rank] for xq in xs], "SUM"), label)
    chk.finish()


# ---------------------------------------------------------------------------
# data movement: bcast, gather, scatter, allgather, alltoall (b2_k_move)
# ---------------------------------------------------------------------------
MOVE_DTYPES = (torch.uint8, torch.bfloat16, torch.float32, torch.float64, torch.complex128)   # 1, 2, 4, 8, 16 B


def _bits(shape, dtype, case, q):
    """Arbitrary bit patterns (NaN payloads included): the movers must copy them exactly."""
    nbytes = int(np.prod(shape, dtype=np.int64)) * dtype.itemsize
    raw = torch.from_numpy(np.frombuffer(_rng(case, q).bytes(nbytes), dtype=np.uint8).copy())
    return raw.view(dtype).reshape(shape)


def _same_bytes(got, want, label):
    got = got.detach().cpu().contiguous()
    assert got.shape == want.shape and got.dtype == want.dtype, (label, got.shape, want.shape)
    g, w = got.view(torch.uint8).reshape(-1), want.contiguous().view(torch.uint8).reshape(-1)
    diff = g != w
    assert not diff.any(), f"{label}: {int(diff.sum())} bytes differ, first at byte {int(diff.nonzero()[0])}"


def _move_all(device, chk, case, shape, dtype, make=None, roots=None):
    """bcast / gather / scatter / allgather / alltoall of rank inputs of ``shape`` (``make(t)``: the view of
    a locally built base tensor that is passed, e.g. a transpose); byte-exact against the inputs."""
    make = make or (lambda t: t)
    label = f"{case} {dtype} shape={tuple(shape)} P={size}"
    roots = roots if roots is not None else sorted({size - 1, 1 % size})
    bases = [_bits(shape, dtype, case, q) for q in range(size)]
    views = [make(b) for b in bases]                 # the logical value rank q passes
    want = [v.contiguous() for v in views]
    mine = make(bases[rank].to(device))
    mine0 = mine.clone()
    # allgather
    g = m.allgather(mine, comm=comm)
    chk(_same_bytes, g, torch.stack(want), f"allgather {label}")
    chk.add(f"allgather {label}", g)
    for root in roots:
        # bcast (the root's contiguous buffer)
        src = want[rank].to(device) if rank == root else torch.empty(want[0].shape, dtype=dtype, device=device)
        chk(_same_bytes, m.bcast(src, root, comm=comm), want[root], f"bcast root={root} {label}")
        # gather
        r = m.gather(mine, root, comm=comm)
        if rank == root:
            chk(_same_bytes, r, torch.stack(want), f"gather root={root} {label}")
        else:
            chk(_expect, r is mine, f"gather root={root} {label}: a non-root rank gets its input back")
    chk(_same_bytes, mine, mine0.cpu(), f"{label}: input changed")


def _move_lead(device, chk, case, shape, dtype, make=None, roots=None):
    """alltoall and scatter, whose inputs are (P, *block): block q goes to rank q."""
    make = make or (lambda t: t)
    label = f"{case} {dtype} shape={tuple(shape)} P={size}"
    roots = roots if roots is not None else sorted({size - 1, 1 % size})
    bases = [_bits(shape, dtype, case, q) for q in range(size)]
    views = [make(b) for b in bases]
    assert views[0].shape[0] == size
    mine = make(bases[rank].to(device))
    mine0 = mine.clone()
    a = m.alltoall(mine, comm=comm)
    chk(_same_bytes, a, torch.stack([views[q][rank] for q in range(size)]), f"alltoall {label}")
    for root in roots:
        x = mine if rank == root else torch.empty(views[0].shape[1:], dtype=dtype, device=device)
        chk(_same_bytes, m.scatter(x, root, comm=comm), views[root][rank], f"scatter root={root} {label}")
    chk(_same_bytes, mine, mine0.cpu(), f"{label}: input changed")


@peers
def test_move_element_sizes_and_tails(device):
    """Element sizes 1 / 2 / 4 / 8 / 16, blocks of 1, 15, 17 elements (tails), 256 elements (whole
    vectors: the fused pull-and-stage loop), roots != 0."""
    chk = _Checks()
    for dtype in MOVE_DTYPES:
        for n in (1, 15, 17, 256):
            _move_all(device, chk, ("tails", n), (n,), dtype)
            _move_lead(device, chk, ("tails lead", n), (size, n), dtype)
    chk.finish()


@peers
def test_move_multichunk_one_cta(device):
    """max_blocks = 1 and blocks above 512 KiB: one CTA walks several chunks and stages the next one
    while it pulls the current one (b2_k_move's software pipeline), with and without a tail."""
    chk = _Checks()
    with _options(device, max_blocks=1):
        for dtype, n in ((torch.uint8, (1 << 20) + 17), (torch.float32, (600 << 10) // 4 * 3),
                         (torch.complex128, (1 << 20) // 16 + 1)):
            _move_all(device, chk, ("chunks", n), (n,), dtype, roots=[size - 1])
            _move_lead(device, chk, ("chunks lead", n), (size, n), dtype, roots=[size - 1])
    chk.finish()


@peers
def test_move_strided_inputs(device):
    """Non-contiguous inputs that the movers gather element by element while they stage (the fused
    pack): a transpose, a stepped slice whose base is not 16-byte aligned, a lead stride other than the
    block size, a 4-d layout that does not merge, and a 5-d one (packed by a copy instead)."""
    chk = _Checks()
    for dtype in MOVE_DTYPES:
        _move_all(device, chk, "transpose", (7, 12), dtype, make=lambda t: t.t())
        _move_all(device, chk, "stepped slice", (2 * 45 + 1,), dtype, make=lambda t: t[1::2])
        _move_all(device, chk, "4-d permuted", (5, 4, 3, 2), dtype, make=lambda t: t.permute(3, 2, 1, 0))
        _move_all(device, chk, "5-d permuted", (3, 2, 3, 2, 2), dtype, make=lambda t: t.permute(4, 3, 2, 1, 0))
        _move_lead(device, chk, "lead stride", (size, 21), dtype, make=lambda t: t[:, 2:19])
        _move_lead(device, chk, "lead transpose", (size, 6, 5), dtype, make=lambda t: t.transpose(1, 2))
        _move_lead(device, chk, "lead stepped", (size, 31), dtype, make=lambda t: t[:, 1::2])
        _move_lead(device, chk, "lead 4-d", (size, 5, 4, 3, 2), dtype, make=lambda t: t.permute(0, 4, 3, 2, 1))
        _move_lead(device, chk, "lead 5-d", (size, 3, 2, 3, 2, 2), dtype,
                   make=lambda t: t.permute(0, 5, 4, 3, 2, 1))
    chk.finish()


@three_or_more
def test_move_bcast_multicast(device):
    """The multicast bcast (forced with bcast_mc_min) needs a multicast object: >= 3 ranks on distinct GPUs."""
    nc = comm._native_comm() if device.type == "cuda" else None
    if nc is None or size < 3 or not nc.has_nvls:
        pytest.skip("the multicast bcast needs >= 3 ranks on distinct GPUs with multicast support")
    chk = _Checks()
    with _options(device, bcast_mc_min=16):
        for n in (16, 4096 + 3, (1 << 20) + 5):
            want = _bits((n,), torch.uint8, "mc", size - 1)
            src = want.to(device) if rank == size - 1 else torch.empty(n, dtype=torch.uint8, device=device)
            chk(_same_bytes, m.bcast(src, size - 1, comm=comm), want, f"multicast bcast n={n} P={size}")
    chk.finish()


# ---------------------------------------------------------------------------
# the same tests with three and five ranks
# ---------------------------------------------------------------------------
_inside_job = size > 1 or "MPI4JAX_B200_NESTED" in os.environ


def _job(nranks, select, env):
    from mpi4jax_b200.run import launch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    repo = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    test_file = os.path.relpath(os.path.abspath(__file__), repo)
    args = ["-m", "pytest", test_file, "-q", "-rp", "-m", "gpu", "-k", select, "-p", "no:cacheprovider"]
    cwd = os.getcwd()
    os.chdir(repo)
    try:
        with tempfile.TemporaryDirectory(prefix=f"mpi4jax-b200-kernels-{nranks}-") as logs:
            code, _ = launch(nranks, args, timeout=900, output_dir=logs,
                             env_extra={"MPI4JAX_B200_NESTED": "1", **env})
            outs = [open(os.path.join(logs, f"rank{r}.log")).read() for r in range(nranks)]
    finally:
        os.chdir(cwd)
    return code, outs


def _expect_passed(code, outs, nranks, tests):
    for r, out in enumerate(outs):
        missing = [t for t in tests if not re.search(rf"^PASSED .*::{t}\[cuda\]", out, re.M)]
        assert code == 0 and not missing, \
            f"rank {r} of the {nranks}-rank job (exit code {code}), not passed: {missing}:\n{out[-4000:]}"


@pytest.mark.gpu
@pytest.mark.skipif(_inside_job, reason="already inside a multi-rank job")
def test_collective_kernels_three_ranks_gpu():
    """P = 3: a non-power-of-two world (chunk unit 48 B, uneven two-shot splits), the two-phase scan,
    and the <3,1,2> (allgather) and <4,4,1> (alltoall) pull-and-stage loops."""
    code, outs = _job(3, "not nvls and not multicast", {})
    _expect_passed(code, outs, 3, [
        "test_allreduce_every_dtype_op_and_transport", "test_allreduce_sizes_around_vector_and_ll_limits",
        "test_allreduce_multichunk_with_one_or_two_ctas", "test_allreduce_edge_values",
        "test_reduce_roots_dtypes_and_sizes", "test_scan_one_phase", "test_scan_two_phase",
        "test_mixed_call_sequences_eager_and_jit", "test_reduce_scatter_names_its_transport",
        "test_move_element_sizes_and_tails",
        "test_move_multichunk_one_cta", "test_move_strided_inputs"])


@pytest.mark.gpu
@pytest.mark.skipif(_inside_job, reason="already inside a multi-rank job")
def test_collective_kernels_five_ranks_gpu():
    """P = 5, data movement only: the <8,1,1> (allgather) and <8,8,1,SPLIT> (alltoall) instantiations,
    which otherwise need >= 5 GPUs.  Smaller p2p ring slots keep five contexts' rings small."""
    code, outs = _job(5, "test_move_element_sizes_and_tails or test_move_multichunk_one_cta",
                      {"MPI4JAX_B200_P2P_SLOT_BYTES": "1048576"})
    _expect_passed(code, outs, 5, ["test_move_element_sizes_and_tails", "test_move_multichunk_one_cta"])
