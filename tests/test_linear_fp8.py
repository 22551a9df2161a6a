"""Scaled float8 linear layers (``scale_x`` / ``scale_w`` of ``ops.linear_allreduce``, ``linear_reduce_scatter``
and ``linear_allgather``): the e4m3 wgmma kernels of csrc/b2_gemm_f8.cu and the fallback, against oracles
that never call the library.

Rank q's operands and scales come from a seed of (case, q), so every rank rebuilds every rank's and
computes the expected result itself, in float64.  The operands are the small integers of
tests/test_gemm.py in float8 (|x| <= 3, |w| <= 4, every |S| <= 2^11: exact in any accumulator of 12 or more
bits) and the scales powers of two in [2^-2, 2^2], one per tensor or one per row / column by rank.  So
rank q's partial ``rn_bf16(S_q * sx_q[i] * sw_q[j])`` is exact in float64, the partials' fp32 sum is exact
(magnitudes in [2^-4, 2^18)), and the kernels and the fallback must match the oracle to the bit.

The bound test uses normal float8 operands, arbitrary scales and this accumulator model: the float8
wgmma adds each 32-wide k-slice into the fp32 accumulators keeping at least 13 significant bits, so each
of the K / 32 additions errs by at most 2^-12 sum_k |x w| (DESIGN section 3, scaled float8).

The tests that take ``device`` run at world size 1 and in jobs launched from this file: 2 and 3 CPU ranks,
and on the GPUs there are 2 ranks (sharing the GPU when there is one), 2 ranks with NVLS off, and 3 to 8
ranks when there are that many GPUs."""

import os
import re
import subprocess
import sys

import pytest
import torch

import mpi4jax_b200 as m
from mpi4jax_b200 import MPI
from mpi4jax_b200.ops import linear_allgather, linear_allreduce, linear_reduce_scatter

from ._peer_job import REPO, Checks, job
from .test_gemm import CASES, TILE, _assert_same, _expect, _gen, _offset_view, _sm_count, _ulp_bf16, exact_operands

comm = MPI.COMM_WORLD
rank, size = comm.Get_rank(), comm.Get_size()
inside_job = size > 1 or "MPI4JAX_B200_NESTED" in os.environ

E4M3, E5M2 = torch.float8_e4m3fn, torch.float8_e5m2
OPS = {"allreduce": linear_allreduce, "reduce_scatter": linear_reduce_scatter, "allgather": linear_allgather}
F8_METHODS = ("gemm_allreduce_f8", "gemm_reduce_scatter_f8", "gemm_allgather_f8")


@pytest.fixture
def kernel_calls(monkeypatch):
    """Shapes (rows, N, K) of every call of the six GEMM entry points while the test runs, by entry point."""
    from mpi4jax_b200._src.backends.cuda import NativeComm

    calls = {n: [] for n in ("gemm_allreduce", "gemm_reduce_scatter", "gemm_allgather") + F8_METHODS}
    for name in calls:
        real = getattr(NativeComm, name)

        def spy(self, x, weight, *scales, _real=real, _name=name):
            calls[_name].append((x.shape[0], weight.shape[0], x.shape[1]))
            return _real(self, x, weight, *scales)

        monkeypatch.setattr(NativeComm, name, spy)
    return calls


def _fused_method(op, device, dx, dw, rows, N):
    """The NativeComm method a scaled call must run, or None for the fallback.  ``rows``: M of the
    allreduce and reduce-scatter, m of the allgather.  The forms of the scales play no part."""
    if device.type != "cuda" or dx != E4M3 or dw != E4M3 or comm.transport != "native" or rows == 0:
        return None
    if op == "allgather":
        return None if (size * rows) % TILE else ("gemm_allreduce_f8" if size == 1 else "gemm_allgather_f8")
    if N == 0 or rows % TILE or N % TILE:
        return None
    if size == 1:
        return "gemm_allreduce_f8"
    if op == "allreduce":
        return "gemm_allreduce_f8" if comm._native_comm().has_nvls else None
    return "gemm_reduce_scatter_f8"


def _check_path(chk, calls, method, label, n=1):
    """``method`` ran ``n`` times and no other GEMM entry point did (all of them when ``method`` is None)."""
    ran = {k: len(v) for k, v in calls.items() if v}
    want = {method: n} if method else {}
    chk(_expect, ran == want, f"{label}: GEMM entry points ran {ran}, expected {want}")
    for v in calls.values():
        v.clear()


# ---------------------------------------------------------------------------
# operands, scales and the oracle
# ---------------------------------------------------------------------------
def f8_operands(case, q, M, N, K, device, dx=E4M3, dw=E4M3):
    x, w = exact_operands(case, q, M, N, K, device, torch.float32)
    return x.to(dx), w.to(dw)


def pow2_scales(case, q, M, N, device, form=None):
    """Rank q's scales: powers of two in [2^-2, 2^2], per tensor or per row / column.  ``form`` = (x per row,
    w per column); by default it differs between neighbouring ranks."""
    gen = _gen(f"{case}/scales", q, device)
    fx, fw = form if form is not None else (q % 2 == 1, q % 3 != 1)
    sx = torch.exp2(torch.randint(-2, 3, (M,) if fx else (), generator=gen, device=device).float())
    sw = torch.exp2(torch.randint(-2, 3, (N,) if fw else (), generator=gen, device=device).float())
    return sx, sw


def partial(x, w, sx, sw):
    """``rn_bf16(S * (sx[i] * sw[j]))`` with S and the scaling in float64 (exact for the operands here)."""
    S = x.double() @ w.double().t()
    return (S * (sx.double().reshape(-1, 1) * sw.double().reshape(1, -1))).to(torch.bfloat16)


def want_sum(parts):
    """``rn(sum_q P_q)``: exact here, so the same as the fp32 sum rounded once."""
    return sum(p.double() for p in parts).to(torch.bfloat16)


class Case:
    """One scaled call of ``op`` on every rank: rank q's operands ``(x_q, w_q)`` and scales ``(sx_q, sw_q)``
    (``ks[q]``: rank q's K, allreduce and reduce-scatter only), this rank's arguments, and the expected
    result."""

    def __init__(self, op, label, rows, N, K, device, ks=None, form=None, dx=E4M3, dw=E4M3, edit=None):
        self.op, self.label, self.rows, self.N = op, label, rows, N
        ks = ks or [K] * size
        self.ops = [f8_operands(label, q, rows, N, ks[q], device, dx, dw) for q in range(size)]
        self.scales = [pow2_scales(label, q, rows, N, device, form) for q in range(size)]
        if edit is not None:
            for q in range(size):
                edit(q, self.ops[q], self.scales[q])
        self.x, self.w = self.ops[rank]
        self.sx, self.sw = self.scales[rank]

    def want(self):
        if self.op == "allgather":
            X = torch.cat([x for x, _ in self.ops])
            SX = torch.cat([sx.expand(self.rows) for sx, _ in self.scales])
            return partial(X, self.w, SX, self.sw)
        full = want_sum([partial(x, w, sx, sw) for (x, w), (sx, sw) in zip(self.ops, self.scales)])
        if self.op == "reduce_scatter":
            r = self.rows // size
            return full[rank * r:(rank + 1) * r]
        return full

    def run(self, x=None, w=None, sx=None, sw=None):
        return OPS[self.op](self.x if x is None else x, self.w if w is None else w, comm=comm,
                            scale_x=self.sx if sx is None else sx, scale_w=self.sw if sw is None else sw)


def _rows(op, num_m):
    """M (allreduce, reduce-scatter: tile rows rounded up to a multiple of P) or m (allgather) of a grid."""
    tiles = -(-num_m // size) * size
    return tiles * TILE // size if op == "allgather" else tiles * TILE


def _over_rasters(case, device):
    """[(gemm_raster, output)] over the tile orders auto, 0, 1, 2, 3, 5 and 17; one call where there is no
    native communicator."""
    if device.type != "cuda" or comm.transport != "native":
        return [("auto", case.run())]
    nc = comm._native_comm()
    outs = []
    try:
        for r in (-1, 0, 1, 2, 3, 5, 17):
            nc.set_option("gemm_raster", r)
            outs.append((r, case.run()))
    finally:
        nc.set_option("gemm_raster", -1)
    return outs


def _same_bits(outs, label):
    first = outs[0][1].contiguous().view(torch.int16)
    for r, out in outs[1:]:
        assert torch.equal(out.contiguous().view(torch.int16), first), f"{label}: {r} and {outs[0][0]} differ in bits"


def _exercises_every_k32(case, M, N, K, device):
    """Outputs between 257 and 2048 (where bf16 rounds), odd ones among them, and a nonzero of x in every
    32-wide k-slice of a row with such outputs: a k-slice of a wgmma or a 128-wide k-block that the kernel
    drops, misplaces or reads twice changes outputs."""
    x, w = f8_operands(case, 0, M, N, K, device)
    s = (x.double() @ w.double().t()).abs()
    mid = (s > 256) & (s <= 2 ** 11)
    assert mid.any() and (mid & (s % 2 == 1)).any(), (case, s.max().item())
    hit = (x[mid.any(1)].float() != 0).reshape(-1, K // 32, 32).any(2).any(0)
    assert hit.all(), f"{case}: k32 slices {(~hit).nonzero().flatten().tolist()} hold no nonzero of such a row"


# ---------------------------------------------------------------------------
# exact mode
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("op", list(OPS))
def test_scaled_exact(op, device, kernel_calls):
    """Every CASES grid in every tile order, scales per tensor and per row / column differing between ranks,
    to the bit; the same bits in every tile order and on every rank."""
    chk = Checks()
    g = _sm_count(device)
    for label, grid, K in CASES:
        num_m, num_n = grid(g)
        rows, N = _rows(op, num_m), num_n * TILE
        _exercises_every_k32(label, num_m * TILE, N, K, device)
        case = Case(op, label, rows, N, K, device)
        outs = _over_rasters(case, device)
        want = case.want()
        for r, out in outs:
            chk(_assert_same, out, want, f"{op} {label} ({rows} x {N} x {K}), gemm_raster {r}")
        chk(_same_bits, outs, label)
        _check_path(chk, kernel_calls, _fused_method(op, device, E4M3, E4M3, rows, N), label, len(outs))
        if op == "allreduce":
            chk.add(label, outs[0][1])
    chk.finish()


@pytest.mark.parametrize("op", list(OPS))
def test_equals_the_bf16_kernel_times_the_scale(op, device, kernel_calls):
    """One power-of-two per-tensor scale pair on every rank: the float8 result is the bf16 op on the same
    integers times that power of two, bit for bit."""
    chk = Checks()
    g = _sm_count(device)
    for label, grid, K in (CASES[2], CASES[4], CASES[5]):
        num_m, num_n = grid(g)
        rows, N = _rows(op, num_m), num_n * TILE
        case = Case(op, label, rows, N, K, device)
        sx, sw = torch.tensor(4.0, device=device), torch.tensor(0.125, device=device)
        got = case.run(sx=sx, sw=sw)
        ref = OPS[op](case.x.to(torch.bfloat16), case.w.to(torch.bfloat16), comm=comm)
        chk(_expect, torch.equal(got.view(torch.int16), (ref.double() * 0.5).to(torch.bfloat16).view(torch.int16)),
            f"{op} {label}: float8 result and bf16 result x 2^-1 differ")
        for v in kernel_calls.values():
            v.clear()
    chk.finish()


@pytest.mark.parametrize("op", list(OPS))
def test_nan_and_overflow_placement(op, device, kernel_calls):
    """A NaN in rank q's x (row a_q), in its scale_x (row b_q) and in this rank's scale_w (column c) give NaN
    in exactly those rows and that column; a scale product of 2^120 gives +-inf where |S| >= 2^8, with the
    sign of S, and exact values elsewhere."""
    label, grid, K = CASES[4]
    num_m, num_n = grid(_sm_count(device))
    rows, N = _rows(op, num_m), num_n * TILE
    spots = [((37 + 101 * q) % rows, (5 + 3 * q) % K, (11 + 29 * q) % rows, (53 + 67 * q) % N) for q in range(size)]

    def edit(q, xw, s):
        a, k, b, c = spots[q]
        xw[0].view(torch.uint8)[a, k] = 0x7F          # e4m3fn NaN (the format has no inf)
        s[0][b] = float("nan")
        s[1][c] = float("nan")

    chk = Checks()
    case = Case(op, label, rows, N, K, device, form=(True, True), edit=edit)
    want = case.want()
    out = case.run()
    chk(_assert_same, out, want, f"{op} {label} with NaN")
    # where the NaN are: the oracle's rows and columns, no more
    if op == "allgather":
        nan_rows = sorted({q * rows + spots[q][i] for q in range(size) for i in (0, 2)})
        nan_cols = [spots[rank][3]]
    else:
        nan_rows = sorted({spots[q][i] for q in range(size) for i in (0, 2)})
        nan_cols = sorted({spots[q][3] for q in range(size)})
        if op == "reduce_scatter":
            r = rows // size
            nan_rows = [i - rank * r for i in nan_rows if rank * r <= i < (rank + 1) * r]
    nan = torch.zeros(out.shape, dtype=torch.bool, device=device)
    nan[nan_rows] = True
    nan[:, nan_cols] = True
    chk(_expect, torch.equal(out.isnan(), nan), f"{op}: NaN outside the edited rows and columns, or missing")
    _check_path(chk, kernel_calls, _fused_method(op, device, E4M3, E4M3, rows, N), label)
    # overflow: scale products of 2^120 on rank 0's rows, 0 on every other rank's (their partials are 0)
    big = Case(op, label + "/inf", rows, N, K, device)
    big.scales = [(torch.tensor(2.0 ** 60 if q == 0 else 0.0, device=device), torch.tensor(2.0 ** 60, device=device))
                  for q in range(size)]
    big.sx, big.sw = big.scales[rank]
    out = big.run()
    want = big.want()
    chk(_assert_same, out, want, f"{op} {label}, overflow")
    chk(_expect, bool(want.isinf().any()) and not want.isnan().any(), "the overflow case has no inf")
    _check_path(chk, kernel_calls, _fused_method(op, device, E4M3, E4M3, rows, N), label)
    chk.finish()


@pytest.mark.parametrize("op", list(OPS))
def test_repeated_calls_and_graph_replay(op, device, kernel_calls):
    """Eager calls with new scales each time, then a CUDA graph of the call replayed four times (both
    staging halves) with operands and scales copied in place before every replay: each gives its set's
    exact result.  The allgather's row scales change on every call, so one read before its chunk arrived
    would show the previous launch's value."""
    label, grid, K = CASES[4]
    num_m, num_n = grid(_sm_count(device))
    rows, N = _rows(op, num_m), num_n * TILE
    chk = Checks()
    sets = [Case(op, f"{label}/{i}", rows, N, K, device, form=(True, i % 2 == 0)) for i in range(3)]
    base = sets[0]
    n = 0
    for i in (0, 1, 2, 0):
        chk(_assert_same, sets[i].run(), sets[i].want(), f"{op} {label}, eager call with set {i}")
        n += 1
    if device.type == "cuda":
        xs, ws = base.x.clone(), base.w.clone()
        sxs, sws = base.sx.clone(), base.sw.expand(N).clone()
        graph = torch.cuda.CUDAGraph()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            base.run(xs, ws, sxs, sws)                      # warm-up on the capture stream
            with torch.cuda.graph(graph, stream=side, capture_error_mode="thread_local"):
                out_g = base.run(xs, ws, sxs, sws)
        torch.cuda.current_stream().wait_stream(side)
        for i in (1, 2, 0, 1):
            s = sets[i]
            xs.copy_(s.x)
            ws.copy_(s.w)
            sxs.copy_(s.sx.expand(rows))
            sws.copy_(s.sw.expand(N))
            graph.replay()
            chk(_assert_same, out_g, s.want(), f"{op} {label}, graph replayed with set {i}")
        n += 2
    _check_path(chk, kernel_calls, _fused_method(op, device, E4M3, E4M3, rows, N), label, n)
    chk.finish()


def test_jit_equals_eager(device, kernel_calls):
    """``mpi4jax_b200.jit`` of a scaled call gives the eager bits."""
    case = Case("allgather", "jit", TILE, 256, 128, device)
    fast = m.jit(lambda a, b, c, d: linear_allgather(a, b, comm=comm, scale_x=c, scale_w=d))
    for _ in range(2):
        _assert_same(fast(case.x, case.w, case.sx, case.sw), case.want(), "jit")


#: rank q % 4's N; with K = 96, which the kernel pads to 128
UNEVEN_N = [0, 100, 128, 384]

#: (label, rows per rank m, tile columns, K): m = 64 puts a shard boundary inside a tile at P >= 2
SHARD_CASES = [("m64-k320", 64, 3, 320), ("m192-k448", 192, 2, 448), ("m16-k64", 16, 5, 64)]


def test_allgather_uneven_n_and_shard_boundaries(device, kernel_calls):
    """Ranks with N of 0, 100, 128 and 384, one x a byte into its buffer and a K the kernel pads; then shard
    boundaries inside a tile.  Every rank makes the same fuse decision."""
    chk = Checks()
    N = UNEVEN_N[rank % 4]
    case = Case("allgather", "uneven-n", TILE, max(N, 1), 96, device)
    case.w, case.sw = case.w[:N], (case.sw[:N] if case.sw.dim() else case.sw)
    x = _offset_view(case.x) if rank % 4 == 1 else case.x
    if rank % 4 == 1:
        assert x.is_contiguous() and x.data_ptr() % 16 == 1
    chk(_assert_same, case.run(x=x), case.want(), f"uneven N = {N}")
    _check_path(chk, kernel_calls, _fused_method("allgather", device, E4M3, E4M3, TILE, N), "uneven-n")
    for label, rows, tn, K in SHARD_CASES:
        case = Case("allgather", label, rows, tn * TILE, K, device)
        chk(_assert_same, case.run(), case.want(), label)
        _check_path(chk, kernel_calls, _fused_method("allgather", device, E4M3, E4M3, rows, tn * TILE), label)
    chk.finish()


#: K shard of rank q % 4; "64@1" is K = 64 a byte into its buffer
UNEVEN_K = ["64@1", 0, 96, 256]


@pytest.mark.parametrize("op", ["allreduce", "reduce_scatter"])
def test_uneven_and_misaligned_k_shards(op, device, kernel_calls):
    """K shards of different lengths and alignment, one empty: the same fuse decision, the sum of the
    ranks' scaled partials."""
    M, N = 256 * size, 384
    ks = [int(str(UNEVEN_K[q % 4]).split("@")[0]) for q in range(size)]
    case = Case(op, "uneven-k", M, N, 0, device, ks=ks)
    x, w = case.x, case.w
    if UNEVEN_K[rank % 4] == "64@1":
        x, w = _offset_view(x), _offset_view(w)
        assert x.data_ptr() % 16 == 1
    chk = Checks()
    chk(_assert_same, case.run(x=x, w=w), case.want(), f"{op}: K shards {ks}")
    _check_path(chk, kernel_calls, _fused_method(op, device, E4M3, E4M3, M, N), op)
    chk.finish()


# (label, x dtype, w dtype, rows (M, or m of the allgather), N, K): what the kernels do not take
FALLBACK_CASES = [
    ("e5m2", E5M2, E5M2, TILE * 2, 256, 128),
    ("e4m3-x-e5m2-w", E4M3, E5M2, TILE * 2, 128, 192),
    ("e5m2-x-e4m3-w", E5M2, E4M3, TILE * 2, 128, 64),
    ("m-unaligned", E4M3, E4M3, 120, 128, 128),
    ("n-unaligned", E4M3, E4M3, TILE * 2, 200, 128),
]


@pytest.mark.parametrize("op", list(OPS))
def test_fallbacks_are_exact(op, device, kernel_calls):
    """e5m2, mixed float8 types and unaligned shapes (and every case on the CPU) run the fallback, with the
    same exact results; the spy shows which path ran.  A shape the allgather kernel takes runs it."""
    chk = Checks()
    for label, dx, dw, rows, N, K in FALLBACK_CASES:
        if op == "reduce_scatter" and rows % size:
            continue
        case = Case(op, label, rows, N, K, device, dx=dx, dw=dw)
        chk(_assert_same, case.run(), case.want(), f"{op} {label}")
        _check_path(chk, kernel_calls, _fused_method(op, device, dx, dw, rows, N), f"{op} {label}")
    chk.finish()


# ---------------------------------------------------------------------------
# bound mode
# ---------------------------------------------------------------------------
BOUND_CASES = [("normal-k4096", 2, 3, 4096), ("normal-k448", 3, 2, 448), ("normal-k128", 1, 1, 128)]


@pytest.mark.parametrize("op", list(OPS))
def test_scaled_within_bound(op, device, kernel_calls):
    """Normal float8 operands and arbitrary fp32 scales, every element within the bound of the accumulator
    model: per rank ``e_q = (K / 32) 2^-12 sum_k |x w|`` on S_q, the scaling (2 fp32 roundings) and the
    bf16 rounding of the partial, then (allreduce, reduce-scatter) the fp32 sum of the partials and its
    rounding.  Prints the worst err / bound and the worst |S_hat - S| / sum_k |x w| it implies."""
    chk = Checks()
    for label, tm, tn, K in BOUND_CASES:
        rows, N = _rows(op, tm), tn * TILE
        xs, scales = [], []
        for q in range(size):
            gen = _gen(label, q, device)
            x = torch.randn(rows, K, generator=gen, device=device).to(E4M3)
            w = torch.randn(N, K, generator=gen, device=device).to(E4M3)
            sx = 0.5 + 1.5 * torch.rand(rows, generator=gen, device=device)
            sw = torch.rand((), generator=gen, device=device) * 3e-2 + 1e-3 if q % 2 else \
                0.5 + torch.rand(N, generator=gen, device=device)
            xs.append((x, w))
            scales.append((sx, sw))
        x, w = xs[rank]
        out = OPS[op](x, w, comm=comm, scale_x=scales[rank][0], scale_w=scales[rank][1]).double()

        def rank_part(xq, wq, sx, sw):
            xd, wd = xq.double(), wq.double()
            s = sx.double().reshape(-1, 1) * sw.double().reshape(1, -1)
            S, A = xd @ wd.t(), xd.abs() @ wd.abs().t()
            e = (K / 32) * 2.0 ** -12 * A * s + 2.0 ** -23 * (S.abs() * s)
            return S * s, e, A * s

        if op == "allgather":
            X = torch.cat([xq for xq, _ in xs])
            SX = torch.cat([sx for sx, _ in scales])
            S, E, A = rank_part(X, w, SX, scales[rank][1])
            bound = 0.5 * _ulp_bf16(S.abs() + E) + E
        else:
            S = E = A = mags = 0
            for (xq, wq), (sx, sw) in zip(xs, scales):
                s, e, a = rank_part(xq, wq, sx, sw)
                d = e + 0.5 * _ulp_bf16(s.abs() + e) if size > 1 else e
                S, E, A, mags = S + s, E + d, A + a, mags + s.abs() + d
            E = E + (size - 1) * 2.0 ** -24 * mags
            bound = 0.5 * _ulp_bf16(S.abs() + E) + E
            if op == "reduce_scatter":
                r = rows // size
                S, bound, A = (t[rank * r:(rank + 1) * r] for t in (S, bound, A))
        err = (out - S).abs()
        worst = (err / bound).nan_to_num(float("inf")).max().item()
        rel = (err / A).nan_to_num(0.0).max().item()
        print(f"linear_{op} float8 {label} ({rows} x {N} x {K}) on {device.type}, rank {rank}: worst err / bound "
              f"{worst:.4f}, worst |err| / sum|x w| {rel:.3g}")
        chk(_expect, worst <= 1.0, f"{op} {label}: err / bound {worst:.4f}")
        _check_path(chk, kernel_calls, _fused_method(op, device, E4M3, E4M3, rows, N), label)
    chk.finish()


# ---------------------------------------------------------------------------
# arguments, launches, transports
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("op", list(OPS))
def test_bad_arguments_raise_everywhere(op, device, kernel_calls):
    """One scale without the other, scales with bf16 operands, a wrong scale shape, dtype or device raise
    ValueError, and a scale or operand that requires grad NotImplementedError, on every rank before any
    device work; the unscaled call still returns what it returns without this feature."""
    f = OPS[op]
    M, N, K = TILE * size, TILE, 64
    x, w = f8_operands("bad", rank, M, N, K, device)
    one = torch.tensor(1.0, device=device)
    other = torch.device("meta")
    bad = [dict(scale_x=one), dict(scale_w=one),
           dict(scale_x=one, scale_w=torch.ones(N + 1, device=device)),
           dict(scale_x=torch.ones(M - 1, device=device), scale_w=one),
           dict(scale_x=torch.ones(1, M, device=device), scale_w=one),
           dict(scale_x=one.double(), scale_w=one),
           dict(scale_x=one, scale_w=one.half()),
           dict(scale_x=torch.ones((), device=other), scale_w=one)]
    for kw in bad:
        with pytest.raises(ValueError, match=f"linear_{op}"):
            f(x, w, comm=comm, **kw)
    with pytest.raises(ValueError, match="float8"):
        f(x.to(torch.bfloat16), w.to(torch.bfloat16), comm=comm, scale_x=one, scale_w=one)
    with pytest.raises(ValueError, match="float8"):
        f(x, w.to(torch.bfloat16), comm=comm, scale_x=one, scale_w=one)
    with pytest.raises(NotImplementedError):
        f(x, w, comm=comm, scale_x=one.clone().requires_grad_(), scale_w=one)
    with pytest.raises(NotImplementedError):
        f(x, w, comm=comm, scale_x=one, scale_w=torch.ones(N, device=device, requires_grad=True))
    assert not any(kernel_calls.values()), kernel_calls
    # the unscaled path: bf16 as before; CPU float8 keeps its float8 product
    xb, wb = exact_operands("bad", rank, M, N, K, device)
    got = f(xb, wb, comm=comm)
    assert got.dtype == torch.bfloat16
    if device.type == "cpu":
        assert f(x, w, comm=comm).dtype == E4M3
    out = m.allreduce(torch.full((5,), float(rank), device=device), MPI.SUM, comm=comm)
    assert torch.equal(out, torch.full((5,), float(size * (size - 1) // 2), device=device))


@pytest.mark.parametrize("op", list(OPS))
def test_one_native_launch_per_fused_call(op, device):
    """A fused call is one native launch, K and N padding included (those are torch ops)."""
    from mpi4jax_b200._src import native

    for label, rows, N, K in (("aligned", TILE * size, 256, 256), ("padded", TILE * size, 200, 96)):
        case = Case(op, label, rows, N, K, device)
        if op == "allgather":
            case.x, case.sx = case.x[:TILE], case.sx[:TILE] if case.sx.dim() else case.sx
            case.ops = [(xq[:TILE], wq) for xq, wq in case.ops]
            case.scales = [(sx[:TILE] if sx.dim() else sx, sw) for sx, sw in case.scales]
            case.rows = TILE
        method = _fused_method(op, device, E4M3, E4M3, case.rows, N)
        if method is None or (op != "allgather" and N % TILE):
            continue
        torch.cuda.synchronize()
        before = native.launch_count()
        out = case.run()
        launched = native.launch_count() - before
        _assert_same(out, case.want(), f"{op} {label}")
        assert launched == 1, f"{op} {label}: {launched} native launches"


HOST_SCRIPT = r"""
import torch
from mpi4jax_b200 import MPI
from mpi4jax_b200.ops import linear_allgather, linear_allreduce, linear_reduce_scatter

comm = MPI.COMM_WORLD
assert comm.transport == "host", comm.transport
gen = torch.Generator().manual_seed(7)
x = torch.randint(-3, 4, (128, 128), generator=gen).float()
w = torch.randint(-4, 5, (256, 128), generator=gen).float()
sx, sw = torch.full((128,), 0.5), torch.tensor(4.0)
want = (x.double() @ w.double().t() * 2).to(torch.bfloat16)
d = comm.device
for f in (linear_allreduce, linear_reduce_scatter, linear_allgather):
    out = f(x.to(torch.float8_e4m3fn).to(d), w.to(torch.float8_e4m3fn).to(d), comm=comm, scale_x=sx.to(d),
            scale_w=sw.to(d))
    assert torch.equal(out.cpu(), want), f
print("host transport ok")
"""


@pytest.mark.gpu
def test_host_transport_falls_back():
    """With host staging the scaled ops run the fallback, even at world size 1, and give the exact result."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    if inside_job:
        pytest.skip("a world-size-1 check")
    env = {**os.environ, "MPI4JAX_B200_TRANSPORT": "host", "MPI4JAX_B200_ABORT_ON_ERROR": "0"}
    res = subprocess.run([sys.executable, "-c", HOST_SCRIPT], cwd=REPO, env=env, capture_output=True, text=True,
                         timeout=600)
    assert res.returncode == 0 and "host transport ok" in res.stdout, res.stdout[-2000:] + res.stderr[-4000:]


def test_allgather_byte_offsets_past_2_31(device, kernel_calls):
    """Two ranks gathering 2 x 32768 x 33024 float8 bytes (2.16e9, past 2^31), so the row-scale region starts
    past 2^31 too: rows of both shards, with per-row scales, against the oracle.  Run by its own job."""
    if device.type != "cuda" or size != 2:
        pytest.skip("a two-rank GPU check")
    rows, N, K = 32768, TILE, 33024
    assert size * rows * K > 2 ** 31

    def shard(q):
        gen = _gen("2^31", q, device)
        x = torch.randint(-2, 3, (rows, K), generator=gen, device=device, dtype=torch.int8).to(torch.float16)
        return x.to(E4M3), torch.exp2(torch.randint(-2, 3, (rows,), generator=gen, device=device).float())

    w = torch.randint(-2, 3, (N, K), generator=_gen("2^31/w", rank, device), device=device,
                      dtype=torch.int8).to(torch.float16).to(E4M3)
    sw = torch.tensor(0.5, device=device)
    x, sx = shard(rank)
    out = linear_allgather(x, w, comm=comm, scale_x=sx, scale_w=sw)
    assert kernel_calls["gemm_allgather_f8"] == [(rows, N, K)]
    del x
    for r0 in (0, rows - TILE, rows, 2 * rows - 2 * TILE, 2 * rows - TILE):
        q, lo = divmod(r0, rows)
        xq, sq = shard(q)
        _assert_same(out[r0:r0 + TILE], partial(xq[lo:lo + TILE], w, sq[lo:lo + TILE], sw), f"rows {r0}..{r0 + TILE}")
        del xq
    del out


# ---------------------------------------------------------------------------
# jobs
# ---------------------------------------------------------------------------
PEER_TESTS = ["test_scaled_exact", "test_equals_the_bf16_kernel_times_the_scale", "test_nan_and_overflow_placement",
              "test_repeated_calls_and_graph_replay", "test_jit_equals_eager",
              "test_allgather_uneven_n_and_shard_boundaries", "test_uneven_and_misaligned_k_shards",
              "test_fallbacks_are_exact", "test_scaled_within_bound", "test_bad_arguments_raise_everywhere",
              "test_one_native_launch_per_fused_call"]


def _passed(out, t, dev):
    return re.search(rf"^PASSED .*::{t}\[(\w+-)?{dev}\]", out, re.M) or re.search(
        rf"^PASSED .*::{t}\[{dev}(-\w+)?\]", out, re.M)


@pytest.mark.skipif(inside_job, reason="already inside a multi-rank job")
@pytest.mark.parametrize("nranks", [2, 3])
def test_cpu_job(nranks):
    """The CPU variants as a job of ``nranks`` CPU ranks."""
    from mpi4jax_b200.run import launch

    args = ["-m", "pytest", os.path.relpath(__file__, REPO), "-q", "-rp", "-m", "not gpu", "-p", "no:cacheprovider"]
    cwd = os.getcwd()
    os.chdir(REPO)
    try:
        code, outs = launch(nranks, args, cpu=True, timeout=900, capture=True,
                            env_extra={"MPI4JAX_B200_NESTED": "1"})
    finally:
        os.chdir(cwd)
    for r, out in enumerate(outs):
        missing = [t for t in PEER_TESTS if not _passed(out, t, "cpu")]
        assert code == 0 and not missing, f"rank {r} of the {nranks}-rank CPU job (exit code {code}), not passed: " \
                                          f"{missing}:\n{out[-4000:]}"


def _gpu_job(nranks, env=None, tests=PEER_TESTS):
    code, outs = job(__file__, nranks, " or ".join(tests), env)
    for r, out in enumerate(outs):
        missing = [t for t in tests if not _passed(out, t, "cuda")]
        assert code == 0 and not missing, f"rank {r} of the {nranks}-rank job (exit code {code}), not passed: " \
                                          f"{missing}:\n{out[-4000:]}"


@pytest.mark.gpu
@pytest.mark.skipif(inside_job, reason="already inside a multi-rank job")
def test_job_two_ranks():
    """Two ranks on the GPUs there are; on one GPU both share it (the allreduce then has no NVLS and takes
    the fallback, which the spy checks)."""
    _gpu_job(2)


@pytest.mark.gpu
@pytest.mark.skipif(inside_job, reason="already inside a multi-rank job")
def test_job_two_ranks_past_2_31_bytes():
    """The byte-offset check as a two-rank job; it needs about 24 GiB of device memory for both ranks."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    need = (24 << 30) if torch.cuda.device_count() < 2 else (12 << 30)
    if torch.cuda.mem_get_info()[0] < need:
        pytest.skip("not enough free device memory")
    _gpu_job(2, tests=["test_allgather_byte_offsets_past_2_31"])


@pytest.mark.gpu
@pytest.mark.skipif(inside_job, reason="already inside a multi-rank job")
def test_job_two_ranks_without_nvls():
    """Two ranks with NVLS off: the allreduce takes the fallback, the other two still run their kernels."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    _gpu_job(2, {"MPI4JAX_B200_NVLS": "0"})


@pytest.mark.gpu
@pytest.mark.skipif(inside_job, reason="already inside a multi-rank job")
@pytest.mark.parametrize("nranks", [3, 4, 5, 7, 8])
def test_job_more_ranks(nranks):
    """One rank per GPU: uneven row slices of the allreduce epilogue, shard boundaries inside tiles."""
    if not torch.cuda.is_available() or torch.cuda.device_count() < nranks:
        pytest.skip(f"needs {nranks} GPUs")
    _gpu_job(nranks)
