"""Tensor-parallel linear (``ops.linear_allreduce``): the wgmma GEMM + in-switch allreduce kernel of
csrc/b2_gemm.cu, and its fallback, against an oracle that never calls the library.

Rank q's operands come from a seed of (case, q), so every rank rebuilds every rank's operands and
computes the expected result itself, in float64 with plain torch.  Two kinds of operands:

* exact: small integers with ``sum_k |x_mk| |w_nk| <= 2^11`` for every output, so every partial sum is
  exact in any accumulator of 12 or more significant bits.  Rank q's partial is rounded once to the
  output dtype (the kernel stages it, the fallback's matmul returns it), and the ranks' partials are
  summed in fp32 and rounded once: the expected output is ``rn(sum_q rn(S_q))`` to the bit.  Every 8th
  row and column is dense and positive, so outputs between 257 and 2048 exercise bf16's rounding,
  ties to even included.
* bound: normal operands, and rows that mix 2^10 entries (which cancel) with 2^-8 ones.  Each element
  must lie within ``1/2 ulp_bf16(|S| + e) + e`` of the exact S, ``e = K 2^-22 sum_k |x| |w|``, plus the
  staging roundings and the fp32 sum of the ranks' partials above one rank.

The tests that take ``device`` run at world size 1 on the CPU fallback and through the kernel, and in
multi-rank jobs (a two-rank job on the GPUs there are; 3, 5 and 7 ranks on the fused NVLS path when
the machine has that many GPUs), where each rank checks its own result and all ranks must hold the
same bits."""

import os
import re
import subprocess
import sys
import zlib

import pytest
import torch

import mpi4jax_b200 as m
from mpi4jax_b200 import MPI
from mpi4jax_b200.ops import linear_allreduce

from ._peer_job import REPO, Checks, expect_passed, job

comm = MPI.COMM_WORLD
rank, size = comm.Get_rank(), comm.Get_size()
inside_job = size > 1 or "MPI4JAX_B200_NESTED" in os.environ

TILE = 128
EXACT_MAX = 2 ** 11


def _grid(tiles):
    """(num_m, num_n) with num_m the largest divisor of ``tiles`` that is at most its square root."""
    d = max(i for i in range(1, int(tiles ** 0.5) + 1) if tiles % i == 0)
    return d, tiles // d


# (label, tile grid (num_m, num_n) as a function of g = SM count, K).  K = 64 is one k-block, 320 fewer
# k-blocks than the 6 ring stages, 384 exactly 6, 448 wraps the ring inside a tile.  The tile counts 1,
# g - 1, g, g + 1, 3g and 4g + 3 leave every remainder of the persistent wave and, above one rank, of the
# epilogue's batches of 4 tiles; g + 1 = 133 is a 7 x 19 grid on an H100, a row count that bands of 2
# and 3 do not divide.
CASES = [
    ("one-tile-k64", lambda g: (1, 1), 64),
    ("one-tile-k4096", lambda g: (1, 1), 4096),
    ("tall-g-1-k320", lambda g: (g - 1, 1), 320),
    ("wide-g-k384", lambda g: (1, g), 384),
    ("grid-g+1-k448", lambda g: _grid(g + 1), 448),
    ("grid-3g-k4096", lambda g: (3, g), 4096),
    ("tall-4g+3-k448", lambda g: (4 * g + 3, 1), 448),
    ("wide-4g+3-k64", lambda g: (1, 4 * g + 3), 64),
]


def _sm_count(device):
    """g: the kernel's persistent grid size on CUDA; on the CPU a small stand-in keeps the shapes cheap."""
    if device.type != "cuda":
        return 4
    return comm._native_comm().get_option("sm_count")


def _gen(case, q, device):
    gen = torch.Generator(device=device)
    gen.manual_seed(zlib.crc32(f"{case}/{q}".encode()))
    return gen


def exact_operands(case, q, M, N, K, device, dtype=torch.bfloat16):
    """Rank q's small-integer operands: |x| <= 3 with at most 512 in every row's sum of |x|, |w| <= 4, so
    ``sum_k |x_mk| |w_nk| <= 2^11``.  Rows of x and w with (index + q) % 8 == 0 are positive (w's dense).
    A row of x keeps about 160 nonzeros at most, spread over the whole of K, so every k-block counts."""
    gen = _gen(case, q, device)
    spread = min(1.0, 160 / max(K, 1))

    def draw(rows, lo, hi, keep_hot, keep):
        hot = (torch.arange(rows, device=device) + q) % 8 == 0
        dense = torch.randint(lo, hi + 1, (rows, K), generator=gen, device=device, dtype=torch.float32)
        sparse = torch.randint(-hi, hi + 1, (rows, K), generator=gen, device=device, dtype=torch.float32)
        t = torch.where(hot[:, None], dense, sparse)
        return t * (torch.rand(rows, K, generator=gen, device=device) < torch.where(hot, keep_hot, keep)[:, None])

    x = draw(M, 2, 3, spread, min(0.5, spread))
    w = draw(N, 1, 4, 1.0, 0.5)
    x[x.abs().cumsum(1) > 512] = 0         # a safeguard: rows reach about 400 on average
    return x.to(dtype), w.to(dtype)


def exact_want(case, M, N, ks, dtype, device, edit=None):
    """``rn(sum_q rn(S_q))`` from every rank's rebuilt operands (``ks[q]``: rank q's K); ``edit(q, x, w)``
    changes rank q's operands first, as the test does."""
    acc = torch.zeros(M, N, dtype=torch.float64, device=device)
    for q in range(size):
        x, w = exact_operands(case, q, M, N, ks[q], device)
        if edit is not None:
            edit(q, x, w)
        xd, wd = x.double(), w.double()
        bound = xd.abs().nan_to_num(0, 0, 0) @ wd.abs().nan_to_num(0, 0, 0).t()
        if bound.numel():
            assert bound.max().item() <= EXACT_MAX, (case, q, bound.max().item())
        acc += (xd @ wd.t()).to(dtype).double()
    return acc.to(dtype)


def _exercises_rounding_and_every_k16(case, M, N, K, device):
    """The exact operands have outputs between 257 and 2048 (where bf16 rounds), odd ones among them, and
    every 16-wide k-slice holds a nonzero of x in a row with such outputs: a k-slice or k-block that the
    kernel drops, misplaces or reads twice changes outputs."""
    x, w = exact_operands(case, 0, M, N, K, device)
    s = (x.double() @ w.double().t()).abs()
    mid = (s > 256) & (s <= EXACT_MAX)
    assert mid.any() and (mid & (s % 2 == 1)).any(), (case, s.max().item())
    hit = (x[mid.any(1)] != 0).reshape(-1, K // 16, 16).any(2).any(0)
    assert hit.all(), f"{case}: k16 slices {(~hit).nonzero().flatten().tolist()} hold no nonzero of such a row"


def _assert_same(out, want, label):
    """Equal values (+-0 equal), NaN exactly where ``want`` has NaN."""
    assert out.dtype == want.dtype and out.shape == want.shape, (label, out.dtype, want.dtype, out.shape)
    o, w = out.double(), want.double()
    nan = w.isnan()
    bad = (o.isnan() != nan) | (~nan & (o != w))
    if bad.any():
        at = tuple(bad.nonzero()[0].tolist())
        raise AssertionError(f"{label}: {int(bad.sum())} of {bad.numel()} elements differ, first at {at}: "
                             f"got {o[at].item()!r}, want {w[at].item()!r}")


def _assert_bitwise(outs, label):
    first = outs[0][1].contiguous().view(torch.uint8)
    for r, out in outs[1:]:
        assert torch.equal(out.contiguous().view(torch.uint8), first), \
            f"{label}: gemm_raster {r} changed bits against gemm_raster {outs[0][0]}"


def _expect(ok, message):
    assert ok, message


@pytest.fixture
def kernel_calls(monkeypatch):
    """Shapes (M, N, K) of every call of the fused kernel's entry point while the test runs."""
    from mpi4jax_b200._src.backends.cuda import NativeComm

    calls = []
    real = NativeComm.gemm_allreduce

    def spy(self, x, weight):
        calls.append((x.shape[0], weight.shape[0], x.shape[1]))
        return real(self, x, weight)

    monkeypatch.setattr(NativeComm, "gemm_allreduce", spy)
    return calls


def _kernel_expected(device, dtype, M, N):
    """Whether linear_allreduce must run the kernel: bf16 tile-aligned CUDA operands on the native
    transport, at world size 1 or with NVLS."""
    if device.type != "cuda" or dtype != torch.bfloat16 or M == 0 or N == 0 or M % TILE or N % TILE:
        return False
    if comm.transport != "native":
        return False
    return size == 1 or comm._native_comm().has_nvls


def _check_path(chk, calls, expected, label, n=1):
    ran = len(calls)
    chk(_expect, ran == (n if expected else 0),
        f"{label}: the fused kernel ran {ran} times, expected {n if expected else 0}")
    calls.clear()


def _over_rasters(x, w, num_m, device):
    """[(gemm_raster, output)] over the tile orders 0 (row-major), bands of 1, 2, 3, num_m and num_m + 1
    tile rows, and the automatic choice (-1); one call where there is no native communicator."""
    if device.type != "cuda" or comm.transport != "native":
        return [("auto", linear_allreduce(x, w, comm=comm))]
    nc = comm._native_comm()
    outs = []
    try:
        for r in dict.fromkeys((-1, 0, 1, 2, 3, num_m, num_m + 1)):
            nc.set_option("gemm_raster", r)
            outs.append((r, linear_allreduce(x, w, comm=comm)))
    finally:
        nc.set_option("gemm_raster", -1)      # get_option reports the automatic choice as 0
    return outs


# ---------------------------------------------------------------------------
# exact mode
# ---------------------------------------------------------------------------
def test_linear_allreduce_exact(device, kernel_calls):
    """Every case and tile order to the bit against ``rn(sum_q rn(S_q))``."""
    chk = Checks()
    g = _sm_count(device)
    for label, grid, K in CASES:
        num_m, num_n = grid(g)
        M, N = num_m * TILE, num_n * TILE
        _exercises_rounding_and_every_k16(label, M, N, K, device)
        x, w = exact_operands(label, rank, M, N, K, device)
        want = exact_want(label, M, N, [K] * size, torch.bfloat16, device)
        outs = _over_rasters(x, w, num_m, device)
        for r, out in outs:
            chk(_assert_same, out, want, f"{label} ({M} x {N} x {K}), gemm_raster {r}")
        chk(_assert_bitwise, outs, label)
        _check_path(chk, kernel_calls, _kernel_expected(device, x.dtype, M, N), label, len(outs))
        chk.add(label, outs[0][1])
    chk.finish()


def test_nan_and_inf_stay_in_their_row_and_column(device, kernel_calls):
    """Rank q puts a NaN at x[m_q, k] and an inf in w[n_q, :].  Rows m_q become NaN, column n_q inf or NaN,
    and every other element still matches the oracle: no crosstalk between rows, columns or tiles."""
    label, grid, K = CASES[4]
    chk = Checks()
    num_m, num_n = grid(_sm_count(device))
    M, N = num_m * TILE, num_n * TILE
    where = [((37 + 101 * q) % M, (5 + 3 * q) % K, (53 + 67 * q) % N, (K - 1 - q) % K) for q in range(size)]

    def edit(q, x, w):
        m0, k0, n0, k1 = where[q]
        x[m0, k0] = float("nan")
        w[n0, k1] = float("inf")

    x, w = exact_operands(label, rank, M, N, K, device)
    edit(rank, x, w)
    want = exact_want(label, M, N, [K] * size, torch.bfloat16, device, edit)
    rows = sorted({m0 for m0, _, _, _ in where})
    cols = sorted({n0 for _, _, n0, _ in where})
    assert want[rows].isnan().all()
    outs = _over_rasters(x, w, num_m, device)
    for r, out in outs:
        chk(_assert_same, out, want, f"{label} with NaN / inf, gemm_raster {r}")
        finite = torch.ones(M, N, dtype=torch.bool, device=device)
        finite[rows] = False
        finite[:, cols] = False
        chk(_expect, out[finite].isfinite().all().item(), f"gemm_raster {r}: a NaN or inf left its row or column")
    chk(_assert_bitwise, outs, label)
    _check_path(chk, kernel_calls, _kernel_expected(device, x.dtype, M, N), label, len(outs))
    chk.add(label, outs[0][1].view(torch.int16))
    chk.finish()


def test_repeated_calls_and_graph_replay(device, kernel_calls):
    """Three eager calls give the same bits, and so does a CUDA graph of the call replayed with new
    operands copied into its inputs."""
    label, grid, K = CASES[4]
    chk = Checks()
    num_m, num_n = grid(_sm_count(device))
    M, N = num_m * TILE, num_n * TILE
    x, w = exact_operands(label, rank, M, N, K, device)
    x2, w2 = exact_operands(label + "/2", rank, M, N, K, device)
    want = exact_want(label, M, N, [K] * size, torch.bfloat16, device)
    want2 = exact_want(label + "/2", M, N, [K] * size, torch.bfloat16, device)
    outs = [(i, linear_allreduce(x, w, comm=comm)) for i in range(3)]
    chk(_assert_same, outs[0][1], want, f"{label}, eager")
    chk(_assert_bitwise, outs, f"{label}, repeated calls")
    if device.type == "cuda":
        xs, ws = x.clone(), w.clone()
        graph = torch.cuda.CUDAGraph()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            linear_allreduce(xs, ws, comm=comm)          # warm-up on the capture stream
            with torch.cuda.graph(graph, stream=side, capture_error_mode="thread_local"):
                out_g = linear_allreduce(xs, ws, comm=comm)
        torch.cuda.current_stream().wait_stream(side)
        for xn, wn, wt, tag in ((x2, w2, want2, "new"), (x, w, want, "first")):
            xs.copy_(xn)
            ws.copy_(wn)
            graph.replay()
            chk(_assert_same, out_g, wt, f"{label}, graph replayed with the {tag} operands")
        chk(_assert_bitwise, [("eager", outs[0][1]), ("graph", out_g)], f"{label}, graph replay")
        n = 3 + 2             # eager calls, warm-up and capture; a replay does not go through Python
        _check_path(chk, kernel_calls, _kernel_expected(device, x.dtype, M, N), label, n)
    chk.add(label, outs[0][1])
    chk.finish()


# (label, dtype, M, N, K): shapes and dtypes the kernel does not take go through matmul + allreduce
# against the same oracle; a bf16 K of 63 is padded for the kernel
FALLBACK_CASES = [
    ("bf16-m127", torch.bfloat16, 127, 128, 64),
    ("bf16-m129", torch.bfloat16, 129, 256, 64),
    ("bf16-k63", torch.bfloat16, 128, 256, 63),
    ("f16", torch.float16, 128, 128, 64),
    ("f16-m129-k63", torch.float16, 129, 128, 63),
    ("f32", torch.float32, 256, 128, 64),
    ("f32-m127-k63", torch.float32, 127, 128, 63),
]


def test_fallback_shapes(device, kernel_calls):
    chk = Checks()
    for label, dtype, M, N, K in FALLBACK_CASES:
        x, w = exact_operands(label, rank, M, N, K, device, dtype)
        want = exact_want(label, M, N, [K] * size, dtype, device)
        out = linear_allreduce(x, w, comm=comm)
        chk(_assert_same, out, want, label)
        _check_path(chk, kernel_calls, _kernel_expected(device, dtype, M, N), label)
        chk.add(label, out)
    chk.finish()


def _offset_view(t, elems=1):
    """A contiguous copy of ``t`` whose storage starts ``elems`` elements into a buffer (2 bytes in bf16:
    not 16-byte aligned)."""
    flat = torch.zeros(t.numel() + elems, dtype=t.dtype, device=t.device)
    view = flat[elems:elems + t.numel()].view(t.shape)
    view.copy_(t)
    return view


#: K shard of rank q % 4; "64@2" is K = 64 at a 2-byte offset
UNEVEN_K = ["64@2", 0, 96, 128]


def test_uneven_k_shards(device, kernel_calls):
    """Ranks with K shards of different lengths and alignment, one of them empty, must make the same fuse
    decision and compute the sum of their products."""
    label, M, N = "uneven-k", 256, 384
    chk = Checks()
    ks = [int(str(UNEVEN_K[q % 4]).split("@")[0]) for q in range(size)]
    x, w = exact_operands(label, rank, M, N, ks[rank], device)
    if UNEVEN_K[rank % 4] == "64@2":
        x, w = _offset_view(x), _offset_view(w)
        assert x.is_contiguous() and x.data_ptr() % 16 == 2
    want = exact_want(label, M, N, ks, torch.bfloat16, device)
    out = linear_allreduce(x, w, comm=comm)
    chk(_assert_same, out, want, f"{label}: K shards {ks}")
    _check_path(chk, kernel_calls, _kernel_expected(device, x.dtype, M, N), label)
    chk.add(label, out)
    chk.finish()


def _ints(case, q, n, device):
    gen = _gen(case, q, device)
    return torch.randint(-1000, 1001, (n,), generator=gen, device=device, dtype=torch.float32)


def test_gemm_interleaved_with_allreduces(device, kernel_calls):
    """A small GEMM, then one large enough to grow the staging segment, with allreduces of other sizes
    (so other grid sizes advance the per-block epochs the fused epilogue shares) between them."""
    chk = Checks()
    big = (4096, 8192, 64) if device.type == "cuda" else (512, 1024, 64)
    steps = [("gemm", (128, 128, 64)), ("allreduce", 1000), ("gemm", big), ("allreduce", 3 << 20),
             ("gemm", (128, 128, 64)), ("allreduce", 17), ("gemm", (384, 640, 192)), ("gemm", big)]
    for i, (kind, arg) in enumerate(steps):
        label = f"step {i}: {kind} {arg}"
        if kind == "gemm":
            M, N, K = arg
            x, w = exact_operands(label, rank, M, N, K, device)
            out = linear_allreduce(x, w, comm=comm)
            chk(_assert_same, out, exact_want(label, M, N, [K] * size, torch.bfloat16, device), label)
            _check_path(chk, kernel_calls, _kernel_expected(device, x.dtype, M, N), label)
        else:
            out = m.allreduce(_ints(label, rank, arg, device), MPI.SUM, comm=comm)
            want = sum(_ints(label, q, arg, device).double() for q in range(size)).float()
            chk(_assert_same, out, want, label)
        chk.add(label, out)
    chk.finish()


# ---------------------------------------------------------------------------
# bound mode
# ---------------------------------------------------------------------------
def normal_operands(case, q, M, N, K, device):
    """Normal operands; ``range`` cases: even rows of x hold 2^10-sized entries in k-block 0, their
    negation against the same w in k-block 1 (the sum cancels exactly) and 2^-8-sized ones after, odd rows
    only 2^-8-sized ones.  A kernel that rounded to bf16 between k-blocks would lose the small ones."""
    gen = _gen(case, q, device)
    x = torch.randn(M, K, generator=gen, device=device)
    w = torch.randn(N, K, generator=gen, device=device)
    if case.startswith("range"):
        x *= 2.0 ** -8
        x[0::2, :64] = 1024 * (1 + torch.rand(M, 64, generator=gen, device=device)[0::2])
        w[:, :64] = 0.5 + 0.5 * torch.rand(N, 64, generator=gen, device=device)
    x, w = x.to(torch.bfloat16), w.to(torch.bfloat16)
    if case.startswith("range"):
        x[0::2, 64:128] = -x[0::2, :64]
        w[:, 64:128] = w[:, :64]
    return x, w


def _ulp_bf16(a):
    """ulp of bf16 at |a| (float64): 2^(exponent - 7), at least the smallest subnormal 2^-133."""
    _, ex = torch.frexp(a)
    ex = torch.where(a > 0, ex, torch.full_like(ex, -125))
    return torch.exp2((ex - 8).clamp(min=-133).double())


def bound_reference(case, M, N, K, device):
    """(S, bound): the exact sum over the ranks and the largest error a correct result can have.  Each
    rank's fp32 accumulation is within e_q = K 2^-22 sum_k |x||w| of S_q; above one rank it is staged
    as bf16 (1/2 ulp) and the partials are summed in fp32 ((P - 1) 2^-24 sum_q |partial|)."""
    S = torch.zeros(M, N, dtype=torch.float64, device=device)
    E = torch.zeros_like(S)
    mags = torch.zeros_like(S)
    for q in range(size):
        x, w = (t.double() for t in normal_operands(case, q, M, N, K, device))
        s = x @ w.t()
        e = K * 2.0 ** -22 * (x.abs() @ w.abs().t())
        d = e if size == 1 else e + 0.5 * _ulp_bf16(s.abs() + e)
        S += s
        E += d
        mags += s.abs() + d
    E += (size - 1) * 2.0 ** -24 * mags
    return S, 0.5 * _ulp_bf16(S.abs() + E) + E


# (label, tile grid as a function of g, K)
BOUND_CASES = [
    ("normal-grid-3g-k4096", lambda g: (3, g), 4096),
    ("normal-tall-g-1-k320", lambda g: (g - 1, 1), 320),
    ("normal-grid-g+1-k448", lambda g: _grid(g + 1), 448),
    ("range-k256", lambda g: (2, 3), 256),
]


def test_linear_allreduce_within_bound(device, kernel_calls):
    """Every element within its own bound (not a fraction of the largest one), the same bits in every tile
    order; prints the worst err / bound."""
    chk = Checks()
    g = _sm_count(device)
    for label, grid, K in BOUND_CASES:
        num_m, num_n = grid(g)
        M, N = num_m * TILE, num_n * TILE
        x, w = normal_operands(label, rank, M, N, K, device)
        S, bound = bound_reference(label, M, N, K, device)
        outs = _over_rasters(x, w, num_m, device)
        ratio = ((outs[0][1].double() - S).abs() / bound).nan_to_num(float("inf"))
        worst = ratio.max().item()
        print(f"linear_allreduce {label} ({M} x {N} x {K}) at {size} rank(s) on {device.type}: "
              f"worst err / bound {worst:.4f}")
        at = divmod(int(ratio.argmax().item()), N)
        chk(_expect, worst <= 1.0, f"{label}: err / bound {worst:.4f} at {at}: got "
                                   f"{outs[0][1][at].item()!r}, exact {S[at].item()!r}, bound {bound[at].item():.3g}")
        chk(_assert_bitwise, outs, label)
        _check_path(chk, kernel_calls, _kernel_expected(device, x.dtype, M, N), label, len(outs))
        chk.add(label, outs[0][1])
    chk.finish()


# ---------------------------------------------------------------------------
# world size 1: operands the kernel cannot read as given, transports, a 4 GiB output, the adjoint
# ---------------------------------------------------------------------------
def test_kernel_operands_are_padded_and_aligned():
    """Each rank's operands are brought into the kernel's form locally: K zero-padded up to a multiple of
    64 that is at least 64, storage contiguous and 16-byte aligned; the product does not change."""
    from mpi4jax_b200.ops.linear import _kernel_operands

    for K in (0, 1, 63, 64, 65, 96, 128, 448):
        for offset in (0, 1, 3):
            x, w = exact_operands(f"prep-{K}", 0, 8, 16, K, torch.device("cpu"))
            if offset:
                x, w = _offset_view(x, offset), _offset_view(w, offset)
            px, pw = _kernel_operands(x, w)
            Kp = max(64, -(-K // 64) * 64)
            for p, t in ((px, x), (pw, w)):
                assert p.shape == (t.shape[0], Kp) and p.dtype == t.dtype and p.is_contiguous(), (K, offset, p.shape)
                assert p.data_ptr() % 16 == 0, (K, offset)
                assert torch.equal(p[:, :K], t) and not p[:, K:].any(), (K, offset)
            assert torch.equal((px.double() @ pw.double().t()), x.double() @ w.double().t())
            if offset == 0 and K == Kp:
                assert px.data_ptr() == x.data_ptr() and pw.data_ptr() == w.data_ptr(), "needless copy"
    x = torch.zeros(8, 4, dtype=torch.bfloat16)
    with pytest.raises(ValueError):
        _kernel_operands(x, torch.zeros(8, 5, dtype=torch.bfloat16))
    xt = torch.zeros(64, 8, dtype=torch.bfloat16).t()             # a transposed view is copied
    px, _ = _kernel_operands(xt, torch.zeros(128, 64, dtype=torch.bfloat16))
    assert px.is_contiguous() and torch.equal(px, xt)


@pytest.mark.gpu
@pytest.mark.parametrize("shard", ["offset", "k0", "k96"])
def test_unaligned_or_short_shard_at_world_size_1(shard, kernel_calls, monkeypatch):
    """A view 2 bytes into its buffer, an empty K and a K that is no multiple of 64 all run the kernel
    (errors raise here instead of ending the process) and give the exact product."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    if size > 1:
        pytest.skip("a world-size-1 check")
    monkeypatch.setenv("MPI4JAX_B200_ABORT_ON_ERROR", "0")
    device = comm.device
    M, N, K = 256, 384, {"offset": 64, "k0": 0, "k96": 96}[shard]
    x, w = exact_operands(shard, 0, M, N, K, device)
    if shard == "offset":
        x, w = _offset_view(x), _offset_view(w)
    out = linear_allreduce(x, w, comm=comm)
    _assert_same(out, exact_want(shard, M, N, [K], torch.bfloat16, device), shard)
    assert kernel_calls == [(M, N, max(64, -(-K // 64) * 64))]


HOST_SCRIPT = r"""
import torch
from mpi4jax_b200 import MPI
from mpi4jax_b200.ops import linear_allreduce

comm = MPI.COMM_WORLD
gen = torch.Generator().manual_seed(7)
x = torch.randint(-3, 4, (128, 64), generator=gen).to(torch.bfloat16)
w = torch.randint(-4, 5, (256, 64), generator=gen).to(torch.bfloat16)
want = (x.double() @ w.double().t()).to(torch.bfloat16)        # |S| <= 768: exact, one rounding
out = linear_allreduce(x.to(comm.device), w.to(comm.device), comm=comm)
assert comm.transport == "host", comm.transport
assert torch.equal(out.cpu(), want)
print("host transport ok")
"""


@pytest.mark.gpu
@pytest.mark.parametrize("env", [{"MPI4JAX_B200_TRANSPORT": "host"}, {"MPI4JAX_USE_CUDA_MPI": "0"}],
                         ids=["transport-host", "use-cuda-mpi-0"])
def test_host_transport_falls_back_at_world_size_1(env):
    """With host staging the kernel is not used, even at world size 1: matmul + allreduce instead."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    if inside_job:
        pytest.skip("a world-size-1 check")
    run_env = {**os.environ, **env, "MPI4JAX_B200_ABORT_ON_ERROR": "0"}
    res = subprocess.run([sys.executable, "-c", HOST_SCRIPT], cwd=REPO, env=run_env, capture_output=True,
                         text=True, timeout=600)
    assert res.returncode == 0 and "host transport ok" in res.stdout, res.stdout[-2000:] + res.stderr[-4000:]


@pytest.mark.gpu
def test_output_past_2_31_elements(kernel_calls):
    """(65536 + 256) x 32768 outputs, 4 GiB: the tiles past element 2^31 against the oracle."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    if size > 1:
        pytest.skip("a world-size-1 check")
    if torch.cuda.mem_get_info()[0] < 8 << 30:
        pytest.skip("needs 8 GiB of free device memory")
    device = comm.device
    M, N, K = 65536 + 256, 32768, 64
    x, w = exact_operands("2^31", 0, M, N, K, device)
    out = linear_allreduce(x, w, comm=comm)
    assert kernel_calls == [(M, N, K)]
    wd = w.double().t()
    for r0 in (0, 65536 - 2 * TILE, 65536 - TILE, 65536, M - TILE):     # 65536 * N = 2^31
        want = (x[r0:r0 + TILE].double() @ wd).to(torch.bfloat16)
        _assert_same(out[r0:r0 + TILE], want, f"rows {r0}..{r0 + TILE}")
    del out


def test_linear_allreduce_adjoint_gradcheck():
    """The autograd rule of linear.py against finite differences, in float64 on the CPU."""
    if size > 1:
        pytest.skip("finite differences perturb every rank's operands at once")
    gen = torch.Generator().manual_seed(3)
    x = torch.randn(5, 7, generator=gen, dtype=torch.float64, requires_grad=True)
    w = torch.randn(3, 7, generator=gen, dtype=torch.float64, requires_grad=True)
    assert torch.autograd.gradcheck(lambda a, b: linear_allreduce(a, b, comm=comm), (x, w))


@pytest.mark.gpu
def test_linear_allreduce_grad():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    gen = torch.Generator().manual_seed(1234 + rank)
    x = (torch.randn(128, 128, generator=gen) * 0.5).to(torch.bfloat16).to(comm.device)
    w = (torch.randn(128, 128, generator=gen) * 0.5).to(torch.bfloat16).to(comm.device)
    x.requires_grad_(True)
    w.requires_grad_(True)
    out = linear_allreduce(x, w, comm=comm)
    out.float().sum().backward()
    g = torch.ones(128, 128, dtype=torch.bfloat16, device=comm.device)
    assert torch.allclose(x.grad.float(), (g @ w.detach()).float(), rtol=2e-2, atol=1e-2)
    assert torch.allclose(w.grad.float(), (g.t() @ x.detach()).float(), rtol=2e-2, atol=1e-2)


def test_linear_allreduce_fallback_cpu():
    x = torch.randn(6, 10)
    w = torch.randn(4, 10)
    out = linear_allreduce(x, w, comm=comm)
    assert torch.allclose(out, (x @ w.t()) * 1.0 if size == 1 else m.allreduce(x @ w.t(), MPI.SUM, comm=comm))


# ---------------------------------------------------------------------------
# the tests that take ``device`` as jobs of 2, 3, 5 and 7 ranks
# ---------------------------------------------------------------------------
PEER_TESTS = ["test_linear_allreduce_exact", "test_nan_and_inf_stay_in_their_row_and_column",
              "test_repeated_calls_and_graph_replay", "test_fallback_shapes", "test_uneven_k_shards",
              "test_gemm_interleaved_with_allreduces", "test_linear_allreduce_within_bound"]


def test_job_reports_nvls(device):
    """Passes inside a multi-rank job whose communicator has NVLS, so that the fused path runs there."""
    if device.type != "cuda" or size == 1:
        pytest.skip("reports on a multi-rank CUDA job")
    if comm.transport != "native" or not comm._native_comm().has_nvls:
        pytest.skip("no NVLS: linear_allreduce runs matmul + allreduce")


def _peer_job(nranks, env=None, need_nvls=False):
    code, outs = job(__file__, nranks, " or ".join(PEER_TESTS + ["test_job_reports_nvls"]), env)
    if need_nvls and code == 0 and not re.search(r"^PASSED .*::test_job_reports_nvls\[cuda\]", outs[0], re.M):
        pytest.skip(f"the {nranks}-rank job has no NVLS, so the fused path did not run")
    expect_passed(code, outs, nranks, PEER_TESTS)


@pytest.mark.gpu
@pytest.mark.skipif(inside_job, reason="already inside a multi-rank job")
def test_job_two_ranks():
    """Two ranks on the GPUs there are: the fused path on two NVLS GPUs, matmul + allreduce when the
    ranks share one GPU."""
    _peer_job(2)


@pytest.mark.gpu
@pytest.mark.skipif(inside_job, reason="already inside a multi-rank job")
def test_job_two_ranks_without_nvls():
    """The multi-rank fallback (matmul + allreduce) on two GPUs.  On one GPU test_job_two_ranks runs it."""
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    _peer_job(2, {"MPI4JAX_B200_NVLS": "0"})


@pytest.mark.gpu
@pytest.mark.skipif(inside_job, reason="already inside a multi-rank job")
@pytest.mark.parametrize("nranks", [3, 5, 7])
def test_job_fused_uneven_row_splits(nranks):
    """One rank per GPU with NVLS: the fused epilogue splits each tile's 128 rows into slices of
    ceil(128 / P) rows, the last one shorter.  Runs when the job reports NVLS; every rank must then run
    the kernel."""
    from mpi4jax_b200._src.torch_compat import device_capabilities

    if not torch.cuda.is_available() or torch.cuda.device_count() < nranks:
        pytest.skip(f"needs {nranks} GPUs")
    if not device_capabilities(0)["multicast"]:
        pytest.skip("needs NVLS multicast")
    _peer_job(nranks, need_nvls=True)
