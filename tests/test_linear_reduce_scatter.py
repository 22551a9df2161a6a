"""Sequence-parallel linear (``ops.linear_reduce_scatter``): the wgmma GEMM + pull-and-fold reduce-scatter
kernel of csrc/b2_gemm_rs.cu, and its fallback, against the oracle of tests/test_gemm.py.

Rank r's expected result is rows ``[r M/P, (r+1) M/P)`` of that oracle, ``rn(sum_q rn(S_q))``: exact for
the small-integer operands, so the kernel and the fallback must both match it to the bit.  The kernel
needs no multicast, so it runs wherever the native transport does: at world size 1 as the stand-alone
GEMM of linear_allreduce, above one rank also with NVLS off and with two ranks sharing one GPU.

The tests that take ``device`` run at world size 1, and in jobs launched from this file: 2 and 3 CPU
ranks, and on the GPUs there are 2 ranks (sharing the GPU when there is one), 2 ranks with NVLS off, and
3, 4, 5, 7 and 8 ranks when there are that many GPUs."""

import os
import re

import pytest
import torch

import mpi4jax_b200 as m
from mpi4jax_b200 import MPI
from mpi4jax_b200.models import ParallelMLP
from mpi4jax_b200.ops import linear_allreduce, linear_reduce_scatter

from ._peer_job import REPO, Checks, expect_passed, job
from .test_gemm import (BOUND_CASES, CASES, FALLBACK_CASES, TILE, UNEVEN_K, _assert_bitwise, _assert_same,
                        _exercises_rounding_and_every_k16, _expect, _gen, _ints, _offset_view, _sm_count,
                        bound_reference, exact_operands, exact_want, normal_operands)

comm = MPI.COMM_WORLD
rank, size = comm.Get_rank(), comm.Get_size()
inside_job = size > 1 or "MPI4JAX_B200_NESTED" in os.environ

#: tile grids with an odd number of tile rows: at P = 2, 4 and 8 a shard boundary falls inside a tile, and
#: the 1-row grid gives 64-row shards at P = 2
ODD_CASES = [
    ("odd-1x3-k64", lambda g: (1, 3), 64),
    ("odd-3x2-k320", lambda g: (3, 2), 320),
    ("odd-5xg-k448", lambda g: (5, g), 448),
]


def _mine(t, q=None):
    """Rank q's (this rank's) row shard of a full (M, N) result."""
    q = rank if q is None else q
    M = t.shape[0]
    return t[q * M // size:(q + 1) * M // size]


def _round_up(num_m):
    return -(-num_m // size) * size


@pytest.fixture
def kernel_calls(monkeypatch):
    """Shapes (M, N, K) of every call of the two GEMM entry points while the test runs, by entry point."""
    from mpi4jax_b200._src.backends.cuda import NativeComm

    calls = {"gemm_reduce_scatter": [], "gemm_allreduce": []}
    for name in calls:
        real = getattr(NativeComm, name)

        def spy(self, x, weight, _real=real, _name=name):
            calls[_name].append((x.shape[0], weight.shape[0], x.shape[1]))
            return _real(self, x, weight)

        monkeypatch.setattr(NativeComm, name, spy)
    return calls


def _kernel_expected(device, dtype, M, N):
    """Whether linear_reduce_scatter must run a kernel: bf16 tile-aligned CUDA operands on the native
    transport, NVLS or not."""
    if device.type != "cuda" or dtype != torch.bfloat16 or M == 0 or N == 0 or M % TILE or N % TILE:
        return False
    return comm.transport == "native"


def _check_path(chk, calls, expected, label, n=1):
    """The fused reduce-scatter kernel ran ``n`` times above one rank; at world size 1 the stand-alone GEMM
    of linear_allreduce ran instead."""
    fused, plain = len(calls["gemm_reduce_scatter"]), len(calls["gemm_allreduce"])
    want = (0, 0) if not expected else (n, 0) if size > 1 else (0, n)
    chk(_expect, (fused, plain) == want,
        f"{label}: gemm_reduce_scatter ran {fused} times and gemm_allreduce {plain}, expected {want}")
    for v in calls.values():
        v.clear()


def _over_rasters(x, w, num_m, device):
    """[(gemm_raster, output)] over the tile orders 0, 1, 2, 3, num_m, num_m + 1 and auto (-1); one call
    where there is no native communicator."""
    if device.type != "cuda" or comm.transport != "native":
        return [("auto", linear_reduce_scatter(x, w, comm=comm))]
    nc = comm._native_comm()
    outs = []
    try:
        for r in dict.fromkeys((-1, 0, 1, 2, 3, num_m, num_m + 1)):
            nc.set_option("gemm_raster", r)
            outs.append((r, linear_reduce_scatter(x, w, comm=comm)))
    finally:
        nc.set_option("gemm_raster", -1)
    return outs


# ---------------------------------------------------------------------------
# exact mode
# ---------------------------------------------------------------------------
def test_linear_reduce_scatter_exact(device, kernel_calls):
    """Every case (tile rows rounded up to a multiple of P) and the odd grids, in every tile order, to the
    bit against this rank's rows of ``rn(sum_q rn(S_q))``."""
    chk = Checks()
    g = _sm_count(device)
    cases = [(lb, (lambda gr: lambda g: (_round_up(gr(g)[0]), gr(g)[1]))(gr), K) for lb, gr, K in CASES]
    for label, grid, K in cases + ODD_CASES:
        num_m, num_n = grid(g)
        M, N = num_m * TILE, num_n * TILE
        if M % size:
            continue                        # an odd grid that P does not divide (P = 3, 5, 7)
        _exercises_rounding_and_every_k16(label, M, N, K, device)
        x, w = exact_operands(label, rank, M, N, K, device)
        full = exact_want(label, M, N, [K] * size, torch.bfloat16, device)
        outs = _over_rasters(x, w, num_m, device)
        for r, out in outs:
            chk(_assert_same, out, _mine(full), f"{label} ({M} x {N} x {K}), gemm_raster {r}")
        chk(_assert_bitwise, outs, label)
        _check_path(chk, kernel_calls, _kernel_expected(device, x.dtype, M, N), label, len(outs))
        chk.add(label, outs[0][1], [_mine(full, q) for q in range(size)])     # every rank holds its own rows
    chk.finish()


def test_nan_and_inf_stay_in_their_row_and_column(device, kernel_calls):
    """Rank q puts a NaN at x[m_q, k] and an inf in w[n_q, :].  Rows m_q become NaN, column n_q inf or NaN,
    in whichever rank's shard they lie, and every other element still matches the oracle."""
    label, grid, K = CASES[4]
    chk = Checks()
    num_m, num_n = grid(_sm_count(device))
    num_m = _round_up(num_m)
    M, N = num_m * TILE, num_n * TILE
    where = [((37 + 101 * q) % M, (5 + 3 * q) % K, (53 + 67 * q) % N, (K - 1 - q) % K) for q in range(size)]

    def edit(q, x, w):
        m0, k0, n0, k1 = where[q]
        x[m0, k0] = float("nan")
        w[n0, k1] = float("inf")

    x, w = exact_operands(label, rank, M, N, K, device)
    edit(rank, x, w)
    full = exact_want(label, M, N, [K] * size, torch.bfloat16, device, edit)
    want = _mine(full)
    rows = sorted({m0 for m0, _, _, _ in where})
    cols = sorted({n0 for _, _, n0, _ in where})
    assert full[rows].isnan().all()
    lo = rank * M // size
    outs = _over_rasters(x, w, num_m, device)
    for r, out in outs:
        chk(_assert_same, out, want, f"{label} with NaN / inf, gemm_raster {r}")
        finite = torch.ones(M // size, N, dtype=torch.bool, device=device)
        finite[[m0 - lo for m0 in rows if lo <= m0 < lo + M // size]] = False
        finite[:, cols] = False
        chk(_expect, out[finite].isfinite().all().item(), f"gemm_raster {r}: a NaN or inf left its row or column")
    chk(_assert_bitwise, outs, label)
    _check_path(chk, kernel_calls, _kernel_expected(device, x.dtype, M, N), label, len(outs))
    chk.finish()


def test_repeated_calls_and_graph_replay(device, kernel_calls):
    """Three eager calls give the same bits, and so does a CUDA graph of the call replayed with new
    operands copied into its inputs."""
    label, grid, K = CASES[4]
    chk = Checks()
    num_m, num_n = grid(_sm_count(device))
    num_m = _round_up(num_m)
    M, N = num_m * TILE, num_n * TILE
    x, w = exact_operands(label, rank, M, N, K, device)
    x2, w2 = exact_operands(label + "/2", rank, M, N, K, device)
    want = _mine(exact_want(label, M, N, [K] * size, torch.bfloat16, device))
    want2 = _mine(exact_want(label + "/2", M, N, [K] * size, torch.bfloat16, device))
    outs = [(i, linear_reduce_scatter(x, w, comm=comm)) for i in range(3)]
    chk(_assert_same, outs[0][1], want, f"{label}, eager")
    chk(_assert_bitwise, outs, f"{label}, repeated calls")
    n = 3
    if device.type == "cuda":
        xs, ws = x.clone(), w.clone()
        graph = torch.cuda.CUDAGraph()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            linear_reduce_scatter(xs, ws, comm=comm)          # warm-up on the capture stream
            with torch.cuda.graph(graph, stream=side, capture_error_mode="thread_local"):
                out_g = linear_reduce_scatter(xs, ws, comm=comm)
        torch.cuda.current_stream().wait_stream(side)
        for xn, wn, wt, tag in ((x2, w2, want2, "new"), (x, w, want, "first")):
            xs.copy_(xn)
            ws.copy_(wn)
            graph.replay()
            chk(_assert_same, out_g, wt, f"{label}, graph replayed with the {tag} operands")
        chk(_assert_bitwise, [("eager", outs[0][1]), ("graph", out_g)], f"{label}, graph replay")
        n += 2                # warm-up and capture; a replay does not go through Python
    _check_path(chk, kernel_calls, _kernel_expected(device, x.dtype, M, N), label, n)
    chk.finish()


def test_fallback_shapes(device, kernel_calls):
    """The shapes and dtypes the kernel does not take go through matmul + reduce_scatter against the same
    oracle; an M that P does not divide raises ValueError on every rank."""
    chk = Checks()
    for label, dtype, M, N, K in FALLBACK_CASES:
        x, w = exact_operands(label, rank, M, N, K, device, dtype)
        if M % size:
            with pytest.raises(ValueError, match="not divisible"):
                linear_reduce_scatter(x, w, comm=comm)
            _check_path(chk, kernel_calls, False, label)
            continue
        out = linear_reduce_scatter(x, w, comm=comm)
        chk(_assert_same, out, _mine(exact_want(label, M, N, [K] * size, dtype, device)), label)
        _check_path(chk, kernel_calls, _kernel_expected(device, dtype, M, N), label)
    chk.finish()


def test_rows_not_divisible_by_ranks_raise_everywhere(device, kernel_calls):
    """M % P != 0 raises ValueError on every rank before any device work, on the kernel's shapes too, and the
    next collective still works."""
    if size == 1:
        pytest.skip("every M is divisible by one rank")
    for M in [TILE * size + 1, TILE * size - 1] + ([TILE] if TILE % size else []):
        x, w = exact_operands(f"bad-{M}", rank, M, TILE, 64, device)
        with pytest.raises(ValueError, match="not divisible"):
            linear_reduce_scatter(x, w, comm=comm)
    assert not any(kernel_calls.values())
    out = m.allreduce(torch.full((5,), float(rank), device=device), MPI.SUM, comm=comm)
    assert torch.equal(out, torch.full((5,), float(size * (size - 1) // 2), device=device))


def test_uneven_k_shards(device, kernel_calls):
    """Ranks with K shards of different lengths and alignment, one of them empty, make the same fuse
    decision and compute the sum of their products."""
    label, M, N = "uneven-k-rs", 256 * size, 384
    chk = Checks()
    ks = [int(str(UNEVEN_K[q % 4]).split("@")[0]) for q in range(size)]
    x, w = exact_operands(label, rank, M, N, ks[rank], device)
    if UNEVEN_K[rank % 4] == "64@2":
        x, w = _offset_view(x), _offset_view(w)
        assert x.is_contiguous() and x.data_ptr() % 16 == 2
    out = linear_reduce_scatter(x, w, comm=comm)
    chk(_assert_same, out, _mine(exact_want(label, M, N, ks, torch.bfloat16, device)), f"{label}: K shards {ks}")
    _check_path(chk, kernel_calls, _kernel_expected(device, x.dtype, M, N), label)
    chk.finish()


def test_interleaved_with_other_collectives(device, kernel_calls):
    """Small and large GEMM reduce-scatters (the large ones grow the staging segment) mixed with
    linear_allreduce, allreduce and reduce_scatter of other sizes, whose grids advance the per-block epochs
    the fused epilogue shares."""
    chk = Checks()
    big = (TILE * size * 16, 8192, 64) if device.type == "cuda" else (TILE * size * 2, 1024, 64)
    steps = [("rs", (TILE * size, 128, 64)), ("allreduce", 1000), ("ar", (384, 640, 192)),
             ("rs", big), ("reduce_scatter", 3 << 18), ("rs", (TILE * size, 384, 128)), ("allreduce", 17),
             ("reduce_scatter", 5), ("ar", (256, 128, 64)), ("rs", big)]
    for i, (kind, arg) in enumerate(steps):
        label = f"step {i}: {kind} {arg}"
        if kind in ("rs", "ar"):
            M, N, K = arg
            x, w = exact_operands(label, rank, M, N, K, device)
            full = exact_want(label, M, N, [K] * size, torch.bfloat16, device)
            if kind == "rs":
                chk(_assert_same, linear_reduce_scatter(x, w, comm=comm), _mine(full), label)
                _check_path(chk, kernel_calls, _kernel_expected(device, x.dtype, M, N), label)
            else:
                chk(_assert_same, linear_allreduce(x, w, comm=comm), full, label)
                for v in kernel_calls.values():
                    v.clear()
        elif kind == "allreduce":
            out = m.allreduce(_ints(label, rank, arg, device), MPI.SUM, comm=comm)
            chk(_assert_same, out, sum(_ints(label, q, arg, device).double() for q in range(size)).float(), label)
        else:
            out = m.reduce_scatter(_ints(label, rank, size * arg, device).reshape(size, arg), MPI.SUM, comm=comm)
            want = sum(_ints(label, q, size * arg, device).double() for q in range(size)).float()
            chk(_assert_same, out, want.reshape(size, arg)[rank], label)
    chk.finish()


# ---------------------------------------------------------------------------
# bound mode
# ---------------------------------------------------------------------------
def test_linear_reduce_scatter_within_bound(device, kernel_calls):
    """Every element within its own bound, the same bits in every tile order; prints the worst err / bound."""
    chk = Checks()
    g = _sm_count(device)
    for label, grid, K in BOUND_CASES:
        num_m, num_n = grid(g)
        num_m = _round_up(num_m)
        M, N = num_m * TILE, num_n * TILE
        x, w = normal_operands(label, rank, M, N, K, device)
        S, bound = bound_reference(label, M, N, K, device)
        S, bound = _mine(S), _mine(bound)
        outs = _over_rasters(x, w, num_m, device)
        ratio = ((outs[0][1].double() - S).abs() / bound).nan_to_num(float("inf"))
        worst = ratio.max().item()
        print(f"linear_reduce_scatter {label} ({M} x {N} x {K}) at {size} rank(s) on {device.type}, rank {rank}: "
              f"worst err / bound {worst:.4f}")
        chk(_expect, worst <= 1.0, f"{label}: err / bound {worst:.4f}")
        chk(_assert_bitwise, outs, label)
        _check_path(chk, kernel_calls, _kernel_expected(device, x.dtype, M, N), label, len(outs))
    chk.finish()


# ---------------------------------------------------------------------------
# the adjoint
# ---------------------------------------------------------------------------
def test_linear_reduce_scatter_adjoint_gradcheck():
    """The autograd rule against finite differences, in float64 on the CPU."""
    if size > 1:
        pytest.skip("finite differences perturb every rank's operands at once")
    gen = torch.Generator().manual_seed(5)
    x = torch.randn(6, 7, generator=gen, dtype=torch.float64, requires_grad=True)
    w = torch.randn(3, 7, generator=gen, dtype=torch.float64, requires_grad=True)
    assert torch.autograd.gradcheck(lambda a, b: linear_reduce_scatter(a, b, comm=comm), (x, w))


def _tern(case, q, shape, density, device):
    """Entries in {-1, 0, 1}, nonzero with probability ``density``."""
    gen = _gen(case, q, device)
    v = torch.randint(0, 2, shape, generator=gen, device=device, dtype=torch.float32) * 2 - 1
    return v * (torch.rand(shape, generator=gen, device=device) < density)


def test_adjoint_identities_exact(device, kernel_calls):
    """With integer operands whose every sum is exact in bf16, ``sum_r <y_r, g_r>`` equals
    ``sum_r <x_r, grad_x_r>`` and ``sum_r <w_r, grad_w_r>`` exactly, and the gradients are ``G @ w`` and
    ``G.T @ x`` with G every rank's cotangent, in rank order."""
    M, N, K = TILE * size, TILE, 32          # |y| <= K P <= 256, |grad_x| <= N = 128
    dtype = torch.bfloat16 if device.type == "cuda" else torch.float32
    x = _tern("adj-x", rank, (M, K), 0.25, device).to(dtype).requires_grad_()
    w = _tern("adj-w", rank, (N, K), 0.5, device).to(dtype).requires_grad_()
    gs = [_tern("adj-g", q, (M // size, N), 1 / 16, device) for q in range(size)]
    G = torch.cat(gs)
    bound = G.abs().t().double() @ _tern("adj-x", rank, (M, K), 0.25, device).abs().double()
    assert bound.max().item() <= 256, bound.max().item()
    y = linear_reduce_scatter(x, w, comm=comm)
    gx, gw = torch.autograd.grad(y, (x, w), gs[rank].to(dtype))
    assert torch.equal(gx.double(), G.double() @ w.detach().double())
    assert torch.equal(gw.double(), G.double().t() @ x.detach().double())
    dots = [(y.detach().double() * gs[rank].double()).sum().item(), (x.detach().double() * gx.double()).sum().item(),
            (w.detach().double() * gw.double()).sum().item()]
    total = [sum(v) for v in zip(*comm.allgather(dots))]
    assert total[0] == total[1] == total[2], total
    _check_path(Checks(), kernel_calls, _kernel_expected(device, dtype, M, N), "adjoint")


# ---------------------------------------------------------------------------
# ParallelMLP(mode="sp")
# ---------------------------------------------------------------------------
def _mlp_data(q, B, d_in, d_out, device, dtype):
    gen = torch.Generator().manual_seed(2000 + q)
    return torch.randn(B, d_in, generator=gen).to(device, dtype), torch.randn(B, d_out, generator=gen).to(device, dtype)


def _reference_mlp(d_in, d_hidden, d_out, B, device, dtype, seed=0):
    """Loss and full gradients of the same MLP on ONE process, on every rank's rows concatenated."""
    gen = torch.Generator().manual_seed(seed)
    w1 = (torch.randn(d_in, d_hidden, generator=gen) / d_in ** 0.5).to(device, dtype).requires_grad_()
    w2 = (torch.randn(d_hidden, d_out, generator=gen) / d_hidden ** 0.5).to(device, dtype).requires_grad_()
    data = [_mlp_data(q, B, d_in, d_out, device, dtype) for q in range(size)]
    xs, ys = torch.cat([d[0] for d in data]), torch.cat([d[1] for d in data])
    loss = ((torch.tanh(xs @ w1) @ w2 - ys) ** 2).mean()
    g1, g2 = torch.autograd.grad(loss, (w1, w2))
    return loss.detach(), g1, g2


def _sp_check(device, dtype, d_in, d_hidden, d_out, B, rtol):
    mlp = ParallelMLP(d_in, d_hidden, d_out, comm=comm, device=device, dtype=dtype, mode="sp")
    x, y = _mlp_data(rank, B, d_in, d_out, device, dtype)
    loss = mlp.loss(x, y)
    g1, g2 = torch.autograd.grad(loss, mlp.parameters())
    ref_loss, r1, r2 = _reference_mlp(d_in, d_hidden, d_out, B, device, dtype)
    k = d_hidden // size
    r1, r2 = r1[:, rank * k:(rank + 1) * k], r2[rank * k:(rank + 1) * k]
    assert abs(loss.item() - ref_loss.item()) <= rtol * abs(ref_loss.item()), (loss.item(), ref_loss.item())
    for got, ref, name in ((g1, r1, "w1"), (g2, r2, "w2")):
        err = ((got.double() - ref.double()).norm() / ref.double().norm()).item()
        assert err <= rtol, f"{name}: relative error {err:.3g}"


def test_parallel_mlp_sp_matches_one_process(device, kernel_calls):
    """Loss and gradient shards of the sequence-parallel MLP against one process on the concatenated rows;
    in bf16 on CUDA through the fused kernel (relative tolerance 3e-2: bf16 operands, activations and
    gradients)."""
    _sp_check(device, torch.float32, 24, 8 * size, 6, 5, 1e-5)
    if device.type == "cuda":
        B = TILE                                       # P B rows, tile-aligned
        _sp_check(device, torch.bfloat16, 64, 64 * size, TILE, B, 3e-2)
        fused = kernel_calls["gemm_reduce_scatter" if size > 1 else "gemm_allreduce"]
        assert fused == [(size * B, TILE, 64)], kernel_calls


def test_parallel_mlp_sp_jit_step_equals_eager(device, kernel_calls):
    """One ``mpi4jax_b200.jit`` step of the sequence-parallel MLP equals an eager step of a twin model."""
    dtype, B, d_out = (torch.bfloat16, TILE, TILE) if device.type == "cuda" else (torch.float32, 5, 6)
    x, y = _mlp_data(rank, B, 32, d_out, device, dtype)
    eager = ParallelMLP(32, 16 * size, d_out, comm=comm, device=device, dtype=dtype, mode="sp")
    twin = ParallelMLP(32, 16 * size, d_out, comm=comm, device=device, dtype=dtype, mode="sp")
    fast = m.jit(lambda a, b: twin.step(a, b))
    for i in range(3):
        l0 = eager.step(x, y)
        l1 = fast(x, y)
        assert torch.equal(l0, l1), (i, l0.item(), l1.item())
        for p, q in zip(eager.parameters(), twin.parameters()):
            assert torch.equal(p, q), i


# ---------------------------------------------------------------------------
# jobs
# ---------------------------------------------------------------------------
PEER_TESTS = ["test_linear_reduce_scatter_exact", "test_nan_and_inf_stay_in_their_row_and_column",
              "test_repeated_calls_and_graph_replay", "test_fallback_shapes",
              "test_rows_not_divisible_by_ranks_raise_everywhere", "test_uneven_k_shards",
              "test_interleaved_with_other_collectives", "test_linear_reduce_scatter_within_bound",
              "test_adjoint_identities_exact", "test_parallel_mlp_sp_matches_one_process",
              "test_parallel_mlp_sp_jit_step_equals_eager"]


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
        missing = [t for t in PEER_TESTS if not re.search(rf"^PASSED .*::{t}\[cpu\]", out, re.M)]
        assert code == 0 and not missing, f"rank {r} of the {nranks}-rank CPU job (exit code {code}), not passed: " \
                                          f"{missing}:\n{out[-4000:]}"


def _gpu_job(nranks, env=None):
    code, outs = job(__file__, nranks, " or ".join(PEER_TESTS), env)
    expect_passed(code, outs, nranks, PEER_TESTS)


@pytest.mark.gpu
@pytest.mark.skipif(inside_job, reason="already inside a multi-rank job")
def test_job_two_ranks():
    """Two ranks on the GPUs there are; on one GPU both share it and run the fused kernel."""
    _gpu_job(2)


@pytest.mark.gpu
@pytest.mark.skipif(inside_job, reason="already inside a multi-rank job")
def test_job_two_ranks_without_nvls():
    """Two ranks on two GPUs with NVLS off: the kernel needs no multicast, so it still runs."""
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    _gpu_job(2, {"MPI4JAX_B200_NVLS": "0"})


@pytest.mark.gpu
@pytest.mark.skipif(inside_job, reason="already inside a multi-rank job")
@pytest.mark.parametrize("nranks", [3, 4, 5, 7, 8])
def test_job_more_ranks(nranks):
    """One rank per GPU: slices of ceil(128 / P) rows, shard boundaries inside tiles at P = 4 and 8."""
    if not torch.cuda.is_available() or torch.cuda.device_count() < nranks:
        pytest.skip(f"needs {nranks} GPUs")
    _gpu_job(nranks)
