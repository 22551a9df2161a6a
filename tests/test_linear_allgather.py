"""Sequence-parallel column-parallel linear (``ops.linear_allgather``): the allgather + wgmma GEMM kernel of
csrc/b2_gemm_ag.cu, and its fallback, against oracles that never call the library.

Rank q's operands come from a seed of (case, q), so every rank rebuilds every rank's rows and computes the
gathered matrix X itself.  Rank r's expected result is ``rn(X @ W_r^T)``, computed in float64: exact for
the small-integer operands of tests/test_gemm.py, so the kernel and the fallback must match it to the bit.
The kernel needs no multicast, so it runs wherever the native transport does: at world size 1 as the
stand-alone GEMM of linear_allreduce, above one rank also with NVLS off and with two ranks sharing one GPU.

The tests that take ``device`` run at world size 1, and in jobs launched from this file: 2 and 3 CPU
ranks, and on the GPUs there are 2 ranks (sharing the GPU when there is one), 2 ranks with NVLS off, and
3, 4, 5, 7 and 8 ranks when there are that many GPUs."""

import os
import re

import pytest
import torch

import mpi4jax_b200 as m
from mpi4jax_b200 import MPI
from mpi4jax_b200.ops import linear_allgather, linear_allreduce, linear_reduce_scatter

from ._peer_job import REPO, Checks, expect_passed, job
from .test_gemm import (BOUND_CASES, CASES, FALLBACK_CASES, TILE, _assert_bitwise, _assert_same, _expect, _gen,
                        _ints, _offset_view, _sm_count, _ulp_bf16, exact_operands, normal_operands)

comm = MPI.COMM_WORLD
rank, size = comm.Get_rank(), comm.Get_size()
inside_job = size > 1 or "MPI4JAX_B200_NESTED" in os.environ

#: (label, rows per rank m, tile columns, K): shard boundaries inside a tile (m = 64 and 192 at P >= 2,
#: m = 16 at P = 8; elsewhere m = 16 leaves P m unaligned and takes the fallback)
SHARD_CASES = [
    ("m64-k320", 64, 3, 320),
    ("m192-k448", 192, 2, 448),
    ("m16-k64", 16, 5, 64),
]


def _round_up(num_m):
    return -(-num_m // size) * size


@pytest.fixture
def kernel_calls(monkeypatch):
    """Shapes (rows, N, K) of every call of the three GEMM entry points while the test runs, by entry point."""
    from mpi4jax_b200._src.backends.cuda import NativeComm

    calls = {"gemm_allgather": [], "gemm_allreduce": [], "gemm_reduce_scatter": []}
    for name in calls:
        real = getattr(NativeComm, name)

        def spy(self, x, weight, _real=real, _name=name):
            calls[_name].append((x.shape[0], weight.shape[0], x.shape[1]))
            return _real(self, x, weight)

        monkeypatch.setattr(NativeComm, name, spy)
    return calls


def _kernel_expected(device, dtype, rows):
    """Whether linear_allgather must run a kernel: bf16 CUDA operands, P m tile-aligned, the native
    transport; NVLS and this rank's N play no part."""
    if device.type != "cuda" or dtype != torch.bfloat16 or rows == 0 or (size * rows) % TILE:
        return False
    return comm.transport == "native"


def _check_path(chk, calls, expected, label, n=1):
    """The allgather kernel ran ``n`` times above one rank; at world size 1 the stand-alone GEMM of
    linear_allreduce ran instead."""
    fused, plain = len(calls["gemm_allgather"]), len(calls["gemm_allreduce"])
    want = (0, 0) if not expected else (n, 0) if size > 1 else (0, n)
    chk(_expect, (fused, plain) == want,
        f"{label}: gemm_allgather ran {fused} times and gemm_allreduce {plain}, expected {want}")
    for v in calls.values():
        v.clear()


def _gathered(make, case, rows, N, K, device):
    """Every rank's rows ``make(case, q, rows, N, K, device)[0]`` in rank order, and this rank's weight."""
    xs = [make(case, q, rows, N, K, device)[0] for q in range(size)]
    return torch.cat(xs), make(case, rank, rows, N, K, device)[1]


def _exact_want(X, w):
    return (X.double() @ w.double().t()).to(w.dtype)


def _over_rasters(x, w, device):
    """[(gemm_raster, output)] over the tile orders 0, 1, 2, 3, 5, 17 and auto (-1); one call where there is
    no native communicator."""
    if device.type != "cuda" or comm.transport != "native":
        return [("auto", linear_allgather(x, w, comm=comm))]
    nc = comm._native_comm()
    outs = []
    try:
        for r in (-1, 0, 1, 2, 3, 5, 17):
            nc.set_option("gemm_raster", r)
            outs.append((r, linear_allgather(x, w, comm=comm)))
    finally:
        nc.set_option("gemm_raster", -1)
    return outs


def _cases(device):
    """(label, rows per rank, N, K) of the CASES grids (tile rows rounded up to a multiple of P) and the
    shard-boundary cases."""
    g = _sm_count(device)
    out = []
    for label, grid, K in CASES:
        num_m, num_n = grid(g)
        out.append((label, _round_up(num_m) * TILE // size, num_n * TILE, K))
    return out + [(label, rows, tn * TILE, K) for label, rows, tn, K in SHARD_CASES]


# ---------------------------------------------------------------------------
# exact mode
# ---------------------------------------------------------------------------
def test_linear_allgather_exact(device, kernel_calls):
    """Every case in every tile order, to the bit, against ``rn(X @ W_r^T)``."""
    chk = Checks()
    for label, rows, N, K in _cases(device):
        X, w = _gathered(exact_operands, label, rows, N, K, device)
        x = X[rank * rows:(rank + 1) * rows].clone()
        outs = _over_rasters(x, w, device)
        for r, out in outs:
            chk(_assert_same, out, _exact_want(X, w), f"{label} ({size} x {rows} x {N} x {K}), gemm_raster {r}")
        chk(_assert_bitwise, outs, label)
        _check_path(chk, kernel_calls, _kernel_expected(device, x.dtype, rows), label, len(outs))
    chk.finish()


def test_bitwise_equal_to_the_standalone_gemm(device, kernel_calls):
    """Normal operands: the same bits as linear_allreduce of the gathered matrix on a one-rank communicator,
    which runs the same mainloop."""
    chk = Checks()
    solo = comm.Split(rank, 0)
    for label, rows, N, K in _cases(device)[3:6] + [("range-k256", 2 * TILE, 384, 256)]:
        X, w = _gathered(normal_operands, label, rows, N, K, device)
        out = linear_allgather(X[rank * rows:(rank + 1) * rows].clone(), w, comm=comm)
        ref = linear_allreduce(X, w, comm=solo)
        chk(_expect, torch.equal(out.view(torch.int16), ref.view(torch.int16)),
            f"{label}: linear_allgather and the stand-alone GEMM differ in bits")
        for v in kernel_calls.values():
            v.clear()
    chk.finish()


def test_nan_and_inf_stay_in_their_row_and_column(device, kernel_calls):
    """Rank q puts a NaN in its row m_q and rank r an inf in its weight row n_r.  Global row q m + m_q is NaN
    on every rank, column n_r inf or NaN on rank r only, and every other element matches the oracle."""
    label, rows, N, K = _cases(device)[4]
    chk = Checks()
    where = [((37 + 101 * q) % rows, (5 + 3 * q) % K, (53 + 67 * q) % N, (K - 1 - q) % K) for q in range(size)]
    X, w = _gathered(exact_operands, label, rows, N, K, device)
    for q in range(size):
        X[q * rows + where[q][0], where[q][1]] = float("nan")
    w[where[rank][2], where[rank][3]] = float("inf")
    want = _exact_want(X, w)
    nan_rows = [q * rows + where[q][0] for q in range(size)]
    assert want[nan_rows].isnan().all()
    outs = _over_rasters(X[rank * rows:(rank + 1) * rows].clone(), w, device)
    for r, out in outs:
        chk(_assert_same, out, want, f"{label} with NaN / inf, gemm_raster {r}")
        finite = torch.ones(size * rows, N, dtype=torch.bool, device=device)
        finite[nan_rows] = False
        finite[:, where[rank][2]] = False
        chk(_expect, out[finite].isfinite().all().item(), f"gemm_raster {r}: a NaN or inf left its row or column")
    chk(_assert_bitwise, outs, label)
    _check_path(chk, kernel_calls, _kernel_expected(device, X.dtype, rows), label, len(outs))
    chk.finish()


def test_repeated_calls_and_graph_replay(device, kernel_calls):
    """Three eager calls give the same bits, and a CUDA graph of the call replayed four times with new
    operands copied into its inputs (both staging halves reused) gives each set's exact result."""
    label, rows, N, K = _cases(device)[4]
    chk = Checks()
    sets = [_gathered(exact_operands, f"{label}/{i}", rows, N, K, device) for i in range(3)]
    x, w = sets[0][0][rank * rows:(rank + 1) * rows].clone(), sets[0][1]
    outs = [(i, linear_allgather(x, w, comm=comm)) for i in range(3)]
    chk(_assert_same, outs[0][1], _exact_want(*sets[0]), f"{label}, eager")
    chk(_assert_bitwise, outs, f"{label}, repeated calls")
    n = 3
    if device.type == "cuda":
        xs, ws = x.clone(), w.clone()
        graph = torch.cuda.CUDAGraph()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            linear_allgather(xs, ws, comm=comm)          # warm-up on the capture stream
            with torch.cuda.graph(graph, stream=side, capture_error_mode="thread_local"):
                out_g = linear_allgather(xs, ws, comm=comm)
        torch.cuda.current_stream().wait_stream(side)
        for i in (1, 2, 0, 1):
            X, wn = sets[i]
            xs.copy_(X[rank * rows:(rank + 1) * rows])
            ws.copy_(wn)
            graph.replay()
            chk(_assert_same, out_g, _exact_want(X, wn), f"{label}, graph replayed with operand set {i}")
        chk(_assert_bitwise, [("eager", outs[0][1]), ("graph", linear_allgather(x, w, comm=comm))], label)
        n += 3                # warm-up, capture and the last eager call; a replay does not go through Python
    _check_path(chk, kernel_calls, _kernel_expected(device, x.dtype, rows), label, n)
    chk.finish()


def test_jit_equals_eager(device, kernel_calls):
    """``mpi4jax_b200.jit`` of the op gives the eager bits, call after call."""
    rows, N, K = TILE, 256, 128
    X, w = _gathered(exact_operands, "jit", rows, N, K, device)
    x = X[rank * rows:(rank + 1) * rows].clone()
    fast = m.jit(lambda a, b: linear_allgather(a, b, comm=comm))
    for i in range(3):
        assert torch.equal(fast(x, w), linear_allgather(x, w, comm=comm)), i
    _assert_same(fast(x, w), _exact_want(X, w), "jit")


#: rank q % 4's N; with the K = 96 of the test, which the kernel pads to 128
UNEVEN_N = [0, 100, 128, 384]


def test_uneven_n_shards(device, kernel_calls):
    """Ranks with N of 0, 100, 128 and 384 columns, one x 2 bytes into its buffer, and a K the kernel pads
    make the same fuse decision; each rank gets its own (P m, N_r) result."""
    label, rows, K = "uneven-n", TILE, 96
    chk = Checks()
    N = UNEVEN_N[rank % 4]
    xs = [exact_operands(label, q, rows, 8, K, device)[0] for q in range(size)]
    X = torch.cat(xs)
    w = exact_operands(f"{label}/w", rank, 8, max(N, 1), K, device)[1][:N]
    x = X[rank * rows:(rank + 1) * rows].clone()
    if rank % 4 == 1:
        x = _offset_view(x)
        assert x.is_contiguous() and x.data_ptr() % 16 == 2
    out = linear_allgather(x, w, comm=comm)
    chk(_assert_same, out, _exact_want(X, w), f"{label}: N = {N}")
    _check_path(chk, kernel_calls, _kernel_expected(device, x.dtype, rows), label)
    chk.finish()


def test_fallback_shapes(device, kernel_calls):
    """The shapes and dtypes the kernel does not take go through allgather + matmul against the same oracle
    (FALLBACK_CASES' M is the rows per rank here); the kernel-call counts show which path ran."""
    chk = Checks()
    for label, dtype, rows, N, K in FALLBACK_CASES:
        X, w = _gathered(lambda *a: exact_operands(*a, dtype), label, rows, N, K, device)
        out = linear_allgather(X[rank * rows:(rank + 1) * rows].clone(), w, comm=comm)
        chk(_assert_same, out, _exact_want(X, w), label)
        _check_path(chk, kernel_calls, _kernel_expected(device, dtype, rows), label)
    chk.finish()


def test_interleaved_with_other_collectives(device, kernel_calls):
    """Small and large allgather GEMMs (the large ones grow the staging segment) mixed with
    linear_reduce_scatter, linear_allreduce, allreduce and allgather of other sizes, which advance the same
    ticket and write the staging halves the kernel gathers into."""
    chk = Checks()
    big = (TILE * 16, 1024, 2048) if device.type == "cuda" else (TILE, 512, 128)
    steps = [("ag", (TILE, 128, 64)), ("allreduce", 1000), ("rs", (TILE * size, 256, 128)), ("ag", big),
             ("allgather", 3 << 18), ("ar", (384, 640, 192)), ("ag", (64, 384, 128)), ("allreduce", 17),
             ("rs", (TILE * size * 4, 2048, 64)), ("allgather", 5), ("ag", big), ("ag", (TILE, 128, 64))]
    for i, (kind, arg) in enumerate(steps):
        label = f"step {i}: {kind} {arg}"
        if kind == "ag":
            rows, N, K = arg
            X, w = _gathered(exact_operands, label, rows, N, K, device)
            x = X[rank * rows:(rank + 1) * rows].clone()
            chk(_assert_same, linear_allgather(x, w, comm=comm), _exact_want(X, w), label)
            _check_path(chk, kernel_calls, _kernel_expected(device, x.dtype, rows), label)
        elif kind in ("rs", "ar"):
            M, N, K = arg
            parts = [exact_operands(label, q, M, N, K, device) for q in range(size)]
            full = sum((x.double() @ w.double().t()).to(torch.bfloat16).double() for x, w in parts).to(torch.bfloat16)
            x, w = parts[rank]
            if kind == "rs":
                got, want = linear_reduce_scatter(x, w, comm=comm), full[rank * M // size:(rank + 1) * M // size]
            else:
                got, want = linear_allreduce(x, w, comm=comm), full
            chk(_assert_same, got, want, label)
            for v in kernel_calls.values():
                v.clear()
        elif kind == "allreduce":
            out = m.allreduce(_ints(label, rank, arg, device), MPI.SUM, comm=comm)
            chk(_assert_same, out, sum(_ints(label, q, arg, device).double() for q in range(size)).float(), label)
        else:
            out = m.allgather(_ints(label, rank, arg, device), comm=comm)
            chk(_assert_same, out, torch.stack([_ints(label, q, arg, device) for q in range(size)]), label)
    chk.finish()


# ---------------------------------------------------------------------------
# bound mode
# ---------------------------------------------------------------------------
def test_linear_allgather_within_bound(device, kernel_calls):
    """Every element within ``1/2 ulp_bf16(|S| + e) + e`` of the exact S, ``e = K 2^-22 sum_k |x| |w|`` (one
    fp32 accumulation, one rounding: no partials to sum), the same bits in every tile order; prints the
    worst err / bound."""
    chk = Checks()
    g = _sm_count(device)
    for label, grid, K in BOUND_CASES:
        num_m, num_n = grid(g)
        rows, N = _round_up(num_m) * TILE // size, num_n * TILE
        X, w = _gathered(normal_operands, label, rows, N, K, device)
        Xd, wd = X.double(), w.double()
        S = Xd @ wd.t()
        e = K * 2.0 ** -22 * (Xd.abs() @ wd.abs().t())
        bound = 0.5 * _ulp_bf16(S.abs() + e) + e
        outs = _over_rasters(X[rank * rows:(rank + 1) * rows].clone(), w, device)
        ratio = ((outs[0][1].double() - S).abs() / bound).nan_to_num(float("inf"))
        worst = ratio.max().item()
        print(f"linear_allgather {label} ({size} x {rows} x {N} x {K}) on {device.type}, rank {rank}: "
              f"worst err / bound {worst:.4f}")
        chk(_expect, worst <= 1.0, f"{label}: err / bound {worst:.4f}")
        chk(_assert_bitwise, outs, label)
        _check_path(chk, kernel_calls, _kernel_expected(device, X.dtype, rows), label, len(outs))
    chk.finish()


def test_byte_offsets_past_2_31(device, kernel_calls):
    """Two ranks gathering 2 x 32768 x 16448 bf16 (2.16e9 bytes, past 2^31): rows whose staging offsets lie
    past 2^31 bytes, and rows of both shards, against the oracle.  Run by its own two-rank GPU job."""
    if device.type != "cuda" or size != 2:
        pytest.skip("a two-rank GPU check")
    rows, N, K = 32768, TILE, 16448
    assert size * rows * K * 2 > 2 ** 31

    def shard(q):
        gen = _gen("2^31", q, device)
        return torch.randint(-2, 3, (rows, K), generator=gen, device=device, dtype=torch.int8).to(torch.bfloat16)

    w = torch.randint(-2, 3, (N, K), generator=_gen("2^31/w", rank, device), device=device,
                      dtype=torch.int8).to(torch.bfloat16)
    out = linear_allgather(shard(rank), w, comm=comm)
    assert kernel_calls["gemm_allgather"] == [(rows, N, K)]
    wd = w.double().t()
    for r0 in (0, rows - TILE, rows, 2 * rows - 2 * TILE, 2 * rows - TILE):   # past row 65281: byte 2^31
        q, lo = divmod(r0, rows)
        xq = shard(q)[lo:lo + TILE]
        _assert_same(out[r0:r0 + TILE], (xq.double() @ wd).to(torch.bfloat16), f"rows {r0}..{r0 + TILE}")
    del out


# ---------------------------------------------------------------------------
# the adjoint
# ---------------------------------------------------------------------------
def test_linear_allgather_adjoint_gradcheck():
    """The autograd rule against finite differences, in float64 on the CPU."""
    if size > 1:
        pytest.skip("finite differences perturb every rank's operands at once")
    gen = torch.Generator().manual_seed(9)
    x = torch.randn(6, 7, generator=gen, dtype=torch.float64, requires_grad=True)
    w = torch.randn(3, 7, generator=gen, dtype=torch.float64, requires_grad=True)
    assert torch.autograd.gradcheck(lambda a, b: linear_allgather(a, b, comm=comm), (x, w))


def _tern(case, q, shape, density, device):
    """Entries in {-1, 0, 1}, nonzero with probability ``density``."""
    gen = _gen(case, q, device)
    v = torch.randint(0, 2, shape, generator=gen, device=device, dtype=torch.float32) * 2 - 1
    return v * (torch.rand(shape, generator=gen, device=device) < density)


def test_adjoint_identities_exact(device, kernel_calls):
    """With ternary operands whose every sum is exact in bf16 and N_q = 128 or 256 by rank,
    ``sum_r <y_r, g_r> = sum_r <x_r, grad_x_r> = sum_r <w_r, grad_w_r>`` exactly, grad_x is rows r of
    ``sum_q g_q @ W_q`` and grad_w is ``g_r^T @ X``."""
    rows, K = TILE, TILE
    ns = [TILE * (1 + q % 2) for q in range(size)]
    dtype = torch.bfloat16 if device.type == "cuda" else torch.float32
    xs = [_tern("adj-x", q, (rows, K), 0.25, device) for q in range(size)]
    ws = [_tern("adj-w", q, (ns[q], K), 0.5, device) for q in range(size)]
    gs = [_tern("adj-g", q, (size * rows, ns[q]), 1 / 16, device) for q in range(size)]
    X = torch.cat(xs).double()
    assert max((g.abs().double() @ w.abs().double()).max().item() for g, w in zip(gs, ws)) * size <= 256
    assert (gs[rank].abs().double().t() @ X.abs()).max().item() <= 256
    x = xs[rank].to(dtype).requires_grad_()
    w = ws[rank].to(dtype).requires_grad_()
    y = linear_allgather(x, w, comm=comm)
    gx, gw = torch.autograd.grad(y, (x, w), gs[rank].to(dtype))
    full_gx = sum(g.double() @ wq.double() for g, wq in zip(gs, ws))
    assert torch.equal(gx.double(), full_gx[rank * rows:(rank + 1) * rows])
    assert torch.equal(gw.double(), gs[rank].double().t() @ X)
    dots = [(y.detach().double() * gs[rank].double()).sum().item(), (x.detach().double() * gx.double()).sum().item(),
            (w.detach().double() * gw.double()).sum().item()]
    total = [sum(v) for v in zip(*comm.allgather(dots))]
    assert total[0] == total[1] == total[2], total
    # forward and the grad_x reduce-scatter; at world size 1 both are the stand-alone GEMM
    ran = {k: len(v) for k, v in kernel_calls.items()}
    if not _kernel_expected(device, dtype, rows):
        assert not any(ran.values()), ran
    else:
        want = {"gemm_allgather": 1, "gemm_allreduce": 0, "gemm_reduce_scatter": 1} if size > 1 else \
            {"gemm_allgather": 0, "gemm_allreduce": 2, "gemm_reduce_scatter": 0}
        assert ran == want, ran


def test_bad_operands_raise_everywhere(device, kernel_calls):
    """Operands that are not 2-D, or whose K differ, raise ValueError on every rank before any device work,
    and the next collective still works."""
    x = torch.zeros(TILE, 64, dtype=torch.bfloat16, device=device)
    for a, b in ((x[0], torch.zeros(TILE, 64, dtype=torch.bfloat16, device=device)),
                 (x, torch.zeros(2, TILE, 64, dtype=torch.bfloat16, device=device)),
                 (x, torch.zeros(TILE, 63, dtype=torch.bfloat16, device=device))):
        with pytest.raises(ValueError, match="linear_allgather"):
            linear_allgather(a, b, comm=comm)
    assert not any(kernel_calls.values())
    out = m.allreduce(torch.full((5,), float(rank), device=device), MPI.SUM, comm=comm)
    assert torch.equal(out, torch.full((5,), float(size * (size - 1) // 2), device=device))


# ---------------------------------------------------------------------------
# jobs
# ---------------------------------------------------------------------------
PEER_TESTS = ["test_linear_allgather_exact", "test_bitwise_equal_to_the_standalone_gemm",
              "test_nan_and_inf_stay_in_their_row_and_column", "test_repeated_calls_and_graph_replay",
              "test_jit_equals_eager", "test_uneven_n_shards", "test_fallback_shapes",
              "test_interleaved_with_other_collectives", "test_linear_allgather_within_bound",
              "test_adjoint_identities_exact", "test_bad_operands_raise_everywhere"]


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


def _gpu_job(nranks, env=None, tests=PEER_TESTS):
    code, outs = job(__file__, nranks, " or ".join(tests), env)
    expect_passed(code, outs, nranks, tests)


@pytest.mark.gpu
@pytest.mark.skipif(inside_job, reason="already inside a multi-rank job")
def test_job_two_ranks():
    """Two ranks on the GPUs there are; on one GPU both share it and run the kernel."""
    _gpu_job(2)


@pytest.mark.gpu
@pytest.mark.skipif(inside_job, reason="already inside a multi-rank job")
def test_job_two_ranks_past_2_31_bytes():
    """The byte-offset check as a two-rank job; it needs about 40 GiB of device memory for both ranks."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    need = (40 << 30) if torch.cuda.device_count() < 2 else (20 << 30)
    if torch.cuda.mem_get_info()[0] < need:
        pytest.skip("not enough free device memory")
    _gpu_job(2, tests=["test_byte_offsets_past_2_31"])


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
    """One rank per GPU: shard boundaries inside tiles, m = 16 at P = 8."""
    if not torch.cuda.is_available() or torch.cuda.device_count() < nranks:
        pytest.skip(f"needs {nranks} GPUs")
    _gpu_job(nranks)
