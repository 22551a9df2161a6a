"""reduce_scatter's two device kernels with peers, against the rank-order oracle of test_collective_kernels.py.

Rank q's input is rebuilt on every rank from a seed of (case, q), and the result of rank r is
``_fold([x_q[r] for q])``: rank order, fp32 accumulation for f16 / bf16, integers wrapped back to the dtype,
one rounding.  Results compare bitwise (NaNs by position); floats are also checked against an
extended-precision fold.  Every rank checks its own block and, over the control plane, every other rank's.

The two transports run code no other collective runs (csrc/b2_reduce.cuh):

* LL: ``b2_k_allreduce_ll`` with ``src_stride`` = the block's bytes -- peer p receives block p of the input,
  and a block length that is not a multiple of 16 B loads every vector through ``b2_ll_load``'s byte loop;
* pull: the ``B2_OPC_REDUCE_SCATTER`` branch of ``b2_k_reduce_chunked`` -- chunks index into one block,
  block q is staged from ``in + q * nbytes`` to ``q * round16(nbytes)``, one barrier per chunk, then block
  ``rank`` is pulled from every peer; the tail goes through ``b2_store_partial``.

The debug line of every GPU call names the transport it took, which must be the one ``reduce_algo``
(csrc/b2_collectives.cu) picks; the tests force one with the communicator's ``ll_max``.  In a
single-process run the CUDA tests run in a two-rank job whose ranks share the GPU; the launchers at the
end run them with three and five ranks, and the LL kernel past one wave of CTAs with a larger LL buffer."""

import os
import re

import pytest
import torch

import mpi4jax_b200 as m
from mpi4jax_b200 import MPI
from mpi4jax_b200._src.native import set_logging

from .._peer_job import expect_passed, job, needs_peers
from .test_collective_kernels import (ALL_DTYPES, OPS, Checks, _assert_same, _check_accuracy, _edge_cases, _expect,
                                      _fold, _input, _logged, _n_for, _ops_for, _options, _run_allreduce)

comm = MPI.COMM_WORLD
rank = comm.Get_rank()
size = comm.Get_size()

peers = needs_peers("reduce-scatter kernels between ranks")

# the LL buffer per (parity, source): MPI4JAX_B200_LL_BYTES rounded up to 4 KiB (csrc/b2_runtime.cpp: make_layout);
# an LL block travels as 2x its bytes, so LL_LIMIT is the longest block the LL kernel takes
LL_BUF = (int(os.environ.get("MPI4JAX_B200_LL_BYTES", 128 << 10)) + 4095) // 4096 * 4096
LL_LIMIT = LL_BUF // 2
CPU_MAX = 1 << 20          # the CPU variants (the multi-rank CPU jobs) skip blocks above this


def _rs_transport(nc, nbytes):
    """What reduce_algo picks for a reduce_scatter block of ``nbytes`` (csrc/b2_collectives.cu)."""
    return "ll" if size > 1 and nbytes <= nc.get_option("ll_max") and 2 * nbytes <= LL_BUF else "oneshot"


def _settings(device, auto=False):
    """(name, ll_max) of the transports a test runs: on the GPU LL (``ll_max`` high) and pull (``ll_max`` = 0),
    and with ``auto`` the size table's own choice; on the CPU, whose backend has one path, a single pass."""
    if device.type != "cuda":
        return (("cpu", None),)
    return ((("auto", None),) if auto else ()) + (("ll", 1 << 30), ("pull", 0))


def _ll_max(device, value):
    return _options(device) if value is None else _options(device, ll_max=value)


def _canon(t):
    """``t`` flattened (``digest`` views 1-d bytes), every NaN the same NaN and -0.0 as +0.0: the bits
    ``_assert_same`` compares."""
    t = t.detach().cpu().reshape(-1)
    if t.dtype.is_complex:
        t = torch.view_as_real(t)
    if t.dtype.is_floating_point:
        t = torch.where(torch.isnan(t), torch.tensor(float("nan"), dtype=t.dtype), t + 0)
    return t


def _blocks(case, n, dtype, opname):
    """Every rank's input of ``case``: P blocks of ``n`` elements."""
    return [_input(case, q, size * n, dtype, opname).reshape(size, n) for q in range(size)]


def _run(device, capsys, chk, how, xs, opname, mine=None):
    """reduce_scatter of this rank's ``xs[rank]`` (``mine``: the view of it that is passed, on the device),
    against the rank-order fold of block p on every rank p; ``how`` names the transport setting."""
    dtype, shape = xs[0].dtype, tuple(xs[0].shape[1:])
    nbytes = xs[0][0].numel() * dtype.itemsize
    label = f"reduce_scatter {how} {dtype} {opname} block {shape} ({nbytes} B) P={size}"
    x = xs[rank].to(device) if mine is None else mine
    x0 = x.clone()
    res, via = _logged(capsys, device, "Reduce_scatter_block",
                       lambda: m.reduce_scatter(x, getattr(MPI, opname), comm=comm))
    if via is not None:
        want_via = _rs_transport(comm._native_comm(), nbytes)
        chk(_expect, via == want_via, f"{label}: took the {via} transport, expected {want_via}")
    flat = [xq.reshape(size, xs[0][0].numel()) for xq in xs]
    wants = [_fold([f[p] for f in flat], opname).reshape(shape) for p in range(size)]
    chk(_assert_same, res, wants[rank], label)
    if dtype.is_floating_point or dtype.is_complex:
        chk(_check_accuracy, res.cpu().reshape(-1), [f[rank] for f in flat], opname, label)
    chk(_assert_same, x, x0, f"{label}: input changed")
    chk.add(label, _canon(res), [_canon(w) for w in wants])


@peers
def test_reduce_scatter_every_dtype_op_and_transport(device, capsys):
    """Every dtype x op (bool with all ten) through LL and pull, at blocks of 1, 17 and 4095 bytes (odd block
    lengths: blocks q >= 1 start at unaligned addresses, tails); full-bit integers, so sums and products wrap."""
    chk = Checks()
    for how, ll_max in _settings(device):
        with _ll_max(device, ll_max):
            for dtype in ALL_DTYPES:
                for opname in _ops_for(dtype) if dtype != torch.bool else OPS:
                    for nbytes in (1, 17, 4095):
                        n = _n_for(nbytes, dtype)
                        xs = _blocks(("matrix", how, str(dtype), opname, n), n, dtype, opname)
                        _run(device, capsys, chk, how, xs, opname)
    chk.finish()


@peers
def test_reduce_scatter_block_lengths_around_vector_and_ll_limits(device, capsys):
    """Blocks of 15, 16, 17, 4095 and 4096 + 16 bytes, the LL limit - 16, at and + 16 bytes, and 8 x the LL
    limit + 48, with element sizes 1, 2, 4, 8 and 16, under the size table's choice and under each transport
    where it is legal.  Odd lengths put blocks q >= 1 at unaligned addresses in both kernels: the LL kernel
    loads them byte by byte, the pull kernel stages them to a 16-byte stride."""
    chk = Checks()
    cases = ((torch.uint8, "SUM"), (torch.bfloat16, "SUM"), (torch.float32, "SUM"), (torch.int32, "BXOR"),
             (torch.float64, "PROD"), (torch.uint64, "MAX"), (torch.complex128, "SUM"))
    lengths = (15, 16, 17, 4095, 4096 + 16, LL_LIMIT - 16, LL_LIMIT, LL_LIMIT + 16, 8 * LL_LIMIT + 48)
    for how, ll_max in _settings(device, auto=True):
        with _ll_max(device, ll_max):
            for dtype, opname in cases:
                for nbytes in lengths:
                    if (how == "ll" and nbytes > LL_LIMIT) or (device.type != "cuda" and nbytes > CPU_MAX):
                        continue
                    n = _n_for(nbytes, dtype)
                    xs = _blocks(("lengths", how, str(dtype), opname, n), n, dtype, opname)
                    _run(device, capsys, chk, how, xs, opname)
    chk.finish()


@peers
def test_reduce_scatter_edge_values(device, capsys):
    """NaN in one rank, +-inf and +-0.0, fp32 subnormals, INT_MIN / INT_MAX, uint64 >= 2^63, wrapping sums
    and products, through both transports.  Rank q's block p is the case's vector of rank q rolled by p,
    so every rank's result differs."""
    chk = Checks()
    for how, ll_max in _settings(device):
        with _ll_max(device, ll_max):
            for name, dtype, opname, vecs in _edge_cases():
                xs = [torch.stack([v.roll(p) for p in range(size)]) for v in vecs]
                _run(device, capsys, chk, f"{how} {name}", xs, opname)
    chk.finish()


@peers
def test_reduce_scatter_multichunk_pull(device, capsys):
    """The pull kernel with max_blocks 1 and 2 and blocks of 2-3 MiB: chunks are capped at 512 KiB, so every
    CTA stages and pulls several chunks of the block, one barrier epoch each; and a 4 MiB block on the full
    grid.  The uint8 blocks have an odd length (unaligned staging sources, a 1-byte tail)."""
    if device.type != "cuda":
        pytest.skip("multi-MiB blocks and the grid cap: GPU only")
    chk = Checks()
    for blocks, nbytes in ((1, (2 << 20) + 16), (2, (3 << 20) + 4), (None, 4 << 20)):
        opts = dict(ll_max=0) if blocks is None else dict(ll_max=0, max_blocks=blocks)
        with _options(device, **opts):
            for dtype, opname in ((torch.float32, "SUM"), (torch.bfloat16, "SUM"), (torch.int16, "MAX"),
                                  (torch.uint8, "SUM")):
                n = _n_for(nbytes + (dtype == torch.uint8), dtype)
                xs = _blocks(("chunks", blocks, str(dtype), n), n, dtype, opname)
                _run(device, capsys, chk, f"pull max_blocks={blocks}", xs, opname)
    chk.finish()


@peers
def test_reduce_scatter_shapes(device, capsys):
    """x of shape (P,) (a 0-dim result), non-contiguous inputs (a transpose; a slice whose start is not
    16-byte aligned), and an empty block (P, 0, 4), which launches nothing: the LL call after it shows that
    every rank's LL ticket stayed in step."""
    chk = Checks()
    for how, ll_max in _settings(device):
        with _ll_max(device, ll_max):
            for dtype, opname in ((torch.float64, "SUM"), (torch.int8, "PROD"), (torch.bool, "LXOR")):
                xs = [_input(("scalar", how, str(dtype), opname), q, size, dtype, opname) for q in range(size)]
                _run(device, capsys, chk, f"{how} x of shape (P,)", xs, opname)
            for dtype in (torch.float32, torch.uint8):
                bases = [_input(("transpose", how, str(dtype)), q, 45 * size, dtype).reshape(45, size)
                         for q in range(size)]
                _run(device, capsys, chk, f"{how} transposed", [b.t() for b in bases], "SUM",
                     mine=bases[rank].to(device).t())
                bases = _blocks(("offset", how, str(dtype)), 38, dtype, "MAX")
                _run(device, capsys, chk, f"{how} offset slice", [b[:, 1:] for b in bases], "MAX",
                     mine=bases[rank].to(device)[:, 1:])
    with _ll_max(device, 1 << 30 if device.type == "cuda" else None):
        empty = [torch.empty((size, 0, 4)) for _ in range(size)]
        _run(device, capsys, chk, "empty block", empty, "SUM")
        _run(device, capsys, chk, "LL after an empty block", _blocks("after empty", 33, torch.float32, "SUM"), "SUM")
    chk.finish()


# ---------------------------------------------------------------------------
# reduce_scatter between the other collectives: the LL buffers and ticket, the staging parity and the
# per-CTA epochs are shared with allreduce, allgather and reduce_scatterv
# ---------------------------------------------------------------------------
ROWS = 7
# (kind, elements per block / rank, dtype, op); block sizes pick the transport, so a captured graph keeps both
MIXED = (("rs", 33, torch.float32, "SUM"), ("ar", 1000, torch.float32, "SUM"), ("rs", 20000, torch.float32, "MAX"),
         ("ar", 5000, torch.float32, "SUM"), ("rs", 1000, torch.int32, "BXOR"), ("rsv", ROWS * 3, torch.float32, "SUM"),
         ("ag", 77, torch.float64, None), ("rs", 77, torch.float64, "PROD"))


def _rs_sequence(a, b, c, d, e, f, g, h, counts):
    return (m.reduce_scatter(a, MPI.SUM, comm=comm),                           # LL
            m.allreduce(b, MPI.SUM, comm=comm, algorithm="ll"),
            m.reduce_scatter(c, MPI.MAX, comm=comm),                           # pull: 80000 B > the LL limit
            m.allreduce(d, MPI.SUM, comm=comm, algorithm="twoshot"),
            m.reduce_scatter(e, MPI.BXOR, comm=comm),                          # LL
            m.reduce_scatterv(f, counts, MPI.SUM, recv_capacity=ROWS, comm=comm)[0],
            m.allgather(g, comm=comm),
            m.reduce_scatter(h, MPI.PROD, comm=comm))                          # LL


def _mixed_inputs(call):
    out = []
    for k, (kind, n, dtype, opname) in enumerate(MIXED):
        xs = [_input(("rs mixed", call, k), q, n * (size if kind in ("rs", "rsv") else 1), dtype, opname or "SUM")
              for q in range(size)]
        out.append([x.reshape(size, n) if kind == "rs" else x.reshape(size * ROWS, 3) if kind == "rsv" else x
                    for x in xs])
    return out


def _mixed_wants(ins, p):
    """What rank p holds after the sequence."""
    wants = []
    for (kind, _, _, opname), xs in zip(MIXED, ins):
        if kind == "rs":
            wants.append(_fold([x[p] for x in xs], opname))
        elif kind == "rsv":
            wants.append(_fold([x.reshape(size, ROWS * 3)[p] for x in xs], opname).reshape(ROWS, 3))
        elif kind == "ar":
            wants.append(_fold(xs, opname))
        else:
            wants.append(torch.stack(xs))
    return wants


@peers
def test_reduce_scatter_mixed_sequences_eager_and_jit(device, capsys):
    """reduce_scatter LL -> allreduce LL -> reduce_scatter pull -> allreduce two-shot -> reduce_scatter LL
    (int32 BXOR) -> reduce_scatterv -> allgather -> reduce_scatter LL (f64 PROD), eagerly (where the debug log
    shows each reduce_scatter's transport) and as a captured CUDA graph replayed with new inputs."""
    chk = Checks()
    f = m.jit(_rs_sequence)
    counts = torch.full((size,), ROWS, dtype=torch.int64, device=device)
    rs_bytes = [n * dt.itemsize for kind, n, dt, _ in MIXED if kind == "rs"]
    for call in range(5):
        ins = _mixed_inputs(call)
        wants = [_mixed_wants(ins, p) for p in range(size)]
        args = [x[rank].to(device) for x in ins]
        for mode, fn in (("eager", _rs_sequence), ("jit", f)):
            logged = device.type == "cuda" and mode == "eager"
            if logged:
                capsys.readouterr()
                set_logging(True)
            try:
                got = fn(*args, counts)
            finally:
                set_logging(False)
            if logged:
                vias = re.findall(rf"^r{rank} \| \w{{8}} \| MPI_Reduce_scatter_block \(GPU\) with .* via (\w+)$",
                                  capsys.readouterr().out, re.M)
                want_vias = [_rs_transport(comm._native_comm(), b) for b in rs_bytes]
                chk(_expect, vias == want_vias, f"mixed sequence call {call}: transports {vias}, expected {want_vias}")
            for k, ((kind, _, _, opname), g) in enumerate(zip(MIXED, got)):
                label = f"mixed sequence call {call} {mode}: {kind} {opname} P={size}"
                chk(_assert_same, g, wants[rank][k], label)
                chk.add(label, _canon(g), [_canon(w[k]) for w in wants])
    chk.finish()


# ---------------------------------------------------------------------------
# the LL kernel past one wave of threads: its grid-stride loop runs once a payload has more vectors than
# sm_count x 512 (1.06 MiB on a 132-SM H100), which needs an LL buffer of more than the default 128 KiB
# ---------------------------------------------------------------------------
GRID_BYTES = (3 << 19) + 16         # 1.5 MiB + 16 B
big_ll = pytest.mark.skipif(size < 2 or LL_LIMIT < GRID_BYTES,
                            reason="needs a multi-rank job whose LL buffer (MPI4JAX_B200_LL_BYTES) is >= 3 MiB")


@big_ll
def test_ll_grid_stride(device, capsys):
    """reduce_scatter (ll_max high) and allreduce(algorithm="ll") at 1.5 MiB + 16 B and at half the LL buffer:
    a full grid in which every thread handles more than one vector.  The int8 payloads have an odd length,
    so the reduce_scatter loads all of them through the byte loop."""
    if device.type != "cuda":
        pytest.skip("the LL kernel runs on the GPU")
    chk = Checks()
    sms = comm._native_comm().get_option("sm_count")
    with _options(device, ll_max=1 << 30):
        for nbytes in (GRID_BYTES, LL_LIMIT):
            chk(_expect, nbytes > sms * 512 * 16, f"{nbytes} B fit in one wave of {sms} x 512 threads")
            for dtype, opname in ((torch.float32, "SUM"), (torch.bfloat16, "SUM"), (torch.int8, "MAX"),
                                  (torch.complex128, "PROD")):
                n = _n_for(nbytes - (dtype == torch.int8), dtype)
                xs = _blocks(("grid", str(dtype), n), n, dtype, opname)
                _run(device, capsys, chk, "ll grid stride", xs, opname)
                _run_allreduce(device, capsys, chk, ("grid allreduce", str(dtype), n), dtype, opname, n, "ll")
    chk.finish()


# ---------------------------------------------------------------------------
# the same tests with three and five ranks, and with a large LL buffer
# ---------------------------------------------------------------------------
_inside_job = size > 1 or "MPI4JAX_B200_NESTED" in os.environ
PEER_TESTS = ["test_reduce_scatter_every_dtype_op_and_transport",
              "test_reduce_scatter_block_lengths_around_vector_and_ll_limits", "test_reduce_scatter_edge_values",
              "test_reduce_scatter_multichunk_pull", "test_reduce_scatter_shapes",
              "test_reduce_scatter_mixed_sequences_eager_and_jit"]


@pytest.mark.gpu
@pytest.mark.skipif(_inside_job, reason="already inside a multi-rank job")
def test_reduce_scatter_kernels_three_ranks_gpu():
    """P = 3: a non-power-of-two world, chunk unit 48 B."""
    code, outs = job(__file__, 3, "not grid_stride")
    expect_passed(code, outs, 3, PEER_TESTS)


@pytest.mark.gpu
@pytest.mark.skipif(_inside_job, reason="already inside a multi-rank job")
def test_reduce_scatter_kernels_five_ranks_gpu():
    """P = 5: the LL kernel pushes to four peers, the pull kernel stages five blocks.  Smaller p2p ring
    slots keep five contexts' rings small."""
    tests = ["test_reduce_scatter_block_lengths_around_vector_and_ll_limits", "test_reduce_scatter_multichunk_pull"]
    code, outs = job(__file__, 5, " or ".join(tests), {"MPI4JAX_B200_P2P_SLOT_BYTES": "1048576"})
    expect_passed(code, outs, 5, tests)


@pytest.mark.gpu
@pytest.mark.skipif(_inside_job, reason="already inside a multi-rank job")
@pytest.mark.parametrize("nranks", [2, 3])
def test_ll_grid_stride_with_8_mib_ll_buffer_gpu(nranks):
    code, outs = job(__file__, nranks, "test_ll_grid_stride", {"MPI4JAX_B200_LL_BYTES": str(8 << 20)})
    expect_passed(code, outs, nranks, ["test_ll_grid_stride"])
