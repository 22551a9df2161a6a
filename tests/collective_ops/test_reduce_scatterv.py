"""reduce_scatterv: rank r receives ``op`` over the ranks' segments for r, folded row by row in rank order,
``(M_r, *S) -> (recv_capacity, *S)``.

Oracle: every rank gathers all inputs and counts with the object API, clamps the counts in rank order
to each rank's rows, and folds each output row over the ranks whose segment reaches it -- in rank order,
in the accumulate type (fp32 for f16/bf16, int64 wrapped back for integers), rounded once -- in plain
torch on the CPU.  Results compare bitwise; NaNs compare by position.  The CUDA variants need peers: in
a single-process run they are checked in a two-rank job whose ranks share the GPU, and
``test_reduce_scatterv_three_ranks_gpu`` runs them with three ranks."""

import contextlib
import os
import re
import tempfile

import pytest
import torch
from torch.func import jvp, vjp, vmap

import mpi4jax_b200 as m
from mpi4jax_b200 import MPI
from mpi4jax_b200._src.native import codes

from .._peer_job import needs_peers

comm = MPI.COMM_WORLD
rank = comm.Get_rank()
size = comm.Get_size()

peers = needs_peers("reduce_scatterv between ranks")

def _clamp(counts, rows):
    out, used = [], 0
    for c in counts:
        k = min(max(int(c), 0), rows - used)
        out.append(k)
        used += k
    return out


def _gathered(x, counts):
    """(inputs, counts clamped in rank order to each rank's rows) of every rank, in rank order."""
    cl = counts.tolist() if isinstance(counts, torch.Tensor) else list(counts)
    raw = x.detach().cpu().contiguous().reshape(-1).view(torch.uint8)      # every dtype pickles as bytes
    everything = comm.allgather((raw, tuple(x.shape), _clamp(cl, x.shape[0])))
    return [e[0].view(x.dtype).reshape(e[1]) for e in everything], [e[2] for e in everything]


def _fold(parts, opname):
    """Rank-order fold of equally shaped CPU tensors, in the accumulate type, rounded once."""
    dt = parts[0].dtype
    if len(parts) == 1:
        return parts[0].clone()
    if dt == torch.bool:
        v = [p.to(torch.int64) for p in parts]
    elif dt in (torch.float16, torch.bfloat16):
        v = [p.float() for p in parts]
    elif dt.is_floating_point or dt.is_complex:
        v = list(parts)
    else:
        v = [p.to(torch.int64) for p in parts]
    acc = v[0].clone()
    for b in v[1:]:
        if opname == "SUM":
            acc = acc + b
        elif opname == "PROD":
            acc = acc * b
        elif opname == "MIN":
            acc = torch.where((b < acc) | (b != b), b, acc)
        elif opname == "MAX":
            acc = torch.where((b > acc) | (b != b), b, acc)
        elif opname == "LAND":
            acc = ((acc != 0) & (b != 0)).to(acc.dtype)
        elif opname == "LOR":
            acc = ((acc != 0) | (b != 0)).to(acc.dtype)
        elif opname == "LXOR":
            acc = ((acc != 0) ^ (b != 0)).to(acc.dtype)
        elif opname == "BAND":
            acc = acc & b
        elif opname == "BOR":
            acc = acc | b
        else:
            acc = acc ^ b
    if dt == torch.bool:
        return acc != 0
    return acc.to(dt)


def _oracle(x, counts, opname, cap):
    xs, cs = _gathered(x, counts)
    recv = [min(cs[q][rank], cap) for q in range(size)]
    displ = [sum(cs[q][:rank]) for q in range(size)]
    out = torch.zeros((cap, *x.shape[1:]), dtype=x.dtype)
    for i in range(max(recv, default=0)):
        out[i] = _fold([xs[q][displ[q] + i] for q in range(size) if i < recv[q]], opname)
    return out, torch.tensor(recv, dtype=torch.int64)


def _same(a, b):
    """Bitwise equality; NaNs compare by position."""
    a, b = a.cpu(), b.cpu()
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    if a.dtype.is_complex:
        a, b = torch.view_as_real(a), torch.view_as_real(b)
    if a.dtype.is_floating_point:
        na, nb = torch.isnan(a), torch.isnan(b)
        if not torch.equal(na, nb):
            return False
        a, b = a.masked_fill(na, 0), b.masked_fill(nb, 0)
    return torch.equal(a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8))


def _check(x, counts, opname="SUM", cap=None):
    _x = x.clone()
    out, rc = m.reduce_scatterv(x, counts, getattr(MPI, opname), recv_capacity=cap, comm=comm)
    cap = x.shape[0] if cap is None else cap
    want, want_rc = _oracle(x, counts, opname, cap)
    assert out.shape == (cap, *x.shape[1:]) and out.dtype == x.dtype and out.device == x.device
    assert rc.dtype == torch.int64 and rc.shape == (size,) and rc.device == x.device
    assert torch.equal(rc.cpu(), want_rc), (counts, cap)
    assert _same(out, want), (opname, counts, cap)
    assert _same(x, _x)
    return out, rc


def _count_cases(n):
    """(rows of x on this rank, send counts, capacity); the counts and the rows differ between ranks, the
    capacity never does."""
    even = [n // size] * size
    even[-1] += n - sum(even)
    return [
        (n, even, None),                                            # MPI_Reduce_scatter: counts sum to M
        (n, [(q + rank) % 4 for q in range(size)], None),           # different per rank
        (n, [0] * size, None),                                      # nothing at all
        (n, [-2 + q + rank for q in range(size)], None),            # negative counts
        (n, [n + 3] * size, None),                                  # past M: the first rank takes all
        (n, [n] * size, 2),                                         # N below a segment: clipped
        (n + 2 * rank, [3 + rank] * size, n + 4),                   # M differs per rank
        (n, even, 0),                                               # capacity 0
        (n, [n - 1 - q for q in range(size)], 2 * n),               # capacity past every segment
    ]


@peers
def test_reduce_scatterv_cases(device):
    n = 7
    for rows, counts, cap in _count_cases(n):
        x = (torch.arange(rows * 3, dtype=torch.float32).reshape(rows, 3) + 100 * rank).to(device)
        _check(x, torch.tensor(counts, device=device), "SUM", cap)
        _check(x, torch.tensor(counts, device=device), "MAX", cap)
    x = (torch.arange(n * 3, dtype=torch.float32).reshape(n, 3) + rank).to(device)
    # a sequence of ints and an int32 tensor are accepted too
    out, _ = _check(x, [1 + q for q in range(size)])
    assert torch.equal(out, _check(x, torch.tensor([1 + q for q in range(size)], dtype=torch.int32,
                                                   device=device))[0])
    # M = 0 on every rank
    e = torch.empty((0, 3), device=device)
    out, rc = _check(e, torch.ones(size, dtype=torch.int64, device=device), "SUM", 4)
    assert not out.any() and rc.tolist() == [0] * size


@peers
def test_reduce_scatterv_is_reduce_scatter(device):
    """M = P * B with every count B: bit for bit the reduce_scatter of x.view(P, B, ...), over every dtype x
    op that reduce_scatter supports."""
    B = 3
    counts = torch.full((size,), B, dtype=torch.int64, device=device)
    for k, dtype in enumerate(codes.DTYPE_CODE):
        g = torch.Generator().manual_seed(31 * k + rank)
        v = torch.randint(-40, 40, (size * B, 5), generator=g)
        x = ((v % 2) == 0) if dtype == torch.bool else (v.abs() if not dtype.is_signed else v).to(dtype)
        if dtype.is_floating_point or dtype.is_complex:
            x = (torch.randn(size * B, 5, generator=g) * 4).to(dtype)
        x = x.to(device)
        for opname in ("SUM", "PROD", "MIN", "MAX", "LAND", "LOR", "LXOR", "BAND", "BOR", "BXOR"):
            op = getattr(MPI, opname)
            try:
                want = m.reduce_scatter(x.view(size, B, 5), op, comm=comm)
            except NotImplementedError as exc:
                with pytest.raises(NotImplementedError, match=re.escape(str(exc))):
                    m.reduce_scatterv(x, counts, op, comm=comm)
                continue
            out, rc = m.reduce_scatterv(x, counts, op, recv_capacity=B, comm=comm)
            assert _same(out, want), (dtype, opname)
            assert rc.tolist() == [B] * size


@peers
def test_reduce_scatterv_odd_rows_and_layouts(device):
    """Row sizes that are not multiples of 16 bytes (segments end inside a 16-byte vector), complex128,
    and non-contiguous inputs."""
    torch.manual_seed(5 + rank)
    for dtype, row in ((torch.int8, (3,)), (torch.uint8, (5, 1)), (torch.float32, (3,)), (torch.float16, (7,)),
                       (torch.complex128, (1,)), (torch.bfloat16, (1,))):
        x = (torch.randn(11, *row) * 50).to(dtype).to(device)
        for _, counts, cap in _count_cases(11):         # (x keeps 11 rows: the counts are clamped to them)
            _check(x, torch.tensor(counts, device=device), "SUM", cap)
            if not dtype.is_complex:
                _check(x, torch.tensor(counts, device=device), "MIN", cap)
    base = torch.randn(4, 9, device=device)
    xt = base.t()                                                       # (9, 4), not contiguous
    assert not xt.is_contiguous()
    _check(xt, torch.tensor([2 + (q + rank) % 3 for q in range(size)], device=device), "SUM", 5)
    _check(torch.randn(12, 6, device=device)[::2, 1:4], torch.tensor([2] * size, device=device), "PROD", 4)


@contextlib.contextmanager
def _max_blocks(device, n):
    """The collective grid cap set to ``n`` CTAs for the block (CUDA), restored afterwards."""
    if device.type != "cuda":
        yield
        return
    nc = comm._native_comm()
    old = nc.get_option("max_blocks")
    nc.set_option("max_blocks", n)
    try:
        yield
    finally:
        m.flush()
        nc.set_option("max_blocks", old)


@peers
def test_reduce_scatterv_multi_chunk(device):
    """Blocks of 2 MiB: with the full grid every CTA folds one chunk; with one or two CTAs (max_blocks) each
    CTA walks several 512 KiB chunks, staging the next one between its arrive and its wait.  Segments end
    inside chunks, the loop bound comes from another rank's segment, and 2046-byte rows end inside vectors."""
    n = 1024
    gen = torch.Generator(device).manual_seed(rank)
    x = torch.randn(size * n, 512, device=device, generator=gen)                     # 2 MiB per block
    xo = torch.randn(size * n, 1023, device=device, generator=gen).to(torch.bfloat16)   # 2046-byte rows
    for blocks in (0, 1, 2):
        with _max_blocks(device, blocks) if blocks else contextlib.nullcontext():
            _check(x, torch.tensor([n] * size, device=device), "SUM", n)
            _check(x, torch.tensor([n - 37 * ((q + rank) % 3) - 1 for q in range(size)], device=device), "SUM", n)
            _check(x, torch.tensor([n * (q + 1) // size + rank for q in range(size)], device=device), "MAX", n - 100)
            _check(x, torch.tensor([300 * (rank == q) + 5 for q in range(size)], device=device), "SUM", n)
            _check(xo, torch.tensor([n - 1 - rank - q for q in range(size)], device=device), "SUM", n)


@peers
def test_reduce_scatterv_values(device):
    """NaN in one rank's row, +-inf, and fp16 / bf16 sums that differ between fp32 and native accumulation."""
    n = 6
    counts = torch.tensor([n - q for q in range(size)], device=device)
    x = torch.ones(size * n, 4)
    if rank == size - 1:
        x[0, 0] = float("nan")
    x[1, 1] = float("inf") if rank == 0 else 1.0
    x[2, 2] = float("-inf") if rank == 0 else float("inf") if rank == 1 else 0.0
    for opname in ("SUM", "PROD", "MIN", "MAX"):
        _check(x.to(device), counts, opname, n)
    # 2048 + 1 + 1 in fp16 is 2048 when rounded per step, 2050 in fp32 rounded once
    for dtype in (torch.float16, torch.bfloat16):
        big = 2048.0 if dtype == torch.float16 else 256.0
        y = torch.full((size * n, 8), big if rank == 0 else 1.0, dtype=dtype)
        out, _ = _check(y.to(device), counts, "SUM", n)
        if size >= 3:
            assert out[0, 0].item() == big + size - 1


def test_reduce_scatterv_single_rank(device):
    """A one-rank communicator: the rows of the one segment (clipped to N), then zeros."""
    solo = comm.Split(rank, 0)
    try:
        x = torch.randn(5, 3, device=device)
        out, rc = m.reduce_scatterv(x, torch.tensor([3], device=device), MPI.SUM, comm=solo)
        assert out.shape == (5, 3) and rc.tolist() == [3]
        assert torch.equal(out[:3], x[:3]) and not out[3:].any()
        out, rc = m.reduce_scatterv(x, [9], MPI.PROD, recv_capacity=2, comm=solo)
        assert torch.equal(out, x[:2]) and rc.tolist() == [2]
    finally:
        m.flush()
        solo.Free()


def test_reduce_scatterv_errors(device):
    x = torch.ones((4, 2), device=device)
    good = torch.ones(size, dtype=torch.int64, device=device)
    other = "meta" if device.type == "cpu" else "cpu"
    with pytest.raises(ValueError, match=re.escape("Reduce_scatterv input must have shape (rows, ...)")):
        m.reduce_scatterv(torch.tensor(1.0, device=device), good, MPI.SUM, comm=comm)
    with pytest.raises(ValueError, match=re.escape("Reduce_scatterv send_counts must have shape (nproc,)")):
        m.reduce_scatterv(x, torch.ones(size + 1, dtype=torch.int64, device=device), MPI.SUM, comm=comm)
    with pytest.raises(ValueError, match=re.escape("Reduce_scatterv send_counts must have shape (nproc,)")):
        m.reduce_scatterv(x, torch.tensor(1, device=device), MPI.SUM, comm=comm)
    with pytest.raises(TypeError, match="Reduce_scatterv send_counts must be an integer tensor"):
        m.reduce_scatterv(x, good.float(), MPI.SUM, comm=comm)
    with pytest.raises(TypeError, match="Reduce_scatterv send_counts must be an integer tensor"):
        m.reduce_scatterv(x, good.bool(), MPI.SUM, comm=comm)
    with pytest.raises(TypeError):
        m.reduce_scatterv(x, [1.5] * size, MPI.SUM, comm=comm)
    with pytest.raises(ValueError, match="Reduce_scatterv send_counts must live on the device of x"):
        m.reduce_scatterv(x, good.to(other), MPI.SUM, comm=comm)
    with pytest.raises(ValueError, match=re.escape("Reduce_scatterv recv_capacity must be >= 0")):
        m.reduce_scatterv(x, good, MPI.SUM, recv_capacity=-1, comm=comm)
    with pytest.raises(TypeError, match='unexpected type for argument "recv_capacity"'):
        m.reduce_scatterv(x, good, MPI.SUM, recv_capacity=2.0, comm=comm)
    with pytest.raises(RuntimeError, match="Explicit token management"):
        m.reduce_scatterv(x, good, MPI.SUM, comm=comm, token=1)
    # a pair the kernels do not define is refused on every call, even when no row has two contributors
    zero = torch.zeros(size, dtype=torch.int64, device=device)
    with pytest.raises(NotImplementedError, match="logical/bitwise reductions need an integer or bool dtype"):
        m.reduce_scatterv(x, zero, MPI.BAND, comm=comm)
    with pytest.raises(NotImplementedError, match="only SUM and PROD are defined for complex dtypes"):
        m.reduce_scatterv(x.to(torch.complex64), zero, MPI.MIN, comm=comm)
    xr = x.clone().requires_grad_(True)
    with pytest.raises(NotImplementedError, match="reduce_scatterv for MAX is not defined"):
        m.reduce_scatterv(xr, good, MPI.MAX, comm=comm)[0].sum().backward()


def test_reduce_scatterv_compiled_errors(device):
    """compiled.reduce_scatterv, the raw torch.ops op and its fake kernel refuse what the eager op refuses."""
    from torch._subclasses.fake_tensor import FakeTensorMode

    x = torch.ones((4, 2), device=device)
    other = "meta" if device.type == "cpu" else "cpu"
    good = torch.ones(size, dtype=torch.int64, device=device)
    bad = [
        (ValueError, "must live on the device of x", x, good.to(other), None),
        (ValueError, re.escape("must have shape (nproc,)"), x, torch.ones(size + 1, dtype=torch.int64,
                                                                           device=device), None),
        (TypeError, "must be an integer tensor", x, good.float(), None),
        (ValueError, re.escape("recv_capacity must be >= 0"), x, good, -1),
        (ValueError, re.escape("input must have shape (rows, ...)"), torch.tensor(1.0, device=device), good, None),
    ]
    for exc, msg, xx, counts, cap in bad:
        with pytest.raises(exc, match=msg):
            m.compiled.reduce_scatterv(xx, counts, MPI.SUM, recv_capacity=cap, comm=comm)
        with pytest.raises(exc, match=msg):
            torch.ops.mpi4jax_b200.reduce_scatterv(xx, counts, 4 if cap is None else cap, MPI.SUM.code, comm._id)
    with FakeTensorMode():
        with pytest.raises(ValueError, match=re.escape("must have shape (nproc,)")):
            m.compiled.reduce_scatterv(torch.empty(4, 2), torch.empty((), dtype=torch.int64), MPI.SUM, comm=comm)
        with pytest.raises(ValueError, match=re.escape("must have shape (nproc,)")):
            torch.ops.mpi4jax_b200.reduce_scatterv(torch.empty(4, 2), torch.empty((), dtype=torch.int64), 4,
                                                   MPI.SUM.code, comm._id)


def test_reduce_scatterv_fake_shape_and_effect():
    from torch._higher_order_ops.effects import _EffectType, _get_effect
    from torch._subclasses.fake_tensor import FakeTensorMode

    with FakeTensorMode():
        out, rc = m.compiled.reduce_scatterv(torch.empty(4, 3, 2), torch.empty(size, dtype=torch.int64), MPI.SUM,
                                             recv_capacity=7, comm=comm)
        assert out.shape == (7, 3, 2) and rc.shape == (size,) and rc.dtype == torch.int64
        out, _ = m.compiled.reduce_scatterv(torch.empty(4, 3), torch.empty(size, dtype=torch.int64), MPI.SUM,
                                            comm=comm)
        assert out.shape == (4, 3)
    assert _get_effect("mpi4jax_b200::reduce_scatterv") == _EffectType.ORDERED


@peers
def test_reduce_scatterv_jit_and_graph_replays(device):
    """Captured once, replayed with the counts changed in place: oracle-exact every time."""
    if device.type != "cuda":
        pytest.skip("CUDA graphs")
    n, cap = 9, 6
    x = torch.randn(n, 5, device=device, generator=torch.Generator(device).manual_seed(rank))
    counts = torch.zeros(size, dtype=torch.int64, device=device)
    f = m.jit(lambda t, c: m.reduce_scatterv(t * 2, c, MPI.SUM, recv_capacity=cap, comm=comm))
    cases = [c for _, c, _ in _count_cases(n)]
    for c in cases:                                     # eager warm-up, capture, replays
        counts.copy_(torch.tensor(c))
        out, rc = f(x, counts)
        want, want_rc = _oracle(x * 2, counts, "SUM", cap)
        assert _same(out, want) and torch.equal(rc.cpu(), want_rc), c
    m.flush()


def _grad_oracle(ct, counts, rows, cap):
    """Cotangent of x: rows [D(p), D(p) + min(s[p], N)) get rank p's first cotangent rows, others zero."""
    cts, _ = _gathered(ct, torch.zeros(size, dtype=torch.int64))
    cl = _clamp(counts.tolist(), rows)
    g = torch.zeros((rows, *ct.shape[1:]), dtype=ct.dtype)
    d = 0
    for p in range(size):
        k = min(cl[p], cap)
        g[d: d + k] = cts[p][:k]
        d += cl[p]
    return g


@peers
def test_reduce_scatterv_derivatives(device):
    """vjp / backward: the reverse-mode allgatherv of the cotangent (bitwise).  jvp: reduce_scatterv of the
    tangent.  Double backward: the adjoint of the adjoint is the op again."""
    n = 6
    gen = torch.Generator().manual_seed(7 + rank)
    for rows, counts, cap in ((n, [2 + (q + rank) % 3 for q in range(size)], 4),
                              (n + rank, [n] * size, 3), (n, [-1 + q for q in range(size)], n + 1)):
        counts = torch.tensor(counts, device=device)
        x = torch.randn(rows, 2, generator=gen).to(device)
        ct = torch.randn(cap, 2, generator=gen).to(device)
        t = torch.randn(rows, 2, generator=gen).to(device)

        def f(v):
            return m.reduce_scatterv(v, counts, MPI.SUM, recv_capacity=cap, comm=comm)[0]

        res, pullback = vjp(f, x)
        assert _same(res, _oracle(x, counts, "SUM", cap)[0])
        (g,) = pullback(ct)
        want = _grad_oracle(ct, counts, rows, cap)
        assert torch.equal(g.cpu(), want), (counts, cap)
        _, tan = jvp(f, (x,), (t,))
        assert _same(tan, _oracle(t, counts, "SUM", cap)[0])
        xr = x.clone().requires_grad_(True)
        ctr = ct.clone().requires_grad_(True)
        out, rc = m.reduce_scatterv(xr, counts, MPI.SUM, recv_capacity=cap, comm=comm)
        assert not rc.requires_grad
        (gx,) = torch.autograd.grad((out * ctr).sum(), xr, create_graph=True)
        assert torch.equal(gx.detach().cpu(), want)
        (gct,) = torch.autograd.grad((gx * t).sum(), ctr)
        assert _same(gct, _oracle(t, counts, "SUM", cap)[0]), (counts, cap)
        xr.grad = None
        (m.reduce_scatterv(xr, counts, MPI.SUM, recv_capacity=cap, comm=comm)[0] * ct).sum().backward()
        assert torch.equal(xr.grad.cpu(), want)


@peers
def test_reduce_scatterv_vmap(device):
    n = 5
    counts = torch.tensor([1 + (q + rank) % 3 for q in range(size)], device=device)
    xb = (torch.arange(3 * n * 2, dtype=torch.float32).reshape(3, n, 2) + 100 * rank).to(device)
    want = torch.stack([m.reduce_scatterv(xb[i], counts, MPI.SUM, recv_capacity=4, comm=comm)[0] for i in range(3)])
    f = vmap(lambda v: m.reduce_scatterv(v, counts, MPI.SUM, recv_capacity=4, comm=comm)[0], in_dims=0, out_dims=0)
    assert torch.equal(f(xb), want)
    f1 = vmap(lambda v: m.reduce_scatterv(v, counts, MPI.SUM, recv_capacity=4, comm=comm)[0], in_dims=1,
              out_dims=0)
    assert torch.equal(f1(xb.movedim(0, 1).contiguous()), want)
    with pytest.raises(ValueError, match="counts must not be batched"):
        vmap(lambda v, c: m.reduce_scatterv(v, c, MPI.SUM, comm=comm)[0])(xb, counts.expand(3, size).contiguous())


@peers
def test_reduce_scatterv_compiled_and_grad(device):
    """torch.compile(fullgraph=True) of compiled.reduce_scatterv and its gradient; the eager and the compiled
    adjoints are equal."""
    n, cap = 6 + rank, 4
    counts = torch.tensor([1 + (q + rank) % 4 for q in range(size)], device=device)
    ct = torch.randn(cap, 2, generator=torch.Generator().manual_seed(rank)).to(device)
    f = torch.compile(lambda v, c: m.compiled.reduce_scatterv(v * 2, c, MPI.SUM, recv_capacity=cap, comm=comm)[0],
                      backend="aot_eager", fullgraph=True)
    x = (torch.arange(n * 2, dtype=torch.float32).reshape(n, 2) + rank).to(device).requires_grad_(True)
    out = f(x, counts)
    assert _same(out.detach(), _oracle(x.detach() * 2, counts, "SUM", cap)[0])
    (out * ct).sum().backward()
    assert torch.equal(x.grad.cpu(), 2 * _grad_oracle(ct, counts, n, cap))
    xe = x.detach().clone().requires_grad_(True)
    (m.reduce_scatterv(xe * 2, counts, MPI.SUM, recv_capacity=cap, comm=comm)[0] * ct).sum().backward()
    assert torch.equal(xe.grad, x.grad)
    m.flush()


def _parent_allgatherv_grad(g, recv_counts, rows):
    """allgatherv's former adjoint: every received segment copied into a zero-padded (P, rows, *S) tensor,
    then reduce_scatter."""
    P = recv_counts.shape[0]
    offsets = torch.cumsum(recv_counts, 0) - recv_counts
    i = torch.arange(rows, device=g.device)
    idx = torch.where(i < recv_counts.view(P, 1), offsets.view(P, 1) + i, g.shape[0])
    padded = torch.cat([g, g.new_zeros((1, *g.shape[1:]))])[idx]
    return m.reduce_scatter(padded, MPI.SUM, comm=comm)


@peers
def test_allgatherv_backward_matches_padded_formulation(device):
    """allgatherv's backward through reduce_scatterv equals the padded reduce_scatter formulation on seeded
    inputs with capacities that differ per rank, bitwise up to the sign of zero."""
    n = 9
    gen = torch.Generator().manual_seed(11 + rank)
    for count, cap in ((4 + rank, None), (n, 3 + 2 * rank), (-1 + 3 * rank, n + rank), (2, 0)):
        counts = torch.tensor(count, device=device)
        x = torch.randn(n, 3, generator=gen).to(device).requires_grad_(True)
        out, rc = m.allgatherv(x, counts, recv_capacity=cap, comm=comm)
        ct = torch.randn(out.shape, generator=gen).to(device)
        ct[:1] = -0.0                           # cotangents of -0.0: the sign of zero may differ
        (out * ct).sum().backward()
        want = _parent_allgatherv_grad(ct, rc, n)
        got = x.grad
        assert torch.equal(got, want), (count, cap)
        nz = want != 0
        assert torch.equal(got[nz].view(torch.int32), want[nz].view(torch.int32))


@peers
def test_allgatherv_reverse_mode(device):
    """The reverse mode: each rank's rows land where a reduce_scatterv with these send counts took them from."""
    from mpi4jax_b200._src.collective_ops.allgatherv import allgatherv_reverse

    n, rows = 4, 11 + rank
    y = (torch.arange(n * 2, dtype=torch.float32).reshape(n, 2) + 100 * rank).to(device)
    for counts in ([1 + (q + rank) % 3 for q in range(size)], [-1] + [n + 2] * (size - 1), [20] * size):
        got = allgatherv_reverse(y, torch.tensor(counts, device=device), rows, comm)
        assert torch.equal(got.cpu(), _grad_oracle(y, torch.tensor(counts), rows, n)), counts


def test_reduce_scatterv_user_op(device):
    """MPI.Op.Create: a non-commutative 2x2 matrix product, folded in rank order over the contributors."""
    matmul = MPI.Op.Create(lambda a, b: a @ b, commute=False)
    n = 3
    x = torch.stack([torch.tensor([[1.0, float((rank + 1) * (i + 1))], [float(i), 1.0]])
                     for i in range(size * n)])
    counts = [n - (q + rank) % 2 for q in range(size)]
    out, rc = m.reduce_scatterv(x.to(device), counts, matmul, recv_capacity=n, comm=comm)
    xs, cs = _gathered(x, counts)
    recv = [min(cs[q][rank], n) for q in range(size)]
    assert rc.tolist() == recv
    want = torch.zeros(n, 2, 2)
    for i in range(max(recv)):
        parts = [xs[q][sum(cs[q][:rank]) + i] for q in range(size) if i < recv[q]]
        acc = parts[0]
        for p in parts[1:]:
            acc = acc @ p
        want[i] = acc
    assert torch.equal(out.cpu(), want)
    with pytest.raises(NotImplementedError, match="derivative of reduce_scatterv"):
        m.reduce_scatterv(x.to(device).requires_grad_(True), counts, matmul, comm=comm)


def test_host_staged_reduce_scatterv(device, monkeypatch):
    from mpi4jax_b200._src.backends import host_staged

    monkeypatch.setattr(host_staged, "ACTIVE", host_staged.ACTIVE)      # restore the flag afterwards
    host_staged_comm = comm.Clone()
    hs = host_staged.HostStagedComm(host_staged_comm, "unit test")
    try:
        n = 5 + rank
        x = (torch.arange(n * 2, dtype=torch.float32).reshape(n, 2) + 10 * rank).to(device)
        counts = torch.tensor([(q + rank + 1) % 4 for q in range(size)], device=device)
        out, rc = hs.reduce_scatterv(x, counts, 4, codes.SUM)
        want, want_rc = _oracle(x, counts, "SUM", 4)
        assert out.device == x.device and rc.device == x.device
        assert _same(out, want) and torch.equal(rc.cpu(), want_rc)
        y = (torch.arange(8, dtype=torch.float32).reshape(4, 2) + rank).to(device)
        place = torch.tensor([1 + q for q in range(size)], device=device)
        back, _ = hs.allgatherv(y, torch.tensor(4, device=device), n, place)
        assert torch.equal(back.cpu(), _grad_oracle(y, place.cpu(), n, 4))
    finally:
        host_staged_comm.Free()


def test_staging_formula_reduce_scatterv():
    from mpi4jax_b200._src import native
    from mpi4jax_b200._src.backends.cuda import stage_need

    if not native.HAS_CUDA_EXT:
        pytest.skip(f"native library not loaded: {native.CUDA_EXT_ERROR}")
    assert codes.OPC_REDUCE_SCATTERV == 16 and codes.OPC_ALLGATHERV == 15
    for nranks in range(1, 17):
        for nbytes in [0, 1, 15, 16, 17, 4095, 4096, 65537, (1 << 20) + 3, 1 << 30]:
            want = 128 + (nbytes + 15) // 16 * 16 * nranks + 4096
            assert stage_need(16, nranks, nbytes) == native.lib.b2_stage_need(16, nranks, nbytes) == want


def test_reduce_scatterv_debug_log(device, capsys):
    from mpi4jax_b200._src.native import set_logging

    x = torch.ones((4, 3), device=device)
    counts = torch.ones(size, dtype=torch.int64, device=device)
    m.reduce_scatterv(x, counts, MPI.SUM, comm=comm)
    m.flush()
    capsys.readouterr()
    set_logging(True)
    try:
        m.reduce_scatterv(x, counts, MPI.SUM, comm=comm)
        m.flush()
    finally:
        set_logging(False)
    out = capsys.readouterr().out
    via = " via pull" if device.type == "cuda" else ""
    assert re.search(rf"^r{rank} \| \w{{8}} \| MPI_Reduce_scatterv( \(\w+\))? with 4 rows of 12 bytes{via}", out,
                     re.M), out
    assert re.search(rf"^r{rank} \| \w{{8}} \| MPI_Reduce_scatterv( \(\w+\))? done with code 0", out, re.M), out


_inside_job = size > 1 or "MPI4JAX_B200_NESTED" in os.environ


@pytest.mark.gpu
@pytest.mark.skipif(_inside_job, reason="already inside a multi-rank job")
def test_reduce_scatterv_three_ranks_gpu():
    """A non-power-of-two world: the CUDA tests of this file in a three-rank job (the ranks share the
    GPUs there are)."""
    from mpi4jax_b200.run import launch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    repo = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    test_file = os.path.relpath(os.path.abspath(__file__), repo)
    args = ["-m", "pytest", test_file, "-q", "-rp", "-m", "gpu", "-k", "not compiled",
            "-p", "no:cacheprovider"]
    cwd = os.getcwd()
    os.chdir(repo)
    try:
        with tempfile.TemporaryDirectory(prefix="mpi4jax-b200-rsv-job-") as logs:
            code, _ = launch(3, args, timeout=900, output_dir=logs, env_extra={"MPI4JAX_B200_NESTED": "1"})
            outs = [open(os.path.join(logs, f"rank{r}.log")).read() for r in range(3)]
    finally:
        os.chdir(cwd)
    for r, out in enumerate(outs):
        assert code == 0 and re.search(r"PASSED .*test_reduce_scatterv_multi_chunk\[cuda\]", out), \
            f"rank {r} of the 3-rank job (exit code {code}):\n{out[-4000:]}"
