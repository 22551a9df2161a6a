"""gatherv: every rank's first ``count`` rows, packed in rank order on the root,
``(N, *S) -> (recv_capacity, *S)``; the other ranks get their input back.

Oracle: every rank gathers all inputs, counts and the root's capacity with the object API and applies the
documented rules (clamp the count to ``[0, N]``, pack the segments in source-rank order, clip them to the
capacity, zero the rest) in plain torch on the CPU; results compare bitwise.  The gradient oracle is the
root's cotangent rows that came from this rank, plus this rank's own cotangent off the root.  The CUDA
variants need peers: in a single-process run they are checked in a two-rank job whose ranks share the
GPU, and ``test_gatherv_three_ranks_gpu`` runs them with three ranks."""

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

peers = needs_peers("gatherv between ranks")


def _roots():
    """Every root at 3 ranks; 0 and the last one otherwise."""
    return list(range(size)) if size <= 3 else [0, size - 1]


def _gathered(x, count, n):
    """(inputs, counts clamped to [0, n]) of every rank, in rank order."""
    c = int(count.item()) if isinstance(count, torch.Tensor) else int(count)
    raw = x.detach().cpu().contiguous().reshape(-1).view(torch.uint8)      # every dtype pickles as bytes
    everything = comm.allgather((raw, tuple(x.shape), min(max(c, 0), n)))
    return [e[0].view(x.dtype).reshape(e[1]) for e in everything], [e[2] for e in everything]


def _segments(ns, cap):
    """(offset, rows) on the root of every rank's segment."""
    out, filled = [], 0
    for n in ns:
        k = min(n, cap - filled)
        out.append((filled, k))
        filled += k
    return out


def _oracle(x, count, root, cap):
    """(out, recv_counts) of this rank, from everybody's x and count."""
    xs, ns = _gathered(x, count, x.shape[0])
    if rank != root:
        return x.detach().cpu(), torch.zeros(size, dtype=torch.int64)
    out = torch.zeros((cap, *x.shape[1:]), dtype=x.dtype)
    recv = []
    for q, (off, k) in enumerate(_segments(ns, cap)):
        out[off: off + k] = xs[q][:k]
        recv.append(k)
    return out, torch.tensor(recv, dtype=torch.int64)


def _oracle_grad(ct, count, root, n):
    """Cotangent of x: the root's cotangent rows (as many as its capacity) that came from this rank,
    zero-padded to n rows; off the root this rank's own cotangent adds (its result was x)."""
    cts = comm.allgather(ct.detach().cpu())
    _, ns = _gathered(torch.zeros(n), count, n)
    off, k = _segments(ns, cts[root].shape[0])[rank]
    g = torch.zeros((n, *ct.shape[1:]), dtype=ct.dtype)
    g[:k] = cts[root][off: off + k]
    return g if rank == root else g + ct.detach().cpu()


def _check(x, count, root, cap=None):
    _x = x.clone()
    _c = count.clone() if isinstance(count, torch.Tensor) else count
    out, rc = m.gatherv(x, count, root, recv_capacity=cap, comm=comm)
    cap = x.shape[0] * size if cap is None else cap
    want, want_rc = _oracle(x, count, root, cap)
    if rank == root:
        assert out.shape == (cap, *x.shape[1:]) and out.dtype == x.dtype and out.device == x.device
    else:
        assert out is x
    assert rc.dtype == torch.int64 and rc.shape == (size,) and rc.device == x.device
    assert torch.equal(out.cpu(), want), (int(count), root, cap)
    assert torch.equal(rc.cpu(), want_rc), (int(count), root, cap)
    assert torch.equal(x, _x)
    if isinstance(count, torch.Tensor):
        assert torch.equal(count, _c)
    return out, rc


def _count_cases(n):
    """(count, capacity) cases; the counts differ between ranks, the capacity is read on the root only."""
    return [
        (n, None),                        # everything: the gather of x
        (n // 2, None),                   # balanced, half
        (0, None),                        # nothing at all
        (rank % 3, None),                 # below N, different per rank
        (n + 5 + rank, None),             # past N: clamped to N
        (-3 + rank, None),                # negative on rank 0 (and on rank 1 / 2 of a 3-rank job: -2, -1)
        (n - rank, 2 + rank),             # capacity below the sum: drops (and differs, unread, elsewhere)
        (n // 2 + rank, n + 1),           # capacity between N and the sum
        (n, n * size + 5),                # capacity > N * nproc
        (n, 0),                           # capacity 0
    ]


@peers
def test_gatherv_cases(device):
    n = 7
    x = (torch.arange(n * 3, dtype=torch.float32).reshape(n, 3) + 100 * rank).to(device)
    for root in _roots():
        for count, cap in _count_cases(n):
            _check(x, torch.tensor(count, device=device), root, cap)
    # a Python int and an int32 tensor are accepted too
    out, _ = _check(x, 2 + rank, 0)
    assert torch.equal(out, _check(x, torch.tensor(2 + rank, dtype=torch.int32, device=device), 0)[0])
    # N = 0
    e = torch.empty((0, 3), device=device)
    out, rc = _check(e, torch.tensor(1, device=device), size - 1, 4)
    assert rc.tolist() == [0] * size


@peers
def test_gatherv_odd_rows_and_noncontiguous(device):
    """Row sizes that are not multiples of 16 bytes, and a non-contiguous x."""
    torch.manual_seed(5 + rank)
    for dtype, row in ((torch.int8, (3,)), (torch.int8, (5, 1)), (torch.float16, (7,)), (torch.float64, (3,))):
        x = (torch.randn(11, *row) * 50).to(dtype).to(device)
        for count, cap in _count_cases(11):
            _check(x, torch.tensor(count, device=device), size - 1, cap)
    base = torch.randn(4, 9, device=device)
    xt = base.t()                                                       # (9, 4), not contiguous
    assert not xt.is_contiguous()
    for root in _roots():
        _check(xt, torch.tensor(5 + rank, device=device), root, 11)


@peers
def test_gatherv_dtypes(device):
    for k, dtype in enumerate(codes.DTYPE_CODE):
        g = torch.Generator().manual_seed(10 * k + rank)
        v = torch.randint(0, 100, (6, 2), generator=g)
        x = (v % 2 == 0) if dtype == torch.bool else v.to(dtype)
        _check(x.to(device), torch.tensor((k + rank) % 7, device=device), k % size, 9)


@peers
def test_gatherv_multi_chunk(device):
    """4 MiB per rank: more chunks than CTAs, segments that end inside chunks and land at offsets that
    are not chunk-aligned; the other ranks walk the same chunks without pulling."""
    n = 1024
    x = torch.randn(n, 1024, device=device, generator=torch.Generator(device).manual_seed(rank))   # 4 MiB
    root = size - 1
    _check(x, torch.tensor(n, device=device), root)
    _check(x, torch.tensor(n - 37 * rank - 1, device=device), 0)
    _check(x, torch.tensor(n * (rank + 1) // size, device=device), root)          # skewed
    _check(x, torch.tensor(n // 2 + 3 * rank, device=device), 0, n + 5)           # drops at the root
    xo = torch.randn(n, 1023, device=device).to(torch.bfloat16)                  # 2046-byte rows
    _check(xo, torch.tensor(n - 1 - rank, device=device), root)


def test_gatherv_single_rank(device):
    """A one-rank communicator: the clamped rows, in order, then zeros."""
    solo = comm.Split(rank, 0)
    try:
        x = torch.randn(5, 3, device=device)
        out, rc = m.gatherv(x, torch.tensor(3, device=device), 0, comm=solo)
        assert out.shape == (5, 3) and rc.tolist() == [3]
        assert torch.equal(out[:3], x[:3]) and not out[3:].any()
        out, rc = m.gatherv(x, 9, 0, recv_capacity=2, comm=solo)
        assert torch.equal(out, x[:2]) and rc.tolist() == [2]
    finally:
        m.flush()
        solo.Free()


def test_gatherv_errors(device, monkeypatch):
    x = torch.ones((4, 2), device=device)
    good = torch.tensor(1, device=device)
    other = "meta" if device.type == "cpu" else "cpu"
    with pytest.raises(ValueError, match=re.escape("Gatherv input must have shape (rows, ...)")):
        m.gatherv(torch.tensor(1.0, device=device), good, 0, comm=comm)
    with pytest.raises(ValueError, match=re.escape("Gatherv count must have shape ()")):
        m.gatherv(x, torch.ones(1, dtype=torch.int64, device=device), 0, comm=comm)
    with pytest.raises(ValueError, match=re.escape("Gatherv count must have shape ()")):
        m.gatherv(x, torch.ones(size, dtype=torch.int64, device=device), 0, comm=comm)
    with pytest.raises(TypeError, match="Gatherv count must be an integer tensor"):
        m.gatherv(x, torch.tensor(1.0, device=device), 0, comm=comm)
    with pytest.raises(TypeError, match="Gatherv count must be an integer tensor"):
        m.gatherv(x, torch.tensor(True, device=device), 0, comm=comm)
    with pytest.raises(TypeError):
        m.gatherv(x, 1.5, 0, comm=comm)
    with pytest.raises(ValueError, match="Gatherv count must live on the device of x"):
        m.gatherv(x, torch.tensor(1, device=other), 0, comm=comm)
    if rank == 0:                       # the capacity is read on the root only
        with pytest.raises(ValueError, match=re.escape("Gatherv recv_capacity must be >= 0")):
            m.gatherv(x, good, 0, recv_capacity=-1, comm=comm)
    with pytest.raises(TypeError, match='unexpected type for argument "recv_capacity"'):
        m.gatherv(x, good, 0, recv_capacity=2.0, comm=comm)
    with pytest.raises(TypeError, match='unexpected type for argument "root"'):
        m.gatherv(x, good, 0.0, comm=comm)
    with pytest.raises(RuntimeError, match="Explicit token management"):
        m.gatherv(x, good, 0, comm=comm, token=1)
    # an invalid root takes gather's abort path (here: raise)
    monkeypatch.setenv("MPI4JAX_B200_ABORT_ON_ERROR", "0")
    with pytest.raises(MPI.MPIError, match=re.escape(f"MPI_Gatherv returned error code 4: invalid root rank {size}")):
        m.gatherv(x, good, size, comm=comm)


@peers
def test_gatherv_jit_and_graph_replays(device):
    """Captured once, replayed with the count changed in place: oracle-exact every time (the count is
    read on the device; a host read of it could not be captured)."""
    if device.type != "cuda":
        pytest.skip("CUDA graphs")
    n, cap, root = 9, 9 + size, size - 1
    x = torch.randn(n, 5, device=device, generator=torch.Generator(device).manual_seed(rank))
    count = torch.zeros((), dtype=torch.int64, device=device)
    f = m.jit(lambda t, c: m.gatherv(t * 2, c, root, recv_capacity=cap, comm=comm))
    cases = [c for c, _ in _count_cases(n)]
    for c in cases:                                     # eager warm-up, capture, replays
        count.fill_(c)
        out, rc = f(x, count)
        want, want_rc = _oracle(x * 2, count, root, cap)
        assert torch.equal(out.cpu(), want) and torch.equal(rc.cpu(), want_rc), c
    # a direct capture
    static_count = torch.tensor(cases[0], device=device)
    m.gatherv(x, static_count, 0, recv_capacity=cap, comm=comm)      # staging sized before the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        g_out, g_rc = m.gatherv(x, static_count, 0, recv_capacity=cap, comm=comm)
    for c in cases:
        static_count.fill_(c)
        g.replay()
        want, want_rc = _oracle(x, static_count, 0, cap)
        assert torch.equal(g_out.cpu(), want) and torch.equal(g_rc.cpu(), want_rc), c
    m.flush()


@peers
def test_gatherv_derivatives(device):
    """vjp / backward: the root's cotangent rows from this rank (plus its own cotangent off the root; random
    fp32, bitwise); rows past the count and rows the root dropped get nothing from it.  jvp: gatherv of
    the tangent.  Double backward: the adjoint of the adjoint (scatterv's, gatherv's reverse mode) is the
    forward."""
    n = 6
    gen = torch.Generator().manual_seed(7 + rank)
    for root in _roots():
        for count, cap in ((4 - rank % 2, None), (n, 2 + 3 * rank), (-1 + 2 * rank, n + 1)):
            c = n * size if cap is None else cap
            rows = c if rank == root else n
            counts = torch.tensor(count, device=device)
            x = torch.randn(n, 2, generator=gen).to(device)
            ct = torch.randn(rows, 2, generator=gen).to(device)
            t = torch.randn(n, 2, generator=gen).to(device)

            def f(v):
                return m.gatherv(v, counts, root, recv_capacity=cap, comm=comm)[0]

            res, pullback = vjp(f, x)
            assert torch.equal(res.cpu(), _oracle(x, counts, root, c)[0])
            (g,) = pullback(ct)
            want = _oracle_grad(ct, counts, root, n)
            assert torch.equal(g.cpu(), want), (root, count, cap)
            if rank == root:
                assert not g[min(max(count, 0), n):].any()     # rows never contributed get no gradient
            _, tan = jvp(f, (x,), (t,))
            assert torch.equal(tan.cpu(), _oracle(t, counts, root, c)[0])
            xr = x.clone().requires_grad_(True)
            ctr = ct.clone().requires_grad_(True)
            out, rc = m.gatherv(xr, counts, root, recv_capacity=cap, comm=comm)
            assert not rc.requires_grad
            (gx,) = torch.autograd.grad((out * ctr).sum(), xr, create_graph=True)
            assert torch.equal(gx.detach().cpu(), want)
            (gct,) = torch.autograd.grad((gx * t).sum(), ctr)
            assert torch.equal(gct.cpu(), _oracle(t, counts, root, c)[0]), (root, count, cap)
            xr.grad = None
            (m.gatherv(xr, counts, root, recv_capacity=cap, comm=comm)[0] * ct).sum().backward()
            assert torch.equal(xr.grad.cpu(), want)


@peers
def test_gatherv_vmap(device):
    n = 5
    count = torch.tensor(2 + rank % 3, device=device)
    root = size - 1
    xb = (torch.arange(3 * n * 2, dtype=torch.float32).reshape(3, n, 2) + 100 * rank).to(device)
    want = torch.stack([m.gatherv(xb[i], count, root, recv_capacity=4, comm=comm)[0] for i in range(3)])
    f = vmap(lambda v: m.gatherv(v, count, root, recv_capacity=4, comm=comm)[0], in_dims=0, out_dims=0)
    assert torch.equal(f(xb), want)
    f1 = vmap(lambda v: m.gatherv(v, count, root, recv_capacity=4, comm=comm)[0], in_dims=1, out_dims=0)
    assert torch.equal(f1(xb.movedim(0, 1).contiguous()), want)
    with pytest.raises(ValueError, match="count must not be batched"):
        vmap(lambda v, c: m.gatherv(v, c, root, comm=comm)[0])(xb, count.expand(3).contiguous())


def test_gatherv_fake_shape_and_effect():
    """The root op has the capacity's rows, the leaf op the shape of x; no device work."""
    from torch._higher_order_ops.effects import _EffectType, _get_effect
    from torch._subclasses.fake_tensor import FakeTensorMode

    with FakeTensorMode():
        x, count = torch.empty(4, 3, 2), torch.empty((), dtype=torch.int64)
        out, rc = torch.ops.mpi4jax_b200.gatherv_root(x, count, 0, 7, 4, comm._id, False)
        assert out.shape == (7, 3, 2) and rc.shape == (size,) and rc.dtype == torch.int64
        out, rc = torch.ops.mpi4jax_b200.gatherv_leaf(x, count, 0, 4, comm._id)
        assert out.shape == (4, 3, 2) and rc.shape == (size,) and rc.dtype == torch.int64
        out, rc = m.compiled.gatherv(torch.empty(4, 3), count, 0, comm=comm)
        assert out.shape == ((4 * size, 3) if rank == 0 else (4, 3)) and rc.shape == (size,)
        assert rc.device == out.device
    for name in ("gatherv_root", "gatherv_leaf"):
        assert _get_effect(f"mpi4jax_b200::{name}") == _EffectType.ORDERED


def test_gatherv_compiled_errors(device):
    """compiled.gatherv, the raw torch.ops ops and their fake kernels refuse what the eager op refuses, on
    the host."""
    from torch._subclasses.fake_tensor import FakeTensorMode

    x = torch.ones((4, 2), device=device)
    other = "meta" if device.type == "cpu" else "cpu"
    bad = [
        (ValueError, "must live on the device of x", x, torch.tensor(1, device=other)),
        (ValueError, re.escape("must have shape ()"), x, torch.ones(1, dtype=torch.int64, device=device)),
        (TypeError, "must be an integer tensor", x, torch.tensor(1.0, device=device)),
    ]
    for exc, msg, xx, count in bad:
        with pytest.raises(exc, match=msg):
            m.compiled.gatherv(xx, count, 0, comm=comm)
        with pytest.raises(exc, match=msg):
            torch.ops.mpi4jax_b200.gatherv_root(xx, count, 0, 4, 4, comm._id, False)
        with pytest.raises(exc, match=msg):
            torch.ops.mpi4jax_b200.gatherv_leaf(xx, count, 0, 4, comm._id)
    with pytest.raises(ValueError, match=re.escape("recv_capacity must be >= 0")):
        torch.ops.mpi4jax_b200.gatherv_root(x, torch.tensor(1, device=device), 0, -1, 4, comm._id, False)
    with FakeTensorMode():
        with pytest.raises(ValueError, match=re.escape("must have shape ()")):
            torch.ops.mpi4jax_b200.gatherv_leaf(torch.empty(4, 2), torch.empty(2, dtype=torch.int64), 0, 4, comm._id)


@peers
def test_gatherv_compiled_and_grad(device):
    """compiled.gatherv forward and gradient, bitwise equal to the eager op's, on every rank and root."""
    n = 6
    for root in _roots():
        cap = 5 + root
        count = torch.tensor(3 + rank, device=device)
        rows = cap if rank == root else n
        ct = torch.randn(rows, 2, generator=torch.Generator().manual_seed(rank)).to(device)

        def loss(F, v, c):
            return (F.gatherv(v * 2, c, root, recv_capacity=cap, comm=comm)[0] * ct).sum()

        f = torch.compile(lambda v, c: loss(m.compiled, v, c), backend="aot_eager", fullgraph=True)
        x = (torch.arange(n * 2, dtype=torch.float32).reshape(n, 2) + rank).to(device)
        xc, xe = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
        y, ye = f(xc, count), loss(m, xe, count)
        assert torch.equal(y, ye)
        y.backward()
        ye.backward()
        assert torch.equal(xc.grad, xe.grad)
        assert torch.equal(xc.grad.cpu(), 2 * _oracle_grad(ct, count, root, n))
    m.flush()


def test_host_staged_gatherv(device, monkeypatch):
    from mpi4jax_b200._src.backends import host_staged

    monkeypatch.setattr(host_staged, "ACTIVE", host_staged.ACTIVE)      # restore the flag afterwards
    host_staged_comm = comm.Clone()
    hs = host_staged.HostStagedComm(host_staged_comm, "unit test")
    try:
        n, root = 5, size - 1
        x = (torch.arange(n * 2, dtype=torch.float32).reshape(n, 2) + 10 * rank).to(device)
        count = torch.tensor((rank + 2) % 4, device=device)
        out, rc = hs.gatherv(x, count, root, 4, n)
        want, want_rc = _oracle(x, count, root, 4)
        assert rc.device == x.device and torch.equal(rc.cpu(), want_rc)
        if rank == root:
            assert out.device == x.device and torch.equal(out.cpu(), want)
        else:
            assert out is None
    finally:
        host_staged_comm.Free()


def test_staging_formula_gatherv():
    from mpi4jax_b200._src import native
    from mpi4jax_b200._src.backends.cuda import stage_need

    if not native.HAS_CUDA_EXT:
        pytest.skip(f"native library not loaded: {native.CUDA_EXT_ERROR}")
    assert codes.OPC_GATHERV == 17
    for nranks in range(1, 17):
        for nbytes in [0, 1, 15, 16, 17, 4095, 4096, 65537, (1 << 20) + 3, 1 << 30]:
            want = 128 + (nbytes + 15) // 16 * 16 + 4096
            assert stage_need(17, nranks, nbytes) == native.lib.b2_stage_need(17, nranks, nbytes) == want


def test_gatherv_debug_log(device, capsys):
    from mpi4jax_b200._src.native import set_logging

    x = torch.ones((4, 3), device=device)
    count = torch.tensor(2, device=device)
    m.gatherv(x, count, 0, comm=comm)
    m.flush()
    capsys.readouterr()
    set_logging(True)
    try:
        m.gatherv(x, count, 0, comm=comm)
        m.flush()
    finally:
        set_logging(False)
    out = capsys.readouterr().out
    assert re.search(rf"^r{rank} \| \w{{8}} \| MPI_Gatherv( \(\w+\))? with 4 rows of 12 bytes to root 0", out, re.M), out
    assert re.search(rf"^r{rank} \| \w{{8}} \| MPI_Gatherv( \(\w+\))? done with code 0", out, re.M), out


_inside_job = size > 1 or "MPI4JAX_B200_NESTED" in os.environ


@pytest.mark.gpu
@pytest.mark.skipif(_inside_job, reason="already inside a multi-rank job")
def test_gatherv_three_ranks_gpu():
    """A non-power-of-two world, every root: the CUDA tests of this file in a three-rank job (the ranks
    share the GPUs there are)."""
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
        with tempfile.TemporaryDirectory(prefix="mpi4jax-b200-gv-job-") as logs:
            code, _ = launch(3, args, timeout=900, output_dir=logs, env_extra={"MPI4JAX_B200_NESTED": "1"})
            outs = [open(os.path.join(logs, f"rank{r}.log")).read() for r in range(3)]
    finally:
        os.chdir(cwd)
    for r, out in enumerate(outs):
        assert code == 0 and re.search(r"PASSED .*test_gatherv_derivatives\[cuda\]", out), \
            f"rank {r} of the 3-rank job (exit code {code}):\n{out[-4000:]}"
