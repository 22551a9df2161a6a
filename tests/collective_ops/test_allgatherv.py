"""allgatherv: every rank's first ``count`` rows, packed in rank order, ``(N, *S) -> (recv_capacity, *S)``.

Oracle: every rank gathers all inputs, counts and capacities with the object API and applies the
documented rules (clamp the count to ``[0, N]``, pack the segments in source-rank order, clip them to
the capacity, zero the rest) in plain torch on the CPU; results compare bitwise.  The gradient oracle is
the rank-order fold of the zero-padded cotangent segments.  The CUDA variants need peers: in a
single-process run they are checked in a two-rank job whose ranks share the GPU, and
``test_allgatherv_three_ranks_gpu`` runs them with three ranks."""

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

peers = needs_peers("allgatherv between ranks")


def _gathered(x, count, cap, n):
    """(inputs, counts clamped to [0, n], capacities) of every rank, in rank order."""
    c = int(count.item()) if isinstance(count, torch.Tensor) else int(count)
    raw = x.detach().cpu().contiguous().reshape(-1).view(torch.uint8)      # every dtype pickles as bytes
    everything = comm.allgather((raw, tuple(x.shape), min(max(c, 0), n), cap))
    xs = [e[0].view(x.dtype).reshape(e[1]) for e in everything]
    return xs, [e[2] for e in everything], [e[3] for e in everything]


def _oracle(x, count, cap):
    """(out, recv_counts) of this rank, from everybody's x and count."""
    xs, ns, _ = _gathered(x, count, cap, x.shape[0])
    out = torch.zeros((cap, *x.shape[1:]), dtype=x.dtype)
    recv, filled = [], 0
    for q in range(size):
        k = min(ns[q], cap - filled)
        out[filled: filled + k] = xs[q][:k]
        recv.append(k)
        filled += k
    return out, torch.tensor(recv, dtype=torch.int64)


def _oracle_grad(ct, count, n, cap):
    """Cotangent of x: receiver q's kept rows of this rank's segment, zero-padded to n rows, folded over q
    in rank order.  ``cap`` (the rows of ``ct``) may differ between ranks."""
    cts, ns, caps = _gathered(ct, count, cap, n)
    parts = []
    for q in range(size):
        seg = torch.zeros((n, *ct.shape[1:]), dtype=ct.dtype)
        filled = 0
        for p in range(size):
            k = min(ns[p], caps[q] - filled)
            if p == rank:
                seg[:k] = cts[q][filled: filled + k]
            filled += k
        parts.append(seg)
    acc = parts[0].clone()
    for seg in parts[1:]:
        acc += seg
    return acc


def _check(x, count, cap=None):
    _x = x.clone()
    _c = count.clone() if isinstance(count, torch.Tensor) else count
    out, rc = m.allgatherv(x, count, recv_capacity=cap, comm=comm)
    cap = x.shape[0] * size if cap is None else cap
    want, want_rc = _oracle(x, count, cap)
    assert out.shape == (cap, *x.shape[1:]) and out.dtype == x.dtype and out.device == x.device
    assert rc.dtype == torch.int64 and rc.shape == (size,) and rc.device == x.device
    assert torch.equal(out.cpu(), want), (int(count), cap)
    assert torch.equal(rc.cpu(), want_rc), (int(count), cap)
    assert torch.equal(x, _x)
    if isinstance(count, torch.Tensor):
        assert torch.equal(count, _c)
    return out, rc


def _count_cases(n):
    """(count, capacity) cases; the counts differ between ranks."""
    return [
        (n, None),                        # everything: the allgather of x
        (n // 2, None),                   # balanced, half
        (0, None),                        # nothing at all
        (rank % 3, None),                 # below N, different per rank
        (n + 5 + rank, None),             # past N: clamped to N
        (-3 + rank, None),                # negative on rank 0 (and on rank 1 / 2 of a 3-rank job: -2, -1)
        (n - rank, 2 + rank),             # capacity below the sum: drops, capacities differ between ranks
        (n // 2 + rank, n + 1),           # capacity between N and the sum
        (n, n * size + 5),                # capacity > N * nproc
        (n, 0),                           # capacity 0
    ]


@peers
def test_allgatherv_cases(device):
    n = 7
    x = (torch.arange(n * 3, dtype=torch.float32).reshape(n, 3) + 100 * rank).to(device)
    for count, cap in _count_cases(n):
        _check(x, torch.tensor(count, device=device), cap)
    # a Python int and an int32 tensor are accepted too
    out, rc = _check(x, 2 + rank)
    assert torch.equal(out, _check(x, torch.tensor(2 + rank, dtype=torch.int32, device=device))[0])
    # N = 0
    e = torch.empty((0, 3), device=device)
    out, rc = _check(e, torch.tensor(1, device=device), 4)
    assert out.shape == (4, 3) and rc.tolist() == [0] * size


@peers
def test_allgatherv_odd_rows_and_noncontiguous(device):
    """Row sizes that are not multiples of 16 bytes, and a non-contiguous x."""
    torch.manual_seed(5 + rank)
    for dtype, row in ((torch.int8, (3,)), (torch.int8, (5, 1)), (torch.float16, (7,)), (torch.float64, (3,))):
        x = (torch.randn(11, *row) * 50).to(dtype).to(device)
        for count, cap in _count_cases(11):
            _check(x, torch.tensor(count, device=device), cap)
    base = torch.randn(4, 9, device=device)
    xt = base.t()                                                       # (9, 4), not contiguous
    assert not xt.is_contiguous()
    _check(xt, torch.tensor(5 + rank, device=device), 11)


@peers
def test_allgatherv_dtypes(device):
    for k, dtype in enumerate(codes.DTYPE_CODE):
        g = torch.Generator().manual_seed(10 * k + rank)
        v = torch.randint(0, 100, (6, 2), generator=g)
        x = (v % 2 == 0) if dtype == torch.bool else v.to(dtype)
        _check(x.to(device), torch.tensor((k + rank) % 7, device=device), 9)


@peers
def test_allgatherv_multi_chunk(device):
    """4 MiB per rank: more chunks than CTAs, segments that end inside chunks and land at offsets that
    are not chunk-aligned."""
    n = 1024
    x = torch.randn(n, 1024, device=device, generator=torch.Generator(device).manual_seed(rank))   # 4 MiB
    _check(x, torch.tensor(n, device=device))
    _check(x, torch.tensor(n - 37 * rank - 1, device=device))
    _check(x, torch.tensor(n * (rank + 1) // size, device=device))                # skewed
    _check(x, torch.tensor(n // 2 + 3 * rank, device=device), n + 5)              # drops at the receivers
    xo = torch.randn(n, 1023, device=device).to(torch.bfloat16)                  # 2046-byte rows
    _check(xo, torch.tensor(n - 1 - rank, device=device))


def test_allgatherv_single_rank(device):
    """A one-rank communicator: the clamped rows, in order, then zeros."""
    solo = comm.Split(rank, 0)
    try:
        x = torch.randn(5, 3, device=device)
        out, rc = m.allgatherv(x, torch.tensor(3, device=device), comm=solo)
        assert out.shape == (5, 3) and rc.tolist() == [3]
        assert torch.equal(out[:3], x[:3]) and not out[3:].any()
        out, rc = m.allgatherv(x, 9, recv_capacity=2, comm=solo)
        assert torch.equal(out, x[:2]) and rc.tolist() == [2]
    finally:
        m.flush()
        solo.Free()


def test_allgatherv_errors(device):
    x = torch.ones((4, 2), device=device)
    good = torch.tensor(1, device=device)
    other = "meta" if device.type == "cpu" else "cpu"
    with pytest.raises(ValueError, match=re.escape("Allgatherv input must have shape (rows, ...)")):
        m.allgatherv(torch.tensor(1.0, device=device), good, comm=comm)
    with pytest.raises(ValueError, match=re.escape("Allgatherv count must have shape ()")):
        m.allgatherv(x, torch.ones(1, dtype=torch.int64, device=device), comm=comm)
    with pytest.raises(ValueError, match=re.escape("Allgatherv count must have shape ()")):
        m.allgatherv(x, torch.ones(size, dtype=torch.int64, device=device), comm=comm)
    with pytest.raises(TypeError, match="Allgatherv count must be an integer tensor"):
        m.allgatherv(x, torch.tensor(1.0, device=device), comm=comm)
    with pytest.raises(TypeError, match="Allgatherv count must be an integer tensor"):
        m.allgatherv(x, torch.tensor(True, device=device), comm=comm)
    with pytest.raises(TypeError):
        m.allgatherv(x, 1.5, comm=comm)
    with pytest.raises(ValueError, match="Allgatherv count must live on the device of x"):
        m.allgatherv(x, torch.tensor(1, device=other), comm=comm)
    with pytest.raises(ValueError, match=re.escape("Allgatherv recv_capacity must be >= 0")):
        m.allgatherv(x, good, recv_capacity=-1, comm=comm)
    with pytest.raises(TypeError, match='unexpected type for argument "recv_capacity"'):
        m.allgatherv(x, good, recv_capacity=2.0, comm=comm)
    with pytest.raises(RuntimeError, match="Explicit token management"):
        m.allgatherv(x, good, comm=comm, token=1)


@peers
def test_allgatherv_jit_and_graph_replays(device):
    """Captured once, replayed with the count changed in place: oracle-exact every time (the count is
    read on the device; a host read of it could not be captured)."""
    if device.type != "cuda":
        pytest.skip("CUDA graphs")
    n, cap = 9, 9 + size
    x = torch.randn(n, 5, device=device, generator=torch.Generator(device).manual_seed(rank))
    count = torch.zeros((), dtype=torch.int64, device=device)
    f = m.jit(lambda t, c: m.allgatherv(t * 2, c, recv_capacity=cap, comm=comm))
    cases = [c for c, _ in _count_cases(n)]
    for c in cases:                                     # eager warm-up, capture, replays
        count.fill_(c)
        out, rc = f(x, count)
        want, want_rc = _oracle(x * 2, count, cap)
        assert torch.equal(out.cpu(), want) and torch.equal(rc.cpu(), want_rc), c
    # a direct capture
    static_count = torch.tensor(cases[0], device=device)
    m.allgatherv(x, static_count, recv_capacity=cap, comm=comm)       # staging sized before the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        g_out, g_rc = m.allgatherv(x, static_count, recv_capacity=cap, comm=comm)
    for c in cases:
        static_count.fill_(c)
        g.replay()
        want, want_rc = _oracle(x, static_count, cap)
        assert torch.equal(g_out.cpu(), want) and torch.equal(g_rc.cpu(), want_rc), c
    m.flush()


@peers
def test_allgatherv_derivatives(device):
    """vjp / backward: the rank-order fold of the kept cotangent rows (random fp32, bitwise); rows past
    the count and rows a receiver dropped get nothing from it.  jvp: allgatherv of the tangent.  Double
    backward: the adjoint of the adjoint is the forward."""
    n = 6
    gen = torch.Generator().manual_seed(7 + rank)
    for count, cap in ((4 - rank % 2, None), (n, 2 + 3 * rank), (-1 + 2 * rank, n + 1)):
        c = n * size if cap is None else cap
        counts = torch.tensor(count, device=device)
        x = torch.randn(n, 2, generator=gen).to(device)
        ct = torch.randn(c, 2, generator=gen).to(device)
        t = torch.randn(n, 2, generator=gen).to(device)

        def f(v):
            return m.allgatherv(v, counts, recv_capacity=cap, comm=comm)[0]

        res, pullback = vjp(f, x)
        assert torch.equal(res.cpu(), _oracle(x, counts, c)[0])
        (g,) = pullback(ct)
        want = _oracle_grad(ct, counts, n, c)
        assert torch.equal(g.cpu(), want), (count, cap)
        assert not g[min(max(count, 0), n):].any()     # rows never contributed get no gradient
        _, tan = jvp(f, (x,), (t,))
        assert torch.equal(tan.cpu(), _oracle(t, counts, c)[0])
        xr = x.clone().requires_grad_(True)
        ctr = ct.clone().requires_grad_(True)
        out, rc = m.allgatherv(xr, counts, recv_capacity=cap, comm=comm)
        assert not rc.requires_grad
        (gx,) = torch.autograd.grad((out * ctr).sum(), xr, create_graph=True)
        assert torch.equal(gx.detach().cpu(), want)
        (gct,) = torch.autograd.grad((gx * t).sum(), ctr)
        assert torch.equal(gct.cpu(), _oracle(t, counts, c)[0]), (count, cap)
        xr.grad = None
        (m.allgatherv(xr, counts, recv_capacity=cap, comm=comm)[0] * ct).sum().backward()
        assert torch.equal(xr.grad.cpu(), want)


@peers
def test_allgatherv_vmap(device):
    n = 5
    count = torch.tensor(2 + rank % 3, device=device)
    xb = (torch.arange(3 * n * 2, dtype=torch.float32).reshape(3, n, 2) + 100 * rank).to(device)
    want = torch.stack([m.allgatherv(xb[i], count, recv_capacity=4, comm=comm)[0] for i in range(3)])
    f = vmap(lambda v: m.allgatherv(v, count, recv_capacity=4, comm=comm)[0], in_dims=0, out_dims=0)
    assert torch.equal(f(xb), want)
    f1 = vmap(lambda v: m.allgatherv(v, count, recv_capacity=4, comm=comm)[0], in_dims=1, out_dims=0)
    assert torch.equal(f1(xb.movedim(0, 1).contiguous()), want)
    with pytest.raises(ValueError, match="count must not be batched"):
        vmap(lambda v, c: m.allgatherv(v, c, comm=comm)[0])(xb, count.expand(3).contiguous())


def test_allgatherv_fake_shape_and_effect():
    from torch._higher_order_ops.effects import _EffectType, _get_effect
    from torch._subclasses.fake_tensor import FakeTensorMode

    with FakeTensorMode():
        out, rc = m.compiled.allgatherv(torch.empty(4, 3, 2), torch.empty((), dtype=torch.int64),
                                        recv_capacity=7, comm=comm)
        assert out.shape == (7, 3, 2) and rc.shape == (size,) and rc.dtype == torch.int64
        assert rc.device == out.device
        out, _ = m.compiled.allgatherv(torch.empty(4, 3), torch.empty((), dtype=torch.int64), comm=comm)
        assert out.shape == (4 * size, 3)
    assert _get_effect("mpi4jax_b200::allgatherv") == _EffectType.ORDERED


def test_allgatherv_compiled_errors(device):
    """compiled.allgatherv, the raw torch.ops op and its fake kernel refuse what the eager op refuses, on
    the host: the kernel would otherwise dereference a count that is not one int64 in x's memory."""
    from torch._subclasses.fake_tensor import FakeTensorMode

    x = torch.ones((4, 2), device=device)
    other = "meta" if device.type == "cpu" else "cpu"
    good = torch.tensor(1, device=device)
    bad = [
        (ValueError, "must live on the device of x", x, torch.tensor(1, device=other), None),
        (ValueError, re.escape("must have shape ()"), x, torch.ones(1, dtype=torch.int64, device=device), None),
        (TypeError, "must be an integer tensor", x, torch.tensor(1.0, device=device), None),
        (ValueError, re.escape("recv_capacity must be >= 0"), x, good, -1),
        (ValueError, re.escape("input must have shape (rows, ...)"), torch.tensor(1.0, device=device), good, None),
    ]
    for exc, msg, xx, count, cap in bad:
        with pytest.raises(exc, match=msg):
            m.compiled.allgatherv(xx, count, recv_capacity=cap, comm=comm)
        with pytest.raises(exc, match=msg):
            torch.ops.mpi4jax_b200.allgatherv(xx, count, 4 if cap is None else cap, comm._id)
    with pytest.raises(TypeError, match="must be an integer tensor"):      # the op's schema takes a tensor
        m.compiled.allgatherv(x, 1, comm=comm)
    with FakeTensorMode():
        with pytest.raises(ValueError, match=re.escape("must have shape ()")):
            m.compiled.allgatherv(torch.empty(4, 2), torch.empty(2, dtype=torch.int64), comm=comm)
        with pytest.raises(ValueError, match=re.escape("must have shape ()")):
            torch.ops.mpi4jax_b200.allgatherv(torch.empty(4, 2), torch.empty(2, dtype=torch.int64), 4, comm._id)


@peers
def test_allgatherv_compiled_and_grad(device):
    n, cap = 6, 5 + rank
    count = torch.tensor(3 + rank, device=device)
    ct = torch.randn(cap, 2, generator=torch.Generator().manual_seed(rank)).to(device)
    f = torch.compile(lambda v, c: (m.compiled.allgatherv(v * 2, c, recv_capacity=cap, comm=comm)[0] * ct).sum(),
                      backend="aot_eager", fullgraph=True)
    x = (torch.arange(n * 2, dtype=torch.float32).reshape(n, 2) + rank).to(device).requires_grad_(True)
    y = f(x, count)
    assert y.item() == (_oracle(x.detach() * 2, count, cap)[0] * ct.cpu()).sum().item()
    y.backward()
    assert torch.equal(x.grad.cpu(), 2 * _oracle_grad(ct, count, n, cap))
    m.flush()


def test_host_staged_allgatherv(device, monkeypatch):
    from mpi4jax_b200._src.backends import host_staged

    monkeypatch.setattr(host_staged, "ACTIVE", host_staged.ACTIVE)      # restore the flag afterwards
    host_staged_comm = comm.Clone()
    hs = host_staged.HostStagedComm(host_staged_comm, "unit test")
    try:
        n = 5
        x = (torch.arange(n * 2, dtype=torch.float32).reshape(n, 2) + 10 * rank).to(device)
        count = torch.tensor((rank + 2) % 4, device=device)
        out, rc = hs.allgatherv(x, count, 4)
        want, want_rc = _oracle(x, count, 4)
        assert out.device == x.device and rc.device == x.device
        assert torch.equal(out.cpu(), want) and torch.equal(rc.cpu(), want_rc)
    finally:
        host_staged_comm.Free()


def test_staging_formula_allgatherv():
    from mpi4jax_b200._src import native
    from mpi4jax_b200._src.backends.cuda import stage_need

    if not native.HAS_CUDA_EXT:
        pytest.skip(f"native library not loaded: {native.CUDA_EXT_ERROR}")
    assert codes.OPC_ALLGATHERV == 15
    for nranks in range(1, 17):
        for nbytes in [0, 1, 15, 16, 17, 4095, 4096, 65537, (1 << 20) + 3, 1 << 30]:
            want = 128 + (nbytes + 15) // 16 * 16 + 4096
            assert stage_need(15, nranks, nbytes) == native.lib.b2_stage_need(15, nranks, nbytes) == want


def test_allgatherv_debug_log(device, capsys):
    from mpi4jax_b200._src.native import set_logging

    x = torch.ones((4, 3), device=device)
    count = torch.tensor(2, device=device)
    m.allgatherv(x, count, comm=comm)
    m.flush()
    capsys.readouterr()
    set_logging(True)
    try:
        m.allgatherv(x, count, comm=comm)
        m.flush()
    finally:
        set_logging(False)
    out = capsys.readouterr().out
    assert re.search(rf"^r{rank} \| \w{{8}} \| MPI_Allgatherv( \(\w+\))? with 4 rows of 12 bytes", out, re.M), out
    assert re.search(rf"^r{rank} \| \w{{8}} \| MPI_Allgatherv( \(\w+\))? done with code 0", out, re.M), out


_inside_job = size > 1 or "MPI4JAX_B200_NESTED" in os.environ


@pytest.mark.gpu
@pytest.mark.skipif(_inside_job, reason="already inside a multi-rank job")
def test_allgatherv_three_ranks_gpu():
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
        with tempfile.TemporaryDirectory(prefix="mpi4jax-b200-agv-job-") as logs:
            code, _ = launch(3, args, timeout=900, output_dir=logs, env_extra={"MPI4JAX_B200_NESTED": "1"})
            outs = [open(os.path.join(logs, f"rank{r}.log")).read() for r in range(3)]
    finally:
        os.chdir(cwd)
    for r, out in enumerate(outs):
        assert code == 0 and re.search(r"PASSED .*test_allgatherv_multi_chunk\[cuda\]", out), \
            f"rank {r} of the 3-rank job (exit code {code}):\n{out[-4000:]}"
