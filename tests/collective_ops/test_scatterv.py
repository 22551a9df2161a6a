"""scatterv: rank q receives a variable-length slice of the root's rows, ``(N, *S) -> (recv_capacity, *S)``.

Oracle: every rank gathers the root's input and send counts and every rank's capacity with the object API
and applies the documented rules (clamp the root's counts in rank order to its ``N`` rows, cut its rows
into one segment per rank, clip each to the receiver's capacity, zero the rest) in plain torch on the
CPU; results compare bitwise.  The gradient oracle places every rank's kept cotangent rows where they were
taken from on the root; the other ranks' templates get zeros.  The CUDA variants need peers: in a
single-process run they are checked in a two-rank job whose ranks share the GPU, and
``test_scatterv_three_ranks_gpu`` runs them with three ranks."""

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

peers = needs_peers("scatterv between ranks")


def _roots():
    """Every root at 3 ranks; 0 and the last one otherwise."""
    return list(range(size)) if size <= 3 else [0, size - 1]


def _clamped(counts, n):
    out, used = [], 0
    for c in counts:
        k = min(max(int(c), 0), n - used)
        out.append(k)
        used += k
    return out


def _plan(x, send_counts, root, cap):
    """(root's x, its clamped counts, displacements, every rank's capacity)."""
    mine = None
    if rank == root:
        mine = (x.detach().cpu().contiguous().reshape(-1).view(torch.uint8), tuple(x.shape),
                [int(c) for c in torch.as_tensor(send_counts).tolist()])
    everything = comm.allgather((mine, cap))
    raw, shape, counts = everything[root][0]
    s = _clamped(counts, shape[0])
    return raw.view(x.dtype).reshape(shape), s, [sum(s[:q]) for q in range(size)], [e[1] for e in everything]


def _oracle(x, send_counts, root, cap):
    """(out, recv_count) of this rank."""
    xr, s, d, _ = _plan(x, send_counts, root, cap)
    k = min(s[rank], cap)
    out = torch.zeros((cap, *x.shape[1:]), dtype=x.dtype)
    out[:k] = xr[d[rank]: d[rank] + k]
    return out, torch.tensor(k, dtype=torch.int64)


def _oracle_grad(ct, send_counts, root, n, cap):
    """Cotangent of x: on the root every rank's first k_q cotangent rows at d_q, zero elsewhere; zeros on
    the other ranks (their x is a template)."""
    _, s, d, caps = _plan(torch.zeros(n, *ct.shape[1:], dtype=ct.dtype), send_counts, root, cap)
    cts = comm.allgather(ct.detach().cpu())
    g = torch.zeros((n, *ct.shape[1:]), dtype=ct.dtype)
    if rank == root:
        for q in range(size):
            k = min(s[q], caps[q])
            g[d[q]: d[q] + k] = cts[q][:k]
    return g


def _check(x, send_counts, root, cap=None, template=True):
    """``template``: the other ranks pass ``torch.empty`` of x's shape and None for the counts."""
    if rank != root and template:
        x = torch.empty_like(x)
        send_counts = None
    _x = x.clone()
    _c = send_counts.clone() if isinstance(send_counts, torch.Tensor) else send_counts
    out, rc = m.scatterv(x, send_counts, root, recv_capacity=cap, comm=comm)
    cap = x.shape[0] if cap is None else cap
    want, want_rc = _oracle(x, send_counts, root, cap)
    assert out.shape == (cap, *x.shape[1:]) and out.dtype == x.dtype and out.device == x.device
    assert rc.dtype == torch.int64 and rc.shape == () and rc.device == x.device
    assert torch.equal(out.cpu(), want), (send_counts, root, cap)
    assert torch.equal(rc.cpu(), want_rc), (send_counts, root, cap)
    if rank == root:
        assert torch.equal(x, _x)
    if isinstance(send_counts, torch.Tensor):
        assert torch.equal(send_counts, _c)
    return out, rc


def _count_cases(n):
    """(send_counts, capacity) cases: the root's counts (read on the root only) and this rank's capacity."""
    P = size
    return [
        ([n // P] * P, None),                                    # an even split
        ([n] + [0] * (P - 1), None),                             # everything to rank 0
        ([0] * P, None),                                         # nothing at all
        ([q % 3 for q in range(P)], None),                       # below N, different per rank
        ([n + 5] * P, None),                                     # past N: rank 0 gets all, the others none
        ([-3 + q for q in range(P)], None),                      # negative
        ([3] * P, None),                                         # summing past N (P = 3)
        ([n // 2 + q for q in range(P)], 1 + rank),              # capacity below the segment, per rank
        ([2] * P, 0),                                            # capacity 0
        ([n - 1] + [1] * (P - 1), n + 4),                        # capacity > N
    ]


@peers
def test_scatterv_cases(device):
    n = 7
    x = (torch.arange(n * 3, dtype=torch.float32).reshape(n, 3) + 100 * rank).to(device)
    for root in _roots():
        for counts, cap in _count_cases(n):
            _check(x, torch.tensor(counts, device=device), root, cap)
    # a list of ints, int32 counts, and counts passed (and not read) on every rank
    counts = [2 + q for q in range(size)]
    out, _ = _check(x, counts, 0)
    assert torch.equal(out, _check(x, torch.tensor(counts, dtype=torch.int32, device=device), 0)[0])
    assert torch.equal(out, _check(x, torch.tensor([rank - 9] * size, device=device) if rank else
                                   torch.tensor(counts, device=device), 0, template=False)[0])
    # N = 0
    e = torch.empty((0, 3), device=device)
    out, rc = _check(e, torch.ones(size, dtype=torch.int64, device=device), size - 1, 4)
    assert rc.item() == 0 and not out.any()


@peers
def test_scatterv_odd_rows_and_noncontiguous(device):
    """Row sizes that are not multiples of 16 bytes, and a non-contiguous x on the root."""
    torch.manual_seed(5 + rank)
    for dtype, row in ((torch.int8, (3,)), (torch.int8, (5, 1)), (torch.float16, (7,)), (torch.float64, (3,))):
        x = (torch.randn(11, *row) * 50).to(dtype).to(device)
        for counts, cap in _count_cases(11):
            _check(x, torch.tensor(counts, device=device), size - 1, cap)
    base = torch.randn(4, 9, device=device)
    xt = base.t()                                                       # (9, 4), not contiguous
    assert not xt.is_contiguous()
    for root in _roots():
        _check(xt, torch.tensor([5 - q for q in range(size)], device=device), root, 4, template=False)


@peers
def test_scatterv_dtypes(device):
    for k, dtype in enumerate(codes.DTYPE_CODE):
        g = torch.Generator().manual_seed(10 * k + rank)
        v = torch.randint(0, 100, (9, 2), generator=g)
        x = (v % 2 == 0) if dtype == torch.bool else v.to(dtype)
        counts = torch.tensor([(k + q) % 5 for q in range(size)], device=device)
        _check(x.to(device), counts, k % size, 3 + rank)


@peers
def test_scatterv_multi_chunk(device):
    """4 MiB on the root: more chunks than CTAs, segments that start and end inside chunks."""
    n = 1024
    x = torch.randn(n, 1024, device=device, generator=torch.Generator(device).manual_seed(rank))   # 4 MiB
    root = size - 1
    _check(x, torch.tensor([n // size] * size, device=device), root)
    _check(x, torch.tensor([n // size - 37 * q - 1 for q in range(size)], device=device), 0)
    _check(x, torch.tensor([n * (q + 1) // (size * size) for q in range(size)], device=device), root)   # skewed
    _check(x, torch.tensor([n // 2 + 3 * q for q in range(size)], device=device), 0, n // 3 + rank)    # drops
    xo = torch.randn(n, 1023, device=device).to(torch.bfloat16)                  # 2046-byte rows
    _check(xo, torch.tensor([n - 1 - q for q in range(size)], device=device), root)


def test_scatterv_single_rank(device):
    """A one-rank communicator: the clamped rows, then zeros."""
    solo = comm.Split(rank, 0)
    try:
        x = torch.randn(5, 3, device=device)
        out, rc = m.scatterv(x, torch.tensor([3], device=device), 0, comm=solo)
        assert out.shape == (5, 3) and rc.item() == 3 and rc.shape == ()
        assert torch.equal(out[:3], x[:3]) and not out[3:].any()
        out, rc = m.scatterv(x, [9], 0, recv_capacity=2, comm=solo)
        assert torch.equal(out, x[:2]) and rc.item() == 2
    finally:
        m.flush()
        solo.Free()


def test_scatterv_errors(device, monkeypatch):
    x = torch.ones((4, 2), device=device)
    good = torch.ones(size, dtype=torch.int64, device=device)
    other = "meta" if device.type == "cpu" else "cpu"
    with pytest.raises(ValueError, match=re.escape("Scatterv input must have shape (rows, ...)")):
        m.scatterv(torch.tensor(1.0, device=device), good, 0, comm=comm)
    with pytest.raises(ValueError, match=re.escape("Scatterv send_counts must have shape (nproc,)")):
        m.scatterv(x, torch.ones(size + 1, dtype=torch.int64, device=device), 0, comm=comm)
    with pytest.raises(ValueError, match=re.escape("Scatterv send_counts must have shape (nproc,)")):
        m.scatterv(x, torch.tensor(1, device=device), 0, comm=comm)
    with pytest.raises(TypeError, match="Scatterv send_counts must be an integer tensor"):
        m.scatterv(x, good.float(), 0, comm=comm)
    with pytest.raises(TypeError, match="Scatterv send_counts must be an integer tensor"):
        m.scatterv(x, good.bool(), 0, comm=comm)
    with pytest.raises(TypeError):
        m.scatterv(x, [1.5] * size, 0, comm=comm)
    with pytest.raises(ValueError, match="Scatterv send_counts must live on the device of x"):
        m.scatterv(x, good.to(other), 0, comm=comm)
    with pytest.raises(ValueError, match=re.escape("Scatterv recv_capacity must be >= 0")):
        m.scatterv(x, good, 0, recv_capacity=-1, comm=comm)
    if rank == 0:
        with pytest.raises(ValueError, match="Scatterv send_counts must be given on the root"):
            m.scatterv(x, None, 0, comm=comm)
    else:
        with pytest.raises(ValueError, match=re.escape("Scatterv recv_capacity must be >= 0")):
            m.scatterv(x, None, 0, recv_capacity=-1, comm=comm)
    with pytest.raises(TypeError, match='unexpected type for argument "recv_capacity"'):
        m.scatterv(x, good, 0, recv_capacity=2.0, comm=comm)
    with pytest.raises(RuntimeError, match="Explicit token management"):
        m.scatterv(x, good, 0, comm=comm, token=1)
    monkeypatch.setenv("MPI4JAX_B200_ABORT_ON_ERROR", "0")
    with pytest.raises(MPI.MPIError, match=re.escape(f"MPI_Scatterv returned error code 4: invalid root rank -1")):
        m.scatterv(x, good, -1, comm=comm)


@peers
def test_scatterv_jit_and_graph_replays(device):
    """Captured once, replayed with the counts changed in place: oracle-exact every time."""
    if device.type != "cuda":
        pytest.skip("CUDA graphs")
    n, cap, root = 9, 4 + rank, size - 1
    x = torch.randn(n, 5, device=device, generator=torch.Generator(device).manual_seed(rank))
    counts = torch.zeros(size, dtype=torch.int64, device=device)
    f = m.jit(lambda t, c: m.scatterv(t * 2, c, root, recv_capacity=cap, comm=comm))
    cases = [c for c, _ in _count_cases(n)]
    for c in cases:                                     # eager warm-up, capture, replays
        counts.copy_(torch.tensor(c))
        out, rc = f(x, counts)
        want, want_rc = _oracle(x * 2, counts, root, cap)
        assert torch.equal(out.cpu(), want) and torch.equal(rc.cpu(), want_rc), c
    # a direct capture
    static_counts = torch.tensor(cases[0], device=device)
    m.scatterv(x, static_counts, 0, recv_capacity=cap, comm=comm)     # staging sized before the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        g_out, g_rc = m.scatterv(x, static_counts, 0, recv_capacity=cap, comm=comm)
    for c in cases:
        static_counts.copy_(torch.tensor(c))
        g.replay()
        want, want_rc = _oracle(x, static_counts, 0, cap)
        assert torch.equal(g_out.cpu(), want) and torch.equal(g_rc.cpu(), want_rc), c
    m.flush()


@peers
def test_scatterv_derivatives(device):
    """vjp / backward: each rank's kept cotangent rows land on the root where they came from (random fp32,
    bitwise), templates get zeros.  jvp: scatterv of the tangent.  Double backward: the adjoint of the
    adjoint (gatherv's reverse mode, whose adjoint is a scatterv again) is the forward, on every rank."""
    n = 6
    gen = torch.Generator().manual_seed(7 + rank)
    for root in _roots():
        for raw, cap in (([2, 3, 1], None), ([n, -1, 4], 2 + rank), ([1 + q for q in range(size)], n + 1)):
            counts = torch.tensor((raw * size)[:size], device=device)
            c = n if cap is None else cap
            x = torch.randn(n, 2, generator=gen).to(device)
            ct = torch.randn(c, 2, generator=gen).to(device)
            t = torch.randn(n, 2, generator=gen).to(device)

            def f(v):
                return m.scatterv(v, counts, root, recv_capacity=cap, comm=comm)[0]

            res, pullback = vjp(f, x)
            assert torch.equal(res.cpu(), _oracle(x, counts, root, c)[0])
            (g,) = pullback(ct)
            want = _oracle_grad(ct, counts, root, n, c)
            assert torch.equal(g.cpu(), want), (root, raw, cap)
            _, tan = jvp(f, (x,), (t,))
            assert torch.equal(tan.cpu(), _oracle(t, counts, root, c)[0])
            xr = x.clone().requires_grad_(True)
            ctr = ct.clone().requires_grad_(True)
            out, rc = m.scatterv(xr, counts, root, recv_capacity=cap, comm=comm)
            assert not rc.requires_grad
            (gx,) = torch.autograd.grad((out * ctr).sum(), xr, create_graph=True)
            assert torch.equal(gx.detach().cpu(), want)
            (gct,) = torch.autograd.grad((gx * t).sum(), ctr)
            assert torch.equal(gct.cpu(), _oracle(t, counts, root, c)[0]), (root, raw, cap)
            xr.grad = None
            (m.scatterv(xr, counts, root, recv_capacity=cap, comm=comm)[0] * ct).sum().backward()
            assert torch.equal(xr.grad.cpu(), want)


@peers
def test_scatterv_vmap(device):
    n = 5
    counts = torch.tensor([2 + q % 3 for q in range(size)], device=device)
    root = size - 1
    xb = (torch.arange(3 * n * 2, dtype=torch.float32).reshape(3, n, 2) + 100 * rank).to(device)
    want = torch.stack([m.scatterv(xb[i], counts, root, recv_capacity=4, comm=comm)[0] for i in range(3)])
    f = vmap(lambda v: m.scatterv(v, counts, root, recv_capacity=4, comm=comm)[0], in_dims=0, out_dims=0)
    assert torch.equal(f(xb), want)
    f1 = vmap(lambda v: m.scatterv(v, counts, root, recv_capacity=4, comm=comm)[0], in_dims=1, out_dims=0)
    assert torch.equal(f1(xb.movedim(0, 1).contiguous()), want)
    with pytest.raises(ValueError, match="counts must not be batched"):
        vmap(lambda v, c: m.scatterv(v, c, root, comm=comm)[0])(xb, counts.expand(3, size).contiguous())


def test_scatterv_fake_shape_and_effect():
    from torch._higher_order_ops.effects import _EffectType, _get_effect
    from torch._subclasses.fake_tensor import FakeTensorMode

    with FakeTensorMode():
        counts = torch.empty(size, dtype=torch.int64)
        out, rc = m.compiled.scatterv(torch.empty(4, 3, 2), counts, 0, recv_capacity=7, comm=comm)
        assert out.shape == (7, 3, 2) and rc.shape == () and rc.dtype == torch.int64
        assert rc.device == out.device
        out, _ = m.compiled.scatterv(torch.empty(4, 3), counts, 0, comm=comm)
        assert out.shape == (4, 3)
    assert _get_effect("mpi4jax_b200::scatterv") == _EffectType.ORDERED


def test_scatterv_compiled_errors(device):
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
            m.compiled.scatterv(xx, counts, 0, recv_capacity=cap, comm=comm)
        with pytest.raises(exc, match=msg):
            torch.ops.mpi4jax_b200.scatterv(xx, counts, 0, 4 if cap is None else cap, 4, comm._id)
    with FakeTensorMode():
        with pytest.raises(ValueError, match=re.escape("must have shape (nproc,)")):
            torch.ops.mpi4jax_b200.scatterv(torch.empty(4, 2), torch.empty(size + 1, dtype=torch.int64), 0, 4, 4,
                                            comm._id)
        if rank == 0:
            with pytest.raises(ValueError, match="send_counts must be given on the root"):
                torch.ops.mpi4jax_b200.scatterv(torch.empty(4, 2), None, 0, 4, 4, comm._id)


@peers
def test_scatterv_compiled_and_grad(device):
    """compiled.scatterv forward and gradient, bitwise equal to the eager op's, on every rank and root."""
    n = 6
    for root in _roots():
        cap = 2 + rank
        counts = torch.tensor([3 + q for q in range(size)], device=device)
        ct = torch.randn(cap, 2, generator=torch.Generator().manual_seed(rank)).to(device)

        def loss(F, v, c):
            return (F.scatterv(v * 2, c, root, recv_capacity=cap, comm=comm)[0] * ct).sum()

        f = torch.compile(lambda v, c: loss(m.compiled, v, c), backend="aot_eager", fullgraph=True)
        x = (torch.arange(n * 2, dtype=torch.float32).reshape(n, 2) + rank).to(device)
        xc, xe = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
        y, ye = f(xc, counts), loss(m, xe, counts)
        assert torch.equal(y, ye)
        y.backward()
        ye.backward()
        assert torch.equal(xc.grad, xe.grad)
        assert torch.equal(xc.grad.cpu(), 2 * _oracle_grad(ct, counts, root, n, cap))
    m.flush()


def test_host_staged_scatterv(device, monkeypatch):
    from mpi4jax_b200._src.backends import host_staged

    monkeypatch.setattr(host_staged, "ACTIVE", host_staged.ACTIVE)      # restore the flag afterwards
    host_staged_comm = comm.Clone()
    hs = host_staged.HostStagedComm(host_staged_comm, "unit test")
    try:
        n, root = 5, size - 1
        x = (torch.arange(n * 2, dtype=torch.float32).reshape(n, 2) + 10 * rank).to(device)
        counts = torch.tensor([(q + 2) % 4 for q in range(size)], device=device)
        out, rc = hs.scatterv(x, counts if rank == root else None, root, 3, n)
        want, want_rc = _oracle(x, counts, root, 3)
        assert out.device == x.device and rc.device == x.device
        assert torch.equal(out.cpu(), want) and torch.equal(rc.cpu(), want_rc)
    finally:
        host_staged_comm.Free()


def test_staging_formula_scatterv():
    from mpi4jax_b200._src import native
    from mpi4jax_b200._src.backends.cuda import stage_need

    if not native.HAS_CUDA_EXT:
        pytest.skip(f"native library not loaded: {native.CUDA_EXT_ERROR}")
    assert codes.OPC_SCATTERV == 18
    for nranks in range(1, 17):
        for nbytes in [0, 1, 15, 16, 17, 4095, 4096, 65537, (1 << 20) + 3, 1 << 30]:
            want = 128 + (nbytes + 15) // 16 * 16 + 4096
            assert stage_need(18, nranks, nbytes) == native.lib.b2_stage_need(18, nranks, nbytes) == want


def test_scatterv_debug_log(device, capsys):
    from mpi4jax_b200._src.native import set_logging

    x = torch.ones((4, 3), device=device)
    counts = torch.ones(size, dtype=torch.int64, device=device)
    m.scatterv(x, counts, 0, comm=comm)
    m.flush()
    capsys.readouterr()
    set_logging(True)
    try:
        m.scatterv(x, counts, 0, comm=comm)
        m.flush()
    finally:
        set_logging(False)
    out = capsys.readouterr().out
    assert re.search(rf"^r{rank} \| \w{{8}} \| MPI_Scatterv( \(\w+\))? with 4 rows of 12 bytes from root 0", out,
                     re.M), out
    assert re.search(rf"^r{rank} \| \w{{8}} \| MPI_Scatterv( \(\w+\))? done with code 0", out, re.M), out


_inside_job = size > 1 or "MPI4JAX_B200_NESTED" in os.environ


@pytest.mark.gpu
@pytest.mark.skipif(_inside_job, reason="already inside a multi-rank job")
def test_scatterv_three_ranks_gpu():
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
        with tempfile.TemporaryDirectory(prefix="mpi4jax-b200-sv-job-") as logs:
            code, _ = launch(3, args, timeout=900, output_dir=logs, env_extra={"MPI4JAX_B200_NESTED": "1"})
            outs = [open(os.path.join(logs, f"rank{r}.log")).read() for r in range(3)]
    finally:
        os.chdir(cwd)
    for r, out in enumerate(outs):
        assert code == 0 and re.search(r"PASSED .*test_scatterv_derivatives\[cuda\]", out), \
            f"rank {r} of the 3-rank job (exit code {code}):\n{out[-4000:]}"
