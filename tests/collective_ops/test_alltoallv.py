"""alltoallv: rows exchanged by device-resident counts, ``(N, *S) -> (recv_capacity, *S)``.

Oracle: every rank gathers all inputs and all send counts and applies the documented rules (clamp the
sends in rank order, pack the received segments in source order, clip them to the capacity, zero the
rest) in plain torch on the CPU; results compare bitwise.  The CUDA variants need peers: in a
single-process run they are checked in a two-rank job whose ranks share the GPU, and
``test_alltoallv_three_ranks_gpu`` runs them with three ranks."""

import os
import re
import tempfile

import pytest
import torch
from torch.func import jvp, vjp, vmap

import mpi4jax_b200 as m
from mpi4jax_b200 import MPI
from mpi4jax_b200._src.native import codes
from mpi4jax_b200.parallel import expert_combine, expert_dispatch

from .._peer_job import needs_peers

comm = MPI.COMM_WORLD
rank = comm.Get_rank()
size = comm.Get_size()

peers = needs_peers("alltoallv between ranks")


def _clamp(counts, n):
    out, used = [], 0
    for c in counts:
        k = min(max(int(c), 0), n - used)
        out.append(k)
        used += k
    return out


def _sent(send_counts, n):
    """s'[q][p] of every rank q (gathered)."""
    cs = m.allgather(send_counts.to(torch.int64), comm=comm).tolist()
    return [_clamp(cs[q], n) for q in range(size)]


def _oracle(x, send_counts, cap):
    """(out, recv_counts) of this rank, from everybody's x and counts."""
    xs = m.allgather(x.contiguous(), comm=comm).cpu()
    sp = _sent(send_counts, x.shape[0])
    out = torch.zeros((cap, *x.shape[1:]), dtype=x.dtype)
    recv, filled = [], 0
    for q in range(size):
        d = sum(sp[q][:rank])
        k = min(sp[q][rank], cap - filled)
        out[filled: filled + k] = xs[q, d: d + k]
        recv.append(k)
        filled += k
    return out, torch.tensor(recv, dtype=torch.int64)


def _oracle_grad(ct, send_counts, n, cap):
    """Cotangent of x: row i of x sent to q and kept at row e there gets ct_q[e]; dropped rows get 0.
    ``cap`` (this rank's capacity, the rows of ``ct``) may differ between ranks."""
    caps = m.allgather(torch.tensor([cap], device=ct.device), comm=comm).view(-1).tolist()
    padded = torch.zeros((max(caps), *ct.shape[1:]), dtype=ct.dtype, device=ct.device)
    padded[:cap] = ct
    cts = m.allgather(padded, comm=comm).cpu()
    sp = _sent(send_counts, n)
    g = torch.zeros((n, *ct.shape[1:]), dtype=ct.dtype)
    for q in range(size):
        filled = 0
        for p in range(size):
            k = min(sp[p][q], caps[q] - filled)
            if p == rank:
                d = sum(sp[rank][:q])
                g[d: d + k] = cts[q, filled: filled + k]
            filled += k
    return g


def _check(x, counts, cap=None):
    _x, _c = x.clone(), counts.clone()
    out, rc = m.alltoallv(x, counts, recv_capacity=cap, comm=comm)
    cap = x.shape[0] * size if cap is None else cap
    want, want_rc = _oracle(x, counts, cap)
    assert out.shape == (cap, *x.shape[1:]) and out.dtype == x.dtype and out.device == x.device
    assert rc.dtype == torch.int64 and rc.shape == (size,) and rc.device == x.device
    assert torch.equal(out.cpu(), want), (counts.tolist(), cap)
    assert torch.equal(rc.cpu(), want_rc), (counts.tolist(), cap)
    assert torch.equal(x, _x) and torch.equal(counts, _c)
    return out, rc


def _count_cases(n):
    """(send_counts, capacity) cases; the counts differ between ranks."""
    bal = [n // size] * size
    return [
        (bal, None),                                                  # balanced
        ([n if q == 0 else 0 for q in range(size)], None),            # everything to rank 0
        ([0] * size, None),                                           # nothing at all
        ([(rank + q) % 3 for q in range(size)], None),                # below N
        ([n - 1 + q for q in range(size)], None),                     # past N: clamped in rank order
        ([-2 if q % 2 == 0 else 3 for q in range(size)], None),       # negative counts send nothing
        ([n if q == 0 else 1 for q in range(size)], 2 + rank),        # capacity < incoming: drops
        (bal, n * size + 5),                                          # capacity > N * nproc
        ([n if q == size - 1 else 0 for q in range(size)], 0),        # capacity 0
    ]


@peers
def test_alltoallv_cases(device):
    n = 7
    x = (torch.arange(n * 3, dtype=torch.float32).reshape(n, 3) + 100 * rank).to(device)
    for counts, cap in _count_cases(n):
        _check(x, torch.tensor(counts, device=device), cap)
    # a list of ints is accepted; int32 counts too
    out, rc = m.alltoallv(x, [1] * size, comm=comm)
    assert torch.equal(out, _check(x, torch.ones(size, dtype=torch.int32, device=device))[0])
    # N = 0
    e = torch.empty((0, 3), device=device)
    out, rc = _check(e, torch.tensor([1] * size, device=device), 4)
    assert out.shape == (4, 3) and rc.tolist() == [0] * size


@peers
def test_alltoallv_odd_rows_and_noncontiguous(device):
    """Row sizes that are not multiples of 16 bytes, and a non-contiguous x."""
    torch.manual_seed(5 + rank)
    for dtype, row in ((torch.int8, (3,)), (torch.int8, (5, 1)), (torch.float16, (7,)), (torch.float64, (3,))):
        x = (torch.randn(11, *row) * 50).to(dtype).to(device)
        for counts, cap in _count_cases(11):
            _check(x, torch.tensor(counts, device=device), cap)
    base = torch.randn(4, 9, device=device)
    xt = base.t()                                                       # (9, 4), not contiguous
    assert not xt.is_contiguous()
    _check(xt, torch.tensor([(q + rank) % 4 for q in range(size)], device=device), 6)


@peers
def test_alltoallv_dtypes(device):
    for k, dtype in enumerate(codes.DTYPE_CODE):
        g = torch.Generator().manual_seed(10 * k + rank)
        v = torch.randint(0, 100, (6, 2), generator=g)
        x = (v % 2 == 0) if dtype == torch.bool else v.to(dtype)
        _check(x.to(device), torch.tensor([(q + k + rank) % 4 for q in range(size)], device=device), 5)


@peers
def test_alltoallv_multi_chunk(device):
    """A few MiB per rank: more chunks than CTAs, segments that start and end inside chunks."""
    n = 1024
    x = torch.randn(n, 1024, device=device, generator=torch.Generator(device).manual_seed(rank))   # 4 MiB
    skew = [n // 2 + 3 if q == rank else (n // 2) // max(size - 1, 1) for q in range(size)]
    _check(x, torch.tensor(skew, device=device))
    _check(x, torch.tensor([n // size + 1] * size, device=device), n)       # drops at the receivers
    xo = torch.randn(n, 1023, device=device).to(torch.bfloat16)            # 2046-byte rows
    _check(xo, torch.tensor([n // size - 1] * size, device=device))


def test_alltoallv_single_rank(device):
    """A one-rank communicator: the clamped rows to rank 0, in order, then zeros."""
    solo = comm.Split(rank, 0)
    try:
        x = torch.randn(5, 3, device=device)
        out, rc = m.alltoallv(x, torch.tensor([3], device=device), comm=solo)
        assert out.shape == (5, 3) and rc.tolist() == [3]
        assert torch.equal(out[:3], x[:3]) and not out[3:].any()
        out, rc = m.alltoallv(x, [9], recv_capacity=2, comm=solo)
        assert torch.equal(out, x[:2]) and rc.tolist() == [2]
    finally:
        m.flush()
        solo.Free()


def test_alltoallv_errors(device):
    x = torch.ones((4, 2), device=device)
    good = torch.zeros(size, dtype=torch.int64, device=device)
    with pytest.raises(ValueError, match=re.escape("Alltoallv input must have shape (rows, ...)")):
        m.alltoallv(torch.tensor(1.0, device=device), good, comm=comm)
    with pytest.raises(ValueError, match=re.escape("Alltoallv send_counts must have shape (nproc,)")):
        m.alltoallv(x, torch.zeros(size + 1, dtype=torch.int64, device=device), comm=comm)
    with pytest.raises(ValueError, match=re.escape("Alltoallv send_counts must have shape (nproc,)")):
        m.alltoallv(x, torch.zeros(1, size, dtype=torch.int64, device=device), comm=comm)
    with pytest.raises(TypeError, match="Alltoallv send_counts must be an integer tensor"):
        m.alltoallv(x, torch.zeros(size, device=device), comm=comm)
    with pytest.raises(TypeError, match="Alltoallv send_counts must be an integer tensor"):
        m.alltoallv(x, torch.zeros(size, dtype=torch.bool, device=device), comm=comm)
    with pytest.raises(ValueError, match="Alltoallv send_counts must live on the device of x"):
        m.alltoallv(x, torch.zeros(size, dtype=torch.int64, device="meta"), comm=comm)
    with pytest.raises(ValueError, match=re.escape("Alltoallv recv_capacity must be >= 0")):
        m.alltoallv(x, good, recv_capacity=-1, comm=comm)
    with pytest.raises(TypeError, match='unexpected type for argument "recv_capacity"'):
        m.alltoallv(x, good, recv_capacity=2.0, comm=comm)
    with pytest.raises(RuntimeError, match="Explicit token management"):
        m.alltoallv(x, good, comm=comm, token=1)


@peers
def test_alltoallv_jit_and_graph_replays(device):
    """Captured once, replayed with counts changed in place: oracle-exact every time (the counts are
    read on the device; a host read of them could not be captured)."""
    if device.type != "cuda":
        pytest.skip("CUDA graphs")
    n = 9
    x = torch.randn(n, 5, device=device, generator=torch.Generator(device).manual_seed(rank))
    counts = torch.zeros(size, dtype=torch.int64, device=device)
    f = m.jit(lambda t, c: m.alltoallv(t * 2, c, recv_capacity=n, comm=comm))
    cases = [c for c, _ in _count_cases(n)]
    for c in cases:                                     # eager warm-up, capture, replays
        counts.copy_(torch.tensor(c))
        out, rc = f(x, counts)
        want, want_rc = _oracle(x * 2, counts, n)
        assert torch.equal(out.cpu(), want) and torch.equal(rc.cpu(), want_rc), c
    # a direct capture
    static_counts = torch.tensor(cases[0], device=device)
    m.alltoallv(x, static_counts, recv_capacity=n, comm=comm)          # staging sized before the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        g_out, g_rc = m.alltoallv(x, static_counts, recv_capacity=n, comm=comm)
    for c in cases:
        static_counts.copy_(torch.tensor(c))
        g.replay()
        want, want_rc = _oracle(x, static_counts, n)
        assert torch.equal(g_out.cpu(), want) and torch.equal(g_rc.cpu(), want_rc), c
    m.flush()


@peers
def test_alltoallv_derivatives(device):
    n, cap = 6, 5                                       # every rank sends 2 rows to rank 0: drops there
    counts = torch.tensor([2 + rank if q == 0 else 1 for q in range(size)], device=device)
    x = (torch.arange(n * 2, dtype=torch.float32).reshape(n, 2) + 10 * rank).to(device)
    ct = (torch.arange(cap * 2, dtype=torch.float32).reshape(cap, 2) * (rank + 1) + 1).to(device)
    t = torch.randn(n, 2, device=device, generator=torch.Generator(device).manual_seed(rank))

    def f(v):
        return m.alltoallv(v, counts, recv_capacity=cap, comm=comm)[0]

    res, pullback = vjp(f, x)
    assert torch.equal(res.cpu(), _oracle(x, counts, cap)[0])
    (g,) = pullback(ct)
    want = _oracle_grad(ct, counts, n, cap)
    assert torch.equal(g.cpu(), want)
    _, tan = jvp(f, (x,), (t,))
    assert torch.equal(tan.cpu(), _oracle(t, counts, cap)[0])
    xr = x.clone().requires_grad_(True)
    out, rc = m.alltoallv(xr, counts, recv_capacity=cap, comm=comm)
    assert not rc.requires_grad
    (out * ct).sum().backward()
    assert torch.equal(xr.grad.cpu(), want)
    sent = sum(_clamp(counts.tolist(), n))
    assert not xr.grad[sent:].any()                    # rows never sent get no gradient


@peers
def test_alltoallv_derivatives_clamped_counts_and_rank_capacities(device):
    """The adjoint where the clamps matter: capacities that differ between ranks (drops everywhere), a
    negative count, and counts that run past N (the reverse mode re-applies the rank-order clamp to the
    raw send counts it gets as place counts)."""
    n = 6
    cap = 2 + rank
    x = (torch.arange(n * 3, dtype=torch.float32).reshape(n, 3) + 10 * rank).to(device)
    ct = (torch.arange(cap * 3, dtype=torch.float32).reshape(cap, 3) * (rank + 1) + 1).to(device)
    for first in (-1, 2):                              # [-1, n, n, ...] and [2, n, n, ...]: the sum passes N
        counts = torch.tensor([first] + [n] * (size - 1), device=device)
        res, pullback = vjp(lambda v: m.alltoallv(v, counts, recv_capacity=cap, comm=comm)[0], x)
        assert torch.equal(res.cpu(), _oracle(x, counts, cap)[0]), first
        (g,) = pullback(ct)
        assert torch.equal(g.cpu(), _oracle_grad(ct, counts, n, cap)), first
        xr = x.clone().requires_grad_(True)
        (m.alltoallv(xr, counts, recv_capacity=cap, comm=comm)[0] * ct).sum().backward()
        assert torch.equal(xr.grad.cpu(), _oracle_grad(ct, counts, n, cap)), first


@peers
def test_alltoallv_vmap(device):
    n = 5
    counts = torch.tensor([(q + rank) % 3 for q in range(size)], device=device)
    xb = (torch.arange(3 * n * 2, dtype=torch.float32).reshape(3, n, 2) + 100 * rank).to(device)
    want = torch.stack([m.alltoallv(xb[i], counts, recv_capacity=4, comm=comm)[0] for i in range(3)])
    f = vmap(lambda v: m.alltoallv(v, counts, recv_capacity=4, comm=comm)[0], in_dims=0, out_dims=0)
    assert torch.equal(f(xb), want)
    f1 = vmap(lambda v: m.alltoallv(v, counts, recv_capacity=4, comm=comm)[0], in_dims=1, out_dims=0)
    assert torch.equal(f1(xb.movedim(0, 1).contiguous()), want)
    with pytest.raises(ValueError, match="counts must not be batched"):
        vmap(lambda v, c: m.alltoallv(v, c, comm=comm)[0])(xb, counts.expand(3, size).contiguous())


def test_alltoallv_fake_shape_and_effect():
    from torch._higher_order_ops.effects import _EffectType, _get_effect
    from torch._subclasses.fake_tensor import FakeTensorMode

    with FakeTensorMode():
        out, rc = m.compiled.alltoallv(torch.empty(4, 3, 2), torch.empty(size, dtype=torch.int64),
                                       recv_capacity=7, comm=comm)
        assert out.shape == (7, 3, 2) and rc.shape == (size,) and rc.dtype == torch.int64
        assert rc.device == out.device
        out, _ = m.compiled.alltoallv(torch.empty(4, 3), torch.empty(size, dtype=torch.int64), comm=comm)
        assert out.shape == (4 * size, 3)
    assert _get_effect("mpi4jax_b200::alltoallv") == _EffectType.ORDERED


def test_alltoallv_compiled_errors(device):
    """compiled.alltoallv and the raw torch.ops op refuse what the eager op refuses, on the host: the
    kernel would otherwise dereference counts that are not nproc int64 values in x's memory."""
    from torch._subclasses.fake_tensor import FakeTensorMode

    x = torch.ones((4, 2), device=device)
    other = "meta" if device.type == "cpu" else "cpu"
    bad = [
        (ValueError, "must live on the device of x", torch.zeros(size, dtype=torch.int64, device=other), None),
        (ValueError, re.escape("must have shape (nproc,)"), torch.zeros(size + 1, dtype=torch.int64, device=device), None),
        (TypeError, "must be an integer tensor", torch.zeros(size, device=device), None),
        (ValueError, re.escape("recv_capacity must be >= 0"), torch.zeros(size, dtype=torch.int64, device=device), -1),
    ]
    for exc, msg, counts, cap in bad:
        with pytest.raises(exc, match=msg):
            m.compiled.alltoallv(x, counts, recv_capacity=cap, comm=comm)
        with pytest.raises(exc, match=msg):
            torch.ops.mpi4jax_b200.alltoallv(x, counts, 4 if cap is None else cap, None, comm._id)
    with FakeTensorMode():
        with pytest.raises(ValueError, match=re.escape("must have shape (nproc,)")):
            m.compiled.alltoallv(torch.empty(4, 2), torch.empty(size + 1, dtype=torch.int64), comm=comm)


@peers
def test_alltoallv_compiled_and_grad(device):
    n, cap = 6, 5
    counts = torch.tensor([2 + rank if q == 0 else 1 for q in range(size)], device=device)
    ct = (torch.arange(cap * 2, dtype=torch.float32).reshape(cap, 2) + rank).to(device)
    f = torch.compile(lambda v, c: (m.compiled.alltoallv(v * 2, c, recv_capacity=cap, comm=comm)[0] * ct).sum(),
                      backend="aot_eager", fullgraph=True)
    x = (torch.arange(n * 2, dtype=torch.float32).reshape(n, 2) + rank).to(device).requires_grad_(True)
    y = f(x, counts)
    assert y.item() == (_oracle(x.detach() * 2, counts, cap)[0] * ct.cpu()).sum().item()
    y.backward()
    assert torch.equal(x.grad.cpu(), 2 * _oracle_grad(ct, counts, n, cap))
    m.flush()


def test_host_staged_alltoallv(device, monkeypatch):
    from mpi4jax_b200._src.backends import host_staged

    monkeypatch.setattr(host_staged, "ACTIVE", host_staged.ACTIVE)      # restore the flag afterwards
    host_staged_comm = comm.Clone()
    hs = host_staged.HostStagedComm(host_staged_comm, "unit test")
    try:
        n = 5
        x = (torch.arange(n * 2, dtype=torch.float32).reshape(n, 2) + 10 * rank).to(device)
        counts = torch.tensor([(q + rank) % 3 for q in range(size)], device=device)
        out, rc = hs.alltoallv(x, counts, 4)
        want, want_rc = _oracle(x, counts, 4)
        assert out.device == x.device and rc.device == x.device
        assert torch.equal(out.cpu(), want) and torch.equal(rc.cpu(), want_rc)
    finally:
        host_staged_comm.Free()


def test_staging_formula_alltoallv():
    from mpi4jax_b200._src import native
    from mpi4jax_b200._src.backends.cuda import stage_need

    if not native.HAS_CUDA_EXT:
        pytest.skip(f"native library not loaded: {native.CUDA_EXT_ERROR}")
    assert codes.OPC_ALLTOALLV == 14
    for nranks in range(1, 17):
        for nbytes in [0, 1, 15, 16, 17, 4095, 4096, 65537, (1 << 20) + 3, 1 << 30]:
            want = 128 + (nbytes + 15) // 16 * 16 + 4096
            assert stage_need(14, nranks, nbytes) == native.lib.b2_stage_need(14, nranks, nbytes) == want


def test_alltoallv_debug_log(device, capsys):
    from mpi4jax_b200._src.native import set_logging

    x = torch.ones((4, 3), device=device)
    counts = torch.ones(size, dtype=torch.int64, device=device)
    m.alltoallv(x, counts, comm=comm)
    m.flush()
    capsys.readouterr()
    set_logging(True)
    try:
        m.alltoallv(x, counts, comm=comm)
        m.flush()
    finally:
        set_logging(False)
    out = capsys.readouterr().out
    assert re.search(rf"^r{rank} \| \w{{8}} \| MPI_Alltoallv( \(\w+\))? with 4 rows of 12 bytes", out, re.M), out
    assert re.search(rf"^r{rank} \| \w{{8}} \| MPI_Alltoallv( \(\w+\))? done with code 0", out, re.M), out


@peers
def test_expert_dispatch_combine(device):
    """combine(dispatch(x)) is x for the tokens that were kept and zero for dropped ones (and for tokens
    whose destination is not a rank); the gradient flows back the same way."""
    n, hidden = 12, 4
    g = torch.Generator().manual_seed(3 + rank)
    dest = torch.randint(-1, size + 1, (n,), generator=g).to(device)          # includes invalid ranks
    x = torch.randn(n, hidden, generator=g).to(device)
    for cap in (None, 3):
        rows, rc, plan = expert_dispatch(x, dest, capacity=cap, comm=comm)
        back = expert_combine(rows * 2, plan)
        # oracle: which tokens did the receivers keep?
        valid = (dest >= 0) & (dest < size)
        order = torch.argsort(torch.where(valid, dest, size), stable=True).cpu()
        counts = [int((dest == q).sum()) for q in range(size)]
        _, kept_rc = _oracle(x[order.to(device)], torch.tensor(counts, device=device),
                             n * size if cap is None else cap)
        sent_back = m.alltoall(kept_rc.view(size, 1).to(device), comm=comm).view(size).cpu()  # rows kept per dest
        keep = torch.zeros(n, dtype=torch.bool)
        start = 0
        for q in range(size):
            keep[order[start: start + int(sent_back[q])]] = True
            start += counts[q]
        want = torch.where(keep.view(n, 1), x.cpu() * 2, torch.zeros(()))
        assert torch.equal(back.cpu(), want), cap
        assert torch.equal(rc.cpu(), kept_rc)
        xr = x.clone().requires_grad_(True)
        rows, _, plan = expert_dispatch(xr, dest, capacity=cap, comm=comm)
        (expert_combine(rows * 3, plan) * x).sum().backward()
        assert torch.equal(xr.grad.cpu(), torch.where(keep.view(n, 1), 3 * x.cpu(), torch.zeros(()))), cap


_inside_job = size > 1 or "MPI4JAX_B200_NESTED" in os.environ


@pytest.mark.gpu
@pytest.mark.skipif(_inside_job, reason="already inside a multi-rank job")
def test_alltoallv_three_ranks_gpu():
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
        with tempfile.TemporaryDirectory(prefix="mpi4jax-b200-a2av-job-") as logs:
            code, _ = launch(3, args, timeout=900, output_dir=logs, env_extra={"MPI4JAX_B200_NESTED": "1"})
            outs = [open(os.path.join(logs, f"rank{r}.log")).read() for r in range(3)]
    finally:
        os.chdir(cwd)
    for r, out in enumerate(outs):
        assert code == 0 and re.search(r"PASSED .*test_alltoallv_multi_chunk\[cuda\]", out), \
            f"rank {r} of the 3-rank job (exit code {code}):\n{out[-4000:]}"
