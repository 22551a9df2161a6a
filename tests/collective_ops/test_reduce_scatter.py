"""reduce_scatter: rank r receives op over ranks q of x_q[r], ``(nproc, *S) -> S``.

Oracle: every rank gathers all inputs and folds its own block in rank order with the CPU backend's
``reduce_stack`` (fp32 accumulation for f16/bf16, as the device kernels do), so results compare
bitwise.  The CUDA variants need peers: in a single-process run they are checked in a two-rank job
whose ranks share the GPU, and ``test_reduce_scatter_three_ranks_gpu`` runs them with three ranks."""

import os
import re
import tempfile

import pytest
import torch
from torch.func import jvp, vjp, vmap

import mpi4jax_b200 as m
from mpi4jax_b200 import MPI
from mpi4jax_b200._src.backends.cpu import reduce_stack
from mpi4jax_b200._src.native import codes

from .._peer_job import needs_peers

comm = MPI.COMM_WORLD
rank = comm.Get_rank()
size = comm.Get_size()

peers = needs_peers("reduce-scatter between ranks")

OPS = ("SUM", "PROD", "MIN", "MAX", "LAND", "LOR", "LXOR", "BAND", "BOR", "BXOR")


_WIDE_UINT = (torch.uint16, torch.uint32, torch.uint64)     # CPU torch lacks arithmetic on these


def _oracle(x, opname, on_cpu=False):
    stack = m.allgather(x, comm=comm)[:, rank]
    if on_cpu:
        stack = stack.cpu()
        if stack.dtype in _WIDE_UINT:      # small non-negative integers: exact in int64 for every op
            return reduce_stack(stack.to(torch.int64), getattr(codes, opname)).to(stack.dtype)
    return reduce_stack(stack, getattr(codes, opname))


def _integer_valued(shape, dtype, device, seed):
    """Small integers (and their bool / complex images): every op of every dtype is exact on them."""
    g = torch.Generator().manual_seed(seed)
    v = torch.randint(0, 4, shape, generator=g) + 1
    if dtype == torch.bool:
        t = v % 2 == 0
    elif dtype.is_complex:
        t = torch.complex(v.double(), (v % 3).double()).to(dtype)
    else:
        t = v.to(dtype)
    return t.to(device)


@peers
def test_reduce_scatter(device):
    x = torch.arange(size * 6, dtype=torch.float32, device=device).reshape(size, 3, 2) + rank
    _x = x.clone()
    res = m.reduce_scatter(x, MPI.SUM, comm=comm)
    want = torch.arange(rank * 6, rank * 6 + 6, dtype=torch.float32, device=device).reshape(3, 2) * size
    want += sum(range(size))
    assert res.shape == (3, 2) and res.dtype == x.dtype and res.device == x.device
    assert torch.equal(res, want)
    assert torch.equal(x, _x)
    # x of shape (nproc,): a 0-dim result
    v = torch.arange(size, dtype=torch.int64, device=device) * 10 + rank
    r0 = m.reduce_scatter(v, MPI.SUM, comm=comm)
    assert r0.shape == () and r0.item() == 10 * rank * size + sum(range(size))
    # an empty block
    e = m.reduce_scatter(torch.empty((size, 0, 4), device=device), MPI.SUM, comm=comm)
    assert e.shape == (0, 4)


def test_reduce_scatter_wrong_shape(device):
    with pytest.raises(ValueError, match=re.escape("Reduce_scatter input must have shape (nproc, ...)")):
        m.reduce_scatter(torch.ones((size + 1, 2), device=device), MPI.SUM, comm=comm)
    with pytest.raises(ValueError, match=re.escape("Reduce_scatter input must have shape (nproc, ...)")):
        m.reduce_scatter(torch.tensor(1.0, device=device), MPI.SUM, comm=comm)


def test_reduce_scatter_single_rank_is_a_copy(device):
    """A one-rank communicator returns x[0] (through the same entry point)."""
    solo = comm.Split(rank, 0)
    try:
        x = torch.randn(1, 37, device=device)
        out = m.reduce_scatter(x, MPI.PROD, comm=solo)
        assert torch.equal(out, x[0]) and out.data_ptr() != x.data_ptr()
    finally:
        m.flush()
        solo.Free()


@peers
def test_reduce_scatter_dtypes_and_ops(device):
    """Every dtype x op: valid combinations equal the oracle bitwise, invalid ones raise what
    allreduce raises."""
    for k, dtype in enumerate(codes.DTYPE_CODE):
        x = _integer_valued((size, 5), dtype, device, seed=100 * k + rank)
        for opname in OPS:
            op = getattr(MPI, opname)
            try:
                m.allreduce(x[0], op, comm=comm)
                expected_error = None
            except NotImplementedError as exc:
                expected_error = exc
            if expected_error is not None:
                with pytest.raises(type(expected_error), match=re.escape(str(expected_error))):
                    m.reduce_scatter(x, op, comm=comm)
                continue
            res = m.reduce_scatter(x, op, comm=comm)
            assert res.dtype == dtype and res.shape == (5,), (dtype, opname)
            assert torch.equal(res.cpu(), _oracle(x, opname, on_cpu=True)), (dtype, opname)


@peers
def test_reduce_scatter_odd_sizes(device):
    """Block byte lengths that are not multiples of 16, and a non-contiguous input."""
    torch.manual_seed(7 + rank)
    for dtype in (torch.int8, torch.float16, torch.float32):
        for n in (1, 3, 15, 17, 4095):
            if dtype == torch.int8:
                x = torch.randint(-100, 100, (size, n), dtype=dtype, device=device)
            else:
                x = torch.randn(size, n, device=device).to(dtype)
            for opname in ("SUM", "MAX"):
                res = m.reduce_scatter(x, getattr(MPI, opname), comm=comm)
                assert torch.equal(res, _oracle(x, opname)), (dtype, n, opname)
    base = torch.randn(33, size, device=device)
    xt = base.t()                                  # (size, 33), not contiguous
    assert not xt.is_contiguous()
    assert torch.equal(m.reduce_scatter(xt, MPI.SUM, comm=comm), m.reduce_scatter(xt.contiguous(), MPI.SUM, comm=comm))


@peers
def test_reduce_scatter_transports(device):
    """Both GPU transports (LL: ll_max high; pull through the staging: ll_max = 0) at a block near the
    LL limit and at a multi-chunk block of a few MiB.  Both equal the oracle and the one-shot allreduce's
    own block, bitwise; the communicator's option is restored afterwards."""
    nc = comm._native_comm() if device.type == "cuda" else None
    ll_max0 = nc.get_option("ll_max") if nc is not None else None
    torch.manual_seed(11 + rank)
    blocks = (16384, (1 << 20) + 3)               # 64 KiB = half the default LL buffer; ~4 MiB
    try:
        for ll_max in (1 << 30, 0):
            if nc is not None:
                nc.set_option("ll_max", ll_max)
            for n in blocks:
                x = torch.randn(size, n, device=device)
                res = m.reduce_scatter(x, MPI.SUM, comm=comm)
                assert torch.equal(res, _oracle(x, "SUM")), (ll_max, n)
                ar = m.allreduce(x, MPI.SUM, comm=comm, algorithm="oneshot")[rank]
                assert torch.equal(res, ar), (ll_max, n)
                xb = torch.randn(size, n // 7 + 1, device=device).to(torch.bfloat16)
                assert torch.equal(m.reduce_scatter(xb, MPI.SUM, comm=comm), _oracle(xb, "SUM")), (ll_max, n)
    finally:
        m.flush()
        if nc is not None:
            nc.set_option("ll_max", ll_max0)
    if nc is not None:
        assert nc.get_option("ll_max") == ll_max0


@peers
def test_reduce_scatter_jit(device):
    x = torch.randn(size, 40, device=device, generator=torch.Generator(device).manual_seed(rank))
    f = m.jit(lambda t: m.reduce_scatter(t * 2, MPI.SUM, comm=comm))
    want = m.reduce_scatter(x * 2, MPI.SUM, comm=comm)
    for _ in range(3):                             # eager warm-up, capture, replay
        assert torch.equal(f(x), want)


@peers
def test_reduce_scatter_vmap(device):
    xb = torch.arange(4 * size * 3, dtype=torch.float32, device=device).reshape(4, size, 3) + rank
    want = torch.stack([m.reduce_scatter(xb[i], MPI.SUM, comm=comm) for i in range(4)])
    f = vmap(lambda t: m.reduce_scatter(t, MPI.SUM, comm=comm), in_dims=0, out_dims=0)
    assert torch.equal(f(xb), want)
    x1 = xb.movedim(0, 1).contiguous()             # (size, 4, 3), batch dimension at 1
    f1 = vmap(lambda t: m.reduce_scatter(t, MPI.SUM, comm=comm), in_dims=1, out_dims=0)
    assert torch.equal(f1(x1), want)


@peers
def test_reduce_scatter_derivatives(device):
    x = torch.arange(size * 3, dtype=torch.float32, device=device).reshape(size, 3) + rank
    ct = torch.arange(3, dtype=torch.float32, device=device) * (rank + 1)
    t = torch.ones(size, 3, device=device) * (rank + 2)

    def f(v):
        return m.reduce_scatter(v, MPI.SUM, comm=comm)

    res, pullback = vjp(f, x)
    assert torch.equal(res, m.reduce_scatter(x, MPI.SUM, comm=comm))
    (g,) = pullback(ct)
    assert torch.equal(g, m.allgather(ct, comm=comm))
    res, tan = jvp(f, (x,), (t,))
    assert torch.equal(tan, m.reduce_scatter(t, MPI.SUM, comm=comm))
    (lt,) = m.linear_transpose(f, x)(ct)
    assert torch.equal(lt, m.allgather(ct, comm=comm))
    # classic autograd
    xr = x.clone().requires_grad_(True)
    (f(xr) * ct).sum().backward()
    assert torch.equal(xr.grad, m.allgather(ct, comm=comm))
    # non-SUM derivatives are not defined
    xm = x.clone().requires_grad_(True)
    with pytest.raises(NotImplementedError, match="adjoint of reduce_scatter for MAX"):
        m.reduce_scatter(xm, MPI.MAX, comm=comm).sum().backward()
    with pytest.raises(NotImplementedError, match="derivative of reduce_scatter for MIN"):
        jvp(lambda v: m.reduce_scatter(v, MPI.MIN, comm=comm), (x,), (t,))


@peers
def test_reduce_scatter_user_op(device):
    """MPI.Op.Create: a non-commutative 2x2 matrix product of every rank's block, folded in rank order."""
    matmul = MPI.Op.Create(lambda a, b: a @ b, commute=False)
    # block q of rank r: shear by (r + 1) * (q + 1)
    x = torch.stack([torch.tensor([[1.0, float((rank + 1) * (q + 1))], [0.0, 1.0]]) for q in range(size)])
    res = m.reduce_scatter(x.to(device), matmul, comm=comm)
    want = torch.tensor([[1.0, float((rank + 1) * size * (size + 1) // 2)], [0.0, 1.0]], device=device)
    assert torch.equal(res, want)
    parts = [torch.tensor([[1.0, float((q + 1) * (rank + 1))], [0.0, 1.0]]) for q in range(size)]
    fold = parts[0]
    for p in parts[1:]:
        fold = fold @ p
    assert torch.equal(res.cpu(), fold)


def test_reduce_scatter_fake_shape():
    from torch._subclasses.fake_tensor import FakeTensorMode

    with FakeTensorMode():
        assert m.compiled.reduce_scatter(torch.empty(size, 3, 2), MPI.SUM, comm=comm).shape == (3, 2)


def test_reduce_scatter_is_effectful():
    from torch._higher_order_ops.effects import _EffectType, _get_effect

    assert _get_effect("mpi4jax_b200::reduce_scatter") == _EffectType.ORDERED


@peers
def test_reduce_scatter_compiled_and_grad(device):
    w = torch.arange(1, 4, dtype=torch.float32, device=device)
    f = torch.compile(lambda v: (m.compiled.reduce_scatter(v * 2, MPI.SUM, comm=comm) * w).sum(),
                      backend="aot_eager", fullgraph=True)
    x = (torch.arange(size * 3, dtype=torch.float32, device=device).reshape(size, 3) + rank).requires_grad_(True)
    y = f(x)
    assert y.item() == (m.reduce_scatter(x.detach() * 2, MPI.SUM, comm=comm) * w).sum().item()
    y.backward()
    assert torch.equal(x.grad, (2 * w).expand(size, 3))
    m.flush()


def test_host_staged_reduce_scatter(device, monkeypatch):
    from mpi4jax_b200._src.backends import host_staged

    monkeypatch.setattr(host_staged, "ACTIVE", host_staged.ACTIVE)      # restore the flag afterwards
    hs = host_staged.HostStagedComm(comm.Clone(), "unit test")
    try:
        x = torch.arange(size * 6, dtype=torch.float32, device=device).reshape(size, 3, 2) + rank
        _x = x.clone()
        res = hs.reduce_scatter(x, codes.SUM)
        want = torch.arange(rank * 6, rank * 6 + 6, dtype=torch.float32, device=device).reshape(3, 2) * size
        assert res.device == x.device and res.dtype == x.dtype
        assert torch.equal(res, want + sum(range(size)))
        assert torch.equal(x, _x)
        v = torch.arange(size, dtype=torch.int32, device=device) + rank
        assert hs.reduce_scatter(v, codes.MAX).item() == rank + size - 1
    finally:
        hs.comm.Free()


def test_staging_formula_reduce_scatter():
    from mpi4jax_b200._src import native
    from mpi4jax_b200._src.backends.cuda import stage_need

    if not native.HAS_CUDA_EXT:
        pytest.skip(f"native library not loaded: {native.CUDA_EXT_ERROR}")
    assert codes.OPC_REDUCE_SCATTER == 13
    for nranks in range(1, 17):
        for nbytes in [0, 1, 15, 16, 17, 4095, 4096, 65537, (1 << 20) + 3, 1 << 30]:
            want = ((nbytes + 15) // 16 * 16) * nranks + 4096
            assert stage_need(13, nranks, nbytes) == native.lib.b2_stage_need(13, nranks, nbytes) == want


def test_reduce_scatter_debug_log(device, capsys):
    from mpi4jax_b200._src.native import set_logging

    x = torch.ones((size, 4), device=device)
    m.reduce_scatter(x, MPI.SUM, comm=comm)
    m.flush()
    capsys.readouterr()
    set_logging(True)
    try:
        m.reduce_scatter(x, MPI.SUM, comm=comm)
        m.flush()
    finally:
        set_logging(False)
    out = capsys.readouterr().out
    assert re.search(rf"^r{rank} \| \w{{8}} \| MPI_Reduce_scatter_block( \(\w+\))? with 4 items per block", out,
                     re.M), out
    assert re.search(rf"^r{rank} \| \w{{8}} \| MPI_Reduce_scatter_block( \(\w+\))? done with code 0", out, re.M), out


_inside_job = size > 1 or "MPI4JAX_B200_NESTED" in os.environ


@pytest.mark.gpu
@pytest.mark.skipif(_inside_job, reason="already inside a multi-rank job")
def test_reduce_scatter_three_ranks_gpu():
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
        with tempfile.TemporaryDirectory(prefix="mpi4jax-b200-rs-job-") as logs:
            code, _ = launch(3, args, timeout=900, output_dir=logs, env_extra={"MPI4JAX_B200_NESTED": "1"})
            outs = [open(os.path.join(logs, f"rank{r}.log")).read() for r in range(3)]
    finally:
        os.chdir(cwd)
    for r, out in enumerate(outs):
        assert code == 0 and re.search(r"PASSED .*test_reduce_scatter_transports\[cuda\]", out), \
            f"rank {r} of the 3-rank job (exit code {code}):\n{out[-4000:]}"
