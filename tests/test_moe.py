"""moe_dispatch / moe_combine: top-k expert routing and the weighted combine.

Oracle: every rank gathers all ranks' ``x``, ``topk_idx``, ``weights`` and expert rows, then builds the expected
rows, counts, ``pos`` / ``dest`` and combine output pair by pair in plain torch on the CPU, with the sequential
fp32 fold; results compare bit for bit (NaN compares by position).  At world size 1 the tests run in-process;
``test_moe_jobs_*`` run them again as 2- and 3-rank jobs, on the CPU (gloo) and on the GPUs there are (the
ranks share them)."""

import os
import re

import pytest
import torch

import mpi4jax_b200 as m
from mpi4jax_b200 import MPI
from mpi4jax_b200._src.native import codes
from mpi4jax_b200.ops import MoePlan, moe_combine, moe_dispatch
from mpi4jax_b200.parallel import expert_combine, expert_dispatch
from mpi4jax_b200.run import launch

from ._peer_job import REPO, expect_passed, job

comm = MPI.COMM_WORLD
rank = comm.Get_rank()
size = comm.Get_size()

_FP8 = tuple(codes.FP8_DTYPE_CODE)
_inside_job = size > 1 or "MPI4JAX_B200_NESTED" in os.environ


def _gather(t):
    """Every rank's ``t`` (the same shape everywhere), stacked on the CPU."""
    return m.allgather(t.contiguous(), comm=comm).cpu()


def _bits(t):
    t = t.detach().cpu().contiguous()
    return t.view({1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])


def _same(a, b):
    """Bit-identical tensors; NaNs must sit at the same places (their payloads are not compared)."""
    a, b = a.detach().cpu(), b.detach().cpu()
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    if a.is_floating_point() and a.dtype not in _FP8:
        na, nb = a.isnan(), b.isnan()
        if not torch.equal(na, nb):
            return False
        a, b = torch.where(na, 0, a), torch.where(nb, 0, b)
    return torch.equal(_bits(a), _bits(b))


def _oracle_dispatch(x, idx, E, R):
    """(rows, recv_counts (L, P), pos, dest) of this rank, pair by pair from every rank's inputs."""
    L = E // size
    xs = _gather(x.view(torch.uint8) if x.dtype in _FP8 else x)
    ids = _gather(idx.to(torch.int64)).view(size, -1)
    k = idx.shape[1]
    rows = torch.zeros((R, *x.shape[1:]), dtype=xs.dtype)
    counts = torch.zeros((L, size), dtype=torch.int64)
    pos = torch.full((idx.numel(),), -1, dtype=torch.int64)
    dest = torch.full((idx.numel(),), -1, dtype=torch.int64)
    for d in range(size):
        at = 0
        for l in range(L):
            for q in range(size):
                for p in (ids[q] == d * L + l).nonzero().flatten().tolist():      # (token, slot) order
                    if at < R:
                        if d == rank:
                            rows[at] = xs[q, p // k]
                            counts[l, q] += 1
                        if q == rank:
                            pos[p], dest[p] = at, d
                    at += 1
    rows = rows.view(x.dtype) if x.dtype in _FP8 else rows
    return rows, counts, pos.view(idx.shape), dest.view(idx.shape)


def _oracle_combine(y, pos, dest, w=None, pairs=False):
    """Token t: its delivered pairs' rows, weighted and folded in slot order in fp32 (f64 for f64)."""
    ys = _gather(y)
    pos, dest = pos.cpu(), dest.cpu()
    N, k = pos.shape
    if pairs:
        out = torch.zeros((N, k, *y.shape[1:]), dtype=y.dtype)
        for t in range(N):
            for j in range(k):
                if dest[t, j] >= 0:
                    out[t, j] = ys[dest[t, j], pos[t, j]]
        return out
    acc_dt = torch.float64 if y.dtype == torch.float64 else torch.float32
    out = torch.zeros((N, *y.shape[1:]), dtype=y.dtype)
    for t in range(N):
        acc = None
        for j in range(k):
            if dest[t, j] < 0:
                continue
            v = ys[dest[t, j], pos[t, j]].to(acc_dt)
            if w is not None:
                v = w[t, j].cpu().to(acc_dt) * v
            acc = v if acc is None else acc + v
        if acc is not None:
            out[t] = acc.to(y.dtype)
    return out


def _check(x, idx, E, R=None):
    rows, expert_counts, plan = moe_dispatch(x, idx, E, recv_capacity=R, comm=comm)
    R = x.shape[0] * idx.shape[1] * size if R is None else R
    want, counts, pos, dest = _oracle_dispatch(x, idx, E, R)
    assert rows.shape == (R, *x.shape[1:]) and rows.dtype == x.dtype and rows.device == x.device
    assert _same(rows, want), (E, R, idx.shape)
    assert isinstance(plan, MoePlan) and plan.recv_capacity == R and plan.k == idx.shape[1]
    assert expert_counts.dtype == torch.int64 and expert_counts.device == x.device
    assert torch.equal(plan.recv_counts.cpu(), counts) and torch.equal(expert_counts.cpu(), counts.sum(1))
    assert torch.equal(plan.pos.cpu(), pos) and torch.equal(plan.dest.cpu(), dest), (E, R)
    return rows, plan


def _check_combine(y, plan, w=None):
    out = moe_combine(y, plan, w)
    assert out.shape == (plan.pos.shape[0], *y.shape[1:]) and out.dtype == y.dtype and out.device == y.device
    assert _same(out, _oracle_combine(y, plan.pos, plan.dest, w)), (y.dtype, w is None)
    return out


def _ids(n, k, E, seed, device, invalid=True):
    g = torch.Generator().manual_seed(seed)
    lo, hi = (-1, E + 1) if invalid else (0, E)
    idx = torch.randint(lo, hi, (n, k), generator=g)
    if n and k > 1:
        idx[0, 1] = idx[0, 0] = min(max(idx[0, 0], 0), E - 1)            # a token that lists an expert twice
    return idx.to(device)


def test_moe_routing(device):
    """k in {1, 2, 8}; E in {P, 4P, the largest multiple of P up to 256}; invalid and repeated ids; cuts at R
    (below one segment too); 12-byte rows (the byte path); N = 0."""
    n = 6
    for k in (1, 2, 8):
        for E in (size, 4 * size, 256 // size * size):
            idx = _ids(n, k, E, 100 * k + E + rank, device)
            x = (torch.arange(n * 3, dtype=torch.float32).reshape(n, 3) + 100 * rank).to(device)
            w = torch.rand(n, k, generator=torch.Generator().manual_seed(k + rank)).to(device)
            for R in (None, 2, n * k + 1):
                rows, plan = _check(x, idx, E, R)
                _check_combine(rows * 3 - 1, plan, w)
                _check_combine(rows, plan)
    for R in (None, 4):
        empty = torch.empty((0, 3), device=device)
        rows, plan = _check(empty, torch.empty((0, 2), dtype=torch.int32, device=device), 2 * size, R)
        assert not rows.any()
        assert _check_combine(rows, plan).shape == (0, 3)


def test_moe_rows_and_dtypes(device):
    """Multi-dimensional rows, expert outputs of another row shape, float8 rows byte for byte, the combine in
    every dtype with and without weights, rows of 16-byte multiples (the vector path)."""
    n, k, E = 9, 2, 2 * size
    idx = _ids(n, k, E, 7 + rank, device)
    g = torch.Generator().manual_seed(3 + rank)
    x = torch.randn(n, 2, 3, 4, generator=g).to(torch.bfloat16).to(device)
    rows, plan = _check(x, idx, E)
    w = torch.randn(n, k, generator=g).to(device)
    R = rows.shape[0]
    for dt in (torch.bfloat16, torch.float16, torch.float32, torch.float64):
        for shape in ((5,), (8,), (2, 16)):
            y = (torch.randn(R, *shape, generator=g) * 3).to(dt).to(device)
            _check_combine(y, plan, w)
            _check_combine(y, plan)
    f8 = (torch.randn(n, 32, generator=g) * 4).to(device).to(torch.float8_e4m3fn)
    _check(f8, idx, E, 5)
    _check(f8[:, :7], idx, E)


def test_moe_nan_inf_and_signed_zero(device):
    """NaN, inf and -0.0 in the expert rows, some of their pairs dropped; a lone -0.0 keeps its sign and a token
    with no delivered pair gets +0."""
    n, k, E = 8, 3, size
    idx = _ids(n, k, E, 11 + rank, device)
    idx[1] = -1                                                            # a token that sends nothing
    x = torch.randn(n, 4).to(device)
    for R in (None, 5):
        rows, plan = _check(x, idx, E, R)
        y = torch.randn(rows.shape, generator=torch.Generator().manual_seed(rank)).to(device)
        y[::3, 0] = float("nan")
        y[1::4, 1] = float("inf")
        y[2::4, 1] = -float("inf")
        y[:, 2] = -0.0
        out = _check_combine(y, plan, torch.rand(n, k).to(device) + 0.5)
        lone = (plan.dest.cpu() >= 0).sum(1) == 1
        assert (out[:, 2].cpu()[lone].view(torch.int32) == -(2**31)).all()     # -0.0
        none = (plan.dest.cpu() >= 0).sum(1) == 0
        assert none[1] and (_bits(out.cpu()[none]) == 0).all()                   # +0
        _check_combine(y.to(torch.bfloat16), plan)


def test_moe_matches_expert_dispatch(device):
    """k = 1 and E = P: the rows and counts of parallel.expert_dispatch, and expert_combine's output."""
    n = 10
    dest = torch.randint(-1, size + 1, (n,), generator=torch.Generator().manual_seed(rank)).to(device)
    x = torch.randn(n, 6).to(device)
    for cap in (None, 3):
        rows, rc, old = expert_dispatch(x, dest, capacity=cap, comm=comm)
        got, counts, plan = moe_dispatch(x, dest.view(n, 1), size, recv_capacity=cap, comm=comm)
        assert _same(got, rows) and torch.equal(plan.recv_counts.view(-1), rc) and counts.tolist() == [rc.sum().item()]
        assert _same(moe_combine(got * 2, plan), expert_combine(rows * 2, old))


@pytest.mark.filterwarnings("ignore:Input #0 requires gradient and is not a double")
def test_moe_gradients_gradcheck(device):
    """gradcheck in float64 (weights: float32, their only dtype) on a one-rank communicator, where the local
    Jacobian is the whole one."""
    solo = comm.Split(rank, 0)
    try:
        n, k, E = 5, 2, 3
        idx = _ids(n, k, E, 5, device)
        g = torch.Generator().manual_seed(9)
        x = torch.randn(n, 3, dtype=torch.float64, generator=g).to(device).requires_grad_(True)
        assert torch.autograd.gradcheck(lambda v: moe_dispatch(v, idx, E, recv_capacity=7, comm=solo)[0], (x,))
        rows, _, plan = moe_dispatch(x.detach(), idx, E, recv_capacity=7, comm=solo)
        y = torch.randn(rows.shape, dtype=torch.float64, generator=g).to(device).requires_grad_(True)
        w = (torch.rand(n, k, generator=g) + 0.5).to(device).requires_grad_(True)
        assert torch.autograd.gradcheck(lambda v: moe_combine(v, plan, w.detach()), (y,))
        assert torch.autograd.gradcheck(lambda v: moe_combine(v, plan), (y,))
        assert torch.autograd.gradcheck(lambda v: moe_combine(y.detach(), plan, v), (w,), eps=1e-2, atol=1e-4,
                                        rtol=1e-3)
        assert torch.autograd.gradcheck(lambda v: moe_combine(moe_dispatch(v, idx, E, comm=solo)[0] * 2,
                                                              moe_dispatch(v, idx, E, comm=solo)[2]), (x,))
    finally:
        m.flush()
        solo.Free()


def test_moe_gradients_bf16(device):
    """bf16 gradients of x and y equal the oracle bit for bit; the weights' gradient within fp32 rounding."""
    n, k, E = 7, 3, 2 * size
    idx = _ids(n, k, E, 21 + rank, device)
    g = torch.Generator().manual_seed(31 + rank)
    x = torch.randn(n, 8, generator=g).to(torch.bfloat16).to(device).requires_grad_(True)
    for R in (None, 6):
        rows, _, plan = moe_dispatch(x, idx, E, recv_capacity=R, comm=comm)
        ct_rows = torch.randn(rows.shape, generator=g).to(torch.bfloat16).to(device)
        x.grad = None
        (rows.float() * ct_rows.float()).sum().backward()
        assert _same(x.grad, _oracle_combine(ct_rows, plan.pos, plan.dest))
        y = torch.randn(rows.shape, generator=g).to(torch.bfloat16).to(device).requires_grad_(True)
        w = torch.randn(n, k, generator=g).to(device).requires_grad_(True)
        ct = torch.randn(n, 8, generator=g).to(torch.bfloat16).to(device)
        (moe_combine(y, plan, w).float() * ct.float()).sum().backward()
        # y: the row of pair (q, t, j) gets rn(w_q[t, j] * ct_q[t]); rows nobody filled get zero
        ps, ds, ws, cts = _gather(plan.pos), _gather(plan.dest), _gather(w.detach()), _gather(ct)
        want_y = torch.zeros(y.shape, dtype=torch.bfloat16)
        ys = _gather(y.detach()).float()
        want_w = torch.zeros(n, k)
        for q in range(size):
            for t in range(n):
                for j in range(k):
                    if ds[q, t, j] == rank:
                        want_y[ps[q, t, j]] = (ws[q, t, j] * cts[q, t].float()).to(torch.bfloat16)
                    if q == rank and ds[q, t, j] >= 0:
                        want_w[t, j] = (ys[ds[q, t, j], ps[q, t, j]] * cts[q, t].float()).sum()
        assert _same(y.grad, want_y), R
        assert torch.allclose(w.grad.cpu(), want_w, rtol=1e-5, atol=1e-5), R
        assert not w.grad.cpu()[plan.dest.cpu() < 0].any()


def test_moe_graph_replays(device):
    """mpi4jax_b200.jit captures dispatch -> per-expert matmul -> combine; replays with topk_idx and weights
    changed in place match eager calls."""
    if device.type != "cuda":
        pytest.skip("CUDA graphs")
    n, k, E, H = 16, 2, 2 * size, 32
    L = E // size
    gen = torch.Generator(device).manual_seed(rank)
    experts = torch.randn(L, H, H, device=device, generator=gen) / H
    x = torch.randn(n, H, device=device, generator=gen)

    def layer(x, idx, w):
        rows, counts, plan = moe_dispatch(x, idx, E, comm=comm)
        # expert of each received row from the group offsets (rows past the filled ones are zero)
        which = torch.searchsorted(counts.cumsum(0), torch.arange(rows.shape[0], device=x.device), right=True)
        y = torch.bmm(rows[:, None], experts[which.clamp(max=L - 1)])[:, 0]
        return moe_combine(y, plan, w)

    f = m.jit(layer)
    idx = torch.zeros(n, k, dtype=torch.int64, device=device)
    w = torch.zeros(n, k, device=device)
    for s in range(4):                               # eager warm-up, capture, replays
        idx.copy_(_ids(n, k, E, 50 + 10 * s + rank, device))
        w.copy_(torch.rand(n, k, device=device, generator=gen))
        assert _same(f(x, idx, w), layer(x, idx, w)), s
    m.flush()


def test_moe_launches_and_no_host_sync(device):
    """One native launch per dispatch and per combine, and no host synchronisation."""
    if device.type != "cuda":
        pytest.skip("native launches")
    from mpi4jax_b200._src import native

    n, k, E = 32, 4, 4 * size
    x = torch.randn(n, 64, device=device)
    idx = _ids(n, k, E, rank, device)
    w = torch.rand(n, k, device=device)
    rows, _, plan = moe_dispatch(x, idx, E, comm=comm)               # sizes the staging
    moe_combine(rows, plan, w)
    torch.cuda.synchronize()
    before = native.launch_count()
    torch.cuda.set_sync_debug_mode("error")
    try:
        rows, _, plan = moe_dispatch(x, idx, E, comm=comm)
        mid = native.launch_count()
        out = moe_combine(rows, plan, w)
        end = native.launch_count()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert (mid - before, end - mid) == (1, 1)
    assert _same(out, _oracle_combine(rows, plan.pos, plan.dest, w))


def test_moe_deterministic(device):
    n, k, E = 40, 4, 4 * size
    idx = _ids(n, k, E, 3 + rank, device)
    x = torch.randn(n, 24).to(device)
    w = torch.randn(n, k).to(device)
    a_rows, _, a_plan = moe_dispatch(x, idx, E, comm=comm)
    b_rows, _, b_plan = moe_dispatch(x, idx, E, comm=comm)
    assert _same(a_rows, b_rows) and torch.equal(a_plan.pos, b_plan.pos)
    y = torch.randn(a_rows.shape).to(device)
    assert _same(moe_combine(y, a_plan, w), moe_combine(y, b_plan, w))


def test_moe_errors(device):
    """Argument errors, raised on every rank before any device work."""
    x = torch.ones(4, 3, device=device)
    idx = torch.zeros(4, 2, dtype=torch.int64, device=device)
    E = size
    bad = [
        (ValueError, "x must be a tensor of shape", (torch.tensor(1.0, device=device), idx, E), {}),
        (TypeError, "topk_idx must be an int32 or int64", (x, idx.float(), E), {}),
        (ValueError, re.escape("topk_idx must have shape (N, k)"), (x, idx[:3], E), {}),
        (ValueError, re.escape("topk_idx must have shape (N, k)"), (x, idx[:, :0], E), {}),
        (ValueError, re.escape("topk_idx must have shape (N, k)"), (x, idx.view(-1), E), {}),
        (ValueError, "must live on the device of x", (x, idx.to("meta"), E), {}),
        (ValueError, "num_experts must be a positive multiple", (x, idx, 0), {}),
        (ValueError, "num_experts must be a positive multiple", (x, idx, 257 // size * size + size), {}),
        (TypeError, "num_experts must be an int", (x, idx, 2.0), {}),
        (ValueError, re.escape("recv_capacity must be >= 0"), (x, idx, E), {"recv_capacity": -1}),
        (TypeError, "recv_capacity must be an int", (x, idx, E), {"recv_capacity": 2.0}),
    ]
    if size > 1:
        bad.append((ValueError, "num_experts must be a positive multiple", (x, idx, size + 1), {}))
    for exc, msg, args, kw in bad:
        with pytest.raises(exc, match=msg):
            moe_dispatch(*args, comm=comm, **kw)
    rows, _, plan = moe_dispatch(x, idx, E, comm=comm)
    with pytest.raises(ValueError, match="y must have shape"):
        moe_combine(rows[1:], plan)
    with pytest.raises(TypeError, match="y must be float16, bfloat16, float32 or float64"):
        moe_combine(rows.to(torch.int32), plan)
    with pytest.raises(TypeError, match="weights must be a float32 tensor"):
        moe_combine(rows, plan, torch.ones(4, 2, dtype=torch.float64, device=device))
    with pytest.raises(ValueError, match="weights must have shape"):
        moe_combine(rows, plan, torch.ones(4, 3, device=device))
    with pytest.raises(TypeError, match="plan must be the MoePlan"):
        moe_combine(rows, tuple(plan))


def test_moe_host_staged(device, monkeypatch):
    """The host-staged transport runs the CPU rules on host copies of the same arguments."""
    from mpi4jax_b200._src.backends import host_staged

    monkeypatch.setattr(host_staged, "ACTIVE", host_staged.ACTIVE)
    hs_comm = comm.Clone()
    hs = host_staged.HostStagedComm(hs_comm, "unit test")
    try:
        n, k, E, R = 6, 2, 2 * size, 7
        idx = _ids(n, k, E, 13 + rank, device)
        x = torch.randn(n, 5).to(device)
        _, _, plan = moe_dispatch(x, idx, E, recv_capacity=R, comm=comm)
        rows, counts, pos, dest = hs.moe_dispatch(x, plan.order, plan.send_counts, k, E, R)
        want, want_counts, want_pos, want_dest = _oracle_dispatch(x, idx, E, R)
        assert rows.device == x.device and _same(rows, want) and torch.equal(counts.cpu(), want_counts)
        assert torch.equal(pos.view(n, k).cpu(), want_pos) and torch.equal(dest.view(n, k).cpu(), want_dest)
        w = torch.rand(n, k).to(device)
        out = hs.moe_combine(rows, plan.pos, plan.dest, w, plan.recv_counts)
        assert out.device == x.device and _same(out, _oracle_combine(rows, plan.pos, plan.dest, w))
        pairs = hs.moe_combine(rows, plan.pos, plan.dest, None, plan.recv_counts, pairs=True)
        assert _same(pairs, _oracle_combine(rows, plan.pos, plan.dest, pairs=True))
    finally:
        hs_comm.Free()


def test_staging_formula_moe():
    from mpi4jax_b200._src import native
    from mpi4jax_b200._src.backends.cuda import stage_need

    if not native.HAS_CUDA_EXT:
        pytest.skip(f"native library not loaded: {native.CUDA_EXT_ERROR}")
    assert (codes.OPC_MOE_DISPATCH, codes.OPC_MOE_COMBINE) == (19, 20)
    for nranks in (1, 2, 3, 8, 16):
        for nbytes in (0, 1, 12, 16, 65537, 1 << 30):
            for opc, want in ((codes.OPC_MOE_DISPATCH, 2048 + (nbytes + 15) // 16 * 16 + 4096),
                              (codes.OPC_MOE_COMBINE, (nbytes + 15) // 16 * 16 + 4096)):
                assert stage_need(opc, nranks, nbytes) == native.lib.b2_stage_need(opc, nranks, nbytes) == want


_TESTS = ["test_moe_routing", "test_moe_rows_and_dtypes", "test_moe_nan_inf_and_signed_zero",
          "test_moe_matches_expert_dispatch", "test_moe_gradients_gradcheck", "test_moe_gradients_bf16",
          "test_moe_deterministic", "test_moe_errors", "test_moe_host_staged"]


@pytest.mark.skipif(_inside_job, reason="already inside a multi-rank job")
@pytest.mark.parametrize("nranks", [2, 3])
def test_moe_jobs_cpu(nranks, tmp_path):
    """This file's CPU tests as an nranks-rank job over gloo."""
    test_file = os.path.relpath(os.path.abspath(__file__), REPO)
    args = ["-m", "pytest", test_file, "-q", "-rp", "-m", "not gpu", "-k", "not jobs", "-p", "no:cacheprovider"]
    cwd = os.getcwd()
    os.chdir(REPO)
    try:
        code, _ = launch(nranks, args, cpu=True, timeout=900, output_dir=str(tmp_path),
                         env_extra={"MPI4JAX_B200_NESTED": "1"})
    finally:
        os.chdir(cwd)
    for r in range(nranks):
        out = (tmp_path / f"rank{r}.log").read_text()
        missing = [t for t in _TESTS if not re.search(rf"^PASSED .*::{t}\[cpu\]", out, re.M)]
        assert code == 0 and not missing, f"rank {r} (exit code {code}), not passed: {missing}:\n{out[-4000:]}"


@pytest.mark.gpu
@pytest.mark.skipif(_inside_job, reason="already inside a multi-rank job")
@pytest.mark.parametrize("nranks", [2, 3])
def test_moe_jobs_gpu(nranks):
    """This file's CUDA tests as an nranks-rank job on the GPUs there are."""
    code, outs = job(__file__, nranks, select="not jobs")
    expect_passed(code, outs, nranks, _TESTS + ["test_moe_graph_replays", "test_moe_launches_and_no_host_sync"])
