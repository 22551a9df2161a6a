"""float8 (e4m3fn, e5m2) through every collective.

Data movement is byte-exact.  A reduction's result is ``cast(fold)``: the contributions widened exactly to
fp32 and folded in rank order (SUM ``a + b``, PROD ``a * b``, MIN ``b if b < a or isnan(b) else a``, MAX with
``>``), then rounded once with torch's ``Tensor.to(float8)``; a NaN that SUM or PROD computes is the positive
NaN.  The oracle below is written from that rule in numpy and compared byte for byte.  Rank 0 holds all 256
bit patterns tiled and rank 1 each pattern repeated, so the first 65536 elements hold every (a, b) pair;
higher ranks hold seeded random bytes.  The CUDA variants need peers: in a single-process run they are
checked in a two-rank job whose ranks share the GPU, and ``test_fp8_three_ranks_gpu`` runs them with three
ranks (the two-phase scan and two-shot at P > 2)."""

import os

import numpy as np
import pytest
import torch

import mpi4jax_b200 as m
from mpi4jax_b200 import MPI
from mpi4jax_b200.parallel import expert_dispatch

from .._peer_job import expect_passed, job, needs_peers

comm = MPI.COMM_WORLD
rank = comm.Get_rank()
size = comm.Get_size()

peers = needs_peers("float8 collectives between ranks")

FP8 = [torch.float8_e4m3fn, torch.float8_e5m2]
OPS = {"SUM": MPI.SUM, "PROD": MPI.PROD, "MIN": MPI.MIN, "MAX": MPI.MAX}
PAIRS = 1 << 16


def _bytes(q, n, seed=0):
    """Rank q's input bytes (uint8, CPU)."""
    k = torch.arange(n)
    if q == 0:
        return (k % 256).to(torch.uint8)
    if q == 1 and seed == 0:
        return (k // 256 % 256).to(torch.uint8)
    g = torch.Generator().manual_seed(1000 * seed + q)
    return torch.randint(0, 256, (n,), generator=g, dtype=torch.uint8)


def _expect(parts, dt, opname):
    """cast(fold) of the contributions ``parts`` (uint8 tensors, in rank order), as uint8."""
    vals = [p.view(dt).to(torch.float32).numpy() for p in parts]
    acc = vals[0]
    with np.errstate(all="ignore"):
        for b in vals[1:]:
            if opname == "SUM":
                acc = acc + b
            elif opname == "PROD":
                acc = acc * b
            else:
                wins = b < acc if opname == "MIN" else b > acc
                acc = np.where(wins | np.isnan(b), b, acc)
    if opname in ("SUM", "PROD") and len(vals) > 1:
        acc = np.where(np.isnan(acc), np.float32(np.nan), acc)
    return torch.from_numpy(np.asarray(acc, dtype=np.float32)).to(dt).view(torch.uint8)


def _check(got, want, what):
    got = got.detach().cpu().contiguous().view(torch.uint8).reshape(-1)
    want = want.reshape(-1)
    assert got.shape == want.shape, f"{what}: {got.numel()} bytes, want {want.numel()}"
    bad = (got != want).nonzero()
    assert bad.numel() == 0, (f"{what}: {bad.numel()} bytes differ, first at {int(bad[0])}: "
                              f"got {int(got[bad[0]]):#04x}, want {int(want[bad[0]]):#04x}")


def _on(device, raw, dt):
    return raw.view(dt).to(device)


# ---------------------------------------------------------------------------
# reductions
# ---------------------------------------------------------------------------
def _reductions(device, dt, opname, n, seed=0, algos=("auto", "ll", "oneshot", "twoshot")):
    op = OPS[opname]
    parts = [_bytes(q, n, seed) for q in range(size)]
    x = _on(device, parts[rank], dt)
    want = _expect(parts, dt, opname)
    tag = f"{dt} {opname} n={n} P={size}"
    for algo in algos:
        if algo == "ll" and 2 * n > 128 << 10:
            continue
        _check(m.allreduce(x, op, comm=comm, algorithm=algo), want, f"allreduce {algo} {tag}")
    for root in sorted({0, size - 1}):
        out = m.reduce(x, op, root, comm=comm)
        if rank == root:
            _check(out, want, f"reduce root {root} {tag}")
    _check(m.scan(x, op, comm=comm), _expect(parts[: rank + 1], dt, opname), f"scan {tag}")
    blocks = [_bytes(q, size * n, seed) for q in range(size)]
    got = m.reduce_scatter(_on(device, blocks[rank], dt).reshape(size, n), op, comm=comm)
    _check(got, _expect([b[rank * n: (rank + 1) * n] for b in blocks], dt, opname), f"reduce_scatter {tag}")


@peers
def test_fp8_reductions_every_pair(device):
    """Every (a, b) pair of bit patterns, both formats, SUM / PROD / MIN / MAX, allreduce on every transport,
    reduce at both end roots, scan and reduce_scatter."""
    for dt in FP8:
        for opname in OPS:
            _reductions(device, dt, opname, PAIRS)
    m.flush()


@peers
def test_fp8_reductions_chunks_and_tails(device):
    """A multi-chunk payload (4 MiB + an odd tail) and short odd lengths."""
    for n in (1, 15, 17, 4099):
        _reductions(device, torch.float8_e5m2, "MAX", n, seed=1)
    _reductions(device, torch.float8_e4m3fn, "SUM", (4 << 20) + 13, seed=2, algos=("auto", "oneshot", "twoshot"))
    m.flush()


def _rsv_counts(q):
    """Rows rank q sends to each rank: 5..15 rows of 7 elements, so segments end inside 16-byte vectors."""
    return [5 + (3 * q + 7 * p) % 11 for p in range(size)]


@peers
def test_fp8_reduce_scatterv(device):
    """Rows of 7 elements: the per-element fold where a segment ends inside a vector; rows reached by one
    rank are that rank's bytes rounded, rows reached by none are zero."""
    row, cap = 7, 14
    for dt in FP8:
        for opname, op in OPS.items():
            counts = [_rsv_counts(q) for q in range(size)]
            parts = [_bytes(q, sum(counts[q]) * row, seed=3).reshape(-1, row) for q in range(size)]
            x = _on(device, parts[rank], dt)
            sc = torch.tensor(counts[rank], dtype=torch.int64, device=device)
            out, recv = m.reduce_scatterv(x, sc, op, recv_capacity=cap, comm=comm)
            reach = [min(counts[q][rank], cap) for q in range(size)]
            segs = [parts[q][sum(counts[q][:rank]):][:reach[q]] for q in range(size)]
            want = torch.zeros((cap, row), dtype=torch.uint8)
            for j in range(cap):
                qs = [q for q in range(size) if reach[q] > j]
                if qs:
                    want[j] = _expect([segs[q][j] for q in qs], dt, opname)
            _check(out, want, f"reduce_scatterv {dt} {opname} P={size}")
            assert recv.cpu().tolist() == reach
    m.flush()


def test_fp8_single_contribution(device):
    """A one-rank communicator still rounds: every byte comes back unchanged except the non-canonical e5m2
    NaNs, which become 0x7F / 0xFF by sign."""
    solo = comm.Split(rank, 0)
    try:
        raw = torch.arange(256, dtype=torch.uint8)
        for dt in FP8:
            want = raw.clone()
            if dt == torch.float8_e5m2:
                want[[0x7D, 0x7E]], want[[0xFD, 0xFE]] = 0x7F, 0xFF
            x = _on(device, raw, dt)
            for opname, op in OPS.items():
                tag = f"{dt} {opname}"
                _check(m.allreduce(x, op, comm=solo), want, f"allreduce {tag}")
                _check(m.reduce(x, op, 0, comm=solo), want, f"reduce {tag}")
                _check(m.scan(x, op, comm=solo), want, f"scan {tag}")
                _check(m.reduce_scatter(x.reshape(1, 256), op, comm=solo), want, f"reduce_scatter {tag}")
                sc = torch.tensor([16], dtype=torch.int64, device=device)
                out, _ = m.reduce_scatterv(x.reshape(16, 16), sc, op, comm=solo)
                _check(out, want, f"reduce_scatterv {tag}")
    finally:
        m.flush()
        solo.Free()


@peers
def test_fp8_scan_nan_payloads(device):
    """Rank 0's prefix is its own contribution rounded, on the two-phase scan too (> oneshot_max bytes at
    P > 2): its non-canonical e5m2 NaNs come back canonical."""
    n = (4 << 20) + 32
    raw = torch.tensor([0x7D, 0x7E, 0xFD, 0xFE, 0x7C, 0x01], dtype=torch.uint8).repeat(n // 6 + 1)[:n]
    parts = [raw if q == 0 else _bytes(q, n, seed=4) for q in range(size)]
    out = m.scan(_on(device, parts[rank], torch.float8_e5m2), MPI.MAX, comm=comm)
    _check(out, _expect(parts[: rank + 1], torch.float8_e5m2, "MAX"), f"scan e5m2 NaN payloads P={size}")
    m.flush()


# ---------------------------------------------------------------------------
# data movement
# ---------------------------------------------------------------------------
def _perm(q, salt=0):
    """All 256 bit patterns in an order that depends on the rank."""
    return ((torch.arange(256) * 5 + 17 * q + salt) % 256).to(torch.uint8)


@peers
def test_fp8_data_movement(device):
    """All 256 patterns of both formats arrive unchanged through every data-movement op."""
    p = size
    for dt in FP8:
        mine = _on(device, _perm(rank), dt)
        every = torch.stack([_perm(q) for q in range(p)])
        _check(m.allgather(mine, comm=comm), every, f"allgather {dt}")
        blocks = torch.stack([_perm(rank, 5 * d) for d in range(p)])
        _check(m.alltoall(_on(device, blocks, dt), comm=comm), torch.stack([_perm(q, 5 * rank) for q in range(p)]),
               f"alltoall {dt}")
        for root in sorted({0, p - 1}):
            _check(m.bcast(_on(device, _perm(rank), dt), root, comm=comm), _perm(root), f"bcast {dt} root {root}")
            out = m.gather(mine, root, comm=comm)
            if rank == root:
                _check(out, every, f"gather {dt} root {root}")
            src = torch.stack([_perm(root, 3 * d) for d in range(p)]) if rank == root else _perm(rank)
            _check(m.scatter(_on(device, src, dt), root, comm=comm), _perm(root, 3 * rank), f"scatter {dt} root {root}")
        nxt, prv = (rank + 1) % p, (rank - 1) % p
        got = m.sendrecv(mine, torch.empty_like(mine), prv, nxt, comm=comm)
        _check(got, _perm(prv), f"sendrecv {dt}")
        if rank == 0 and p > 1:
            m.send(mine, 1, tag=8, comm=comm)
        elif rank == 1:
            _check(m.recv(torch.empty_like(mine), 0, tag=8, comm=comm), _perm(0), f"send/recv {dt}")
        # variable-count ops on rows of all 256 patterns: rank q sends 1 + (q + d) % 3 rows to rank d
        rows = lambda q: torch.stack([_perm(q, 11 * k) for k in range(3 * p)])          # noqa: E731
        cnt = lambda q: [1 + (q + d) % 3 for d in range(p)]                              # noqa: E731
        sc = torch.tensor(cnt(rank), dtype=torch.int64, device=device)
        out, recv = m.alltoallv(_on(device, rows(rank), dt), sc, comm=comm)
        want = torch.cat([rows(q)[sum(cnt(q)[:rank]):][: cnt(q)[rank]] for q in range(p)])
        _check(out[: want.shape[0]], want, f"alltoallv {dt}")
        k = 1 + rank % 3
        out, _ = m.allgatherv(_on(device, rows(rank), dt), k, comm=comm)
        want = torch.cat([rows(q)[: 1 + q % 3] for q in range(p)])
        _check(out[: want.shape[0]], want, f"allgatherv {dt}")
        out, _ = m.gatherv(_on(device, rows(rank), dt), k, p - 1, comm=comm)
        if rank == p - 1:
            _check(out[: want.shape[0]], want, f"gatherv {dt}")
        out, _ = m.scatterv(_on(device, rows(0), dt), cnt(0), 0, comm=comm)
        _check(out[: cnt(0)[rank]], rows(0)[sum(cnt(0)[:rank]):][: cnt(0)[rank]], f"scatterv {dt}")
    m.flush()


@peers
def test_fp8_expert_dispatch(device):
    """fp8 tokens reach the ranks their routing names, packed by source rank in token order."""
    p = size
    tokens = lambda q: torch.stack([_perm(q, 7 * t) for t in range(2 * p + 1)])               # noqa: E731
    dest = lambda q: torch.tensor([(q + 3 * t) % (p + 1) for t in range(2 * p + 1)]) % p     # noqa: E731
    for dt in FP8:
        rows, recv, _ = expert_dispatch(_on(device, tokens(rank), dt), dest(rank).to(device), comm=comm)
        want = torch.cat([tokens(q)[dest(q) == rank] for q in range(p)])
        assert recv.cpu().tolist() == [int((dest(q) == rank).sum()) for q in range(p)]
        _check(rows[: want.shape[0]], want, f"expert_dispatch {dt}")
    m.flush()


# ---------------------------------------------------------------------------
# graphs, tracing
# ---------------------------------------------------------------------------
@peers
def test_fp8_jit_replays(device):
    """mpi4jax_b200.jit captures an fp8 allreduce and alltoallv and replays them with new inputs."""
    if device.type != "cuda":
        pytest.skip("CUDA graphs")
    sc = torch.ones(size, dtype=torch.int64, device=device)
    f = m.jit(lambda x, y: (m.allreduce(x, MPI.SUM, comm=comm), m.alltoallv(y, sc, recv_capacity=size, comm=comm)[0]))
    for seed in (5, 6, 7):
        parts = [_bytes(q, 4096, seed) for q in range(size)]
        rows = [_bytes(q, size * 256, seed + 50).reshape(size, 256) for q in range(size)]
        red, moved = f(_on(device, parts[rank], torch.float8_e4m3fn), _on(device, rows[rank], torch.float8_e5m2))
        _check(red, _expect(parts, torch.float8_e4m3fn, "SUM"), f"jit allreduce seed {seed}")
        _check(moved, torch.stack([rows[q][rank] for q in range(size)]), f"jit alltoallv seed {seed}")
    m.flush()


@peers
def test_fp8_compiled(device):
    """torch.compile(fullgraph=True) of compiled.allreduce and compiled.allgather with fp8 operands."""
    parts = [_bytes(q, 1000, 8) for q in range(size)]
    x = _on(device, parts[rank], torch.float8_e5m2)
    fn = torch.compile(lambda t: (m.compiled.allreduce(t, MPI.MIN, comm=comm), m.compiled.allgather(t, comm=comm)),
                       backend="aot_eager", fullgraph=True)
    red, gathered = fn(x)
    _check(red, _expect(parts, torch.float8_e5m2, "MIN"), "compiled allreduce")
    _check(gathered, torch.stack(parts), "compiled allgather")
    m.flush()


# ---------------------------------------------------------------------------
# errors
# ---------------------------------------------------------------------------
def _outcome(fn):
    try:
        fn()
    except Exception as exc:            # noqa: BLE001 - the outcome is compared, not handled
        return type(exc), str(exc).replace("float64", "<dtype>").replace(str(torch.float64), "<dtype>")
    return None


def test_fp8_errors(device, monkeypatch):
    monkeypatch.setenv("MPI4JAX_B200_ABORT_ON_ERROR", "0")
    for dt in FP8:
        x = torch.zeros(8, dtype=dt, device=device)
        for op in (MPI.LAND, MPI.LOR, MPI.LXOR, MPI.BAND, MPI.BOR, MPI.BXOR):
            with pytest.raises(NotImplementedError):
                m.allreduce(x, op, comm=comm)
            with pytest.raises(NotImplementedError):
                m.reduce_scatter(x.repeat(size).reshape(size, 8), op, comm=comm)
        with pytest.raises(TypeError):
            m.allreduce((x, torch.zeros(8, dtype=torch.int64, device=device)), MPI.MAXLOC, comm=comm)
        # the in-switch paths do not take fp8: what float64 gets
        for fn in (lambda t: m.allreduce(t, MPI.SUM, comm=comm, algorithm="nvls"),
                   lambda t: m.allreduce_(m.symmetric_empty((16,), t.dtype, comm=comm).zero_(), comm=comm)):
            want = _outcome(lambda: fn(torch.zeros(16, dtype=torch.float64, device=device)))
            m.flush()
            got = _outcome(lambda: fn(torch.zeros(16, dtype=dt, device=device)))
            m.flush()
            assert (got and got[0]) == (want and want[0]), (dt, got, want)
    for dt in (torch.float8_e4m3fnuz, torch.float8_e5m2fnuz, torch.float8_e8m0fnu):
        x = torch.zeros(4, dtype=torch.uint8, device=device).view(dt)
        with pytest.raises(RuntimeError, match="Unknown MPI type"):
            m.allreduce(x, MPI.SUM, comm=comm)
        with pytest.raises(RuntimeError, match="Unknown MPI type"):
            m.allgather(x, comm=comm)


_inside_job = size > 1 or "MPI4JAX_B200_NESTED" in os.environ


@pytest.mark.gpu
@pytest.mark.skipif(_inside_job, reason="already inside a multi-rank job")
def test_fp8_three_ranks_gpu():
    """A non-power-of-two world: the CUDA reductions of this file in a three-rank job (the ranks share the
    GPUs there are), where large payloads take the two-shot allreduce and the two-phase scan."""
    tests = ["test_fp8_reductions_every_pair", "test_fp8_reductions_chunks_and_tails", "test_fp8_reduce_scatterv",
             "test_fp8_scan_nan_payloads", "test_fp8_data_movement"]
    code, outs = job(__file__, 3, select=" or ".join(tests))
    expect_passed(code, outs, 3, tests)
