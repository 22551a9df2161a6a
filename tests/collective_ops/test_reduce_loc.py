"""MAXLOC / MINLOC: allreduce, reduce, scan and reduce_scatter of ``(values, indices)`` pairs.

Oracle: every rank builds every rank's inputs from a seed and folds them in rank order with numpy -- MAXLOC
takes the next pair when its value is larger, or equal (+0 == -0) with a smaller index; a NaN value beats
every other value, two NaNs tie -- and compares the result bit for bit (values as their raw bits, so signed
zeros and NaN payloads count).  The CUDA variants need peers: in a single-process run they are checked in a
two-rank job whose ranks share the GPU, and ``test_reduce_loc_three_ranks_gpu`` runs them with three ranks."""

import contextlib
import os
import re
import tempfile

import numpy as np
import pytest
import torch

import mpi4jax_b200 as m
from mpi4jax_b200 import MPI
from mpi4jax_b200._src.native import codes

from .._peer_job import needs_peers

comm = MPI.COMM_WORLD
rank = comm.Get_rank()
size = comm.Get_size()

peers = needs_peers("MAXLOC / MINLOC between ranks")

VALUE_DTYPES = [torch.float16, torch.bfloat16, torch.float32, torch.float64, torch.int16, torch.int32, torch.int64]
INDEX_DTYPES = [torch.int32, torch.int64]
KINDS = ["allreduce", "reduce", "scan", "reduce_scatter"]
_INT = {2: torch.int16, 4: torch.int32, 8: torch.int64}
_QNAN = {torch.float16: 0x7E00, torch.bfloat16: 0x7FC0, torch.float32: 0x7FC00000,
         torch.float64: 0x7FF8000000000000}


def _pair(seed, q, shape, vdt, idt, special=True):
    """Rank q's inputs: few distinct values and indices (ties in value, and in value and index), and with
    ``special`` +-0, +-inf and NaNs whose payload names the rank (floats) or the integer extremes."""
    g = torch.Generator().manual_seed(seed * 131 + q)
    v = torch.randint(-3, 4, shape, generator=g).to(vdt)
    i = torch.randint(0, 4, shape, generator=g).to(idt)
    if special:
        r = torch.randint(0, 12, shape, generator=g)
        if vdt.is_floating_point:
            v = torch.where(r == 0, torch.tensor(-0.0, dtype=vdt), v)
            v = torch.where(r == 1, torch.tensor(float("inf"), dtype=vdt), v)
            v = torch.where(r == 2, torch.tensor(float("-inf"), dtype=vdt), v)
            bits = v.view(_INT[v.element_size()])
            nan = torch.full(shape, _QNAN[vdt] + 1 + q, dtype=bits.dtype)
            v = torch.where(r == 3, nan, bits).view(vdt)
        else:
            info = torch.iinfo(vdt)
            v = torch.where(r == 0, torch.tensor(info.min, dtype=vdt), v)
            v = torch.where(r == 1, torch.tensor(info.max, dtype=vdt), v)
    return v, i


def _bits(v):
    v = v.detach().cpu()
    return (v.view(_INT[v.element_size()]) if v.dtype.is_floating_point else v).numpy()


def _oracle(pairs, maxloc):
    """numpy fold of ``pairs`` (CPU tensors) in the given order: (value bits, indices)."""
    keys = [(v.double() if v.dtype.is_floating_point else v.to(torch.int64)).numpy() for v, _ in pairs]
    bits = [_bits(v) for v, _ in pairs]
    idx = [i.to(torch.int64).numpy() for _, i in pairs]
    ak, ab, ai = keys[0], bits[0], idx[0]
    for bk, bb, bi in zip(keys[1:], bits[1:], idx[1:]):
        an, bn = np.isnan(ak), np.isnan(bk)
        with np.errstate(invalid="ignore"):
            beats = bk > ak if maxloc else bk < ak
            take = np.where(an | bn, bn & (~an | (bi < ai)), beats | ((bk == ak) & (bi < ai)))
        ak, ab, ai = np.where(take, bk, ak), np.where(take, bb, ab), np.where(take, bi, ai)
    return ab, ai


def _run(kind, x, op, root=0, c=comm):
    if kind == "allreduce":
        return m.allreduce(x, op, comm=c)
    if kind == "reduce":
        return m.reduce(x, op, root, comm=c)
    if kind == "scan":
        return m.scan(x, op, comm=c)
    return m.reduce_scatter(x, op, comm=c)


def _check(device, kind, pairs, opname, root=0):
    """``kind`` of this rank's pair of ``pairs`` (every rank's CPU inputs), against the oracle."""
    op = getattr(MPI, opname)
    v, i = pairs[rank]
    x = (v.to(device), i.to(device))
    x0 = (x[0].clone(), x[1].clone())
    out = _run(kind, x, op, root)
    assert isinstance(out, tuple) and len(out) == 2
    assert np.array_equal(_bits(x[0]), _bits(x0[0])) and torch.equal(x[1], x0[1])      # inputs untouched
    if kind == "reduce" and rank != root:
        assert out[0] is x[0] and out[1] is x[1]
        return out
    src = pairs[: rank + 1] if kind == "scan" else pairs
    if kind == "reduce_scatter":
        src = [(pv[rank], pi[rank]) for pv, pi in src]
    want_v, want_i = _oracle(src, opname == "MAXLOC")
    shape = v.shape[1:] if kind == "reduce_scatter" else v.shape
    for t, dt in zip(out, (v.dtype, i.dtype)):
        assert t.shape == shape and t.dtype == dt and t.device == x[0].device, (kind, t.shape, t.dtype)
    assert np.array_equal(_bits(out[0]), want_v), (kind, opname, v.dtype, i.dtype)
    assert np.array_equal(out[1].cpu().to(torch.int64).numpy(), want_i), (kind, opname, v.dtype, i.dtype)
    return out


def _all_pairs(seed, shape, vdt, idt, special=True):
    return [_pair(seed, q, shape, vdt, idt, special) for q in range(size)]


@peers
def test_reduce_loc_dtypes_and_collectives(device):
    """Every value x index dtype, both ops, the four collectives and every root of reduce, on an odd count
    (a tail that is not a whole vector) with ties, +-0, +-inf, NaNs and integer extremes."""
    for a, vdt in enumerate(VALUE_DTYPES):
        for b, idt in enumerate(INDEX_DTYPES):
            pairs = _all_pairs(10 * a + b, (37,), vdt, idt)
            blocks = _all_pairs(10 * a + b, (size, 3, 5), vdt, idt)
            for opname in ("MAXLOC", "MINLOC"):
                for kind in ("allreduce", "scan"):
                    _check(device, kind, pairs, opname)
                for root in range(size):
                    _check(device, "reduce", pairs, opname, root)
                _check(device, "reduce_scatter", blocks, opname)


@peers
def test_reduce_loc_engineered_ties(device):
    """Ties in value, in value and index, +0 against -0, NaNs at several ranks (payloads tell them apart), and
    a NaN against +-inf and the integer extremes."""
    n = 6
    nan = lambda q: torch.tensor([_QNAN[torch.float32] + 1 + q], dtype=torch.int32).view(torch.float32)[0]
    pairs = []
    for q in range(size):
        v = torch.tensor([1.0, 2.0, 0.0, 5.0, float("inf"), 7.0])
        v[2] = -0.0 if q % 2 else 0.0                                    # +0 == -0: the index decides
        if q > 0:
            v[3] = nan(q)                                                # NaN at every rank but 0
        if q == size - 1:
            v[5] = nan(q)
        i = torch.tensor([size - q, 3, size - q, size - q, 3, q], dtype=torch.int64)   # col 1, 4: full ties
        pairs.append((v, i))
    for opname in ("MAXLOC", "MINLOC"):
        for kind in ("allreduce", "scan"):
            out = _check(device, kind, pairs, opname)
        assert out[1][1].item() == 3                   # column 1: every rank ties in value and index
    ints = [(torch.tensor([torch.iinfo(torch.int64).min if q % 2 else torch.iinfo(torch.int64).max] * n),
             torch.arange(n, dtype=torch.int32) + q) for q in range(size)]
    for opname in ("MAXLOC", "MINLOC"):
        _check(device, "allreduce", ints, opname)


@peers
def test_reduce_loc_shapes_and_layouts(device):
    """0-d pairs, Python scalars, empty tensors, an odd number of pairs and non-contiguous inputs."""
    for kind in ("allreduce", "reduce", "scan"):
        _check(device, kind, _all_pairs(3, (), torch.float32, torch.int64), "MAXLOC")
        _check(device, kind, _all_pairs(4, (0,), torch.float64, torch.int32), "MINLOC")
        _check(device, kind, _all_pairs(5, (2, 0, 3), torch.int16, torch.int64), "MAXLOC")
        _check(device, kind, _all_pairs(6, (3, 7), torch.bfloat16, torch.int32), "MINLOC")
    _check(device, "reduce_scatter", _all_pairs(7, (size,), torch.float16, torch.int64), "MAXLOC")
    _check(device, "reduce_scatter", _all_pairs(8, (size, 0), torch.float32, torch.int64), "MINLOC")
    # Python scalars become tensors as in every op: a float32 value and an int64 index
    err = float(rank % 2) + 0.5
    v, i = m.allreduce((err, rank), MPI.MAXLOC, comm=comm)
    assert v.dtype == torch.float32 and i.dtype == torch.int64 and v.shape == ()
    want = max(range(size), key=lambda q: (float(q % 2) + 0.5, -q))
    assert v.item() == float(want % 2) + 0.5 and i.item() == want
    # non-contiguous values and indices: the results of their contiguous copies
    g = torch.Generator().manual_seed(rank)
    base_v = torch.randint(-2, 3, (8, 6), generator=g).float().to(device)
    base_i = torch.randint(0, 3, (6, 8), generator=g).to(device)
    for kind in KINDS:
        if kind == "reduce_scatter":
            xv, xi = base_v[:size * 2:2, ::2], base_i.t()[:size, 1::2]
        else:
            xv, xi = base_v[:, ::2], base_i.t()[:, 1::2]
        assert not xv.is_contiguous() and not xi.is_contiguous()
        got = _run(kind, (xv, xi), MPI.MINLOC)
        want = _run(kind, (xv.contiguous(), xi.contiguous()), MPI.MINLOC)
        assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1]), kind


@contextlib.contextmanager
def _max_blocks(device, n):
    """The collective grid cap set to ``n`` CTAs for the block (CUDA), restored afterwards."""
    if device.type != "cuda" or not n:
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
def test_reduce_loc_multi_chunk(device):
    """~200 Ki pairs (3.2 MB of records): many CTAs with one chunk each, and with one or two CTAs (max_blocks)
    several chunks per CTA, the next staged between this one's arrive and its wait.  Results agree across
    ranks."""
    pairs = _all_pairs(21, (200_003,), torch.float32, torch.int64)
    blocks = _all_pairs(22, (size, 70_001), torch.float64, torch.int32)
    for blocks_cap in (0, 1, 2):
        with _max_blocks(device, blocks_cap):
            out = _check(device, "allreduce", pairs, "MAXLOC")
            _check(device, "scan", pairs, "MINLOC")
            _check(device, "reduce", pairs, "MAXLOC", size - 1)
            _check(device, "reduce_scatter", blocks, "MINLOC")
    digests = comm.allgather((_bits(out[0]).tobytes(), out[1].cpu().numpy().tobytes()))
    assert all(d == digests[0] for d in digests)


def test_reduce_loc_single_rank(device):
    """A one-rank communicator: every collective returns its input pair (reduce-scatter: block 0)."""
    solo = comm.Split(rank, 0)
    try:
        v, i = _pair(1, 0, (1, 9), torch.float32, torch.int32)
        for kind in KINDS:
            out = _run(kind, (v.to(device), i.to(device)), MPI.MAXLOC, c=solo)
            want = (v[0], i[0]) if kind == "reduce_scatter" else (v, i)
            assert np.array_equal(_bits(out[0]), _bits(want[0])) and torch.equal(out[1].cpu(), want[1]), kind
    finally:
        m.flush()
        solo.Free()


def _mpi4py_maxloc(x, y):
    """mpi4py's MAXLOC on Python pairs (no NaNs)."""
    (u, i), (v, j) = x, y
    if u > v:
        return u, i
    if v > u:
        return v, j
    return (v, j) if j < i else (u, i)


def _mpi4py_minloc(x, y):
    (u, i), (v, j) = x, y
    if u < v:
        return u, i
    if v < u:
        return v, j
    return (v, j) if j < i else (u, i)


def test_reduce_loc_object_api():
    """``comm.allreduce((v, i), op=MPI.MAXLOC)`` and ``comm.reduce`` behave as mpi4py's; ``Op.__call__`` on tensor
    pairs is the elementwise rule; the operators pickle by name and map from mpi4py's names."""
    import functools
    import pickle
    from types import SimpleNamespace

    from mpi4jax_b200._src.comm import as_op

    everyone = [(float((3 * q) % 4), (5 * q) % 3) for q in range(size)]
    for op, rule in ((MPI.MAXLOC, _mpi4py_maxloc), (MPI.MINLOC, _mpi4py_minloc)):
        want = functools.reduce(rule, everyone)
        assert comm.allreduce(everyone[rank], op=op) == want
        assert comm.reduce(everyone[rank], op=op, root=0) == (want if rank == 0 else None)
        assert pickle.loads(pickle.dumps(op)) is op
        assert as_op(SimpleNamespace(name=f"MPI_{op.name}")) is op
    assert MPI.MAXLOC((1.0, 2), (1.0, 1)) == (1.0, 1) and MPI.MAXLOC((1.0, 1), (1.0, 1)) == (1.0, 1)
    assert MPI.MINLOC((0.0, 3), (-0.0, 2)) == (-0.0, 2) and MPI.MAXLOC((1.0, 5), (float("nan"), 9))[1] == 9
    pairs = [_pair(31, q, (40,), vdt, torch.int64) for q, vdt in enumerate([torch.bfloat16] * 2 + [torch.float64] * 2)]
    for a, b in ((pairs[0], pairs[1]), (pairs[2], pairs[3])):
        for op in (MPI.MAXLOC, MPI.MINLOC):
            v, i = op(a, b)
            want_v, want_i = _oracle([a, b], op is MPI.MAXLOC)
            assert np.array_equal(_bits(v), want_v) and np.array_equal(i.numpy(), want_i)


def test_reduce_loc_errors(device):
    v = torch.ones(4, device=device)
    i = torch.zeros(4, dtype=torch.int64, device=device)
    for call in (lambda x, **k: m.allreduce(x, MPI.MAXLOC, comm=comm, **k),
                 lambda x: m.reduce(x, MPI.MINLOC, 0, comm=comm), lambda x: m.scan(x, MPI.MAXLOC, comm=comm)):
        with pytest.raises(TypeError, match=re.escape("takes a pair (values, indices)")):
            call(v)
        with pytest.raises(TypeError, match="takes a pair"):
            call((v, i, i))
        for bad in (torch.bool, torch.uint8, torch.int8, torch.complex64):
            with pytest.raises(TypeError, match="values must be float16, bfloat16"):
                call((v.to(bad), i))
        for bad in (torch.int16, torch.float32, torch.uint32):
            with pytest.raises(TypeError, match="indices must be int32 or int64"):
                call((v, i.to(bad)))
        with pytest.raises(ValueError, match="must have the same shape"):
            call((v, i[:3]))
        with pytest.raises(ValueError, match="must live on the same device"):
            call((v, i.to("meta" if device.type == "cpu" else "cpu")))
    with pytest.raises(ValueError, match="algorithm must be 'auto'"):
        m.allreduce((v, i), MPI.MAXLOC, comm=comm, algorithm="ll")
    with pytest.raises(ValueError, match=re.escape("Reduce_scatter input must have shape (nproc, ...)")):
        m.reduce_scatter((v[:size + 1], i[:size + 1]), MPI.MAXLOC, comm=comm)
    vr = v.clone().requires_grad_(True)
    for name, call in (("allreduce", lambda x: m.allreduce(x, MPI.MAXLOC, comm=comm)),
                       ("reduce", lambda x: m.reduce(x, MPI.MAXLOC, 0, comm=comm)),
                       ("scan", lambda x: m.scan(x, MPI.MINLOC, comm=comm))):
        op = "MINLOC" if name == "scan" else "MAXLOC"
        with pytest.raises(NotImplementedError, match=f"The derivative of {name} for {op} is not defined"):
            call((vr, i))
    with pytest.raises(NotImplementedError, match="is not defined"):
        torch.func.vmap(lambda t: m.allreduce((t, i), MPI.MAXLOC, comm=comm)[0])(v.expand(2, 4))
    counts = torch.ones(size, dtype=torch.int64, device=device)
    with pytest.raises(NotImplementedError, match="reduce_scatterv does not support MAXLOC"):
        m.reduce_scatterv(v.reshape(4, 1), counts, MPI.MAXLOC, comm=comm)
    with pytest.raises(NotImplementedError, match="reduce_scatterv does not support MINLOC"):
        m.compiled.reduce_scatterv(v.reshape(4, 1), counts, MPI.MINLOC, comm=comm)


def test_tuples_with_other_ops_unchanged(device):
    """A tuple passed with any other operator is one tensor, as it always was."""
    out = m.allreduce((1.0, 2.0), MPI.SUM, comm=comm)
    assert torch.equal(out.cpu(), torch.tensor([1.0, 2.0]) * size) and out.dtype == torch.float32
    out = m.scan((3, 1), MPI.MAX, comm=comm)
    assert torch.equal(out.cpu(), torch.tensor([3, 1]))


@peers
def test_reduce_loc_jit_replays(device):
    """Captured once, replayed with new inputs: the new winners every time."""
    if device.type != "cuda":
        pytest.skip("CUDA graphs")
    f = m.jit(lambda v, i: (m.allreduce((v, i), MPI.MAXLOC, comm=comm),
                            m.reduce_scatter((v.view(size, -1), i.view(size, -1)), MPI.MINLOC, comm=comm)))
    n = size * 1000
    for step in range(4):                              # eager warm-up, capture, replays
        pairs = _all_pairs(40 + step, (n,), torch.float32, torch.int64)
        v, i = pairs[rank]
        (av, ai), (rv, ri) = f(v.to(device), i.to(device))
        want_v, want_i = _oracle(pairs, True)
        assert np.array_equal(_bits(av), want_v) and np.array_equal(ai.cpu().numpy(), want_i), step
        want_v, want_i = _oracle([(pv.view(size, -1)[rank], pi.view(size, -1)[rank]) for pv, pi in pairs], False)
        assert np.array_equal(_bits(rv), want_v) and np.array_equal(ri.cpu().numpy(), want_i), step
    m.flush()


@peers
def test_reduce_loc_compiled(device):
    """torch.compile(fullgraph=True) of the compiled.* ops with pairs: the eager results."""
    pairs = _all_pairs(50, (size, 9), torch.bfloat16, torch.int32)
    x = tuple(t.to(device) for t in pairs[rank])
    calls = {
        "allreduce": lambda v, i: m.compiled.allreduce((v, i), MPI.MAXLOC, comm=comm),
        "reduce": lambda v, i: m.compiled.reduce((v, i), MPI.MINLOC, size - 1, comm=comm),
        "scan": lambda v, i: m.compiled.scan((v, i), MPI.MINLOC, comm=comm),
        "reduce_scatter": lambda v, i: m.compiled.reduce_scatter((v, i), MPI.MAXLOC, comm=comm),
    }
    for kind, fn in calls.items():
        got = torch.compile(fn, backend="aot_eager", fullgraph=True)(*x)
        op = MPI.MINLOC if kind in ("reduce", "scan") else MPI.MAXLOC
        want = _run(kind, x, op, size - 1)
        assert np.array_equal(_bits(got[0]), _bits(want[0])) and torch.equal(got[1], want[1]), kind
    m.flush()


def test_reduce_loc_fake_shape_and_effect():
    from torch._higher_order_ops.effects import _EffectType, _get_effect
    from torch._subclasses.fake_tensor import FakeTensorMode

    from mpi4jax_b200._src import compile_ops

    with FakeTensorMode():
        v, i = torch.empty(size, 3, dtype=torch.float16), torch.empty(size, 3, dtype=torch.int32)
        for opcode, shape in ((codes.OPC_ALLREDUCE, (size, 3)), (codes.OPC_REDUCE, (size, 3)),
                              (codes.OPC_SCAN, (size, 3)), (codes.OPC_REDUCE_SCATTER, (3,))):
            ov, oi = torch.ops.mpi4jax_b200.reduce_loc(v, i, codes.MAXLOC, opcode, 0, comm._id)
            assert ov.shape == shape and oi.shape == shape and ov.dtype == torch.float16 and oi.dtype == torch.int32
        ov, oi = m.compiled.reduce_scatter((v, i), MPI.MINLOC, comm=comm)
        assert ov.shape == (3,) and oi.dtype == torch.int32
    assert "reduce_loc" in compile_ops.ALL_OPS
    assert _get_effect("mpi4jax_b200::reduce_loc") == _EffectType.ORDERED


def test_host_staged_reduce_loc(device, monkeypatch):
    from mpi4jax_b200._src.backends import host_staged

    monkeypatch.setattr(host_staged, "ACTIVE", host_staged.ACTIVE)      # restore the flag afterwards
    host_staged_comm = comm.Clone()
    hs = host_staged.HostStagedComm(host_staged_comm, "unit test")
    try:
        pairs = _all_pairs(60, (size, 11), torch.float16, torch.int64)
        v, i = (t.to(device) for t in pairs[rank])
        out = hs.reduce_loc(codes.OPC_REDUCE_SCATTER, v, i, codes.MINLOC, 0)
        want_v, want_i = _oracle([(pv[rank], pi[rank]) for pv, pi in pairs], False)
        assert out[0].device == v.device and out[1].device == v.device
        assert np.array_equal(_bits(out[0]), want_v) and np.array_equal(out[1].cpu().numpy(), want_i)
        out = hs.reduce_loc(codes.OPC_REDUCE, v, i, codes.MAXLOC, 0)
        assert (out is None) == (rank != 0)
    finally:
        host_staged_comm.Free()


def test_reduce_loc_debug_log(device, capsys):
    from mpi4jax_b200._src.native import set_logging

    x = (torch.ones(4, device=device), torch.zeros(4, dtype=torch.int32, device=device))
    blocks = (torch.ones(size, 4, device=device), torch.zeros(size, 4, dtype=torch.int32, device=device))
    m.allreduce(x, MPI.MAXLOC, comm=comm)
    m.flush()
    capsys.readouterr()
    set_logging(True)
    try:
        m.allreduce(x, MPI.MAXLOC, comm=comm)
        m.reduce(x, MPI.MINLOC, 0, comm=comm)
        m.reduce_scatter(blocks, MPI.MAXLOC, comm=comm)
        m.flush()
    finally:
        set_logging(False)
    out = capsys.readouterr().out
    via = " via oneshot" if device.type == "cuda" else ""
    for name, details in (("Allreduce", "with 4 pairs"), ("Reduce", "with 4 pairs to root 0"),
                          ("Reduce_scatter_block", "with 4 pairs per block")):
        assert re.search(rf"^r{rank} \| \w{{8}} \| MPI_{name}( \(\w+\))? {details}{via}$", out, re.M), out
        assert re.search(rf"^r{rank} \| \w{{8}} \| MPI_{name}( \(\w+\))? done with code 0", out, re.M), out


_inside_job = size > 1 or "MPI4JAX_B200_NESTED" in os.environ


@pytest.mark.gpu
@pytest.mark.skipif(_inside_job, reason="already inside a multi-rank job")
def test_reduce_loc_three_ranks_gpu():
    """A non-power-of-two world: the CUDA tests of this file in a three-rank job (the ranks share the GPUs
    there are)."""
    from mpi4jax_b200.run import launch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    repo = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    test_file = os.path.relpath(os.path.abspath(__file__), repo)
    args = ["-m", "pytest", test_file, "-q", "-rp", "-m", "gpu", "-k", "not compiled", "-p", "no:cacheprovider"]
    cwd = os.getcwd()
    os.chdir(repo)
    try:
        with tempfile.TemporaryDirectory(prefix="mpi4jax-b200-loc-job-") as logs:
            code, _ = launch(3, args, timeout=900, output_dir=logs, env_extra={"MPI4JAX_B200_NESTED": "1"})
            outs = [open(os.path.join(logs, f"rank{r}.log")).read() for r in range(3)]
    finally:
        os.chdir(cwd)
    for r, out in enumerate(outs):
        assert code == 0 and re.search(r"PASSED .*test_reduce_loc_dtypes_and_collectives\[cuda\]", out), \
            f"rank {r} of the 3-rank job (exit code {code}):\n{out[-4000:]}"
