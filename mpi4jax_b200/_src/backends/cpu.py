"""CPU backend: the 15 ops on host tensors over ``torch.distributed`` (gloo).

Role: what the reference's CPU bridge (mpi_xla_bridge_cpu.cpp, one blocking MPI call
per op) is to its GPU bridge -- the correctness path that runs anywhere, including the
GPU-less CI box.  The image has no MPI, so gloo carries the bytes; semantics follow MPI:

* collectives move raw bytes (every dtype incl. bool/complex) with ``all_gather`` /
  ``broadcast`` and reduce locally in rank order (deterministic, all 10 ops);
* point-to-point keeps MPI matching semantics on top of gloo's FIFO channels: each
  message is a (header, payload) pair, the receiver keeps an unexpected-message queue
  per source, so tags may be consumed out of order, ``ANY_SOURCE`` / ``ANY_TAG`` work
  and ``Status`` is filled.  Sends are eager (``isend``) for every size, completed at
  ``flush()``; self-sends never touch the network.
"""

from __future__ import annotations

import time
from collections import deque
from typing import Optional

import torch
import torch.distributed as dist

from ..comm import ANY_SOURCE, ANY_TAG, Comm, Status
from ..native import codes

_HDR_WORDS = 4  # tag, nbytes, dtype code (informational), magic
_MAGIC = 0x6232_6D70  # "b2mp"


def _bytes_view(x: torch.Tensor) -> torch.Tensor:
    return x.contiguous().reshape(-1).view(torch.uint8)


def reduce_stack(stack: torch.Tensor, op_code: int) -> torch.Tensor:
    """Reduce ``stack`` (P, *shape) over dim 0 with MPI op semantics, in rank order."""
    dt = stack.dtype
    if dt in codes.FP8_DTYPE_CODE:
        return _reduce_fp8(stack, op_code)
    if stack.shape[0] == 1:
        return stack[0].clone()     # a single contribution passes through unchanged (as in MPI)
    if dt == torch.bool:
        if op_code in (codes.SUM, codes.MAX, codes.LOR, codes.BOR):
            return stack.any(dim=0)
        if op_code in (codes.PROD, codes.MIN, codes.LAND, codes.BAND):
            return stack.all(dim=0)
        if op_code in (codes.LXOR, codes.BXOR):
            return (stack.to(torch.int32).sum(dim=0) % 2).to(torch.bool)
    if dt in (torch.uint16, torch.uint32, torch.uint64) and op_code in (codes.SUM, codes.PROD, codes.MIN, codes.MAX):
        # CPU torch has no arithmetic on these: int64 holds the same bits modulo 2^64 (sums and products
        # wrap alike), and a flipped sign bit makes its order the unsigned order of uint64
        wide = stack.view(torch.int64) if dt == torch.uint64 else stack.to(torch.int64)
        if op_code in (codes.MIN, codes.MAX):
            bias = -(1 << 63) if dt == torch.uint64 else 0
            res = reduce_stack(wide ^ bias, op_code) ^ bias
        else:
            res = reduce_stack(wide, op_code)
        return res.view(dt) if dt == torch.uint64 else res.to(dt)
    is_float = dt.is_floating_point
    is_cplx = dt.is_complex
    if op_code == codes.SUM:
        acc_dt = torch.float32 if dt in (torch.float16, torch.bfloat16) else dt
        acc = stack[0].to(acc_dt).clone()
        for q in range(1, stack.shape[0]):
            acc += stack[q].to(acc_dt)
        return acc.to(dt)
    if op_code == codes.PROD:
        acc_dt = torch.float32 if dt in (torch.float16, torch.bfloat16) else dt
        acc = stack[0].to(acc_dt).clone()
        for q in range(1, stack.shape[0]):
            acc *= stack[q].to(acc_dt)
        return acc.to(dt)
    if is_cplx:
        raise NotImplementedError("only SUM and PROD are defined for complex dtypes")
    if op_code == codes.MIN:
        return stack.amin(dim=0) if not is_float else torch.min(stack, dim=0).values
    if op_code == codes.MAX:
        return stack.amax(dim=0) if not is_float else torch.max(stack, dim=0).values
    if is_float:
        raise NotImplementedError("logical/bitwise reductions need an integer or bool dtype")
    if op_code == codes.LAND:
        return (stack != 0).all(dim=0).to(dt)
    if op_code == codes.LOR:
        return (stack != 0).any(dim=0).to(dt)
    if op_code == codes.LXOR:
        return ((stack != 0).to(torch.int32).sum(dim=0) % 2).to(dt)
    wide = stack.to(torch.int64) if dt in (torch.uint16, torch.uint32, torch.uint64) else stack
    acc = wide[0].clone()
    for q in range(1, stack.shape[0]):
        if op_code == codes.BAND:
            acc &= wide[q]
        elif op_code == codes.BOR:
            acc |= wide[q]
        else:
            acc ^= wide[q]
    return acc.to(dt)


def _reduce_fp8(stack: torch.Tensor, op_code: int) -> torch.Tensor:
    """The float8 rule of the kernels (csrc/b2_device.cuh): widen exactly to fp32, fold in rank order with
    ``b2_apply`` (the later NaN wins MIN / MAX), round once with torch's cast -- a single contribution too.
    A NaN that SUM or PROD computes is the positive NaN, as the GPU's fp32 arithmetic makes it."""
    check_op(stack.dtype, op_code)
    wide = stack.to(torch.float32)
    acc = wide[0]
    for b in wide[1:]:
        if op_code == codes.SUM:
            acc = acc + b
        elif op_code == codes.PROD:
            acc = acc * b
        else:
            wins = b < acc if op_code == codes.MIN else b > acc
            acc = torch.where(wins | b.isnan(), b, acc)
    if op_code in (codes.SUM, codes.PROD) and stack.shape[0] > 1:
        acc = torch.where(acc.isnan(), float("nan"), acc)
    return acc.to(stack.dtype)


def check_op(dtype: torch.dtype, op_code: int) -> None:
    """Refuse a dtype / op pair that ``reduce_stack`` (and the CUDA kernels) do not define, with its error."""
    if dtype.is_complex and op_code not in (codes.SUM, codes.PROD):
        raise NotImplementedError("only SUM and PROD are defined for complex dtypes")
    if dtype.is_floating_point and op_code not in (codes.SUM, codes.PROD, codes.MIN, codes.MAX):
        raise NotImplementedError("logical/bitwise reductions need an integer or bool dtype")


class CpuState:
    """Per-communicator host-side p2p state (unexpected queues, pending sends)."""

    def __init__(self, comm: Comm):
        self.comm = comm
        self.pending: list = []                      # (work, keepalive tensors)
        self.unexpected = [deque() for _ in range(comm.size)]   # per source: (tag, payload)
        self.self_queue: deque = deque()

    def prune(self) -> None:
        self.pending = [(w, k) for (w, k) in self.pending if not w.is_completed()]

    def flush(self) -> None:
        for work, _ in self.pending:
            work.wait()
        self.pending.clear()


# ---------------------------------------------------------------------------
# collectives
# ---------------------------------------------------------------------------
def _allgather_bytes(comm: Comm, x: torch.Tensor) -> list:
    flat = _bytes_view(x)
    if comm.size == 1:
        return [flat.clone()]
    outs = [torch.empty_like(flat) for _ in range(comm.size)]
    dist.all_gather(outs, flat, group=comm._group)
    return comm._in_rank_order(outs)


def _gather_stack(comm: Comm, x: torch.Tensor) -> torch.Tensor:
    parts = _allgather_bytes(comm, x)
    return torch.stack([p.view(x.dtype).reshape(x.shape) for p in parts], dim=0)


def barrier(comm: Comm) -> None:
    dist.barrier(group=comm._group)


def allreduce(comm: Comm, x: torch.Tensor, op_code: int) -> torch.Tensor:
    return reduce_stack(_gather_stack(comm, x), op_code)


def reduce(comm: Comm, x: torch.Tensor, op_code: int, root: int) -> Optional[torch.Tensor]:
    stack = _gather_stack(comm, x)
    return reduce_stack(stack, op_code) if comm.rank == root else None


def scan(comm: Comm, x: torch.Tensor, op_code: int) -> torch.Tensor:
    stack = _gather_stack(comm, x)
    return reduce_stack(stack[: comm.rank + 1], op_code)


def reduce_scatter(comm: Comm, x: torch.Tensor, op_code: int) -> torch.Tensor:
    # x: (P, *S).  Everybody gathers everything and reduces its own block (correctness path).
    return reduce_stack(_gather_stack(comm, x)[:, comm.rank], op_code)


def reduce_loc(comm: Comm, opcode: int, values: torch.Tensor, indices: torch.Tensor, op_code: int, root: int):
    """MAXLOC / MINLOC: everybody gathers both tensors and folds the pairs of its source ranks in rank order
    through ``Op.__call__`` (correctness path).  None off the root of a reduce."""
    from ..comm import MAXLOC, MINLOC

    op = MAXLOC if op_code == codes.MAXLOC else MINLOC
    vals, idxs = _gather_stack(comm, values), _gather_stack(comm, indices)
    if opcode == codes.OPC_REDUCE_SCATTER:
        vals, idxs = vals[:, comm.rank], idxs[:, comm.rank]
    if opcode == codes.OPC_REDUCE and comm.rank != root:
        return None
    acc = (vals[0], idxs[0])
    for q in range(1, comm.rank + 1 if opcode == codes.OPC_SCAN else comm.size):
        acc = op(acc, (vals[q], idxs[q]))
    return acc[0].clone(), acc[1].clone()


def allgather(comm: Comm, x: torch.Tensor) -> torch.Tensor:
    return _gather_stack(comm, x)


def alltoall(comm: Comm, x: torch.Tensor) -> torch.Tensor:
    # x: (P, *S).  Everybody gathers everything and keeps its column (correctness path).
    stack = _gather_stack(comm, x)            # (P_src, P_dst, *S)
    return stack[:, comm.rank].clone()


def _clamp_in_order(counts, n: int) -> list:
    """Counts clamped in rank order to ``n`` rows: negative -> 0, nothing past row ``n``."""
    out, used = [], 0
    for c in counts:
        k = min(max(int(c), 0), n - used)
        out.append(k)
        used += k
    return out


def _pack(stack: torch.Tensor, counts: list, displs: list, out_rows: int, place: Optional[list] = None):
    """Rows ``[displs[q], displs[q] + counts[q])`` of ``stack[q]`` for every rank q, packed in rank order
    into ``out_rows`` rows and clipped to them (``place``: at most ``place[q]`` rows each, at the sum of
    the lower ranks' ``place``), zero elsewhere; and the rows written from each rank."""
    out = torch.zeros((out_rows, *stack.shape[2:]), dtype=stack.dtype)
    recv, filled = [], 0
    for q, (n, d) in enumerate(zip(counts, displs)):
        slot = out_rows - filled if place is None else place[q]
        k = min(n, slot)
        out[filled: filled + k] = stack[q, d: d + k]
        recv.append(k)
        filled += k if place is None else slot
    return out, torch.tensor(recv, dtype=torch.int64)


def _gather_segments(comm: Comm, x: torch.Tensor, counts: list, n: int):
    """Every rank's ``counts`` clamped in rank order to its first ``n`` rows, ``[q][p]``, and the rows they
    cover, zero-padded to a common width, ``(P, width, *S)``."""
    sent = _clamp_in_order(counts, n)
    counts = _gather_stack(comm, torch.tensor(sent, dtype=torch.int64)).tolist()
    mine = torch.zeros((max(sum(row) for row in counts), *x.shape[1:]), dtype=x.dtype)
    mine[: sum(sent)] = x[: sum(sent)]
    return counts, _gather_stack(comm, mine)


def alltoallv(comm: Comm, x: torch.Tensor, send_counts: torch.Tensor, out_rows: int,
              place_counts: Optional[torch.Tensor] = None):
    """Same rules as the kernel (csrc/b2_collectives.cu: b2_k_rowsv): everybody gathers every
    rank's clamped counts and sent rows, then assembles its own output (correctness path)."""
    P, r = comm.size, comm.rank
    rows = x.shape[0]
    max_rows = rows if place_counts is None else P * out_rows
    counts, stack = _gather_segments(comm, x, send_counts.tolist(), min(rows, max_rows))
    place = None if place_counts is None else _clamp_in_order(place_counts.tolist(), out_rows)
    return _pack(stack, [row[r] for row in counts], [sum(row[:r]) for row in counts], out_rows, place)


def allgatherv(comm: Comm, x: torch.Tensor, count: torch.Tensor, out_rows: int,
               place_counts: Optional[torch.Tensor] = None):
    """Same rules as the kernel's gather mode (csrc/b2_collectives.cu: b2_k_rowsv): alltoallv where every rank
    sends its first ``count`` rows to every rank, each segment from row 0 of its source (correctness
    path)."""
    n = min(max(int(count), 0), x.shape[0])
    counts = _gather_stack(comm, torch.tensor(n, dtype=torch.int64)).tolist()
    place = None if place_counts is None else _clamp_in_order(place_counts.tolist(), out_rows)
    return _pack(_gather_stack(comm, x), counts, [0] * comm.size, out_rows, place)


def reduce_scatterv(comm: Comm, x: torch.Tensor, send_counts: torch.Tensor, out_rows: int, op_code: int):
    """Same rules as the kernel (csrc/b2_reduce.cuh: b2_k_reduce_scatterv): everybody gathers every rank's
    clamped counts and rows, padded to a common width, then folds the segments for its own rank -- each
    run of rows over the ranks whose segment reaches it, in rank order (correctness path)."""
    P, r = comm.size, comm.rank
    check_op(x.dtype, op_code)         # on every call, also when no row has two contributors
    counts, stack = _gather_segments(comm, x, send_counts.tolist(), x.shape[0])
    recv = [min(row[r], out_rows) for row in counts]
    displ = [sum(row[:r]) for row in counts]
    out = torch.zeros((out_rows, *x.shape[1:]), dtype=x.dtype)
    lo = 0
    for hi in sorted(set(recv) - {0}):          # rows [lo, hi) have the same contributors
        qs = [q for q in range(P) if recv[q] >= hi]
        out[lo:hi] = reduce_stack(torch.stack([stack[q, displ[q] + lo: displ[q] + hi] for q in qs]), op_code)
        lo = hi
    return out, torch.tensor(recv, dtype=torch.int64)


def gatherv(comm: Comm, x: torch.Tensor, count: torch.Tensor, root: int, out_rows: int, max_rows: int,
            place_counts: Optional[torch.Tensor] = None):
    """Same rules as the kernel's gather mode with output rows on the root only (csrc/b2_collectives.cu:
    b2_k_rowsv): everybody gathers every rank's clamped count and rows, the root assembles its output
    (correctness path).  The other ranks get ``(None, zeros)``."""
    counts, stack = _gather_segments(comm, x, [count], min(x.shape[0], max_rows))
    if comm.rank != root:
        return None, torch.zeros(comm.size, dtype=torch.int64)
    place = None if place_counts is None else _clamp_in_order(place_counts.tolist(), out_rows)
    return _pack(stack, [n for (n,) in counts], [0] * comm.size, out_rows, place)


def scatterv(comm: Comm, x: torch.Tensor, send_counts: Optional[torch.Tensor], root: int, out_rows: int,
             max_rows: int):
    """Same rules as the kernel's rooted mode (csrc/b2_collectives.cu: b2_k_rowsv): the root broadcasts its
    send counts, clamped in rank order to its rows, then the rows they cover; each rank keeps its segment,
    clipped to ``out_rows`` (correctness path)."""
    P, r = comm.size, comm.rank
    if r == root:
        sent = torch.tensor(_clamp_in_order(send_counts.tolist(), min(x.shape[0], max_rows)), dtype=torch.int64)
    else:
        sent = torch.zeros(P, dtype=torch.int64)
    sent = bcast(comm, sent, root).tolist()
    width = sum(sent)
    rows = x[:width] if r == root else torch.empty((width, *x.shape[1:]), dtype=x.dtype)
    rows = bcast(comm, rows, root)
    k = min(sent[r], out_rows)
    out = torch.zeros((out_rows, *x.shape[1:]), dtype=x.dtype)
    d = sum(sent[:r])
    out[:k] = rows[d: d + k]
    return out, torch.tensor(k, dtype=torch.int64)


def bcast(comm: Comm, x: torch.Tensor, root: int) -> torch.Tensor:
    buf = _bytes_view(x).clone()
    if comm.size > 1:
        dist.broadcast(buf, src=comm._global(root), group=comm._group)
    return buf.view(x.dtype).reshape(x.shape)


def gather(comm: Comm, x: torch.Tensor, root: int) -> Optional[torch.Tensor]:
    stack = _gather_stack(comm, x)
    return stack if comm.rank == root else None


def scatter(comm: Comm, x: torch.Tensor, root: int, out_shape, dtype) -> torch.Tensor:
    # root holds (P, *S); others pass a template of shape S
    numel = 1
    for s in out_shape:
        numel *= s
    nbytes = numel * torch.empty((), dtype=dtype).element_size()
    if comm.rank == root:
        buf = _bytes_view(x).clone()
    else:
        buf = torch.empty(nbytes * comm.size, dtype=torch.uint8)
    if comm.size > 1:
        dist.broadcast(buf, src=comm._global(root), group=comm._group)
    mine = buf[comm.rank * nbytes : (comm.rank + 1) * nbytes].clone()
    return mine.view(dtype).reshape(out_shape)


# ---------------------------------------------------------------------------
# point to point
# ---------------------------------------------------------------------------
def send(comm: Comm, x: torch.Tensor, dest: int, tag: int) -> None:
    st = comm._cpu()
    payload = _bytes_view(x).clone()
    if dest == comm.rank:
        st.self_queue.append((tag, payload))
        return
    hdr = torch.tensor([tag, payload.numel(), codes.DTYPE_CODE.get(x.dtype, -1), _MAGIC],
                       dtype=torch.int64)
    g = comm._global(dest)
    w1 = dist.isend(hdr, dst=g, group=comm._group)
    st.pending.append((w1, hdr))
    if payload.numel() > 0:
        w2 = dist.isend(payload, dst=g, group=comm._group)
        st.pending.append((w2, payload))
    st.prune()


def _pull_one(comm: Comm, source: int):
    """Blocking receive of the next (tag, payload) from ``source`` (rank in comm)."""
    hdr = torch.empty(_HDR_WORDS, dtype=torch.int64)
    dist.recv(hdr, src=comm._global(source), group=comm._group)
    if int(hdr[3]) != _MAGIC:
        raise RuntimeError("mpi4jax_b200 CPU p2p protocol error (foreign traffic on the group?)")
    payload = torch.empty(int(hdr[1]), dtype=torch.uint8)
    if payload.numel() > 0:
        dist.recv(payload, src=comm._global(source), group=comm._group)
    return int(hdr[0]), payload


def _match(queue: deque, tag: int):
    for k, (t, payload) in enumerate(queue):
        if tag == ANY_TAG or t == tag:
            del queue[k]
            return t, payload
    return None


def recv_bytes(comm: Comm, source: int, tag: int):
    """Blocking matched receive of one message: returns ``(source, tag, payload uint8 tensor)``."""
    st = comm._cpu()
    got = None
    src = source
    if source == comm.rank or (source == ANY_SOURCE and st.self_queue):
        got = _match(st.self_queue, tag)
        if got is not None:
            src = comm.rank
        elif source == comm.rank:
            raise RuntimeError("recv from self: no matching message was sent (would deadlock)")
    if got is None and source != ANY_SOURCE:
        got = _match(st.unexpected[source], tag)
        while got is None:
            t, payload = _pull_one(comm, source)
            if tag == ANY_TAG or t == tag:
                got = (t, payload)
            else:
                st.unexpected[source].append((t, payload))
    if got is None:
        # ANY_SOURCE: first look at what already arrived, then take whoever sends next
        for q in range(comm.size):
            got = _match(st.unexpected[q], tag)
            if got is not None:
                src = q
                break
        while got is None:
            hdr = torch.empty(_HDR_WORDS, dtype=torch.int64)
            g = dist.recv(hdr, src=None, group=comm._group)
            q = comm._ranks.index(g)
            payload = torch.empty(int(hdr[1]), dtype=torch.uint8)
            if payload.numel() > 0:
                dist.recv(payload, src=g, group=comm._group)
            if tag == ANY_TAG or int(hdr[0]) == tag:
                got, src = (int(hdr[0]), payload), q
            else:
                st.unexpected[q].append((int(hdr[0]), payload))
    t, payload = got
    return src, t, payload


def recv(comm: Comm, template: torch.Tensor, source: int, tag: int,
         status: Optional[Status]) -> torch.Tensor:
    src, t, payload = recv_bytes(comm, source, tag)
    want = template.numel() * template.element_size()
    if payload.numel() != want:
        # same rule as the GPU transport (csrc/b2_p2p.cu: B2_ERR_TRUNCATE): the template fixes the message
        # size.  (MPI would accept a shorter message; the reference never relies on that, and a
        # transport-dependent answer is worse than a strict one.)
        raise RuntimeError(
            f"message size mismatch: received {payload.numel()} bytes into a {want}-byte buffer "
            "(send and recv must agree on the size, docs/sharp-bits.md)")
    out = torch.empty(template.shape, dtype=template.dtype)
    out.reshape(-1).view(torch.uint8)[:] = payload
    if status is not None:
        status._set(src, t, payload.numel(), template.element_size())
    return out


def send_object(comm: Comm, obj, dest: int, tag: int) -> None:
    """Pickle-based message (mpi4py's lower-case ``comm.send``)."""
    import pickle

    send(comm, torch.frombuffer(bytearray(pickle.dumps(obj)), dtype=torch.uint8), dest, tag)


def recv_object(comm: Comm, source: int, tag: int, status: Optional[Status]):
    import pickle

    src, t, payload = recv_bytes(comm, source, tag)
    if status is not None:
        status._set(src, t, payload.numel(), 1)
    return pickle.loads(payload.numpy().tobytes())


def sendrecv(comm: Comm, sendbuf: torch.Tensor, recv_template: torch.Tensor, source: int,
             dest: int, sendtag: int, recvtag: int, status: Optional[Status]) -> torch.Tensor:
    send(comm, sendbuf, dest, sendtag)         # eager -> cannot deadlock against the recv
    return recv(comm, recv_template, source, recvtag, status)


def log_call(rank: int, opname: str, details: str):
    """Debug trace with the reference's line format (mpi_ops_common.h:154-206)."""
    import random
    import string

    ident = "".join(random.choices(string.ascii_letters + string.digits, k=8))
    prefix = f"r{rank} | {ident} | MPI_{opname}"
    print(f"{prefix} {details}".rstrip(), flush=True)
    t0 = time.perf_counter()

    def done(code: int = 0):
        print(f"{prefix} done with code {code} ({time.perf_counter() - t0:.2e}s)", flush=True)

    return done
