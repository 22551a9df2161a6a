"""Backend dispatch for the 15 ops: CUDA tensors -> native kernels, CPU tensors -> gloo.

This is the analogue of the per-platform lowering registration each reference op does
(``register_lowering(..., platform="cpu"|"cuda"|"xpu")``, e.g.
/root/reference/mpi4jax/_src/collective_ops/allreduce.py:162-173): one op, several
device back ends, chosen by where the operand lives.
"""

from __future__ import annotations

import math
import operator
from typing import Optional

import torch

from .. import native
from ..backends import cpu as _cpu
from ..comm import Comm, Status
from ..native import codes


def _on_cpu(comm: Comm, opname: str, details: str, fn, *args):
    """``fn(comm, *args)``, a call of the CPU backend, between its ``MPI4JAX_DEBUG`` lines."""
    done = _cpu.log_call(comm.rank, opname, details) if native.get_logging() else None
    out = fn(comm, *args)
    if done:
        done()
    return out


def _rows_text(x: torch.Tensor) -> str:
    return f"with {x.shape[0]} rows of {math.prod(x.shape[1:]) * x.element_size()} bytes"


_is_wrapped = torch._C._functorch.is_functorch_wrapped_tensor


def _plain(x: torch.Tensor) -> torch.Tensor:
    """Backends need real storage (the CUDA path takes raw pointers).  A torch.func wrapper here
    means an op's autograd rule called the backend directly instead of going through a
    ``torch.autograd.Function`` (which peels the transform levels) -- caught on every backend so the
    CPU suite sees it too."""
    if _is_wrapped(x):
        raise RuntimeError("mpi4jax_b200 internal error: a torch.func-wrapped tensor reached the "
                           "communication backend; use run_opaque() / a differentiable op in the rule")
    return x


class _Opaque(torch.autograd.Function):
    """Runs ``fn(x)`` with the torch.func transform levels peeled off ``x``."""

    @staticmethod
    def forward(fn, x):
        out = fn(x)
        return x.new_empty(0) if out is None else out

    @staticmethod
    def setup_context(ctx, inputs, output):
        pass

    @staticmethod
    def backward(ctx, g):
        raise NotImplementedError("higher-order derivatives through this communication rule are not defined")

    @staticmethod
    def vmap(info, in_dims, fn, x):
        return _Opaque.apply(fn, x), in_dims[1]     # rank-wise elementwise rules: the batch rides along


def run_opaque(fn, x: torch.Tensor):
    """Call a non-differentiable backend function from inside an autograd rule (where ``x`` may be a
    GradTrackingTensor / BatchedTensor of an active torch.func transform)."""
    if _is_wrapped(x) or torch._C._functorch.peek_interpreter_stack() is not None:
        return _Opaque.apply(fn, x)
    return fn(x)


def _is_cuda(*tensors) -> bool:
    return any(t is not None and t.is_cuda for t in tensors)


def barrier(comm: Comm) -> None:
    if comm.device.type == "cuda":
        comm._native_comm().barrier()
        return
    _on_cpu(comm, "Barrier", "", _cpu.barrier)


def allreduce(comm: Comm, x: torch.Tensor, op_code: int, algo: int = codes.ALGO_AUTO) -> torch.Tensor:
    _plain(x)
    if x.is_cuda:
        return comm._native_comm().allreduce(x, op_code, algo)
    return _on_cpu(comm, "Allreduce", f"with {x.numel()} items", _cpu.allreduce, x, op_code)


def reduce(comm: Comm, x: torch.Tensor, op_code: int, root: int) -> Optional[torch.Tensor]:
    _plain(x)
    if x.is_cuda:
        return comm._native_comm().reduce(x, op_code, root)
    return _on_cpu(comm, "Reduce", f"with {x.numel()} items to root {root}", _cpu.reduce, x, op_code, root)


def scan(comm: Comm, x: torch.Tensor, op_code: int) -> torch.Tensor:
    _plain(x)
    if x.is_cuda:
        return comm._native_comm().scan(x, op_code)
    return _on_cpu(comm, "Scan", f"with {x.numel()} items", _cpu.scan, x, op_code)


def reduce_scatter(comm: Comm, x: torch.Tensor, op_code: int) -> torch.Tensor:
    _plain(x)
    if x.is_cuda:
        return comm._native_comm().reduce_scatter(x, op_code)
    return _on_cpu(comm, "Reduce_scatter_block", f"with {x.numel() // x.shape[0]} items per block",
                   _cpu.reduce_scatter, x, op_code)


def reduce_loc(comm: Comm, opcode: int, values: torch.Tensor, indices: torch.Tensor, op_code: int, root: int):
    """MAXLOC / MINLOC of ``(values, indices)`` pairs for the reduction collective ``opcode`` (collective_ops/_loc.py
    states the rule): ``(values, indices)``, or None off the root of a reduce."""
    _plain(values)
    _plain(indices)
    if values.is_cuda:
        return comm._native_comm().reduce_loc(opcode, values, indices, op_code, root)
    n = values.numel() // values.shape[0] if opcode == codes.OPC_REDUCE_SCATTER else values.numel()
    details = f"with {n} pairs" + (f" to root {root}" if opcode == codes.OPC_REDUCE else
                                   " per block" if opcode == codes.OPC_REDUCE_SCATTER else "")
    return _on_cpu(comm, codes.OPC_REDUCTION_NAME[opcode], details, _cpu.reduce_loc, opcode, values, indices, op_code,
                   root)


def allgather(comm: Comm, x: torch.Tensor) -> torch.Tensor:
    _plain(x)
    if x.is_cuda:
        return comm._native_comm().allgather(x)
    return _on_cpu(comm, "Allgather", f"sending {x.numel() * x.element_size()} bytes", _cpu.allgather, x)


def alltoall(comm: Comm, x: torch.Tensor) -> torch.Tensor:
    _plain(x)
    if x.is_cuda:
        return comm._native_comm().alltoall(x)
    return _on_cpu(comm, "Alltoall", f"with {x.numel()} items", _cpu.alltoall, x)


def check_rows(opname: str, x: torch.Tensor) -> None:
    if x.dim() == 0:
        raise ValueError(f"{opname} input must have shape (rows, ...)")


def as_counts(counts, x: torch.Tensor, scalar: bool = False) -> torch.Tensor:
    """One int (``scalar``) or a sequence of ints becomes an int64 tensor on x's device; tensors are
    checked, not moved."""
    if isinstance(counts, torch.Tensor):
        return counts
    value = operator.index(counts) if scalar else [operator.index(c) for c in counts]
    return torch.tensor(value, dtype=torch.int64, device=x.device)


def check_rowsv_args(opname: str, comm: Comm, x: torch.Tensor, counts: torch.Tensor, out_rows: int,
                     name: str) -> None:
    """Host-side checks of a variable-count call.  Every entry point (the op, its ``compiled`` twin, the raw
    ``torch.ops`` op and its fake kernel, the backends) passes through them: the kernel dereferences the
    counts as int64 values in x's device memory -- one for the ``count`` of allgatherv and gatherv,
    ``nproc`` for every other counts argument -- so anything else must be refused before the launch."""
    shape, shape_text = ((), "()") if name == "count" else ((comm.Get_size(),), "(nproc,)")
    check_rows(opname, x)
    if not isinstance(counts, torch.Tensor):
        raise TypeError(f"{opname} {name} must be an integer tensor (got {type(counts).__name__})")
    if counts.dtype.is_floating_point or counts.dtype.is_complex or counts.dtype == torch.bool:
        raise TypeError(f"{opname} {name} must be an integer tensor (got {counts.dtype})")
    if tuple(counts.shape) != shape:
        raise ValueError(f"{opname} {name} must have shape {shape_text} (got {tuple(counts.shape)})")
    if counts.device != x.device:
        raise ValueError(f"{opname} {name} must live on the device of x ({x.device}, got {counts.device})")
    if out_rows < 0:
        raise ValueError(f"{opname} recv_capacity must be >= 0 (got {out_rows})")


def rowsv_capacity(opname: str, comm: Comm, x: torch.Tensor, counts: torch.Tensor, recv_capacity,
                   name: str, fan_in: int):
    """The output rows of a public variable-count call or its ``compiled`` twin, after the checks:
    ``recv_capacity``, or by default ``fan_in * N``, the rows that never drop one -- ``fan_in`` is nproc for
    the gathering ops, 1 for reduce_scatterv (when every rank passes ``N`` rows) and scatterv."""
    check_rows(opname, x)
    out_rows = x.shape[0] * fan_in if recv_capacity is None else recv_capacity
    check_rowsv_args(opname, comm, x, counts, out_rows, name)
    return out_rows


def gatherv_capacity(comm: Comm, x: torch.Tensor, count: torch.Tensor, root: int, recv_capacity):
    """gatherv's output rows after the checks: the capacity is read on the root only, the other ranks
    receive nothing (0)."""
    if comm.Get_rank() == root:
        return rowsv_capacity("Gatherv", comm, x, count, recv_capacity, "count", comm.Get_size())
    check_rowsv_args("Gatherv", comm, x, count, 0, "count")
    return 0


def scatterv_capacity(comm: Comm, x: torch.Tensor, send_counts: Optional[torch.Tensor], root: int,
                      recv_capacity):
    """scatterv's output rows after the checks: ``send_counts`` are required on the root and may be None
    elsewhere; the capacity defaults to ``N`` and must be >= 0."""
    if send_counts is not None:
        return rowsv_capacity("Scatterv", comm, x, send_counts, recv_capacity, "send_counts", 1)
    if comm.Get_rank() == root:
        raise ValueError("Scatterv send_counts must be given on the root")
    check_rows("Scatterv", x)
    out_rows = x.shape[0] if recv_capacity is None else recv_capacity
    if out_rows < 0:
        raise ValueError(f"Scatterv recv_capacity must be >= 0 (got {out_rows})")
    return out_rows


def alltoallv(comm: Comm, x: torch.Tensor, send_counts: torch.Tensor, out_rows: int,
              place_counts: Optional[torch.Tensor] = None):
    _plain(x)
    check_rowsv_args("Alltoallv", comm, x, send_counts, out_rows, "send_counts")
    if place_counts is not None:
        check_rowsv_args("Alltoallv", comm, x, place_counts, out_rows, "place_counts")
    if x.is_cuda:
        return comm._native_comm().alltoallv(x, send_counts, out_rows, place_counts)
    return _on_cpu(comm, "Alltoallv", _rows_text(x), _cpu.alltoallv, x, send_counts, out_rows, place_counts)


def allgatherv(comm: Comm, x: torch.Tensor, count: torch.Tensor, out_rows: int,
               place_counts: Optional[torch.Tensor] = None):
    _plain(x)
    check_rowsv_args("Allgatherv", comm, x, count, out_rows, "count")
    if place_counts is not None:
        check_rowsv_args("Allgatherv", comm, x, place_counts, out_rows, "place_counts")
    if x.is_cuda:
        return comm._native_comm().allgatherv(x, count, out_rows, place_counts)
    return _on_cpu(comm, "Allgatherv", _rows_text(x), _cpu.allgatherv, x, count, out_rows, place_counts)


def reduce_scatterv(comm: Comm, x: torch.Tensor, send_counts: torch.Tensor, out_rows: int, op_code: int):
    _plain(x)
    check_rowsv_args("Reduce_scatterv", comm, x, send_counts, out_rows, "send_counts")
    if x.is_cuda:
        return comm._native_comm().reduce_scatterv(x, send_counts, out_rows, op_code)
    return _on_cpu(comm, "Reduce_scatterv", _rows_text(x), _cpu.reduce_scatterv, x, send_counts, out_rows, op_code)


def gatherv(comm: Comm, x: torch.Tensor, count: torch.Tensor, root: int, out_rows: int, max_rows: int,
            place_counts: Optional[torch.Tensor] = None):
    """``(out, recv_counts)``; ``out`` is None on the ranks other than ``root``, which read neither
    ``out_rows`` nor ``place_counts``.  ``max_rows``: the rows any rank may contribute, the same on every
    rank (it sizes the staging)."""
    _plain(x)
    is_root = comm.Get_rank() == root
    check_rowsv_args("Gatherv", comm, x, count, out_rows, "count")
    if place_counts is not None and is_root:
        check_rowsv_args("Gatherv", comm, x, place_counts, out_rows, "place_counts")
    if x.is_cuda:
        return comm._native_comm().gatherv(x, count, root, out_rows, max_rows, place_counts)
    return _on_cpu(comm, "Gatherv", f"{_rows_text(x)} to root {root}", _cpu.gatherv, x, count, root, out_rows,
                   max_rows, place_counts)


def scatterv(comm: Comm, x: torch.Tensor, send_counts: Optional[torch.Tensor], root: int, out_rows: int,
             max_rows: int):
    """``(out, recv_count)``.  ``x`` and ``send_counts`` are read on ``root`` only (elsewhere ``x`` gives
    the row shape and dtype, and ``send_counts`` may be None); ``max_rows``: the root rows that may be
    sent, the same on every rank (it sizes the staging)."""
    _plain(x)
    scatterv_capacity(comm, x, send_counts, root, out_rows)
    if x.is_cuda:
        return comm._native_comm().scatterv(x, send_counts, root, out_rows, max_rows)
    return _on_cpu(comm, "Scatterv", f"{_rows_text(x)} from root {root}", _cpu.scatterv, x, send_counts, root,
                   out_rows, max_rows)


def moe_dispatch(comm: Comm, x: torch.Tensor, order: torch.Tensor, send_counts: torch.Tensor, k: int,
                 num_experts: int, out_rows: int, with_plan: bool = True):
    """``(rows, recv_counts, pos, dest)`` of a top-k dispatch whose pairs are already sorted (ops/moe.py states
    the rules); ``with_plan`` False: the rows only, the rest None."""
    _plain(x)
    if x.is_cuda:
        return comm._native_comm().moe_dispatch(x, order, send_counts, k, num_experts, out_rows, with_plan)
    return _on_cpu(comm, "Moe_dispatch", f"with {order.shape[0]} pairs to {num_experts} experts", _cpu.moe_dispatch,
                   x, order, send_counts, k, num_experts, out_rows, with_plan)


def moe_combine(comm: Comm, y: torch.Tensor, pos: torch.Tensor, dest: torch.Tensor, weights: Optional[torch.Tensor],
                recv_counts: torch.Tensor, pairs: bool = False) -> torch.Tensor:
    _plain(y)
    if y.is_cuda:
        return comm._native_comm().moe_combine(y, pos, dest, weights, recv_counts, pairs)
    return _on_cpu(comm, "Moe_combine", f"with {pos.shape[0]} tokens x {pos.shape[1]} pairs", _cpu.moe_combine, y,
                   pos, dest, weights, recv_counts, pairs)


def bcast(comm: Comm, x: torch.Tensor, root: int) -> torch.Tensor:
    _plain(x)
    if x.is_cuda:
        return comm._native_comm().bcast(x, root)
    return _on_cpu(comm, "Bcast", f"{x.numel()} items from root {root}", _cpu.bcast, x, root)


def gather(comm: Comm, x: torch.Tensor, root: int) -> Optional[torch.Tensor]:
    _plain(x)
    if x.is_cuda:
        return comm._native_comm().gather(x, root)
    return _on_cpu(comm, "Gather", f"{x.numel()} items to root {root}", _cpu.gather, x, root)


def scatter(comm: Comm, x: torch.Tensor, root: int, out_shape, dtype) -> torch.Tensor:
    _plain(x)
    if x.is_cuda:
        return comm._native_comm().scatter(x, root, out_shape, dtype)
    return _on_cpu(comm, "Scatter", f"from root {root}", _cpu.scatter, x, root, out_shape, dtype)


def send(comm: Comm, x: torch.Tensor, dest: int, tag: int) -> None:
    _plain(x)
    if x.is_cuda:
        comm._native_comm().send(x, dest, tag)
        return
    _on_cpu(comm, "Send", f"{x.numel()} items to {dest} with tag {tag}", _cpu.send, x, dest, tag)


def recv(comm: Comm, template: torch.Tensor, source: int, tag: int,
         status: Optional[Status]) -> torch.Tensor:
    if template.is_cuda:
        return comm._native_comm().recv(template, source, tag, status)
    return _on_cpu(comm, "Recv", f"{template.numel()} items from {source} with tag {tag}", _cpu.recv, template,
                   source, tag, status)


def sendrecv(comm: Comm, sendbuf: torch.Tensor, recv_template: torch.Tensor, source: int,
             dest: int, sendtag: int, recvtag: int, status: Optional[Status]) -> torch.Tensor:
    if sendbuf.is_cuda != recv_template.is_cuda:
        raise ValueError("sendrecv: sendbuf and recvbuf must live on the same device type")
    if sendbuf.is_cuda:
        return comm._native_comm().sendrecv(sendbuf, recv_template, source, dest, sendtag,
                                            recvtag, status)
    return _on_cpu(comm, "Sendrecv", f"<{source} (tag {recvtag}) / >{dest} (tag {sendtag})", _cpu.sendrecv,
                   sendbuf, recv_template, source, dest, sendtag, recvtag, status)
