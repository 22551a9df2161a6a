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


def _log(comm: Comm, opname: str, details: str):
    if native.get_logging():
        return _cpu.log_call(comm.rank, opname, details)
    return None


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
    done = _log(comm, "Barrier", "")
    _cpu.barrier(comm)
    if done:
        done()


def allreduce(comm: Comm, x: torch.Tensor, op_code: int, algo: int = codes.ALGO_AUTO) -> torch.Tensor:
    _plain(x)
    if x.is_cuda:
        return comm._native_comm().allreduce(x, op_code, algo)
    done = _log(comm, "Allreduce", f"with {x.numel()} items")
    out = _cpu.allreduce(comm, x, op_code)
    if done:
        done()
    return out


def reduce(comm: Comm, x: torch.Tensor, op_code: int, root: int) -> Optional[torch.Tensor]:
    _plain(x)
    if x.is_cuda:
        return comm._native_comm().reduce(x, op_code, root)
    done = _log(comm, "Reduce", f"with {x.numel()} items to root {root}")
    out = _cpu.reduce(comm, x, op_code, root)
    if done:
        done()
    return out


def scan(comm: Comm, x: torch.Tensor, op_code: int) -> torch.Tensor:
    _plain(x)
    if x.is_cuda:
        return comm._native_comm().scan(x, op_code)
    done = _log(comm, "Scan", f"with {x.numel()} items")
    out = _cpu.scan(comm, x, op_code)
    if done:
        done()
    return out


def reduce_scatter(comm: Comm, x: torch.Tensor, op_code: int) -> torch.Tensor:
    _plain(x)
    if x.is_cuda:
        return comm._native_comm().reduce_scatter(x, op_code)
    done = _log(comm, "Reduce_scatter_block", f"with {x.numel() // x.shape[0]} items per block")
    out = _cpu.reduce_scatter(comm, x, op_code)
    if done:
        done()
    return out


def allgather(comm: Comm, x: torch.Tensor) -> torch.Tensor:
    _plain(x)
    if x.is_cuda:
        return comm._native_comm().allgather(x)
    done = _log(comm, "Allgather", f"sending {x.numel() * x.element_size()} bytes")
    out = _cpu.allgather(comm, x)
    if done:
        done()
    return out


def alltoall(comm: Comm, x: torch.Tensor) -> torch.Tensor:
    _plain(x)
    if x.is_cuda:
        return comm._native_comm().alltoall(x)
    done = _log(comm, "Alltoall", f"with {x.numel()} items")
    out = _cpu.alltoall(comm, x)
    if done:
        done()
    return out


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
                   name: str):
    """The output rows of a public variable-count call or its ``compiled`` twin, after the checks:
    ``recv_capacity``, or by default the rows that never drop one -- ``N * nproc`` for the gathering ops,
    ``N`` for reduce_scatterv (when every rank passes ``N`` rows) and scatterv."""
    check_rows(opname, x)
    if recv_capacity is not None:
        out_rows = recv_capacity
    else:
        out_rows = x.shape[0] * (1 if opname in ("Reduce_scatterv", "Scatterv") else comm.Get_size())
    check_rowsv_args(opname, comm, x, counts, out_rows, name)
    return out_rows


def _cpu_rowsv(opname: str, fn, comm: Comm, x: torch.Tensor, *args):
    """``fn(comm, x, *args)``, the CPU backend's alltoallv / allgatherv / reduce_scatterv, with its log line."""
    row_bytes = math.prod(x.shape[1:]) * x.element_size()
    done = _log(comm, opname, f"with {x.shape[0]} rows of {row_bytes} bytes")
    out = fn(comm, x, *args)
    if done:
        done()
    return out


def alltoallv(comm: Comm, x: torch.Tensor, send_counts: torch.Tensor, out_rows: int,
              place_counts: Optional[torch.Tensor] = None):
    _plain(x)
    check_rowsv_args("Alltoallv", comm, x, send_counts, out_rows, "send_counts")
    if place_counts is not None:
        check_rowsv_args("Alltoallv", comm, x, place_counts, out_rows, "place_counts")
    if x.is_cuda:
        return comm._native_comm().alltoallv(x, send_counts, out_rows, place_counts)
    return _cpu_rowsv("Alltoallv", _cpu.alltoallv, comm, x, send_counts, out_rows, place_counts)


def allgatherv(comm: Comm, x: torch.Tensor, count: torch.Tensor, out_rows: int,
               place_counts: Optional[torch.Tensor] = None):
    _plain(x)
    check_rowsv_args("Allgatherv", comm, x, count, out_rows, "count")
    if place_counts is not None:
        check_rowsv_args("Allgatherv", comm, x, place_counts, out_rows, "place_counts")
    if x.is_cuda:
        return comm._native_comm().allgatherv(x, count, out_rows, place_counts)
    return _cpu_rowsv("Allgatherv", _cpu.allgatherv, comm, x, count, out_rows, place_counts)


def reduce_scatterv(comm: Comm, x: torch.Tensor, send_counts: torch.Tensor, out_rows: int, op_code: int):
    _plain(x)
    check_rowsv_args("Reduce_scatterv", comm, x, send_counts, out_rows, "send_counts")
    if x.is_cuda:
        return comm._native_comm().reduce_scatterv(x, send_counts, out_rows, op_code)
    return _cpu_rowsv("Reduce_scatterv", _cpu.reduce_scatterv, comm, x, send_counts, out_rows, op_code)


def _cpu_rooted(opname: str, fn, comm: Comm, x: torch.Tensor, root: int, where: str, *args):
    """``fn(comm, x, *args)``, the CPU backend's gatherv / scatterv, with its log line."""
    row_bytes = math.prod(x.shape[1:]) * x.element_size()
    done = _log(comm, opname, f"with {x.shape[0]} rows of {row_bytes} bytes {where} root {root}")
    out = fn(comm, x, *args)
    if done:
        done()
    return out


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
    return _cpu_rooted("Gatherv", _cpu.gatherv, comm, x, root, "to", count, root, out_rows, max_rows, place_counts)


def scatterv(comm: Comm, x: torch.Tensor, send_counts: Optional[torch.Tensor], root: int, out_rows: int,
             max_rows: int):
    """``(out, recv_count)``.  ``x`` and ``send_counts`` are read on ``root`` only (elsewhere ``x`` gives
    the row shape and dtype, and ``send_counts`` may be None); ``max_rows``: the root rows that may be
    sent, the same on every rank (it sizes the staging)."""
    _plain(x)
    if send_counts is not None:
        check_rowsv_args("Scatterv", comm, x, send_counts, out_rows, "send_counts")
    elif comm.Get_rank() == root:
        raise ValueError("Scatterv send_counts must be given on the root")
    else:
        check_rows("Scatterv", x)
        if out_rows < 0:
            raise ValueError(f"Scatterv recv_capacity must be >= 0 (got {out_rows})")
    if x.is_cuda:
        return comm._native_comm().scatterv(x, send_counts, root, out_rows, max_rows)
    return _cpu_rooted("Scatterv", _cpu.scatterv, comm, x, root, "from", send_counts, root, out_rows, max_rows)


def bcast(comm: Comm, x: torch.Tensor, root: int) -> torch.Tensor:
    _plain(x)
    if x.is_cuda:
        return comm._native_comm().bcast(x, root)
    done = _log(comm, "Bcast", f"{x.numel()} items from root {root}")
    out = _cpu.bcast(comm, x, root)
    if done:
        done()
    return out


def gather(comm: Comm, x: torch.Tensor, root: int) -> Optional[torch.Tensor]:
    _plain(x)
    if x.is_cuda:
        return comm._native_comm().gather(x, root)
    done = _log(comm, "Gather", f"{x.numel()} items to root {root}")
    out = _cpu.gather(comm, x, root)
    if done:
        done()
    return out


def scatter(comm: Comm, x: torch.Tensor, root: int, out_shape, dtype) -> torch.Tensor:
    _plain(x)
    if x.is_cuda:
        return comm._native_comm().scatter(x, root, out_shape, dtype)
    done = _log(comm, "Scatter", f"from root {root}")
    out = _cpu.scatter(comm, x, root, out_shape, dtype)
    if done:
        done()
    return out


def send(comm: Comm, x: torch.Tensor, dest: int, tag: int) -> None:
    _plain(x)
    if x.is_cuda:
        comm._native_comm().send(x, dest, tag)
        return
    done = _log(comm, "Send", f"{x.numel()} items to {dest} with tag {tag}")
    _cpu.send(comm, x, dest, tag)
    if done:
        done()


def recv(comm: Comm, template: torch.Tensor, source: int, tag: int,
         status: Optional[Status]) -> torch.Tensor:
    if template.is_cuda:
        return comm._native_comm().recv(template, source, tag, status)
    done = _log(comm, "Recv", f"{template.numel()} items from {source} with tag {tag}")
    out = _cpu.recv(comm, template, source, tag, status)
    if done:
        done()
    return out


def sendrecv(comm: Comm, sendbuf: torch.Tensor, recv_template: torch.Tensor, source: int,
             dest: int, sendtag: int, recvtag: int, status: Optional[Status]) -> torch.Tensor:
    if sendbuf.is_cuda != recv_template.is_cuda:
        raise ValueError("sendrecv: sendbuf and recvbuf must live on the same device type")
    if sendbuf.is_cuda:
        return comm._native_comm().sendrecv(sendbuf, recv_template, source, dest, sendtag,
                                            recvtag, status)
    done = _log(comm, "Sendrecv", f"<{source} (tag {recvtag}) / >{dest} (tag {sendtag})")
    out = _cpu.sendrecv(comm, sendbuf, recv_template, source, dest, sendtag, recvtag, status)
    if done:
        done()
    return out
