"""``torch.library`` registration of the ops -- the traceable frontend.

The reference's ops are JAX *primitives*: abstract-eval rules give shapes, an ordered effect
threads a token through every custom call so XLA keeps them in program order
(/root/reference/mpi4jax/_src/utils.py:45-53, jax_compat.py:82-100, e.g. allreduce.py:87-111).
The torch analogue: every op is a ``torch.library.custom_op`` with a fake (meta) kernel =
the abstract-eval rule, and is registered as an **ORDERED effectful op**
(``torch._higher_order_ops.effects``), which makes AOTAutograd thread effect tokens through
them exactly like JAX does -- ``send`` (no result) and ``barrier`` (no operands) can neither be
dead-code-eliminated nor reordered inside ``torch.compile(fullgraph=True)``.

The eager/CUDA-graph path (``mpi4jax_b200.jit``) does not need any of this; it is provided so
that functions using the ops can be traced by ``torch.compile`` / ``torch.export``:

    from mpi4jax_b200 import compiled as mc
    f = torch.compile(lambda x: mc.allreduce(x, MPI.SUM, comm=comm), fullgraph=True)

Communicators and reduction ops travel through the graph as plain integers (comm id, op code),
the counterpart of the reference's int64 handle attributes.
"""

from __future__ import annotations

from typing import Optional

import torch
from torch.library import custom_op

from . import comm as _comm_mod
from .collective_ops import _adjoints, _dispatch, _loc
from .comm import ANY_SOURCE, ANY_TAG, SUM, Comm, as_op
from .native import codes
from .utils import get_default_comm

def _register(comm: Optional[Comm]) -> int:
    """Communicator -> integer graph attribute.  No registration side effect here: Dynamo defers
    Python side effects of a traced frame until after the graph has run, so the lookup table must
    exist beforehand -- it is the registry every ``Comm`` enters at construction."""
    comm = comm or get_default_comm()
    return comm._id


def _c(comm_id: int) -> Comm:
    for comm in list(_comm_mod._comm_registry):
        if comm._id == comm_id:
            return comm
    raise RuntimeError(f"mpi4jax_b200: communicator #{comm_id} no longer exists (it was freed or garbage "
                       "collected after the function using it was compiled)")


def _st(status_id: int):
    """Status id -> object (0 = no status requested)."""
    if status_id == 0:
        return None
    st = _comm_mod._status_registry.get(status_id)
    if st is None:
        raise RuntimeError(f"mpi4jax_b200: Status #{status_id} was garbage collected after the function "
                           "using it was compiled; keep a reference to it")
    return st


def _rowsv_fake(opname: str, comm: Comm, x, counts, name: str, out_rows: int, place_counts=None,
                counts_shape=None):
    """A variable-count op's fake kernel: the backends' checks of ``counts`` and ``place_counts`` (each when
    given) against ``out_rows``, then ``(out, out_counts)``: ``out_rows`` rows like ``x`` and int64 counts of
    ``counts_shape`` (default ``(nproc,)``)."""
    if counts is not None:
        _dispatch.check_rowsv_args(opname, comm, x, counts, out_rows, name)
    if place_counts is not None:
        _dispatch.check_rowsv_args(opname, comm, x, place_counts, out_rows, "place_counts")
    counts_shape = (comm.Get_size(),) if counts_shape is None else counts_shape
    return x.new_empty((out_rows, *x.shape[1:])), x.new_empty(counts_shape, dtype=torch.int64)


# ---------------------------------------------------------------- op definitions
@custom_op("mpi4jax_b200::allreduce", mutates_args=())
def _allreduce(x: torch.Tensor, op: int, comm_id: int) -> torch.Tensor:
    return _dispatch.allreduce(_c(comm_id), x.contiguous(), op, codes.ALGO_AUTO)


@_allreduce.register_fake
def _(x, op, comm_id):
    return torch.empty_like(x, memory_format=torch.contiguous_format)


def _allreduce_setup(ctx, inputs, output):
    _, ctx.op, ctx.comm_id = inputs


def _allreduce_backward(ctx, g):
    if ctx.op != SUM.code:
        raise NotImplementedError("The adjoint of allreduce is only defined for SUM")
    return g, None, None            # transpose of allreduce(SUM) = identity on the local cotangent


_allreduce.register_autograd(_allreduce_backward, setup_context=_allreduce_setup)


@custom_op("mpi4jax_b200::reduce_scatter", mutates_args=())
def _reduce_scatter(x: torch.Tensor, op: int, comm_id: int) -> torch.Tensor:
    return _dispatch.reduce_scatter(_c(comm_id), x.contiguous(), op)


@_reduce_scatter.register_fake
def _(x, op, comm_id):
    return x.new_empty(x.shape[1:])


def _reduce_scatter_setup(ctx, inputs, output):
    _, ctx.op, ctx.comm_id = inputs


def _reduce_scatter_backward(ctx, g):
    if ctx.op != SUM.code:
        raise NotImplementedError("The adjoint of reduce_scatter is only defined for SUM")
    return _adjoints.reduce_scatter(compiled, g, _c(ctx.comm_id)), None, None


_reduce_scatter.register_autograd(_reduce_scatter_backward, setup_context=_reduce_scatter_setup)


@custom_op("mpi4jax_b200::reduce_loc", mutates_args=())
def _reduce_loc(values: torch.Tensor, indices: torch.Tensor, op: int, kind: int, root: int,
                comm_id: int) -> tuple[torch.Tensor, torch.Tensor]:
    # MAXLOC / MINLOC of (values, indices) pairs; `kind`: the collective's opcode.  Off the root of a reduce:
    # copies of the input pair.  No autograd rule: the eager op has none either.
    out = _dispatch.reduce_loc(_c(comm_id), kind, values.contiguous(), indices.contiguous(), op, root)
    return (values.clone(), indices.clone()) if out is None else out


@_reduce_loc.register_fake
def _(values, indices, op, kind, root, comm_id):
    shape = values.shape[1:] if kind == codes.OPC_REDUCE_SCATTER else values.shape
    return values.new_empty(shape), indices.new_empty(shape)


@custom_op("mpi4jax_b200::allgather", mutates_args=())
def _allgather(x: torch.Tensor, comm_id: int, size: int) -> torch.Tensor:
    return _dispatch.allgather(_c(comm_id), x.contiguous())


@_allgather.register_fake
def _(x, comm_id, size):
    return x.new_empty((size, *x.shape))


def _allgather_setup(ctx, inputs, output):
    _, ctx.comm_id, _ = inputs


def _allgather_backward(ctx, g):
    return _adjoints.allgather(compiled, g, _c(ctx.comm_id)), None, None


_allgather.register_autograd(_allgather_backward, setup_context=_allgather_setup)


@custom_op("mpi4jax_b200::alltoall", mutates_args=())
def _alltoall(x: torch.Tensor, comm_id: int) -> torch.Tensor:
    return _dispatch.alltoall(_c(comm_id), x.contiguous())


@_alltoall.register_fake
def _(x, comm_id):
    return torch.empty_like(x, memory_format=torch.contiguous_format)


def _alltoall_setup(ctx, inputs, output):
    _, ctx.comm_id = inputs


def _alltoall_backward(ctx, g):
    return _adjoints.alltoall(compiled, g, _c(ctx.comm_id)), None


_alltoall.register_autograd(_alltoall_backward, setup_context=_alltoall_setup)


@custom_op("mpi4jax_b200::alltoallv", mutates_args=())
def _alltoallv(x: torch.Tensor, send_counts: torch.Tensor, out_rows: int, place_counts: Optional[torch.Tensor],
               comm_id: int) -> tuple[torch.Tensor, torch.Tensor]:
    return _dispatch.alltoallv(_c(comm_id), x.contiguous(), send_counts, out_rows, place_counts)


@_alltoallv.register_fake
def _(x, send_counts, out_rows, place_counts, comm_id):
    return _rowsv_fake("Alltoallv", _c(comm_id), x, send_counts, "send_counts", out_rows)


def _alltoallv_setup(ctx, inputs, output):
    x, send_counts, _, place_counts, ctx.comm_id = inputs
    ctx.in_rows = x.shape[0]
    ctx.save_for_backward(send_counts, place_counts, output[1])


def _alltoallv_backward(ctx, g, _g_counts):
    send_counts, place_counts, recv_counts = ctx.saved_tensors
    back = _adjoints.alltoallv(compiled, g, _c(ctx.comm_id), ctx.in_rows, send_counts, recv_counts, place_counts)
    return back, None, None, None, None


_alltoallv.register_autograd(_alltoallv_backward, setup_context=_alltoallv_setup)


@custom_op("mpi4jax_b200::allgatherv", mutates_args=())
def _allgatherv(x: torch.Tensor, count: torch.Tensor, out_rows: int, comm_id: int,
                place_counts: Optional[torch.Tensor] = None) -> tuple[torch.Tensor, torch.Tensor]:
    return _dispatch.allgatherv(_c(comm_id), x.contiguous(), count, out_rows, place_counts)


@_allgatherv.register_fake
def _(x, count, out_rows, comm_id, place_counts=None):
    return _rowsv_fake("Allgatherv", _c(comm_id), x, count, "count", out_rows, place_counts)


def _allgatherv_setup(ctx, inputs, output):
    x, _, _, ctx.comm_id, place_counts = inputs
    ctx.in_rows = x.shape[0]
    ctx.save_for_backward(output[1], place_counts)


def _allgatherv_backward(ctx, g, _g_counts):
    recv_counts, place_counts = ctx.saved_tensors
    counts = recv_counts if place_counts is None else place_counts
    return _adjoints.allgatherv(compiled, g, _c(ctx.comm_id), ctx.in_rows, counts), None, None, None, None


_allgatherv.register_autograd(_allgatherv_backward, setup_context=_allgatherv_setup)


@custom_op("mpi4jax_b200::reduce_scatterv", mutates_args=())
def _reduce_scatterv(x: torch.Tensor, send_counts: torch.Tensor, out_rows: int, op: int,
                     comm_id: int) -> tuple[torch.Tensor, torch.Tensor]:
    return _dispatch.reduce_scatterv(_c(comm_id), x.contiguous(), send_counts, out_rows, op)


@_reduce_scatterv.register_fake
def _(x, send_counts, out_rows, op, comm_id):
    return _rowsv_fake("Reduce_scatterv", _c(comm_id), x, send_counts, "send_counts", out_rows)


def _reduce_scatterv_setup(ctx, inputs, output):
    x, send_counts, _, ctx.op, ctx.comm_id = inputs
    ctx.in_rows = x.shape[0]
    ctx.save_for_backward(send_counts)


def _reduce_scatterv_backward(ctx, g, _g_counts):
    if ctx.op != SUM.code:
        raise NotImplementedError("The adjoint of reduce_scatterv is only defined for SUM")
    (send_counts,) = ctx.saved_tensors
    return _adjoints.reduce_scatterv(compiled, g, _c(ctx.comm_id), ctx.in_rows, send_counts), None, None, None, None


_reduce_scatterv.register_autograd(_reduce_scatterv_backward, setup_context=_reduce_scatterv_setup)


@custom_op("mpi4jax_b200::bcast", mutates_args=())
def _bcast(x: torch.Tensor, root: int, comm_id: int) -> torch.Tensor:
    out = _dispatch.bcast(_c(comm_id), x.contiguous(), root)
    return out.clone() if out.data_ptr() == x.data_ptr() else out   # custom ops may not alias inputs


@_bcast.register_fake
def _(x, root, comm_id):
    return torch.empty_like(x, memory_format=torch.contiguous_format)


def _bcast_setup(ctx, inputs, output):
    _, ctx.root, ctx.comm_id = inputs


def _bcast_backward(ctx, g):
    return _adjoints.bcast(compiled, g, ctx.root, _c(ctx.comm_id)), None, None


_bcast.register_autograd(_bcast_backward, setup_context=_bcast_setup)


@custom_op("mpi4jax_b200::scan", mutates_args=())
def _scan(x: torch.Tensor, op: int, comm_id: int) -> torch.Tensor:
    return _dispatch.scan(_c(comm_id), x.contiguous(), op)


@_scan.register_fake
def _(x, op, comm_id):
    return torch.empty_like(x, memory_format=torch.contiguous_format)


@custom_op("mpi4jax_b200::reduce", mutates_args=())
def _reduce(x: torch.Tensor, op: int, root: int, comm_id: int) -> torch.Tensor:
    comm = _c(comm_id)
    out = _dispatch.reduce(comm, x.contiguous(), op, root)
    return out if comm.Get_rank() == root else x.clone()


@_reduce.register_fake
def _(x, op, root, comm_id):
    return torch.empty_like(x, memory_format=torch.contiguous_format)


@custom_op("mpi4jax_b200::gather_root", mutates_args=())
def _gather_root(x: torch.Tensor, root: int, comm_id: int, size: int) -> torch.Tensor:
    return _dispatch.gather(_c(comm_id), x.contiguous(), root)


@_gather_root.register_fake
def _(x, root, comm_id, size):
    return x.new_empty((size, *x.shape))


@custom_op("mpi4jax_b200::gather_leaf", mutates_args=())
def _gather_leaf(x: torch.Tensor, root: int, comm_id: int) -> torch.Tensor:
    _dispatch.gather(_c(comm_id), x.contiguous(), root)
    return x.clone()


@_gather_leaf.register_fake
def _(x, root, comm_id):
    return torch.empty_like(x, memory_format=torch.contiguous_format)


@custom_op("mpi4jax_b200::gatherv_root", mutates_args=())
def _gatherv_root(x: torch.Tensor, count: torch.Tensor, root: int, out_rows: int, max_rows: int, comm_id: int,
                  reverse: bool, place_counts: Optional[torch.Tensor] = None) -> tuple[torch.Tensor, torch.Tensor]:
    # the root's output; in the reverse mode (scatterv's adjoint) also run on the other ranks, which get zeros
    comm = _c(comm_id)
    out, recv_counts = _dispatch.gatherv(comm, x.contiguous(), count, root, out_rows, max_rows, place_counts)
    return (out if comm.Get_rank() == root else x.new_zeros((out_rows, *x.shape[1:]))), recv_counts


@_gatherv_root.register_fake
def _(x, count, root, out_rows, max_rows, comm_id, reverse, place_counts=None):
    return _rowsv_fake("Gatherv", _c(comm_id), x, count, "count", out_rows, place_counts)


def _gatherv_root_setup(ctx, inputs, output):
    x, _, ctx.root, _, ctx.max_rows, ctx.comm_id, ctx.reverse, place_counts = inputs
    ctx.in_rows = x.shape[0]
    ctx.save_for_backward(output[1], place_counts)


def _gatherv_root_backward(ctx, g, _g_counts):
    recv_counts, place_counts = ctx.saved_tensors
    comm = _c(ctx.comm_id)
    if ctx.reverse:
        back = _adjoints.gatherv_reverse(compiled, g, comm, ctx.root, ctx.in_rows, ctx.max_rows, place_counts)
    else:
        back = _adjoints.gatherv(compiled, g, comm, ctx.root, ctx.in_rows, ctx.max_rows, recv_counts)
    return back, None, None, None, None, None, None, None


_gatherv_root.register_autograd(_gatherv_root_backward, setup_context=_gatherv_root_setup)


@custom_op("mpi4jax_b200::gatherv_leaf", mutates_args=())
def _gatherv_leaf(x: torch.Tensor, count: torch.Tensor, root: int, max_rows: int,
                  comm_id: int) -> tuple[torch.Tensor, torch.Tensor]:
    _, recv_counts = _dispatch.gatherv(_c(comm_id), x.contiguous(), count, root, 0, max_rows)
    return x.clone(), recv_counts


@_gatherv_leaf.register_fake
def _(x, count, root, max_rows, comm_id):
    _, recv_counts = _rowsv_fake("Gatherv", _c(comm_id), x, count, "count", 0)
    return torch.empty_like(x, memory_format=torch.contiguous_format), recv_counts


def _gatherv_leaf_setup(ctx, inputs, output):
    x, _, ctx.root, ctx.max_rows, ctx.comm_id = inputs
    ctx.in_rows = x.shape[0]


def _gatherv_leaf_backward(ctx, g, _g_counts):
    back = _adjoints.gatherv(compiled, g, _c(ctx.comm_id), ctx.root, ctx.in_rows, ctx.max_rows, None)
    return back, None, None, None, None


_gatherv_leaf.register_autograd(_gatherv_leaf_backward, setup_context=_gatherv_leaf_setup)


@custom_op("mpi4jax_b200::scatterv", mutates_args=())
def _scatterv(x: torch.Tensor, send_counts: Optional[torch.Tensor], root: int, out_rows: int, max_rows: int,
              comm_id: int) -> tuple[torch.Tensor, torch.Tensor]:
    return _dispatch.scatterv(_c(comm_id), x.contiguous(), send_counts, root, out_rows, max_rows)


@_scatterv.register_fake
def _(x, send_counts, root, out_rows, max_rows, comm_id):
    comm = _c(comm_id)
    _dispatch.scatterv_capacity(comm, x, send_counts, root, out_rows)
    return _rowsv_fake("Scatterv", comm, x, send_counts, "send_counts", out_rows, counts_shape=())


def _scatterv_setup(ctx, inputs, output):
    x, send_counts, ctx.root, _, ctx.max_rows, ctx.comm_id = inputs
    ctx.in_rows = x.shape[0]
    ctx.save_for_backward(send_counts, output[1])


def _scatterv_backward(ctx, g, _g_count):
    send_counts, recv_count = ctx.saved_tensors
    back = _adjoints.scatterv(compiled, g, _c(ctx.comm_id), ctx.root, ctx.in_rows, ctx.max_rows, recv_count,
                              send_counts)
    return back, None, None, None, None, None


_scatterv.register_autograd(_scatterv_backward, setup_context=_scatterv_setup)


@custom_op("mpi4jax_b200::scatter", mutates_args=())
def _scatter(x: torch.Tensor, root: int, comm_id: int, is_root: bool) -> torch.Tensor:
    shape = tuple(x.shape[1:]) if is_root else tuple(x.shape)
    return _dispatch.scatter(_c(comm_id), x.contiguous(), root, shape, x.dtype)


@_scatter.register_fake
def _(x, root, comm_id, is_root):
    return x.new_empty(tuple(x.shape[1:]) if is_root else tuple(x.shape))


@custom_op("mpi4jax_b200::barrier", mutates_args=())
def _barrier(comm_id: int) -> None:
    _dispatch.barrier(_c(comm_id))


@_barrier.register_fake
def _(comm_id):
    return None


@custom_op("mpi4jax_b200::send", mutates_args=())
def _send(x: torch.Tensor, dest: int, tag: int, comm_id: int) -> None:
    _dispatch.send(_c(comm_id), x.contiguous(), dest, tag)


@_send.register_fake
def _(x, dest, tag, comm_id):
    return None


@custom_op("mpi4jax_b200::recv", mutates_args=())
def _recv(template: torch.Tensor, source: int, tag: int, comm_id: int, status_id: int) -> torch.Tensor:
    return _dispatch.recv(_c(comm_id), template, source, tag, _st(status_id))


@_recv.register_fake
def _(template, source, tag, comm_id, status_id):
    return torch.empty_like(template, memory_format=torch.contiguous_format)


@custom_op("mpi4jax_b200::sendrecv", mutates_args=())
def _sendrecv(sendbuf: torch.Tensor, recvbuf: torch.Tensor, source: int, dest: int, sendtag: int,
              recvtag: int, comm_id: int, status_id: int) -> torch.Tensor:
    return _dispatch.sendrecv(_c(comm_id), sendbuf.contiguous(), recvbuf, source, dest, sendtag, recvtag,
                              _st(status_id))


@_sendrecv.register_fake
def _(sendbuf, recvbuf, source, dest, sendtag, recvtag, comm_id, status_id):
    return torch.empty_like(recvbuf, memory_format=torch.contiguous_format)


def _sendrecv_setup(ctx, inputs, output):
    sendbuf, _, ctx.source, ctx.dest, ctx.sendtag, ctx.recvtag, ctx.comm_id, _ = inputs
    ctx.send_meta = (tuple(sendbuf.shape), sendbuf.dtype, sendbuf.device)


def _sendrecv_backward(ctx, g):
    shape, dtype, device = ctx.send_meta
    template = torch.empty(shape, dtype=dtype, device=device)
    back = _adjoints.sendrecv(compiled, g, template, ctx.source, ctx.dest, ctx.sendtag, ctx.recvtag,
                              _c(ctx.comm_id))
    return back, None, None, None, None, None, None, None


_sendrecv.register_autograd(_sendrecv_backward, setup_context=_sendrecv_setup)


ALL_OPS = ("allreduce", "allgather", "alltoall", "bcast", "scan", "reduce", "gather_root", "gather_leaf",
           "scatter", "barrier", "send", "recv", "sendrecv", "reduce_scatter", "alltoallv", "allgatherv",
           "reduce_scatterv", "gatherv_root", "gatherv_leaf", "scatterv", "reduce_loc")
ORDERED_EFFECT = False
try:  # the ordered effect: AOTAutograd threads a token through these ops in program order
    from torch._higher_order_ops.effects import _EffectType, _register_effectful_op

    for _name in ALL_OPS:
        _register_effectful_op(f"mpi4jax_b200::{_name}", _EffectType.ORDERED)
    ORDERED_EFFECT = True
except Exception:  # pragma: no cover - private API moved; ops then still rely on "has side effects"
    pass


# ---------------------------------------------------------------- public, traceable wrappers
class compiled:
    """Namespace of ``torch.compile``-traceable ops (static arguments are plain Python values)."""

    @staticmethod
    def allreduce(x, op, *, comm=None):
        """With ``MPI.MAXLOC`` / ``MPI.MINLOC``, ``x`` and the result are ``(values, indices)`` pairs (the
        ``reduce_loc`` op); the same holds for ``reduce``, ``scan`` and ``reduce_scatter``."""
        op = as_op(op)
        if _loc.is_loc(op):
            return _loc.compiled_loc("allreduce", codes.OPC_ALLREDUCE, x, op, comm or get_default_comm())
        return torch.ops.mpi4jax_b200.allreduce(x, op.code, _register(comm))

    @staticmethod
    def reduce_scatter(x, op, *, comm=None):
        comm = comm or get_default_comm()
        op = as_op(op)
        if _loc.is_loc(op):
            return _loc.compiled_loc("reduce_scatter", codes.OPC_REDUCE_SCATTER, x, op, comm)
        if x.dim() == 0 or x.shape[0] != comm.Get_size():
            raise ValueError("Reduce_scatter input must have shape (nproc, ...)")
        return torch.ops.mpi4jax_b200.reduce_scatter(x, op.code, comm._id)

    @staticmethod
    def allgather(x, *, comm=None):
        comm = comm or get_default_comm()     # plain attribute reads only: this code is traced by Dynamo
        return torch.ops.mpi4jax_b200.allgather(x, comm._id, comm.Get_size())

    @staticmethod
    def alltoall(x, *, comm=None):
        return torch.ops.mpi4jax_b200.alltoall(x, _register(comm))

    @staticmethod
    def alltoallv(x, send_counts, *, recv_capacity=None, comm=None):
        """``(out, recv_counts)`` of :func:`mpi4jax_b200.alltoallv`; ``send_counts`` must be a device
        tensor of shape ``(nproc,)``."""
        comm = comm or get_default_comm()
        cap = _dispatch.rowsv_capacity("Alltoallv", comm, x, send_counts, recv_capacity, "send_counts",
                                       comm.Get_size())
        return torch.ops.mpi4jax_b200.alltoallv(x, send_counts, cap, None, comm._id)

    @staticmethod
    def _alltoallv_reverse(y, recv_counts, send_counts, rows, comm):
        # the counterpart of the eager alltoallv_reverse, for alltoallv's adjoint (collective_ops/_adjoints.py)
        return torch.ops.mpi4jax_b200.alltoallv(y, recv_counts, rows, send_counts, comm._id)[0]

    @staticmethod
    def allgatherv(x, count, *, recv_capacity=None, comm=None):
        """``(out, recv_counts)`` of :func:`mpi4jax_b200.allgatherv`; ``count`` must be an integer device
        tensor of shape ``()``."""
        comm = comm or get_default_comm()
        cap = _dispatch.rowsv_capacity("Allgatherv", comm, x, count, recv_capacity, "count", comm.Get_size())
        return torch.ops.mpi4jax_b200.allgatherv(x, count, cap, comm._id)

    @staticmethod
    def _allgatherv_reverse(y, place_counts, rows, comm):
        # the counterpart of the eager allgatherv_reverse, for reduce_scatterv's adjoint (collective_ops/_adjoints.py)
        count = torch.full((), y.shape[0], dtype=torch.int64, device=y.device)
        return torch.ops.mpi4jax_b200.allgatherv(y, count, rows, comm._id, place_counts)[0]

    @staticmethod
    def reduce_scatterv(x, send_counts, op, *, recv_capacity=None, comm=None):
        """``(out, recv_counts)`` of :func:`mpi4jax_b200.reduce_scatterv` for the built-in operators;
        ``send_counts`` must be a device tensor of shape ``(nproc,)``."""
        comm = comm or get_default_comm()
        op = as_op(op)
        _loc.refuse(op, "reduce_scatterv")
        cap = _dispatch.rowsv_capacity("Reduce_scatterv", comm, x, send_counts, recv_capacity, "send_counts", 1)
        return torch.ops.mpi4jax_b200.reduce_scatterv(x, send_counts, cap, op.code, comm._id)

    @staticmethod
    def gatherv(x, count, root, *, recv_capacity=None, comm=None):
        """``(out, recv_counts)`` of :func:`mpi4jax_b200.gatherv`; ``count`` must be an integer device tensor
        of shape ``()``.  On the root the ``gatherv_root`` op, elsewhere ``gatherv_leaf``, whose result is a
        copy of ``x``."""
        comm = comm or get_default_comm()
        cap = _dispatch.gatherv_capacity(comm, x, count, root, recv_capacity)
        if comm.Get_rank() == root:
            return torch.ops.mpi4jax_b200.gatherv_root(x, count, int(root), cap, x.shape[0], comm._id, False)
        return torch.ops.mpi4jax_b200.gatherv_leaf(x, count, int(root), x.shape[0], comm._id)

    @staticmethod
    def _gatherv_reverse(y, count, place_counts, root, rows, max_rows, comm):
        # the counterpart of the eager gatherv_reverse, for scatterv's adjoint (collective_ops/_adjoints.py)
        if comm.Get_rank() != root:
            place_counts = None
        return torch.ops.mpi4jax_b200.gatherv_root(y, count, root, rows, max_rows, comm._id, True, place_counts)[0]

    @staticmethod
    def scatterv(x, send_counts, root, *, recv_capacity=None, comm=None):
        """``(out, recv_count)`` of :func:`mpi4jax_b200.scatterv`; ``send_counts`` must be a device tensor of
        shape ``(nproc,)`` on the root (None or such a tensor elsewhere)."""
        comm = comm or get_default_comm()
        _dispatch.check_rows("Scatterv", x)
        cap = _dispatch.scatterv_capacity(comm, x, send_counts, root, recv_capacity)
        return torch.ops.mpi4jax_b200.scatterv(x, send_counts, int(root), cap, x.shape[0], comm._id)

    @staticmethod
    def _scatterv_bounded(x, send_counts, root, rows, max_rows, comm):
        # the counterpart of the eager scatterv_bounded, for gatherv's adjoint (collective_ops/_adjoints.py)
        return torch.ops.mpi4jax_b200.scatterv(x, send_counts, root, rows, max_rows, comm._id)[0]

    @staticmethod
    def bcast(x, root, *, comm=None):
        return torch.ops.mpi4jax_b200.bcast(x, int(root), _register(comm))

    @staticmethod
    def scan(x, op, *, comm=None):
        op = as_op(op)
        if _loc.is_loc(op):
            return _loc.compiled_loc("scan", codes.OPC_SCAN, x, op, comm or get_default_comm())
        return torch.ops.mpi4jax_b200.scan(x, op.code, _register(comm))

    @staticmethod
    def reduce(x, op, root, *, comm=None):
        op = as_op(op)
        if _loc.is_loc(op):
            return _loc.compiled_loc("reduce", codes.OPC_REDUCE, x, op, comm or get_default_comm(), root)
        return torch.ops.mpi4jax_b200.reduce(x, op.code, int(root), _register(comm))

    @staticmethod
    def gather(x, root, *, comm=None):
        comm = comm or get_default_comm()
        if comm.Get_rank() == root:
            return torch.ops.mpi4jax_b200.gather_root(x, int(root), comm._id, comm.Get_size())
        return torch.ops.mpi4jax_b200.gather_leaf(x, int(root), comm._id)

    @staticmethod
    def scatter(x, root, *, comm=None):
        comm = comm or get_default_comm()
        return torch.ops.mpi4jax_b200.scatter(x, int(root), comm._id, comm.Get_rank() == root)

    @staticmethod
    def barrier(*, comm=None):
        torch.ops.mpi4jax_b200.barrier(_register(comm))

    @staticmethod
    def send(x, dest, *, tag=0, comm=None):
        torch.ops.mpi4jax_b200.send(x, int(dest), int(tag), _register(comm))

    @staticmethod
    def recv(x, source=ANY_SOURCE, *, tag=ANY_TAG, comm=None, status=None):
        """``status``: an ``MPI.Status`` filled when the compiled function runs (as under ``jax.jit`` in
        the reference, tests/collective_ops/test_send_and_recv.py:113-153); keep it alive."""
        return torch.ops.mpi4jax_b200.recv(x, int(source), int(tag), _register(comm),
                                           0 if status is None else status._id)

    @staticmethod
    def sendrecv(sendbuf, recvbuf, source, dest, *, sendtag=0, recvtag=ANY_TAG, comm=None, status=None):
        return torch.ops.mpi4jax_b200.sendrecv(sendbuf, recvbuf, int(source), int(dest), int(sendtag),
                                               int(recvtag), _register(comm), 0 if status is None else status._id)
