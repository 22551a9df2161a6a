"""MAXLOC and MINLOC: the value-index reductions of allreduce, reduce, scan and reduce_scatter.

With ``op=MPI.MAXLOC`` or ``MPI.MINLOC`` those four ops take a pair ``(values, indices)`` and return one:
the extreme value and where it is, e.g. ``allreduce((local_max, global_argmax), MPI.MAXLOC)``.

The fold rule -- the one rule of every path: the sm_90a kernel (csrc/b2_reduce_loc.cu), the gloo backend,
the host-staged transport and the object API (``Op.python_function`` / ``Op.__call__``).  Ranks fold in rank
order.  Folding the accumulator ``a`` (earlier ranks) with the next rank's pair ``b``:

* ``MAXLOC``: ``b`` wins if ``b.v > a.v``.  On equal values (``+0 == -0``) the smaller index wins; on equal
  value and index, ``a`` wins.
* NaN propagates, as in MAX / MIN: a NaN value beats every non-NaN value; two NaNs tie and go to the
  smaller index.
* ``MINLOC``: the same with ``<``.

The result is always one input pair, both fields from the same rank: values are copied, never recomputed,
so results are bit-identical across ranks and backends, signed zeros and NaN payloads included.  Values
compare as their dtype (float16 / bfloat16 exactly as float32).  For pairs without NaN the rule is mpi4py's.

Value dtypes: float16, bfloat16, float32, float64, int16, int32, int64 (MPI's SHORT_INT, 2INT, LONG_INT,
FLOAT_INT, DOUBLE_INT and the half types); index dtypes: int32, int64.
"""

from __future__ import annotations

import torch

from ..native import codes
from ..utils import as_tensor, needs_autograd
from . import _dispatch

VALUE_DTYPES = (torch.float16, torch.bfloat16, torch.float32, torch.float64, torch.int16, torch.int32, torch.int64)
INDEX_DTYPES = (torch.int32, torch.int64)
_SAME_WIDTH_INT = {2: torch.int16, 4: torch.int32, 8: torch.int64}


def is_loc(op) -> bool:
    return op.code in (codes.MAXLOC, codes.MINLOC)


def refuse(op, opname: str) -> None:
    """A loc operator passed to a collective other than the four reductions."""
    if is_loc(op):
        raise NotImplementedError(f"{opname} does not support {op.name}; use allreduce, reduce, scan or "
                                  "reduce_scatter with a (values, indices) pair")


def fold(a, b, maxloc: bool):
    """The fold rule on two pairs: ``(value, index)`` tuples of Python numbers (returns one of them), or of
    tensors (elementwise; returns the winning values and indices, bit for bit)."""
    (av, ai), (bv, bi) = a, b
    if not isinstance(av, torch.Tensor):
        an, bn = av != av, bv != bv
        if an or bn:
            takes = bn and (not an or bi < ai)
        else:
            takes = (bv > av if maxloc else bv < av) or (bv == av and bi < ai)
        return tuple(b) if takes else tuple(a)
    an, bn = torch.isnan(av), torch.isnan(bv)
    beats = bv > av if maxloc else bv < av
    takes = torch.where(an | bn, bn & (~an | (bi < ai)), beats | ((bv == av) & (bi < ai)))
    as_int = _SAME_WIDTH_INT[av.element_size()]                # select bits: NaN payloads stay as they are
    return torch.where(takes, bv.view(as_int), av.view(as_int)).view(av.dtype), torch.where(takes, bi, ai)


def check_pair(opname: str, x, op, comm):
    """``(values, indices)`` of a loc call, after the checks (Python scalars become tensors as in every op)."""
    if not isinstance(x, (tuple, list)) or len(x) != 2:
        raise TypeError(f"{opname} with {op.name} takes a pair (values, indices), got {type(x).__name__}")
    values, indices = (as_tensor(t, comm) for t in x)
    if values.dtype not in VALUE_DTYPES:
        raise TypeError(f"{opname} with {op.name}: values must be float16, bfloat16, float32, float64, int16, int32 "
                        f"or int64 (got {values.dtype})")
    if indices.dtype not in INDEX_DTYPES:
        raise TypeError(f"{opname} with {op.name}: indices must be int32 or int64 (got {indices.dtype})")
    if values.shape != indices.shape:
        raise ValueError(f"{opname} with {op.name}: values and indices must have the same shape "
                         f"(got {tuple(values.shape)} and {tuple(indices.shape)})")
    if values.device != indices.device:
        raise ValueError(f"{opname} with {op.name}: values and indices must live on the same device "
                         f"(got {values.device} and {indices.device})")
    return values, indices


def reduce_loc(opname: str, opcode: int, x, op, comm, root: int = 0, algorithm: str = "auto"):
    """The four public ops with a loc operator: ``(values, indices)``; reduce returns the input pair off the
    root."""
    values, indices = check_pair(opname, x, op, comm)
    if algorithm != "auto":
        raise ValueError(f"{opname} with {op.name} has one transport; algorithm must be 'auto' (got {algorithm!r})")
    if needs_autograd(values):
        raise NotImplementedError(f"The derivative of {opname} for {op.name} is not defined")
    if opcode == codes.OPC_REDUCE_SCATTER and (values.dim() == 0 or values.shape[0] != comm.Get_size()):
        raise ValueError("Reduce_scatter input must have shape (nproc, ...)")
    out = _dispatch.reduce_loc(comm, opcode, values, indices, op.code, root)
    return (values, indices) if out is None else out


def compiled_loc(opname: str, opcode: int, x, op, comm, root: int = 0):
    """The ``compiled`` twin of :func:`reduce_loc`: the ``mpi4jax_b200::reduce_loc`` custom op."""
    values, indices = check_pair(opname, x, op, comm)
    if torch.is_grad_enabled() and values.requires_grad:
        raise NotImplementedError(f"The derivative of {opname} for {op.name} is not defined")
    if opcode == codes.OPC_REDUCE_SCATTER and (values.dim() == 0 or values.shape[0] != comm.Get_size()):
        raise ValueError("Reduce_scatter input must have shape (nproc, ...)")
    return torch.ops.mpi4jax_b200.reduce_loc(values, indices, op.code, opcode, int(root), comm._id)
