"""moe_dispatch / moe_combine -- top-k mixture-of-experts routing with a deterministic weighted combine.

``rows, expert_counts, plan = moe_dispatch(x, topk_idx, num_experts)`` sends each token to the k experts its
router picked, the experts spread over the ranks; ``out = moe_combine(y, plan, weights)`` brings the experts'
results back and sums each token's k results with its gate weights.  Every count stays on the device, so the
pair can be captured into a CUDA graph, and the combine folds in a fixed order, so its result is the same bits
on every call.  Extension: the reference has no expert routing.

Rules, on rank r of P (``E = num_experts``, ``L = E / P`` experts per rank):

* inputs: ``x`` is ``(N, *S)`` of any dtype the data movers take, float8 included; ``topk_idx`` is ``(N, k)``
  int32 or int64 on x's device, ``k >= 1``.  Expert e lives on rank ``e // L`` as local expert ``e % L``.  Pair
  ``(t, j)`` sends row t of ``x`` to expert ``topk_idx[t, j]``; an id outside ``[0, E)`` is not sent, and a
  token that lists an expert twice sends both pairs.
* the same on every rank, and not checked on the device: N, k, S, the dtype, E and ``recv_capacity`` (as
  alltoallv's N).  E must be divisible by P and at most 256 (every rank's per-expert counts live in the
  kernel's shared memory).
* dispatch output ``rows (R, *S)``, ``R = recv_capacity`` (default ``N * k * P``, which never drops a pair):
  grouped by local expert; within an expert by source rank; within (expert, source) in the sender's
  ``(token, slot)`` order.  The layout is cut at R in that order, and rows past the filled ones are zero.
  ``expert_counts`` is ``(L,)`` int64, the rows each local expert received after the cut: its cumulative sum
  gives the group offsets of a grouped GEMM.
* ``plan`` (:class:`MoePlan`) holds what the combine and the backward passes need; ``plan.dest`` and
  ``plan.pos`` ``(N, k)`` name the rank and row each pair landed in, -1 for a pair that was not delivered
  (invalid id, or cut at R).
* combine: ``y`` is ``(R, *S')`` in the layout of the dispatched rows (S' may differ from S), f16, bf16, f32 or
  f64; ``weights`` is ``(N, k)`` float32 or None (unit weights).  ``out[t] = rn(sum_j w[t,j] *
  y_{dest[t,j]}[pos[t,j]])`` over the delivered pairs only, in slot order j = 0..k-1: the accumulator starts
  as the first delivered product (so a lone -0.0 keeps its sign), products and sums are separate fp32
  round-to-nearest operations with no FMA contraction (f64 rows: f64), and the result is rounded once.  A
  token with no delivered pair gets +0.

GPU: ``b2_k_moe_dispatch`` gathers each pair's token row while it stages it behind a header of its
per-expert counts, and pulls its own experts' segments from the peers after one barrier;
``b2_k_moe_combine`` stages the filled expert rows and, after a full barrier, pulls each token's k rows and
folds them (csrc/b2_moe.cu).  One launch each.  The sort is torch ``argsort`` + ``searchsorted`` on the
device.  Differentiable (eager autograd, once): the dispatch's adjoint is a unit-weight combine; the combine's
adjoint replays the dispatch of the cotangent from the plan, scaled by the pair weights (sent to the experts
by a dispatch of one float per pair), and gathers each weight's gradient, the fp32 dot product of the
cotangent and y rows on the expert side, with a combine that keeps the pairs apart.
"""

from __future__ import annotations

import operator
from typing import NamedTuple, Optional

import torch
from torch.autograd.function import once_differentiable

from .._src.collective_ops import _dispatch
from .._src.comm import Comm
from .._src.native import codes
from .._src.utils import check_dtype, get_default_comm, needs_autograd

_COMBINE_DTYPES = (torch.float16, torch.bfloat16, torch.float32, torch.float64)
_MAX_ROWS = 2**31 - 1          # the kernels count rows in 32 bits


class MoePlan(NamedTuple):
    """What :func:`moe_combine` and the backward passes need to undo a :func:`moe_dispatch` (all on the device)."""

    order: torch.Tensor          # (N * k,) int64: the pair t * k + j at each position of the pairs sorted by expert
    send_counts: torch.Tensor    # (E,) int64: this rank's pairs for each expert
    recv_counts: torch.Tensor    # (L, P) int64: rows received per (local expert, source rank), after the cut
    dest: torch.Tensor           # (N, k) int64: the rank each pair went to, -1 if not delivered
    pos: torch.Tensor            # (N, k) int64: the row it landed in there, -1 if not delivered
    recv_capacity: int           # R
    k: int
    num_experts: int
    comm: Comm


def _check_dispatch(x, topk_idx, num_experts, recv_capacity, comm: Comm) -> int:
    """The argument checks of moe_dispatch (the same verdict on every rank); returns R."""
    if not isinstance(x, torch.Tensor) or x.dim() == 0:
        raise ValueError("moe_dispatch x must be a tensor of shape (N, ...)")
    check_dtype(x)
    if not isinstance(topk_idx, torch.Tensor) or topk_idx.dtype not in (torch.int32, torch.int64):
        raise TypeError(f"moe_dispatch topk_idx must be an int32 or int64 tensor (got "
                        f"{getattr(topk_idx, 'dtype', type(topk_idx).__name__)})")
    if topk_idx.dim() != 2 or topk_idx.shape[0] != x.shape[0] or topk_idx.shape[1] < 1:
        raise ValueError(f"moe_dispatch topk_idx must have shape (N, k) with N = {x.shape[0]} and k >= 1 "
                         f"(got {tuple(topk_idx.shape)})")
    if topk_idx.device != x.device:
        raise ValueError(f"moe_dispatch topk_idx must live on the device of x ({x.device}, got {topk_idx.device})")
    try:
        E = operator.index(num_experts)
    except TypeError:
        raise TypeError(f"moe_dispatch num_experts must be an int (got {type(num_experts).__name__})") from None
    P = comm.Get_size()
    if E < 1 or E % P or E > codes.MOE_MAX_EXPERTS:
        raise ValueError(f"moe_dispatch num_experts must be a positive multiple of the {P} ranks and at most "
                         f"{codes.MOE_MAX_EXPERTS} (got {E})")
    n_pairs = x.shape[0] * topk_idx.shape[1]
    R = n_pairs * P if recv_capacity is None else recv_capacity
    if not isinstance(R, int) or isinstance(R, bool):
        raise TypeError(f"moe_dispatch recv_capacity must be an int (got {type(R).__name__})")
    if R < 0:
        raise ValueError(f"moe_dispatch recv_capacity must be >= 0 (got {R})")
    if n_pairs * P > _MAX_ROWS or R > _MAX_ROWS:
        raise ValueError(f"moe_dispatch: {n_pairs} pairs on {P} ranks, or {R} rows, exceed 2^31 - 1 rows")
    return R


class _Dispatch(torch.autograd.Function):
    @staticmethod
    def forward(x, order, send_counts, k, num_experts, R, comm):
        return _dispatch.moe_dispatch(comm, x, order, send_counts, k, num_experts, R)

    @staticmethod
    def setup_context(ctx, inputs, output):
        ctx.N, ctx.comm = inputs[0].shape[0], inputs[-1]
        ctx.mark_non_differentiable(*output[1:])
        ctx.save_for_backward(*output[1:])

    @staticmethod
    @once_differentiable
    def backward(ctx, g, *_):
        recv, pos, dest = ctx.saved_tensors
        N = ctx.N
        grad = _dispatch.moe_combine(ctx.comm, g, pos.view(N, -1), dest.view(N, -1), None, recv)
        return grad, None, None, None, None, None, None


def moe_dispatch(x: torch.Tensor, topk_idx: torch.Tensor, num_experts: int, *, recv_capacity: Optional[int] = None,
                 comm: Optional[Comm] = None):
    """Send row t of ``x`` to each of the experts ``topk_idx[t]`` names (module docstring states the rules).

    Arguments:
        x: tokens ``(N, ...)``; N, the row shape and the dtype must be the same on every rank.
        topk_idx: ``(N, k)`` int32 or int64 expert ids on x's device; ids outside ``[0, num_experts)`` are not
            sent.
        num_experts: E, a multiple of the world size and at most 256; rank ``e // (E / nproc)`` holds expert e.
        recv_capacity: rows of the output, the same on every rank (default ``N * k * nproc``: no pair is
            dropped).
        comm: the communicator (defaults to a clone of ``COMM_WORLD``).

    Returns:
        Tuple[Tensor, Tensor, MoePlan]: the received rows ``(recv_capacity, ...)``, grouped by local expert, then
        source rank, then the sender's (token, slot) order, zero past the filled ones; the rows each local
        expert received, int64 ``(E / nproc,)``; and the plan :func:`moe_combine` takes.  Differentiable in
        ``x``; no host synchronisation.
    """
    comm = comm or get_default_comm()
    R = _check_dispatch(x, topk_idx, num_experts, recv_capacity, comm)
    N, k = topk_idx.shape
    E = operator.index(num_experts)
    key = topk_idx.reshape(-1).to(torch.int64)
    key = torch.where((key >= 0) & (key < E), key, E)           # invalid ids sort last and count for no expert
    order = torch.argsort(key, stable=True)
    # counts from the sorted keys: torch.bincount would read its maximum back to the host
    send_counts = torch.searchsorted(key[order], torch.arange(E + 1, device=key.device)).diff()
    fn = _Dispatch.apply if needs_autograd(x) else _Dispatch.forward
    rows, recv, pos, dest = fn(x, order, send_counts, k, E, R, comm)
    plan = MoePlan(order, send_counts, recv, dest.view(N, k), pos.view(N, k), R, k, E, comm)
    return rows, recv.sum(1), plan


def _replay(t: torch.Tensor, plan: MoePlan, pairs: bool = False) -> torch.Tensor:
    """The dispatch of ``t`` (``(N, ...)``, or one row per pair with ``pairs``) that ``plan`` describes, without
    sorting again."""
    return _dispatch.moe_dispatch(plan.comm, t, plan.order, plan.send_counts, 1 if pairs else plan.k,
                                  plan.num_experts, plan.recv_capacity, with_plan=False)[0]


class _Combine(torch.autograd.Function):
    @staticmethod
    def forward(y, weights, plan):
        return _dispatch.moe_combine(plan.comm, y, plan.pos, plan.dest, weights, plan.recv_counts)

    @staticmethod
    def setup_context(ctx, inputs, output):
        y, weights, ctx.plan = inputs
        ctx.save_for_backward(y, weights)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        y, w = ctx.saved_tensors
        plan = ctx.plan
        need_y, need_w = ctx.needs_input_grad[:2]
        acc = torch.float64 if y.dtype == torch.float64 else torch.float32
        g_rows = _replay(g, plan)                                 # (R, *S'): zero on the rows nobody filled
        gy = gw = None
        if need_y:
            if w is None:
                gy = g_rows
            else:
                w_rows = _replay(w.reshape(-1, 1), plan, pairs=True).view(-1, *[1] * (y.dim() - 1))
                gy = (g_rows.to(acc) * w_rows.to(acc)).to(y.dtype)
        if need_w:
            dots = (g_rows.to(acc) * y.to(acc)).reshape(y.shape[0], -1).sum(1, keepdim=True).float()
            gw = _dispatch.moe_combine(plan.comm, dots, plan.pos, plan.dest, None, plan.recv_counts, pairs=True)
            gw = gw.view(plan.pos.shape)
        return gy, gw, None


def moe_combine(y: torch.Tensor, plan: MoePlan, weights: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Return each token the weighted sum of its experts' results (module docstring states the rules).

    Arguments:
        y: ``(R, ...)`` rows laid out like :func:`moe_dispatch`'s output (e.g. the experts' results), float16,
            bfloat16, float32 or float64.
        plan: the :class:`MoePlan` of that dispatch.
        weights: ``(N, k)`` float32 gate weights on y's device, or None for unit weights.

    Returns:
        Tensor: ``(N, ...)``, row t the fold of its delivered pairs' rows in slot order, +0 if none was
        delivered.  Differentiable in ``y`` and ``weights``; no host synchronisation.
    """
    if not isinstance(plan, MoePlan):
        raise TypeError(f"moe_combine plan must be the MoePlan of a moe_dispatch (got {type(plan).__name__})")
    if not isinstance(y, torch.Tensor) or y.dim() == 0 or y.shape[0] != plan.recv_capacity:
        raise ValueError(f"moe_combine y must have shape ({plan.recv_capacity}, ...), the dispatch's recv_capacity "
                         f"rows (got {tuple(getattr(y, 'shape', ()))})")
    if y.dtype not in _COMBINE_DTYPES:
        raise TypeError(f"moe_combine y must be float16, bfloat16, float32 or float64 (got {y.dtype})")
    if y.device != plan.pos.device:
        raise ValueError(f"moe_combine y must live on the device of the plan ({plan.pos.device}, got {y.device})")
    if weights is not None:
        if not isinstance(weights, torch.Tensor) or weights.dtype != torch.float32:
            raise TypeError(f"moe_combine weights must be a float32 tensor (got "
                            f"{getattr(weights, 'dtype', type(weights).__name__)})")
        if tuple(weights.shape) != tuple(plan.pos.shape) or weights.device != y.device:
            raise ValueError(f"moe_combine weights must have shape {tuple(plan.pos.shape)} on {y.device} (got "
                             f"{tuple(weights.shape)} on {weights.device})")
        weights = weights.contiguous()
    grad = needs_autograd(y) if weights is None else needs_autograd(y, weights)
    return (_Combine.apply if grad else _Combine.forward)(y, weights, plan)
