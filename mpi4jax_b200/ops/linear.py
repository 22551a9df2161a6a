"""Row-parallel linear layers with the allreduce or the reduce-scatter fused into the GEMM kernel.

``linear_allreduce(x, weight)`` = ``allreduce(x @ weight.T, SUM)`` where every rank holds a
K-shard of both operands -- the tensor-parallel pattern of the reference's matvec tests
(/root/reference/tests/collective_ops/test_allreduce_matvec.py:41-65).  On CUDA with bf16
operands and tile-aligned shapes it runs as ONE hand-written sm_90a kernel (wgmma MMAs,
TMA-fed, accumulators in registers, every finished tile all-reduced in the NVSwitch with
``multimem.ld_reduce`` / ``multimem.st`` while the next tile's operands are loaded, csrc/b2_gemm.cu);
otherwise it falls back to ``torch.matmul`` + ``allreduce``.
Differentiable: the adjoint of the allreduce is the identity on the replicated cotangent, so
``grad_x = g @ weight`` and ``grad_weight = g.T @ x`` are plain local GEMMs.

The K shards may differ between ranks, in length and in memory layout.  The fused kernel pairs tile t
of every rank in its epilogue, so either every rank runs it or none does: the choice depends only on
what all ranks share (M, N, the dtype, the transport and NVLS), and each rank then brings its own
operands into the form the kernel needs (:func:`_kernel_operands`).

``linear_reduce_scatter(x, weight)`` is the sequence-parallel twin: rank r keeps only rows
``[r M/P, (r+1) M/P)`` of the same sum, ``reduce_scatter((x @ weight.T).reshape(P, M/P, N), SUM)``.
Its kernel (csrc/b2_gemm_rs.cu) shares the GEMM and reduces each group of tiles by pulling every rank's
staged partial, with no multicast, so it also runs where NVLS is off or the ranks share a GPU.  The
adjoint of a reduce-scatter is an allgather: with ``G = allgather(g)``, ``grad_x = G @ weight`` and
``grad_weight = G.T @ x``.

``linear_allgather(x, weight)`` is the column-parallel layer in front of it: ``allgather(x) @ weight.T``
with rank q's rows first gathered at ``[q m, (q+1) m)``, and this rank's own column shard of the weight.
Its kernel (csrc/b2_gemm_ag.cu) runs the same GEMM on the gathered matrix while the ranks push their
shards into every rank's staging, so the allgather's NVLink traffic overlaps the tiles already computable.
The fuse decision depends only on what the ranks share (m, K, the dtype and the transport), never on this
rank's N, so a rank with no columns at all still pushes its rows.  The adjoint pairs the two layers:
``grad_x = linear_reduce_scatter(g, weight.T)`` and ``grad_weight = g.T @ allgather(x)``.

Scaled float8: each op takes ``scale_x`` and ``scale_w`` (both or neither).  With them, ``x`` and ``weight``
are float8 (``float8_e4m3fn`` or ``float8_e5m2``) and rank q's partial is ``rn_bf16(S_q * (sx_q[i] * sw_q[j]))``
with ``S_q = x_q @ w_q.T`` as the tensor core accumulates it and the scale product in fp32; the partials are
then summed, scattered or stored as the bf16 op does, and the output is bf16.  A scale is float32 of shape
``()`` (per tensor) or one per row of ``x`` / row of ``weight``, and its form may differ between ranks.  Two
e4m3 operands on the bf16 op's fused path run the e4m3 twin of its kernel (csrc/b2_gemm_f8.cu); everything
else computes ``S`` as ``x.float() @ w.float().T``, scales and rounds it the same way and calls the bf16
collective.  The scaled path is forward-only, like the float8 collectives.
"""

from __future__ import annotations

from typing import Optional

import torch
import torch.nn.functional as F

from .._src.collective_ops import _dispatch
from .._src.comm import SUM, Comm
from .._src.utils import get_default_comm, needs_autograd

_BM, _BN, _BK = 128, 128, 64     # tile of csrc/b2_gemm_body.cuh
_BK8 = 128                         # the float8 kernels' k-block: 128 one-byte elements
_F8 = (torch.float8_e4m3fn, torch.float8_e5m2)


def _kernel_shape(x: torch.Tensor, w: torch.Tensor, comm: Comm, dtype: torch.dtype = torch.bfloat16) -> bool:
    """CUDA operands of the kernel's ``dtype`` (bf16, or e4m3 for the float8 twins) with tile-aligned M and N
    on the native transport: what both kernels need.  The same answer on every rank of ``comm``."""
    if not (x.is_cuda and w.is_cuda and x.dtype == dtype and w.dtype == dtype
            and x.dim() == 2 and w.dim() == 2):
        return False
    M, N = x.shape[0], w.shape[0]
    return not (M == 0 or N == 0 or M % _BM or N % _BN or comm.transport != "native")


def _fuse(x: torch.Tensor, w: torch.Tensor, comm: Comm, dtype: torch.dtype = torch.bfloat16) -> bool:
    """Whether to run the fused allreduce kernel; the same answer on every rank of ``comm``."""
    if not _kernel_shape(x, w, comm, dtype):
        return False
    return comm.Get_size() == 1 or comm._native_comm().has_nvls


def _aligned(t: torch.Tensor) -> torch.Tensor:
    t = t.contiguous()
    return t if t.data_ptr() % 16 == 0 else t.clone()     # TMA needs 16-byte aligned rows


def _kernel_operands(x: torch.Tensor, w: torch.Tensor):
    """This rank's operands as the fused kernel takes them: K zero-padded to a multiple of 64 that is at
    least 64 (zero columns add nothing to ``x @ w.T``), contiguous and 16-byte aligned."""
    if x.shape[1] != w.shape[1]:
        raise ValueError(f"linear_allreduce: x has {x.shape[1]} columns, weight {w.shape[1]}")
    K = x.shape[1]
    pad = max(_BK, -(-K // _BK) * _BK) - K
    if pad:
        x, w = F.pad(x, (0, pad)), F.pad(w, (0, pad))
    return _aligned(x), _aligned(w)


def _forward(x: torch.Tensor, w: torch.Tensor, comm: Comm) -> torch.Tensor:
    if _fuse(x, w, comm):
        return comm._native_comm().gemm_allreduce(*_kernel_operands(x, w))
    return _dispatch.allreduce(comm, (x @ w.t()).contiguous(), SUM.code)


class _LinearAllreduce(torch.autograd.Function):
    @staticmethod
    def forward(x, w, comm):
        return _forward(x, w, comm)

    @staticmethod
    def setup_context(ctx, inputs, output):
        x, w, ctx.comm = inputs
        ctx.save_for_backward(x, w)

    @staticmethod
    def backward(ctx, g):
        x, w = ctx.saved_tensors
        return g @ w, g.t() @ x, None


def linear_allreduce(x: torch.Tensor, weight: torch.Tensor, *, comm: Optional[Comm] = None,
                     scale_x: Optional[torch.Tensor] = None, scale_w: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``x (M, K_local) @ weight (N, K_local).T`` summed over the ranks of ``comm``.  With ``scale_x`` and
    ``scale_w``: float8 operands, each rank's partial scaled by its own scales (module docstring), bf16 out."""
    comm = comm or get_default_comm()
    if _scaled("linear_allreduce", x, weight, scale_x, scale_w):
        return _forward_f8(x, weight, scale_x, scale_w, comm)
    if not needs_autograd(x, weight):
        return _forward(x, weight, comm)
    return _LinearAllreduce.apply(x, weight, comm)


def _forward_rs(x: torch.Tensor, w: torch.Tensor, comm: Comm) -> torch.Tensor:
    P = comm.Get_size()
    if _kernel_shape(x, w, comm):
        nc = comm._native_comm()
        xk, wk = _kernel_operands(x, w)
        # one rank: the reduce-scatter is the identity and the kernel the stand-alone GEMM
        return nc.gemm_allreduce(xk, wk) if P == 1 else nc.gemm_reduce_scatter(xk, wk)
    y = (x @ w.t()).contiguous()
    return _dispatch.reduce_scatter(comm, y.reshape(P, y.shape[0] // P, y.shape[1]), SUM.code)


class _LinearReduceScatter(torch.autograd.Function):
    @staticmethod
    def forward(x, w, comm):
        return _forward_rs(x, w, comm)

    @staticmethod
    def setup_context(ctx, inputs, output):
        x, w, ctx.comm = inputs
        ctx.save_for_backward(x, w)

    @staticmethod
    def backward(ctx, g):
        x, w = ctx.saved_tensors
        G = _dispatch.allgather(ctx.comm, g.contiguous()).reshape(x.shape[0], g.shape[1])
        return G @ w, G.t() @ x, None


def linear_reduce_scatter(x: torch.Tensor, weight: torch.Tensor, *, comm: Optional[Comm] = None,
                          scale_x: Optional[torch.Tensor] = None,
                          scale_w: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Rows ``[r M/P, (r+1) M/P)`` of ``x (M, K_local) @ weight (N, K_local).T`` summed over the P ranks of
    ``comm``, on rank r: shape ``(M / P, N)``.  ``M`` must be divisible by P.  With ``scale_x`` (over all M
    rows) and ``scale_w``: float8 operands, bf16 out (module docstring)."""
    comm = comm or get_default_comm()
    P = comm.Get_size()
    if x.dim() != 2 or weight.dim() != 2:
        raise ValueError(f"linear_reduce_scatter: x and weight must be 2-D (got {x.dim()}-D and {weight.dim()}-D)")
    if x.shape[0] % P:
        raise ValueError(f"linear_reduce_scatter: M = {x.shape[0]} rows are not divisible by the {P} ranks")
    if _scaled("linear_reduce_scatter", x, weight, scale_x, scale_w):
        return _forward_rs_f8(x, weight, scale_x, scale_w, comm)
    if not needs_autograd(x, weight):
        return _forward_rs(x, weight, comm)
    return _LinearReduceScatter.apply(x, weight, comm)


def _fuse_ag(x: torch.Tensor, w: torch.Tensor, comm: Comm, dtype: torch.dtype = torch.bfloat16) -> bool:
    """CUDA operands of the kernel's ``dtype``, ``P m`` a multiple of the tile height, the native transport:
    whether to run the allgather kernel.  The same answer on every rank of ``comm``: it never looks at this
    rank's N."""
    P, m = comm.Get_size(), x.shape[0]
    return (x.is_cuda and w.is_cuda and x.dtype == dtype and w.dtype == dtype and m > 0
            and (P * m) % _BM == 0 and comm.transport == "native")


def _forward_ag(x: torch.Tensor, w: torch.Tensor, comm: Comm) -> torch.Tensor:
    P, (m, K), N = comm.Get_size(), x.shape, w.shape[0]
    if _fuse_ag(x, w, comm):
        nc = comm._native_comm()
        # this rank's N up to a multiple of the tile width (at least one tile, so that a rank without
        # columns still runs the kernel and pushes its rows) with zero rows of the weight
        Np = max(_BN, -(-N // _BN) * _BN)
        xk, wk = _kernel_operands(x, F.pad(w, (0, 0, 0, Np - N)) if Np != N else w)
        y = nc.gemm_allreduce(xk, wk) if P == 1 else nc.gemm_allgather(xk, wk)
        return y if Np == N else y[:, :N].contiguous()
    X = _dispatch.allgather(comm, x.contiguous()).reshape(P * m, K)
    return X @ w.t()


class _LinearAllgather(torch.autograd.Function):
    @staticmethod
    def forward(x, w, comm):
        return _forward_ag(x, w, comm)

    @staticmethod
    def setup_context(ctx, inputs, output):
        x, w, ctx.comm = inputs
        ctx.save_for_backward(x, w)

    @staticmethod
    def backward(ctx, g):
        x, w = ctx.saved_tensors
        P = ctx.comm.Get_size()
        # rows r of sum_q g_q @ w_q (the N_q may differ), then the gathered x again, on every rank in this order
        grad_x = _forward_rs(g, w.t(), ctx.comm)
        X = _dispatch.allgather(ctx.comm, x.contiguous()).reshape(P * x.shape[0], x.shape[1])
        return grad_x, g.t() @ X, None


def linear_allgather(x: torch.Tensor, weight: torch.Tensor, *, comm: Optional[Comm] = None,
                     scale_x: Optional[torch.Tensor] = None, scale_w: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``allgather(x).reshape(P m, K) @ weight.T`` over the P ranks of ``comm``: shape ``(P m, N)``, rank q's
    rows at ``[q m, (q+1) m)``.  ``x (m, K)`` has the same shape on every rank; ``weight (N, K)`` is this
    rank's column shard, and N may differ between ranks.  With ``scale_x`` and ``scale_w``: float8 operands,
    output row ``q m + i`` scaled by rank q's ``scale_x[i]`` and this rank's ``scale_w``, bf16 out."""
    comm = comm or get_default_comm()
    if x.dim() != 2 or weight.dim() != 2:
        raise ValueError(f"linear_allgather: x and weight must be 2-D (got {x.dim()}-D and {weight.dim()}-D)")
    if x.shape[1] != weight.shape[1]:
        raise ValueError(f"linear_allgather: x has {x.shape[1]} columns, weight {weight.shape[1]}")
    if _scaled("linear_allgather", x, weight, scale_x, scale_w):
        return _forward_ag_f8(x, weight, scale_x, scale_w, comm)
    if not needs_autograd(x, weight):
        return _forward_ag(x, weight, comm)
    return _LinearAllgather.apply(x, weight, comm)


# ---------------------------------------------------------------------------
# scaled float8
# ---------------------------------------------------------------------------
def _scaled(op: str, x: torch.Tensor, w: torch.Tensor, sx: Optional[torch.Tensor], sw: Optional[torch.Tensor]) -> bool:
    """Whether the call takes the scaled float8 path; raises for bad arguments before any device work, on
    every rank alike (the checks look at nothing another rank could see differently)."""
    if sx is None and sw is None:
        return False
    if sx is None or sw is None:
        raise ValueError(f"{op}: pass both scale_x and scale_w, or neither")
    if x.dtype not in _F8 or w.dtype not in _F8:
        raise ValueError(f"{op}: scales need float8 operands (float8_e4m3fn or float8_e5m2), got {x.dtype} "
                         f"and {w.dtype}")
    if x.dim() != 2 or w.dim() != 2:
        raise ValueError(f"{op}: x and weight must be 2-D (got {x.dim()}-D and {w.dim()}-D)")
    if x.shape[1] != w.shape[1]:
        raise ValueError(f"{op}: x has {x.shape[1]} columns, weight {w.shape[1]}")
    for name, s, t, n, what in (("scale_x", sx, x, x.shape[0], "rows of x"), ("scale_w", sw, w, w.shape[0], "N")):
        if not isinstance(s, torch.Tensor) or s.dtype != torch.float32:
            raise ValueError(f"{op}: {name} must be a float32 tensor")
        if s.device != t.device:
            raise ValueError(f"{op}: {name} is on {s.device}, its operand on {t.device}")
        if s.dim() > 1 or (s.dim() == 1 and s.shape[0] != n):
            raise ValueError(f"{op}: {name} must have shape () or ({what},) = ({n},), got {tuple(s.shape)}")
    if needs_autograd(x, w, sx, sw):
        raise NotImplementedError(f"{op}: the scaled float8 path is forward-only (float8 has no derivative rules)")
    return True


def _bytes(t: torch.Tensor) -> torch.Tensor:
    return t.contiguous().view(torch.uint8)


def _kernel_operands_f8(x: torch.Tensor, w: torch.Tensor):
    """:func:`_kernel_operands` for the float8 kernels: K zero-padded to a multiple of 128 that is at least
    128 (a zero byte is +0 in e4m3), contiguous, 16-byte aligned.  Padded as bytes."""
    K = x.shape[1]
    pad = max(_BK8, -(-K // _BK8) * _BK8) - K
    xb, wb = _bytes(x), _bytes(w)
    if pad:
        xb, wb = F.pad(xb, (0, pad)), F.pad(wb, (0, pad))
    return _aligned(xb).view(x.dtype), _aligned(wb).view(w.dtype)


def _scaled_partial(S: torch.Tensor, sx: torch.Tensor, sw: torch.Tensor) -> torch.Tensor:
    """``rn_bf16(S * (sx[i] * sw[j]))`` in fp32, the kernels' epilogue."""
    return (S * (sx.reshape(-1, 1) * sw.reshape(1, -1))).to(torch.bfloat16)


def _product(x: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    return x.float() @ w.float().t()


def _forward_f8(x, w, sx, sw, comm: Comm) -> torch.Tensor:
    if _fuse(x, w, comm, torch.float8_e4m3fn):
        xk, wk = _kernel_operands_f8(x, w)
        return comm._native_comm().gemm_allreduce_f8(xk, wk, sx.contiguous(), sw.contiguous())
    return _dispatch.allreduce(comm, _scaled_partial(_product(x, w), sx, sw), SUM.code)


def _forward_rs_f8(x, w, sx, sw, comm: Comm) -> torch.Tensor:
    P = comm.Get_size()
    if _kernel_shape(x, w, comm, torch.float8_e4m3fn):
        nc = comm._native_comm()
        xk, wk = _kernel_operands_f8(x, w)
        sx, sw = sx.contiguous(), sw.contiguous()
        return nc.gemm_allreduce_f8(xk, wk, sx, sw) if P == 1 else nc.gemm_reduce_scatter_f8(xk, wk, sx, sw)
    y = _scaled_partial(_product(x, w), sx, sw)
    return _dispatch.reduce_scatter(comm, y.reshape(P, y.shape[0] // P, y.shape[1]), SUM.code)


def _forward_ag_f8(x, w, sx, sw, comm: Comm) -> torch.Tensor:
    P, (m, K), N = comm.Get_size(), x.shape, w.shape[0]
    if _fuse_ag(x, w, comm, torch.float8_e4m3fn):
        nc = comm._native_comm()
        Np = max(_BN, -(-N // _BN) * _BN)
        if Np != N:      # zero weight rows, and a per-column scale for each (sliced off with them)
            w = F.pad(_bytes(w), (0, 0, 0, Np - N)).view(w.dtype)
            if sw.dim() == 1:
                sw = F.pad(sw, (0, Np - N), value=1.0)
        xk, wk = _kernel_operands_f8(x, w)
        sx, sw = sx.contiguous(), sw.contiguous()
        y = nc.gemm_allreduce_f8(xk, wk, sx, sw) if P == 1 else nc.gemm_allgather_f8(xk, wk, sx, sw)
        return y if Np == N else y[:, :N].contiguous()
    # every rank's rows as bytes, and its row scales, one per row whatever form this rank passed
    X = _dispatch.allgather(comm, _bytes(x)).reshape(P * m, K).view(x.dtype)
    SX = _dispatch.allgather(comm, sx.expand(m).contiguous()).reshape(P * m)
    return _scaled_partial(_product(X, w), SX, sw)
