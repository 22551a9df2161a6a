"""Row-parallel linear layer with the allreduce fused into the GEMM kernel.

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
"""

from __future__ import annotations

from typing import Optional

import torch
import torch.nn.functional as F

from .._src.collective_ops import _dispatch
from .._src.comm import SUM, Comm
from .._src.utils import get_default_comm, needs_autograd

_BM, _BN, _BK = 128, 128, 64     # tile of csrc/b2_gemm.cu


def _fuse(x: torch.Tensor, w: torch.Tensor, comm: Comm) -> bool:
    """Whether to run the fused kernel; the same answer on every rank of ``comm``."""
    if not (x.is_cuda and w.is_cuda and x.dtype == torch.bfloat16 and w.dtype == torch.bfloat16
            and x.dim() == 2 and w.dim() == 2):
        return False
    M, N = x.shape[0], w.shape[0]
    if M == 0 or N == 0 or M % _BM or N % _BN or comm.transport != "native":
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


def linear_allreduce(x: torch.Tensor, weight: torch.Tensor, *, comm: Optional[Comm] = None) -> torch.Tensor:
    """``x (M, K_local) @ weight (N, K_local).T`` summed over the ranks of ``comm``."""
    comm = comm or get_default_comm()
    if not needs_autograd(x, weight):
        return _forward(x, weight, comm)
    return _LinearAllreduce.apply(x, weight, comm)
