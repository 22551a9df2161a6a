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
"""

from __future__ import annotations

from typing import Optional

import torch

from .._src.collective_ops import _dispatch
from .._src.comm import SUM, Comm
from .._src.utils import get_default_comm, needs_autograd


def _fusable(x: torch.Tensor, w: torch.Tensor) -> bool:
    return (
        x.is_cuda and w.is_cuda and x.dtype == torch.bfloat16 and w.dtype == torch.bfloat16
        and x.dim() == 2 and w.dim() == 2 and x.shape[1] == w.shape[1]
        and x.shape[0] % 128 == 0 and w.shape[0] % 128 == 0 and x.shape[1] % 64 == 0
    )


def _forward(x: torch.Tensor, w: torch.Tensor, comm: Comm) -> torch.Tensor:
    if _fusable(x, w):
        nc = comm._native_comm()
        if comm.Get_size() == 1 or nc.has_nvls:
            return nc.gemm_allreduce(x.contiguous(), w.contiguous())
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
