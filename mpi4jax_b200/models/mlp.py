"""A small MLP trained data-parallel / tensor-parallel through the differentiable ops.

BASELINE.json config 5 ("grad through allreduce+bcast on a jitted MLP loss"): parameters
are created on rank 0 and broadcast (``bcast``, whose VJP is a reduce-to-root), the loss
is averaged with ``allreduce`` (VJP = identity), hidden activations of the tensor-parallel
variant are summed with ``allreduce`` exactly like the reference's column-sharded mat-vec
pattern (/root/reference/tests/collective_ops/test_allreduce_matvec.py:41-65).
"""

from __future__ import annotations

from typing import Optional

import torch

from .. import _src as ops
from .._src.comm import SUM, Comm
from .._src.utils import get_default_comm


class ParallelMLP:
    """``mode="dp"``: replicated weights, batch sharded, gradients all-reduced.
    ``mode="tp"``: first layer column-sharded, second layer row-sharded + allreduce."""

    def __init__(self, d_in: int, d_hidden: int, d_out: int, comm: Optional[Comm] = None,
                 device=None, dtype=torch.float32, mode: str = "dp", seed: int = 0):
        self.comm = comm or get_default_comm()
        self.device = torch.device(device) if device is not None else self.comm.device
        self.mode = mode
        P, r = self.comm.Get_size(), self.comm.Get_rank()
        gen = torch.Generator().manual_seed(seed)
        w1 = torch.randn(d_in, d_hidden, generator=gen, dtype=torch.float32) / d_in**0.5
        w2 = torch.randn(d_hidden, d_out, generator=gen, dtype=torch.float32) / d_hidden**0.5
        if mode == "tp":
            if d_hidden % P:
                raise ValueError("d_hidden must be divisible by the number of ranks")
            k = d_hidden // P
            w1, w2 = w1[:, r * k:(r + 1) * k], w2[r * k:(r + 1) * k]
        elif r != 0:
            w1, w2 = torch.zeros_like(w1), torch.zeros_like(w2)   # only the root's values matter
        self.w1 = w1.to(self.device, dtype).contiguous().requires_grad_(True)
        self.w2 = w2.to(self.device, dtype).contiguous().requires_grad_(True)

    def parameters(self):
        return [self.w1, self.w2]

    def forward(self, x: torch.Tensor, weights=None) -> torch.Tensor:
        w1_, w2_ = weights if weights is not None else (self.w1, self.w2)
        if self.mode == "tp":
            h = torch.tanh(x @ w1_)                           # column-parallel
            if h.is_cuda and h.dtype == torch.bfloat16:
                # row-parallel GEMM and its allreduce as ONE wgmma + multimem.red kernel
                from ..ops.linear import linear_allreduce

                return linear_allreduce(h, w2_.t(), comm=self.comm)
            return ops.allreduce(h @ w2_, SUM, comm=self.comm)       # row-parallel + sum
        w1 = ops.bcast(w1_, 0, comm=self.comm)                # parameters live on the root
        w2 = ops.bcast(w2_, 0, comm=self.comm)
        return torch.tanh(x @ w1) @ w2

    def loss(self, x: torch.Tensor, y: torch.Tensor, weights=None) -> torch.Tensor:
        local = ((self.forward(x, weights) - y) ** 2).mean()
        if self.mode == "tp":
            return local
        return ops.allreduce(local, SUM, comm=self.comm) / self.comm.Get_size()

    def step(self, x, y, lr: float = 1e-2) -> torch.Tensor:
        """One SGD step; returns the (global) loss.  In dp mode the gradient of the bcast
        parameters arrives on the root already summed over ranks (reduce-to-root VJP)."""
        params = list(self.parameters())
        # Differentiate with respect to VIEWS of the parameters, with autograd.grad: the backward pass then
        # never touches the parameters' AccumulateGrad nodes, which belong to the stream the parameters were
        # created on (the legacy default stream) -- the engine would make that stream wait for the backward
        # pass, which is illegal while the step is being captured into a CUDA graph
        # (mpi4jax_b200.jit(mlp.step): forward, backward through the collectives' VJPs and update as ONE
        # graph -- BASELINE config 5, bench/mlp_grad.py).
        views = [p.view_as(p) for p in params]
        loss = self.loss(x, y, views)
        grads = torch.autograd.grad(loss, views, allow_unused=True)
        with torch.no_grad():
            for p, g in zip(params, grads):
                p.grad = g
                if g is not None:
                    p -= lr * g
        return loss.detach()
