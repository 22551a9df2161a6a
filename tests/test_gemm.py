"""Tensor-parallel linear: wgmma GEMM + in-switch allreduce in one kernel (csrc/b2_gemm.cu)
against a plain fp32 PyTorch reference of the same op."""

import pytest
import torch

import mpi4jax_b200 as m
from mpi4jax_b200 import MPI
from mpi4jax_b200.ops import linear_allreduce

comm = MPI.COMM_WORLD
rank, size = comm.Get_rank(), comm.Get_size()


def _operands(M, N, K, device):
    gen = torch.Generator().manual_seed(1234 + rank)
    x = (torch.randn(M, K, generator=gen) * 0.5).to(torch.bfloat16).to(device)
    w = (torch.randn(N, K, generator=gen) * 0.5).to(torch.bfloat16).to(device)
    return x, w


def _reference(x, w):
    local = (x.float() @ w.float().t()).contiguous()
    return m.allreduce(local, MPI.SUM, comm=comm)


@pytest.mark.gpu
# (2048, 2048, 256): 256 tiles, more than one per CTA on any GPU -- the operand ring and the fused
# epilogue's batches then carry across tile boundaries
@pytest.mark.parametrize("shape", [(128, 128, 64), (256, 384, 512), (1024, 512, 2048), (128, 256, 4096),
                                   (2048, 2048, 256)])
def test_linear_allreduce_matches_fp32_reference(shape):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    M, N, K = shape
    x, w = _operands(M, N, K, comm.device)
    ref = _reference(x, w)
    for _ in range(3):                      # repeated calls: accumulator re-zeroing, parity
        out = linear_allreduce(x, w, comm=comm)
        assert out.dtype == torch.bfloat16 and out.shape == (M, N)
        err = (out.float() - ref).abs().max().item()
        scale = ref.abs().max().item()
        assert err <= 1e-2 * scale + 1e-3, (err, scale)     # one bf16 rounding of an fp32 sum


@pytest.mark.gpu
def test_linear_allreduce_grad():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    x, w = _operands(128, 128, 128, comm.device)
    x.requires_grad_(True)
    w.requires_grad_(True)
    out = linear_allreduce(x, w, comm=comm)
    out.float().sum().backward()
    g = torch.ones(128, 128, dtype=torch.bfloat16, device=comm.device)
    assert torch.allclose(x.grad.float(), (g @ w.detach()).float(), rtol=2e-2, atol=1e-2)
    assert torch.allclose(w.grad.float(), (g.t() @ x.detach()).float(), rtol=2e-2, atol=1e-2)


def test_linear_allreduce_fallback_cpu():
    x = torch.randn(6, 10)
    w = torch.randn(4, 10)
    out = linear_allreduce(x, w, comm=comm)
    assert torch.allclose(out, (x @ w.t()) * 1.0 if size == 1 else m.allreduce(x @ w.t(), MPI.SUM, comm=comm))
