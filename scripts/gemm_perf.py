"""Fused wgmma GEMM+allreduce vs cuBLAS GEMM followed by an allreduce (ours / NCCL)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import mpi4jax_b200 as m  # noqa: E402
from mpi4jax_b200 import MPI  # noqa: E402
from mpi4jax_b200.ops import linear_allreduce  # noqa: E402
from mpi4jax_b200.utils import max_over_ranks  # noqa: E402

comm = MPI.COMM_WORLD
rank, size = comm.Get_rank(), comm.Get_size()
dev = comm.device
nccl = dist.new_group(backend="nccl") if size > 1 else None


def timeit(fn, iters=10):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    comm.Barrier()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    e.synchronize()
    return max_over_ranks(s.elapsed_time(e) / iters * 1e3, comm)


for (M, N, K) in [(4096, 4096, 4096 // size), (8192, 8192, 8192 // size), (8192, 4096, 1024), (2048, 4096, 4096)]:
    x = torch.randn(M, K, device=dev).bfloat16()
    w = torch.randn(N, K, device=dev).bfloat16()
    flops = 2.0 * M * N * K
    rows = {}
    rows["fused wgmma+NVLS (one kernel)"] = timeit(lambda: linear_allreduce(x, w, comm=comm))
    rows["cublas + our allreduce"] = timeit(lambda: m.allreduce(x @ w.t(), MPI.SUM, comm=comm))
    if nccl is not None:
        def f():
            y = x @ w.t()
            dist.all_reduce(y, group=nccl)
            return y
        rows["cublas + nccl allreduce"] = timeit(f)
    rows["cublas gemm only"] = timeit(lambda: x @ w.t())
    if rank == 0:
        print(f"M={M} N={N} K/rank={K} (bf16 out {M * N * 2 / 2**20:.0f} MiB): " +
              "; ".join(f"{k} {v:.1f} us ({flops / v / 1e6:.0f} TF/s/GPU)" for k, v in rows.items()), flush=True)
m.flush()
