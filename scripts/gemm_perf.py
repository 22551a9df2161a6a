"""Fused wgmma GEMM+allreduce vs cuBLAS GEMM followed by an allreduce (ours / NCCL), and for M divisible by
the world size the same for GEMM+reduce-scatter over the rows and for allgather (of M / P rows per rank)+GEMM.
Then the same in scaled float8 (e4m3, bf16 out) against torch._scaled_mm with fast accumulation; at world size
1 the fused rows are the stand-alone float8 GEMM.  The first line names the card and its power limit."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import mpi4jax_b200 as m  # noqa: E402
from mpi4jax_b200 import MPI  # noqa: E402
from mpi4jax_b200.ops import linear_allgather, linear_allreduce, linear_reduce_scatter  # noqa: E402
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


if rank == 0:
    try:
        import subprocess
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                            str(dev.index or 0)], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = torch.cuda.get_device_name(dev)
    print(f"device: {q}", flush=True)

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
    if M % size == 0:
        rows["fused wgmma+reduce-scatter (one kernel)"] = timeit(lambda: linear_reduce_scatter(x, w, comm=comm))
        rows["cublas + our reduce_scatter"] = timeit(
            lambda: m.reduce_scatter((x @ w.t()).reshape(size, M // size, N), MPI.SUM, comm=comm))
        if nccl is not None:
            def g():
                y = x @ w.t()
                out = torch.empty(M // size, N, device=dev, dtype=y.dtype)
                dist.reduce_scatter_tensor(out, y, group=nccl)
                return out
            rows["cublas + nccl reduce_scatter_tensor"] = timeit(g)
        xs = x[:M // size].contiguous()           # this rank's rows of the gathered (M, K) operand
        rows["fused allgather+wgmma (one kernel)"] = timeit(lambda: linear_allgather(xs, w, comm=comm))
        rows["our allgather + cublas"] = timeit(lambda: m.allgather(xs, comm=comm).reshape(M, K) @ w.t())
        if nccl is not None:
            def h():
                X = torch.empty(M, K, device=dev, dtype=xs.dtype)
                dist.all_gather_into_tensor(X, xs, group=nccl)
                return X @ w.t()
            rows["nccl all_gather_into_tensor + cublas"] = timeit(h)
    rows["cublas gemm only"] = timeit(lambda: x @ w.t())
    # scaled float8 (e4m3): the fused kernels, torch._scaled_mm (fast accumulation) + our collective, and + NCCL
    x8, w8 = x.to(torch.float8_e4m3fn), w.to(torch.float8_e4m3fn)
    sx, sw = torch.ones(M, 1, device=dev), torch.ones(1, N, device=dev)     # _scaled_mm's row-wise scale shapes
    sxv, swv = sx.reshape(M), sw.reshape(N)

    def smm(a, sa):
        return torch._scaled_mm(a, w8.t(), scale_a=sa, scale_b=sw, out_dtype=torch.bfloat16, use_fast_accum=True)

    rows["f8 fused wgmma+NVLS (one kernel)"] = timeit(
        lambda: linear_allreduce(x8, w8, comm=comm, scale_x=sxv, scale_w=swv))
    rows["f8 _scaled_mm + our allreduce"] = timeit(lambda: m.allreduce(smm(x8, sx), MPI.SUM, comm=comm))
    if nccl is not None:
        def f8():
            y = smm(x8, sx)
            dist.all_reduce(y, group=nccl)
            return y
        rows["f8 _scaled_mm + nccl allreduce"] = timeit(f8)
    if M % size == 0 and size > 1:
        rows["f8 fused wgmma+reduce-scatter (one kernel)"] = timeit(
            lambda: linear_reduce_scatter(x8, w8, comm=comm, scale_x=sxv, scale_w=swv))
        x8s, sxs = x8[:M // size].contiguous(), sxv[:M // size]
        rows["f8 fused allgather+wgmma (one kernel)"] = timeit(
            lambda: linear_allgather(x8s, w8, comm=comm, scale_x=sxs, scale_w=swv))
        rows["f8 our allgather + _scaled_mm"] = timeit(
            lambda: smm(m.allgather(x8s.view(torch.uint8), comm=comm).reshape(M, K).view(torch.float8_e4m3fn),
                        m.allgather(sxs, comm=comm).reshape(M, 1)))
        if nccl is not None:
            def h8():
                X = torch.empty(M, K, device=dev, dtype=torch.uint8)
                dist.all_gather_into_tensor(X, x8s.view(torch.uint8), group=nccl)
                return smm(X.view(torch.float8_e4m3fn), sx)
            rows["f8 nccl all_gather_into_tensor + _scaled_mm"] = timeit(h8)
    rows["f8 _scaled_mm only"] = timeit(lambda: smm(x8, sx))
    if rank == 0:
        print(f"M={M} N={N} K/rank={K} (bf16 out {M * N * 2 / 2**20:.0f} MiB): " +
              "; ".join(f"{k} {v:.1f} us ({flops / v / 1e6:.0f} TF/s/GPU)" for k, v in rows.items()), flush=True)
m.flush()
