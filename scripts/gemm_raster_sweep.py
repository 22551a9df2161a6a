"""Tile order of the persistent wgmma GEMM (csrc/b2_gemm_raster.h): device time per shape for several
band heights G (communicator option "gemm_raster"; 0 = row-major), next to cuBLAS.  One GPU.
    python scripts/gemm_raster_sweep.py"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import mpi4jax_b200 as m  # noqa: E402
from mpi4jax_b200 import MPI  # noqa: E402
from mpi4jax_b200.ops import linear_allreduce  # noqa: E402

comm = MPI.COMM_WORLD
dev = comm.device
nc = comm._native_comm()


def timeit(fn, iters=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / iters * 1e3


for (M, N, K) in [(4096, 4096, 4096), (8192, 8192, 8192), (8192, 4096, 1024), (2048, 4096, 4096), (16384, 8192, 4096)]:
    x = torch.randn(M, K, device=dev).bfloat16()
    w = torch.randn(N, K, device=dev).bfloat16()
    flops = 2.0 * M * N * K
    ref = (x @ w.t()).float()
    row = {}
    for G in (0, 2, 4, 8, 16, 32):
        nc.set_option("gemm_raster", G)
        out = linear_allreduce(x, w, comm=comm).float()
        err = ((out - ref).abs().max() / ref.abs().max()).item()
        us = timeit(lambda: linear_allreduce(x, w, comm=comm))
        row[f"G={G}"] = f"{us:.1f} us {flops / us / 1e6:.0f} TF/s (err {err:.1e})"
    us = timeit(lambda: x @ w.t())
    row["cublas"] = f"{us:.1f} us {flops / us / 1e6:.0f} TF/s"
    print(f"M={M} N={N} K={K}:", row, flush=True)
nc.set_option("gemm_raster", 0)
m.flush()
