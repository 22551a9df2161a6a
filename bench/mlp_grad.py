"""BASELINE.json config 5: ``grad`` through allreduce + bcast on a jitted MLP loss (step time,
gradient correctness), data-parallel and tensor-parallel, eager and under ``mpi4jax_b200.jit``.

* dp: parameters live on rank 0 and reach the ranks through ``bcast`` (VJP = reduce-to-root), the
  loss is averaged with ``allreduce`` (VJP = identity): one SGD step = forward, backward through
  both collectives, update.  The reference's counterpart is ``jax.grad`` of a jitted loss that
  calls ``mpi4jax.allreduce`` / ``bcast`` (README.rst:59-96, tests/collective_ops/test_allreduce.py:141-223).
* tp: first layer column-sharded, second layer row-sharded; in bf16 the row-parallel GEMM and its
  allreduce are ONE wgmma + multimem kernel (csrc/b2_gemm.cu).
* sp: batch sharded, weights sharded as in tp; the rows are all-gathered before the first layer and the
  row-parallel GEMM and its reduce-scatter are ONE wgmma kernel in bf16 (csrc/b2_gemm_rs.cu).  Rank q
  uses data(q), so its gradient shards are checked against the single-process gradient as for dp.

Device-timed (CUDA events on the launching stream, barrier + synchronize before, max over ranks).

    python -m mpi4jax_b200.run -n 8 bench/mlp_grad.py --out gpurun_out/mlp_grad.json
"""

import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

import mpi4jax_b200 as m  # noqa: E402
from mpi4jax_b200 import MPI  # noqa: E402
from mpi4jax_b200.models import ParallelMLP  # noqa: E402
from mpi4jax_b200.utils import max_over_ranks  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--d-in", type=int, default=1024)
ap.add_argument("--d-hidden", type=int, default=4096)
ap.add_argument("--d-out", type=int, default=1024)
ap.add_argument("--batch", type=int, default=512, help="samples per rank")
ap.add_argument("--steps", type=int, default=50)
ap.add_argument("--out", default="gpurun_out/mlp_grad.json")
ns = ap.parse_args()

comm = MPI.COMM_WORLD
rank, size = comm.Get_rank(), comm.Get_size()
dev = comm.device


def timed(fn, steps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    comm.Barrier()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    m.barrier(comm=comm)
    s.record()
    for _ in range(steps):
        fn()
    e.record()
    e.synchronize()
    return max_over_ranks(s.elapsed_time(e) * 1e3 / steps, comm)


def reference_grads(dtype):
    """The same loss on ONE process: every rank's shard concatenated, plain torch autograd."""
    gen = torch.Generator().manual_seed(0)
    w1 = (torch.randn(ns.d_in, ns.d_hidden, generator=gen) / ns.d_in ** 0.5).to(dev, dtype).requires_grad_()
    w2 = (torch.randn(ns.d_hidden, ns.d_out, generator=gen) / ns.d_hidden ** 0.5).to(dev, dtype).requires_grad_()
    xs = torch.cat([data(q, dtype)[0] for q in range(size)])
    ys = torch.cat([data(q, dtype)[1] for q in range(size)])
    loss = ((torch.tanh(xs @ w1) @ w2 - ys) ** 2).mean()
    loss.backward()
    return loss.detach(), w1.grad, w2.grad


def data(q, dtype):
    gen = torch.Generator().manual_seed(1000 + q)
    x = torch.randn(ns.batch, ns.d_in, generator=gen).to(dev, dtype)
    y = torch.randn(ns.batch, ns.d_out, generator=gen).to(dev, dtype)
    return x, y


result = {"world": size, "shape": [ns.d_in, ns.d_hidden, ns.d_out], "batch_per_rank": ns.batch}
for mode, dtype in (("dp", torch.float32), ("tp", torch.float32), ("tp", torch.bfloat16), ("sp", torch.bfloat16)):
    name = f"{mode}_{'bf16' if dtype == torch.bfloat16 else 'fp32'}"
    mlp = ParallelMLP(ns.d_in, ns.d_hidden, ns.d_out, comm=comm, device=dev, dtype=dtype, mode=mode)
    x, y = data(rank if mode != "tp" else 0, dtype)           # tp: every rank sees the same batch
    # ---- gradient correctness against the single-process loss -----------------------------
    for p in mlp.parameters():
        p.grad = None
    loss = mlp.loss(x, y)
    loss.backward()
    row = {}
    if mode == "dp":
        ref_loss, g1, g2 = reference_grads(dtype)
        row["loss_rel_err"] = abs(loss.item() - ref_loss.item()) / abs(ref_loss.item())
        if rank == 0:       # the root's parameters receive the gradient summed over ranks (reduce-to-root)
            row["grad_rel_err"] = max(((mlp.w1.grad - g1).norm() / g1.norm()).item(),
                                      ((mlp.w2.grad - g2).norm() / g2.norm()).item())
    elif mode == "sp":      # every rank holds its column / row shard of the single-process gradient
        ref_loss, g1, g2 = reference_grads(dtype)
        k = ns.d_hidden // size
        s1, s2 = g1[:, rank * k:(rank + 1) * k], g2[rank * k:(rank + 1) * k]
        row["loss_rel_err"] = abs(loss.item() - ref_loss.item()) / abs(ref_loss.item())
        row["grad_rel_err"] = max(((mlp.w1.grad - s1).float().norm() / s1.float().norm()).item(),
                                  ((mlp.w2.grad - s2).float().norm() / s2.float().norm()).item())
    else:
        row["loss_finite"] = bool(torch.isfinite(loss).item())
    # ---- step time: eager and as one CUDA graph --------------------------------------------
    row["eager_us"] = round(timed(lambda: mlp.step(x, y), ns.steps), 1)
    fast = m.jit(lambda a, b: mlp.step(a, b))
    fast(x, y)
    try:
        fast(x, y)
        row["jit_us"] = round(timed(lambda: fast(x, y), ns.steps), 1)
    except Exception as exc:  # pragma: no cover - capture of the autograd engine failed
        import traceback

        row["jit_error"] = str(exc)[:200]
        if rank == 0:
            traceback.print_exc()
    flops = 6 * ns.batch * (ns.d_in * ns.d_hidden / (size if mode == "tp" else 1) + ns.d_hidden * ns.d_out
                            / (size if mode == "tp" else 1))
    row["tflops_per_gpu_jit"] = round(flops / row.get("jit_us", row["eager_us"]) / 1e6, 2)
    errs = comm.allgather(row.get("grad_rel_err"))
    row["grad_rel_err"] = max((v for v in errs if v is not None), default=None)
    result[name] = row
    if rank == 0:
        print(name, row, flush=True)
    del mlp, fast
if rank == 0:
    os.makedirs(os.path.dirname(ns.out) or ".", exist_ok=True)
    with open(ns.out, "w") as f:
        json.dump(result, f, indent=1)
m.flush()
