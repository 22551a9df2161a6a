"""Device-timed sweeps for the BASELINE.json collective configs:

* allreduce 1 KB - 1 GB, fp32 + bf16, every transport (ll / oneshot / twoshot / nvls / auto)
  next to NCCL on the same box                                   (configs 2)
* allgather and alltoall 1 KB - 1 GB per-rank payload vs NCCL     (config 4)
* reduce_scatter (P, n) fp32 + bf16, 1 KB - 1 GB per-rank input, vs NCCL and vs allreduce
* alltoallv bf16 token rows, balanced and skewed counts, 64 KiB - 256 MiB per rank, vs NCCL
  all_to_all_single (with its counts exchange and host read-back) and vs the equal-split alltoall;
  plus balanced rows of 8190 bytes (the byte-wise path for rows that are not a multiple of 16 bytes)
* allgatherv bf16 rows, full / half / skewed counts, 64 KiB - 256 MiB per rank, vs the allgather of the
  padded rows (alone and followed by a device-side compaction) and vs NCCL all_gather_into_tensor
* reduce_scatterv bf16 rows, equal / skewed / small counts, 64 KiB - 256 MiB output per rank, vs the
  reduce_scatter of the zero-padded segments (with the padding gather) and vs NCCL reduce_scatter_tensor
* gatherv / scatterv bf16 rows (root = last rank), full / half / skewed counts, 64 KiB - 256 MiB per rank, vs
  gather / scatter of the padded blocks followed by the device-side compaction a user would otherwise write
* bcast, reduce, gather, scatter (root = last rank) vs NCCL, scan (no NCCL counterpart)
* sendrecv ring, halo exchange latency

Timing: ``reps`` back-to-back ops captured in ONE CUDA graph, one replay timed with CUDA
events on the launching stream (barrier + synchronize before), max over ranks -- i.e. the
kernels' time, not the Python launch path.  Bus bandwidth uses the NCCL-tests conventions:
allreduce S/t*2(P-1)/P, allgather/alltoall/reduce_scatter (P-1)/P * total/t.

    python -m mpi4jax_b200.run -n 8 bench/collectives_sweep.py [--max-bytes 1073741824] [--out f.json]
"""

import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
os.environ.setdefault("MPI4JAX_B200_ABORT_ON_ERROR", "0")

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import mpi4jax_b200 as m  # noqa: E402
from mpi4jax_b200 import MPI  # noqa: E402
from mpi4jax_b200.utils import max_over_ranks  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--max-bytes", type=int, default=1 << 30)
ap.add_argument("--out", default="gpurun_out/collectives_sweep.json")
ap.add_argument("--quick", action="store_true", help="every fourth size")
ap.add_argument("--skip-allreduce-algos", action="store_true", help="time only the automatic choice")
ap.add_argument("--only-allreduce", action="store_true", help="stop after the allreduce tables")
ap.add_argument("--only-p2p", action="store_true", help="only the p2p ring, barrier and halo lines")
ap.add_argument("--only-allgatherv", action="store_true", help="only the allgatherv rows")
ap.add_argument("--only-reduce-scatterv", action="store_true", help="only the reduce_scatterv rows")
ap.add_argument("--only-gatherv", action="store_true", help="only the gatherv rows")
ap.add_argument("--only-scatterv", action="store_true", help="only the scatterv rows")
ap.add_argument("--max-blocks", type=int, default=0, help="override the collective grid cap")
ap.add_argument("--nvls-pipeline", type=int, default=-1, help="0 / 1: software pipelining of the NVLS allreduce")
ap.add_argument("--min-bytes", type=int, default=1 << 10)
ns = ap.parse_args()

comm = MPI.COMM_WORLD
rank, size = comm.Get_rank(), comm.Get_size()
dev = comm.device
nccl = None
try:
    nccl = dist.new_group(backend="nccl")
    t = torch.ones(8, device=dev)
    dist.all_reduce(t, group=nccl)
    torch.cuda.synchronize()
except Exception as exc:  # pragma: no cover
    if rank == 0:
        print("NCCL comparison unavailable:", exc)
    nccl = None
nc = comm._native_comm()
has_nvls = nc.has_nvls
if ns.max_blocks:
    nc.set_option("max_blocks", ns.max_blocks)
if ns.nvls_pipeline >= 0:
    nc.set_option("nvls_pipeline", ns.nvls_pipeline)


def reps_for(nbytes):
    return 50 if nbytes <= (1 << 16) else 20 if nbytes <= (1 << 22) else 5 if nbytes <= (1 << 27) else 3


def time_graph(fn, reps):
    """fn() enqueues ONE op; returns us per op (device time, max over ranks)."""
    fn()
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side), torch.cuda.graph(g, stream=side, capture_error_mode="thread_local"):
        for _ in range(reps):
            fn()
    torch.cuda.current_stream().wait_stream(side)
    g.replay()
    torch.cuda.synchronize()
    best = None
    for _ in range(3):
        comm.Barrier()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        g.replay()
        e.record()
        e.synchronize()
        us = s.elapsed_time(e) * 1e3 / reps
        best = us if best is None else min(best, us)
    del g
    return max_over_ranks(best, comm)


def time_eager(fn, reps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    best = None
    for _ in range(3):
        comm.Barrier()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(reps):
            fn()
        e.record()
        e.synchronize()
        us = s.elapsed_time(e) * 1e3 / reps
        best = us if best is None else min(best, us)
    return max_over_ranks(best, comm)


def time_nccl(fn, reps):
    try:
        return time_graph(fn, reps)
    except Exception:
        torch.cuda.synchronize()
        return time_eager(fn, max(reps, 10))


sizes = [] if ns.only_p2p else [1 << k for k in range(10, 31, 2 if ns.quick else 1) if ns.min_bytes <= (1 << k) <= ns.max_bytes]
result = {"world": size, "nvls": has_nvls, "allreduce": {}, "allgather": {}, "alltoall": {}, "p2p": {}}


# ---------------------------------------------------------------- allgatherv (per-rank |x| = nbytes, 64 KiB - 256 MiB)
# bf16 rows of hidden size 4096 (8 KiB), every rank contributing count_r of its N rows: "full" (N), "half"
# (N / 2) and "skewed" (rank r contributes N * (r + 1) / P).  Next to the allgather of the padded N rows,
# to that allgather followed by the device-side compaction a user would write without allgatherv (gather
# the counts too, scatter the valid rows to their packed positions: capturable, no host read), and to
# NCCL's all_gather_into_tensor of the padded rows.  Bandwidth: the bytes a rank receives from its peers,
# sum_{q != r} count_q * row_bytes (the most over ranks), divided by the time -- the same numerator for
# every column, so the columns compare as times do.
def allgatherv_rows():
    result["allgatherv"] = {"full": {}, "half": {}, "skewed": {}}
    hidden = 4096
    for nbytes in [b for b in sizes if (64 << 10) <= b <= (256 << 20)]:
        n = nbytes // (hidden * 2)
        for kind in ("full", "half", "skewed"):
            counts = [n if kind == "full" else n // 2 if kind == "half" else n * (q + 1) // size
                      for q in range(size)]
            useful = max(sum(counts) - counts[q] for q in range(size)) * hidden * 2
            bw = lambda us: round(useful / us / 1e3, 1)
            x = torch.ones(n, hidden, dtype=torch.bfloat16, device=dev)
            count = torch.tensor(counts[rank], dtype=torch.int64, device=dev)
            reps = reps_for(nbytes * size // 2)
            row = {}
            us = time_graph(lambda: m.allgatherv(x, count, comm=comm), reps)
            row["ours"] = {"us": round(us, 2), "busbw": bw(us)}
            us = time_graph(lambda: m.allgather(x, comm=comm), reps)
            row["allgather"] = {"us": round(us, 2), "busbw": bw(us)}
            rows = torch.arange(n, device=dev)

            def allgather_compact():
                xs = m.allgather(x, comm=comm)                                      # (P, N, hidden)
                cs = m.allgather(count.view(1), comm=comm).view(size, 1)
                dest = torch.where(rows < cs, torch.cumsum(cs, 0) - cs + rows, n * size)   # invalid -> pad row
                out = torch.zeros(n * size + 1, hidden, dtype=x.dtype, device=dev)
                return out.index_copy_(0, dest.view(-1), xs.view(-1, hidden))[: n * size]

            us = time_graph(allgather_compact, reps)
            row["allgather_compact"] = {"us": round(us, 2), "busbw": bw(us)}
            if nccl is not None:
                out = torch.empty(size * n, hidden, dtype=x.dtype, device=dev)
                us = time_nccl(lambda: dist.all_gather_into_tensor(out, x, group=nccl), reps)
                row["nccl"] = {"us": round(us, 2), "busbw": bw(us)}
                del out
            result["allgatherv"][kind][str(nbytes)] = row
            if rank == 0:
                print("allgatherv", kind, nbytes, {k: (v["us"], v["busbw"]) for k, v in row.items()}, flush=True)
            del x


# ------------------------------------------------------------ reduce_scatterv (N rows out = nbytes, 64 KiB - 256 MiB)
# bf16 rows of hidden size 4096 (8 KiB); every rank holds P segments of up to N rows (x has P * N rows) and sends
# s[p] rows to rank p: "equal" (N: the reduce_scatter of x.view(P, N, hidden)), "skewed" (N * (p + 1) / P) and
# "small" (N / 8, the case of a capacity far above the counts).  Next to what a user writes without
# reduce_scatterv -- the segments zero-padded into (P, N, hidden) with a device-side gather (capturable, no
# host read), then reduce_scatter -- and to NCCL's reduce_scatter_tensor of that padded tensor (alone).
# Bandwidth: the rows a rank receives from its peers, sum_{q != r} s_q[r] * row_bytes (the most over ranks),
# divided by the time.
def reduce_scatterv_rows():
    result["reduce_scatterv"] = {"equal": {}, "skewed": {}, "small": {}}
    hidden = 4096
    for nbytes in [b for b in sizes if (64 << 10) <= b <= (256 << 20) and b * size <= (1 << 30)]:
        n = nbytes // (hidden * 2)
        for kind in ("equal", "skewed", "small"):
            counts = [n if kind == "equal" else n * (p + 1) // size if kind == "skewed" else n // 8
                      for p in range(size)]
            useful = max(counts) * (size - 1) * hidden * 2
            bw = lambda us: round(useful / us / 1e3, 1) if useful else 0.0
            x = torch.ones(size * n, hidden, dtype=torch.bfloat16, device=dev)
            send = torch.tensor(counts, dtype=torch.int64, device=dev)
            reps = reps_for(nbytes * size // 2)
            row = {}
            us = time_graph(lambda: m.reduce_scatterv(x, send, MPI.SUM, recv_capacity=n, comm=comm), reps)
            row["ours"] = {"us": round(us, 2), "busbw": bw(us)}
            i = torch.arange(n, device=dev)
            idx = torch.where(i < send.view(size, 1), (torch.cumsum(send, 0) - send).view(size, 1) + i, size * n)
            padded = torch.zeros(size, n, hidden, dtype=x.dtype, device=dev)

            def pad_reduce_scatter():
                xp = torch.cat([x, x.new_zeros(1, hidden)])
                return m.reduce_scatter(xp[idx], MPI.SUM, comm=comm)

            us = time_graph(pad_reduce_scatter, reps)
            row["pad_reduce_scatter"] = {"us": round(us, 2), "busbw": bw(us)}
            if nccl is not None:
                out = torch.empty(n, hidden, dtype=x.dtype, device=dev)
                us = time_nccl(lambda: dist.reduce_scatter_tensor(out, padded.view(size * n, hidden), group=nccl), reps)
                row["nccl_padded"] = {"us": round(us, 2), "busbw": bw(us)}
                del out
            result["reduce_scatterv"][kind][str(nbytes)] = row
            if rank == 0:
                print("reduce_scatterv", kind, nbytes, {k: (v["us"], v["busbw"]) for k, v in row.items()}, flush=True)
            del x, padded


# ----------------------------------------------------- gatherv / scatterv (root = last rank, 64 KiB - 256 MiB)
# bf16 rows of hidden size 4096 (8 KiB).  gatherv: every rank holds N rows (nbytes) and contributes count_r of
# them, "full" (N), "half" (N / 2) or "skewed" (N * (r + 1) / P).  scatterv: the root holds N rows and sends
# s[q] to rank q, "full" (N / P each: all of them), "half" (N / 2P) or "skewed" (proportional to q + 1).  Next
# to what a user writes without them: gather / scatter of (P, N, hidden) blocks with the counts, and the
# device-side compaction on the receiving side (the root packs the gathered rows; the root pads its rows into
# blocks before the scatter).  Both are capturable, with no host read.  Bandwidth: the rows that cross between
# the root and the other ranks, times the row bytes, over the time.
def gatherv_rows():
    result["gatherv"] = {"full": {}, "half": {}, "skewed": {}}
    hidden, root = 4096, size - 1
    for nbytes in [b for b in sizes if (64 << 10) <= b <= (256 << 20)]:
        n = nbytes // (hidden * 2)
        for kind in ("full", "half", "skewed"):
            counts = [n if kind == "full" else n // 2 if kind == "half" else n * (q + 1) // size for q in range(size)]
            useful = (sum(counts) - counts[root]) * hidden * 2
            bw = lambda us: round(useful / us / 1e3, 1) if useful else 0.0
            x = torch.ones(n, hidden, dtype=torch.bfloat16, device=dev)
            count = torch.tensor(counts[rank], dtype=torch.int64, device=dev)
            reps = reps_for(nbytes * size // 2)
            row = {}
            us = time_graph(lambda: m.gatherv(x, count, root, comm=comm), reps)
            row["ours"] = {"us": round(us, 2), "busbw": bw(us)}
            rows = torch.arange(n, device=dev)

            def gather_compact():
                xs = m.gather(x, root, comm=comm)                                   # root: (P, N, hidden)
                cs = m.gather(count.view(1), root, comm=comm)
                if rank != root:
                    return xs
                cs = cs.view(size, 1)
                dest = torch.where(rows < cs, torch.cumsum(cs, 0) - cs + rows, n * size)   # invalid -> pad row
                out = torch.zeros(n * size + 1, hidden, dtype=x.dtype, device=dev)
                return out.index_copy_(0, dest.view(-1), xs.view(-1, hidden))[: n * size]

            us = time_graph(gather_compact, reps)
            row["gather_compact"] = {"us": round(us, 2), "busbw": bw(us)}
            result["gatherv"][kind][str(nbytes)] = row
            if rank == 0:
                print("gatherv", kind, nbytes, {k: (v["us"], v["busbw"]) for k, v in row.items()}, flush=True)
            del x


def scatterv_rows():
    result["scatterv"] = {"full": {}, "half": {}, "skewed": {}}
    hidden, root = 4096, size - 1
    for nbytes in [b for b in sizes if (64 << 10) <= b <= (256 << 20)]:
        n = nbytes // (hidden * 2)
        for kind in ("full", "half", "skewed"):
            counts = [n // size if kind == "full" else n // (2 * size) if kind == "half"
                      else 2 * n * (q + 1) // (size * (size + 1)) for q in range(size)]
            useful = (sum(counts) - counts[root]) * hidden * 2
            bw = lambda us: round(useful / us / 1e3, 1) if useful else 0.0
            x = torch.ones(n, hidden, dtype=torch.bfloat16, device=dev)
            send = torch.tensor(counts, dtype=torch.int64, device=dev)
            reps = reps_for(nbytes)
            row = {}
            us = time_graph(lambda: m.scatterv(x, send, root, comm=comm), reps)
            row["ours"] = {"us": round(us, 2), "busbw": bw(us)}
            i = torch.arange(n, device=dev)
            idx = torch.where(i < send.view(size, 1), (torch.cumsum(send, 0) - send).view(size, 1) + i, n)
            template = torch.empty(n, hidden, dtype=x.dtype, device=dev)

            def pad_scatter():
                if rank == root:
                    padded = torch.cat([x, x.new_zeros(1, hidden)])[idx]                # (P, N, hidden)
                    return m.scatter(padded, root, comm=comm), m.scatter(send.view(size, 1), root, comm=comm)
                return m.scatter(template, root, comm=comm), m.scatter(send[:1], root, comm=comm)

            us = time_graph(pad_scatter, reps)
            row["pad_scatter"] = {"us": round(us, 2), "busbw": bw(us)}
            result["scatterv"][kind][str(nbytes)] = row
            if rank == 0:
                print("scatterv", kind, nbytes, {k: (v["us"], v["busbw"]) for k, v in row.items()}, flush=True)
            del x, template


if ns.only_gatherv or ns.only_scatterv:
    if ns.only_gatherv:
        gatherv_rows()
    else:
        scatterv_rows()
    if rank == 0:
        os.makedirs(os.path.dirname(ns.out) or ".", exist_ok=True)
        with open(ns.out, "w") as f:
            json.dump(result, f, indent=1)
    m.flush()
    sys.exit(0)

if ns.only_reduce_scatterv:
    reduce_scatterv_rows()
    if rank == 0:
        os.makedirs(os.path.dirname(ns.out) or ".", exist_ok=True)
        with open(ns.out, "w") as f:
            json.dump(result, f, indent=1)
    m.flush()
    sys.exit(0)

if ns.only_allgatherv:
    allgatherv_rows()
    if rank == 0:
        os.makedirs(os.path.dirname(ns.out) or ".", exist_ok=True)
        with open(ns.out, "w") as f:
            json.dump(result, f, indent=1)
    m.flush()
    sys.exit(0)

# ---------------------------------------------------------------- allreduce
sym_pool = None
if sizes and size > 1 and dev.type == "cuda":
    sym_pool = m.symmetric_empty((max(sizes),), torch.uint8, comm=comm)
for dtype, dname in ((torch.float32, "fp32"), (torch.bfloat16, "bf16")):
    table = {}
    for nbytes in sizes:
        x = torch.ones(nbytes // torch.empty((), dtype=dtype).element_size(), dtype=dtype, device=dev)
        row = {}
        reps = reps_for(nbytes)
        for algo in (("auto",) if ns.skip_allreduce_algos else ("auto", "ll", "oneshot", "twoshot", "nvls")):
            if algo == "ll" and nbytes > (64 << 10):
                continue
            if algo == "nvls" and not has_nvls:
                continue
            if algo == "oneshot" and size > 2 and nbytes > (1 << 27):
                continue
            try:
                us = time_graph(lambda: m.allreduce(x, MPI.SUM, comm=comm, algorithm=algo), reps)
                row[algo] = {"us": round(us, 2), "busbw": round(nbytes / us / 1e3 * 2 * (size - 1) / size, 1)}
            except Exception as exc:
                row[algo] = {"error": str(exc)[:120]}
        if nccl is not None:
            us = time_nccl(lambda: dist.all_reduce(x, group=nccl), reps)
            row["nccl"] = {"us": round(us, 2), "busbw": round(nbytes / us / 1e3 * 2 * (size - 1) / size, 1)}
        if sym_pool is not None and has_nvls and nbytes >= 16:
            # the same reduction on a SYMMETRIC tensor, in place (no staging copies): mpi4jax_b200.allreduce_
            xs = sym_pool[: nbytes].view(dtype)
            xs.fill_(1)
            try:
                us = time_graph(lambda: m.allreduce_(xs, comm=comm), reps)
                row["sym"] = {"us": round(us, 2), "busbw": round(nbytes / us / 1e3 * 2 * (size - 1) / size, 1)}
            except Exception as exc:
                row["sym"] = {"error": str(exc)[:120]}
        table[str(nbytes)] = row
        if rank == 0:
            print(dname, nbytes, {k: (v.get("us"), v.get("busbw")) for k, v in row.items()}, flush=True)
        del x
    result["allreduce"][dname] = table

if ns.only_allreduce:
    if rank == 0:
        os.makedirs(os.path.dirname(ns.out) or ".", exist_ok=True)
        with open(ns.out, "w") as f:
            json.dump(result, f, indent=1)
    m.flush()
    sys.exit(0)

# ---------------------------------------------------------------- allgather / alltoall (per-rank payload = nbytes)
for nbytes in sizes:
    if nbytes * size > (8 << 30):
        continue
    reps = reps_for(nbytes * size // 2)
    x = torch.ones(nbytes // 4, device=dev)
    row = {}
    us = time_graph(lambda: m.allgather(x, comm=comm), reps)
    row["ours"] = {"us": round(us, 2), "busbw": round(nbytes * (size - 1) / us / 1e3, 1)}
    if nccl is not None:
        out = torch.empty(size * x.numel(), device=dev)
        us = time_nccl(lambda: dist.all_gather_into_tensor(out, x, group=nccl), reps)
        row["nccl"] = {"us": round(us, 2), "busbw": round(nbytes * (size - 1) / us / 1e3, 1)}
        del out
    result["allgather"][str(nbytes)] = row
    if nbytes >= size * 4:
        y = torch.ones(size, nbytes // 4 // size, device=dev)        # total payload = nbytes per rank
        tot = y.numel() * 4
        row2 = {}
        us = time_graph(lambda: m.alltoall(y, comm=comm), reps)
        row2["ours"] = {"us": round(us, 2), "busbw": round(tot * (size - 1) / size / us / 1e3, 1)}
        if nccl is not None:
            out = torch.empty_like(y)
            us = time_nccl(lambda: dist.all_to_all_single(out, y, group=nccl), reps)
            row2["nccl"] = {"us": round(us, 2), "busbw": round(tot * (size - 1) / size / us / 1e3, 1)}
            del out
        result["alltoall"][str(nbytes)] = row2
        del y
    if rank == 0:
        print("allgather/alltoall", nbytes, row, result["alltoall"].get(str(nbytes)), flush=True)
    del x

# ---------------------------------------------------------------- reduce_scatter (per-rank input |x| = nbytes)
# next to NCCL's reduce_scatter_tensor and to allreduce(x)[rank], what a user without it would call
result["reduce_scatter"] = {}
for dtype, dname in ((torch.float32, "fp32"), (torch.bfloat16, "bf16")):
    table = {}
    esize = torch.empty((), dtype=dtype).element_size()
    for nbytes in sizes:
        if nbytes < size * 16:
            continue
        x = torch.ones(size, nbytes // esize // size, dtype=dtype, device=dev)
        tot = x.numel() * esize
        reps = reps_for(nbytes)
        bw = lambda us: round(tot * (size - 1) / size / us / 1e3, 1)
        row = {}
        us = time_graph(lambda: m.reduce_scatter(x, MPI.SUM, comm=comm), reps)
        row["ours"] = {"us": round(us, 2), "busbw": bw(us)}
        us = time_graph(lambda: m.allreduce(x, MPI.SUM, comm=comm), reps)
        row["allreduce"] = {"us": round(us, 2), "busbw": bw(us)}
        if nccl is not None:
            out = torch.empty(x.shape[1:], dtype=dtype, device=dev)
            us = time_nccl(lambda: dist.reduce_scatter_tensor(out, x, group=nccl), reps)
            row["nccl"] = {"us": round(us, 2), "busbw": bw(us)}
            del out
        table[str(nbytes)] = row
        if rank == 0:
            print("reduce_scatter", dname, nbytes, {k: (v["us"], v["busbw"]) for k, v in row.items()}, flush=True)
        del x
    result["reduce_scatter"][dname] = table

# ---------------------------------------------------------------- alltoallv (per-rank input |x| = nbytes, 64 KiB - 256 MiB)
# bf16 token rows of hidden size 4096 (8 KiB), the layout of an expert-parallel MoE dispatch.  Balanced:
# N / P rows to every rank; skewed: half of every rank's rows to rank 0, the rest spread evenly.  Next to
# the equal-split alltoall at the same bytes, and to what an NCCL-based MoE layer does: exchange the
# counts, read them back to the host (.tolist(), a device synchronisation), then all_to_all_single with
# split lists -- which cannot be captured into a CUDA graph, so it is timed eagerly.
# "odd_rows": balanced again with hidden size 4095 (8190-byte rows), which takes the byte-wise path of the
# kernel (rows that are not a multiple of 16 bytes).
result["alltoallv"] = {"balanced": {}, "skewed": {}, "odd_rows": {}}


def alltoallv_counts(kind, n):
    rest = (n - n // 2) // max(size - 1, 1)
    if kind == "skewed":
        return [n // 2 + (rest if size == 1 else 0)] + [rest] * (size - 1)
    return [n // size] * size


for nbytes in [b for b in sizes if (64 << 10) <= b <= (256 << 20)]:
    for kind, hidden in (("balanced", 4096), ("skewed", 4096), ("odd_rows", 4095)):
        n = nbytes // (hidden * 2)
        if n < size:
            continue
        x = torch.ones(n, hidden, dtype=torch.bfloat16, device=dev)
        counts = torch.tensor(alltoallv_counts(kind, n), dtype=torch.int64, device=dev)
        reps = reps_for(nbytes)
        bw = lambda us: round(n * hidden * 2 * (size - 1) / size / us / 1e3, 1)
        row = {}
        us = time_graph(lambda: m.alltoallv(x, counts, comm=comm), reps)
        row["ours"] = {"us": round(us, 2), "busbw": bw(us)}
        y = x[: n // size * size].view(size, n // size, hidden)
        us = time_graph(lambda: m.alltoall(y, comm=comm), reps)
        row["alltoall"] = {"us": round(us, 2), "busbw": bw(us)}
        if nccl is not None:
            def nccl_alltoallv():
                recv = torch.empty_like(counts)
                dist.all_to_all_single(recv, counts, group=nccl)
                send_split, recv_split = counts.tolist(), recv.tolist()
                out = torch.empty(sum(recv_split), hidden, dtype=x.dtype, device=dev)
                dist.all_to_all_single(out, x[: sum(send_split)], recv_split, send_split, group=nccl)
            us = time_eager(nccl_alltoallv, max(reps, 5))
            row["nccl"] = {"us": round(us, 2), "busbw": bw(us)}
        result["alltoallv"][kind][str(nbytes)] = row
        if rank == 0:
            print("alltoallv", kind, nbytes, {k: (v["us"], v["busbw"]) for k, v in row.items()}, flush=True)
        del x, y

allgatherv_rows()
reduce_scatterv_rows()
gatherv_rows()
scatterv_rows()

# ---------------------------------------------------------------- rooted ops + scan (per-rank payload = nbytes)
result.update({"bcast": {}, "reduce": {}, "gather": {}, "scatter": {}, "scan": {}})
root = size - 1
for nbytes in [b for b in sizes if b >= 1 << 10][::1 if ns.quick else 2]:
    reps = reps_for(nbytes)
    x = torch.ones(nbytes // 4, device=dev)
    rows = {k: {} for k in ("bcast", "reduce", "scan")}
    us = time_graph(lambda: m.bcast(x, root, comm=comm), reps)
    rows["bcast"]["ours"] = {"us": round(us, 2), "gbs": round(nbytes / us / 1e3, 1)}
    us = time_graph(lambda: m.reduce(x, MPI.SUM, root, comm=comm), reps)
    rows["reduce"]["ours"] = {"us": round(us, 2), "gbs": round(nbytes / us / 1e3, 1)}
    us = time_graph(lambda: m.scan(x, MPI.SUM, comm=comm), reps)
    rows["scan"]["ours"] = {"us": round(us, 2), "gbs": round(nbytes / us / 1e3, 1)}
    if nccl is not None:
        y = x.clone()
        us = time_nccl(lambda: dist.broadcast(y, src=root, group=nccl), reps)
        rows["bcast"]["nccl"] = {"us": round(us, 2), "gbs": round(nbytes / us / 1e3, 1)}
        us = time_nccl(lambda: dist.reduce(y, dst=root, group=nccl), reps)
        rows["reduce"]["nccl"] = {"us": round(us, 2), "gbs": round(nbytes / us / 1e3, 1)}
        del y
    for k in rows:
        result[k][str(nbytes)] = rows[k]
    if nbytes * size <= (2 << 30):
        rows2 = {"gather": {}, "scatter": {}}
        us = time_graph(lambda: m.gather(x, root, comm=comm), reps)
        rows2["gather"]["ours"] = {"us": round(us, 2), "gbs": round(nbytes * (size - 1) / us / 1e3, 1)}
        big = torch.ones(size, nbytes // 4, device=dev) if rank == root else x
        us = time_graph(lambda: m.scatter(big, root, comm=comm), reps)
        rows2["scatter"]["ours"] = {"us": round(us, 2), "gbs": round(nbytes * (size - 1) / us / 1e3, 1)}
        if nccl is not None:
            try:
                outs = [torch.empty_like(x) for _ in range(size)] if rank == root else None
                us = time_eager(lambda: dist.gather(x, outs, dst=root, group=nccl), max(reps, 5))
                rows2["gather"]["nccl"] = {"us": round(us, 2), "gbs": round(nbytes * (size - 1) / us / 1e3, 1)}
                ins = [torch.ones_like(x) for _ in range(size)] if rank == root else None
                y = torch.empty_like(x)
                us = time_eager(lambda: dist.scatter(y, ins, src=root, group=nccl), max(reps, 5))
                rows2["scatter"]["nccl"] = {"us": round(us, 2), "gbs": round(nbytes * (size - 1) / us / 1e3, 1)}
                del outs, ins, y
            except Exception as exc:  # pragma: no cover
                rows2["gather"]["nccl"] = {"error": str(exc)[:100]}
        for k in rows2:
            result[k][str(nbytes)] = rows2[k]
        del big
    if rank == 0:
        print("rooted", nbytes, {k: v for k, v in rows.items()}, {k: result[k].get(str(nbytes)) for k in ("gather", "scatter")},
              flush=True)
    del x

# ---------------------------------------------------------------- p2p ring + halo
for nbytes in (8, 4096, 1 << 16, 1 << 20, 1 << 24, 1 << 28):
    x = torch.ones(max(nbytes // 4, 1), device=dev)
    us = time_graph(lambda: m.sendrecv(x, x, source=(rank - 1) % size, dest=(rank + 1) % size, comm=comm),
                    reps_for(nbytes))
    result["p2p"][str(nbytes)] = {"us": round(us, 2), "gbs": round(nbytes / us / 1e3, 1)}
us = time_graph(lambda: m.barrier(comm=comm), 50)
result["barrier_us"] = round(us, 2)
if size in (1, 2, 4, 6, 8, 16):
    from mpi4jax_b200.models import ShallowWaterConfig, ShallowWaterModel

    mod = ShallowWaterModel(ShallowWaterConfig.for_resolution(4096, 4096), comm=comm, device=dev)
    for nf in (2, 4):
        fields = [mod.fe, mod.fn, mod.q, mod.ke][:nf]
        kinds = ["u", "v", "h", "h"][:nf]
        us = time_graph(lambda: mod.enforce_boundaries(fields, kinds), 50)
        result[f"halo{nf}_us"] = round(us, 2)
if rank == 0:
    print("p2p", result["p2p"], "barrier", result["barrier_us"], "halo", result.get("halo2_us"), result.get("halo4_us"))
    os.makedirs(os.path.dirname(ns.out) or ".", exist_ok=True)
    with open(ns.out, "w") as f:
        json.dump(result, f, indent=1)
m.flush()
