"""Measure the transport crossovers of the GPU collectives for THIS job's world size on THIS box and write
a tuning file (mpi4jax_b200/_src/tuning.py explains the keys and how the file is picked up).

    python -m mpi4jax_b200.run -n 8 bench/autotune_collectives.py --out mpi4jax_b200/_src/tuning_tables/NVIDIA_H100_80GB_HBM3.json

For every message size (1 KiB .. 64 MiB, powers of two) the allreduce is timed with each forced transport
(`algorithm="ll" | "oneshot" | "twoshot" | "nvls"`), bcast with the multicast path forced on and off; device
time of a CUDA-graph replay of back-to-back calls, max over ranks.  Existing entries of the output file for
other world sizes are kept.  The reference has no counterpart (MPI chooses its own algorithms)."""

import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

import mpi4jax_b200 as m  # noqa: E402
from mpi4jax_b200 import MPI  # noqa: E402
from mpi4jax_b200._src import tuning  # noqa: E402
from mpi4jax_b200.utils import max_over_ranks  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--out", default="gpurun_out/tuning.json")
ap.add_argument("--max-bytes", type=int, default=64 << 20)
ns = ap.parse_args()

comm = MPI.COMM_WORLD
rank, size = comm.Get_rank(), comm.Get_size()
dev = comm.device
if dev.type != "cuda" or size < 2:
    raise SystemExit("autotune needs >= 2 GPU ranks")
nc = comm._native_comm()
m.comm_reserve(ns.max_bytes, comm=comm)


def time_graph(fn, reps):
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
    return max_over_ranks(best, comm)


sizes = [1 << k for k in range(10, 31) if (1 << k) <= ns.max_bytes]
times = {a: [] for a in ("ll", "oneshot", "twoshot", "nvls")}
bcast = {"pull": [], "mc": []}
for nbytes in sizes:
    x = torch.ones(nbytes // 4, device=dev)
    reps = 20 if nbytes <= (8 << 20) else 5
    for algo in times:
        ok = not (algo == "ll" and nbytes > (64 << 10)) and not (algo == "nvls" and not (nc.has_nvls and size > 2))
        try:
            times[algo].append(time_graph(lambda: m.allreduce(x, MPI.SUM, comm=comm, algorithm=algo), reps) if ok else None)
        except Exception:
            times[algo].append(None)
    if nc.has_nvls and size > 2:
        nc.set_option("bcast_mc_min", 1 << 62)
        bcast["pull"].append(time_graph(lambda: m.bcast(x, 0, comm=comm), reps))
        nc.set_option("bcast_mc_min", 0)
        bcast["mc"].append(time_graph(lambda: m.bcast(x, 0, comm=comm), reps))
    if rank == 0:
        print(nbytes, {a: t[-1] for a, t in times.items()}, {k: (v[-1] if v else None) for k, v in bcast.items()}, flush=True)
nc.set_option("bcast_mc_min", nc.tuning["bcast_mc_min"])

# LL against the best of the others; one-shot against two-shot; the switch against the best pull
others = [min((t for t in (times["oneshot"][i], times["twoshot"][i], times["nvls"][i]) if t is not None), default=None)
          for i in range(len(sizes))]
row = {"ll_max": min(tuning.crossover(sizes, times["ll"], others), 64 << 10),
       "oneshot_max": tuning.crossover(sizes, times["oneshot"], times["twoshot"])}
if nc.has_nvls and size > 2:
    pulls = [min((t for t in (times["oneshot"][i], times["twoshot"][i]) if t is not None), default=None)
             for i in range(len(sizes))]
    row["nvls_min"] = max(tuning.crossover(sizes, pulls, times["nvls"]), row["ll_max"]) + 1
    row["bcast_mc_min"] = tuning.crossover(sizes, bcast["pull"], bcast["mc"]) + 1
if rank == 0:
    doc = {"gpu": torch.cuda.get_device_name(dev), "table": {}}
    if os.path.exists(ns.out):
        try:
            doc = json.load(open(ns.out))
        except Exception:
            pass
    doc.setdefault("table", {})[str(size)] = row
    doc["gpu"] = torch.cuda.get_device_name(dev)
    os.makedirs(os.path.dirname(ns.out) or ".", exist_ok=True)
    with open(ns.out, "w") as fh:
        json.dump(doc, fh, indent=1, sort_keys=True)
    print("wrote", ns.out, {str(size): row}, flush=True)
m.flush()
