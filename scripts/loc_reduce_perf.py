"""Device-timed latency and bandwidth of MAXLOC against its neighbours, f32 values + int64 indices:

* ``maxloc``: ``allreduce((v, i), MPI.MAXLOC)`` -- the staged one-shot pull of 16-byte records;
* ``max``: ``allreduce(v, MPI.MAX)`` alone (the LL flag-in-data path at small sizes), the floor a value-only
  reduction reaches;
* ``allgather_argmax``: what a user writes without MAXLOC -- two allgathers, then a tie-correct argmax in
  torch (NaN-propagating max, smallest index among the ranks that hold it).

Timing: ``--reps`` back-to-back calls captured in one CUDA graph, one replay timed with CUDA events after a
barrier, best of ``--trials`` replays, max over ranks (the kernels' time, not the Python launch path); the
graph is warmed up by two eager calls and one untimed replay.  ``GBps`` is the pair bytes per rank (12 per
pair) over that time.  Each JSON line carries the card name and its power limit, read in the same run.

    python -m mpi4jax_b200.run -n 8 scripts/loc_reduce_perf.py [--pairs 1,1024,65536,16777216] [--out f.jsonl]
"""

import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

import mpi4jax_b200 as m  # noqa: E402
from mpi4jax_b200 import MPI  # noqa: E402
from mpi4jax_b200.utils import max_over_ranks  # noqa: E402


def card() -> dict:
    """Name and power limit of this rank's GPU (a read-only nvidia-smi query)."""
    idx = torch.cuda.current_device()
    info = {"gpu": torch.cuda.get_device_name(idx), "power_limit_w": None}
    try:
        out = subprocess.run(["nvidia-smi", f"--id={idx}", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit_w"] = float(out)
    except (OSError, ValueError, subprocess.SubprocessError):
        pass
    return info


def time_graph(comm, fn, reps, trials):
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
    for _ in range(trials):
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


def allgather_argmax(v, i, comm):
    vv, ii = m.allgather(v, comm=comm), m.allgather(i, comm=comm)
    best = vv.amax(0)
    holds = (vv == best) | (vv.isnan() & best.isnan())
    return best, torch.where(holds, ii, torch.iinfo(ii.dtype).max).amin(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", default="1,1024,65536,16777216")
    ap.add_argument("--trials", type=int, default=5)
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file (rank 0)")
    args = ap.parse_args()
    comm = MPI.COMM_WORLD.Clone()
    rank, size = comm.Get_rank(), comm.Get_size()
    dev = comm.device
    if dev.type != "cuda":
        raise SystemExit("loc_reduce_perf.py measures the GPU path: no CUDA device")
    meta = {"ranks": size, "gpus_on_node": torch.cuda.device_count(), **card()}
    meta["ranks_share_a_gpu"] = size > meta["gpus_on_node"]
    lines = []
    for n in (int(s) for s in args.pairs.split(",")):
        gen = torch.Generator(dev).manual_seed(rank)
        v = torch.randn(n, device=dev, generator=gen)
        i = torch.randint(0, 1 << 40, (n,), device=dev, generator=gen)
        want = m.allreduce((v, i), MPI.MAXLOC, comm=comm)
        got = allgather_argmax(v, i, comm)
        assert torch.equal(want[0], got[0]) and torch.equal(want[1], got[1]), "the two MAXLOC forms disagree"
        reps = 200 if n <= 1 << 16 else 20 if n <= 1 << 20 else 3
        variants = {
            "maxloc": lambda: m.allreduce((v, i), MPI.MAXLOC, comm=comm),
            "max": lambda: m.allreduce(v, MPI.MAX, comm=comm),
            "allgather_argmax": lambda: allgather_argmax(v, i, comm),
        }
        for name, fn in variants.items():
            us = time_graph(comm, fn, reps, args.trials)
            lines.append({"variant": name, "pairs": n, "us": round(us, 2), "GBps": round(12 * n / us / 1e3, 3),
                          **meta})
        del v, i, want, got
        torch.cuda.empty_cache()
    if rank == 0:
        for line in lines:
            print(json.dumps(line), flush=True)
        if args.out:
            with open(args.out, "a") as fh:
                fh.writelines(json.dumps(line) + "\n" for line in lines)
    m.flush()


if __name__ == "__main__":
    main()
