"""Device-timed cost of float8 collectives against bf16 and f32 at equal ELEMENT counts:

* reductions: ``allreduce(x, MPI.SUM)`` and ``reduce_scatter`` (blocks of ``n`` elements) for e4m3fn, bf16
  and f32 -- fp8 moves a quarter of f32's bytes and half of bf16's, and widens / narrows in the kernel;
* data movement: ``allgather`` and ``alltoallv`` (``n`` elements split evenly over the ranks) for e4m3fn and
  bf16, which move bytes.

Timing as in ``loc_reduce_perf.py``: ``--reps`` back-to-back calls captured in one CUDA graph, one replay
timed with CUDA events after a barrier, best of ``--trials`` replays, max over ranks.  Each JSON line names
the transport the reduction took (from the debug log of one eager call), the world size, and the card's
name and power limit, read in the same run.  At world size 1 every op is a staging copy in and out plus the
conversions: it measures those, not NVLink.

    python -m mpi4jax_b200.run -n 8 scripts/fp8_collectives_perf.py [--elems 1024,...] [--out f.jsonl]
"""

import argparse
import contextlib
import io
import json
import os
import re
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

import mpi4jax_b200 as m  # noqa: E402
from loc_reduce_perf import card, time_graph  # noqa: E402
from mpi4jax_b200 import MPI  # noqa: E402
from mpi4jax_b200._src.native import set_logging  # noqa: E402

ELEMS = ",".join(str(1 << k) for k in range(10, 27, 2))     # 1 Ki ... 64 Mi


def transport(fn) -> str:
    """The transport named in the debug log line of one eager call of ``fn``."""
    buf = io.StringIO()
    set_logging(True)
    try:
        with contextlib.redirect_stdout(buf):
            fn()
            m.flush()
    finally:
        set_logging(False)
    found = re.findall(r" via (\w+)$", buf.getvalue(), re.M)
    return found[0] if found else "-"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--elems", default=ELEMS)
    ap.add_argument("--trials", type=int, default=5)
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file (rank 0)")
    args = ap.parse_args()
    comm = MPI.COMM_WORLD.Clone()
    rank, size = comm.Get_rank(), comm.Get_size()
    dev = comm.device
    if dev.type != "cuda":
        raise SystemExit("fp8_collectives_perf.py measures the GPU path: no CUDA device")
    meta = {"ranks": size, "gpus_on_node": torch.cuda.device_count(), **card()}
    meta["ranks_share_a_gpu"] = size > meta["gpus_on_node"]
    lines = []
    for n in (int(s) for s in args.elems.split(",")):
        gen = torch.Generator(dev).manual_seed(rank)
        base = torch.randn(n, device=dev, generator=gen)
        blocks = torch.randn(size, n, device=dev, generator=gen)
        per = n // size
        counts = torch.full((size,), per, dtype=torch.int64, device=dev)
        reps = 100 if n <= 1 << 16 else 20 if n <= 1 << 22 else 3
        for dt in (torch.float8_e4m3fn, torch.bfloat16, torch.float32):
            x, xb = base.to(dt), blocks.to(dt)
            rows = x[: per * size].reshape(per * size, 1)
            ops = {"allreduce_sum": lambda: m.allreduce(x, MPI.SUM, comm=comm),
                   "reduce_scatter_sum": lambda: m.reduce_scatter(xb, MPI.SUM, comm=comm)}
            if dt != torch.float32:
                ops["allgather"] = lambda: m.allgather(x, comm=comm)
                ops["alltoallv"] = lambda: m.alltoallv(rows, counts, comm=comm)
            for name, fn in ops.items():
                via = transport(fn) if name.endswith("_sum") else "-"
                us = time_graph(comm, fn, reps, args.trials)
                lines.append({"op": name, "dtype": str(dt).replace("torch.", ""), "elems": n, "via": via,
                              "us": round(us, 2), "GBps": round(n * x.element_size() / us / 1e3, 3), **meta})
            del x, xb, rows
        del base, blocks
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
