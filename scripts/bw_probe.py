"""Where does the large-message bandwidth go?  Times the bandwidth-bound collectives at one size for
several grid caps (communicator option max_blocks) next to the p2p ring (64 lanes), device time of a
CUDA graph of a few launches, max over ranks.  usage: python -m mpi4jax_b200.run -n N scripts/bw_probe.py [MiB]"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import mpi4jax_b200 as m  # noqa: E402
from mpi4jax_b200 import MPI  # noqa: E402

comm = MPI.COMM_WORLD
rank, size = comm.Get_rank(), comm.Get_size()
dev = comm.device
mib = int(sys.argv[1]) if len(sys.argv) > 1 else 256
nbytes = mib << 20
nc = comm._native_comm()
comm_reserve = getattr(m, "comm_reserve", None)
if comm_reserve:
    comm_reserve(nbytes, comm=comm)


def time_graph(fn, reps=4):
    fn(); fn()
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
    best = 1e30
    for _ in range(3):
        comm.Barrier()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record(); g.replay(); e.record(); e.synchronize()
        best = min(best, s.elapsed_time(e) * 1e3 / reps)
    t = torch.tensor([best], device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t)


x = torch.ones(nbytes // 4, device=dev)
blk = torch.ones(nbytes // 4 // size, device=dev)
a2a = torch.ones(size, nbytes // 4 // size, device=dev)
ops = {
    "allreduce": (lambda: m.allreduce(x, MPI.SUM, comm=comm), 2 * (size - 1) / size * nbytes),
    "allreduce_max": (lambda: m.allreduce(x, MPI.MAX, comm=comm), 2 * (size - 1) / size * nbytes),
    "allgather": (lambda: m.allgather(blk, comm=comm), (size - 1) / size * nbytes),
    "alltoall": (lambda: m.alltoall(a2a, comm=comm), (size - 1) / size * nbytes),
    "bcast": (lambda: m.bcast(x, 0, comm=comm), nbytes),
    "reduce": (lambda: m.reduce(x, MPI.SUM, 0, comm=comm), nbytes),
    "sendrecv": (lambda: m.sendrecv(x, x, source=(rank - 1) % size, dest=(rank + 1) % size, comm=comm), nbytes),
}
sms = nc.get_option("sm_count")
for mb in ((sms, 2 * sms) if size > 2 else (64, sms, 2 * sms)):
    nc.set_option("max_blocks", mb)
    for pipe in (0, 1):
        nc.set_option("nvls_pipeline", pipe)
        row = {}
        for name, (fn, moved) in ops.items():
            if pipe == 1 and name not in ("allreduce",):
                continue
            us = time_graph(fn)
            row[name] = (round(us, 1), round(moved / us / 1e3, 1))
        if rank == 0:
            print(f"{mib} MiB max_blocks={mb} nvls_pipeline={pipe}:", row, flush=True)
nc.set_option("max_blocks", sms)
t = x.clone()
us = time_graph(lambda: dist.all_reduce(t))
us2 = time_graph(lambda: dist.broadcast(t, 0))
if rank == 0:
    print(f"nccl allreduce {round(us, 1)} us {round(2 * (size - 1) / size * nbytes / us / 1e3, 1)} GB/s; bcast {round(us2, 1)} us "
          f"{round(nbytes / us2 / 1e3, 1)} GB/s", flush=True)
m.flush()
