"""Device-side timeline of the communication-avoiding shallow-water step INSIDE a CUDA-graph replay:
first-CTA-start / last-CTA-end (%globaltimer) of the four kernels of each step, relative to the
step's first event.  A = frame tendencies, S = bulk (one step; of a pair of steps, S2 in the first and
the ring launch in the second), X = halo exchange,
D = frame friction.  Works at any world size (every rank prints its own table to its log).

    python -m mpi4jax_b200.run -n 8 scripts/swe_timeline.py [grid] [steps]
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import mpi4jax_b200 as m  # noqa: E402
from mpi4jax_b200 import MPI  # noqa: E402
from mpi4jax_b200._src import native  # noqa: E402
from mpi4jax_b200.models import ShallowWaterConfig, ShallowWaterModel  # noqa: E402

grid = int(sys.argv[1]) if len(sys.argv) > 1 else 4096
steps = int(sys.argv[2]) if len(sys.argv) > 2 else 8
comm = MPI.COMM_WORLD
model = ShallowWaterModel(ShallowWaterConfig.for_resolution(grid, grid), comm=comm, device=comm.device)
model.step(first_step=True)
buf = torch.zeros((steps, 4, 2), dtype=torch.int64, device=comm.device)
native.lib.b2_swe_ca_timeline(buf.data_ptr(), steps)
run = m.jit(lambda: model.multistep(steps, first_step=False), warmup=0)
run()                                   # capture + one replay
for _ in range(3):                      # warm replays
    run()
buf[:, :, 0] = torch.iinfo(torch.int64).max
buf[:, :, 1] = 0
torch.cuda.synchronize()
comm.Barrier()
m.barrier(comm=comm)
run()
torch.cuda.synchronize()
native.lib.b2_swe_ca_timeline(None, 0)
t = buf.cpu().double()
names = ["A", "S", "X", "D"]
if comm.Get_rank() in (0, comm.Get_size() - 1):
    print(f"rank {comm.Get_rank()} of {comm.Get_size()}: local block {model.ny_local}x{model.nx_local}", flush=True)
    t0 = t[0, :, 0].min()
    prev_end = None
    for s in range(steps):
        base = t[s, :, 0].min()
        row = "  ".join(f"{names[k]} {(t[s, k, 0] - base) / 1e3:6.1f}-{(t[s, k, 1] - base) / 1e3:6.1f}" for k in range(4))
        end = t[s, :, 1].max()
        print(f"step {s}: start +{(base - t0) / 1e3:7.1f} us | {row} | step {(end - base) / 1e3:6.1f} us", flush=True)
    total = (t[:, :, 1].max() - t0) / 1e3
    print(f"rank {comm.Get_rank()}: {steps} steps in {total:.1f} us = {total / steps:.1f} us/step", flush=True)
m.flush()
