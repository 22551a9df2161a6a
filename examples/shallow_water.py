"""mpi4jax_b200 demo application -- Shallow water

The reference's demo (/root/reference/examples/shallow_water.py), a non-linear shallow-water
solver adapted from https://github.com/dionhaefner/shallow-water, on the H100-native stack.

Usage examples:

    # runs the demo on 4 processes (one GPU each; --cpu for the gloo backend)
    $ python -m mpi4jax_b200.run -n 4 examples/shallow_water.py

    # runs the demo as a benchmark (no output), 4096x4096 grid as in BASELINE.json
    $ python -m mpi4jax_b200.run -n 8 examples/shallow_water.py --benchmark --nx 4096 --ny 4096

    # saves the output animation as shallow-water.mp4 (needs matplotlib + ffmpeg)
    $ python -m mpi4jax_b200.run -n 4 examples/shallow_water.py --save-animation

    # integrate with the public p2p ops instead of the fused native kernels
    $ python -m mpi4jax_b200.run -n 4 examples/shallow_water.py --backend ops
"""

import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

import mpi4jax_b200  # noqa: E402
from mpi4jax_b200 import MPI  # noqa: E402
from mpi4jax_b200.models import (  # noqa: E402
    ModelState,
    ShallowWaterConfig,
    ShallowWaterModel,
    solve_shallow_water,
)

DAY_IN_SECONDS = 86_400
PLOT_EVERY = 100
PLOT_ETA_RANGE = 10
MAX_QUIVERS = (25, 50)


def animate_shallow_water(sol, model):
    """Create a matplotlib animation of the result (rank 0, global fields)."""
    import matplotlib.pyplot as plt
    import numpy as np
    from matplotlib import animation

    cfg = model.cfg
    x = np.arange(-1, model.nx_global - 1) * cfg.dx
    y = np.arange(-1, model.ny_global - 1) * cfg.dy
    qs = (slice(1, -1, max(1, model.ny_global // MAX_QUIVERS[0])),
          slice(1, -1, max(1, model.nx_global // MAX_QUIVERS[1])))
    yy, xx = np.meshgrid(y, x, indexing="ij")
    fig = plt.figure(figsize=(6, 4))
    ax = plt.gca()
    cs = ax.pcolormesh(0.5 * (x[:-1] + x[1:]) / 1e3, 0.5 * (y[:-1] + y[1:]) / 1e3,
                       sol[0].h[1:-1, 1:-1] - cfg.depth, vmin=-PLOT_ETA_RANGE, vmax=PLOT_ETA_RANGE,
                       cmap="RdBu_r")
    cq = ax.quiver(xx[qs] / 1e3, yy[qs] / 1e3, sol[0].u[qs], sol[0].v[qs], clip_on=True)
    label = ax.text(s="", x=0.05, y=0.95, ha="left", va="top", backgroundcolor=(1, 1, 1, 0.8),
                    transform=ax.transAxes)
    ax.set(aspect="equal", xlabel="$x$ (km)", ylabel="$y$ (km)")
    plt.colorbar(cs, orientation="horizontal", label="Surface height anomaly (m)", pad=0.2, shrink=0.8)
    fig.tight_layout()

    def frame(i):
        cs.set_array((sol[i].h - cfg.depth)[1:-1, 1:-1].flatten())
        cq.set_UVC(sol[i].u[qs], sol[i].v[qs])
        label.set_text(f"t = {PLOT_EVERY * cfg.dt * i / DAY_IN_SECONDS:.2f} days")
        return cs, cq, label

    return animation.FuncAnimation(fig, frame, frames=len(sol), interval=50, blit=True,
                                   repeat_delay=3_000)


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--benchmark", action="store_true", help="exit after the solve (no output)")
    ap.add_argument("--save-animation", action="store_true")
    ap.add_argument("--nx", type=int, default=360)
    ap.add_argument("--ny", type=int, default=180)
    ap.add_argument("--days", type=float, default=None, help="model days (default 10; 0.1 with --benchmark)")
    ap.add_argument("--backend", default="auto", choices=["auto", "native", "ops"])
    ns = ap.parse_args(argv)

    comm = MPI.COMM_WORLD
    days = ns.days if ns.days is not None else (0.1 if ns.benchmark else 10.0)
    cfg = (ShallowWaterConfig(nx=ns.nx, ny=ns.ny) if (ns.nx, ns.ny) == (360, 180)
           else ShallowWaterConfig.for_resolution(ns.nx, ns.ny))
    sol = solve_shallow_water(t1=days * DAY_IN_SECONDS, num_multisteps=PLOT_EVERY, config=cfg,
                              comm=comm, backend=ns.backend)
    if ns.benchmark:
        mpi4jax_b200.flush()
        return 0

    # copy the solution to rank 0 (reference :579-584 does one gather of the stacked snapshots)
    model = ShallowWaterModel(cfg, comm=comm, backend=ns.backend)
    stacked = torch.stack([torch.stack(list(s[:3])) for s in sol])       # (time, 3, ny, nx)
    full = mpi4jax_b200.gather(stacked, root=0, comm=comm)
    if comm.Get_rank() == 0:
        import numpy as np

        frames = []
        for t in range(full.shape[1]):
            fields = []
            for k in range(3):
                out = torch.empty((model.ny_global, model.nx_global))
                for r in range(comm.Get_size()):
                    iy, ix = np.unravel_index(r, (model.nproc_y, model.nproc_x))
                    sl = (slice((model.ny_local - 2) * iy, (model.ny_local - 2) * iy + model.ny_local),
                          slice((model.nx_local - 2) * ix, (model.nx_local - 2) * ix + model.nx_local))
                    out[sl] = full[r, t, k].cpu()
                fields.append(out.numpy())
            frames.append(ModelState(*fields, None, None, None))
        anim = animate_shallow_water(frames, model)
        if ns.save_animation:
            anim.save("shallow-water.mp4", writer="ffmpeg", dpi=100)
        else:
            import matplotlib.pyplot as plt

            plt.show()
    return 0


if __name__ == "__main__":
    sys.exit(main())
