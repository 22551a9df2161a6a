"""Device-timed cost of top-k expert routing: ``ops.moe_dispatch`` + ``ops.moe_combine`` (two sm_90a kernels) against
the torch composition a user writes without them, on the same routing:

* dispatch: sort the pairs by expert, repeat every token k times with a gather (N k rows written to HBM), send them
  by destination rank with ``alltoallv`` together with each row's local expert id, and regroup the received rows by
  expert with a stable argsort + gather;
* combine: undo the regroup with ``index_copy``, send the rows back with ``alltoallv_reverse``, put them in their
  ``(N, k)`` slots and take the weighted sum over k.

Timing as in ``loc_reduce_perf.py``: ``--reps`` back-to-back dispatch + combine pairs captured in one CUDA graph, one
replay timed with CUDA events after a barrier, best of ``--trials`` replays, max over ranks.  The card's name and
power limit are read in the same run.  At world size 1 both paths are local copies (the peer is the rank itself):
this measures the gathers, the staging and the folds, not NVLink; a run with several ranks sharing one GPU
measures time-slicing, not the links.

    python scripts/moe_perf.py [--configs N:H:k:E,...] [--out f.jsonl]
    python -m mpi4jax_b200.run -n 8 scripts/moe_perf.py
"""

import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

import mpi4jax_b200 as m  # noqa: E402
from loc_reduce_perf import card, time_graph  # noqa: E402
from mpi4jax_b200 import MPI  # noqa: E402
from mpi4jax_b200._src.collective_ops.alltoallv import alltoallv_reverse  # noqa: E402
from mpi4jax_b200.ops import moe_combine, moe_dispatch  # noqa: E402

# tokens : hidden : k : experts -- Mixtral-like (k = 2, 8 experts) and DeepSeek-like (k = 8, 64 experts) routing
CONFIGS = "4096:4096:2:8,4096:2048:8:64,16384:1024:8:256"


def torch_composition(x, idx, w, E, comm):
    """dispatch (gather + alltoallv + regroup) -> identity experts -> combine (regroup back + alltoallv_reverse +
    weighted sum); returns the combined tokens."""
    N, k = idx.shape
    P = comm.Get_size()
    L = E // P
    key = idx.reshape(-1)
    order = torch.argsort(key, stable=True)
    picked = x[order // k]                                                   # N k rows through HBM
    bounds = torch.searchsorted(key[order], torch.arange(0, E + 1, L, device=x.device))
    send = bounds.diff()
    rows, recv = m.alltoallv(picked, send, comm=comm)
    local = m.alltoallv((key[order] % L).view(-1, 1), send, comm=comm)[0].view(-1)
    filled = torch.arange(rows.shape[0], device=x.device) < recv.sum()
    regroup = torch.argsort(torch.where(filled, local, L), stable=True)      # by expert, then source rank
    grouped = rows[regroup]
    # (the experts would run on `grouped` here)
    back_rows = torch.zeros_like(grouped).index_copy(0, regroup, grouped)
    back = alltoallv_reverse(back_rows, recv, send, N * k, comm)
    slots = torch.zeros_like(back).index_copy(0, order, back).view(N, k, -1)
    return (slots.float() * w[..., None]).sum(1).to(x.dtype)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--configs", default=CONFIGS, help="N:H:k:E,... (bf16 tokens of H elements)")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--trials", type=int, default=5)
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    args = ap.parse_args()
    comm = MPI.COMM_WORLD
    rank, P = comm.Get_rank(), comm.Get_size()
    dev = comm.device
    if dev.type != "cuda":
        raise SystemExit("moe_perf.py measures the GPU path: it needs a CUDA device")
    info = card()
    lines = []
    for cfg in args.configs.split(","):
        N, H, k, E = (int(v) for v in cfg.split(":"))
        E = max(P, E // P * P)
        g = torch.Generator(dev).manual_seed(rank)
        x = torch.randn(N, H, device=dev, generator=g).to(torch.bfloat16)
        idx = torch.rand(N, E, device=dev, generator=g).argsort(1)[:, :k]       # k distinct experts per token
        w = torch.rand(N, k, device=dev, generator=g)

        def fused():
            rows, _, plan = moe_dispatch(x, idx, E, comm=comm)
            return moe_combine(rows, plan, w)

        def composed():
            return torch_composition(x, idx, w, E, comm)

        ref = (x.float() * w.sum(1, keepdim=True)).to(torch.bfloat16)       # identity experts: every pair kept
        for name, fn in (("fused", fused), ("composed", composed)):
            err = (fn().float() - ref.float()).abs().max().item()
            assert err <= 2e-2 * ref.float().abs().max().item(), (name, cfg, err)
        us = {name: time_graph(comm, fn, args.reps, args.trials)
              for name, fn in (("fused", fused), ("composed", composed))}
        row = {"bench": "moe_dispatch_combine", "world": P, "tokens": N, "hidden": H, "k": k, "experts": E,
               "dtype": "bfloat16", "fused_us": round(us["fused"], 1), "composed_us": round(us["composed"], 1),
               "speedup": round(us["composed"] / us["fused"], 2),
               "pair_bytes": N * k * H * 2, **info}
        lines.append(row)
    if rank == 0:
        print(f"# {info['gpu']}, power limit {info['power_limit_w']} W, world size {P}")
        print(f"{'tokens':>7} {'hidden':>6} {'k':>2} {'E':>4} {'fused us':>10} {'torch us':>10} {'speedup':>7}")
        for r in lines:
            print(f"{r['tokens']:>7} {r['hidden']:>6} {r['k']:>2} {r['experts']:>4} {r['fused_us']:>10} "
                  f"{r['composed_us']:>10} {r['speedup']:>7}")
        for r in lines:
            print(json.dumps(r))
        if args.out:
            with open(args.out, "a") as fh:
                for r in lines:
                    fh.write(json.dumps(r) + "\n")
    m.flush()


if __name__ == "__main__":
    main()
