"""``python -m mpi4jax_b200.info`` -- what this installation can do (build, devices, transports).

The reference prints the MPI vendor / rank / size in the pytest header (tests/conftest.py:1-9) and
exposes ``MPI_ABI_INFO``; this is the same information for the NVLink transport, usable in bug
reports and job logs (add ``--json`` for machine-readable output)."""

from __future__ import annotations

import json
import os
import sys


def collect() -> dict:
    import torch

    import mpi4jax_b200 as m
    from mpi4jax_b200._src import native, torch_compat
    from mpi4jax_b200._src.backends import transport

    info = {
        "version": m.__version__,
        "torch": torch.__version__,
        "latest_tested_torch": torch_compat.LATEST_TESTED_TORCH,
        "native_library": native.NATIVE_ABI_INFO["library"],
        "native_loaded": native.HAS_CUDA_EXT,
        "native_error": None if native.HAS_CUDA_EXT else native.CUDA_EXT_ERROR,
        "native_abi": native.NATIVE_ABI_INFO["native"],
        "cuda_available": torch.cuda.is_available(),
        "device_count": torch.cuda.device_count() if torch.cuda.is_available() else 0,
        "requested_transport": transport.requested(),
        "env": {k: v for k, v in sorted(os.environ.items()) if k.startswith(("MPI4JAX_", "RANK", "WORLD_SIZE",
                                                                            "LOCAL_RANK", "MASTER_"))},
    }
    devices = []
    for i in range(info["device_count"]):
        caps = torch_compat.device_capabilities(i)
        props = torch.cuda.get_device_properties(i)
        devices.append({"index": i, "name": props.name, "sm": list(caps["sm"] or ()),
                        "sm_90": caps["sm_90"], "memory_gib": round(props.total_memory / 2**30, 1),
                        "sms": props.multi_processor_count, "vmm": caps["vmm"], "multicast": caps["multicast"]})
    info["devices"] = devices
    return info


def main(argv=None) -> int:
    argv = sys.argv[1:] if argv is None else argv
    info = collect()
    if "--json" in argv:
        print(json.dumps(info, indent=1, default=str))
        return 0
    print(f"mpi4jax_b200 {info['version']}  (torch {info['torch']}, tested up to {info['latest_tested_torch']})")
    state = "loaded" if info["native_loaded"] else f"NOT loaded ({info['native_error']})"
    print(f"native core   : {info['native_library']}  [{state}]")
    if info["native_abi"]:
        print(f"native ABI    : {info['native_abi']}")
    print(f"CUDA          : available={info['cuda_available']}  devices={info['device_count']}  "
          f"transport request={info['requested_transport']}")
    for d in info["devices"]:
        print(f"  cuda:{d['index']}  {d['name']}  sm_{''.join(map(str, d['sm']))}  {d['sms']} SMs  "
              f"{d['memory_gib']} GiB  vmm={d['vmm']}  multicast(NVLS)={d['multicast']}"
              + ("" if d["sm_90"] else "   [not a Hopper sm_90 device: the kernels will not load]"))
    for k, v in info["env"].items():
        print(f"  {k}={v}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
