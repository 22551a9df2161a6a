"""In-tree build of the native core (``libb2mpi.so``) for sm_90a (H100).

``python -m mpi4jax_b200._src.native.build`` (or ``__graft_entry__.build()``)
compiles every translation unit under ``csrc/`` with
``nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo`` in parallel and links
them into ``mpi4jax_b200/_native/libb2mpi.so`` (git-ignored).  nvcc cross-compiles
without a GPU, so the library can be built on a machine that has none.

Counterpart of the reference's ``setup.py`` extension build
(/root/reference/setup.py:81-108, 375-431), which swaps the compiler for
``mpicc`` and passes no GPU architecture flags because it contains no device code.
"""

from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

REPO = Path(__file__).resolve().parents[3]
CSRC = REPO / "csrc"
OUT_DIR = REPO / "mpi4jax_b200" / "_native"
OBJ_DIR = OUT_DIR / "obj"
LIB = OUT_DIR / "libb2mpi.so"

ARCH_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=default"]
# extra nvcc flags, e.g. MPI4JAX_B200_NVCC_FLAGS="-DB2_SWE_EXPLICIT_ROUNDING=1" (part of the cache key)
COMMON += os.environ.get("MPI4JAX_B200_NVCC_FLAGS", "").split()


def _nvcc() -> str:
    roots = [os.environ.get(k) for k in ("CUDA_HOME", "CUDA_PATH", "CUDA_ROOT")]
    cands = [os.environ.get("MPI4JAX_B200_NVCC"), shutil.which("nvcc"),
             *[os.path.join(r, "bin", "nvcc") for r in roots if r], "/usr/local/cuda/bin/nvcc"]
    for cand in cands:
        if cand and Path(cand).exists():
            return cand
    raise RuntimeError("nvcc not found; set MPI4JAX_B200_NVCC")


def sources() -> list[Path]:
    return sorted(list(CSRC.glob("*.cu")) + list(CSRC.glob("*.cpp")))


def _headers_digest() -> str:
    h = hashlib.sha1()
    for p in sorted(list(CSRC.glob("*.h")) + list(CSRC.glob("*.cuh"))):
        h.update(p.read_bytes())
    h.update(" ".join(ARCH_FLAGS + COMMON).encode())
    return h.hexdigest()


def _compile_one(nvcc: str, src: Path, digest: str, verbose: bool) -> Path:
    obj = OBJ_DIR / (src.name + ".o")
    stamp = OBJ_DIR / (src.name + ".stamp")
    key = hashlib.sha1(src.read_bytes() + digest.encode()).hexdigest()
    if obj.exists() and stamp.exists() and stamp.read_text() == key:
        return obj
    cmd = [nvcc, *ARCH_FLAGS, *COMMON, "-I", str(CSRC), "-c", str(src), "-o", str(obj)]
    if src.suffix == ".cpp":
        cmd.insert(1, "-x")
        cmd.insert(2, "cu")
    if verbose:
        cmd += ["-Xptxas", "-v"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src.name}:\n{res.stdout}\n{res.stderr}")
    if verbose:
        sys.stderr.write(res.stderr)
    stamp.write_text(key)
    return obj


def build(force: bool = False, verbose: bool = False) -> Path:
    """Compile (if stale) and link the native library; returns its path."""
    nvcc = _nvcc()
    OBJ_DIR.mkdir(parents=True, exist_ok=True)
    if force:
        for p in OBJ_DIR.glob("*"):
            p.unlink()
    digest = _headers_digest()
    srcs = sources()
    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(lambda s: _compile_one(nvcc, s, digest, verbose), srcs))
    newest = max(o.stat().st_mtime for o in objs)
    if force or not LIB.exists() or LIB.stat().st_mtime < newest:
        cmd = [nvcc, *ARCH_FLAGS, "-shared", "-o", str(LIB), *map(str, objs), "-lpthread"]
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            raise RuntimeError(f"link failed:\n{res.stdout}\n{res.stderr}")
    return LIB


def needs_build() -> bool:
    if not LIB.exists():
        return True
    lib_m = LIB.stat().st_mtime
    return any(p.stat().st_mtime > lib_m for p in list(CSRC.glob("*")))


if __name__ == "__main__":
    path = build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(path)
