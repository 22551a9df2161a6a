"""setuptools entry point: builds the native sm_90a core as part of ``build_ext`` / ``pip install``.

The reference's ``setup.py`` swaps the C compiler for ``mpicc`` and builds up to three
nanobind bridges depending on which toolkits it discovers (/root/reference/setup.py:81-108,
117-179, 375-469).  Here there is one native library with device code, so ``build_ext``
delegates to the parallel nvcc driver in ``mpi4jax_b200/_src/native/build.py`` (CUDA toolkit
discovery: ``$MPI4JAX_B200_NVCC``, ``nvcc`` on PATH, ``$CUDA_HOME``/``$CUDA_PATH``,
``/usr/local/cuda``).  ``MPI4JAX_B200_SKIP_NATIVE_BUILD=1`` installs the pure-Python CPU
(gloo) frontend only, like the reference builds without its CUDA extension when no toolkit
is found.
"""

import importlib.util
import os
import sys
from pathlib import Path

from setuptools import Extension, setup
from setuptools.command.build_ext import build_ext

HERE = Path(__file__).resolve().parent


def _load_builder():
    spec = importlib.util.spec_from_file_location(
        "_b2_build", HERE / "mpi4jax_b200" / "_src" / "native" / "build.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


class nvcc_build_ext(build_ext):
    """Runs the in-tree nvcc build, then places the library where setuptools expects it."""

    def run(self):
        if os.environ.get("MPI4JAX_B200_SKIP_NATIVE_BUILD", "").lower() in ("1", "true", "on"):
            print("mpi4jax_b200: skipping the native build (CPU frontend only)", file=sys.stderr)
            return
        builder = _load_builder()
        try:
            lib = builder.build(verbose=bool(self.verbose > 1))
        except RuntimeError as exc:
            if "nvcc not found" in str(exc):
                print(f"mpi4jax_b200: {exc}; installing the CPU frontend only", file=sys.stderr)
                return
            raise
        if not self.inplace:
            dest = Path(self.build_lib) / "mpi4jax_b200" / "_native"
            dest.mkdir(parents=True, exist_ok=True)
            self.copy_file(str(lib), str(dest / lib.name))

    def get_outputs(self):
        return []


setup(
    # a placeholder Extension makes setuptools run build_ext and tag the wheel as platform-specific
    ext_modules=[Extension("mpi4jax_b200._native.libb2mpi", sources=[])],
    cmdclass={"build_ext": nvcc_build_ext},
)
