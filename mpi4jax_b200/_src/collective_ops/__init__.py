"""The 13 communication primitives (one module per op, like the reference's
mpi4jax/_src/collective_ops/)."""

from types import SimpleNamespace

from . import (allgather, allgatherv, allreduce, alltoall, alltoallv, gatherv, reduce, reduce_scatter, reduce_scatterv,
               scatterv, sendrecv)

# the eager frontend as ``F`` of the shared adjoint rules (_adjoints.py)
eager = SimpleNamespace(allgather=allgather.allgather, allreduce=allreduce.allreduce, alltoall=alltoall.alltoall,
                        alltoallv=alltoallv.alltoallv, _alltoallv_reverse=alltoallv.alltoallv_reverse,
                        _allgatherv_reverse=allgatherv.allgatherv_reverse,
                        _gatherv_reverse=gatherv.gatherv_reverse, _scatterv_bounded=scatterv.scatterv_bounded,
                        reduce=reduce.reduce, reduce_scatter=reduce_scatter.reduce_scatter,
                        reduce_scatterv=reduce_scatterv.reduce_scatterv, sendrecv=sendrecv.sendrecv)
