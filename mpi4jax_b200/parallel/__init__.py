"""Parallelism patterns assembled from the primitives.

The reference is a message-passing substrate and ships no DP/TP/PP/SP library code
(SURVEY.md section 2.5); what it has are user-level patterns in its tests and example.
They are provided here as small, tested helpers:

* ``average_gradients`` / ``broadcast_parameters``   data parallel (test_allreduce.py:251-322)
* ``column_parallel_matvec`` / ``row_parallel_matvec`` tensor parallel (test_allreduce_matvec.py:41-65)
* ``ring_shift``                                      sequence/context-parallel building block
* ``alltoall_reshard``                                Ulysses-style head<->sequence reshard
* ``expert_dispatch`` / ``expert_combine``            mixture-of-experts token routing (alltoallv)
* ``pipeline_send`` / ``pipeline_recv``               differentiable stage boundary (extension)
* ``cartesian_neighbors``                             2-D domain decomposition (shallow_water.py:64-107)
"""

from .patterns import (  # noqa: F401
    alltoall_reshard,
    average_gradients,
    broadcast_parameters,
    cartesian_neighbors,
    column_parallel_matvec,
    expert_combine,
    expert_dispatch,
    pipeline_recv,
    pipeline_send,
    ring_shift,
    row_parallel_matvec,
)
