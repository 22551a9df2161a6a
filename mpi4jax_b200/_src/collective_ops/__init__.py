"""The 13 communication primitives (one module per op, like the reference's
mpi4jax/_src/collective_ops/)."""
