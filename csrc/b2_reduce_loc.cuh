// mpi4jax_b200 -- value-index reductions (MAXLOC / MINLOC): the launch arguments and the launcher table
// shared by the kernel file (b2_reduce_loc.cu) and the entry point (b2_collectives.cu).
#pragma once

#include "b2_device.cuh"

// Staging record of one (value, index) pair: 16 bytes, the value's bits zero-extended to 8 bytes, then the
// index as int64 (int32 indices sign-extended).  A pair is one 16-byte peer load.
#define B2_LOC_RECORD 16

struct B2LocArgs {
  const void* in_val;
  const void* in_idx;
  void* out_val;
  void* out_idx;
  size_t count;       // pairs per block (reduce-scatter: per destination; otherwise the whole input)
  size_t chunk;       // chunk bytes of the staged records; a multiple of 16 * size
  int idx_bytes;      // 4 or 8
  int src_lo;         // the pairs folded: ranks [src_lo, src_hi), in rank order
  int src_hi;
  int has_out;        // this rank stores a result (reduce: root only)
  int nblk;           // blocks staged by every rank: size for reduce-scatter, else 1
  int opcode;
};

typedef void (*b2_loc_launch_fn)(const B2DevComm&, const B2LocArgs&, int grid, cudaStream_t);

// [value dtype][0: MAXLOC, 1: MINLOC]; nullptr for a value dtype without a pair kernel.  b2_loc_kernel holds
// the kernel itself, for the co-residency query.
extern b2_loc_launch_fn b2_loc_table[B2_DTYPE_COUNT][2];
extern const void* b2_loc_kernel[B2_DTYPE_COUNT][2];
void b2_register_reduce_loc();
