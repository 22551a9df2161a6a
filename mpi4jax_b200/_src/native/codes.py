"""Numeric codes shared with the native core (csrc/b2_common.h)."""

from __future__ import annotations

import torch

# enum B2DType
F32, F64, F16, BF16, I8, I16, I32, I64, U8, U16, U32, U64, BOOL, C64, C128 = range(15)

DTYPE_CODE = {
    torch.float32: F32,
    torch.float64: F64,
    torch.float16: F16,
    torch.bfloat16: BF16,
    torch.int8: I8,
    torch.int16: I16,
    torch.int32: I32,
    torch.int64: I64,
    torch.uint8: U8,
    torch.uint16: U16,
    torch.uint32: U32,
    torch.uint64: U64,
    torch.bool: BOOL,
    torch.complex64: C64,
    torch.complex128: C128,
}

# Hopper's two 8-bit float formats (no MPI predefined datatype): every data-movement collective moves them
# as bytes, the reductions widen to fp32, fold, and round once (csrc/b2_device.cuh)
F8E4M3, F8E5M2 = 15, 16
FP8_DTYPE_CODE = {
    torch.float8_e4m3fn: F8E4M3,
    torch.float8_e5m2: F8E5M2,
}

# every dtype with a wire representation
WIRE_DTYPE_CODE = {**DTYPE_CODE, **FP8_DTYPE_CODE}

# enum B2Op
SUM, PROD, MIN, MAX, LAND, LOR, LXOR, BAND, BOR, BXOR = range(10)
MAXLOC, MINLOC = 10, 11         # value-index reductions: not members of the [dtype][op] kernel tables

# enum B2Algo
ALGO_AUTO, ALGO_LL, ALGO_ONESHOT, ALGO_TWOSHOT, ALGO_NVLS = range(5)
ALGO_BY_NAME = {
    "auto": ALGO_AUTO,
    "ll": ALGO_LL,
    "oneshot": ALGO_ONESHOT,
    "twoshot": ALGO_TWOSHOT,
    "nvls": ALGO_NVLS,
}

# enum B2OpCode (subset used from Python)
OPC_ALLREDUCE, OPC_REDUCE, OPC_SCAN, OPC_ALLGATHER, OPC_ALLTOALL = 1, 2, 3, 4, 5
OPC_BCAST, OPC_GATHER, OPC_SCATTER = 6, 7, 8
OPC_REDUCE_SCATTER = 13
OPC_ALLTOALLV = 14
OPC_ALLGATHERV = 15
OPC_REDUCE_SCATTERV = 16
OPC_GATHERV = 17
OPC_SCATTERV = 18
OPC_MOE_DISPATCH = 19
OPC_MOE_COMBINE = 20

# experts a top-k dispatch may route to (B2_MOE_MAX_EXPERTS: the kernel keeps every rank's per-expert counts in
# shared memory)
MOE_MAX_EXPERTS = 256

# MPI names of the reduction collectives (debug log lines, error messages)
OPC_REDUCTION_NAME = {OPC_ALLREDUCE: "Allreduce", OPC_REDUCE: "Reduce", OPC_SCAN: "Scan",
                      OPC_REDUCE_SCATTER: "Reduce_scatter_block"}

ANY = -1  # ANY_SOURCE / ANY_TAG on the wire
