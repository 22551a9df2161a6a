// Typed instantiations of the fused reduce kernels, dtype group 0: float types (see b2_reduce.cuh).
#include "b2_reduce.cuh"

void b2_register_reduce_group_0() {
  B2_REG_ARITH(B2_F32, float)
  B2_REG_ARITH(B2_F64, double)
  B2_REG_ARITH(B2_F16, __half)
  B2_REG_ARITH(B2_BF16, __nv_bfloat16)
}
