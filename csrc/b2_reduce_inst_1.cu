// Typed instantiations of the fused reduce kernels, dtype group 1: signed integers (see b2_reduce.cuh).
#include "b2_reduce.cuh"

void b2_register_reduce_group_1() {
  B2_REG_INT(B2_I8, signed char)
  B2_REG_INT(B2_I16, short)
  B2_REG_INT(B2_I32, int)
  B2_REG_INT(B2_I64, long long)
}
