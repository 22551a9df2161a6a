// Typed instantiations of the fused reduce kernels, dtype group 2: unsigned integers (see b2_reduce.cuh).
#include "b2_reduce.cuh"

void b2_register_reduce_group_2() {
  B2_REG_INT(B2_U8, unsigned char)
  B2_REG_INT(B2_U16, unsigned short)
  B2_REG_INT(B2_U32, unsigned int)
  B2_REG_INT(B2_U64, unsigned long long)
}
