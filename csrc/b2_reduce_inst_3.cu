// Typed instantiations of the fused reduce kernels, dtype group 3: bool and complex (see b2_reduce.cuh).
#include "b2_reduce.cuh"

void b2_register_reduce_group_3() {
  B2_REG(B2_BOOL, b2_boolean, B2_LAND)
  B2_REG(B2_BOOL, b2_boolean, B2_LOR)
  B2_REG(B2_BOOL, b2_boolean, B2_LXOR)
  B2_REG(B2_C64, b2_c64, B2_SUM)
  B2_REG(B2_C64, b2_c64, B2_PROD)
  B2_REG(B2_C128, b2_c128, B2_SUM)
  B2_REG(B2_C128, b2_c128, B2_PROD)
}
