// Typed instantiations of the fused reduce kernels, dtype group 4: float8 e4m3fn and e5m2 (see b2_reduce.cuh).
// No in-switch path: multimem.ld_reduce has no float8 form on sm_90a.
#include "b2_reduce.cuh"

void b2_register_reduce_group_4() {
  B2_REG_ARITH(B2_F8E4M3, b2_f8e4m3)
  B2_REG_ARITH(B2_F8E5M2, b2_f8e5m2)
}
