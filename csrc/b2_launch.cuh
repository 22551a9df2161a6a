// mpi4jax_b200 -- kernel launch helper with programmatic dependent launch (PDL).
//
// The shallow-water step is 7 short kernels (4 stencils + 3 halo exchanges); at 8 GPUs each is
// short enough that the launch/drain gap between stream-ordered kernels is a visible part of
// the step.  With PDL the next kernel's CTAs are scheduled while the previous kernel drains and
// block in `griddepcontrol.wait` until its memory is visible: same semantics, shorter gaps.
// Works in eager mode and inside CUDA-graph capture (programmatic edges).  Every kernel launched
// through b2_launch() MUST call b2_pdl_enter() before its first global memory access.
#pragma once
#include <cuda_runtime.h>
#include <utility>

#ifdef __CUDACC__
// trigger first: the successor may be scheduled as soon as all CTAs of this grid are resident;
// it still blocks in its own wait until this grid has completed and flushed.
__device__ __forceinline__ void b2_pdl_enter() {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");
}
#endif

extern "C" int b2_pdl_enabled(void);
extern "C" void b2_set_pdl(int enable);

template <typename... KArgs, typename... Args>
static inline cudaError_t b2_launch(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem,
                                    cudaStream_t stream, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = b2_pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, KArgs(std::forward<Args>(args))...);
}
