// mpi4jax_b200 -- row-parallel linear layer: GEMM + allreduce in ONE kernel.
//
//   out = allreduce_SUM_over_ranks( X_r (M x K_r, bf16)  @  W_r^T (W_r: N x K_r, bf16) )
//
// This is the tensor-parallel pattern the reference only has as a user-level test
// (column-sharded mat-vec followed by mpi4jax.allreduce,
// tests/collective_ops/test_allreduce_matvec.py:41-65).  There the product is one XLA op and
// the reduction a blocking MPI call afterwards; here both are one sm_90a kernel:
//
//   * Hopper tensor cores: `wgmma.mma_async.m64n128k16.f32.bf16.bf16` (bf16 in, fp32 accumulate in
//     registers), operands read straight from shared memory through GMMA descriptors; the operands
//     are staged by TMA (`cp.async.bulk.tensor.2d`, 128-byte swizzle) through a 6-stage mbarrier
//     ring that the producer warp keeps filling, also across tile boundaries;
//   * the consumer warpgroups turn a finished tile into bf16, store it into this rank's SYMMETRIC
//     staging buffer and then all-reduce that tile right there, tile by tile: block-paired
//     cross-GPU barrier (the same tile is owned by the same CTA index on every rank),
//     `multimem.ld_reduce.add.acc::f32.v4.bf16x2` of this rank's 1/P row-slice of the tile (summed in
//     fp32 INSIDE the NVSwitch), `multimem.st` of the result to every rank, second barrier, copy of
//     the finished tile to the output.  NVLink traffic equals that of a stand-alone bf16 allreduce;
//     the producer prefetches the next tiles' operands meanwhile.
//
// Roles (384 threads): warpgroup 0 = TMA producer (one thread), warpgroups 1 and 2 = MMA + epilogue
// + per-tile collective, each owning 64 rows of the 128 x 128 tile.
// Persistent: grid = min(#tiles, #SMs), every CTA walks tiles blockIdx.x, +gridDim.x, ...
// Shapes: M, N multiples of 128, K multiple of 64 (checked by the host wrapper).
#include "b2_gemm_body.cuh"

namespace {

__global__ void __launch_bounds__(GEMM_THREADS, 1)
b2_k_gemm_allreduce(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b,
                    const B2DevComm c, const GemmArgs g) {
  gemm_body<EPI_ALLREDUCE>(tma_a, tma_b, c, g);
}

}  // namespace

// out (M x N, bf16) = sum over ranks of A (M x K, bf16, row-major) @ B^T (B: N x K, bf16, row-major).
// Multi-rank calls stage the bf16 partial tiles in the communicator's multicast-bound staging
// segment (M*N*2 bytes per parity; grown by the Python layer like for any other collective).
extern "C" int b2_gemm_allreduce(B2Comm* c, const void* A, const void* B, void* out, int M, int N, int K,
                                 cudaStream_t stream) {
  if (!gemm_shape_ok("gemm_allreduce", M, N, K)) return B2_ERR_BAD_ARG;
  const GemmArgs g = gemm_args(M, N, K, out, c->dev.size > 1 ? 1 : 0);
  if (g.fused && c->dev.stage_mc == nullptr) {
    b2_set_error("gemm_allreduce: multi-rank call needs a multicast-bound staging segment (NVLS)");
    return B2_ERR_BAD_ARG;
  }
  static bool attr_set = false;
  return gemm_launch(b2_k_gemm_allreduce, attr_set, c, A, B, g, "gemm_allreduce", stream);
}

