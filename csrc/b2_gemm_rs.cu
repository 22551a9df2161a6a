// mpi4jax_b200 -- sequence-parallel row-parallel linear layer: GEMM + reduce-scatter in ONE kernel.
//
//   out_r = rows [r M/P, (r+1) M/P) of  sum over ranks q of  X_q (M x K_q, bf16) @ W_q^T (W_q: N x K_q, bf16)
//
// The producer, the wgmma mainloop and the tile order are those of b2_k_gemm_allreduce (b2_gemm_body.cuh).
// Only the epilogue differs: per group of up to 4 finished tiles every rank stages its bf16 partial tiles,
// then (between two block-paired barriers) pulls its 1/P row-slice of each tile from every rank's staging,
// folds it in rank order in fp32, rounds once and stores each 16-byte result into the staging of the rank
// whose shard holds that row; after the second barrier each rank copies its own rows to the output.  No
// NVSwitch multicast: it runs wherever the staging segment is peer-mapped, two ranks on one GPU included.
// NVLink bytes per rank: (P-1)/P * M*N*2 pulled (the reduce-scatter lower bound), (P-1)/P^2 * M*N*2 stored.
#include "b2_gemm_body.cuh"

namespace {

__global__ void __launch_bounds__(GEMM_THREADS, 1)
b2_k_gemm_reduce_scatter(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b,
                         const B2DevComm c, const GemmArgs g) {
  gemm_body<EPI_REDUCE_SCATTER>(tma_a, tma_b, c, g);
}

}  // namespace

// out ((M / P) x N, bf16) = rows [rank * M / P, (rank + 1) * M / P) of the sum over the P ranks of A @ B^T.
// Multi-rank calls stage the partial tiles in the staging segment (M*N*2 bytes per parity, no multicast
// needed); one rank is the stand-alone GEMM of b2_gemm_allreduce.
extern "C" int b2_gemm_reduce_scatter(B2Comm* c, const void* A, const void* B, void* out, int M, int N, int K,
                                      cudaStream_t stream) {
  if (!gemm_shape_ok("gemm_reduce_scatter", M, N, K)) return B2_ERR_BAD_ARG;
  if (M % c->dev.size) {
    b2_set_error("gemm_reduce_scatter: M = %d is not divisible by the %d ranks", M, c->dev.size);
    return B2_ERR_BAD_ARG;
  }
  if (c->dev.size == 1) return b2_gemm_allreduce(c, A, B, out, M, N, K, stream);
  static bool attr_set = false;
  return gemm_launch(b2_k_gemm_reduce_scatter, attr_set, c, A, B, gemm_args(M, N, K, out, 1), "gemm_reduce_scatter",
                    stream);
}
