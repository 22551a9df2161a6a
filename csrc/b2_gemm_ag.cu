// mpi4jax_b200 -- sequence-parallel column-parallel linear layer: allgather + GEMM in ONE kernel.
//
//   out_r (P m x N_r) = allgather_q(X_q (m x K, bf16)) @ W_r^T (W_r: N_r x K, bf16)
//
// The producer, the wgmma mainloop and the epilogue are those of the stand-alone GEMM of b2_k_gemm_allreduce
// (b2_gemm_body.cuh, EPI_ALLGATHER).  A is the gathered (P m, K) matrix, built in this launch's half of every
// rank's staging while the GEMM runs: warps 1-3 of the producer warpgroup, idle in the other two kernels, push
// this rank's shard chunk by chunk with plain 16-byte stores into rows [rank m, (rank + 1) m) of every rank's
// gathered matrix (its own included) and publish each chunk in an arrival word of the destination's control
// segment.  Before the TMA loads of a tile, the producer thread waits for every chunk under the tile's 128
// rows, so TMA only ever reads local memory.  Each rank walks the tile rows from its own shard on, so its
// first tiles wait only on its own pushes.  No multicast: it runs wherever the staging segment is
// peer-mapped, two ranks on one GPU included.  NVLink bytes per rank: (P-1) m K 2 out, (P-1) m K 2 in.
#include "b2_gemm_body.cuh"

namespace {

__global__ void __launch_bounds__(GEMM_THREADS, 1)
b2_k_gemm_allgather(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b,
                    const B2DevComm c, const __grid_constant__ GemmArgsAg g) {
  gemm_body<EPI_ALLGATHER>(tma_a, tma_b, c, g);
}

}  // namespace

// out (P m x N, bf16) = the rows of every rank's x_local (m x K, bf16, row-major), in rank order, @ w^T
// (w: N x K, bf16, row-major).  m and K must be the same on every rank, N may differ.  Multi-rank calls
// gather into the staging segment (P m K 2 bytes per parity, grown by the Python layer to the same size on
// every rank); one rank is the stand-alone GEMM of b2_gemm_allreduce.
extern "C" int b2_gemm_allgather(B2Comm* c, const void* x_local, const void* w, void* out, int m, int N, int K,
                                 cudaStream_t stream) {
  const int P = c->dev.size;
  if (m <= 0 || (long long)P * m > 0x7fffffff || !gemm_shape_ok("gemm_allgather", P * m, N, K))
    return B2_ERR_BAD_ARG;
  if (P == 1) return b2_gemm_allreduce(c, x_local, w, out, m, N, K, stream);
  const size_t row_bytes = (size_t)K * 2, need = (size_t)P * m * row_bytes + 4096;
  if (c->stage == nullptr || need > c->dev.stage_half) {
    b2_set_error("gemm_allgather: staging too small (need %zu bytes, have %zu)", need,
                 c->stage ? c->dev.stage_half : (size_t)0);
    return B2_ERR_BAD_ARG;
  }
  GemmArgsAg g;
  static_cast<GemmArgs&>(g) = gemm_args(P * m, N, K, out, 0);
  g.x_local = (const __nv_bfloat16*)x_local;
  g.m = m;
  // at most B2_AG_CHUNKS chunks per shard, each at least 16 KiB: every CTA of a wide grid gets a chunk to
  // push, and a tile waits on few arrival words
  const size_t min_rows = (16384 + row_bytes - 1) / row_bytes;
  size_t rows = ((size_t)m + B2_AG_CHUNKS - 1) / B2_AG_CHUNKS;
  if (rows < min_rows) rows = min_rows;
  g.chunk_rows = rows < (size_t)m ? (int)rows : m;
  if (((uintptr_t)x_local & 15) != 0) {
    b2_set_error("gemm_allgather: x must be 16-byte aligned");
    return B2_ERR_BAD_ARG;
  }
  // A: the gathered matrix in staging half 0 (ta) and 1 (g.tma_a1); the kernel picks one by the ticket's
  // parity, which the host cannot know while a CUDA graph is captured
  CUtensorMap ta, tb;
  const char* gathered = c->dev.stage[c->dev.rank];
  if (b2_tensor_map_2d_bf16(&ta, gathered, (unsigned long long)g.M, (unsigned long long)K, BM, BK) ||
      b2_tensor_map_2d_bf16(&g.tma_a1, gathered + c->dev.stage_half, (unsigned long long)g.M, (unsigned long long)K,
                            BM, BK) ||
      b2_tensor_map_2d_bf16(&tb, w, (unsigned long long)N, (unsigned long long)K, BN, BK))
    return B2_ERR_BAD_ARG;
  static bool attr_set = false;
  size_t smem;
  int grid;
  if (int rc = gemm_geometry(b2_k_gemm_allgather, attr_set, c, g, "gemm_allgather", smem, grid)) return rc;
  b2_k_gemm_allgather<<<grid, GEMM_THREADS, smem, stream>>>(ta, tb, c->dev, g);
  return b2_launched(c, "gemm_allgather");
}
