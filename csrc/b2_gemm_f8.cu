// mpi4jax_b200 -- scaled float8 linear layers: the e4m3 twins of the three GEMM kernels.
//
//   partial_r (i, j) = rn_bf16( S_r[i, j] * (sx_r[i] * sw_r[j]) ),  S_r = X_r (e4m3) @ W_r^T (e4m3), fp32 accumulators
//
// Producer, ring, tile order and epilogues are those of the bf16 kernels (b2_gemm_body.cuh with T = e4m3): a
// 128 x 128 e4m3 tile is 16 KiB like a 128 x 64 bf16 one, so only the TMA element type, the k-block (128
// elements) and the instruction (`wgmma.mma_async.m64n128k32.f32.e4m3.e4m3`) change.  Before its bf16
// conversion every accumulator is multiplied by its row and column scale, read through device pointers, so
// the epilogues see bf16 partial tiles as before: the allreduce sums them in the NVSwitch, the reduce-scatter
// folds them in fp32, the allgather kernel stores them.  The allgather kernel gathers the row scales with the
// rows (ag_push); its gathered matrix is P m K bytes, half the bf16 kernel's NVLink traffic.
//
// The three kernels share this translation unit; the bf16 kernels keep theirs, and their SASS is unchanged.
#include "b2_gemm_body.cuh"

namespace {

using E4M3 = __nv_fp8_e4m3;
constexpr int BK8 = GemmElem<E4M3>::BK;

__global__ void __launch_bounds__(GEMM_THREADS, 1)
b2_k_gemm_allreduce_f8(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b,
                       const B2DevComm c, const __grid_constant__ GemmArgsF8 g) {
  gemm_body<EPI_ALLREDUCE, E4M3>(tma_a, tma_b, c, g);
}

__global__ void __launch_bounds__(GEMM_THREADS, 1)
b2_k_gemm_reduce_scatter_f8(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b,
                            const B2DevComm c, const __grid_constant__ GemmArgsF8 g) {
  gemm_body<EPI_REDUCE_SCATTER, E4M3>(tma_a, tma_b, c, g);
}

__global__ void __launch_bounds__(GEMM_THREADS, 1)
b2_k_gemm_allgather_f8(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b,
                       const B2DevComm c, const __grid_constant__ GemmArgsAgF8 g) {
  gemm_body<EPI_ALLGATHER, E4M3>(tma_a, tma_b, c, g);
}

GemmScales scales(const float* sx, int sx_inc, const float* sw, int sw_inc) {
  GemmScales s;
  s.sx = sx;
  s.sw = sw;
  s.sx_inc = sx_inc;
  s.sw_inc = sw_inc;
  return s;
}

bool scales_ok(const char* what, const float* sx, int sx_inc, const float* sw, int sw_inc) {
  if (sx == nullptr || sw == nullptr || (sx_inc != 0 && sx_inc != 1) || (sw_inc != 0 && sw_inc != 1)) {
    b2_set_error("%s: need scale pointers with an increment of 0 or 1 (got %d, %d)", what, sx_inc, sw_inc);
    return false;
  }
  return true;
}

}  // namespace

// out (M x N, bf16) = sum over ranks of the scaled partials of A (M x K, e4m3, row-major) @ B^T (B: N x K, e4m3,
// row-major); sx has M (or 1) floats, sw N (or 1).  Multi-rank calls need NVLS, as b2_gemm_allreduce does.
extern "C" int b2_gemm_allreduce_f8(B2Comm* c, const void* A, const void* B, void* out, int M, int N, int K,
                                    const float* sx, int sx_inc, const float* sw, int sw_inc, cudaStream_t stream) {
  if (!gemm_shape_ok("gemm_allreduce_f8", M, N, K, BK8) || !scales_ok("gemm_allreduce_f8", sx, sx_inc, sw, sw_inc))
    return B2_ERR_BAD_ARG;
  GemmArgsF8 g;
  static_cast<GemmArgs&>(g) = gemm_args(M, N, K, out, c->dev.size > 1 ? 1 : 0);
  g.s = scales(sx, sx_inc, sw, sw_inc);
  if (g.fused && c->dev.stage_mc == nullptr) {
    b2_set_error("gemm_allreduce_f8: multi-rank call needs a multicast-bound staging segment (NVLS)");
    return B2_ERR_BAD_ARG;
  }
  static bool attr_set = false;
  return gemm_launch<E4M3>(b2_k_gemm_allreduce_f8, attr_set, c, A, B, g, "gemm_allreduce_f8", stream);
}

// out ((M / P) x N, bf16) = rows [rank M / P, (rank + 1) M / P) of the sum over ranks of the scaled partials;
// sx indexes all M rows of A.  One rank is the stand-alone float8 GEMM.
extern "C" int b2_gemm_reduce_scatter_f8(B2Comm* c, const void* A, const void* B, void* out, int M, int N, int K,
                                         const float* sx, int sx_inc, const float* sw, int sw_inc,
                                         cudaStream_t stream) {
  if (!gemm_shape_ok("gemm_reduce_scatter_f8", M, N, K, BK8) ||
      !scales_ok("gemm_reduce_scatter_f8", sx, sx_inc, sw, sw_inc))
    return B2_ERR_BAD_ARG;
  if (M % c->dev.size) {
    b2_set_error("gemm_reduce_scatter_f8: M = %d is not divisible by the %d ranks", M, c->dev.size);
    return B2_ERR_BAD_ARG;
  }
  if (c->dev.size == 1) return b2_gemm_allreduce_f8(c, A, B, out, M, N, K, sx, sx_inc, sw, sw_inc, stream);
  GemmArgsF8 g;
  static_cast<GemmArgs&>(g) = gemm_args(M, N, K, out, 1);
  g.s = scales(sx, sx_inc, sw, sw_inc);
  static bool attr_set = false;
  return gemm_launch<E4M3>(b2_k_gemm_reduce_scatter_f8, attr_set, c, A, B, g, "gemm_reduce_scatter_f8", stream);
}

// out (P m x N, bf16): row q m + i = rn_bf16(S * (sx_q[i] * sw[j])), S from the rows of every rank's x_local
// (m x K, e4m3) in rank order and this rank's w (N x K, e4m3).  Each rank's row scales travel with its rows.
// Staging per parity: the gathered (P m, K) bytes, then P m floats of row scales at a 16-byte aligned offset.
extern "C" int b2_gemm_allgather_f8(B2Comm* c, const void* x_local, const void* w, void* out, int m, int N, int K,
                                    const float* sx, int sx_inc, const float* sw, int sw_inc, cudaStream_t stream) {
  const int P = c->dev.size;
  if (m <= 0 || (long long)P * m > 0x7fffffff || !gemm_shape_ok("gemm_allgather_f8", P * m, N, K, BK8) ||
      !scales_ok("gemm_allgather_f8", sx, sx_inc, sw, sw_inc))
    return B2_ERR_BAD_ARG;
  if (P == 1) return b2_gemm_allreduce_f8(c, x_local, w, out, m, N, K, sx, sx_inc, sw, sw_inc, stream);
  const size_t row_bytes = (size_t)K, sx_off = ((size_t)P * m * row_bytes + 15) & ~(size_t)15;
  const size_t need = sx_off + (size_t)P * m * sizeof(float) + 4096;
  if (c->stage == nullptr || need > c->dev.stage_half) {
    b2_set_error("gemm_allgather_f8: staging too small (need %zu bytes, have %zu)", need,
                 c->stage ? c->dev.stage_half : (size_t)0);
    return B2_ERR_BAD_ARG;
  }
  GemmArgsAgF8 g;
  static_cast<GemmArgs&>(g) = gemm_args(P * m, N, K, out, 0);
  g.x_local = (const __nv_bfloat16*)x_local;
  g.m = m;
  g.s = scales(sx, sx_inc, sw, sw_inc);
  g.sx_off = sx_off;
  // the chunk rule of b2_gemm_allgather, with one byte per element
  const size_t min_rows = (16384 + row_bytes - 1) / row_bytes;
  size_t rows = ((size_t)m + B2_AG_CHUNKS - 1) / B2_AG_CHUNKS;
  if (rows < min_rows) rows = min_rows;
  g.chunk_rows = rows < (size_t)m ? (int)rows : m;
  if (((uintptr_t)x_local & 15) != 0) {
    b2_set_error("gemm_allgather_f8: x must be 16-byte aligned");
    return B2_ERR_BAD_ARG;
  }
  CUtensorMap ta, tb;
  const char* gathered = c->dev.stage[c->dev.rank];
  if (gemm_tensor_map<E4M3>(&ta, gathered, g.M, K) ||
      gemm_tensor_map<E4M3>(&g.tma_a1, gathered + c->dev.stage_half, g.M, K) || gemm_tensor_map<E4M3>(&tb, w, N, K))
    return B2_ERR_BAD_ARG;
  static bool attr_set = false;
  size_t smem;
  int grid;
  if (int rc = gemm_geometry(b2_k_gemm_allgather_f8, attr_set, c, g, "gemm_allgather_f8", smem, grid)) return rc;
  b2_k_gemm_allgather_f8<<<grid, GEMM_THREADS, smem, stream>>>(ta, tb, c->dev, g);
  return b2_launched(c, "gemm_allgather_f8");
}
