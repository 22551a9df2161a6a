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
#include <cstdio>
#include <cstring>

#include <cuda.h>
#include <cuda_bf16.h>

#include "b2_device.cuh"
#include "b2_runtime.h"
#include "b2_gemm_raster.h"

extern "C" void b2_set_error(const char* fmt, ...);
extern "C" void b2_count_launch(B2Comm* c);
extern "C" int b2_tensor_map_2d_bf16(CUtensorMap* out, const void* ptr, unsigned long long rows,
                                     unsigned long long cols, unsigned box_rows, unsigned box_cols);

namespace {

constexpr int BM = 128, BN = 128, BK = 64, STAGES = 6, WGMMA_K = 16;
constexpr int GEMM_THREADS = 384, EPI_THREADS = 256;
constexpr uint32_t A_STAGE_BYTES = BM * BK * 2, B_STAGE_BYTES = BN * BK * 2;

struct GemmArgs {
  int M, N, K;
  __nv_bfloat16* out;
  int fused;           // > 1 rank: per-tile NVLS allreduce through the staging segment
  int raster;          // tile order: 0 = row-major, G > 0 = bands of G tile rows (b2_gemm_raster.h)
};

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t cnt) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(cnt));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t tx) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(tx) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n.reg .pred p;\nWAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra WAIT_DONE;\nbra WAIT_LOOP;\nWAIT_DONE:\n}" ::"r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0,
                                            int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"((uint64_t)map), "r"(bar), "r"(c0), "r"(c1) : "memory");
}
// K-major operand tile in shared memory, 128-byte swizzle (GMMA matrix descriptor):
// start address >> 4 at [0,14), leading byte offset (unused for swizzled K-major, 1) at [16,30),
// stride byte offset = 8 rows x 128 B = 1024 B >> 4 at [32,46), layout SWIZZLE_128B = 1 at [62,64)
__device__ __forceinline__ uint64_t gmma_desc(uint32_t smem_addr) {
  uint64_t d = (uint64_t)((smem_addr & 0x3FFFFu) >> 4);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024u >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}
// d (64 x 128 fp32, this warpgroup's accumulator fragment) (+)= A (64 x 16) @ B^T (B: 128 x 16)
__device__ __forceinline__ void wgmma_bf16(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accum) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(accum));
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from touching the accumulator registers across a wgmma_wait
__device__ __forceinline__ void fence_accumulator(float (&d)[64]) {
#pragma unroll
  for (int i = 0; i < 64; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
__device__ __forceinline__ uint4 mc_ld_reduce_bf16(const void* mc) {
  uint4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.bf16x2 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(mc) : "memory");
  return v;
}
__device__ __forceinline__ void mc_st16(void* mc, uint4 v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc), "r"(v.x), "r"(v.y),
               "r"(v.z), "r"(v.w) : "memory");
}
// cross-GPU barrier executed by the 256 consumer threads only (named barrier 1), CTA b <-> CTA b
__device__ __forceinline__ void epi_barrier_all(const B2DevComm& c, unsigned e, int et) {
  asm volatile("bar.sync 1, 256;" ::: "memory");
  if (et < c.size) {
    unsigned* remote = (unsigned*)(c.heap[et] + c.lay.flags_off) + (size_t)blockIdx.x * B2_MAX_RANKS + c.rank;
    b2_st_release_sys(remote, e);
    const unsigned* local =
        (const unsigned*)(c.heap[c.rank] + c.lay.flags_off) + (size_t)blockIdx.x * B2_MAX_RANKS + et;
    b2_wait_ge(c, local, e, B2_OPC_ALLREDUCE, et);
  }
  asm volatile("bar.sync 1, 256;" ::: "memory");
}

__global__ void __launch_bounds__(GEMM_THREADS, 1)
b2_k_gemm_allreduce(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b,
                    const B2DevComm c, const GemmArgs g) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ uint64_t full_bar[STAGES], empty_bar[STAGES];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2;
  const uint32_t smem_base = ((uint32_t)__cvta_generic_to_shared(smem_raw) + 1023u) & ~1023u;
  const uint32_t smem_a = smem_base, smem_b = smem_base + STAGES * A_STAGE_BYTES;
  auto bar = [](uint64_t* p) { return (uint32_t)__cvta_generic_to_shared(p); };

  unsigned ticket = 0, e = 0;
  if (g.fused) {
    ticket = b2_ticket_read(c.ticket);
    e = b2_ld_volatile(c.epoch + blockIdx.x);
  }
  const size_t par = (size_t)(ticket & 1u) * c.stage_half;

  if (threadIdx.x == 0) {
    // full: the producer's expect_tx arrival + the TMA bytes; empty: one arrival per consumer warpgroup
    for (int s = 0; s < STAGES; ++s) { mbar_init(bar(&full_bar[s]), 1); mbar_init(bar(&empty_bar[s]), 2); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int num_n = g.N / BN, tiles = (g.M / BM) * num_n, num_kb = g.K / BK;

  if (wg == 0) {
    if (threadIdx.x == 0) {
      // ===== TMA producer =====
      uint32_t stage = 0, phase = 0;
      for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        int m_blk, n_blk;
        b2_gemm_tile_coords(tile, g.M / BM, num_n, g.raster, m_blk, n_blk);
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(bar(&empty_bar[stage]), phase ^ 1u);
          mbar_expect_tx(bar(&full_bar[stage]), A_STAGE_BYTES + B_STAGE_BYTES);
          tma_load_2d(smem_a + stage * A_STAGE_BYTES, &tma_a, bar(&full_bar[stage]), kb * BK, m_blk * BM);
          tma_load_2d(smem_b + stage * B_STAGE_BYTES, &tma_b, bar(&full_bar[stage]), kb * BK, n_blk * BN);
          if (++stage == STAGES) { stage = 0; phase ^= 1u; }
        }
      }
    }
  } else {
    // ===== consumers: wgmma -> bf16 -> (staging + per-tile NVLS allreduce | output) =====
    const int cw = wg - 1;                                      // rows cw * 64 .. +64 of the tile
    const int wq = warp & 3;                                    // 16-row slice of the warpgroup's rows
    const int et = threadIdx.x - 128;                           // 0..255 within the consumer group
    const bool leader = (threadIdx.x & 127) == 0;
    __nv_bfloat16* stage_local = (__nv_bfloat16*)(c.stage[c.rank] + par);
    __nv_bfloat16* stage_mc = (__nv_bfloat16*)(c.stage_mc + par);
    uint32_t stage = 0, phase = 0;
    float acc[64];
    constexpr int GROUP = 4;                                    // tiles per collective round
    int pend[GROUP], np = 0;
    for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
      int m_blk, n_blk;
      b2_gemm_tile_coords(tile, g.M / BM, num_n, g.raster, m_blk, n_blk);
      uint32_t prev = 0;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(bar(&full_bar[stage]), phase);                // TMA landed this stage
        const uint64_t adesc = gmma_desc(smem_a + stage * A_STAGE_BYTES + cw * 64 * 128);
        const uint64_t bdesc = gmma_desc(smem_b + stage * B_STAGE_BYTES);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / WGMMA_K; ++k)                  // +32 B per WGMMA_K inside the swizzle atom
          wgmma_bf16(acc, adesc + (uint64_t)(k * 2), bdesc + (uint64_t)(k * 2), (kb | k) != 0);
        wgmma_commit();
        wgmma_wait<1>();                                        // the previous stage's MMAs have retired
        if (kb > 0 && leader) mbar_arrive(bar(&empty_bar[prev]));
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1u; }
      }
      wgmma_wait<0>();
      fence_accumulator(acc);
      if (leader) mbar_arrive(bar(&empty_bar[prev]));           // the producer refills while we store
      // accumulator fragment: acc[4j + {0,1}] = row r, columns 8j + 2(lane % 4) + {0,1}; acc[4j + {2,3}] = row r + 8
      const size_t row = (size_t)m_blk * BM + cw * 64 + wq * 16 + (lane >> 2);
      __nv_bfloat16* dst = (g.fused ? stage_local : g.out) + row * g.N + (size_t)n_blk * BN + 2 * (lane & 3);
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        *reinterpret_cast<__nv_bfloat162*>(dst + 8 * j) = __floats2bfloat162_rn(acc[4 * j], acc[4 * j + 1]);
        *reinterpret_cast<__nv_bfloat162*>(dst + 8 * (size_t)g.N + 8 * j) =
            __floats2bfloat162_rn(acc[4 * j + 2], acc[4 * j + 3]);
      }
      if (g.fused) {
        // --- all-reduce finished tiles across the ranks.  GROUP tiles share one pair of cross-GPU
        // barriers; all loads of a batch are issued before the first dependent store so the
        // NVLink / L2 round trips overlap instead of adding up.
        pend[np++] = tile;
        const bool last = tile + (int)gridDim.x >= tiles;
        if (np == GROUP || last) {
          epi_barrier_all(c, ++e, et);                          // every rank staged these partial tiles
          const int per = (BM + c.size - 1) / c.size;           // my row-slice of every tile
          const int r0 = per * c.rank < BM ? per * c.rank : BM, r1 = r0 + per < BM ? r0 + per : BM;
          const int slice_vec = (r1 - r0) * (BN / 8), nred = np * slice_vec;
          for (int base = et; base < nred; base += EPI_THREADS * 4) {
            uint4 v[4];
            size_t offs[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
              const int i = base + u * EPI_THREADS;
              if (i < nred) {
                const int slot = i / slice_vec, w = i - slot * slice_vec;
                const int tl = pend[slot], r = r0 + w / (BN / 8), v8 = w % (BN / 8);
                int tm, tn;
                b2_gemm_tile_coords(tl, g.M / BM, num_n, g.raster, tm, tn);
                offs[u] = ((size_t)tm * BM + r) * g.N + (size_t)tn * BN + v8 * 8;
                v[u] = mc_ld_reduce_bf16(stage_mc + offs[u]);   // fp32 sum inside the NVSwitch
              }
            }
#pragma unroll
            for (int u = 0; u < 4; ++u)
              if (base + u * EPI_THREADS < nred) mc_st16(stage_mc + offs[u], v[u]);   // broadcast to every rank
          }
          epi_barrier_all(c, ++e, et);                          // all slices of these tiles have landed
          const int ncp = np * BM * (BN / 8);
          for (int base = et; base < ncp; base += EPI_THREADS * 8) {
            uint4 v[8];
            size_t offs[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) {
              const int i = base + u * EPI_THREADS;
              if (i < ncp) {
                const int slot = i / (BM * (BN / 8)), w = i - slot * (BM * (BN / 8));
                const int tl = pend[slot], r = w / (BN / 8), v8 = w % (BN / 8);
                int tm, tn;
                b2_gemm_tile_coords(tl, g.M / BM, num_n, g.raster, tm, tn);
                offs[u] = ((size_t)tm * BM + r) * g.N + (size_t)tn * BN + v8 * 8;
                v[u] = b2_ld_peer16(stage_local + offs[u]);
              }
            }
#pragma unroll
            for (int u = 0; u < 8; ++u)
              if (base + u * EPI_THREADS < ncp) b2_st16(g.out + offs[u], v[u]);
          }
          np = 0;
        }
      }
    }
    if (g.fused && et == 0) b2_st_volatile(c.epoch + blockIdx.x, e);
  }

  __syncthreads();
  if (g.fused) b2_finish_bump(c.ticket, c.ticket + 1, 1u, gridDim.x);
}

}  // namespace

// out (M x N, bf16) = sum over ranks of A (M x K, bf16, row-major) @ B^T (B: N x K, bf16, row-major).
// Multi-rank calls stage the bf16 partial tiles in the communicator's multicast-bound staging
// segment (M*N*2 bytes per parity; grown by the Python layer like for any other collective).
extern "C" int b2_gemm_allreduce(B2Comm* c, const void* A, const void* B, void* out, int M, int N, int K,
                                 cudaStream_t stream) {
  if (M <= 0 || N <= 0 || K <= 0 || M % BM || N % BN || K % BK) {
    b2_set_error("gemm_allreduce: need M %% %d == 0, N %% %d == 0, K %% %d == 0 (got %d, %d, %d)", BM, BN,
                 BK, M, N, K);
    return B2_ERR_BAD_ARG;
  }
  GemmArgs g;
  memset(&g, 0, sizeof g);
  g.M = M; g.N = N; g.K = K;
  g.out = (__nv_bfloat16*)out;
  g.fused = (c->dev.size > 1) ? 1 : 0;
  // banded tile order for the stand-alone GEMM; the fused epilogue recomputes a tile's coordinates per
  // 16-byte vector (integer divisions in front of every multimem load), so it keeps the cheaper
  // row-major formula
  g.raster = c->gemm_raster >= 0 ? c->gemm_raster : (g.fused ? 0 : B2_GEMM_RASTER_GROUP);
  if (g.fused) {
    if (c->dev.stage_mc == nullptr) {
      b2_set_error("gemm_allreduce: multi-rank call needs a multicast-bound staging segment (NVLS)");
      return B2_ERR_BAD_ARG;
    }
    if ((size_t)M * N * 2 + 4096 > c->dev.stage_half) {
      b2_set_error("gemm_allreduce: staging too small (need %zu bytes, have %zu)", (size_t)M * N * 2 + 4096,
                   c->dev.stage_half);
      return B2_ERR_BAD_ARG;
    }
  }
  CUtensorMap ta, tb;
  if (b2_tensor_map_2d_bf16(&ta, A, (unsigned long long)M, (unsigned long long)K, BM, BK) ||
      b2_tensor_map_2d_bf16(&tb, B, (unsigned long long)N, (unsigned long long)K, BN, BK))
    return B2_ERR_BAD_ARG;
  const size_t smem = (size_t)STAGES * (A_STAGE_BYTES + B_STAGE_BYTES) + 1024;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(b2_k_gemm_allreduce, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) {
      b2_set_error("gemm_allreduce: cannot reserve %zu bytes of shared memory: %s", smem,
                   cudaGetErrorString(e));
      return 1000 + (int)e;
    }
    attr_set = true;
  }
  const int tiles = (M / BM) * (N / BN);
  int grid = tiles < c->sm_count ? tiles : c->sm_count;
  if (grid > B2_MAX_BLOCKS) grid = B2_MAX_BLOCKS;
  b2_k_gemm_allreduce<<<grid, GEMM_THREADS, smem, stream>>>(ta, tb, c->dev, g);
  b2_count_launch(c);
  cudaError_t err = cudaGetLastError();
  if (err != cudaSuccess) {
    b2_set_error("gemm_allreduce: kernel launch failed: %s", cudaGetErrorString(err));
    return 1000 + (int)err;
  }
  return 0;
}
