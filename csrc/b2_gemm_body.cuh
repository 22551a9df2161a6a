// mpi4jax_b200 -- the persistent wgmma GEMM that the linear-layer kernels share: TMA producer,
// 6-stage mbarrier ring, wgmma mainloop, tile order and the per-group epilogues.  Each kernel lives in its
// own translation unit (b2_gemm.cu: GEMM + allreduce, b2_gemm_rs.cu: GEMM + reduce-scatter, b2_gemm_ag.cu:
// allgather + GEMM; b2_gemm_f8.cu: the three float8 twins); in one unit together ptxas schedules the allreduce
// kernel differently.
#pragma once

#include <cstring>
#include <type_traits>

#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp8.h>

#include "b2_device.cuh"
#include "b2_runtime.h"
#include "b2_gemm_raster.h"

namespace {

constexpr int BM = 128, BN = 128, BK = 64, STAGES = 6, WGMMA_K = 16;
constexpr int GEMM_THREADS = 384, EPI_THREADS = 256;
constexpr int RS_BATCH = 8;          // peer loads a reduce-scatter thread issues before it folds them
constexpr uint32_t A_STAGE_BYTES = BM * BK * 2, B_STAGE_BYTES = BN * BK * 2;

struct GemmArgs {
  int M, N, K;
  __nv_bfloat16* out;
  int fused;           // > 1 rank: per-tile NVLS allreduce through the staging segment
  int raster;          // tile order: 0 = row-major, G > 0 = bands of G tile rows (b2_gemm_raster.h)
};

// allgather + GEMM: A is the (M = P m, K) gathered matrix in the staging, built while the GEMM runs.  Its
// kernel passes these, and gemm_body reaches them by a downcast of `g`: a larger GemmArgs, or a gemm_body
// with more parameters, changes the register allocation of the other two kernels.
struct GemmArgsAg : GemmArgs {
  CUtensorMap tma_a1;             // A in staging half 1 (the kernel's tma_a: half 0)
  const __nv_bfloat16* x_local;   // this rank's (m, K) shard (float8 kernel: one byte per element)
  int m;                          // rows per rank
  int chunk_rows;                 // rows per pushed chunk; ceil(m / chunk_rows) <= B2_AG_CHUNKS
};

// Scaled float8 operands: partial (i, j) = rn_bf16(S[i, j] * (sx[i * sx_inc] * sw[j * sw_inc])).  The scales
// are read through these pointers at every launch (a graph replay sees scales updated in place); an increment
// of 0 is one scale for the whole tensor, 1 one per row of A / column of the output.
struct GemmScales {
  const float* sx;
  const float* sw;
  int sx_inc, sw_inc;
};
// The float8 kernels' arguments, reached like GemmArgsAg by a downcast of `g`.  Allgather + GEMM: the push
// warps copy this rank's row scales (sx, sx_inc) as m floats per shard into a region `sx_off` bytes into the
// staging half, after the gathered (P m, K) matrix; the epilogue reads them there with an increment of 1.
struct GemmArgsF8 : GemmArgs {
  GemmScales s;
};
struct GemmArgsAgF8 : GemmArgsAg {
  GemmScales s;
  size_t sx_off;
};

// Operand element types of the mainloop.  A k-block is one 128-byte row of the swizzle atom in either
// type: BK = 64 bf16 or 128 e4m3 elements, so the stage sizes, the GMMA descriptors and the +32 B per wgmma
// k-step are the same, and one wgmma takes 16 or 32 elements of K.
template <typename T> struct GemmElem;
template <> struct GemmElem<__nv_bfloat16> { static constexpr int BK = 64, WGMMA_K = 16; };
template <> struct GemmElem<__nv_fp8_e4m3> { static constexpr int BK = 128, WGMMA_K = 32; };

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
// the same for e4m3 operands, 32 elements of K per instruction (float8 wgmma has no transpose immediates)
__device__ __forceinline__ void wgmma_e4m3(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accum) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k32.f32.e4m3.e4m3 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n}"
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
// cross-GPU barrier executed by the 256 consumer threads only (named barrier 1), CTA b <-> CTA b;
// `opcode` names the collective in the watchdog's abort line
__device__ __forceinline__ void epi_barrier_all(const B2DevComm& c, unsigned e, int et, int opcode) {
  asm volatile("bar.sync 1, 256;" ::: "memory");
  if (et < c.size) {
    unsigned* remote = (unsigned*)(c.heap[et] + c.lay.flags_off) + (size_t)blockIdx.x * B2_MAX_RANKS + c.rank;
    b2_st_release_sys(remote, e);
    const unsigned* local =
        (const unsigned*)(c.heap[c.rank] + c.lay.flags_off) + (size_t)blockIdx.x * B2_MAX_RANKS + et;
    b2_wait_ge(c, local, e, opcode, et);
  }
  asm volatile("bar.sync 1, 256;" ::: "memory");
}

// ---------------------------------------------------------------------------
// allgather + GEMM (EPI_ALLGATHER): every rank pushes its (m, K) shard, chunk by chunk, into rows
// [rank m, (rank + 1) m) of the gathered matrix in every rank's staging half, and publishes each chunk in an
// arrival word of the destination (B2_AG_FLAGS_REL); the producer waits for the chunks under a tile's rows.
// ---------------------------------------------------------------------------
__device__ __forceinline__ unsigned* ag_arrivals(const B2DevComm& c, int r) {
  return (unsigned*)(c.heap[r] + c.lay.flags_off + B2_AG_FLAGS_REL);
}

// Warps 1-3 of warpgroup 0 (96 threads): chunk j goes from CTA j % gridDim.x, to this rank first, then to
// rank - 1, rank - 2, ..., so rank r receives shard r + 1 first.  After each (chunk, destination) the pushing
// warps synchronise and one thread publishes the chunk with `val`.  Never waits on anything.  Float8: the
// chunk's row scales go with its rows, to gathered rows [rank m + r0, rank m + r1) of the scale region, before
// the same barrier and arrival word.
template <typename T>
__device__ __forceinline__ void ag_push(const B2DevComm& c, const GemmArgsAg& a, size_t par, unsigned val) {
  const int t = threadIdx.x - 32;
  const size_t row_bytes = (size_t)a.K * sizeof(T);
  const int nch = (a.m + a.chunk_rows - 1) / a.chunk_rows;
  for (int j = blockIdx.x; j < nch; j += gridDim.x) {
    const int r0 = j * a.chunk_rows, r1 = r0 + a.chunk_rows < a.m ? r0 + a.chunk_rows : a.m;
    const size_t nvec = (size_t)(r1 - r0) * row_bytes / 16;
    const char* src = (const char*)a.x_local + (size_t)r0 * row_bytes;
    const size_t off = par + ((size_t)c.rank * a.m + r0) * row_bytes;
    for (int s = 0; s < c.size; ++s) {
      const int d = (c.rank - s + c.size) % c.size;
      char* dst = c.stage[d] + off;
      for (size_t i = t; i < nvec; i += 96 * 4) {
        uint4 v[4];
#pragma unroll
        for (int u = 0; u < 4; ++u)
          if (i + u * 96 < nvec) v[u] = b2_ld_stream16(src + ((i + u * 96) << 4));
#pragma unroll
        for (int u = 0; u < 4; ++u)
          if (i + u * 96 < nvec) b2_st16(dst + ((i + u * 96) << 4), v[u]);
      }
      if constexpr (!std::is_same_v<T, __nv_bfloat16>) {
        const GemmArgsAgF8& f = static_cast<const GemmArgsAgF8&>(a);
        float* sdst = (float*)(c.stage[d] + par + f.sx_off) + (size_t)c.rank * a.m;
        for (int i = r0 + t; i < r1; i += 96) sdst[i] = f.s.sx[(size_t)i * f.s.sx_inc];
      }
      asm volatile("bar.sync 2, 96;" ::: "memory");
      if (t == 0) b2_st_release_sys(ag_arrivals(c, d) + (size_t)c.rank * B2_AG_CHUNKS + j, val);
    }
  }
}

// The producer thread: wait until every chunk under gathered rows [lo, lo + BM) has arrived for this launch
// (arrival word >= val), then order those generic-proxy writes before the TMA's async-proxy reads.
__device__ __forceinline__ void ag_wait_rows(const B2DevComm& c, const GemmArgsAg& a, int lo, unsigned val) {
  const unsigned* arr = ag_arrivals(c, c.rank);
  for (int q = lo / a.m; q < c.size && q * a.m < lo + BM; ++q) {
    const int r0 = lo > q * a.m ? lo - q * a.m : 0;                 // rows [r0, r1) of shard q
    const int r1 = lo + BM < (q + 1) * a.m ? lo + BM - q * a.m : a.m;
    for (int j = r0 / a.chunk_rows; j <= (r1 - 1) / a.chunk_rows; ++j)
      b2_wait_ge(c, arr + (size_t)q * B2_AG_CHUNKS + j, val, B2_OPC_ALLGATHER, q);
  }
  asm volatile("fence.proxy.async.global;" ::: "memory");
}

// The persistent GEMM all three kernels share: producer, wgmma mainloop, 6-stage ring and tile order.  EPI
// picks what the consumers do with a group of finished tiles when the call is fused (> 1 rank);
// EPI_ALLGATHER instead gathers A while the GEMM runs (`g` is a GemmArgsAg: tma_a / g.tma_a1 map the gathered
// matrix in staging half 0 / 1), walks the tile rows from this rank's own shard on, and stores the tiles like
// the stand-alone GEMM.
enum GemmEpilogue { EPI_ALLREDUCE, EPI_REDUCE_SCATTER, EPI_ALLGATHER };

template <int EPI, typename T = __nv_bfloat16>
__device__ __forceinline__ void gemm_body(const CUtensorMap& tma_a, const CUtensorMap& tma_b, const B2DevComm& c,
                                          const GemmArgs& g) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ uint64_t full_bar[STAGES], empty_bar[STAGES];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2;
  const uint32_t smem_base = ((uint32_t)__cvta_generic_to_shared(smem_raw) + 1023u) & ~1023u;
  const uint32_t smem_a = smem_base, smem_b = smem_base + STAGES * A_STAGE_BYTES;
  auto bar = [](uint64_t* p) { return (uint32_t)__cvta_generic_to_shared(p); };

  unsigned ticket = 0, e = 0;
  if (EPI == EPI_ALLGATHER || g.fused) {
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

  constexpr bool F8 = !std::is_same_v<T, __nv_bfloat16>;
  constexpr int KB = GemmElem<T>::BK;                           // elements of K per k-block (128 bytes)
  const int num_n = g.N / BN, tiles = (g.M / BM) * num_n, num_kb = g.K / KB;

  // allgather + GEMM: tile row m_blk of the tile order is gathered tile row (m_blk + rot) mod (M / BM), so
  // the first tiles lie in this rank's own shard
  int rot = 0;
  if constexpr (EPI == EPI_ALLGATHER)
    rot = (int)(((long long)c.rank * static_cast<const GemmArgsAg&>(g).m) / BM);

  if (wg == 0) {
    if (threadIdx.x == 0) {
      // ===== TMA producer =====
      const CUtensorMap* ta = &tma_a;
      if constexpr (EPI == EPI_ALLGATHER)
        if (ticket & 1u) ta = &static_cast<const GemmArgsAg&>(g).tma_a1;
      uint32_t stage = 0, phase = 0;
      int waited = -1;                                          // allgather: the tile row already waited for
      for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        int m_blk, n_blk;
        b2_gemm_tile_coords(tile, g.M / BM, num_n, g.raster, m_blk, n_blk);
        if constexpr (EPI == EPI_ALLGATHER) {
          m_blk = (m_blk + rot) % (g.M / BM);
          if (m_blk != waited) ag_wait_rows(c, static_cast<const GemmArgsAg&>(g), m_blk * BM, ticket + 1u);
          waited = m_blk;
        }
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(bar(&empty_bar[stage]), phase ^ 1u);
          mbar_expect_tx(bar(&full_bar[stage]), A_STAGE_BYTES + B_STAGE_BYTES);
          tma_load_2d(smem_a + stage * A_STAGE_BYTES, ta, bar(&full_bar[stage]), kb * KB, m_blk * BM);
          tma_load_2d(smem_b + stage * B_STAGE_BYTES, &tma_b, bar(&full_bar[stage]), kb * KB, n_blk * BN);
          if (++stage == STAGES) { stage = 0; phase ^= 1u; }
        }
      }
    }
    if constexpr (EPI == EPI_ALLGATHER)
      if (warp > 0) ag_push<T>(c, static_cast<const GemmArgsAg&>(g), par, ticket + 1u);
  } else {
    // ===== consumers: wgmma -> bf16 -> (staging + per-group collective | output) =====
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
      if constexpr (EPI == EPI_ALLGATHER) m_blk = (m_blk + rot) % (g.M / BM);
      uint32_t prev = 0;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(bar(&full_bar[stage]), phase);                // TMA landed this stage
        const uint64_t adesc = gmma_desc(smem_a + stage * A_STAGE_BYTES + cw * 64 * 128);
        const uint64_t bdesc = gmma_desc(smem_b + stage * B_STAGE_BYTES);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < KB / GemmElem<T>::WGMMA_K; ++k) {   // +32 B per wgmma k-step inside the swizzle atom
          if constexpr (F8) wgmma_e4m3(acc, adesc + (uint64_t)(k * 2), bdesc + (uint64_t)(k * 2), (kb | k) != 0);
          else wgmma_bf16(acc, adesc + (uint64_t)(k * 2), bdesc + (uint64_t)(k * 2), (kb | k) != 0);
        }
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
      if constexpr (F8) {
        // acc * (sx[row] * sw[col]) in fp32, then the one bf16 rounding below.  Allgather: the gathered row
        // scales in the staging, written by the ranks' push warps; every full_bar wait of this tile came after
        // the producer's ld.acquire.sys of their arrival words (ag_wait_rows), so they are visible here.  L2
        // loads (.cg): another tile may have brought the same 128-byte line into L1 before all of it arrived.
        float x0, x1;
        const GemmScales* s;
        if constexpr (EPI == EPI_ALLGATHER) {
          s = &static_cast<const GemmArgsAgF8&>(g).s;
          const float* sxg = (const float*)(c.stage[c.rank] + par + static_cast<const GemmArgsAgF8&>(g).sx_off);
          x0 = __ldcg(sxg + row);
          x1 = __ldcg(sxg + row + 8);
        } else {
          s = &static_cast<const GemmArgsF8&>(g).s;
          x0 = __ldg(s->sx + row * s->sx_inc);
          x1 = __ldg(s->sx + (row + 8) * s->sx_inc);
        }
        const float* sw = s->sw + ((size_t)n_blk * BN + 2 * (lane & 3)) * s->sw_inc;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const float w0 = __ldg(sw + (size_t)(8 * j) * s->sw_inc), w1 = __ldg(sw + (size_t)(8 * j + 1) * s->sw_inc);
          acc[4 * j] *= x0 * w0;
          acc[4 * j + 1] *= x0 * w1;
          acc[4 * j + 2] *= x1 * w0;
          acc[4 * j + 3] *= x1 * w1;
        }
      }
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        *reinterpret_cast<__nv_bfloat162*>(dst + 8 * j) = __floats2bfloat162_rn(acc[4 * j], acc[4 * j + 1]);
        *reinterpret_cast<__nv_bfloat162*>(dst + 8 * (size_t)g.N + 8 * j) =
            __floats2bfloat162_rn(acc[4 * j + 2], acc[4 * j + 3]);
      }
      if (g.fused) {
        // --- reduce finished tiles across the ranks.  GROUP tiles share one pair of cross-GPU barriers;
        // all loads of a batch are issued before the first dependent store so the NVLink / L2 round trips
        // overlap instead of adding up.
        pend[np++] = tile;
        const bool last = tile + (int)gridDim.x >= tiles;
        if (np == GROUP || last) {
          // (the first barrier and the slice bounds are written in each branch: shared in front of them,
          // they change the allreduce kernel's instruction schedule)
          if constexpr (EPI == EPI_ALLREDUCE) {
            epi_barrier_all(c, ++e, et, B2_OPC_ALLREDUCE);                   // every rank staged these partial tiles
            const int per = (BM + c.size - 1) / c.size;         // my row-slice of every tile
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
            epi_barrier_all(c, ++e, et, B2_OPC_ALLREDUCE);      // all slices of these tiles have landed
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
          } else {
            epi_barrier_all(c, ++e, et, B2_OPC_REDUCE_SCATTER);                // every rank staged these partial tiles
            const int per = (BM + c.size - 1) / c.size;       // my row-slice of every tile
            const int r0 = per * c.rank < BM ? per * c.rank : BM, r1 = r0 + per < BM ? r0 + per : BM;
            const int slice_vec = (r1 - r0) * (BN / 8), nred = np * slice_vec;
            // reduce-scatter by pull, no multicast: fold this rank's row-slice of each tile over every
            // rank's staged partial in rank order (fp32, one rounding, as the bf16 reduction kernels do),
            // then store the result into the staging of the rank whose shard holds the row.  Only this
            // rank reads or writes slice `rank` of any staging, so the store races with nothing.
            const int shard = g.M / c.size;                     // output rows per rank
            for (int i = et; i < nred; i += EPI_THREADS) {
              const int slot = i / slice_vec, w = i - slot * slice_vec;
              const int tl = pend[slot], r = r0 + w / (BN / 8), v8 = w % (BN / 8);
              int tm, tn;
              b2_gemm_tile_coords(tl, g.M / BM, num_n, g.raster, tm, tn);
              const int row = tm * BM + r;
              const size_t off = par + ((size_t)row * g.N + (size_t)tn * BN + v8 * 8) * sizeof(__nv_bfloat16);
              B2Vec<__nv_bfloat16> sum;
              for (int q0 = 0; q0 < c.size; q0 += RS_BATCH) {
                uint4 x[RS_BATCH];                              // the peers' loads in flight before any fold
#pragma unroll
                for (int k = 0; k < RS_BATCH; ++k)
                  if (q0 + k < c.size) x[k] = b2_ld_peer16(c.stage[q0 + k] + off);
#pragma unroll
                for (int k = 0; k < RS_BATCH; ++k) {
                  if (q0 + k >= c.size) break;
                  if (q0 + k == 0) sum.load(x[k]);
                  else sum.template accumulate<B2_SUM>(x[k]);
                }
              }
              b2_st16(c.stage[row / shard] + off, sum.store());
            }
            epi_barrier_all(c, ++e, et, B2_OPC_REDUCE_SCATTER); // every slice of these tiles has landed
            // copy the rows of these tiles that lie in this rank's shard [lo, lo + shard) to the output
            const int lo = c.rank * shard;
            for (int slot = 0; slot < np; ++slot) {
              int tm, tn;
              b2_gemm_tile_coords(pend[slot], g.M / BM, num_n, g.raster, tm, tn);
              const int a = tm * BM > lo ? tm * BM : lo;
              const int b = tm * BM + BM < lo + shard ? tm * BM + BM : lo + shard;
              const int ncp = (b - a) * (BN / 8);               // <= 0: no row of this tile is mine
              for (int base = et; base < ncp; base += EPI_THREADS * 4) {
                uint4 v[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                  const int i = base + u * EPI_THREADS;
                  if (i < ncp)
                    v[u] = b2_ld_peer16(stage_local + (size_t)(a + i / (BN / 8)) * g.N + (size_t)tn * BN +
                                        (i % (BN / 8)) * 8);
                }
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                  const int i = base + u * EPI_THREADS;
                  if (i < ncp)
                    b2_st16(g.out + (size_t)(a - lo + i / (BN / 8)) * g.N + (size_t)tn * BN + (i % (BN / 8)) * 8,
                            v[u]);
                }
              }
            }
          }
          np = 0;
        }
      }
    }
    if (g.fused && et == 0) b2_st_volatile(c.epoch + blockIdx.x, e);
  }

  __syncthreads();
  if (EPI == EPI_ALLGATHER || g.fused) b2_finish_bump(c.ticket, c.ticket + 1, 1u, gridDim.x);
}

// The tile order, shared-memory reservation and persistent grid of a GEMM kernel; `g` is filled in except
// for the tile order.  `attr_set`: the kernel's own flag that its shared-memory size has been reserved.
template <typename Kernel>
int gemm_geometry(Kernel kernel, bool& attr_set, B2Comm* c, GemmArgs& g, const char* what, size_t& smem, int& grid) {
  // banded tile order for the stand-alone store; the fused epilogues recompute a tile's coordinates per
  // 16-byte vector (integer divisions in front of every staging load), so they keep the cheaper
  // row-major formula
  g.raster = c->gemm_raster >= 0 ? c->gemm_raster : (g.fused ? 0 : B2_GEMM_RASTER_GROUP);
  smem = (size_t)STAGES * (A_STAGE_BYTES + B_STAGE_BYTES) + 1024;
  if (!attr_set) {
    if (int rc = b2_cuda_check(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem),
                               "%s: cannot reserve %zu bytes of shared memory", what, smem))
      return rc;
    attr_set = true;
  }
  const int tiles = (g.M / BM) * (g.N / BN);
  grid = tiles < c->sm_count ? tiles : c->sm_count;
  if (grid > B2_MAX_BLOCKS) grid = B2_MAX_BLOCKS;
  return 0;
}

// TMA map of a row-major (rows x cols) operand of element type T, box BM (= BN) rows x one k-block
template <typename T>
int gemm_tensor_map(CUtensorMap* map, const void* p, int rows, int cols) {
  if constexpr (std::is_same_v<T, __nv_bfloat16>)
    return b2_tensor_map_2d_bf16(map, p, (unsigned long long)rows, (unsigned long long)cols, BM, BK);
  else
    return b2_tensor_map_2d_u8(map, p, (unsigned long long)rows, (unsigned long long)cols, BM, GemmElem<T>::BK);
}

// Tensor maps, staging check and launch of the allreduce and reduce-scatter kernels.  `Args`: GemmArgs, or
// GemmArgsF8 for the float8 kernels (element type T).
template <typename T = __nv_bfloat16, typename Kernel, typename Args>
int gemm_launch(Kernel kernel, bool& attr_set, B2Comm* c, const void* A, const void* B, Args g, const char* what,
                cudaStream_t stream) {
  if (g.fused && (size_t)g.M * g.N * 2 + 4096 > c->dev.stage_half) {
    b2_set_error("%s: staging too small (need %zu bytes, have %zu)", what, (size_t)g.M * g.N * 2 + 4096,
                 c->dev.stage_half);
    return B2_ERR_BAD_ARG;
  }
  CUtensorMap ta, tb;
  if (gemm_tensor_map<T>(&ta, A, g.M, g.K) || gemm_tensor_map<T>(&tb, B, g.N, g.K)) return B2_ERR_BAD_ARG;
  size_t smem;
  int grid;
  if (int rc = gemm_geometry(kernel, attr_set, c, g, what, smem, grid)) return rc;
  kernel<<<grid, GEMM_THREADS, smem, stream>>>(ta, tb, c->dev, g);
  return b2_launched(c, what);
}

// `kb`: the k-block in elements, BK for bf16 and GemmElem<__nv_fp8_e4m3>::BK for float8
inline bool gemm_shape_ok(const char* what, int M, int N, int K, int kb = BK) {
  if (M <= 0 || N <= 0 || K <= 0 || M % BM || N % BN || K % kb) {
    b2_set_error("%s: need M %% %d == 0, N %% %d == 0, K %% %d == 0 (got %d, %d, %d)", what, BM, BN, kb, M, N, K);
    return false;
  }
  return true;
}

inline GemmArgs gemm_args(int M, int N, int K, void* out, int fused) {
  GemmArgs g;
  memset(&g, 0, sizeof g);
  g.M = M; g.N = N; g.K = K;
  g.out = (__nv_bfloat16*)out;
  g.fused = fused;
  return g;
}

}  // namespace
