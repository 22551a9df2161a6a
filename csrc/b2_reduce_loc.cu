// mpi4jax_b200 -- MAXLOC / MINLOC: value-index reductions for allreduce, reduce, scan and reduce-scatter.
//
// One kernel family on the staged one-shot protocol (b2_staged_begin / b2_staged_end, block-paired
// barriers), instantiated per value dtype and operator.  Every rank packs its (value, index) pairs into
// 16-byte records in its staging (B2_LOC_RECORD), so a pair is one peer load and the fold needs no second
// stream; after the barrier each rank pulls the records of the ranks it folds -- all of them issued before
// any is folded -- and folds them in rank order.  The result is always one of the input pairs, copied,
// never recomputed: values keep their bits (signed zeros, NaN payloads), indices are narrowed back to their
// width without loss.
//
// The fold rule (mpi4jax_b200/_src/collective_ops/_loc.py states it for every backend): folding the
// accumulator a (earlier ranks) with the next rank's pair b, MAXLOC takes b when b.v > a.v, or when the
// values are equal (+0 == -0) and b.i < a.i; a NaN value beats every other value, and two NaNs are equal.
// MINLOC is the same with <.  Values compare as their dtype; f16 / bf16 as float.
#include "b2_reduce_loc.cuh"

b2_loc_launch_fn b2_loc_table[B2_DTYPE_COUNT][2];
const void* b2_loc_kernel[B2_DTYPE_COUNT][2];

// The comparison type of a value dtype, and a value from the low bytes of a record.
template <typename V> struct B2LocKey;
template <> struct B2LocKey<float> {
  using K = float;
  static __device__ __forceinline__ K of(unsigned long long b) { return __uint_as_float((unsigned)b); }
};
template <> struct B2LocKey<double> {
  using K = double;
  static __device__ __forceinline__ K of(unsigned long long b) { return __longlong_as_double((long long)b); }
};
template <> struct B2LocKey<__half> {
  using K = float;
  static __device__ __forceinline__ K of(unsigned long long b) { return __half2float(__ushort_as_half((unsigned short)b)); }
};
template <> struct B2LocKey<__nv_bfloat16> {
  using K = float;
  static __device__ __forceinline__ K of(unsigned long long b) {
    return __bfloat162float(__ushort_as_bfloat16((unsigned short)b));
  }
};
template <> struct B2LocKey<short> {
  using K = int;
  static __device__ __forceinline__ K of(unsigned long long b) { return (short)(unsigned short)b; }
};
template <> struct B2LocKey<int> {
  using K = int;
  static __device__ __forceinline__ K of(unsigned long long b) { return (int)(unsigned)b; }
};
template <> struct B2LocKey<long long> {
  using K = long long;
  static __device__ __forceinline__ K of(unsigned long long b) { return (long long)b; }
};

// Does the next rank's pair (bv, bi) replace the accumulator (av, ai)?
template <int OP, typename K>
__device__ __forceinline__ bool b2_loc_takes(K av, long long ai, K bv, long long bi) {
  if constexpr (b2_is_float<K>::value) {
    const bool an = av != av, bn = bv != bv;
    if (an || bn) return bn && (!an || bi < ai);
  }
  return (OP == B2_MAXLOC ? bv > av : bv < av) || (bv == av && bi < ai);
}

// the raw bits of element i of an array of 2-, 4- or 8-byte elements, zero-extended
template <int BYTES>
__device__ __forceinline__ unsigned long long b2_loc_bits(const char* p, size_t i) {
  if constexpr (BYTES == 2) return ((const unsigned short*)p)[i];
  else if constexpr (BYTES == 4) return ((const unsigned*)p)[i];
  else return ((const unsigned long long*)p)[i];
}

#define LOC_BATCH 8   // peer loads in flight per pair before the first one is folded (P <= 8 on HGX H100)

template <typename V, int OP>
__global__ void __launch_bounds__(B2_THREADS, 1)
b2_k_reduce_loc(const __grid_constant__ B2DevComm c, const __grid_constant__ B2LocArgs a) {
  using K = typename B2LocKey<V>::K;
  constexpr int VB = (int)sizeof(V);
  auto [par, e] = b2_staged_begin(c);
  const int t = threadIdx.x, nt = blockDim.x;
  const char* in_val = (const char*)a.in_val;
  const char* in_idx = (const char*)a.in_idx;
  char* mine = c.stage[c.rank] + par;
  const size_t n = a.count, blk = n * B2_LOC_RECORD;        // records per block, staged bytes per block
  const size_t per = a.chunk / B2_LOC_RECORD;                // records per chunk
  const size_t nch = (blk + a.chunk - 1) / a.chunk;
  // chunk ch of every block this rank sends -> records in its staging
  auto stage = [&](size_t ch) {
    const size_t r0 = ch * per, r1 = r0 + per < n ? r0 + per : n;
    for (int b = 0; b < a.nblk; ++b) {
      const size_t base = (size_t)b * n;
      for (size_t i = r0 + t; i < r1; i += nt) {
        const unsigned long long v = b2_loc_bits<VB>(in_val, base + i);
        const long long x = a.idx_bytes == 4 ? (long long)((const int*)in_idx)[base + i]
                                             : ((const long long*)in_idx)[base + i];
        b2_st16(mine + (size_t)b * blk + i * B2_LOC_RECORD,
                make_uint4((unsigned)v, (unsigned)(v >> 32), (unsigned)x, (unsigned)((unsigned long long)x >> 32)));
      }
    }
  };
  // the block this rank folds: its own for reduce-scatter, the only one otherwise
  const size_t src = par + (a.nblk > 1 ? (size_t)c.rank * blk : 0);
  size_t ch = blockIdx.x;                                    // the grid never exceeds the chunks
  stage(ch);
  b2_barrier_arrive(c, ++e);
  unsigned e_cur = e;
  for (; ch < nch; ch += gridDim.x) {
    const size_t nxt = ch + gridDim.x;
    if (nxt < nch) stage(nxt);                               // between this chunk's arrive and its wait
    b2_barrier_wait(c, e_cur, a.opcode);                     // every rank staged this chunk
    if (a.has_out) {
      const size_t r0 = ch * per, r1 = r0 + per < n ? r0 + per : n;
      for (size_t i = r0 + t; i < r1; i += nt) {
        unsigned long long av = 0;
        long long ai = 0;
        K ak = K(0);
        for (int q0 = a.src_lo; q0 < a.src_hi; q0 += LOC_BATCH) {
          uint4 r[LOC_BATCH];
#pragma unroll
          for (int k = 0; k < LOC_BATCH; ++k)
            if (q0 + k < a.src_hi) r[k] = b2_ld_peer16(c.stage[q0 + k] + src + i * B2_LOC_RECORD);
#pragma unroll
          for (int k = 0; k < LOC_BATCH; ++k) {
            if (q0 + k >= a.src_hi) break;
            const unsigned long long bv = (unsigned long long)r[k].x | ((unsigned long long)r[k].y << 32);
            const long long bi = (long long)((unsigned long long)r[k].z | ((unsigned long long)r[k].w << 32));
            const K bk = B2LocKey<V>::of(bv);
            if (q0 + k == a.src_lo || b2_loc_takes<OP, K>(ak, ai, bk, bi)) {
              av = bv;
              ai = bi;
              ak = bk;
            }
          }
        }
        if constexpr (VB == 2) ((unsigned short*)a.out_val)[i] = (unsigned short)av;
        else if constexpr (VB == 4) ((unsigned*)a.out_val)[i] = (unsigned)av;
        else ((unsigned long long*)a.out_val)[i] = av;
        if (a.idx_bytes == 4) ((int*)a.out_idx)[i] = (int)ai;
        else ((long long*)a.out_idx)[i] = ai;
      }
    }
    if (nxt < nch) {
      b2_barrier_arrive(c, ++e);
      e_cur = e;
    }
  }
  b2_staged_end(c, e);
}
#undef LOC_BATCH

template <typename V, int OP>
static void b2_launch_loc(const B2DevComm& c, const B2LocArgs& a, int grid, cudaStream_t s) {
  b2_k_reduce_loc<V, OP><<<grid, B2_THREADS, 0, s>>>(c, a);
}

#define B2_REG_LOC(DT, V)                                                        \
  b2_loc_table[DT][0] = &b2_launch_loc<V, B2_MAXLOC>;                            \
  b2_loc_table[DT][1] = &b2_launch_loc<V, B2_MINLOC>;                            \
  b2_loc_kernel[DT][0] = (const void*)&b2_k_reduce_loc<V, B2_MAXLOC>;            \
  b2_loc_kernel[DT][1] = (const void*)&b2_k_reduce_loc<V, B2_MINLOC>;

void b2_register_reduce_loc() {
  B2_REG_LOC(B2_F32, float)
  B2_REG_LOC(B2_F64, double)
  B2_REG_LOC(B2_F16, __half)
  B2_REG_LOC(B2_BF16, __nv_bfloat16)
  B2_REG_LOC(B2_I16, short)
  B2_REG_LOC(B2_I32, int)
  B2_REG_LOC(B2_I64, long long)
}
