// mpi4jax_b200 -- reduction collectives over peer-mapped HBM (allreduce, reduce, scan, reduce-scatter).
//
// Replaces the reference's MPI_Allreduce / MPI_Reduce / MPI_Scan call sites
// (mpi4jax/_src/xla_bridge/mpi_ops_common.h:236-249, 310-338 and their CUDA
// callers mpi_xla_bridge_cuda.cpp:167-209, 523-632) with hand-written sm_90a
// kernels in which the reduction operator and the dtype up/down-cast are FUSED
// into the NVLink transfer: no MPI call, no host sync, no staging through host
// memory, no separate elementwise kernel.
//
// Three transports, chosen per message size by b2_allreduce():
//   * LL        flag-in-data push (8 B = 4 B payload + 4 B flag), no barrier, no
//               fence: one NVLink one-way latency.            (<= ll_max bytes)
//   * ONESHOT   stage -> barrier -> every rank pulls all P copies and reduces.
//   * TWOSHOT   stage -> barrier -> rank r reduces sub-slice r (pull) and pushes
//               the result into every peer's staging -> barrier -> copy out.
// Work is split into chunks owned by CTA (chunk mod grid) ON EVERY RANK, so all
// synchronisation is CTA<->same-CTA across GPUs (block-paired flags): CTAs are
// at different phases at any instant, which overlaps the local copy-in/copy-out
// with the NVLink reduce-scatter and all-gather phases of other chunks.
#pragma once

#include "b2_device.cuh"

struct B2ReduceArgs {
  const void* in;
  void* out;
  size_t nbytes;     // payload bytes per rank
  size_t chunk;      // chunk bytes; multiple of 16 * size
  int algo;          // B2_ALGO_ONESHOT or B2_ALGO_TWOSHOT
  int src_lo;        // contributions reduced: ranks [src_lo, src_hi)
  int src_hi;
  int has_out;       // this rank materialises a result (reduce: root only)
  int opcode;
  int pipeline;      // NVLS allreduce: stage the next chunk / copy the previous one out between arrive and wait
  unsigned long long* trace;   // optional phase timeline of CTA 0 (communicator option "trace_ptr"), else null
  int trace_cap;
};

template <typename T, int OP>
__global__ void __launch_bounds__(B2_THREADS)
b2_k_reduce_chunked(const B2DevComm c, const B2ReduceArgs a) {
  auto [par, e] = b2_staged_begin(c);
  const char* in = (const char*)a.in;
  char* out = (char*)a.out;
  char* mine = c.stage[c.rank] + par;
  const size_t nchunks = (a.nbytes + a.chunk - 1) / a.chunk;
  const int t = threadIdx.x, nt = blockDim.x;

  for (size_t ch = blockIdx.x; ch < nchunks; ch += gridDim.x) {
    const size_t off = ch * a.chunk;
    const size_t len = b2_chunk_len(a.nbytes, a.chunk, ch);
    const size_t nv = (len + 15) >> 4;        // vectors incl. a padded tail vector
    if (a.opcode == B2_OPC_REDUCE_SCATTER) {
      // reduce-scatter: nbytes is ONE block and chunks index into it.  Stage this chunk of all P
      // input blocks (block q at q * bs), then pull block `rank` from every peer and reduce it in
      // rank order.  One barrier: the staging parity alternates per launch as for one-shot.
      const size_t bs = (a.nbytes + 15) & ~(size_t)15;
      for (int q = 0; q < c.size; ++q)
        b2_copy_bytes<false>(mine + (size_t)q * bs + off, in + (size_t)q * a.nbytes + off, len);
      b2_barrier_all(c, ++e, a.opcode);
      const size_t src = (size_t)c.rank * bs + off;
      for (size_t i = t; i < nv; i += nt) {
        B2Vec<T> acc;
        acc.load(b2_ld_peer16(c.stage[0] + par + src + (i << 4)));
        for (int q = 1; q < c.size; ++q)
          acc.template accumulate<OP>(b2_ld_peer16(c.stage[q] + par + src + (i << 4)));
        const uint4 r = acc.store();
        const size_t b = i << 4;
        if (b + 16 <= len) b2_st16(out + off + b, r);
        else b2_store_partial(out + off + b, r, (int)(len - b));
      }
      continue;
    }
    // 1. stage my contribution (local HBM -> local symmetric staging)
    b2_copy_bytes<false>(mine + off, in + off, len);
    // 2. everybody's copy of this chunk is staged
    b2_barrier_all(c, ++e, a.opcode);

    if (a.algo == B2_ALGO_ONESHOT) {
      if (a.has_out) {
        for (size_t i = t; i < nv; i += nt) {
          B2Vec<T> acc;
          acc.load(b2_ld_peer16(c.stage[a.src_lo] + par + off + (i << 4)));
          for (int q = a.src_lo + 1; q < a.src_hi; ++q)
            acc.template accumulate<OP>(b2_ld_peer16(c.stage[q] + par + off + (i << 4)));
          const uint4 r = acc.store();
          const size_t b = i << 4;
          if (b + 16 <= len) b2_st16(out + off + b, r);
          else b2_store_partial(out + off + b, r, (int)(len - b));
        }
      }
    } else {
      // 3. reduce-scatter by pull: rank r owns vectors [v0, v1) of this chunk
      const size_t per = (nv + c.size - 1) / c.size;
      size_t v0 = per * (size_t)c.rank;
      if (v0 > nv) v0 = nv;
      size_t v1 = v0 + per;
      if (v1 > nv) v1 = nv;
      if (a.opcode == B2_OPC_SCAN) {
        // two-phase scan: all P copies of a vector are loaded BEFORE the prefixes overwrite them
        // (prefix q lands where rank q staged its own contribution; this rank is the only reader)
        for (size_t i = v0 + t; i < v1; i += nt) {
          uint4 v[B2_MAX_RANKS];
#pragma unroll
          for (int q = 0; q < B2_MAX_RANKS; ++q)
            if (q < c.size) v[q] = b2_ld_peer16(c.stage[q] + par + off + (i << 4));
          B2Vec<T> acc;
          acc.load(v[0]);
          // float8 rounds every result, rank 0's single contribution too (a non-canonical e5m2 NaN)
          if constexpr (b2_is_fp8<T>::value) b2_st16(c.stage[0] + par + off + (i << 4), acc.store());
#pragma unroll
          for (int q = 1; q < B2_MAX_RANKS; ++q)
            if (q < c.size) {
              acc.template accumulate<OP>(v[q]);
              b2_st16(c.stage[q] + par + off + (i << 4), acc.store());
            }
        }
      } else
      for (size_t i = v0 + t; i < v1; i += nt) {
        B2Vec<T> acc;
        acc.load(b2_ld_peer16(c.stage[0] + par + off + (i << 4)));
        for (int q = 1; q < c.size; ++q)
          acc.template accumulate<OP>(b2_ld_peer16(c.stage[q] + par + off + (i << 4)));
        const uint4 r = acc.store();
        // 4. all-gather by push: result goes straight into every peer's staging
        for (int q = 0; q < c.size; ++q) {
          const int p = (c.rank + q) % c.size;   // stagger destinations across ranks
          b2_st16(c.stage[p] + par + off + (i << 4), r);
        }
      }
      // 5. every sub-slice of this chunk has landed in my staging
      b2_barrier_all(c, ++e, a.opcode);
      // 6. staging -> user output
      if (a.has_out) b2_copy_bytes<true>(out + off, mine + off, len);
    }
  }
  b2_staged_end(c, e);
}

// ---------------------------------------------------------------------------
// LL allreduce.  Wire format per 16-byte payload vector: two 16-byte stores
// {w0, flag, w1, flag} {w2, flag, w3, flag}; each 8-byte half is written
// atomically, so a reader that sees `flag` in a half sees its payload word.
// flag = ticket + 1 (never 0, unique for 2^32 launches; buffers alternate by
// ticket parity so a sender can never overwrite data that is still being read:
// to be two tickets ahead it needs this rank's contribution to the ticket in
// between, which this rank only sends after it finished reading).
//
// Reduce-scatter uses the same kernel with `src_stride` = the block size: peer p receives block p
// (in + p * src_stride) and this rank folds its own block (in + rank * src_stride) with the P - 1 it
// received.  Allreduce passes 0: every peer receives the whole input.
// ---------------------------------------------------------------------------
struct B2LLArgs {
  const void* in;
  void* out;
  size_t nbytes;       // payload bytes per destination (allreduce: all of it; reduce-scatter: one block)
  size_t src_stride;   // bytes between the inputs of consecutive destinations (0: one input for all)
  int opcode;
};

// vector i of a payload of nbytes bytes, zero padded past the end
__device__ __forceinline__ uint4 b2_ll_load(const char* in, size_t b, size_t nbytes, bool aligned) {
  if (aligned && b + 16 <= nbytes) return *reinterpret_cast<const uint4*>(in + b);
  alignas(16) unsigned char tmp[16];
  for (int k = 0; k < 16; ++k) tmp[k] = (b + k < nbytes) ? ((const unsigned char*)in)[b + k] : 0;
  return *reinterpret_cast<const uint4*>(tmp);
}

template <typename T, int OP>
__global__ void __launch_bounds__(B2_THREADS)
b2_k_allreduce_ll(const B2DevComm c, const B2LLArgs a) {
  const unsigned ticket = b2_ticket_read(c.ticket);
  const unsigned flag = ticket + 1u;
  const size_t par_off = c.lay.ll_off + (size_t)(ticket & 1u) * c.size * c.lay.ll_cap;
  const size_t nv = (a.nbytes + 15) >> 4;
  const char* in = (const char*)a.in;
  char* out = (char*)a.out;
  const size_t stride = a.src_stride;
  const bool aligned = ((((uintptr_t)in) | stride) & 15) == 0;     // every block start is 16-byte aligned

  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < nv;
       i += (size_t)gridDim.x * blockDim.x) {
    const size_t b = i << 4;
    const uint4 mine = b2_ll_load(in + (size_t)c.rank * stride, b, a.nbytes, aligned);
    // push to every peer's LL buffer, slot [source = my rank][vector i]
    for (int q = 1; q < c.size; ++q) {
      const int p = (c.rank + q) % c.size;
      const uint4 v = stride ? b2_ll_load(in + (size_t)p * stride, b, a.nbytes, aligned) : mine;
      char* dst = c.heap[p] + par_off + (size_t)c.rank * c.lay.ll_cap + (i << 5);
      b2_st16_sys(dst, make_uint4(v.x, flag, v.y, flag));
      b2_st16_sys(dst + 16, make_uint4(v.z, flag, v.w, flag));
    }
    // gather + reduce in rank order (bitwise identical result on every rank)
    B2Vec<T> acc;
    B2Watchdog<> wd;
    for (int q = 0; q < c.size; ++q) {
      uint4 v;
      if (q == c.rank) {
        v = mine;
      } else {
        const char* src = c.heap[c.rank] + par_off + (size_t)q * c.lay.ll_cap + (i << 5);
        uint4 l, h;
        while (true) {
          l = b2_ld_peer16(src);
          h = b2_ld_peer16(src + 16);
          if (l.y == flag && l.w == flag && h.y == flag && h.w == flag) break;
          if (wd.expired(c)) b2_fatal(c, B2_ERR_TIMEOUT, a.opcode, q, flag, l.y, 2);
        }
        v = make_uint4(l.x, l.z, h.x, h.z);
      }
      if (q == 0) acc.load(v);
      else acc.template accumulate<OP>(v);
    }
    const uint4 r = acc.store();
    if (b + 16 <= a.nbytes) b2_st16(out + b, r);
    else b2_store_partial(out + b, r, (int)(a.nbytes - b));
  }
  b2_finish_bump(c.ticket, c.ticket + 1, 1u, gridDim.x);
}

// ---------------------------------------------------------------------------
// reduce_scatterv: variable row counts that exist only on the device.
//
// Staging parity of every rank: [header: this rank's send counts clamped in rank order to its input
// rows, int64 x B2_MAX_RANKS (B2_A2AV_HDR)] [P blocks of round16(N * row_bytes)].  Block p holds the
// first min(s_r[p], N) rows of this rank's segment for rank p -- only real rows are staged.
//
// The schedule is b2_k_rowsv's: every CTA writes the header and stages its first chunk before its first
// arrive; after the first wait it reads the P x P counts, and the chunks of a block (bytes, up to the
// largest min(s_q[p], N) rows of any pair -- the same on every rank) belong to CTA k mod grid everywhere.
// Chunk k of block r is then folded from every peer's staging, in rank order over the ranks whose
// segment reaches that element; rows [max_q c[q], N) are zero.
// ---------------------------------------------------------------------------
struct B2RsvArgs {
  const void* in;
  void* out;
  const long long* send_counts;    // [P] rows to each rank (any value: clamped here)
  long long* recv_counts;          // [P] rows folded from each rank
  size_t row_bytes;
  size_t in_rows;                  // may differ between ranks
  size_t out_rows;                 // N: the same on every rank (sizes the staging and the chunks)
  size_t chunk;
  int opcode;
};

// Fold the vector at byte v of block `rank` over the ranks q with v < len[q], in rank order.  Segments
// are prefixes of the block, so the ranks that reach element j of the vector are exactly those with
// len[q] > v + j * sizeof(T); `covered` is how far into the vector an earlier rank reached.  The peers'
// loads are issued RSV_BATCH at a time before any of them is folded, so their NVLink round trips overlap.
#define RSV_BATCH 4
template <typename T, int OP>
__device__ __forceinline__ uint4 rsv_fold(const B2DevComm& c, size_t src, size_t v, const size_t* len) {
  using Tr = B2Traits<T>;
  constexpr int N = B2Vec<T>::N;
  B2Vec<T> acc;
  size_t covered = 0;
  for (int q0 = 0; q0 < c.size; q0 += RSV_BATCH) {
    uint4 x[RSV_BATCH];
#pragma unroll
    for (int k = 0; k < RSV_BATCH; ++k) {
      x[k] = make_uint4(0, 0, 0, 0);
      if (q0 + k < c.size && v < len[q0 + k]) x[k] = b2_ld_peer16(c.stage[q0 + k] + src + v);
    }
#pragma unroll
    for (int k = 0; k < RSV_BATCH; ++k) {
      const int q = q0 + k;
      if (q >= c.size || v >= len[q]) continue;
      const size_t nb = len[q] - v < 16 ? len[q] - v : 16;
      if (covered == 0) {
        acc.load(x[k]);
      } else if (nb == 16 && covered == 16) {
        acc.template accumulate<OP>(x[k]);
      } else {             // a segment ends inside this vector (row_bytes % 16 != 0)
        alignas(16) T tmp[N];
        *reinterpret_cast<uint4*>(tmp) = x[k];
#pragma unroll
        for (int j = 0; j < N; ++j) {
          const size_t eb = (size_t)j * sizeof(T);
          if (eb < nb) {
            const typename Tr::Acc u = Tr::up(tmp[j]);
            acc.a[j] = eb < covered ? b2_apply<OP, typename Tr::Acc>(acc.a[j], u) : u;
          }
        }
      }
      if (nb > covered) covered = nb;
    }
  }
  return acc.store();
}
#undef RSV_BATCH

template <typename T, int OP>
__global__ void __launch_bounds__(B2_THREADS, 1)
b2_k_reduce_scatterv(const B2DevComm c, const B2RsvArgs a) {
  __shared__ size_t s_src[B2_MAX_RANKS], s_mine[B2_MAX_RANKS];   // this rank's segments: input byte, staged bytes
  __shared__ size_t s_len[B2_MAX_RANKS];                         // bytes of block `rank` staged by peer q
  __shared__ size_t s_cnt[B2_MAX_RANKS][B2_MAX_RANKS];           // [q][p]: min(s_q[p], N)
  __shared__ size_t s_fold, s_nch;
  auto [par, e] = b2_staged_begin(c);
  const int t = threadIdx.x, nt = blockDim.x, P = c.size, r = c.rank;
  const char* in = (const char*)a.in;
  char* out = (char*)a.out;
  char* mine = c.stage[r] + par;
  const size_t rb = a.row_bytes;
  const size_t bs = (a.out_rows * rb + 15) & ~(size_t)15;
  char* blocks = mine + B2_A2AV_HDR;
  // 1. this rank's counts, clamped in rank order to the rows that exist -> header
  if (t == 0) {
    size_t used = 0;
    for (int p = 0; p < P; ++p) {
      size_t s = a.send_counts[p] > 0 ? (size_t)a.send_counts[p] : 0;
      if (s > a.in_rows - used) s = a.in_rows - used;
      ((volatile unsigned long long*)mine)[p] = s;
      s_src[p] = used * rb;
      s_mine[p] = (s < a.out_rows ? s : a.out_rows) * rb;
      used += s;
    }
  }
  __syncthreads();
  // chunk ch of every block this rank sends (n written out: b2_chunk_len changes this kernel's SASS)
  auto stage = [&](size_t ch) {
    const size_t off = ch * a.chunk;
    for (int p = 0; p < P; ++p)
      if (off < s_mine[p]) {
        const size_t n = s_mine[p] - off < a.chunk ? s_mine[p] - off : a.chunk;
        b2_copy_bytes<false>(blocks + (size_t)p * bs + off, in + s_src[p] + off, n);
      }
  };
  size_t ch = blockIdx.x;
  stage(ch);
  b2_barrier_arrive(c, ++e);
  unsigned e_cur = e;
  b2_barrier_wait(c, e_cur, a.opcode);   // every rank's header and chunk blockIdx.x are staged
  // 2. the peers' headers: what each sends here, and the longest segment of any pair (the loop bound)
  if (t < P * P) {
    const unsigned long long h = ((const volatile unsigned long long*)(c.stage[t / P] + par))[t % P];
    s_cnt[t / P][t % P] = h < a.out_rows ? (size_t)h : a.out_rows;
  }
  __syncthreads();
  if (t == 0) {
    size_t lmax = 0, cmax = 0;
    for (int q = 0; q < P; ++q) {
      for (int p = 0; p < P; ++p)
        if (s_cnt[q][p] > lmax) lmax = s_cnt[q][p];
      const size_t k = s_cnt[q][r];
      s_len[q] = k * rb;
      if (k > cmax) cmax = k;
      if (blockIdx.x == 0) a.recv_counts[q] = (long long)k;
    }
    s_fold = cmax * rb;
    s_nch = (lmax * rb + a.chunk - 1) / a.chunk;        // the same on every rank
  }
  __syncthreads();
  // 3. stage -> arrive -> wait -> fold, software-pipelined over the chunks of this CTA
  const size_t nch = s_nch, fold = s_fold;
  const size_t src = par + B2_A2AV_HDR + (size_t)r * bs;
  for (; ch < nch; ch += gridDim.x) {
    if (ch != blockIdx.x) b2_barrier_wait(c, e_cur, a.opcode);
    const size_t off = ch * a.chunk;
    const size_t end = off + a.chunk < fold ? off + a.chunk : fold;
    for (size_t v = off + ((size_t)t << 4); v < end; v += (size_t)nt << 4) {
      const uint4 res = rsv_fold<T, OP>(c, src, v, s_len);
      if (v + 16 <= end) b2_st16(out + v, res);
      else b2_store_partial(out + v, res, (int)(end - v));
    }
    const size_t nxt = ch + gridDim.x;
    if (nxt < nch) {
      stage(nxt);
      b2_barrier_arrive(c, ++e);
      e_cur = e;
    }
  }
  // 4. rows nobody sends are zero: the output is fully written on every call
  a2av_zero(out, fold, a.out_rows * rb);
  b2_staged_end(c, e);
}

// ---------------------------------------------------------------------------
// host-side typed dispatch.  Each b2_reduce_inst_N.cu registers the launchers of
// one dtype group (keeps nvcc parallel and fast); the caller checks the launch.
// ---------------------------------------------------------------------------
typedef void (*b2_reduce_launch_fn)(const B2DevComm&, const B2ReduceArgs&, int grid, cudaStream_t);
typedef void (*b2_ll_launch_fn)(const B2DevComm&, const B2LLArgs&, int grid, cudaStream_t);
typedef void (*b2_rsv_launch_fn)(const B2DevComm&, const B2RsvArgs&, int grid, cudaStream_t);

template <typename T, int OP>
void b2_launch_reduce(const B2DevComm& c, const B2ReduceArgs& a, int grid, cudaStream_t s) {
  b2_k_reduce_chunked<T, OP><<<grid, B2_THREADS, 0, s>>>(c, a);
}
template <typename T, int OP>
void b2_launch_ll(const B2DevComm& c, const B2LLArgs& a, int grid, cudaStream_t s) {
  b2_k_allreduce_ll<T, OP><<<grid, B2_THREADS, 0, s>>>(c, a);
}
template <typename T, int OP>
void b2_launch_rsv(const B2DevComm& c, const B2RsvArgs& a, int grid, cudaStream_t s) {
  b2_k_reduce_scatterv<T, OP><<<grid, B2_THREADS, 0, s>>>(c, a);
}

// tables filled by the instance files: [dtype][op] -> launcher (nullptr = invalid combo); b2_rsv_kernel
// holds the kernel itself, for the co-residency query
extern b2_reduce_launch_fn b2_reduce_table[B2_DTYPE_COUNT][B2_OP_COUNT];
extern b2_ll_launch_fn b2_ll_table[B2_DTYPE_COUNT][B2_OP_COUNT];
extern b2_rsv_launch_fn b2_rsv_table[B2_DTYPE_COUNT][B2_OP_COUNT];
extern const void* b2_rsv_kernel[B2_DTYPE_COUNT][B2_OP_COUNT];
void b2_register_reduce_group_0();
void b2_register_reduce_group_1();
void b2_register_reduce_group_2();
void b2_register_reduce_group_3();
void b2_register_reduce_group_4();

#define B2_REG(DT, T, OP)                                                \
  b2_reduce_table[DT][OP] = &b2_launch_reduce<T, OP>;                    \
  b2_ll_table[DT][OP] = &b2_launch_ll<T, OP>;                            \
  b2_rsv_table[DT][OP] = &b2_launch_rsv<T, OP>;                          \
  b2_rsv_kernel[DT][OP] = (const void*)&b2_k_reduce_scatterv<T, OP>;

#define B2_REG_ARITH(DT, T) \
  B2_REG(DT, T, B2_SUM) B2_REG(DT, T, B2_PROD) B2_REG(DT, T, B2_MIN) B2_REG(DT, T, B2_MAX)
#define B2_REG_INT(DT, T)                                                              \
  B2_REG_ARITH(DT, T) B2_REG(DT, T, B2_LAND) B2_REG(DT, T, B2_LOR) B2_REG(DT, T, B2_LXOR) \
  B2_REG(DT, T, B2_BAND) B2_REG(DT, T, B2_BOR) B2_REG(DT, T, B2_BXOR)
