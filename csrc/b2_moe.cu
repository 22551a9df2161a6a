// mpi4jax_b200 -- top-k mixture-of-experts dispatch and combine (mpi4jax_b200/ops/moe.py states the rules).
//
// b2_k_moe_dispatch: the staged protocol of b2_k_rowsv with a per-expert schedule.  Staging parity of every
// rank: [header: its E send counts, int64 x B2_MOE_MAX_EXPERTS] [its pairs' rows in expert order].  The rows are
// gathered from the tokens while they are staged (sorted pair s carries token order[s] / k), so the k-fold copy
// of the input never exists in HBM.  Every CTA writes the header before its first arrive; after the first wait
// each CTA reads all P x E counts and derives, the same on every rank:
//   * this rank's E receive segments, (local expert l, source q) at l * P + q: the rows of q's staged expert
//     r L + l, packed in that order and cut at out_rows, then one zero gap up to out_rows;
//   * where each expert's pairs of this rank land on its owner, so that every CTA writes pos / dest for its
//     share of this rank's pairs.
// Chunk c of the staged bytes belongs to CTA c mod grid on every rank, as in b2_k_rowsv: a pull is the
// intersection of a chunk with a segment, and chunk c + grid is staged between the arrive and the wait.
//
// b2_k_moe_combine<T>: every rank stages the filled rows of its expert outputs; a token's k rows may lie in any
// chunk of any peer, so the block-paired barrier is followed by a grid-wide wait (b2_grid_wait) before the
// pulls.  Work goes grid-stride over (token, 16-byte vector); each work item issues up to MOE_BATCH peer loads
// before it folds them, in slot order, with separate round-to-nearest products and sums (no FMA contraction).
#include <climits>
#include <cstring>

#include "b2_device.cuh"
#include "b2_runtime.h"

namespace {

constexpr int MOE_BATCH = 8;     // peer loads in flight per work item of the combine
constexpr int SCAN_PER_THREAD = B2_MAX_RANKS * B2_MOE_MAX_EXPERTS / B2_THREADS;

// Inclusive prefix sums, in place, over runs of `seg` entries of the first `len` entries of each of `nrows`
// rows (seg divides len; nrows x len <= SCAN_PER_THREAD x blockDim).  All threads call.
__device__ __forceinline__ void moe_scan(unsigned (*a)[B2_MOE_MAX_EXPERTS], int nrows, int len, int seg) {
  const int t = threadIdx.x, nt = blockDim.x, n = nrows * len;
  for (int d = 1; d < seg; d <<= 1) {
    unsigned v[SCAN_PER_THREAD];
#pragma unroll
    for (int u = 0; u < SCAN_PER_THREAD; ++u) {
      const int i = t + u * nt, x = i % len;
      v[u] = (i < n && x % seg >= d) ? a[i / len][x - d] : 0u;
    }
    __syncthreads();
#pragma unroll
    for (int u = 0; u < SCAN_PER_THREAD; ++u) {
      const int i = t + u * nt;
      if (i < n) a[i / len][i % len] += v[u];
    }
    __syncthreads();
  }
}

// Stage bytes [off, off + len) of this rank's sorted pair rows: staged row s is row order[s] / k of `in`, moved in
// units of U bytes (U divides the row bytes and the input's alignment).
template <int U>
__device__ __forceinline__ void moe_gather(char* __restrict__ dst, const char* __restrict__ in,
                                           const long long* __restrict__ order, int k, size_t rb, size_t off,
                                           size_t len) {
  for (size_t i = threadIdx.x; i < len / U; i += blockDim.x) {
    const size_t b = off + i * U, s = b / rb;
    const char* src = in + (size_t)(order[s] / k) * rb + (b - s * rb);
    if (U == 16) b2_st16(dst + i * U, b2_ld_stream16(src));
    else if (U == 4) *(unsigned*)(dst + i * U) = *(const unsigned*)src;
    else dst[i * U] = *src;
  }
}

}  // namespace

struct B2MoeDispatchArgs {
  const void* in;
  void* out;
  const long long* order;        // [n_pairs]
  const long long* send_counts;  // [E]
  long long* recv_counts;        // [L x P] or null
  long long* pos;                // [n_pairs] or null
  long long* dest;               // [n_pairs] or null
  size_t row_bytes;
  size_t n_pairs;
  size_t out_rows;
  size_t chunk;
  int k;
  int num_experts;
  int opcode;
};

__global__ void __launch_bounds__(B2_THREADS, 1)
b2_k_moe_dispatch(const __grid_constant__ B2DevComm c, const __grid_constant__ B2MoeDispatchArgs a) {
  __shared__ unsigned s_pre[B2_MAX_RANKS][B2_MOE_MAX_EXPERTS];   // [q][e]: q's sorted pairs of experts <= e
  __shared__ unsigned s_land[1][B2_MOE_MAX_EXPERTS];             // [e]: rows of the owner of e for experts <= e
  __shared__ unsigned s_base[B2_MOE_MAX_EXPERTS];                // [e]: the owner's row of this rank's first pair of e
  __shared__ unsigned s_src[B2_MOE_MAX_EXPERTS], s_dst[B2_MOE_MAX_EXPERTS], s_len[B2_MOE_MAX_EXPERTS];  // rows
  __shared__ size_t s_nch, s_filled;
  auto [par, e] = b2_staged_begin(c);
  const int t = threadIdx.x, P = c.size, r = c.rank, E = a.num_experts, L = E / P;
  const size_t rb = a.row_bytes, n = a.n_pairs;
  char* mine = c.stage[r] + par;
  char* mine_rows = mine + B2_MOE_HDR;
  // 1. this rank's counts, clamped in expert order to its n pairs -> header
  if (t < E) {
    const long long w = a.send_counts[t];
    s_pre[0][t] = w <= 0 ? 0u : (unsigned)((unsigned long long)w < n ? w : n);
  }
  __syncthreads();
  for (int d = 1; d < E; d <<= 1) {            // saturating at n (each term <= n < 2^31: no overflow)
    const unsigned v = (t < E && t >= d) ? s_pre[0][t - d] : 0u;
    __syncthreads();
    if (t < E) s_pre[0][t] = (unsigned)min((size_t)s_pre[0][t] + v, n);
    __syncthreads();
  }
  if (t < E) ((volatile unsigned long long*)mine)[t] = s_pre[0][t] - (t > 0 ? s_pre[0][t - 1] : 0u);
  const size_t mine_bytes = (size_t)s_pre[0][E - 1] * rb;
  const int unit = ((((uintptr_t)a.in) | rb) & 15) == 0 ? 16 : ((((uintptr_t)a.in) | rb) & 3) == 0 ? 4 : 1;
  auto stage = [&](size_t ch) {
    const size_t off = ch * a.chunk;
    if (off >= mine_bytes) return;
    const size_t len = b2_chunk_len(mine_bytes, a.chunk, ch);
    const char* in = (const char*)a.in;
    if (unit == 16) moe_gather<16>(mine_rows + off, in, a.order, a.k, rb, off, len);
    else if (unit == 4) moe_gather<4>(mine_rows + off, in, a.order, a.k, rb, off, len);
    else moe_gather<1>(mine_rows + off, in, a.order, a.k, rb, off, len);
  };
  size_t ch = blockIdx.x;
  stage(ch);
  b2_barrier_arrive(c, ++e);
  unsigned e_cur = e;
  b2_barrier_wait(c, e_cur, a.opcode);            // every rank's header and chunk blockIdx.x are staged
  // 2. every rank's counts; per expert: all ranks' pairs and those of the ranks below this one; per receive
  // segment: its length and the rows of the lower sources in front of it
  for (int i = t; i < P * E; i += blockDim.x)
    s_pre[i / E][i % E] = (unsigned)((const volatile unsigned long long*)(c.stage[i / E] + par))[i % E];
  __syncthreads();
  if (t < E) {
    unsigned tot = 0, below = 0, front = 0;
    const int q = t % P, er = r * L + t / P;      // segment t: source q, expert er of this rank
    for (int p = 0; p < P; ++p) {
      tot += s_pre[p][t];
      if (p < r) below += s_pre[p][t];
      if (p < q) front += s_pre[p][er];
    }
    s_land[0][t] = tot;
    s_base[t] = below;
    s_len[t] = s_pre[q][er];
    s_dst[t] = front;
  }
  __syncthreads();
  moe_scan(s_pre, P, E, E);
  moe_scan(s_land, 1, E, L);
  if (t < E) {
    const int q = t % P, er = r * L + t / P;
    const unsigned len = s_len[t];
    const size_t dst = (size_t)(er % L ? s_land[0][er - 1] : 0u) + s_dst[t];
    s_src[t] = s_pre[q][er] - len;
    s_dst[t] = (unsigned)(dst < a.out_rows ? dst : a.out_rows);
    const size_t keep = dst < a.out_rows ? min((size_t)len, a.out_rows - dst) : 0;
    s_len[t] = (unsigned)keep;
    if (blockIdx.x == 0 && a.recv_counts != nullptr) a.recv_counts[t] = (long long)keep;
    s_base[t] += t % L ? s_land[0][t - 1] : 0u;
  }
  if (t == 0) {
    size_t smax = 0;
    for (int q = 0; q < P; ++q) smax = max(smax, (size_t)s_pre[q][E - 1]);
    s_nch = (smax * rb + a.chunk - 1) / a.chunk;     // the same on every rank
    s_filled = min((size_t)s_land[0][r * L + L - 1], a.out_rows);
  }
  __syncthreads();
  // 3. where this rank's pairs landed: sorted pair s of expert x is pair w = s - (first of x) of its segment
  if (a.pos != nullptr) {
    const size_t gt = (size_t)blockIdx.x * blockDim.x + t, gs = (size_t)gridDim.x * blockDim.x;
    const unsigned sent = s_pre[r][E - 1];
    for (size_t s = gt; s < n; s += gs) {
      const long long pair = a.order[s];
      if (pair < 0 || (size_t)pair >= n) continue;
      long long row = -1, to = -1;
      if (s < sent) {
        int lo = 0, hi = E - 1;                      // the first expert whose prefix passes s
        while (lo < hi) {
          const int mid = (lo + hi) >> 1;
          if (s_pre[r][mid] > s) hi = mid;
          else lo = mid + 1;
        }
        const size_t at = (size_t)s_base[lo] + (s - (lo ? s_pre[r][lo - 1] : 0u));
        if (at < a.out_rows) {
          row = (long long)at;
          to = lo / L;
        }
      }
      a.pos[pair] = row;
      a.dest[pair] = to;
    }
  }
  // 4. stage -> arrive -> wait -> pull, software-pipelined over the chunks of this CTA
  const size_t nch = s_nch;
  char* out = (char*)a.out;
  for (; ch < nch; ch += gridDim.x) {
    if (ch != blockIdx.x) b2_barrier_wait(c, e_cur, a.opcode);
    const size_t off = ch * a.chunk, end = off + a.chunk;
    for (int i = 0; i < E; ++i) {
      const int sg = (i + r) % E, q = sg % P;        // stagger peers across ranks
      const size_t s0 = (size_t)s_src[sg] * rb, s1 = s0 + (size_t)s_len[sg] * rb;
      const size_t lo = off > s0 ? off : s0, hi = end < s1 ? end : s1;
      if (lo < hi)
        b2_copy_bytes<true>(out + (size_t)s_dst[sg] * rb + (lo - s0), c.stage[q] + par + B2_MOE_HDR + lo, hi - lo);
    }
    const size_t nxt = ch + gridDim.x;
    if (nxt < nch) {
      stage(nxt);
      b2_barrier_arrive(c, ++e);
      e_cur = e;
    }
  }
  // 5. rows past the filled ones are zero: the output is fully written on every call
  a2av_zero(out, s_filled * rb, a.out_rows * rb);
  b2_staged_end(c, e);
}

// ---------------------------------------------------------------------------
// combine
// ---------------------------------------------------------------------------
struct B2MoeCombineArgs {
  const void* in;
  void* out;
  const long long* pos;            // [tokens x k]
  const long long* dest;           // [tokens x k]
  const float* weights;            // [tokens x k] or null
  const long long* recv_counts;    // [n_counts]
  size_t row_bytes;
  size_t in_rows;
  size_t tokens;
  size_t chunk;
  int n_counts;
  int k;
  int pairs;
  int opcode;
};

namespace {

template <typename A> __device__ __forceinline__ A moe_mul(A a, A b);
template <> __device__ __forceinline__ float moe_mul(float a, float b) { return __fmul_rn(a, b); }
template <> __device__ __forceinline__ double moe_mul(double a, double b) { return __dmul_rn(a, b); }
template <typename A> __device__ __forceinline__ A moe_add(A a, A b);
template <> __device__ __forceinline__ float moe_add(float a, float b) { return __fadd_rn(a, b); }
template <> __device__ __forceinline__ double moe_add(double a, double b) { return __dadd_rn(a, b); }

// W bytes of a row as raw bits (W = 16: one vector; otherwise one element)
template <int W> struct MoeWord;
template <> struct MoeWord<16> { using type = uint4; };
template <> struct MoeWord<8> { using type = unsigned long long; };
template <> struct MoeWord<4> { using type = unsigned; };
template <> struct MoeWord<2> { using type = unsigned short; };
template <int W> __device__ __forceinline__ typename MoeWord<W>::type moe_load(const char* p) {
  using U = typename MoeWord<W>::type;
  if constexpr (W == 16) return b2_ld_peer16(p);
  else return *(const volatile U*)p;
}
template <int W> __device__ __forceinline__ void moe_store(char* p, typename MoeWord<W>::type v) {
  using U = typename MoeWord<W>::type;
  if constexpr (W == 16) b2_st16(p, v);
  else *(U*)p = v;
}

// Work item (token tk, W-byte piece at byte `at` of its row): fold or (pairs mode) copy its k pairs.
template <typename T, int W>
__device__ __forceinline__ void moe_combine_item(const B2DevComm& c, const B2MoeCombineArgs& a, size_t par,
                                                 size_t tk, size_t at) {
  constexpr int N = W / (int)sizeof(T);
  using A = typename B2Traits<T>::Acc;
  char* out = (char*)a.out;
  const int k = a.k;
  A acc[N];
  bool started = false;
  for (int j0 = 0; j0 < k; j0 += MOE_BATCH) {
    typename MoeWord<W>::type raw[MOE_BATCH];
    bool have[MOE_BATCH];
#pragma unroll
    for (int u = 0; u < MOE_BATCH; ++u) {          // the batch's loads first, then its fold
      const size_t p = tk * (size_t)k + j0 + u;
      have[u] = false;
      if (j0 + u < k) {
        const long long d = a.dest[p], row = a.pos[p];
        have[u] = d >= 0 && d < c.size && row >= 0 && (size_t)row < a.in_rows;
        if (have[u]) raw[u] = moe_load<W>(c.stage[d] + par + (size_t)row * a.row_bytes + at);
      }
    }
#pragma unroll
    for (int u = 0; u < MOE_BATCH; ++u) {
      if (j0 + u >= k) break;
      const size_t p = tk * (size_t)k + j0 + u;
      if (a.pairs) {                                 // one output row per pair, zeros where it was dropped
        moe_store<W>(out + p * a.row_bytes + at, have[u] ? raw[u] : typename MoeWord<W>::type{});
        continue;
      }
      if (!have[u]) continue;
      T v[N];
      memcpy(v, &raw[u], W);
      const bool weighted = a.weights != nullptr;
      const A w = weighted ? (A)a.weights[p] : (A)1;
#pragma unroll
      for (int i = 0; i < N; ++i) {
        A x = B2Traits<T>::up(v[i]);
        if (weighted) x = moe_mul<A>(w, x);
        acc[i] = started ? moe_add<A>(acc[i], x) : x;   // the first product starts the sum (-0 keeps its sign)
      }
      started = true;
    }
  }
  if (a.pairs) return;
  T o[N];
#pragma unroll
  for (int i = 0; i < N; ++i) o[i] = started ? B2Traits<T>::down(acc[i]) : B2Traits<T>::down((A)0);
  typename MoeWord<W>::type b;
  memcpy(&b, o, W);
  moe_store<W>(out + tk * a.row_bytes + at, b);
}

}  // namespace

template <typename T>
__global__ void __launch_bounds__(B2_THREADS, 1)
b2_k_moe_combine(const __grid_constant__ B2DevComm c, const __grid_constant__ B2MoeCombineArgs a) {
  __shared__ size_t s_fill;
  auto [par, e] = b2_staged_begin(c);
  const unsigned gen = b2_ticket_read(c.ticket) + 1u;
  const int t = threadIdx.x;
  // 1. the filled rows (the sum of the counts, clamped to the rows there are) -> staging
  if (t < 32) {
    unsigned long long s = 0;
    for (int i = t; i < a.n_counts; i += 32) {
      const long long v = a.recv_counts[i];
      s += v > 0 ? (unsigned long long)v : 0ull;
    }
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (t == 0) s_fill = (size_t)(s < a.in_rows ? s : a.in_rows);
  }
  __syncthreads();
  const size_t bytes = s_fill * a.row_bytes;
  char* mine = c.stage[c.rank] + par;
  for (size_t ch = blockIdx.x; ch * a.chunk < bytes; ch += gridDim.x)
    b2_copy_bytes<false>(mine + ch * a.chunk, (const char*)a.in + ch * a.chunk, b2_chunk_len(bytes, a.chunk, ch));
  // 2. full barrier: CTA b of every rank has staged (block-paired), then so has every CTA (grid-wide)
  b2_barrier_all(c, ++e, a.opcode);
  b2_grid_wait(c, c.ticket + TK_GRID, gen, a.opcode);
  // 3. pull and fold, grid-stride over (token or pair, piece of a row)
  const size_t gt = (size_t)blockIdx.x * blockDim.x + t, gs = (size_t)gridDim.x * blockDim.x;
  const size_t rows = a.tokens;
  const bool vec = ((a.row_bytes | (uintptr_t)a.out) & 15) == 0;
  const size_t per = vec ? a.row_bytes / 16 : a.row_bytes / sizeof(T);
  for (size_t it = gt; it < rows * per; it += gs) {
    const size_t tk = it / per, piece = it - tk * per;
    if (vec) moe_combine_item<T, 16>(c, a, par, tk, piece * 16);
    else moe_combine_item<T, (int)sizeof(T)>(c, a, par, tk, piece * sizeof(T));
  }
  b2_staged_end(c, e);
}

// ---------------------------------------------------------------------------
// host entry points
// ---------------------------------------------------------------------------
extern "C" int b2_moe_dispatch(B2Comm* c, const void* in, void* out, size_t row_bytes, size_t n_pairs, int k,
                               const long long* order, const long long* send_counts, int num_experts,
                               size_t out_rows, long long* recv_counts, long long* pos, long long* dest,
                               cudaStream_t stream) {
  B2DebugScope* dbg = b2_debug_begin(c, "Moe_dispatch", stream, "with %zu pairs of %zu bytes to %d experts", n_pairs,
                                     row_bytes, num_experts);
  const int P = c->dev.size;
  int rc = 0;
  if (num_experts < 1 || num_experts > B2_MOE_MAX_EXPERTS || num_experts % P != 0 || k < 1) {
    b2_set_error("moe_dispatch: %d experts on %d ranks (need a multiple of the ranks, at most %d) and k = %d",
                 num_experts, P, B2_MOE_MAX_EXPERTS, k);
    rc = B2_ERR_BAD_ARG;
  } else if ((order == nullptr && n_pairs > 0) || send_counts == nullptr || (pos == nullptr) != (dest == nullptr) ||
             (out == nullptr && out_rows > 0)) {
    b2_set_error("moe_dispatch: order (unless there are no pairs) and send_counts must be device arrays, pos and "
                 "dest both given or both null");
    rc = B2_ERR_BAD_ARG;
  } else if (n_pairs * (size_t)P > (size_t)INT_MAX || out_rows > (size_t)INT_MAX) {
    b2_set_error("moe_dispatch: %zu pairs on %d ranks or %zu output rows do not fit the 31-bit row counts", n_pairs,
                 P, out_rows);
    rc = B2_ERR_BAD_ARG;
  } else {
    B2MoeDispatchArgs a;
    memset(&a, 0, sizeof a);
    a.in = in; a.out = out; a.order = order; a.send_counts = send_counts;
    a.recv_counts = recv_counts; a.pos = pos; a.dest = dest;
    a.row_bytes = row_bytes; a.n_pairs = n_pairs; a.out_rows = out_rows; a.k = k; a.num_experts = num_experts;
    a.opcode = B2_OPC_MOE_DISPATCH;
    int grid;
    rc = b2_plan_staged(c, a.opcode, n_pairs * row_bytes, (const void*)b2_k_moe_dispatch, "moe_dispatch", &a.chunk,
                        &grid);
    if (rc == 0) {
      b2_k_moe_dispatch<<<grid, B2_THREADS, 0, stream>>>(c->dev, a);
      rc = b2_launched(c, "moe_dispatch");
    }
  }
  b2_debug_end(dbg, rc);
  return rc;
}

typedef void (*b2_moe_combine_kernel)(const B2DevComm, const B2MoeCombineArgs);
static b2_moe_combine_kernel moe_combine_kernel(int dtype) {
  switch (dtype) {
    case B2_F32: return b2_k_moe_combine<float>;
    case B2_F64: return b2_k_moe_combine<double>;
    case B2_F16: return b2_k_moe_combine<__half>;
    case B2_BF16: return b2_k_moe_combine<__nv_bfloat16>;
    default: return nullptr;
  }
}

extern "C" int b2_moe_combine(B2Comm* c, const void* in, void* out, size_t row_bytes, size_t in_rows, size_t tokens,
                              int k, const long long* pos, const long long* dest, const float* weights,
                              const long long* recv_counts, int n_counts, int dtype, int pairs,
                              cudaStream_t stream) {
  B2DebugScope* dbg = b2_debug_begin(c, "Moe_combine", stream, "with %zu tokens x %d pairs of %zu bytes", tokens, k,
                                     row_bytes);
  const b2_moe_combine_kernel kern = moe_combine_kernel(dtype);
  int rc = 0;
  if (kern == nullptr) {
    b2_set_error("moe_combine: rows must be float32, float64, float16 or bfloat16 (dtype %d)", dtype);
    rc = B2_ERR_BAD_ARG;
  } else if (k < 1 || row_bytes % b2_dtype_size(dtype) != 0 || ((pos == nullptr || dest == nullptr) && tokens > 0) ||
             recv_counts == nullptr || n_counts < 0) {
    b2_set_error("moe_combine: k = %d, %zu-byte rows of dtype %d, and pos, dest and recv_counts device arrays", k,
                 row_bytes, dtype);
    rc = B2_ERR_BAD_ARG;
  } else {
    B2MoeCombineArgs a;
    memset(&a, 0, sizeof a);
    a.in = in; a.out = out; a.pos = pos; a.dest = dest; a.weights = pairs ? nullptr : weights;
    a.recv_counts = recv_counts; a.n_counts = n_counts;
    a.row_bytes = row_bytes; a.in_rows = in_rows; a.tokens = pairs ? tokens * (size_t)k : tokens;
    a.k = pairs ? 1 : k; a.pairs = pairs != 0; a.opcode = B2_OPC_MOE_COMBINE;
    int grid;
    rc = b2_plan_staged(c, a.opcode, in_rows * row_bytes, (const void*)kern, "moe_combine", &a.chunk, &grid);
    if (rc == 0) {
      kern<<<grid, B2_THREADS, 0, stream>>>(c->dev, a);
      rc = b2_launched(c, "moe_combine");
    }
  }
  b2_debug_end(dbg, rc);
  return rc;
}
