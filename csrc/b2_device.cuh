// mpi4jax_b200 -- device-side building blocks shared by every kernel:
//   * system-scope acquire/release accessors for flags that live in peer HBM
//   * the %globaltimer watchdog of every spin wait (deadlock -> diagnostics + trap,
//     the analogue of the reference's abort_on_error, mpi_ops_common.h:60-78) and
//     the spin-waits on one flag word
//   * the flag-in-data word ({value, flag} as one 8-byte store) and its poll
//   * the last-arrival counter (the last CTA of a launch to finish does the epilogue)
//   * the block-paired cross-GPU barrier (CTA b on every rank <-> CTA b)
//   * the per-kernel ticket (staging parity + unique flag values, advanced on
//     the device so CUDA-graph replays stay correct)
//   * 16-byte vector movers and the typed reduction functors (10 ops x 17 dtypes,
//     fp32 accumulation for f16/bf16 and the two float8 formats)
#pragma once

#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include "b2_common.h"

#define B2_THREADS 512

// ---------------------------------------------------------------------------
// memory-model helpers
// ---------------------------------------------------------------------------
__device__ __forceinline__ void b2_st_release_sys(unsigned* p, unsigned v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void b2_st_relaxed_sys(unsigned* p, unsigned v) {
  asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned b2_ld_acquire_sys(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ unsigned b2_ld_relaxed_sys(const unsigned* p) {
  unsigned v;
  asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ unsigned b2_ld_volatile(const unsigned* p) {
  unsigned v;
  asm volatile("ld.volatile.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void b2_st_volatile(unsigned* p, unsigned v) {
  asm volatile("st.volatile.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void b2_fence_sys() { asm volatile("fence.acq_rel.sys;" ::: "memory"); }

// 16-byte accessors.  Peer data is read with strong.sys loads (no stale L1 line
// can be returned) and written with plain 16-byte stores.
__device__ __forceinline__ uint4 b2_ld_peer16(const void* p) {
  uint4 v;
  asm volatile("ld.volatile.global.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p)
               : "memory");
  return v;
}
__device__ __forceinline__ uint4 b2_ld_stream16(const void* p) {
  uint4 v;
  asm volatile("ld.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p));
  return v;
}
__device__ __forceinline__ void b2_st16(void* p, uint4 v) {
  asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z),
               "r"(v.w)
               : "memory");
}
__device__ __forceinline__ void b2_st16_sys(void* p, uint4 v) {
  asm volatile("st.relaxed.sys.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y),
               "r"(v.z), "r"(v.w)
               : "memory");
}

__device__ __forceinline__ unsigned long long b2_gtime() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// ---------------------------------------------------------------------------
// watchdog: fatal diagnostics then trap (host side prints "r<rank> | ... aborting")
// ---------------------------------------------------------------------------
static __device__ __noinline__ void b2_fatal(const B2DevComm& c, int code, int opcode, int peer,
                                      unsigned expected, unsigned observed, int aux) {
  B2ErrorRecord* e = c.err;
  if (e != nullptr && atomicCAS((int*)&e->code, 0, code) == 0) {
    e->rank = c.rank;
    e->opcode = opcode;
    e->peer = peer;
    e->expected = expected;
    e->observed = observed;
    e->block = (int)blockIdx.x;
    e->aux = aux;
    __threadfence_system();
  }
  __trap();
}

// The watchdog of one spin wait: every PERIOD + 1 polls it reads %globaltimer; the first reading
// starts the wait.  The caller reports with its own b2_fatal arguments:
//   B2Watchdog<> wd;  while (!ready()) if (wd.expired(c)) b2_fatal(c, B2_ERR_TIMEOUT, ...);
// (Keep the counter test, the clock read and the timeout test nested as written: a form that
// returns early, or that computes the result into a flag, adds instructions to every kernel that spins.)
template <unsigned PERIOD = 0xfffu>
struct B2Watchdog {
  unsigned long long t0 = 0;
  unsigned spins = 0;
  __device__ __forceinline__ bool expired(const B2DevComm& c) {
    if ((++spins & PERIOD) == 0) {
      const unsigned long long now = b2_gtime();
      if (t0 == 0) t0 = now;
      else if (now - t0 > c.timeout_ns) return true;
    }
    return false;
  }
};

// Spin until `(int)(load(p) - want) >= 0` (monotone epochs, wrap-safe).
__device__ __forceinline__ void b2_wait_ge(const B2DevComm& c, const unsigned* p, unsigned want,
                                           int opcode, int peer) {
  unsigned v = b2_ld_acquire_sys(p);
  if ((int)(v - want) >= 0) return;
  B2Watchdog<> wd;
  while (true) {
    v = b2_ld_acquire_sys(p);
    if ((int)(v - want) >= 0) return;
    if (wd.expired(c)) b2_fatal(c, B2_ERR_TIMEOUT, opcode, peer, want, v, 0);
  }
}

// Spin until `load(p) == want` exactly (used where stale values may be larger).
__device__ __forceinline__ void b2_wait_eq(const B2DevComm& c, const unsigned* p, unsigned want,
                                           int opcode, int peer) {
  unsigned v = b2_ld_acquire_sys(p);
  if (v == want) return;
  B2Watchdog<> wd;
  while (true) {
    v = b2_ld_acquire_sys(p);
    if (v == want) return;
    if (wd.expired(c)) b2_fatal(c, B2_ERR_TIMEOUT, opcode, peer, want, v, 1);
  }
}

// ---------------------------------------------------------------------------
// flag-in-data ("LL") words: {value, flag} travels as ONE 8-byte store; 8-byte stores are single
// transactions, so a reader that sees the flag sees the value: no fence, no separate signal, one
// NVLink one-way latency.  Used by the halo exchanges (b2_halo_ll.cuh) and small p2p messages.
// ---------------------------------------------------------------------------
__device__ __forceinline__ void b2_ll_put(uint2* p, unsigned v, unsigned flag) {
  // no "memory" clobber: the value comes from registers and nothing in the kernel reads the
  // (remote) target, so the compiler stays free to overlap other loads with the push
  asm volatile("st.relaxed.sys.global.v2.u32 [%0], {%1, %2};" ::"l"(p), "r"(v), "r"(flag));
}
// Spin until the word at `p` carries `flag`; return its value.  opcode, peer, aux: the diagnostics.
__device__ __forceinline__ unsigned b2_ll_poll(const B2DevComm& c, const uint2* p, unsigned flag,
                                               int opcode, int peer, int aux) {
  unsigned v, f;
  B2Watchdog<> wd;
  while (true) {
    asm volatile("ld.volatile.global.v2.u32 {%0, %1}, [%2];" : "=r"(v), "=r"(f) : "l"(p) : "memory");
    if (f == flag) return v;
    if (wd.expired(c)) b2_fatal(c, B2_ERR_TIMEOUT, opcode, peer, flag, f, aux);
  }
}

// ---------------------------------------------------------------------------
// block-paired cross-GPU barrier.
// CTA b of this rank signals CTA b of every peer and waits for all of them.
// All threads of the CTA must call it.  `e` is the CTA's next epoch value.
// release/acquire at .sys scope + bar.sync make every write issued by the CTA
// before the barrier visible to the peers' CTAs after it.
// ---------------------------------------------------------------------------
__device__ __forceinline__ void b2_barrier_all(const B2DevComm& c, unsigned e, int opcode) {
  __syncthreads();
  const int t = threadIdx.x;
  if (t < c.size) {
    unsigned* remote =
        (unsigned*)(c.heap[t] + c.lay.flags_off) + (size_t)blockIdx.x * B2_MAX_RANKS + c.rank;
    b2_st_release_sys(remote, e);
    const unsigned* local =
        (const unsigned*)(c.heap[c.rank] + c.lay.flags_off) + (size_t)blockIdx.x * B2_MAX_RANKS + t;
    b2_wait_ge(c, local, e, opcode, t);
  }
  __syncthreads();
}

// The two halves of b2_barrier_all, for software pipelining: local work placed between the
// arrive and the wait (staging the next chunk, copying the previous one out) hides the NVLink
// round trip of the flags.  Epochs of one CTA must still be used in increasing order.
__device__ __forceinline__ void b2_barrier_arrive(const B2DevComm& c, unsigned e) {
  __syncthreads();
  const int t = threadIdx.x;
  if (t < c.size) {
    unsigned* remote =
        (unsigned*)(c.heap[t] + c.lay.flags_off) + (size_t)blockIdx.x * B2_MAX_RANKS + c.rank;
    b2_st_release_sys(remote, e);
  }
}
__device__ __forceinline__ void b2_barrier_wait(const B2DevComm& c, unsigned e, int opcode) {
  const int t = threadIdx.x;
  if (t < c.size) {
    const unsigned* local =
        (const unsigned*)(c.heap[c.rank] + c.lay.flags_off) + (size_t)blockIdx.x * B2_MAX_RANKS + t;
    b2_wait_ge(c, local, e, opcode, t);
  }
  __syncthreads();
}

// ---------------------------------------------------------------------------
// ticket: one value per kernel launch, identical on every CTA, advanced by the
// LAST CTA TO FINISH (so every CTA has already read it).  Lives in local device
// memory -> graph replays see fresh values without host involvement.
// Usage:  unsigned t = b2_ticket_read(ptr);  ...  b2_finish_bump(ptr, ctr, 1, gridDim.x);
// (staged kernels go through b2_staged_begin / b2_staged_end below)
// ---------------------------------------------------------------------------
__device__ __forceinline__ unsigned b2_ticket_read(const unsigned* ticket) {
  __shared__ unsigned s_ticket;
  if (threadIdx.x == 0) s_ticket = b2_ld_volatile(ticket);
  __syncthreads();
  return s_ticket;
}

// Thread 0 of each of `nblocks` CTAs calls once its CTA is done: fences the CTA's writes and counts
// its arrival in *ctr.  True in the last CTA to arrive, which has reset the counter for the next use.
__device__ __forceinline__ bool b2_last_arrival(unsigned* ctr, unsigned nblocks) {
  __threadfence();
  const bool last = atomicAdd(ctr, 1u) == nblocks - 1;
  if (last) b2_st_volatile(ctr, 0u);
  return last;
}

// Grid-wide wait of a launch whose CTAs are all resident at once (plan_staged's grid): returns in every CTA once
// all gridDim.x CTAs have called it.  ctr[0] counts the arrivals (zero between launches: the last arrival resets
// it) and the last arrival publishes `gen` in ctr[1]; `gen` must grow from launch to launch (the staged kernels
// pass their ticket + 1).  Writes a CTA made before the call, and what it acquired from peers, are visible to
// every CTA after it.  All threads call.
__device__ __forceinline__ void b2_grid_wait(const B2DevComm& c, unsigned* ctr, unsigned gen, int opcode) {
  __syncthreads();
  if (threadIdx.x == 0) {
    if (b2_last_arrival(ctr, gridDim.x)) b2_st_release_sys(ctr + 1, gen);
    else b2_wait_ge(c, ctr + 1, gen, opcode, -1);
  }
  __syncthreads();
}

// All threads call; adds `delta` to *target once every one of `nblocks` CTAs is done.
__device__ __forceinline__ void b2_finish_bump(unsigned* target, unsigned* ctr, unsigned delta,
                                               unsigned nblocks) {
  __syncthreads();
  if (threadIdx.x == 0 && b2_last_arrival(ctr, nblocks)) {
    b2_st_volatile(target, b2_ld_volatile(target) + delta);
    __threadfence();
  }
}

// ---------------------------------------------------------------------------
// staged launch: the protocol of every kernel that stages data and synchronises with the block-paired
// barriers.  The ticket's parity picks the staging half, so a launch (or graph replay) never writes
// staging that a peer may still be reading for the previous one; the CTA's epochs continue where its
// previous launch stopped.  All threads call both:
//   auto [par, e] = b2_staged_begin(c);  ... b2_barrier_all(c, ++e, ...) ...  b2_staged_end(c, e);
// A kernel forms its own staging pointer, c.stage[c.rank] + par: formed in here, it changes the
// register allocation of b2_k_rowsv and b2_k_reduce_root_nvls.
// ---------------------------------------------------------------------------
struct B2Staged {
  size_t par;    // byte offset of this launch's staging half (into any rank's c.stage, and c.stage_mc)
  unsigned e;    // the CTA's last barrier epoch
};
__device__ __forceinline__ B2Staged b2_staged_begin(const B2DevComm& c) {
  B2Staged s;
  s.par = (size_t)(b2_ticket_read(c.ticket) & 1u) * c.stage_half;
  s.e = b2_ld_volatile(c.epoch + blockIdx.x);
  return s;
}
// `e`: the CTA's last epoch.  The last CTA to finish advances the ticket.
__device__ __forceinline__ void b2_staged_end(const B2DevComm& c, unsigned e) {
  __syncthreads();
  if (threadIdx.x == 0) b2_st_volatile(c.epoch + blockIdx.x, e);
  b2_finish_bump(c.ticket, c.ticket + 1, 1u, gridDim.x);
}

// Bytes of chunk `ch` of a `total`-byte payload cut into `chunk`-byte chunks; chunk ch starts at byte
// ch * chunk, which must be below `total`.
__device__ __forceinline__ size_t b2_chunk_len(size_t total, size_t chunk, size_t ch) {
  return total - ch * chunk < chunk ? total - ch * chunk : chunk;
}

// ---------------------------------------------------------------------------
// byte movers (CTA-cooperative).  Fast path: both pointers 16-byte aligned.
// ---------------------------------------------------------------------------
template <bool PEER_SRC>
__device__ __forceinline__ uint4 b2_ld16(const void* p) {
  if (PEER_SRC) return b2_ld_peer16(p);
  return b2_ld_stream16(p);
}

template <bool PEER_SRC>
__device__ __forceinline__ void b2_copy_bytes(void* __restrict__ dst, const void* __restrict__ src,
                                              size_t n) {
  if (n == 0) return;
  const int t = threadIdx.x, nt = blockDim.x;
  if ((((uintptr_t)dst | (uintptr_t)src) & 15) == 0) {
    const size_t nv = n >> 4;
    const char* s = (const char*)src;
    char* d = (char*)dst;
    size_t i = t;
    for (; i + 3 * (size_t)nt < nv; i += 4 * (size_t)nt) {
      uint4 v0 = b2_ld16<PEER_SRC>(s + (i << 4));
      uint4 v1 = b2_ld16<PEER_SRC>(s + ((i + nt) << 4));
      uint4 v2 = b2_ld16<PEER_SRC>(s + ((i + 2 * (size_t)nt) << 4));
      uint4 v3 = b2_ld16<PEER_SRC>(s + ((i + 3 * (size_t)nt) << 4));
      b2_st16(d + (i << 4), v0);
      b2_st16(d + ((i + nt) << 4), v1);
      b2_st16(d + ((i + 2 * (size_t)nt) << 4), v2);
      b2_st16(d + ((i + 3 * (size_t)nt) << 4), v3);
    }
    for (; i < nv; i += nt) b2_st16(d + (i << 4), b2_ld16<PEER_SRC>(s + (i << 4)));
    const size_t tail = n & 15;
    if ((size_t)t < tail) {
      const volatile unsigned char* sb = (const volatile unsigned char*)src + (nv << 4);
      ((unsigned char*)dst)[(nv << 4) + t] = sb[t];
    }
  } else {
    const volatile unsigned char* sb = (const volatile unsigned char*)src;
    unsigned char* db = (unsigned char*)dst;
    for (size_t i = t; i < n; i += nt) db[i] = sb[i];
  }
}

// ---------------------------------------------------------------------------
// typed reductions
// ---------------------------------------------------------------------------
struct b2_c64 { float re, im; };
struct b2_c128 { double re, im; };
struct b2_boolean { unsigned char v; };   // tag type: logical semantics on bytes

template <typename T> struct B2Traits {
  using Acc = T;
  static __device__ __forceinline__ Acc up(T v) { return v; }
  static __device__ __forceinline__ T down(Acc v) { return v; }
};
template <> struct B2Traits<__half> {
  using Acc = float;
  static __device__ __forceinline__ Acc up(__half v) { return __half2float(v); }
  static __device__ __forceinline__ __half down(Acc v) { return __float2half_rn(v); }
};
template <> struct B2Traits<__nv_bfloat16> {
  using Acc = float;
  static __device__ __forceinline__ Acc up(__nv_bfloat16 v) { return __bfloat162float(v); }
  static __device__ __forceinline__ __nv_bfloat16 down(Acc v) { return __float2bfloat16_rn(v); }
};
template <> struct B2Traits<b2_boolean> {
  using Acc = unsigned char;
  static __device__ __forceinline__ Acc up(b2_boolean v) { return v.v != 0 ? 1 : 0; }
  static __device__ __forceinline__ b2_boolean down(Acc v) { b2_boolean r; r.v = v; return r; }
};

// Hopper's float8 formats (tag types: the byte is the value).  Widening is exact: e4m3 through the hardware
// f16x2 conversion, e5m2 as the top byte of an f16; the sign bit is or-ed back in, because the e4m3 conversion
// makes every NaN the positive f16 NaN.  Narrowing is the hardware's round-to-nearest-even with satfinite
// (one F2FP per pair), then a compare-select turns its clamp into torch's Tensor.to(float8) overflow:
// e4m3fn |x| > 464, inf and NaN -> NaN; e5m2 |x| >= 61440 and inf -> inf, NaN -> NaN; the sign kept.
struct b2_f8e4m3 { unsigned char v; };
struct b2_f8e5m2 { unsigned char v; };

template <typename F> struct B2F8;
template <> struct B2F8<b2_f8e4m3> {
  static __device__ __forceinline__ unsigned up2(unsigned short p) {     // two bytes -> f16x2
    unsigned h2;
    asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(h2) : "h"(p));
    return h2;
  }
  static __device__ __forceinline__ unsigned short down2(float lo, float hi) {
    unsigned short p;
    asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(p) : "f"(hi), "f"(lo));
    return p;
  }
  static __device__ __forceinline__ unsigned fix(float x, unsigned b) {
    return fabsf(x) <= 464.f ? b : ((__float_as_uint(x) >> 24) & 0x80u) | 0x7Fu;
  }
};
template <> struct B2F8<b2_f8e5m2> {
  static __device__ __forceinline__ unsigned up2(unsigned short p) { return __byte_perm(p, 0u, 0x1404); }
  static __device__ __forceinline__ unsigned short down2(float lo, float hi) {
    unsigned short p;
    asm("cvt.rn.satfinite.e5m2x2.f32 %0, %1, %2;" : "=h"(p) : "f"(hi), "f"(lo));
    return p;
  }
  static __device__ __forceinline__ unsigned fix(float x, unsigned b) {
    return fabsf(x) < 61440.f ? b : ((__float_as_uint(x) >> 24) & 0x80u) | (x != x ? 0x7Fu : 0x7Cu);
  }
};
// bytes 0 and 1 of `w` (k = 0) or 2 and 3 (k = 1), widened
template <typename F>
__device__ __forceinline__ float2 b2_f8x2_up(unsigned w, int k) {
  const unsigned h2 = B2F8<F>::up2((unsigned short)(w >> (16 * k)));
  const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&h2));
  return make_float2(__uint_as_float(__float_as_uint(f.x) | ((w << (24 - 16 * k)) & 0x80000000u)),
                     __uint_as_float(__float_as_uint(f.y) | ((w << (16 - 16 * k)) & 0x80000000u)));
}
template <typename F>
__device__ __forceinline__ unsigned b2_f8x2_down(float lo, float hi) {
  const unsigned p = B2F8<F>::down2(lo, hi);
  return B2F8<F>::fix(lo, p & 0xFFu) | (B2F8<F>::fix(hi, p >> 8) << 8);
}
template <> struct B2Traits<b2_f8e4m3> {
  using Acc = float;
  static __device__ __forceinline__ Acc up(b2_f8e4m3 v) { return b2_f8x2_up<b2_f8e4m3>(v.v, 0).x; }
  static __device__ __forceinline__ b2_f8e4m3 down(Acc v) {
    b2_f8e4m3 r; r.v = (unsigned char)b2_f8x2_down<b2_f8e4m3>(v, 0.f); return r;
  }
};
template <> struct B2Traits<b2_f8e5m2> {
  using Acc = float;
  static __device__ __forceinline__ Acc up(b2_f8e5m2 v) { return b2_f8x2_up<b2_f8e5m2>(v.v, 0).x; }
  static __device__ __forceinline__ b2_f8e5m2 down(Acc v) {
    b2_f8e5m2 r; r.v = (unsigned char)b2_f8x2_down<b2_f8e5m2>(v, 0.f); return r;
  }
};
template <typename T> struct b2_is_fp8 { static constexpr bool value = false; };
template <> struct b2_is_fp8<b2_f8e4m3> { static constexpr bool value = true; };
template <> struct b2_is_fp8<b2_f8e5m2> { static constexpr bool value = true; };

template <typename A> struct b2_is_complex { static constexpr bool value = false; };
template <> struct b2_is_complex<b2_c64> { static constexpr bool value = true; };
template <> struct b2_is_complex<b2_c128> { static constexpr bool value = true; };
template <typename A> struct b2_is_float { static constexpr bool value = false; };
template <> struct b2_is_float<float> { static constexpr bool value = true; };
template <> struct b2_is_float<double> { static constexpr bool value = true; };

template <int OP, typename A>
__device__ __forceinline__ A b2_apply(A a, A b) {
  if constexpr (b2_is_complex<A>::value) {
    A r;
    if constexpr (OP == B2_SUM) { r.re = a.re + b.re; r.im = a.im + b.im; }
    else { r.re = a.re * b.re - a.im * b.im; r.im = a.re * b.im + a.im * b.re; }
    return r;
  } else if constexpr (b2_is_float<A>::value) {
    if constexpr (OP == B2_SUM) return a + b;
    else if constexpr (OP == B2_PROD) return a * b;
    else if constexpr (OP == B2_MIN) return (b < a || b != b) ? b : a;   // NaN-propagating like numpy
    else return (b > a || b != b) ? b : a;
  } else {
    if constexpr (OP == B2_SUM) return (A)(a + b);
    else if constexpr (OP == B2_PROD) return (A)(a * b);
    else if constexpr (OP == B2_MIN) return b < a ? b : a;
    else if constexpr (OP == B2_MAX) return b > a ? b : a;
    else if constexpr (OP == B2_LAND) return (A)((a != 0) && (b != 0));
    else if constexpr (OP == B2_LOR) return (A)((a != 0) || (b != 0));
    else if constexpr (OP == B2_LXOR) return (A)((a != 0) != (b != 0));
    else if constexpr (OP == B2_BAND) return (A)(a & b);
    else if constexpr (OP == B2_BOR) return (A)(a | b);
    else return (A)(a ^ b);
  }
}

// A 16-byte vector viewed as N elements of T, accumulated in B2Traits<T>::Acc.
template <typename T> struct B2Vec {
  static constexpr int N = 16 / (int)sizeof(T);
  using Acc = typename B2Traits<T>::Acc;
  Acc a[N];
  __device__ __forceinline__ void load(uint4 v) {
    alignas(16) T tmp[N];
    *reinterpret_cast<uint4*>(tmp) = v;
#pragma unroll
    for (int i = 0; i < N; ++i) a[i] = B2Traits<T>::up(tmp[i]);
  }
  template <int OP> __device__ __forceinline__ void accumulate(uint4 v) {
    alignas(16) T tmp[N];
    *reinterpret_cast<uint4*>(tmp) = v;
#pragma unroll
    for (int i = 0; i < N; ++i) a[i] = b2_apply<OP, Acc>(a[i], B2Traits<T>::up(tmp[i]));
  }
  __device__ __forceinline__ uint4 store() const {
    alignas(16) T tmp[N];
#pragma unroll
    for (int i = 0; i < N; ++i) tmp[i] = B2Traits<T>::down(a[i]);
    return *reinterpret_cast<const uint4*>(tmp);
  }
};

// float8: 16 elements per vector, widened and narrowed in pairs (8 packed conversions each way).  `a` stays
// addressable per element for rsv_fold.
template <typename F> struct B2Vec8 {
  static constexpr int N = 16;
  using Acc = float;
  Acc a[N];
  __device__ __forceinline__ void load(uint4 v) {
    const unsigned w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float2 f = b2_f8x2_up<F>(w[i >> 1], i & 1);
      a[2 * i] = f.x;
      a[2 * i + 1] = f.y;
    }
  }
  template <int OP> __device__ __forceinline__ void accumulate(uint4 v) {
    const unsigned w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float2 f = b2_f8x2_up<F>(w[i >> 1], i & 1);
      a[2 * i] = b2_apply<OP, Acc>(a[2 * i], f.x);
      a[2 * i + 1] = b2_apply<OP, Acc>(a[2 * i + 1], f.y);
    }
  }
  __device__ __forceinline__ uint4 store() const {
    unsigned w[4];
#pragma unroll
    for (int j = 0; j < 4; ++j)
      w[j] = b2_f8x2_down<F>(a[4 * j], a[4 * j + 1]) | (b2_f8x2_down<F>(a[4 * j + 2], a[4 * j + 3]) << 16);
    return make_uint4(w[0], w[1], w[2], w[3]);
  }
};
template <> struct B2Vec<b2_f8e4m3> : B2Vec8<b2_f8e4m3> {};
template <> struct B2Vec<b2_f8e5m2> : B2Vec8<b2_f8e5m2> {};

// Store the first `nbytes` (<16) bytes of a vector to an arbitrary address.
__device__ __forceinline__ void b2_store_partial(void* dst, uint4 v, int nbytes) {
  alignas(16) unsigned char tmp[16];
  *reinterpret_cast<uint4*>(tmp) = v;
  unsigned char* d = (unsigned char*)dst;
  for (int i = 0; i < nbytes; ++i) d[i] = tmp[i];
}

// zero bytes [lo, hi) of `out`, spread over every thread of the grid
__device__ __forceinline__ void a2av_zero(char* out, size_t lo, size_t hi) {
  const size_t gt = (size_t)blockIdx.x * blockDim.x + threadIdx.x, gs = (size_t)gridDim.x * blockDim.x;
  if (lo >= hi) return;
  const size_t v0 = lo + ((16 - ((uintptr_t)(out + lo) & 15)) & 15);     // first 16-byte aligned byte
  const size_t tail = (uintptr_t)(out + hi) & 15;
  const size_t v1 = hi - tail;                                           // end of the aligned vectors
  if (hi - lo < 32 || v0 >= v1) {
    for (size_t i = lo + gt; i < hi; i += gs) out[i] = 0;
    return;
  }
  for (size_t i = lo + gt; i < v0; i += gs) out[i] = 0;
  for (size_t i = v0 + (gt << 4); i < v1; i += gs << 4) b2_st16(out + i, make_uint4(0, 0, 0, 0));
  for (size_t i = v1 + gt; i < hi; i += gs) out[i] = 0;
}
