// mpi4jax_b200 -- point-to-point send / recv / sendrecv over peer-mapped HBM.
//
// Replaces the reference's blocking MPI_Send / MPI_Recv / MPI_Sendrecv call
// sites (mpi4jax/_src/xla_bridge/mpi_ops_common.h:340-389 and the CUDA callers
// mpi_xla_bridge_cuda.cpp:650-827, each preceded by a full stream sync and,
// by default, D2H/H2D staging through pageable host memory).
//
// Transport: every directed pair (s -> d) owns a ring of B2_P2P_NSLOT slots in
// d's symmetric heap.  A message is cut into fragments of at most slot_bytes;
// fragment number fs of the pair uses slot fs % NSLOT.  Up to 64 CTAs ("lanes")
// cooperate on a message; lane l of the sender is paired with lane l of the
// receiver (both derive the lane count from the byte count):
//
//   sender lane l          : wait credit(slot)  -> push stripe l into d's slot (NVLink stores)
//                            -> hdr[slot][l] = {fs+1, tag, nbytes} as ONE 16-byte release store
//   receiver lane l        : wait hdr[slot][l].seq == fs+1 -> validate -> copy stripe to the
//                            user buffer -> last lane to finish releases ack[slot] = fs+1 to s
//
// The sender never waits for the receiver unless the ring is full (eager up to
// NSLOT x slot_bytes in flight, like MPI's eager protocol); larger messages
// stream through the ring with the two kernels running concurrently on the two
// GPUs.  sendrecv launches both roles in ONE kernel (disjoint CTA groups), so
// the exchange is deadlock-free for any size.  All sequence numbers live in
// device memory and are advanced by the kernels themselves: the ops are
// CUDA-graph capturable and never synchronise the host.  MPI semantics kept:
// tags (validated against the pair FIFO), ANY_TAG, ANY_SOURCE (device-side
// election over the P inbox heads), Status(source, tag, count), zero-byte
// messages, self-sends.  Tag matching: a receive with a tag takes the EARLIEST
// pending message of that source carrying the tag (MPI's non-overtaking rule);
// a message that fits one slot may thereby be received ahead of earlier
// messages with other tags (per-source bitmap of slots consumed out of order).
// Messages larger than a slot stream through the ring and can only be matched
// at the head of the pair's queue -- like MPI's rendezvous protocol, where the
// blocked sender would not have reached the later send either.
//
// Small messages (<= B2_P2P_LL_MAX bytes) travel flag-in-data: every 4-byte word is pushed as one
// 8-byte {word, seq + 1} store into the slot's LL area and the receiver polls the words themselves,
// so the header needs no release fence over the payload and the message costs ONE NVLink one-way
// latency (b2_ll_put / b2_ll_poll, the halo kernels' transport too).  Matching, tags, Status and
// credits are unchanged: the header is still written, its size field tells the receiver which format
// to read.
#include <cstring>

#include "b2_device.cuh"
#include "b2_runtime.h"

// p2p_ctl words
#define CTL_SEND_FIN 0     // finish counter, send role
#define CTL_RECV_FIN 1     // finish counter, recv role
#define CTL_ELECT 2        // any-source election word: (gen << 8) | source
#define CTL_GEN 3          // election generation
#define CTL_SLOT_DONE 8    // [NSLOT] per-slot receiver-lane completion counters
#define CTL_OOO 16         // [B2_MAX_RANKS] per-source bitmap: bit i = fragment head+i consumed out of order

struct B2P2PArgs {
  const void* sendbuf;
  size_t send_bytes;
  int dest;
  int send_tag;
  int send_lanes;      // 0 = no send role
  void* recvbuf;
  size_t recv_bytes;
  int source;          // -1 = ANY_SOURCE
  int recv_tag;        // -1 = ANY_TAG
  int recv_lanes;      // 0 = no recv role
  B2StatusRecord* status;
  int opcode;
  int anysource_scan;  // communicator option "p2p_anysource_scan" (see the election in p2p_recv_role)
};

// ---- flag-in-data transport of small messages ---------------------------------------------------
__device__ __forceinline__ bool p2p_is_ll(size_t nbytes) { return nbytes > 0 && nbytes <= B2_P2P_LL_MAX; }
__device__ __forceinline__ unsigned p2p_load_word(const char* src, size_t w, size_t nbytes) {
  const size_t b = w << 2;
  if (b + 4 <= nbytes && (((uintptr_t)src) & 3) == 0) return *reinterpret_cast<const unsigned*>(src + b);
  unsigned v = 0;
  for (size_t k = 0; k < 4 && b + k < nbytes; ++k) v |= (unsigned)(unsigned char)src[b + k] << (8 * k);
  return v;
}
__device__ __forceinline__ void p2p_store_word(char* dst, size_t w, size_t nbytes, unsigned v) {
  const size_t b = w << 2;
  if (b + 4 <= nbytes && (((uintptr_t)dst) & 3) == 0) { *reinterpret_cast<unsigned*>(dst + b) = v; return; }
  for (size_t k = 0; k < 4 && b + k < nbytes; ++k) dst[b + k] = (char)(v >> (8 * k));
}
// The 16-byte header {seq + 1, tag, bytes lo, bytes hi} travels as ONE vector store / load: a
// receiver that sees the sequence word sees tag and size of the same store (16-byte aligned vector
// accesses are single transactions on NVLink and in L2 -- what NCCL's LL128 protocol builds on).
// `release`: the payload of a slot message was written with plain stores before (flag-in-data
// messages need no ordering: their words carry the flag themselves).
__device__ __forceinline__ void p2p_hdr_put(unsigned* hdr, unsigned seq1, int tag, size_t nbytes, bool release) {
  const unsigned lo = (unsigned)(nbytes & 0xffffffffull), hi = (unsigned)((unsigned long long)nbytes >> 32);
  if (release)
    asm volatile("st.release.sys.global.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(hdr), "r"(seq1), "r"((unsigned)tag),
                 "r"(lo), "r"(hi) : "memory");
  else
    asm volatile("st.relaxed.sys.global.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(hdr), "r"(seq1), "r"((unsigned)tag),
                 "r"(lo), "r"(hi) : "memory");
}
// Matching reads headers with this plain volatile load, not an acquire: it orders nothing read later.
// Every lane matches for itself, a lane reads slot payload only after its own b2_wait_eq (acquire) on
// its header, flag-in-data words carry their own flags, and the elected source is published after a fence.
struct P2PHdr { unsigned seq1; int tag; unsigned long long nbytes; };
__device__ __forceinline__ P2PHdr p2p_hdr_get(const unsigned* hdr) {
  unsigned a, b, c2, d;
  asm volatile("ld.volatile.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(a), "=r"(b), "=r"(c2), "=r"(d) : "l"(hdr) : "memory");
  P2PHdr h;
  h.seq1 = a; h.tag = (int)b; h.nbytes = (unsigned long long)c2 | ((unsigned long long)d << 32);
  return h;
}

// ---- the ring of pair (s -> d): headers, slots and flag-in-data areas in d's heap (`dheap`), indexed by
// s; acks in s's heap (`sheap`), indexed by d ----
__device__ __forceinline__ unsigned* p2p_hdr(const B2DevComm& c, char* dheap, int s, unsigned slot, int lane) {
  return (unsigned*)(dheap + c.lay.p2p_hdr_off) + (((size_t)s * B2_P2P_NSLOT + slot) * B2_P2P_MAX_LANES + lane) * 4;
}
__device__ __forceinline__ char* p2p_slot(const B2DevComm& c, char* dheap, int s, unsigned slot) {
  return dheap + c.lay.p2p_slot_off + ((size_t)s * B2_P2P_NSLOT + slot) * c.lay.p2p_slot_bytes;
}
__device__ __forceinline__ uint2* p2p_ll(const B2DevComm& c, char* dheap, int s, unsigned slot) {
  return (uint2*)(dheap + c.lay.p2p_ll_off + ((size_t)s * B2_P2P_NSLOT + slot) * (2 * B2_P2P_LL_MAX));
}
__device__ __forceinline__ unsigned* p2p_ack(const B2DevComm& c, char* sheap, int d, unsigned slot) {
  return (unsigned*)(sheap + c.lay.p2p_ack_off) + (size_t)d * B2_P2P_NSLOT + slot;
}

__device__ __forceinline__ size_t p2p_nfrag(size_t nbytes, size_t slot_bytes) {
  return nbytes == 0 ? 1 : (nbytes + slot_bytes - 1) / slot_bytes;
}
// Fragment f of a message whose first fragment is number seq0: its number, slot, offset in the
// message and length, and the stripe [lo, hi) of it that lane `lane` of `lanes` moves.
struct P2PFrag { unsigned fs, slot; size_t off, len, lo, hi; };
__device__ __forceinline__ P2PFrag p2p_frag(size_t slot_bytes, size_t nbytes, unsigned seq0, size_t f, int lanes,
                                            int lane) {
  P2PFrag g;
  g.fs = seq0 + (unsigned)f;
  g.slot = g.fs % B2_P2P_NSLOT;
  g.off = f * slot_bytes;
  g.len = b2_chunk_len(nbytes, slot_bytes, f);
  size_t stripe = (g.len + lanes - 1) / lanes;
  stripe = (stripe + 15) & ~(size_t)15;
  g.lo = stripe * (size_t)lane;
  if (g.lo > g.len) g.lo = g.len;
  g.hi = g.lo + stripe;
  if (g.hi > g.len) g.hi = g.len;
  return g;
}

#define P2P_LL_WORDS_PER_THREAD ((B2_P2P_LL_MAX / 4 + B2_THREADS - 1) / B2_THREADS)

__device__ void p2p_send_role(const B2DevComm& c, const B2P2PArgs& a, int lane) {
  const size_t slot_bytes = c.lay.p2p_slot_bytes;
  const char* src = (const char*)a.sendbuf;
  char* dheap = c.heap[a.dest];
  const bool ll = p2p_is_ll(a.send_bytes);
  // flag-in-data message: fetch the payload BEFORE the sequence number and the credit are known --
  // the three memory round trips overlap instead of following each other (the message is latency)
  unsigned word[P2P_LL_WORDS_PER_THREAD];
  const size_t nw = ll ? (a.send_bytes + 3) >> 2 : 0;
  if (ll) {
#pragma unroll
    for (int k = 0; k < P2P_LL_WORDS_PER_THREAD; ++k) {
      const size_t w = (size_t)k * B2_THREADS + threadIdx.x;
      word[k] = w < nw ? p2p_load_word(src, w, a.send_bytes) : 0u;
    }
  }
  const unsigned seq0 = b2_ticket_read(c.p2p_send_seq + a.dest);
  const size_t nfrag = p2p_nfrag(a.send_bytes, slot_bytes);
  for (size_t f = 0; f < nfrag; ++f) {
    const P2PFrag g = p2p_frag(slot_bytes, a.send_bytes, seq0, f, a.send_lanes, lane);
    // credit: the previous occupant of this slot (fragment fs - NSLOT) has been consumed
    if (threadIdx.x == 0)
      b2_wait_ge(c, p2p_ack(c, c.heap[c.rank], a.dest, g.slot), g.fs + 1u - B2_P2P_NSLOT, a.opcode, a.dest);
    __syncthreads();
    if (ll) {
      uint2* area = p2p_ll(c, dheap, c.rank, g.slot);
#pragma unroll
      for (int k = 0; k < P2P_LL_WORDS_PER_THREAD; ++k) {
        const size_t w = (size_t)k * B2_THREADS + threadIdx.x;
        if (w < nw) b2_ll_put(area + w, word[k], g.fs + 1u);
      }
    } else {
      b2_copy_bytes<false>(p2p_slot(c, dheap, c.rank, g.slot) + g.lo, src + g.off + g.lo, g.hi - g.lo);
      __syncthreads();
    }
    if (threadIdx.x == 0)
      p2p_hdr_put(p2p_hdr(c, dheap, c.rank, g.slot, lane), g.fs + 1u, a.send_tag, a.send_bytes, !ll);
  }
  if (a.send_lanes == 1) {
    // the only CTA of the role knows the new value: no counter, no reload (kernel boundaries order it)
    if (threadIdx.x == 0) b2_st_volatile(c.p2p_send_seq + a.dest, seq0 + (unsigned)nfrag);
  } else {
    b2_finish_bump(c.p2p_send_seq + a.dest, c.p2p_ctl + CTL_SEND_FIN, (unsigned)nfrag, (unsigned)a.send_lanes);
  }
}

// One pass over the window of source `src`: the `window` fragments from `head`, minus those consumed
// out of order (bitmap `ooo`), read through the lane-0 headers (every message has one).  It stops
// at the first fragment that has not arrived, and at the first message with the tag (ANY_TAG: the
// head of the queue).  The pair state (head, bitmap) only changes when a receive kernel finishes
// and headers arrive in sequence order, so every lane that walks the window finds the same message.
enum { P2P_FOUND, P2P_NOT_YET, P2P_STREAMED_BEHIND };
struct P2PFound { int res; unsigned seq; P2PHdr hd; };   // seq, hd: the message with the tag, if any
__device__ P2PFound p2p_walk(const B2DevComm& c, int src, int tag, unsigned head, unsigned ooo, unsigned window) {
  P2PFound m;
  m.res = P2P_NOT_YET;
  unsigned i = 0;
  while (i < window) {
    if ((ooo >> i) & 1u) { ++i; continue; }            // already consumed out of order
    const unsigned sq = head + i;
    const P2PHdr hd = p2p_hdr_get(p2p_hdr(c, c.heap[c.rank], src, sq % B2_P2P_NSLOT, 0));
    if (hd.seq1 != sq + 1u) break;                     // not here yet (nor anything behind it)
    const size_t nf = p2p_nfrag(hd.nbytes, c.lay.p2p_slot_bytes);
    if (tag < 0 || hd.tag == tag) {
      // a streamed message cannot overtake (see the file header)
      m.res = i == 0 || nf == 1 ? P2P_FOUND : P2P_STREAMED_BEHIND;
      m.seq = sq;
      m.hd = hd;
      break;
    }
    if (nf >= window - i) break;                       // its fragments fill the rest of the window
    i += (unsigned)nf;
  }
  return m;
}

// Sequence number of the first fragment of the message a receive (src, tag) consumes.  Executed by
// thread 0 of EVERY receiving lane.
__device__ unsigned p2p_match(const B2DevComm& c, const B2P2PArgs& a, int src, unsigned head, unsigned ooo,
                              P2PHdr* found) {
  B2Watchdog<0x3ffu> wd;
  while (true) {
    const P2PFound m = p2p_walk(c, src, a.recv_tag, head, ooo, B2_P2P_NSLOT);
    if (m.res == P2P_STREAMED_BEHIND)
      b2_fatal(c, B2_ERR_TAG_MISMATCH, a.opcode, src, (unsigned)a.recv_tag, (unsigned)m.hd.tag, 5);
    if (m.res == P2P_FOUND) {
      *found = m.hd;
      return m.seq;
    }
    if (wd.expired(c)) b2_fatal(c, B2_ERR_TIMEOUT, a.opcode, src, (unsigned)a.recv_tag, head, 6);
  }
}

__device__ void p2p_recv_role(const B2DevComm& c, const B2P2PArgs& a, int lane) {
  __shared__ int s_src, s_tag;
  __shared__ unsigned s_seq0, s_head, s_ooo, s_gen;
  const size_t slot_bytes = c.lay.p2p_slot_bytes;

  // ---- resolve the source (ANY_SOURCE: lane 0 elects, the others follow) ----
  if (threadIdx.x == 0) {
    int src = a.source;
    if (src < 0) {
      const unsigned gen = b2_ld_volatile(c.p2p_ctl + CTL_GEN) & 0xffffffu;
      if (lane == 0) {
        // The election probes the sources in turn for a message this receive may take now.  By default
        // it looks at each source's oldest pending message only (a window of one fragment: bit 0 of the
        // bitmap is never set at the head).  Communicator option "p2p_anysource_scan" = 1 looks as deep
        // into every source's window as a receive from a named source does; a streamed message behind
        // the head is "not here" then, since another source may match.  Both are mirrored by the model
        // in tests/_p2p_sim.py (Inbox).
        B2Watchdog<> wd;
        int probe = 0;
        while (src < 0) {
          const unsigned head = b2_ld_volatile(c.p2p_recv_seq + probe);
          const unsigned ooo = a.anysource_scan ? b2_ld_volatile(c.p2p_ctl + CTL_OOO + probe) : 0u;
          const unsigned window = a.anysource_scan ? B2_P2P_NSLOT : 1u;
          if (p2p_walk(c, probe, a.recv_tag, head, ooo, window).res == P2P_FOUND) {
            src = probe;
            break;
          }
          probe = (probe + 1) % c.size;
          if (wd.expired(c)) b2_fatal(c, B2_ERR_TIMEOUT, a.opcode, -1, 0, 0, 3);
        }
        __threadfence();
        b2_st_volatile(c.p2p_ctl + CTL_ELECT, (gen << 8) | (unsigned)src);
      } else {
        B2Watchdog<> wd;
        while (true) {
          const unsigned w = b2_ld_volatile(c.p2p_ctl + CTL_ELECT);
          if ((w >> 8) == gen) { src = (int)(w & 0xffu); break; }
          if (wd.expired(c)) b2_fatal(c, B2_ERR_TIMEOUT, a.opcode, -1, gen, w, 4);
        }
      }
    }
    s_src = src;
    // pair state: three independent loads in flight together (GEN is only needed for the final bump)
    s_head = b2_ld_volatile(c.p2p_recv_seq + src);
    s_ooo = b2_ld_volatile(c.p2p_ctl + CTL_OOO + src);
    s_gen = b2_ld_volatile(c.p2p_ctl + CTL_GEN);
    P2PHdr hd;
    s_seq0 = p2p_match(c, a, src, s_head, s_ooo, &hd);
    // the matched header is lane 0's header of the message's first fragment: check it once, here
    if (a.recv_tag >= 0 && hd.tag != a.recv_tag)
      b2_fatal(c, B2_ERR_TAG_MISMATCH, a.opcode, src, (unsigned)a.recv_tag, (unsigned)hd.tag, 0);
    if (hd.nbytes != (unsigned long long)a.recv_bytes)
      b2_fatal(c, B2_ERR_TRUNCATE, a.opcode, src, (unsigned)a.recv_bytes, (unsigned)hd.nbytes, 0);
    s_tag = hd.tag;
  }
  __syncthreads();
  const int src = s_src;
  const unsigned seq0 = s_seq0;
  const bool ll = p2p_is_ll(a.recv_bytes);

  const size_t nfrag = p2p_nfrag(a.recv_bytes, slot_bytes);
  char* dst = (char*)a.recvbuf;
  char* myheap = c.heap[c.rank];
  for (size_t f = 0; f < nfrag; ++f) {
    const P2PFrag g = p2p_frag(slot_bytes, a.recv_bytes, seq0, f, a.recv_lanes, lane);
    if (ll) {
      // flag-in-data: the words are polled themselves; nothing to wait for, nothing to fence
      const uint2* area = p2p_ll(c, myheap, src, g.slot);
      const size_t nw = (a.recv_bytes + 3) >> 2;
      for (size_t w = threadIdx.x; w < nw; w += blockDim.x)
        p2p_store_word(dst, w, a.recv_bytes, b2_ll_poll(c, area + w, g.fs + 1u, a.opcode, src, 7));
    } else {
      // this lane's stripe of the slot was written by the sender's lane of the same index: its header
      // (acquire) orders the payload loads
      if (threadIdx.x == 0) b2_wait_eq(c, p2p_hdr(c, myheap, src, g.slot, lane), g.fs + 1u, a.opcode, src);
      __syncthreads();
      b2_copy_bytes<true>(dst + g.off + g.lo, p2p_slot(c, myheap, src, g.slot) + g.lo, g.hi - g.lo);
    }
    __syncthreads();
    // credit back to the sender: every load of the slot has returned (their values were stored)
    if (threadIdx.x == 0) {
      unsigned* ack = p2p_ack(c, c.heap[src], c.rank, g.slot);
      if (a.recv_lanes == 1) {
        if (ll) b2_st_relaxed_sys(ack, g.fs + 1u);    // (the polled words were consumed: nothing left to order)
        else b2_st_release_sys(ack, g.fs + 1u);
      } else if (b2_last_arrival(c.p2p_ctl + CTL_SLOT_DONE + g.slot, (unsigned)a.recv_lanes)) {
        b2_st_release_sys(ack, g.fs + 1u);
      }
    }
  }
  if (threadIdx.x == 0 && lane == 0 && a.status != nullptr) {
    a.status->source = src;
    a.status->tag = s_tag;
    a.status->count_bytes = (long long)a.recv_bytes;
    a.status->error = 0;
    __threadfence_system();
    a.status->ready = 1;
  }
  // advance recv_seq[src] (+ election generation) once every lane is done
  bool last = a.recv_lanes == 1;
  if (!last) {
    __syncthreads();
    if (threadIdx.x == 0) last = b2_last_arrival(c.p2p_ctl + CTL_RECV_FIN, (unsigned)a.recv_lanes);
  }
  if (threadIdx.x == 0 && last) {
    // (head, ooo, gen as read at entry: the pair state only changes here, at the end of a receive)
    const unsigned head = s_head;
    unsigned ooo = s_ooo;
    if (seq0 == head) {
      // in order: advance past this message and past anything behind it that was already taken
      unsigned nh = head + (unsigned)nfrag;
      ooo = nfrag >= B2_P2P_NSLOT ? 0u : (ooo >> (unsigned)nfrag);
      while (ooo & 1u) { ooo >>= 1; ++nh; }
      b2_st_volatile(c.p2p_recv_seq + src, nh);
    } else {
      ooo |= 1u << (seq0 - head);                     // single-slot message taken ahead of the head
    }
    b2_st_volatile(c.p2p_ctl + CTL_OOO + src, ooo);
    b2_st_volatile(c.p2p_ctl + CTL_GEN, s_gen + 1u);
    __threadfence();
  }
}

__global__ void __launch_bounds__(B2_THREADS) b2_k_p2p(const B2DevComm c, const B2P2PArgs a) {
  if ((int)blockIdx.x < a.send_lanes) p2p_send_role(c, a, (int)blockIdx.x);
  else p2p_recv_role(c, a, (int)blockIdx.x - a.send_lanes);
}

// lane count: same function of the byte count on both sides of a message
static int lanes_for(const B2Comm* c, size_t nbytes) {
  size_t frag = nbytes < c->dev.lay.p2p_slot_bytes ? nbytes : c->dev.lay.p2p_slot_bytes;
  size_t lanes = (frag + 65535) / 65536;
  if (lanes < 1) lanes = 1;
  if (lanes > B2_P2P_MAX_LANES) lanes = B2_P2P_MAX_LANES;
  return (int)lanes;
}

static int launch_p2p(B2Comm* c, B2P2PArgs& a, const char* name, cudaStream_t stream) {
  const int P = c->dev.size;
  if (a.send_lanes > 0 && (a.dest < 0 || a.dest >= P)) {
    b2_set_error("%s: invalid destination rank %d (communicator size %d)", name, a.dest, P);
    return B2_ERR_BAD_ARG;
  }
  if (a.recv_lanes > 0 && (a.source < -1 || a.source >= P)) {
    b2_set_error("%s: invalid source rank %d (communicator size %d)", name, a.source, P);
    return B2_ERR_BAD_ARG;
  }
  a.anysource_scan = c->p2p_anysource_scan;
  b2_k_p2p<<<a.send_lanes + a.recv_lanes, B2_THREADS, 0, stream>>>(c->dev, a);
  return b2_launched(c, name);
}

extern "C" int b2_send(B2Comm* c, const void* buf, size_t nbytes, int dest, int tag,
                       cudaStream_t stream) {
  B2DebugScope* dbg = b2_debug_begin(c, "Send", stream, "%zu bytes to %d with tag %d", nbytes, dest, tag);
  B2P2PArgs a;
  memset(&a, 0, sizeof a);
  a.sendbuf = buf; a.send_bytes = nbytes; a.dest = dest; a.send_tag = tag;
  a.send_lanes = lanes_for(c, nbytes);
  a.opcode = B2_OPC_SEND;
  int rc = launch_p2p(c, a, "send", stream);
  b2_debug_end(dbg, rc);
  return rc;
}

extern "C" int b2_recv(B2Comm* c, void* buf, size_t nbytes, int source, int tag,
                       B2StatusRecord* status, cudaStream_t stream) {
  B2DebugScope* dbg = b2_debug_begin(c, "Recv", stream, "%zu bytes from %d with tag %d", nbytes, source, tag);
  B2P2PArgs a;
  memset(&a, 0, sizeof a);
  a.recvbuf = buf; a.recv_bytes = nbytes; a.source = source; a.recv_tag = tag;
  a.recv_lanes = lanes_for(c, nbytes);
  a.status = status;
  a.opcode = B2_OPC_RECV;
  int rc = launch_p2p(c, a, "recv", stream);
  b2_debug_end(dbg, rc);
  return rc;
}

extern "C" int b2_sendrecv(B2Comm* c, const void* sendbuf, size_t send_bytes, int dest, int sendtag,
                           void* recvbuf, size_t recv_bytes, int source, int recvtag,
                           B2StatusRecord* status, cudaStream_t stream) {
  B2DebugScope* dbg = b2_debug_begin(c, "Sendrecv", stream, "<%d (%zu bytes, tag %d) / >%d (%zu bytes, tag %d)",
                                     source, recv_bytes, recvtag, dest, send_bytes, sendtag);
  B2P2PArgs a;
  memset(&a, 0, sizeof a);
  a.sendbuf = sendbuf; a.send_bytes = send_bytes; a.dest = dest; a.send_tag = sendtag;
  a.send_lanes = lanes_for(c, send_bytes);
  a.recvbuf = recvbuf; a.recv_bytes = recv_bytes; a.source = source; a.recv_tag = recvtag;
  a.recv_lanes = lanes_for(c, recv_bytes);
  a.status = status;
  a.opcode = B2_OPC_SENDRECV;
  int rc = launch_p2p(c, a, "sendrecv", stream);
  b2_debug_end(dbg, rc);
  return rc;
}
