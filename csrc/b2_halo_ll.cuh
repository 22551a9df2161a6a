// mpi4jax_b200 -- flag-in-data ("LL") halo transport and the one push / poll body of the eight-side
// exchanges: the stand-alone exchange kernel (b2_halo.cu) and the deep exchange of the
// communication-avoiding shallow-water step (b2_swe_ca.cu).  Message geometry: b2_halo_geom.h.
//
// A halo element travels as one flag-in-data word {value, flag} (fz_put / fz_get over b2_ll_put /
// b2_ll_poll in b2_device.cuh): no fence, no separate signal, one NVLink one-way latency.
// flag = (messages sent on this side so far) + 1, buffer parity = that count & 1; both ends of
// a channel count the same messages in device memory (c.ticket[TK_RX + side] / [TK_TX + side]), so
// kernels using this transport can be mixed freely and replayed from CUDA graphs.
#pragma once

#include "b2_device.cuh"
#include "b2_halo_geom.h"
#include "b2_runtime.h"

__device__ __forceinline__ uint2* fz_buf(const B2DevComm& c, int rank, unsigned parity, int side) {
  return (uint2*)(c.heap[rank] + c.lay.halo_ll_off +
                  ((size_t)parity * HALO_NSIDES + side) * c.lay.halo_ll_cap);
}
// one halo element: a float as a flag-in-data word; a poll that times out reports the side (aux 5)
__device__ __forceinline__ void fz_put(uint2* p, float v, unsigned flag) {
  b2_ll_put(p, __float_as_uint(v), flag);
}
__device__ __forceinline__ float fz_get(const B2DevComm& c, const uint2* p, unsigned flag, int side) {
  return __uint_as_float(b2_ll_poll(c, p, flag, B2_OPC_HALO, side, 5));
}

// End of an exchange kernel: after every thread of the CTA is done, the last CTA to finish advances
// the per-side message counters of the sides that have a neighbour.
__device__ __forceinline__ void fz_finish(const B2DevComm& c, const int (&nb)[HALO_NSIDES],
                                          const unsigned* s_rx, const unsigned* s_tx) {
  __syncthreads();
  if (threadIdx.x == 0 && b2_last_arrival(c.ticket + TK_FIN, gridDim.x)) {
    for (int k = 0; k < HALO_NSIDES; ++k)
      if (nb[k] >= 0) {
        b2_st_volatile(c.ticket + TK_RX + k, s_rx[k] + 1u);
        b2_st_volatile(c.ticket + TK_TX + k, s_tx[k] + 1u);
      }
    __threadfence();
  }
}

// The exchange of `nf` fields, DEPTH layers deep, with every neighbour of d: one grid-stride loop pushes
// every element of every message straight from the arrays into the neighbour's receive buffer, a second
// polls every element that lands here and hands it to `recv(side, e, value)`.  Elements are numbered
// through all sides by a prefix of the message sizes.
template <int DEPTH, class Recv>
__device__ __forceinline__ void fz_exchange(const B2DevComm& c, const B2HaloDesc& d, const int nf, Recv recv) {
  __shared__ unsigned s_rx[HALO_NSIDES], s_tx[HALO_NSIDES];
  __shared__ int s_cnt[HALO_NSIDES + 1];
  const int gt = blockIdx.x * blockDim.x + threadIdx.x, gn = gridDim.x * blockDim.x;
  const int ny = d.ny, nx = d.nx;
  const size_t pitch = (size_t)d.pitch;
  const int nb[HALO_NSIDES] = {d.west, d.east, d.south, d.north, d.sw, d.se, d.nw, d.ne};
  if (threadIdx.x < HALO_NSIDES) {
    s_rx[threadIdx.x] = b2_ld_volatile(c.ticket + TK_RX + threadIdx.x);
    s_tx[threadIdx.x] = b2_ld_volatile(c.ticket + TK_TX + threadIdx.x);
  }
  if (threadIdx.x == 0) {
    int acc = 0;
    for (int k = 0; k < HALO_NSIDES; ++k) {
      s_cnt[k] = acc;
      if (nb[k] >= 0) acc += halo_msg_count(nf, DEPTH, ny, nx, k);     // |message towards k| == |landing on k|
    }
    s_cnt[HALO_NSIDES] = acc;
  }
  __syncthreads();
  const int total = s_cnt[HALO_NSIDES];
  for (int k = gt; k < total; k += gn) {
    int s = 0;
    while (k >= s_cnt[s + 1]) ++s;
    const int e = k - s_cnt[s], land = halo_opposite(s);
    int f, js, is, jr, ir, layer;
    halo_msg_elem(DEPTH, ny, nx, land, e, f, js, is, jr, ir, layer);
    fz_put(fz_buf(c, nb[s], s_tx[s] & 1u, land) + e, d.field[f][(size_t)js * pitch + is], s_tx[s] + 1u);
  }
  for (int k = gt; k < total; k += gn) {
    int s = 0;
    while (k >= s_cnt[s + 1]) ++s;
    const int e = k - s_cnt[s];
    recv(s, e, fz_get(c, fz_buf(c, c.rank, s_rx[s] & 1u, s) + e, s_rx[s] + 1u, s));
  }
  fz_finish(c, nb, s_rx, s_tx);
}
