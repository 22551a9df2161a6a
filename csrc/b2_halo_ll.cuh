// mpi4jax_b200 -- flag-in-data ("LL") halo transport shared by the stand-alone exchange kernel
// (b2_halo.cu) and the deep exchange of the communication-avoiding shallow-water step (b2_swe_ca.cu).
//
// A halo element travels as one flag-in-data word {value, flag} (fz_put / fz_get over b2_ll_put /
// b2_ll_poll in b2_device.cuh): no fence, no separate signal, one NVLink one-way latency.
// flag = (messages sent on this side so far) + 1, buffer parity = that count & 1; both ends of
// a channel count the same messages in device memory (c.ticket[TK_RX + side] / [TK_TX + side]), so
// kernels using this transport can be mixed freely and replayed from CUDA graphs.
#pragma once

#include "b2_device.cuh"

enum { FS_W = 0, FS_E, FS_S, FS_N, FS_SW, FS_SE, FS_NW, FS_NE, FS_NSIDES };

__device__ __forceinline__ uint2* fz_buf(const B2DevComm& c, int rank, unsigned parity, int side) {
  return (uint2*)(c.heap[rank] + c.lay.halo_ll_off +
                  ((size_t)parity * FS_NSIDES + side) * c.lay.halo_ll_cap);
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
__device__ __forceinline__ void fz_finish(const B2DevComm& c, const int (&nb)[FS_NSIDES],
                                          const unsigned* s_rx, const unsigned* s_tx) {
  __syncthreads();
  if (threadIdx.x == 0 && b2_last_arrival(c.ticket + TK_FIN, gridDim.x)) {
    for (int k = 0; k < FS_NSIDES; ++k)
      if (nb[k] >= 0) {
        b2_st_volatile(c.ticket + TK_RX + k, s_rx[k] + 1u);
        b2_st_volatile(c.ticket + TK_TX + k, s_tx[k] + 1u);
      }
    __threadfence();
  }
}
