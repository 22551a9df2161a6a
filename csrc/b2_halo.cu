// mpi4jax_b200 -- fused multi-field 2-D halo exchange.
//
// The reference's flagship workload (examples/shallow_water.py:172-264,
// `enforce_boundaries`) exchanges a 1-cell halo with up to four neighbours by
// issuing, per field, 2 sendrecv + 1 send + 1 recv custom calls, each of them a
// blocking MPI call behind a full stream synchronisation, with XLA gather /
// dynamic-update-slice kernels around them for the strided column pack and the
// halo unpack (48 custom calls per model step at 8 ranks, SURVEY.md section 3.4).
//
// Here ONE kernel launch exchanges the halos of up to B2_HALO_MAX_FIELDS fields
// with all EIGHT neighbours in a single phase: strided column pack, NVLink push
// straight into the neighbour's symmetric receive buffer, halo unpack and the
// physical wall conditions, all fused.
//
// Why eight neighbours: the reference's west/north/east/south message order
// makes every corner halo cell end up with the DIAGONAL neighbour's interior
// corner value (it travels through two hops: columns first, then rows carrying
// the fresh corner).  Sending that value directly from the diagonal rank gives
// bit-identical halos with one NVLink latency instead of two.  Where a rank
// touches a y wall the wall-row cells of the halo columns come from the W/E
// neighbours' wall rows, exactly as in the reference's sequence.
//
// Transport and kernel body: b2_halo_ll.cuh.  Every element is pushed as one 8-byte {value, flag}
// store and the receiver polls the data itself -- no release fence, no arrival counter, one NVLink
// one-way latency.  Receive buffers alternate on the device-side per-side message counters, so no
// "ready" handshake is needed and the kernel is CUDA-graph replayable.  The messages are the depth-1
// case of the deep exchange's (b2_halo_geom.h); what is particular to this kernel is the receive rule
// with the wall conditions and the closing wall pass.

#include "b2_device.cuh"
#include "b2_halo_ll.cuh"
#include "b2_runtime.h"

#define HALO_THREADS 256
#define HALO_LL_CTAS 16

__global__ void __launch_bounds__(HALO_THREADS) b2_k_halo_ll(const B2DevComm c, const B2HaloDesc d) {
  const size_t pitch = (size_t)d.pitch;
  const int jlo = (d.south >= 0) ? 1 : 0, jhi = (d.north >= 0) ? d.ny - 1 : d.ny;
  const bool uwall = !d.periodic_x && d.at_east_wall, vwall = d.at_north_wall;
  fz_exchange<1>(c, d, d.nfields, [&](int side, int e, float val) {
    halo_recv_walls(d.ny, d.nx, pitch, side, e, jlo, jhi, uwall, vwall, val, d.field, d.kind);
  });
  halo_wall_pass(d.ny, d.nx, pitch, d.nfields, jlo, jhi, (d.west >= 0) ? 1 : 0, (d.east >= 0) ? d.nx - 1 : d.nx,
                 uwall, vwall, d.field, d.kind, blockIdx.x * blockDim.x + threadIdx.x, gridDim.x * blockDim.x);
}

// halo_exchange / swe_ca: every neighbour rank is -1 (wall) or a rank of the communicator
int b2_halo_check_ranks(B2Comm* c, const B2HaloDesc* d, const char* what) {
  const int nb[HALO_NSIDES] = {d->west, d->east, d->south, d->north, d->sw, d->se, d->nw, d->ne};
  for (int k = 0; k < HALO_NSIDES; ++k)
    if (nb[k] < -1 || nb[k] >= c->dev.size) {
      b2_set_error("%s: invalid neighbour rank %d", what, nb[k]);
      return B2_ERR_BAD_ARG;
    }
  return 0;
}

// the longest message of an exchange of `nfields` fields, `depth` layers deep, fits one halo buffer
int b2_halo_check_cap(B2Comm* c, int nfields, int depth, int ny, int nx, const char* what) {
  const size_t need = (size_t)nfields * depth * (size_t)(ny > nx ? ny : nx) * sizeof(uint2);
  if (need > c->dev.lay.halo_ll_cap) {
    b2_set_error("%s: halo buffers too small (%zu > %zu); raise MPI4JAX_B200_HALO_BYTES", what, need,
                 c->dev.lay.halo_ll_cap);
    return B2_ERR_BAD_ARG;
  }
  return 0;
}

extern "C" int b2_halo_exchange(B2Comm* c, const B2HaloDesc* d, cudaStream_t stream) {
  if (d->nfields < 1 || d->nfields > B2_HALO_MAX_FIELDS) {
    b2_set_error("halo_exchange: nfields must be in [1, %d]", B2_HALO_MAX_FIELDS);
    return B2_ERR_BAD_ARG;
  }
  if (int rc = b2_halo_check_cap(c, d->nfields, 1, d->ny, d->nx, "halo_exchange")) return rc;
  if (d->pitch < d->nx) {
    b2_set_error("halo_exchange: pitch %d < nx %d", d->pitch, d->nx);
    return B2_ERR_BAD_ARG;
  }
  if (int rc = b2_halo_check_ranks(c, d, "halo_exchange")) return rc;
  // about one element per thread and side: the exchange is pure latency, so spread it wide
  const int mx = d->ny > d->nx ? d->ny : d->nx;
  int ctas = (d->nfields * mx + HALO_THREADS - 1) / HALO_THREADS;
  if (ctas < HALO_LL_CTAS) ctas = HALO_LL_CTAS;
  if (ctas > 96) ctas = 96;
  b2_k_halo_ll<<<ctas, HALO_THREADS, 0, stream>>>(c->dev, *d);
  return b2_launched(c, "halo_exchange");
}
