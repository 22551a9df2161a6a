// mpi4jax_b200 -- shallow-water stencil kernels (fp32), the compute side of the
// reference's demo application (examples/shallow_water.py:270-403).  The
// reference leaves this arithmetic to XLA (dozens of fused elementwise kernels
// plus pad / dynamic-update-slice copies per step, separated by 48 blocking MPI
// custom calls).  Here one model step is four stencil launches and three fused
// multi-field halo exchanges (b2_halo.cu):
//
//   K1 fluxes      (h,u,v)                 -> fe, fn, q, ke        [exchange fe,fn,q,ke]
//   K2 tendencies  (h,fe,fn,q,ke,d*_old)   -> dh,du,dv, h',u,v     [exchange h',u,v]
//   K34 friction-u (fluxes inline from u, incl. their halo) + friction-v flux -> u, fe2, fn2
//                                                                   [exchange fe2,fn2]
//   K5 friction-v apply                    -> v
//
// The physics, including the order of boundary updates, the edge-padded `hc`
// rows at the y walls and the `v - u` term of the second friction flux
// (shallow_water.py:387-392), follows the reference line by line so that the
// two programs integrate the same discrete system.  The redundant `hc` halo
// exchange of the reference (:278-279) is elided: after `enforce_boundaries(h)`
// at the end of the previous step, h's halo already holds exactly the values
// that exchange would deliver (see DESIGN.md, "shallow water").
//
// Memory layout / vectorisation: fields are (ny, pitch) with pitch a multiple of
// 4 floats, so every row starts 16-byte aligned.  One thread owns an aligned
// group of 4 cells: centre rows and the rows above/below are single 16-byte
// loads, only the two x-neighbours of the group are scalar loads (L1 hits).
// These kernels are pure streaming stencils (1 FLOP per ~2 bytes): the roofline
// is HBM bandwidth, there is no tensor-core work in this workload.
#include "b2_swe_body.cuh"

__global__ void __launch_bounds__(SWE_THREADS)
swe_k1_fluxes(B2SweParams p, const float* __restrict__ h, const float* __restrict__ u,
              const float* __restrict__ v, float* __restrict__ fe, float* __restrict__ fn,
              float* __restrict__ q, float* __restrict__ ke) {
  int j, i0;
  bool m[4];
  if (!swe_map(p, j, i0, m)) return;
  swe_k1_body(p, h, u, v, fe, fn, q, ke, j, i0, m);
}

__global__ void __launch_bounds__(SWE_THREADS, 3)
swe_k2_tendencies(B2SweParams p, const float* __restrict__ h, float* __restrict__ h_new,
                  float* __restrict__ u, float* __restrict__ v, float* __restrict__ dh,
                  float* __restrict__ du, float* __restrict__ dv, const float* __restrict__ fe,
                  const float* __restrict__ fn, const float* __restrict__ q,
                  const float* __restrict__ ke) {
  int j, i0;
  bool m[4];
  if (!swe_map(p, j, i0, m)) return;
  swe_k2_body(p, h, h_new, u, v, dh, du, dv, fe, fn, q, ke, j, i0, m);
}

__global__ void __launch_bounds__(SWE_THREADS)
swe_k34_friction_u(B2SweParams p, const float* __restrict__ u, float* __restrict__ u_new,
                   const float* __restrict__ v, float* __restrict__ fe2, float* __restrict__ fn2,
                   int has_south) {
  int j, i0 = -1;
  bool m[4];
  // also the group that holds only the east halo column (nx % 4 == 1): u_new's halo cells are copies
  // of u's, there as everywhere else
  if (!swe_map(p, j, i0, m) && i0 != p.nx - 1) return;
  swe_k34_body(p, u, u_new, v, fe2, fn2, j, i0, m, has_south != 0);
}

__global__ void __launch_bounds__(SWE_THREADS)
swe_k5_friction_v(B2SweParams p, float* __restrict__ v, const float* __restrict__ fe2,
                  const float* __restrict__ fn2) {
  int j, i0;
  bool m[4];
  if (!swe_map(p, j, i0, m)) return;
  swe_k5_body(p, v, fe2, fn2, j, i0, m);
}

extern "C" {

// One call = `nsteps` model steps (4 stencil launches + 3 fused halo exchanges each), all
// enqueued on `s` without touching the host again: the whole time loop of the reference's
// `do_multistep` (examples/shallow_water.py:406-411) becomes a launch sequence that CUDA-graph
// capture turns into a single replayable graph.  `h0`/`h1` ping-pong (their wall rows are
// initialised identically and never written); the state is returned in h0 (an odd step count
// ends with one device copy).
int b2_swe_multistep(B2Comm* c, const B2SweParams* p0, const B2SweState* st, const B2HaloDesc* topo,
                     int nsteps, int first_step, cudaStream_t s) {
  B2SweParams p = *p0;
  if (p.pitch % 4 != 0 || p.pitch < p.nx || p.ny < 3 || p.nx < 3) {
    b2_set_error("swe: need ny,nx >= 3 and a row pitch that is a multiple of 4 floats and >= nx "
                 "(got ny=%d nx=%d pitch=%d)", p.ny, p.nx, p.pitch);
    return B2_ERR_BAD_ARG;
  }
  // friction-u is out of place: u and u1 ping-pong
  if (p.viscosity > 0.f && st->u == st->u1) {
    b2_set_error("swe_friction_u_fused: u_new must not alias u (the update reads u's neighbours)");
    return B2_ERR_BAD_ARG;
  }
  const unsigned blocks = (unsigned)(((long long)(p.ny - 2) * (p.pitch / 4) + SWE_THREADS - 1) / SWE_THREADS);
  float* h = st->h0;
  float* hn = st->h1;
  float* u = st->u;
  float* un = st->u1;
  B2HaloDesc d = *topo;
  d.ny = p.ny;
  d.nx = p.nx;
  d.pitch = p.pitch;
  int rc = 0;
  for (int it = 0; it < nsteps && rc == 0; ++it) {
    p.first_step = (first_step && it == 0) ? 1 : 0;
    swe_k1_fluxes<<<blocks, SWE_THREADS, 0, s>>>(p, h, u, st->v, st->fe, st->fn, st->q, st->ke);
    if ((rc = b2_launched(c, "swe_fluxes"))) break;
    d.nfields = 4;
    d.field[0] = st->fe; d.kind[0] = 1;
    d.field[1] = st->fn; d.kind[1] = 2;
    d.field[2] = st->q;  d.kind[2] = 0;
    d.field[3] = st->ke; d.kind[3] = 0;
    if ((rc = b2_halo_exchange(c, &d, s))) break;
    swe_k2_tendencies<<<blocks, SWE_THREADS, 0, s>>>(p, h, hn, u, st->v, st->dh, st->du, st->dv,
                                                     st->fe, st->fn, st->q, st->ke);
    if ((rc = b2_launched(c, "swe_tendencies"))) break;
    d.nfields = 3;
    d.field[0] = hn;    d.kind[0] = 0;
    d.field[1] = u;     d.kind[1] = 1;
    d.field[2] = st->v; d.kind[2] = 2;
    if ((rc = b2_halo_exchange(c, &d, s))) break;
    if (p.viscosity > 0.f) {
      // friction-u fluxes are evaluated inline from u (incl. their halo, from u's fresh halo):
      // no K3 launch, no (fe, fn) exchange, no HBM round trip of the fluxes
      swe_k34_friction_u<<<blocks, SWE_THREADS, 0, s>>>(p, u, un, st->v, st->fe2, st->fn2, topo->south >= 0);
      if ((rc = b2_launched(c, "swe_friction_u_fused"))) break;
      { float* t = u; u = un; un = t; }
      d.nfields = 2;
      d.field[0] = st->fe2; d.kind[0] = 1;
      d.field[1] = st->fn2; d.kind[1] = 2;
      if ((rc = b2_halo_exchange(c, &d, s))) break;
      swe_k5_friction_v<<<blocks, SWE_THREADS, 0, s>>>(p, st->v, st->fe2, st->fn2);
      if ((rc = b2_launched(c, "swe_friction_v"))) break;
    }
    float* t = h; h = hn; hn = t;
  }
  const size_t bytes = (size_t)p.ny * p.pitch * sizeof(float);
  if (rc == 0 && u != st->u)
    rc = b2_cuda_check(cudaMemcpyAsync(st->u, u, bytes, cudaMemcpyDeviceToDevice, s), "swe_multistep: copy failed");
  if (rc == 0 && h != st->h0)
    rc = b2_cuda_check(cudaMemcpyAsync(st->h0, h, bytes, cudaMemcpyDeviceToDevice, s), "swe_multistep: copy failed");
  return rc;
}

}  // extern "C"
