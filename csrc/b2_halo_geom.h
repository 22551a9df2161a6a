// mpi4jax_b200 -- message geometry of the eight-side halo exchanges: the stand-alone one-layer exchange
// (b2_k_halo_ll, b2_halo.cu) and the deep exchange of the communication-avoiding step (b2_k_halo_ca,
// b2_swe_ca.cu).  Both run the one push / poll body of b2_halo_ll.cuh over these messages and differ
// only in the depth and in the receive rule.  Host-compilable (tests/native/swe_host_emu.cpp runs the
// kernels' own index code on the CPU).
//
// A message carries `depth` layers of `nf` fields; element e of the message that LANDS on receiver
// side `side` (HALO_W = it comes from the west neighbour, ...) maps to field f, the sender's cell
// (js, is), the receiver's cell (jr, ir) and the layer (0 = the main arrays' halo cell).  W / E
// messages are full height (rows 0 .. ny-1; at a y wall the wall-row values ride along), S / N messages
// cover the interior columns, corner messages are depth x depth blocks.  The elements of a message are
// contiguous in the receive buffer.
#pragma once

#include <cuda_runtime.h>

enum { HALO_W = 0, HALO_E, HALO_S, HALO_N, HALO_SW, HALO_SE, HALO_NW, HALO_NE, HALO_NSIDES };

// the side a message sent towards `side` lands on at the receiver
__host__ __device__ __forceinline__ int halo_opposite(int side) {
  const int opp[HALO_NSIDES] = {HALO_E, HALO_W, HALO_N, HALO_S, HALO_NE, HALO_NW, HALO_SE, HALO_SW};
  return opp[side];
}

__host__ __device__ inline int halo_msg_count(int nf, int depth, int ny, int nx, int side) {
  if (side <= HALO_E) return nf * depth * ny;
  if (side <= HALO_N) return nf * depth * (nx - 2);
  return nf * depth * depth;
}
__host__ __device__ inline void halo_msg_elem(int depth, int ny, int nx, int side, int e, int& f, int& js, int& is,
                                              int& jr, int& ir, int& layer) {
  if (side <= HALO_E) {
    f = e / (depth * ny);
    const int l = (e / ny) % depth, j = e % ny;
    layer = l; js = jr = j;
    if (side == HALO_W) { is = nx - 2 - l; ir = -l; }
    else                { is = 1 + l;      ir = nx - 1 + l; }
  } else if (side <= HALO_N) {
    const int n = nx - 2;
    f = e / (depth * n);
    const int l = (e / n) % depth, i = 1 + e % n;
    layer = l; is = ir = i;
    if (side == HALO_S) { js = ny - 2 - l; jr = -l; }
    else                { js = 1 + l;      jr = ny - 1 + l; }
  } else {
    f = e / (depth * depth);
    const int lj = (e / depth) % depth, li = e % depth;
    layer = lj > li ? lj : li;
    if (side == HALO_SW)      { js = ny - 2 - lj; is = nx - 2 - li; jr = -lj;         ir = -li; }
    else if (side == HALO_SE) { js = ny - 2 - lj; is = 1 + li;      jr = -lj;         ir = nx - 1 + li; }
    else if (side == HALO_NW) { js = 1 + lj;      is = nx - 2 - li; jr = ny - 1 + lj; ir = -li; }
    else                      { js = 1 + lj;      is = 1 + li;      jr = ny - 1 + lj; ir = nx - 1 + li; }
  }
}

// ---- receive rules ---------------------------------------------------------------------------------
// [jlo, jhi): the rows of the main halo columns the W / E messages fill -- all rows where the receiver
// touches a y wall, otherwise the corner rows come from the diagonal neighbours.

// Deep exchange: every layer into the ext arrays (W / E messages: interior rows only), layer 0 also into
// the main arrays' halo.
__host__ __device__ inline void halo_scatter_deep(int depth, int ny, int nx, size_t pitch, int epitch, int side,
                                                  int e, int jlo, int jhi, float val, float* const* field,
                                                  float* const* ext) {
  int f, js, is, jr, ir, layer;
  halo_msg_elem(depth, ny, nx, side, e, f, js, is, jr, ir, layer);
  const size_t eoff = (size_t)(jr + 2) * epitch + (ir + 2);
  if (side <= HALO_E) {
    if (jr >= 1 && jr <= ny - 2) ext[f][eoff] = val;
    if (layer == 0 && jr >= jlo && jr < jhi) field[f][(size_t)jr * pitch + ir] = val;
  } else {
    ext[f][eoff] = val;
    if (layer == 0) field[f][(size_t)jr * pitch + ir] = val;
  }
}

// One-layer exchange: the main halo cell, with the reference's wall conditions -- v (kind 2) is 0 on
// row ny-2 of a north-wall rank (`vwall`), u (kind 1) on column nx-2 of a non-periodic east-wall rank
// (`uwall`).  A received cell on a wall row / column is zeroed here, not only by halo_wall_pass: the
// sender reads its edge while other CTAs of its own launch may already be zeroing that edge's wall
// cells, so the value that arrives there is not reliably the wall value.
__host__ __device__ inline void halo_recv_walls(int ny, int nx, size_t pitch, int side, int e, int jlo, int jhi,
                                                bool uwall, bool vwall, float val, float* const* field,
                                                const int* kind) {
  int f, js, is, jr, ir, layer;
  halo_msg_elem(1, ny, nx, side, e, f, js, is, jr, ir, layer);
  if (side <= HALO_E) {
    if (jr < jlo || jr >= jhi) return;
    if (kind[f] == 2 && vwall && jr == ny - 2) val = 0.f;
  } else if (side <= HALO_N) {
    if (kind[f] == 1 && uwall && ir == nx - 2) val = 0.f;
  }
  field[f][(size_t)jr * pitch + ir] = val;
}

// The one-layer exchange's closing wall pass, thread t of n: the cells of u's wall column (rows
// [jlo, jhi)) and v's wall row (columns [ilo, ihi)) that no message writes.
__host__ __device__ inline void halo_wall_pass(int ny, int nx, size_t pitch, int nf, int jlo, int jhi, int ilo,
                                               int ihi, bool uwall, bool vwall, float* const* field,
                                               const int* kind, int t, int n) {
  for (int f = 0; f < nf; ++f) {
    if (kind[f] == 1 && uwall)
      for (int j = jlo + t; j < jhi; j += n) field[f][(size_t)j * pitch + (nx - 2)] = 0.f;
    if (kind[f] == 2 && vwall)
      for (int i = ilo + t; i < ihi; i += n) field[f][(size_t)(ny - 2) * pitch + i] = 0.f;
  }
}
