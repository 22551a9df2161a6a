// mpi4jax_b200 -- shallow water, communication-avoiding step ("CA"): ONE halo exchange per model
// step instead of the reference's twelve per-field rounds (three fused exchanges in b2_swe.cu).
//
// The reference's step (examples/shallow_water.py:270-403) alternates local stencils with halo
// exchanges four times: fluxes -> exchange(fe, fn, q, ke) -> tendencies -> exchange(h', u', v')
// -> friction-u -> exchange(fe2, fn2) -> friction-v.  At 8 GPUs a rank owns 2048 x 1024 cells; with
// so little arithmetic per step, the NVLink round trip of every exchange -- not the bandwidth --
// bounds the step.  Here the tendency phase's result (h', u', v') is exchanged ONCE, three cells deep, and everything the other two exchanges
// used to deliver is recomputed from it on a thin frame around the block:
//
//   frame kernel A   h', u', v' on the cells within 3 of the block edge (u', v' two cells further: the
//                    "band").  The fluxes a ring cell needs from its neighbours' side of the edge are
//                    evaluated locally, each with the operands its OWNER would have used (see "views").
//   exchange X       3 layers of (h', u', v') to all eight neighbours (b2_swe_ca.cu).
//   frame kernel D   friction (u' -> u'', v' -> v'') on the frame, and the neighbours' u'', v''
//                    one / two cells beyond the edge, which next step's halo fluxes need.
//   bulk kernel      flux + tendency, then friction, on everything else, one pass (b2_swe_ca_bulk.cuh):
//                    its dependency cone stays inside the step's input arrays, so it needs nothing from
//                    A, X or D and runs concurrently with A -> X -> D.
//
// Views.  The reference's discrete system is decomposition dependent: a rank computes its
// fluxes from u, v whose HALO is stale by the friction update (the halo of u, v is exchanged
// before the friction step and not after it).  A flux at a halo cell therefore has to be
// evaluated as the cell's owner Q does: with the post-friction value u'' at cells Q owns and
// the pre-friction value u' at cells Q only sees as halo.  `ca_vu(Q, d)` implements exactly
// that; with it (and the explicit-rounding helpers of b2_swe_body.cuh) this pipeline and the
// stand-alone one produce the same bits on the same decomposition
// (tests/test_swe_host_emulation.py runs both on 1x1 .. 2x4 process grids).
//
// Storage.  The main (ny, pitch) arrays keep their meaning (1-cell halo; u, v halos stale).  h, u, v,
// du and dv come in three buffer sets: every kernel of a step reads one set and writes another
// (b2_swe_ca.cu: two sets per step, the third for the pair schedule that advances the bulk two steps).
// dh is updated in place by a one-step schedule and moves between three buffers with a pair of steps.
// Five "ext" arrays [(ny + 4) x epitch], cell (j, i) at (j + 2) * epitch + (i + 2), hold what
// lies beyond: hx (h, layers 1..2), upx / vpx (u', v': layers 1..3 and a mirror of this rank's
// own ring cells, i.e. every STALE value a view can ask for), uppx / vppx (u'', v'' of the
// neighbours' cells, layers 1..2 / 1).  Only their outer cells are ever touched.
#pragma once

#include "b2_halo_geom.h"
#include "b2_swe_body.cuh"

#ifndef __CUDACC__
#ifndef __noinline__
#define __noinline__ __attribute__((noinline))      // host emulation build (tests/native/swe_host_emu.cpp)
#endif
#endif
#define CA_L 3        // halo layers exchanged per step (layer 1 = the main arrays' halo cell)
#define CA_NF 3       // fields per exchange: h', u', v'

// everything a frame kernel dereferences
struct CACtx {
  B2SweParams p;
  B2SweCA x;
  const float *h;                 // h of this step (halo fresh)
  float *hn;                      // h' (ping-pong partner of h)
  const float *ua, *va;           // u'', v'' of the previous step (interior; wall rows constant); kernel D
                                  // writes this step's into the partners
  float *dh;                      // the next step's dh (frame cells)
  const float *dh_src = nullptr;  // this step's dh; null: dh, updated cell by cell in place
  const float *du, *dv;           // du, dv of this step (the previous step's tendencies)
  float *du_o, *dv_o;             // their partners: the bulk kernel reads du, dv while kernel A runs
  float *upf, *vpf;               // u', v' of the frame band (cells within 5 of the edge) and, after X, their halo
};

__host__ __device__ inline bool swe_ca_supported(const B2SweParams& p) {
  return p.ny >= 16 && p.nx >= 24;
}
__host__ __device__ inline int swe_ca_cb1(const B2SweParams& p) { return ((p.nx - 4) >> 2) << 2; }   // multiple of 4 <= nx - 4
// frame cells proper: within three of the block edge (plus the columns the bulk's alignment leaves over)
__host__ __device__ __forceinline__ bool ca_is_frame(const B2SweParams& p, int cb1, int j, int i) {
  return j <= 3 || j >= p.ny - 4 || i <= 3 || i >= cb1;
}

__host__ __device__ __forceinline__ int ca_rj(const B2SweParams& p, int j) { return j < 1 ? -1 : (j > p.ny - 2 ? 1 : 0); }
__host__ __device__ __forceinline__ int ca_ri(const B2SweParams& p, int i) { return i < 1 ? -1 : (i > p.nx - 2 ? 1 : 0); }
// rows beyond a physical wall (no rank owns them; the main arrays hold their constant values)
__host__ __device__ __forceinline__ bool ca_wall_row(const B2SweParams& p, int j) {
  return (j < 1 && p.south_wall) || (j > p.ny - 2 && p.north_wall);
}
__host__ __device__ __forceinline__ size_t ca_m(const B2SweParams& p, int j, int i) { return (size_t)j * p.pitch + i; }
__host__ __device__ __forceinline__ size_t ca_e(const B2SweCA& x, int j, int i) {
  return (size_t)(j + 2) * x.epitch + (i + 2);
}
__host__ __device__ __forceinline__ bool ca_mine(const B2SweParams& p, int j, int i) {
  return j >= 1 && j <= p.ny - 2 && i >= 1 && i <= p.nx - 2;
}

// ---- accessors -------------------------------------------------------------------------------
// Straight-line code: every accessor SELECTS an address and issues one load, rows beyond a wall are
// clamped into the main arrays (their values are never used: the wall rules zero what they feed).
// No branch separates the ~100 loads of a frame cell, so they are all in flight together -- the
// frame kernels are on the step's critical path and pure latency.
__device__ __forceinline__ size_t ca_m_safe(const B2SweParams& p, int j, int i) {
  const int jj = j < 0 ? 0 : (j > p.ny - 1 ? p.ny - 1 : j), ii = i < 0 ? 0 : (i > p.nx - 1 ? p.nx - 1 : i);
  return (size_t)jj * p.pitch + ii;
}
__device__ __forceinline__ float ca_h(const CACtx& c, int j, int i) {
  const bool main = ca_mine(c.p, j, i) || ca_wall_row(c.p, j);
  const float* ptr = main ? c.h + ca_m_safe(c.p, j, i) : c.x.hx + ca_e(c.x, j, i);
  return *ptr;
}
// u as cell-owner Q = (qj, qi) sees it at cell (j, i): fresh where Q owns the cell, stale elsewhere
__device__ __forceinline__ float ca_vu(const CACtx& c, int qj, int qi, int j, int i) {
  const int rj = ca_rj(c.p, j), ri = ca_ri(c.p, i);
  const bool own = rj == qj && ri == qi, mine = rj == 0 && ri == 0;
  const float* ext = own ? c.x.uppx : c.x.upx;
  const float* ptr = (ca_wall_row(c.p, j) || (own && mine)) ? c.ua + ca_m_safe(c.p, j, i) : ext + ca_e(c.x, j, i);
  return *ptr;
}
__device__ __forceinline__ float ca_vv(const CACtx& c, int qj, int qi, int j, int i) {
  const int rj = ca_rj(c.p, j), ri = ca_ri(c.p, i);
  const bool own = rj == qj && ri == qi, mine = rj == 0 && ri == 0;
  const float* ext = own ? c.x.vppx : c.x.vpx;
  const float* ptr = (ca_wall_row(c.p, j) || (own && mine)) ? c.va + ca_m_safe(c.p, j, i) : ext + ca_e(c.x, j, i);
  return *ptr;
}

// ---- the four flux-kernel quantities at cell (j, i) in [0, ny) x [0, nx), evaluated as the
// cell's owner does (swe_k1_body's expressions; zero beyond a wall, where nothing is ever stored:
// such a cell is evaluated at the clamped row and the result discarded)
__device__ __forceinline__ int ca_flux_row(const B2SweParams& p, int j) {
  return ca_wall_row(p, j) ? (j < 1 ? 1 : p.ny - 2) : j;
}
__device__ __forceinline__ float ca_fe(const CACtx& c, int j0, int i) {
  const int j = ca_flux_row(c.p, j0);
  const int qj = ca_rj(c.p, j), qi = ca_ri(c.p, i), hj = hc_row(c.p, j);
  const float r = swe_fe(ca_h(c, hj, i), ca_h(c, hj, i + 1), ca_vu(c, qj, qi, j, i));
  return ca_wall_row(c.p, j0) ? 0.f : r;
}
__device__ __forceinline__ float ca_fn(const CACtx& c, int j0, int i) {
  const int j = ca_flux_row(c.p, j0);
  const int qj = ca_rj(c.p, j), qi = ca_ri(c.p, i);
  const float r = swe_fn(ca_h(c, hc_row(c.p, j), i), ca_h(c, hc_row(c.p, j + 1), i), ca_vv(c, qj, qi, j, i));
  return (ca_wall_row(c.p, j0) || (c.p.north_wall && j0 == c.p.ny - 2)) ? 0.f : r;      // "v" wall rule
}
__device__ __forceinline__ float ca_q(const CACtx& c, int j0, int i) {
  const int j = ca_flux_row(c.p, j0);
  const int qj = ca_rj(c.p, j), qi = ca_ri(c.p, i), hj = hc_row(c.p, j), hj1 = hc_row(c.p, j + 1);
  const float r = swe_q(c.p, c.p.coriolis[j], ca_vv(c, qj, qi, j, i + 1), ca_vv(c, qj, qi, j, i),
                        ca_vu(c, qj, qi, j + 1, i), ca_vu(c, qj, qi, j, i), ca_h(c, hj, i), ca_h(c, hj, i + 1),
                        ca_h(c, hj1, i), ca_h(c, hj1, i + 1));
  return ca_wall_row(c.p, j0) ? 0.f : r;
}
__device__ __forceinline__ float ca_ke(const CACtx& c, int j0, int i) {
  const int j = ca_flux_row(c.p, j0);
  const int qj = ca_rj(c.p, j), qi = ca_ri(c.p, i);
  const float r = swe_ke(ca_vu(c, qj, qi, j, i), ca_vu(c, qj, qi, j, i - 1), ca_vv(c, qj, qi, j, i),
                         ca_vv(c, qj, qi, j - 1, i));
  return ca_wall_row(c.p, j0) ? 0.f : r;
}

// ---- frame kernel A: flux + tendency update of one of this rank's cells ------------------------
// Frame cells get everything; the two cells beyond them (distance 4, 5: bulk cells, whose h', dh ..
// the bulk kernel writes) only need their u', v' here, because kernel D's friction stencil on the
// frame reaches that far and must not wait for the bulk kernel.
// The 14 flux values of a cell's tendency stencil, as (kind, dj, di); a warp of kernel A evaluates the
// slots of ONE kind for 32 cells, so the cell's latency is a few flux evaluations, not fourteen in a row.
#define CA_NSLOT 14
__host__ __device__ __forceinline__ int ca_slot_base(int kind) { return kind == 0 ? 0 : kind == 1 ? 4 : kind == 2 ? 8 : 11; }
__host__ __device__ __forceinline__ int ca_slot_count(int kind) { return kind < 2 ? 4 : 3; }
// offset of slot k of `kind` from the cell: fe (0,0) (0,-1) (1,0) (1,-1); fn (0,0) (0,1) (-1,0) (-1,1);
// q (0,0) (0,-1) (-1,0); ke (0,0) (0,1) (1,0)
__host__ __device__ __forceinline__ int ca_slot_dj(int kind, int k) {
  return kind == 0 ? (k >> 1) : kind == 1 ? -(k >> 1) : kind == 2 ? -(k >> 1) : (k >> 1);
}
__host__ __device__ __forceinline__ int ca_slot_di(int kind, int k) {
  return kind == 0 ? -(k & 1) : kind == 1 ? (k & 1) : kind == 2 ? -(k & 1) : (k & 1);
}
// A flux at one of THIS rank's cells is what the stand-alone flux kernel computes there: every operand
// comes from the main arrays, whose halo holds exactly the stale value the view rule asks for (kernel D
// and the exchange keep it so).  Only the fluxes at the cells beyond the edge -- which the reference
// receives by halo exchange -- need the owner's view, i.e. the ext arrays (generic path below); they
// enter the stencils of the outermost ring of cells only.
__device__ __forceinline__ float ca_flux_plain(const CACtx& c, int j, int i, int kind) {
  const B2SweParams& p = c.p;
  const size_t o = ca_m(p, j, i), oh = ca_m(p, hc_row(p, j), i), ohn = ca_m(p, hc_row(p, j + 1), i);
  const size_t P = (size_t)p.pitch;
  switch (kind) {
    case 0: return swe_fe(c.h[oh], c.h[oh + 1], c.ua[o]);
    case 1: return (p.north_wall && j == p.ny - 2) ? 0.f : swe_fn(c.h[oh], c.h[ohn], c.va[o]);
    case 2: return swe_q(p, p.coriolis[j], c.va[o + 1], c.va[o], c.ua[o + P], c.ua[o], c.h[oh], c.h[oh + 1], c.h[ohn],
                         c.h[ohn + 1]);
    default: return swe_ke(c.ua[o], c.ua[o - 1], c.va[o], c.va[o - P]);
  }
}
// the rare path is a real call: inlined, its ~250 instructions per flux would sit in every one of the
// fourteen slots and the kernel would spend its time fetching instructions
static __device__ __noinline__ float ca_flux_generic(const CACtx& c, int j, int i, int kind) {
  switch (kind) {
    case 0: return ca_fe(c, j, i);
    case 1: return ca_fn(c, j, i);
    case 2: return ca_q(c, j, i);
    default: return ca_ke(c, j, i);
  }
}
// all slots of one kind: the plain evaluations first, branch-free (a flux cell beyond the edge is
// evaluated at the clamped cell and replaced afterwards), so every load of the warp is in flight at once
template <int KIND>
__device__ __forceinline__ void ca_flux_kind(const CACtx& c, int j, int i, float* r) {
  constexpr int n = KIND < 2 ? 4 : 3;
  const int ny = c.p.ny, nx = c.p.nx;
#pragma unroll
  for (int k = 0; k < n; ++k) {
    const int fj = j + ca_slot_dj(KIND, k), fi = i + ca_slot_di(KIND, k);
    const int cj = fj < 1 ? 1 : (fj > ny - 2 ? ny - 2 : fj), ci = fi < 1 ? 1 : (fi > nx - 2 ? nx - 2 : fi);
    r[k] = ca_flux_plain(c, cj, ci, KIND);
  }
#pragma unroll
  for (int k = 0; k < n; ++k) {
    const int fj = j + ca_slot_dj(KIND, k), fi = i + ca_slot_di(KIND, k);
    if (!ca_mine(c.p, fj, fi)) r[k] = ca_flux_generic(c, fj, fi, KIND);
  }
}
__device__ __forceinline__ void ca_flux_all(const CACtx& c, int j, int i, float* fl) {
  ca_flux_kind<0>(c, j, i, fl);
  ca_flux_kind<1>(c, j, i, fl + 4);
  ca_flux_kind<2>(c, j, i, fl + 8);
  ca_flux_kind<3>(c, j, i, fl + 11);
}
__device__ __forceinline__ void swe_ca_tend_finish(const CACtx& c, int j, int i, const float* fl) {
  const B2SweParams& p = c.p;
  const size_t off = ca_m(p, j, i);
  SweK2In in;
  in.fe_c = fl[0]; in.fe_w = fl[1]; in.fen_c = fl[2]; in.fen_w = fl[3];
  in.fn_c = fl[4]; in.fn_e = fl[5]; in.fns_c = fl[6]; in.fns_e = fl[7];
  in.q_c = fl[8]; in.q_w = fl[9]; in.qs_c = fl[10];
  in.ke_c = fl[11]; in.ke_e = fl[12]; in.ken_c = fl[13];
  in.h_c = c.h[off]; in.h_e = ca_h(c, j, i + 1); in.h_n = ca_h(c, j + 1, i);
  in.u_o = c.ua[off]; in.v_o = c.va[off];
  const bool frame = ca_is_frame(p, c.x.cb1, j, i);
  // (a band-only cell's h' and dh are the bulk kernel's: its old dh is not needed)
  in.dh_o = (p.first_step || !frame) ? 0.f : (c.dh_src != nullptr ? c.dh_src : c.dh)[off];
  in.du_o = p.first_step ? 0.f : c.du[off];
  in.dv_o = p.first_step ? 0.f : c.dv[off];
  SweK2Out o = swe_k2_cell(p, in);
  if (p.north_wall && j == p.ny - 2) o.v = 0.f;       // "v" wall rule, after the update
  c.upf[off] = o.u; c.vpf[off] = o.v;
  if (frame) {                                        // (the band-only cells are the bulk kernel's)
    c.hn[off] = o.h;
    c.dh[off] = o.dh;
    c.du_o[off] = o.du;
    c.dv_o[off] = o.dv;
  }
}
__device__ __forceinline__ void swe_ca_tend_cell(const CACtx& c, int j, int i) {
  float fl[CA_NSLOT];
  ca_flux_all(c, j, i, fl);
  swe_ca_tend_finish(c, j, i, fl);
}

// ---- frame kernel D: friction ------------------------------------------------------------------
// u', v' of the frame band and of the cells up to three beyond the block (mine: upf / vpf; beyond: the
// exchanged copy)
__device__ __forceinline__ float ca_up(const CACtx& c, int j, int i) {
  const bool main = ca_mine(c.p, j, i) || ca_wall_row(c.p, j);
  const float* ptr = main ? c.upf + ca_m_safe(c.p, j, i) : c.x.upx + ca_e(c.x, j, i);
  return *ptr;
}
__device__ __forceinline__ float ca_vp(const CACtx& c, int j, int i) {
  const bool main = ca_mine(c.p, j, i) || ca_wall_row(c.p, j);
  const float* ptr = main ? c.vpf + ca_m_safe(c.p, j, i) : c.x.vpx + ca_e(c.x, j, i);
  return *ptr;
}
// u'' of cell (j, i) (swe_k34_body's update; the wall rules are functions of the row only, and a
// y neighbour's far wall is out of reach)
__device__ __forceinline__ float ca_upp(const CACtx& c, int j, int i) {
  const B2SweParams& p = c.p;
  return swe_friction_u(p, ca_up(c, j, i), ca_up(c, j, i + 1), ca_up(c, j, i - 1), ca_up(c, j + 1, i),
                        ca_up(c, j - 1, i), p.north_wall && j == p.ny - 2, p.south_wall && j == 1);
}
// v'' of cell (j, i) given u'' of the cell, of its west and of its south neighbour (swe_k34_body's
// fluxes + swe_k5_body's update)
__device__ __forceinline__ float ca_vpp(const CACtx& c, int j, int i, float upp_c, float upp_w, float upp_s) {
  const B2SweParams& p = c.p;
  const float v_c = ca_vp(c, j, i);
  const float fe2_c = swe_visc_flux(p.c_nux, ca_vp(c, j, i + 1), upp_c);
  const float fe2_w = swe_visc_flux(p.c_nux, v_c, upp_w);
  const float fn2_c = swe_visc_flux(p.c_nuy, ca_vp(c, j + 1, i), upp_c);
  const float fn2_s = swe_visc_flux(p.c_nuy, v_c, upp_s);                     // south wall: clamped loads, discarded
  return swe_apply_div(p, v_c, fe2_c, fe2_w, (p.north_wall && j == p.ny - 2) ? 0.f : fn2_c,
                       (p.south_wall && j == 1) ? 0.f : fn2_s);
}
// the three u'' values a cell's friction needs: slot 0 = the cell, 1 = west, 2 = south (a warp of
// kernel D evaluates one slot for 32 cells)
__device__ __forceinline__ float ca_upp_slot(const CACtx& c, int j, int i, int slot) {
  return slot == 0 ? ca_upp(c, j, i) : slot == 1 ? ca_upp(c, j, i - 1) : ca_upp(c, j - 1, i);
}
// cells beyond the first halo layer only need their own u'' (their v'' is never used)
__device__ __forceinline__ bool ca_needs_vpp(const B2SweParams& p, int j, int i) {
  return j >= 0 && j <= p.ny - 1 && i >= 0 && i <= p.nx - 1;
}

// one of this rank's frame cells: u'' -> ua, v'' -> va; ring cells also mirror u', v' into the
// stale store (what the neighbours see in their halo until the next exchange)
__device__ __forceinline__ void swe_ca_fric_finish(const CACtx& c, float* __restrict__ ua_out,
                                                   float* __restrict__ va_out, int j, int i, const float* upp) {
  const B2SweParams& p = c.p;
  const size_t off = ca_m(p, j, i);
  ua_out[off] = upp[0];
  va_out[off] = ca_vpp(c, j, i, upp[0], upp[1], upp[2]);
  if (j == 1 || j == p.ny - 2 || i == 1 || i == p.nx - 2) {
    const size_t e = ca_e(c.x, j, i);
    c.x.upx[e] = c.upf[off];
    c.x.vpx[e] = c.vpf[off];
  }
}
// a neighbour's cell, one or two layers beyond the edge: its u'' (and v'' on layer 1).  Layer 1 is
// also the main arrays' halo: u, v get the exchanged u', v' there -- stale by this friction step,
// which is what the reference's in-place update leaves in the halo.
__device__ __forceinline__ void swe_ca_fric_ext_finish(const CACtx& c, float* __restrict__ ua_out,
                                                       float* __restrict__ va_out, int j, int i, const float* upp) {
  const B2SweParams& p = c.p;
  const size_t e = ca_e(c.x, j, i);
  c.x.uppx[e] = upp[0];
  if (ca_needs_vpp(p, j, i)) {
    c.x.vppx[e] = ca_vpp(c, j, i, upp[0], upp[1], upp[2]);
    ua_out[ca_m(p, j, i)] = c.x.upx[e];
    va_out[ca_m(p, j, i)] = c.x.vpx[e];
  }
}
// ---- task enumeration ----------------------------------------------------------------------------
// Bulk (b2_swe_ca_bulk.cuh) = rows [4, ny-5] x columns [4, cb1); frame = every other interior cell.
// A band of width w: rows [1, w] and [ny-1-w, ny-2] completely, of the rows in between the columns
// [1, w] and [ce, nx-2].  Kernel D walks the frame (w = 3, ce = cb1), kernel A the frame plus the two
// cells beyond it (w = 5, ce = cb1 - 2).
struct CAFrame {
  int w, ce;
  int nfull;          // cells in the 2w full rows
  int per;            // band cells per middle row
  int nrows;          // middle rows
  int total;
};
__host__ __device__ inline CAFrame ca_frame(const B2SweParams& p, int w, int ce) {
  CAFrame f;
  f.w = w; f.ce = ce;
  f.nfull = 2 * w * (p.nx - 2);
  f.per = w + (p.nx - 1 - ce);
  f.nrows = p.ny - 2 - 2 * w;
  f.total = f.nfull + f.nrows * f.per;
  return f;
}
// (32-bit arithmetic throughout: the frame of a block that fits a GPU is a few hundred thousand cells,
// and a 64-bit division costs more than the flux it indexes)
__host__ __device__ inline bool ca_frame_cell(const B2SweParams& p, const CAFrame& f, int idx, int& j, int& i) {
  if (idx >= f.total) return false;
  if (idx < f.nfull) {
    const int n = p.nx - 2;
    const int r = idx / n;
    i = 1 + (idx - r * n);
    j = r < f.w ? 1 + r : (p.ny - 1 - f.w) + (r - f.w);
  } else {
    // side bands column by column (a warp's 32 cells then share their distance from the edge, i.e.
    // take the same path through the accessors)
    const int t = idx - f.nfull;
    const int s = t / f.nrows;
    j = f.w + 1 + (t - s * f.nrows);
    i = s < f.w ? 1 + s : f.ce + (s - f.w);
  }
  return true;
}
// the two layers of cells around the interior ("ext ring"): rows -1, 0, ny-1, ny (columns
// -1 .. nx) and columns -1, 0, nx-1, nx of the rows in between; cells beyond a wall do not exist
__host__ __device__ inline long long ca_ext_total(const B2SweParams& p) {
  return 4LL * (p.nx + 2) + 4LL * (p.ny - 2);
}
__host__ __device__ inline bool ca_ext_cell(const B2SweParams& p, long long idx, int& j, int& i) {
  const long long nrow = 4LL * (p.nx + 2);
  if (idx < nrow) {
    const int r = (int)(idx / (p.nx + 2));
    i = -1 + (int)(idx % (p.nx + 2));
    j = r == 0 ? -1 : r == 1 ? 0 : r == 2 ? p.ny - 1 : p.ny;
  } else {
    const long long t = idx - nrow;
    if (t >= 4LL * (p.ny - 2)) return false;
    const int s = (int)(t & 3);
    j = 1 + (int)(t >> 2);
    i = s == 0 ? -1 : s == 1 ? 0 : s == 2 ? p.nx - 1 : p.nx;
  }
  return !ca_wall_row(p, j);
}
// task t of kernel D -> cell; frame cells first, then the two layers beyond the edge
__device__ __forceinline__ bool ca_fric_task(const B2SweParams& p, const CAFrame& f, long long t, int& j, int& i,
                                             bool& ext) {
  ext = t >= f.total;
  if (!ext) return ca_frame_cell(p, f, (int)t, j, i);
  return ca_ext_cell(p, t - f.total, j, i);
}
__device__ __forceinline__ void swe_ca_fric_task(const CACtx& c, const CAFrame& f, float* __restrict__ ua_out,
                                                 float* __restrict__ va_out, long long t) {
  int j, i;
  bool ext;
  if (!ca_fric_task(c.p, f, t, j, i, ext)) return;
  float upp[3] = {ca_upp_slot(c, j, i, 0), 0.f, 0.f};
  if (ca_needs_vpp(c.p, j, i)) { upp[1] = ca_upp_slot(c, j, i, 1); upp[2] = ca_upp_slot(c, j, i, 2); }
  if (ext) swe_ca_fric_ext_finish(c, ua_out, va_out, j, i, upp);
  else swe_ca_fric_finish(c, ua_out, va_out, j, i, upp);
}

// ---- exchange geometry: the eight-side messages of b2_halo_geom.h at CA_NF fields, CA_L layers deep -----
__host__ __device__ inline int ca_msg_count(int ny, int nx, int side) {
  return halo_msg_count(CA_NF, CA_L, ny, nx, side);
}
__host__ __device__ inline void ca_msg_elem(int ny, int nx, int side, int e, int& f, int& js, int& is, int& jr,
                                            int& ir, int& layer) {
  halo_msg_elem(CA_L, ny, nx, side, e, f, js, is, jr, ir, layer);
}
__host__ __device__ inline void ca_scatter(int ny, int nx, size_t pitch, int epitch, int side, int e, int jlo,
                                           int jhi, float val, float* const* field, float* const* ext) {
  halo_scatter_deep(CA_L, ny, nx, pitch, epitch, side, e, jlo, jhi, val, field, ext);
}
