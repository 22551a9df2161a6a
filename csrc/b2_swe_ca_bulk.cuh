// mpi4jax_b200 -- shallow water, the BULK of the communication-avoiding step (b2_swe_ca.cu): the whole
// model step (flux + tendency + Adams-Bashforth update, then friction) on the cells at least four away
// from the block edge, in one pass over the arrays: h, u, v, dh, du, dv are read once and written once
// (12 array passes per step; the stand-alone kernels of b2_swe.cu make 32).
//
// A warp owns a column strip of 32 float4 groups and walks down a segment of rows.  Each lane keeps
// rolling rows in registers, so every flux quantity is evaluated once per cell row (a row's fluxes are
// the next row's "south" fluxes), and the friction of row t-1 follows the tendency of row t:
//
//   row t+2 (loaded one row ahead)     fluxes of row t+1   (fe, q at i0-1 .. i0+3, fn, ke at i0 .. i0+4)
//   tendency + update of row t         u', v' of row t     (registers only; never stored)
//   friction of row t-1                u'' needs u' of rows t-2 .. t and the west / east lanes' u'
//
// The u' a lane needs beyond its own four columns (two to the west, one to the east) come from its
// neighbour lanes, so lanes 0 and 31 only supply them: a warp stores 30 groups.  A segment also
// evaluates u', v' of the two rows above and the one row below it (and, at the bulk's edge, of the band
// cells at distance 2 and 3): nothing it reads is written by another warp in the same step, because u,
// v, du and dv are ping-pong pairs (the segment reads this step's arrays and writes the partners).  dh
// is updated in place: a cell's new dh is needed only where the cell's h' is stored, and only the
// owning lane reads it.
//
// Bit-compatibility with the stand-alone kernels: the quantities are the shared explicit-rounding
// helpers of b2_swe_body.cuh (swe_fe .. swe_ke, swe_k2_cell, swe_friction_u, swe_visc_flux,
// swe_apply_div), same operands, hence the same bits.  The body is written per lane with the two
// phases of a row (tendency, friction) separated by the lane exchange, so that the host emulation
// (tests/native/swe_host_emu.cpp) runs exactly this code.
#pragma once

#include "b2_swe_body.cuh"

#define CA_BULK_WARPS 4              // warps per CTA (independent: no shared memory, no barrier)
#define CA_BULK_LANES 30             // groups a warp stores; lanes 0 and 31 supply their neighbours' u', v'

// Row of six with index d + 1 for column offset d = -1 .. 4 relative to the group start.
struct Row6A {
  float a[6];
};
__device__ __forceinline__ Row6A ld_row_a(const float* __restrict__ x, int j, int i0, int pitch) {
  const Row6 r = ld_row<true, true>(x, j, i0, pitch);
  Row6A o;
  o.a[0] = r.w; o.a[1] = r.c0; o.a[2] = r.c1; o.a[3] = r.c2; o.a[4] = r.c3; o.a[5] = r.e;
  return o;
}

struct CABulkArgs {
  B2SweParams p;
  int ng;                                            // bulk groups per row: columns [4, 4 + 4 ng)
  int rows;                                          // rows per segment
  int wcols;                                         // warp strips per row of segments
  int nseg;                                          // segments: bulk rows [4, ny - 4)
  const float *h, *u, *v, *du, *dv;                  // this step
  float *h_o, *u_o, *v_o, *du_o, *dv_o;              // the next step (ping-pong partners)
  float* dh;                                         // read, then updated in place (own cell only)
};

// geometry of the launch: a warp's (segment, strip), a lane's group
__host__ __device__ inline void ca_bulk_geometry(const B2SweParams& p, int cb1, int rows, CABulkArgs& a) {
  a.ng = (cb1 >> 2) - 1;
  a.rows = rows;
  a.wcols = (a.ng + CA_BULK_LANES - 1) / CA_BULK_LANES;
  a.nseg = (p.ny - 8 + rows - 1) / rows;
}
__host__ __device__ inline long long ca_bulk_warps(const CABulkArgs& a) { return (long long)a.wcols * a.nseg; }
// group index of `lane` in strip `wc` (-1 = the group west of the bulk, ng = the one east of it;
// lanes beyond that repeat it); the lane stores when it returns true
__host__ __device__ inline bool ca_bulk_lane(const CABulkArgs& a, int wc, int lane, int& i0) {
  int g = wc * CA_BULK_LANES + lane - 1;
  if (g > a.ng) g = a.ng;
  i0 = 4 + 4 * g;
  return lane >= 1 && lane <= CA_BULK_LANES && g < a.ng;
}

// the four flux quantities of row k from rows k-1 (v only), k and k+1 (swe_k1_body's expressions)
struct CAFluxRow {
  float fe[5], q[5];                                 // columns i0-1 .. i0+3
  float fn[5], ke[5];                                // columns i0 .. i0+4
};
__device__ __forceinline__ void ca_bulk_fluxes(const B2SweParams& p, float cor, const Row6A& H, const Row6A& U,
                                               const Row6A& V, const Row6A& Hn, const Row6A& Un, const Row6A& Vs,
                                               CAFluxRow& f) {
#pragma unroll
  for (int t = 0; t < 5; ++t) {
    f.fe[t] = swe_fe(H.a[t], H.a[t + 1], U.a[t]);
    f.q[t] = swe_q(p, cor, V.a[t + 1], V.a[t], Un.a[t], U.a[t], H.a[t], H.a[t + 1], Hn.a[t], Hn.a[t + 1]);
    const int x = t + 1;
    f.fn[t] = swe_fn(H.a[x], Hn.a[x], V.a[x]);
    f.ke[t] = swe_ke(U.a[x], U.a[x - 1], V.a[x], Vs.a[x]);
  }
}

// everything a lane carries from one row to the next
struct CABulkLane {
  int i0;
  bool store;                                        // this lane's group is a bulk group
  Row6A H[3], U[3], V[3];                            // rows t, t+1 and (loaded ahead) t+2
  CAFluxRow Fm, Fc;                                  // fluxes of rows t-1, t
  float4 dh4, du4, dv4;                              // old tendencies of row t
  float upn[4], vpn[4];                              // u', v' of row t (exchanged between the phases)
  float up0[7], up1[7];                              // u' of rows t-2, t-1: index d + 2 <-> column i0 + d
  float vp1[5];                                      // v' of row t-1: columns i0 .. i0+4
  float upp1[4];                                     // u'' of row t-2: columns i0 .. i0+3
};

// rows [s, e) of segment `seg`; its tendency rows are s-2 .. e (rows s-2, s-1 and e only feed the
// friction of rows s .. e-1)
__host__ __device__ inline void ca_bulk_rows(const CABulkArgs& a, int seg, int& s, int& e) {
  s = 4 + seg * a.rows;
  e = s + a.rows < a.p.ny - 4 ? s + a.rows : a.p.ny - 4;
}

// rows s-4 .. s-1 and the fluxes of rows s-3, s-2 of the segment starting at row s
__device__ __forceinline__ void ca_bulk_begin(const CABulkArgs& a, CABulkLane& L, int s) {
  const int P = a.p.pitch, t = s - 2;
  const Row6A Vs = ld_row_a(a.v, t - 2, L.i0, P);
  L.H[0] = ld_row_a(a.h, t - 1, L.i0, P); L.U[0] = ld_row_a(a.u, t - 1, L.i0, P); L.V[0] = ld_row_a(a.v, t - 1, L.i0, P);
  L.H[1] = ld_row_a(a.h, t, L.i0, P); L.U[1] = ld_row_a(a.u, t, L.i0, P); L.V[1] = ld_row_a(a.v, t, L.i0, P);
  L.H[2] = ld_row_a(a.h, t + 1, L.i0, P); L.U[2] = ld_row_a(a.u, t + 1, L.i0, P); L.V[2] = ld_row_a(a.v, t + 1, L.i0, P);
  ca_bulk_fluxes(a.p, a.p.coriolis[t - 1], L.H[0], L.U[0], L.V[0], L.H[1], L.U[1], Vs, L.Fm);
  ca_bulk_fluxes(a.p, a.p.coriolis[t], L.H[1], L.U[1], L.V[1], L.H[2], L.U[2], L.V[0], L.Fc);
  // slots 0, 1 = rows t, t+1 (ca_bulk_tend loads row t+2 into slot 2)
  L.H[0] = L.H[1]; L.U[0] = L.U[1]; L.V[0] = L.V[1];
  L.H[1] = L.H[2]; L.U[1] = L.U[2]; L.V[1] = L.V[2];
  L.dh4 = L.du4 = L.dv4 = make_float4(0.f, 0.f, 0.f, 0.f);
}

// phase 1 of row t: load row t+2 and the old tendencies, fluxes of row t+1, tendency + update of row t;
// stores h', dh, du, dv when `out` (row t is one of the segment's rows)
__device__ __forceinline__ void ca_bulk_tend(const CABulkArgs& a, CABulkLane& L, int t, bool out) {
  const B2SweParams& p = a.p;
  const int P = p.pitch;
  const size_t off = (size_t)t * P + L.i0;
  L.H[2] = ld_row_a(a.h, t + 2, L.i0, P); L.U[2] = ld_row_a(a.u, t + 2, L.i0, P); L.V[2] = ld_row_a(a.v, t + 2, L.i0, P);
  if (!p.first_step) {
    L.du4 = ld4(a.du, off); L.dv4 = ld4(a.dv, off);
    if (out) L.dh4 = ld4(a.dh, off);                 // (rows above / below the segment: h' is not stored)
  }
  CAFluxRow Fp;
  ca_bulk_fluxes(p, p.coriolis[t + 1], L.H[1], L.U[1], L.V[1], L.H[2], L.U[2], L.V[0], Fp);
  const float DHo[4] = {L.dh4.x, L.dh4.y, L.dh4.z, L.dh4.w}, DUo[4] = {L.du4.x, L.du4.y, L.du4.z, L.du4.w},
              DVo[4] = {L.dv4.x, L.dv4.y, L.dv4.z, L.dv4.w};
  float Hn[4], DH[4], DU[4], DV[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    SweK2In in;
    in.fe_c = L.Fc.fe[k + 1]; in.fe_w = L.Fc.fe[k]; in.fen_c = Fp.fe[k + 1]; in.fen_w = Fp.fe[k];
    in.fn_c = L.Fc.fn[k]; in.fn_e = L.Fc.fn[k + 1]; in.fns_c = L.Fm.fn[k]; in.fns_e = L.Fm.fn[k + 1];
    in.q_c = L.Fc.q[k + 1]; in.q_w = L.Fc.q[k]; in.qs_c = L.Fm.q[k + 1];
    in.ke_c = L.Fc.ke[k]; in.ke_e = L.Fc.ke[k + 1]; in.ken_c = Fp.ke[k];
    in.h_c = L.H[0].a[k + 1]; in.h_e = L.H[0].a[k + 2]; in.h_n = L.H[1].a[k + 1];
    in.u_o = L.U[0].a[k + 1]; in.v_o = L.V[0].a[k + 1];
    in.dh_o = DHo[k]; in.du_o = DUo[k]; in.dv_o = DVo[k];
    const SweK2Out o = swe_k2_cell(p, in);
    Hn[k] = o.h; L.upn[k] = o.u; L.vpn[k] = o.v;
    DH[k] = o.dh; DU[k] = o.du; DV[k] = o.dv;
  }
  if (out && L.store) {
    st4(a.h_o, off, make_float4(Hn[0], Hn[1], Hn[2], Hn[3]));
    st4(a.dh, off, make_float4(DH[0], DH[1], DH[2], DH[3]));
    st4(a.du_o, off, make_float4(DU[0], DU[1], DU[2], DU[3]));
    st4(a.dv_o, off, make_float4(DV[0], DV[1], DV[2], DV[3]));
  }
  L.H[0] = L.H[1]; L.U[0] = L.U[1]; L.V[0] = L.V[1];
  L.H[1] = L.H[2]; L.U[1] = L.U[2]; L.V[1] = L.V[2];
  L.Fm = L.Fc; L.Fc = Fp;
}

// phase 2 of row t: friction of row r = t-1 (swe_k34_body's u update and fluxes, swe_k5_body's v update)
// given the west lane's u' of row t at columns i0-2, i0-1 and the east lane's u', v' at i0+4.
// `upp_only`: row r lies above the segment, only its u'' is needed (the south flux of the next row);
// `out`: row r is one of the segment's rows, u'' and v'' are stored.
__device__ __forceinline__ void ca_bulk_fric(const CABulkArgs& a, CABulkLane& L, int t, float uw2, float uw3,
                                             float ue, float ve, bool upp_only, bool out) {
  const B2SweParams& p = a.p;
  const float up2[7] = {uw2, uw3, L.upn[0], L.upn[1], L.upn[2], L.upn[3], ue};
  const float vp2[5] = {L.vpn[0], L.vpn[1], L.vpn[2], L.vpn[3], ve};
  if (upp_only || out) {
    float UPP[5], FE2[5];
#pragma unroll
    for (int d = 0; d < 5; ++d) {                    // column i0 + d - 1
      const int x = d + 1;
      UPP[d] = swe_friction_u(p, L.up1[x], L.up1[x + 1], L.up1[x - 1], up2[x], L.up0[x], false, false);
      FE2[d] = swe_visc_flux(p.c_nux, L.vp1[d], UPP[d]);
    }
    if (out && L.store) {
      float Vn[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float fn2_c = swe_visc_flux(p.c_nuy, vp2[k], UPP[k + 1]);     // fn2[r][i]
        const float fn2_s = swe_visc_flux(p.c_nuy, L.vp1[k], L.upp1[k]);    // fn2[r-1][i]
        Vn[k] = swe_apply_div(p, L.vp1[k], FE2[k + 1], FE2[k], fn2_c, fn2_s);
      }
      const size_t off = (size_t)(t - 1) * p.pitch + L.i0;
      st4(a.u_o, off, make_float4(UPP[1], UPP[2], UPP[3], UPP[4]));
      st4(a.v_o, off, make_float4(Vn[0], Vn[1], Vn[2], Vn[3]));
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) L.upp1[k] = UPP[k + 1];
  }
#pragma unroll
  for (int x = 0; x < 7; ++x) { L.up0[x] = L.up1[x]; L.up1[x] = up2[x]; }
#pragma unroll
  for (int x = 0; x < 5; ++x) L.vp1[x] = vp2[x];
}
