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
// cells at distance 2 and 3): nothing it reads is written by another warp in the same step, because the
// segment reads this step's buffer set and writes another.
//
// The same functions serve the pair kernel (swe_ca_bulk_pair, b2_swe_ca.cu), whose step-2 warp reads its
// rows from the step-1 warp's shared-memory ring instead of the arrays: the row addressing is a template
// parameter (IN_RING / OUT_RING), the arithmetic is the same code.
//
// Bit-compatibility with the stand-alone kernels: the quantities are the shared explicit-rounding
// helpers of b2_swe_body.cuh (swe_fe .. swe_ke, swe_k2_cell, swe_friction_u, swe_visc_flux,
// swe_apply_div), same operands, hence the same bits.  The body is written per lane with the two
// phases of a row (tendency, friction) separated by the lane exchange, so that the host emulation
// (tests/native/swe_host_emu.cpp) runs exactly this code.
#pragma once

#include "b2_swe_body.cuh"

#define CA_BULK_WARPS 4              // warps per CTA (independent: no shared memory, no barrier)

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

// The pair kernel's shared-memory row ring (swe_ca_bulk_pair, b2_swe_ca.cu): the step-1 warp's rows of
// h, u, v, dh, du, dv, CA_RING_SLOTS rows per field, row j in slot j % CA_RING_SLOTS.  A ring row is the
// warp strip's 128 columns with 4 floats of padding on each side (lane l's group at 4 + 4 l), so that the
// west / east neighbours of lanes 0 and 31 are addressable.
#define CA_RING_SLOTS 8
#define CA_RING_PITCH 136
#define CA_RING_FIELD (CA_RING_SLOTS * CA_RING_PITCH)
#define CA_RING_FLOATS (6 * CA_RING_FIELD)
enum { CA_RH = 0, CA_RU, CA_RV, CA_RDH, CA_RDU, CA_RDV };

// where a launch's warps go: its store window and how its warps tile it
struct CAWin {
  int ng;                                            // bulk groups per row: columns [4, 4 + 4 ng)
  int r0, r1, g0, g1;                                // store window: rows [r0, r1) x groups [g0, g1)
  int halo;                                          // lanes on each side of a strip that do not store
  int rows;                                          // rows per segment
  int wcols;                                         // warp strips per row of segments
  int nseg;                                          // segments: window rows [r0, r1)
};
struct CABulkArgs : CAWin {
  B2SweParams p;
  const float *h, *u, *v, *du, *dv;                  // this step
  float *h_o, *u_o, *v_o, *du_o, *dv_o;              // the next step
  float* dh;                                         // the next step's dh (own cells only)
  const float* dh_src = nullptr;                     // this step's dh; null: dh, updated in place
};

// geometry of a launch over the window [r0, r1) x [g0, g1): a warp's (segment, strip), a lane's group.
// The one-step kernel over the whole bulk is the window [4, ny - 4) x [0, ng) with halo 1.
__host__ __device__ inline void ca_bulk_window(int cb1, int r0, int r1, int g0, int g1, int halo, int rows,
                                               CAWin& a) {
  a.ng = (cb1 >> 2) - 1;
  a.r0 = r0; a.r1 = r1; a.g0 = g0; a.g1 = g1; a.halo = halo;
  a.rows = rows;
  a.wcols = (g1 - g0 + 32 - 2 * halo - 1) / (32 - 2 * halo);
  a.nseg = (r1 - r0 + rows - 1) / rows;
}
__host__ __device__ inline void ca_bulk_geometry(const B2SweParams& p, int cb1, int rows, CAWin& a) {
  ca_bulk_window(cb1, 4, p.ny - 4, 0, (cb1 >> 2) - 1, 1, rows, a);
}
__host__ __device__ inline long long ca_bulk_warps(const CAWin& a) { return (long long)a.wcols * a.nseg; }
// group index of `lane` in strip `wc`; lanes beyond the groups the window's stored lanes need repeat the
// last of them (at most ng, the group east of the bulk), so a narrow window loads few distinct columns;
// the lane stores when it returns true
__host__ __device__ inline bool ca_bulk_lane(const CAWin& a, int wc, int lane, int& i0) {
  int g = a.g0 + wc * (32 - 2 * a.halo) + lane - a.halo;
  const int ghi = a.g1 + a.halo - 1 < a.ng ? a.g1 + a.halo - 1 : a.ng;
  if (g > ghi) g = ghi;
  if (g < -1) g = -1;
  i0 = 4 + 4 * g;
  return lane >= a.halo && lane < 32 - a.halo && g < a.g1;
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
  int ic;                                            // the lane's group in a ring row (pair kernel)
  bool store;                                        // this lane's group is stored to the arrays
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
__host__ __device__ inline void ca_bulk_rows(const CAWin& a, int seg, int& s, int& e) {
  s = a.r0 + seg * a.rows;
  e = s + a.rows < a.r1 ? s + a.rows : a.r1;
}

// The pair kernel's step-1 lane (segment `seg`, strip `wc` of the inner bulk `b`) also stores state t+1
// to the arrays where the ring launch and the frame kernels of step t+1 read it: rows < 10 and >= ny-11
// (the ring launch's row windows [4, 8) and [ny-7, ny-4) reach 2 rows north, 4 south) and groups 0, 1,
// ng-2, ng-1 (the side windows' groups and their neighbours).  Each such cell is stored by one lane: the
// owner of its row and group under step 2's partition, extended to rows [4, 8) for the first segment, to
// rows [ny-7, ny-4) for the last, and to groups 0 and ng-1 for the outer strips.  Sets L.store.
struct CAPairBand {
  bool band_g;                                       // the lane's group is a band group
  int lo, hi;                                        // rows the lane owns
};
__host__ __device__ inline CAPairBand ca_pair_band(const CABulkArgs& b, int seg, int wc, int lane, bool own,
                                                   CABulkLane& L) {
  const int g = (L.i0 - 4) >> 2;
  L.store = own || (g == 0 && wc == 0 && lane == 2) || (g == b.g1 && wc == b.wcols - 1);
  int s, e;
  ca_bulk_rows(b, seg, s, e);
  CAPairBand r;
  r.band_g = g < 2 || g >= b.ng - 2;
  r.lo = seg == 0 ? s - 4 : s;
  r.hi = seg == b.nseg - 1 ? e + 3 : e;
  return r;
}
__host__ __device__ __forceinline__ bool ca_pair_hbm(const CAPairBand& B, int ny, int r) {
  return r >= B.lo && r < B.hi && (B.band_g || r < 10 || r >= ny - 11);
}

// Row j of an input field: from the (ny, pitch) array `x` or (RING) from field `f` of the ring.
__host__ __device__ __forceinline__ int ca_ring_off(const CABulkLane& L, int f, int j) {
  return f * CA_RING_FIELD + (j & (CA_RING_SLOTS - 1)) * CA_RING_PITCH + L.ic;
}
template <bool RING>
__device__ __forceinline__ Row6A ca_ld_row(const CABulkArgs& a, const CABulkLane& L, const float* x,
                                           const float* ring, int f, int j) {
  if (!RING) return ld_row_a(x, j, L.i0, a.p.pitch);
  const int o = ca_ring_off(L, f, j);
  const float4 c = ld4(ring, o);
  Row6A r;
  r.a[0] = ring[o - 1]; r.a[1] = c.x; r.a[2] = c.y; r.a[3] = c.z; r.a[4] = c.w; r.a[5] = ring[o + 4];
  return r;
}
// (`off`: the lane's group in row j of the arrays)
template <bool RING>
__device__ __forceinline__ float4 ca_ld4(const CABulkLane& L, const float* x, size_t off, const float* ring, int f,
                                         int j) {
  return RING ? ld4(ring, ca_ring_off(L, f, j)) : ld4(x, off);
}
// Row j of an output field: to the array `x` where `hbm` (and the lane stores), and (RING) to the ring.
template <bool RING>
__device__ __forceinline__ void ca_st4(const CABulkLane& L, float* x, size_t off, float* ring, int f, int j,
                                       bool hbm, float4 v) {
  if (RING) st4(ring, ca_ring_off(L, f, j), v);
  if (hbm && L.store) st4(x, off, v);
}

// rows s-4 .. s-1 and the fluxes of rows s-3, s-2 of the segment starting at row s
template <bool IN_RING = false>
__device__ __forceinline__ void ca_bulk_begin(const CABulkArgs& a, CABulkLane& L, int s, const float* ring = nullptr) {
  const int t = s - 2;
  const Row6A Vs = ca_ld_row<IN_RING>(a, L, a.v, ring, CA_RV, t - 2);
  L.H[0] = ca_ld_row<IN_RING>(a, L, a.h, ring, CA_RH, t - 1); L.U[0] = ca_ld_row<IN_RING>(a, L, a.u, ring, CA_RU, t - 1);
  L.V[0] = ca_ld_row<IN_RING>(a, L, a.v, ring, CA_RV, t - 1);
  L.H[1] = ca_ld_row<IN_RING>(a, L, a.h, ring, CA_RH, t); L.U[1] = ca_ld_row<IN_RING>(a, L, a.u, ring, CA_RU, t);
  L.V[1] = ca_ld_row<IN_RING>(a, L, a.v, ring, CA_RV, t);
  L.H[2] = ca_ld_row<IN_RING>(a, L, a.h, ring, CA_RH, t + 1); L.U[2] = ca_ld_row<IN_RING>(a, L, a.u, ring, CA_RU, t + 1);
  L.V[2] = ca_ld_row<IN_RING>(a, L, a.v, ring, CA_RV, t + 1);
  ca_bulk_fluxes(a.p, a.p.coriolis[t - 1], L.H[0], L.U[0], L.V[0], L.H[1], L.U[1], Vs, L.Fm);
  ca_bulk_fluxes(a.p, a.p.coriolis[t], L.H[1], L.U[1], L.V[1], L.H[2], L.U[2], L.V[0], L.Fc);
  // slots 0, 1 = rows t, t+1 (ca_bulk_tend loads row t+2 into slot 2)
  L.H[0] = L.H[1]; L.U[0] = L.U[1]; L.V[0] = L.V[1];
  L.H[1] = L.H[2]; L.U[1] = L.U[2]; L.V[1] = L.V[2];
  L.dh4 = L.du4 = L.dv4 = make_float4(0.f, 0.f, 0.f, 0.f);
}

// phase 1 of row t: load row t+2 and the old tendencies, fluxes of row t+1, tendency + update of row t;
// stores h', dh, du, dv when `out` (row t is one of the segment's rows): to the ring (OUT_RING), and to
// the arrays where `hbm` as well
template <bool IN_RING = false, bool OUT_RING = false>
__device__ __forceinline__ void ca_bulk_tend(const CABulkArgs& a, CABulkLane& L, int t, bool out,
                                             float* ring = nullptr, bool hbm = true) {
  const B2SweParams& p = a.p;
  const size_t off = (size_t)t * p.pitch + L.i0;
  L.H[2] = ca_ld_row<IN_RING>(a, L, a.h, ring, CA_RH, t + 2);
  L.U[2] = ca_ld_row<IN_RING>(a, L, a.u, ring, CA_RU, t + 2);
  L.V[2] = ca_ld_row<IN_RING>(a, L, a.v, ring, CA_RV, t + 2);
  if (!p.first_step) {
    L.du4 = ca_ld4<IN_RING>(L, a.du, off, ring, CA_RDU, t); L.dv4 = ca_ld4<IN_RING>(L, a.dv, off, ring, CA_RDV, t);
    if (out)                                         // (rows above / below the segment: h' is not stored)
      L.dh4 = ca_ld4<IN_RING>(L, a.dh_src != nullptr ? a.dh_src : a.dh, off, ring, CA_RDH, t);
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
  if (out) {
    ca_st4<OUT_RING>(L, a.h_o, off, ring, CA_RH, t, hbm, make_float4(Hn[0], Hn[1], Hn[2], Hn[3]));
    ca_st4<OUT_RING>(L, a.dh, off, ring, CA_RDH, t, hbm, make_float4(DH[0], DH[1], DH[2], DH[3]));
    ca_st4<OUT_RING>(L, a.du_o, off, ring, CA_RDU, t, hbm, make_float4(DU[0], DU[1], DU[2], DU[3]));
    ca_st4<OUT_RING>(L, a.dv_o, off, ring, CA_RDV, t, hbm, make_float4(DV[0], DV[1], DV[2], DV[3]));
  }
  L.H[0] = L.H[1]; L.U[0] = L.U[1]; L.V[0] = L.V[1];
  L.H[1] = L.H[2]; L.U[1] = L.U[2]; L.V[1] = L.V[2];
  L.Fm = L.Fc; L.Fc = Fp;
}

// phase 2 of row t: friction of row r = t-1 (swe_k34_body's u update and fluxes, swe_k5_body's v update)
// given the west lane's u' of row t at columns i0-2, i0-1 and the east lane's u', v' at i0+4.
// `upp_only`: row r lies above the segment, only its u'' is needed (the south flux of the next row);
// `out`: row r is one of the segment's rows, u'' and v'' are stored (ring and `hbm` as in ca_bulk_tend).
template <bool OUT_RING = false>
__device__ __forceinline__ void ca_bulk_fric(const CABulkArgs& a, CABulkLane& L, int t, float uw2, float uw3,
                                             float ue, float ve, bool upp_only, bool out, float* ring = nullptr,
                                             bool hbm = true) {
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
    if (out && (OUT_RING || L.store)) {
      float Vn[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float fn2_c = swe_visc_flux(p.c_nuy, vp2[k], UPP[k + 1]);     // fn2[r][i]
        const float fn2_s = swe_visc_flux(p.c_nuy, L.vp1[k], L.upp1[k]);    // fn2[r-1][i]
        Vn[k] = swe_apply_div(p, L.vp1[k], FE2[k + 1], FE2[k], fn2_c, fn2_s);
      }
      const size_t off = (size_t)(t - 1) * p.pitch + L.i0;
      ca_st4<OUT_RING>(L, a.u_o, off, ring, CA_RU, t - 1, hbm, make_float4(UPP[1], UPP[2], UPP[3], UPP[4]));
      ca_st4<OUT_RING>(L, a.v_o, off, ring, CA_RV, t - 1, hbm, make_float4(Vn[0], Vn[1], Vn[2], Vn[3]));
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) L.upp1[k] = UPP[k + 1];
  }
#pragma unroll
  for (int x = 0; x < 7; ++x) { L.up0[x] = L.up1[x]; L.up1[x] = up2[x]; }
#pragma unroll
  for (int x = 0; x < 5; ++x) L.vp1[x] = vp2[x];
}
