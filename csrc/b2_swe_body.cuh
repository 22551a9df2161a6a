// mpi4jax_b200 -- shallow-water stencil bodies shared by every launch schedule: the stand-alone
// kernels (b2_swe.cu), the one-pass bulk kernel (b2_swe_ca_bulk.cuh) and the
// scalar frame kernels of the communication-avoiding step (b2_swe_ca_body.cuh).
// Each vector body handles one aligned group of 4 cells of row j: loads, arithmetic, vector stores.
//
// Every rounding is spelled out with __fmul_rn / __fadd_rn / __fmaf_rn (never contracted or split by
// ptxas), so an expression gives the same bits in whatever kernel it is inlined -- which is what
// lets a kernel that RECOMPUTES a quantity at its stencil neighbours agree to the bit with one that
// reads it from memory, and lets the tests compare launch schedules with torch.equal.  The forms
// are chosen for instruction count (the fused kernels are issue-bound, not bandwidth-bound):
// constant factors are folded on the host (B2SweParams::c_*), sums of products are FMA chains.
#pragma once

#include "b2_runtime.h"

#define SWE_THREADS 256

// An aligned group of four cells plus its west / east neighbours.
struct Row6 {
  float w, c0, c1, c2, c3, e;
};

__device__ __forceinline__ float4 ld4(const float* __restrict__ a, size_t off) {
  return *reinterpret_cast<const float4*>(a + off);
}
__device__ __forceinline__ void st4(float* __restrict__ a, size_t off, float4 v) {
  *reinterpret_cast<float4*>(a + off) = v;
}
// row `j`, group starting at column i0 (multiple of 4); neighbours are fetched only when asked
template <bool W, bool E>
__device__ __forceinline__ Row6 ld_row(const float* __restrict__ a, int j, int i0, int pitch) {
  const size_t off = (size_t)j * pitch + i0;
  const float4 v = ld4(a, off);
  Row6 r;
  r.c0 = v.x; r.c1 = v.y; r.c2 = v.z; r.c3 = v.w;
  r.w = (W && i0 > 0) ? a[off - 1] : 0.f;
  r.e = (E && i0 + 4 < pitch) ? a[off + 4] : 0.f;
  return r;
}

// thread -> (row j in [1, ny-2], group g); returns false when out of range
__device__ __forceinline__ bool swe_map(const B2SweParams& p, int& j, int& i0, bool m[4]) {
  const int ngroups = p.pitch >> 2;
  const long long idx = (long long)blockIdx.x * SWE_THREADS + threadIdx.x;
  if (idx >= (long long)(p.ny - 2) * ngroups) return false;
  j = (int)(idx / ngroups) + 1;
  i0 = (int)(idx % ngroups) << 2;
#pragma unroll
  for (int k = 0; k < 4; ++k) m[k] = (i0 + k >= 1) && (i0 + k <= p.nx - 2);
  return m[0] || m[1] || m[2] || m[3];
}

__host__ __device__ __forceinline__ int hc_row(const B2SweParams& p, int j) {
  // hc = h with the physical wall rows replaced by their neighbouring interior row
  if (p.south_wall && j == 0) return 1;
  if (p.north_wall && j == p.ny - 1) return p.ny - 2;
  return j;
}

// ---- flux-kernel quantities (examples/shallow_water.py:283-330) ---------------------------------
__device__ __forceinline__ float swe_fe(float h_c, float h_e, float u_c) {          // mass flux east
  return __fmul_rn(__fmul_rn(__fadd_rn(h_c, h_e), 0.5f), u_c);
}
__device__ __forceinline__ float swe_fn(float h_c, float h_n, float v_c) {          // mass flux north
  return __fmul_rn(__fmul_rn(__fadd_rn(h_c, h_n), 0.5f), v_c);
}
// potential vorticity (f + dv/dx - du/dy) / mean(h)
__device__ __forceinline__ float swe_q(const B2SweParams& p, float cor, float v_e, float v_c, float u_n,
                                       float u_c, float h_c, float h_e, float h_n, float h_ne) {
  const float rel = __fmaf_rn(__fadd_rn(v_e, -v_c), p.rdx, -__fmul_rn(__fadd_rn(u_n, -u_c), p.rdy));
  const float den = __fmul_rn(__fadd_rn(__fadd_rn(h_c, h_e), __fadd_rn(h_n, h_ne)), 0.25f);
  return __fmul_rn(__fadd_rn(cor, rel), __frcp_rn(den));
}
// kinetic energy (u_c^2 + u_w^2 + v_c^2 + v_s^2) / 4
__device__ __forceinline__ float swe_ke(float u_c, float u_w, float v_c, float v_s) {
  const float s = __fmaf_rn(v_s, v_s, __fmaf_rn(v_c, v_c, __fmaf_rn(u_w, u_w, __fmul_rn(u_c, u_c))));
  return __fmul_rn(s, 0.25f);
}

__device__ __forceinline__ void swe_k1_body(const B2SweParams& p, const float* __restrict__ h,
                                            const float* __restrict__ u, const float* __restrict__ v,
                                            float* __restrict__ fe, float* __restrict__ fn,
                                            float* __restrict__ q, float* __restrict__ ke, int j,
                                            int i0, const bool m[4]) {
  const int P = p.pitch;
  const Row6 hc = ld_row<false, true>(h, hc_row(p, j), i0, P);
  const Row6 hn = ld_row<false, true>(h, hc_row(p, j + 1), i0, P);
  const Row6 uc = ld_row<true, false>(u, j, i0, P);
  const Row6 un = ld_row<false, false>(u, j + 1, i0, P);
  const Row6 vc = ld_row<false, true>(v, j, i0, P);
  const Row6 vs = ld_row<false, false>(v, j - 1, i0, P);
  const float cor = p.coriolis[j];
  const float H[5] = {hc.c0, hc.c1, hc.c2, hc.c3, hc.e}, HN[5] = {hn.c0, hn.c1, hn.c2, hn.c3, hn.e};
  const float U[5] = {uc.w, uc.c0, uc.c1, uc.c2, uc.c3}, UN[4] = {un.c0, un.c1, un.c2, un.c3};
  const float V[5] = {vc.c0, vc.c1, vc.c2, vc.c3, vc.e}, VS[4] = {vs.c0, vs.c1, vs.c2, vs.c3};
  float FE[4], FN[4], Q[4], KE[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float uk = U[k + 1], vk = V[k];
    FE[k] = swe_fe(H[k], H[k + 1], uk);
    FN[k] = swe_fn(H[k], HN[k], vk);
    Q[k] = swe_q(p, cor, V[k + 1], vk, UN[k], uk, H[k], H[k + 1], HN[k], HN[k + 1]);
    KE[k] = swe_ke(uk, U[k], vk, VS[k]);
    if (!m[k]) FE[k] = FN[k] = Q[k] = KE[k] = 0.f;   // halo / pad lanes: refreshed by the exchange
    if (p.north_wall && j == p.ny - 2) FN[k] = 0.f;    // "v" wall rule (shallow_water.py:261-262)
  }
  const size_t off = (size_t)j * P + i0;
  st4(fe, off, make_float4(FE[0], FE[1], FE[2], FE[3]));
  st4(fn, off, make_float4(FN[0], FN[1], FN[2], FN[3]));
  st4(q, off, make_float4(Q[0], Q[1], Q[2], Q[3]));
  st4(ke, off, make_float4(KE[0], KE[1], KE[2], KE[3]));
}

// ---- tendencies + Adams-Bashforth update of one cell (shallow_water.py:290-356) ----------------
struct SweK2In {
  float fe_c, fe_w, fen_c, fen_w;      // fe[j][i], fe[j][i-1], fe[j+1][i], fe[j+1][i-1]
  float fn_c, fn_e, fns_c, fns_e;      // fn[j][i], fn[j][i+1], fn[j-1][i], fn[j-1][i+1]
  float q_c, q_w, qs_c;                // q[j][i], q[j][i-1], q[j-1][i]
  float ke_c, ke_e, ken_c;             // ke[j][i], ke[j][i+1], ke[j+1][i]
  float h_c, h_e, h_n;                 // h[j][i], h[j][i+1], h[j+1][i]
  float u_o, v_o, dh_o, du_o, dv_o;    // own cell, old values
};
struct SweK2Out {
  float h, u, v, dh, du, dv;
};

__device__ __forceinline__ SweK2Out swe_k2_cell(const B2SweParams& p, const SweK2In& x) {
  // dh = -(fe_c - fe_w) / dx - (fn_c - fn_s) / dy
  const float dh_new = __fmaf_rn(__fadd_rn(x.fns_c, -x.fn_c), p.rdy, __fmul_rn(__fadd_rn(x.fe_w, -x.fe_c), p.rdx));
  // du = -g (h_e - h_c) / dx + (q_c (fn_c + fn_e) + q_s (fn_s + fn_se)) / 4 - (ke_e - ke_c) / dx
  const float su = __fmaf_rn(x.q_c, __fadd_rn(x.fn_c, x.fn_e), __fmul_rn(x.qs_c, __fadd_rn(x.fns_c, x.fns_e)));
  float du_new = __fmaf_rn(0.25f, su, __fmul_rn(p.c_gx, __fadd_rn(x.h_e, -x.h_c)));
  du_new = __fmaf_rn(__fadd_rn(x.ke_c, -x.ke_e), p.rdx, du_new);
  // dv = -g (h_n - h_c) / dy - (q_c (fe_c + fe_n) + q_w (fe_w + fe_nw)) / 4 - (ke_n - ke_c) / dy
  const float sv = __fmaf_rn(x.q_c, __fadd_rn(x.fe_c, x.fen_c), __fmul_rn(x.q_w, __fadd_rn(x.fe_w, x.fen_w)));
  float dv_new = __fmaf_rn(-0.25f, sv, __fmul_rn(p.c_gy, __fadd_rn(x.h_n, -x.h_c)));
  dv_new = __fmaf_rn(__fadd_rn(x.ke_c, -x.ken_c), p.rdy, dv_new);
  SweK2Out o;
  if (p.first_step) {
    o.u = __fmaf_rn(p.dt, du_new, x.u_o);
    o.v = __fmaf_rn(p.dt, dv_new, x.v_o);
    o.h = __fmaf_rn(p.dt, dh_new, x.h_c);
  } else {
    o.u = __fmaf_rn(p.dt, __fmaf_rn(p.ab_a, du_new, __fmul_rn(p.ab_b, x.du_o)), x.u_o);
    o.v = __fmaf_rn(p.dt, __fmaf_rn(p.ab_a, dv_new, __fmul_rn(p.ab_b, x.dv_o)), x.v_o);
    o.h = __fmaf_rn(p.dt, __fmaf_rn(p.ab_a, dh_new, __fmul_rn(p.ab_b, x.dh_o)), x.h_c);
  }
  o.dh = dh_new; o.du = du_new; o.dv = dv_new;
  return o;
}

__device__ __forceinline__ void swe_k2_body(const B2SweParams& p, const float* __restrict__ h,
                                            float* __restrict__ h_new, float* __restrict__ u,
                                            float* __restrict__ v, float* __restrict__ dh,
                                            float* __restrict__ du, float* __restrict__ dv,
                                            const float* __restrict__ fe, const float* __restrict__ fn,
                                            const float* __restrict__ q, const float* __restrict__ ke,
                                            int j, int i0, const bool m[4]) {
  const int P = p.pitch;
  const size_t off = (size_t)j * P + i0;
  const Row6 fec = ld_row<true, false>(fe, j, i0, P), fen = ld_row<true, false>(fe, j + 1, i0, P);
  const Row6 fnc = ld_row<false, true>(fn, j, i0, P), fns = ld_row<false, true>(fn, j - 1, i0, P);
  const Row6 qc = ld_row<true, false>(q, j, i0, P), qs = ld_row<false, false>(q, j - 1, i0, P);
  const Row6 kec = ld_row<false, true>(ke, j, i0, P), ken = ld_row<false, false>(ke, j + 1, i0, P);
  const Row6 hc = ld_row<false, true>(h, j, i0, P), hn = ld_row<false, false>(h, j + 1, i0, P);
  const float4 u4 = ld4(u, off), v4 = ld4(v, off);
  float4 dh4 = make_float4(0, 0, 0, 0), du4 = dh4, dv4 = dh4;
  if (!p.first_step) { dh4 = ld4(dh, off); du4 = ld4(du, off); dv4 = ld4(dv, off); }
  const float FE[5] = {fec.w, fec.c0, fec.c1, fec.c2, fec.c3}, FEN[5] = {fen.w, fen.c0, fen.c1, fen.c2, fen.c3};
  const float FN[5] = {fnc.c0, fnc.c1, fnc.c2, fnc.c3, fnc.e}, FNS[5] = {fns.c0, fns.c1, fns.c2, fns.c3, fns.e};
  const float Q[5] = {qc.w, qc.c0, qc.c1, qc.c2, qc.c3}, QS[4] = {qs.c0, qs.c1, qs.c2, qs.c3};
  const float KE[5] = {kec.c0, kec.c1, kec.c2, kec.c3, kec.e}, KEN[4] = {ken.c0, ken.c1, ken.c2, ken.c3};
  const float H[5] = {hc.c0, hc.c1, hc.c2, hc.c3, hc.e}, HN[4] = {hn.c0, hn.c1, hn.c2, hn.c3};
  const float Uo[4] = {u4.x, u4.y, u4.z, u4.w}, Vo[4] = {v4.x, v4.y, v4.z, v4.w};
  const float DHo[4] = {dh4.x, dh4.y, dh4.z, dh4.w}, DUo[4] = {du4.x, du4.y, du4.z, du4.w},
              DVo[4] = {dv4.x, dv4.y, dv4.z, dv4.w};
  float Un[4], Vn[4], Hn[4], DH[4], DU[4], DV[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    SweK2In in;
    in.fe_c = FE[k + 1]; in.fe_w = FE[k]; in.fen_c = FEN[k + 1]; in.fen_w = FEN[k];
    in.fn_c = FN[k]; in.fn_e = FN[k + 1]; in.fns_c = FNS[k]; in.fns_e = FNS[k + 1];
    in.q_c = Q[k + 1]; in.q_w = Q[k]; in.qs_c = QS[k];
    in.ke_c = KE[k]; in.ke_e = KE[k + 1]; in.ken_c = KEN[k];
    in.h_c = H[k]; in.h_e = H[k + 1]; in.h_n = HN[k];
    in.u_o = Uo[k]; in.v_o = Vo[k]; in.dh_o = DHo[k]; in.du_o = DUo[k]; in.dv_o = DVo[k];
    const SweK2Out r = swe_k2_cell(p, in);
    Un[k] = r.u; Vn[k] = r.v; Hn[k] = r.h; DH[k] = r.dh; DU[k] = r.du; DV[k] = r.dv;
    if (!m[k]) { Un[k] = Uo[k]; Vn[k] = Vo[k]; Hn[k] = H[k]; DH[k] = DU[k] = DV[k] = 0.f; }
    if (p.north_wall && j == p.ny - 2) Vn[k] = 0.f;    // "v" wall rule, applied after the update
  }
  st4(u, off, make_float4(Un[0], Un[1], Un[2], Un[3]));
  st4(v, off, make_float4(Vn[0], Vn[1], Vn[2], Vn[3]));
  st4(h_new, off, make_float4(Hn[0], Hn[1], Hn[2], Hn[3]));
  st4(dh, off, make_float4(DH[0], DH[1], DH[2], DH[3]));
  st4(du, off, make_float4(DU[0], DU[1], DU[2], DU[3]));
  st4(dv, off, make_float4(DV[0], DV[1], DV[2], DV[3]));
}

// ---- friction phase (shallow_water.py:366-402) ----------------------------------------------------
// viscous flux nu (a - b) / d, with c = nu / d folded
__device__ __forceinline__ float swe_visc_flux(float c, float a, float b) {
  return __fmul_rn(__fadd_rn(a, -b), c);
}
// x + dt ((fe_c - fe_w) / dx + (fn_c - fn_s) / dy)
__device__ __forceinline__ float swe_apply_div(const B2SweParams& p, float x, float fe_c, float fe_w,
                                               float fn_c, float fn_s) {
  const float d = __fmaf_rn(__fadd_rn(fe_c, -fe_w), p.rdx, __fmul_rn(__fadd_rn(fn_c, -fn_s), p.rdy));
  return __fmaf_rn(p.dt, d, x);
}
// The friction update of u at one cell: u + dt nu (d2u/dx2 + d2u/dy2) on the 5-point stencil, the
// second differences formed from the first ones so that a flux the reference's boundary rules zero
// (fn = 0 on row ny-2 of the north-wall ranks, "v" rule; fn's south halo row = 0 on south-wall
// ranks, never received) simply drops out.
__device__ __forceinline__ float swe_friction_u(const B2SweParams& p, float u_c, float u_e, float u_w,
                                                float u_n, float u_s, bool fn_c_zero, bool fn_s_zero) {
  const float d2x = __fadd_rn(__fadd_rn(u_e, -u_c), -__fadd_rn(u_c, -u_w));
  const float dn = fn_c_zero ? 0.f : __fadd_rn(u_n, -u_c);
  const float ds = fn_s_zero ? 0.f : __fadd_rn(u_c, -u_s);
  return __fmaf_rn(p.c_fx, d2x, __fmaf_rn(p.c_fy, __fadd_rn(dn, -ds), u_c));
}

// friction-u + the friction-v fluxes in one pass (no flux round trip through HBM):
//   u_new = friction_u(u);  fe2 = nu (v[c+1] - u_new) / dx;  fn2 = nu (v[c+nx] - u_new) / dy
// (`v - u` mirrors the reference, shallow_water.py:387-392).  u is read with its 5-point
// neighbourhood, so the update must NOT be in place: u -> u_new ping-pong, like h in K2.  The halo
// rows of u_new are copies of u's, i.e. what the in-place update of the reference leaves there
// (u's halo as exchanged before the friction step).
__device__ __forceinline__ void swe_k34_body(const B2SweParams& p, const float* __restrict__ u,
                                             float* __restrict__ u_new,
                                             const float* __restrict__ v, float* __restrict__ fe2,
                                             float* __restrict__ fn2, int j, int i0, const bool m[4],
                                             bool has_south) {
  const int P = p.pitch;
  const size_t off = (size_t)j * P + i0;
  const Row6 uc = ld_row<true, true>(u, j, i0, P);
  const float4 un4 = ld4(u, off + P), us4 = ld4(u, off - P);
  const Row6 vc = ld_row<false, true>(v, j, i0, P);
  const float4 vn = ld4(v, off + P);
  const float U[6] = {uc.w, uc.c0, uc.c1, uc.c2, uc.c3, uc.e};
  const float UN[4] = {un4.x, un4.y, un4.z, un4.w}, US[4] = {us4.x, us4.y, us4.z, us4.w};
  const float V[5] = {vc.c0, vc.c1, vc.c2, vc.c3, vc.e}, VN[4] = {vn.x, vn.y, vn.z, vn.w};
  const bool fn_c_zero = p.north_wall && j == p.ny - 2;
  const bool fn_s_zero = (j == 1) && !has_south;
  float Un[4], FE2[4], FN2[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float uk = U[k + 1];
    const float un = swe_friction_u(p, uk, U[k + 2], U[k], UN[k], US[k], fn_c_zero, fn_s_zero);
    Un[k] = m[k] ? un : uk;
    FE2[k] = m[k] ? swe_visc_flux(p.c_nux, V[k + 1], un) : 0.f;
    FN2[k] = m[k] ? swe_visc_flux(p.c_nuy, VN[k], un) : 0.f;
    if (p.north_wall && j == p.ny - 2) FN2[k] = 0.f;
  }
  st4(u_new, off, make_float4(Un[0], Un[1], Un[2], Un[3]));
  st4(fe2, off, make_float4(FE2[0], FE2[1], FE2[2], FE2[3]));
  st4(fn2, off, make_float4(FN2[0], FN2[1], FN2[2], FN2[3]));
  if (j == 1) st4(u_new, (size_t)i0, us4);                                   // south halo row
  if (j == p.ny - 2) st4(u_new, (size_t)(p.ny - 1) * P + i0, un4);         // north halo row
}

__device__ __forceinline__ void swe_k5_body(const B2SweParams& p, float* __restrict__ v,
                                            const float* __restrict__ fe2,
                                            const float* __restrict__ fn2, int j, int i0,
                                            const bool m[4]) {
  const int P = p.pitch;
  const size_t off = (size_t)j * P + i0;
  const Row6 fec = ld_row<true, false>(fe2, j, i0, P);
  const float4 fnc = ld4(fn2, off), fns = ld4(fn2, off - P), v4 = ld4(v, off);
  const float FE[5] = {fec.w, fec.c0, fec.c1, fec.c2, fec.c3};
  const float FN[4] = {fnc.x, fnc.y, fnc.z, fnc.w}, FNS[4] = {fns.x, fns.y, fns.z, fns.w};
  const float Vo[4] = {v4.x, v4.y, v4.z, v4.w};
  float Vn[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float vn = swe_apply_div(p, Vo[k], FE[k + 1], FE[k], FN[k], FNS[k]);
    Vn[k] = m[k] ? vn : Vo[k];
  }
  st4(v, off, make_float4(Vn[0], Vn[1], Vn[2], Vn[3]));
}
