// Host emulation of the shallow-water stencil bodies (csrc/b2_swe_body.cuh, b2_swe_ca_bulk.cuh,
// b2_swe_ca_body.cuh): the same source, compiled by g++ with the CUDA qualifiers defined away, driven
// by plain loops instead of a grid.  Lets the CPU test-suite check the INDEXING of kernels it cannot
// launch -- in particular the communication-avoiding step as b2_swe_multistep_ca launches it (one-pass
// bulk kernel with its 32 lanes in lockstep, frame kernels with owner views, deep halo exchange
// geometry, bulk / frame partition, ping-pong storage) against the stand-alone K1 -> K2 -> K34 -> K5
// pipeline, bit for bit (every rounding in the bodies is explicit, so host and device agree on the
// arithmetic).  The halo exchanges' message geometry and receive rules (csrc/b2_halo_geom.h) are
// compiled here as well.
// Build: g++ -O1 -ffp-contract=off -shared -fPIC -I csrc -I $CUDA/include tests/native/swe_host_emu.cpp
#include <cmath>
#include <cstring>
#include <cuda_runtime.h>

static inline float __fmul_rn(float a, float b) { return a * b; }
static inline float __fadd_rn(float a, float b) { return a + b; }
static inline float __fmaf_rn(float a, float b, float c) { return fmaf(a, b, c); }
static inline float __frcp_rn(float a) { return 1.0f / a; }      // correctly rounded, like the intrinsic

// swe_map is grid-based; the harness enumerates (j, group) itself
struct FakeIdx { unsigned x; };
static FakeIdx blockIdx, threadIdx;

#include "b2_swe_ca_body.cuh"
#include "b2_swe_ca_bulk.cuh"

static void masks(const B2SweParams& p, int i0, bool m[4]) {
  for (int k = 0; k < 4; ++k) m[k] = (i0 + k >= 1) && (i0 + k <= p.nx - 2);
}

struct EmuStep {      // one rank's arrays for one step, B2SweState roles of b2_swe_multistep_ca
  const float *h, *u, *v, *du, *dv;            // this step
  float *h_o, *u_o, *v_o, *du_o, *dv_o;        // the next step (ping-pong partners)
  float *dh, *upf, *vpf;
};

extern "C" {

// the ABI structs as this compiler lays them out
int emu_sizeof_swe_params() { return (int)sizeof(B2SweParams); }
int emu_sizeof_swe_ca() { return (int)sizeof(B2SweCA); }

// K1 on every interior row / group (what swe_k1_fluxes does)
void emu_k1_all(const B2SweParams* p, const float* h, const float* u, const float* v, float* fe, float* fn,
                float* q, float* ke) {
  for (int j = 1; j <= p->ny - 2; ++j)
    for (int i0 = 0; i0 < p->pitch; i0 += 4) {
      bool m[4];
      masks(*p, i0, m);
      if (!(m[0] || m[1] || m[2] || m[3])) continue;
      swe_k1_body(*p, h, u, v, fe, fn, q, ke, j, i0, m);
    }
}

// K2 everywhere, in place on u, v like swe_k2_tendencies
void emu_k2_all(const B2SweParams* p, const float* h, float* h_new, float* u, float* v, float* dh, float* du,
                float* dv, const float* fe, const float* fn, const float* q, const float* ke) {
  for (int j = 1; j <= p->ny - 2; ++j)
    for (int i0 = 0; i0 < p->pitch; i0 += 4) {
      bool m[4];
      masks(*p, i0, m);
      if (!(m[0] || m[1] || m[2] || m[3])) continue;
      swe_k2_body(*p, h, h_new, u, v, dh, du, dv, fe, fn, q, ke, j, i0, m);
    }
}

void emu_k5(const B2SweParams* p, float* v, const float* fe2, const float* fn2) {
  for (int j = 1; j <= p->ny - 2; ++j)
    for (int i0 = 0; i0 < p->pitch; i0 += 4) {
      bool m[4];
      masks(*p, i0, m);
      if (!(m[0] || m[1] || m[2] || m[3])) continue;
      swe_k5_body(*p, v, fe2, fn2, j, i0, m);
    }
}

// merged friction kernel: u -> u_new, friction-v fluxes (swe_k34_friction_u)
void emu_k34(const B2SweParams* p, const float* u, float* u_new, const float* v, float* fe2, float* fn2,
             int has_south) {
  for (int j = 1; j <= p->ny - 2; ++j)
    for (int i0 = 0; i0 < p->pitch; i0 += 4) {
      bool m[4];
      masks(*p, i0, m);
      if (!(m[0] || m[1] || m[2] || m[3]) && i0 != p->nx - 1) continue;     // (swe_k34_friction_u's groups)
      swe_k34_body(*p, u, u_new, v, fe2, fn2, j, i0, m, has_south != 0);
    }
}

// ---- communication-avoiding step (csrc/b2_swe_ca_body.cuh, b2_swe_ca_bulk.cuh): the kernels of
// b2_swe_ca.cu as loops.  `reverse` walks the tasks backwards: a kernel whose threads only read what no
// thread of the same launch (or phase) writes gives the same bits in any order.
static CACtx make_ctx(const B2SweParams* p, const B2SweCA* x, const EmuStep* e) {
  CACtx c;
  c.p = *p; c.x = *x; c.x.cb1 = swe_ca_cb1(*p);
  c.h = e->h; c.hn = e->h_o; c.ua = e->u; c.va = e->v; c.dh = e->dh;
  c.du = e->du; c.dv = e->dv; c.du_o = e->du_o; c.dv_o = e->dv_o;
  c.upf = e->upf; c.vpf = e->vpf;
  return c;
}

static CABulkArgs bulk_args(const B2SweParams* p, int rows) {
  CABulkArgs a;
  a.p = *p;
  ca_bulk_geometry(*p, swe_ca_cb1(*p), rows, a);
  return a;
}

int emu_ca_supported(const B2SweParams* p) { return swe_ca_supported(*p) ? 1 : 0; }

// kernel A / kernel D
void emu_ca_tend_frame(const B2SweParams* p, const B2SweCA* x, const EmuStep* e, int reverse) {
  const CACtx c = make_ctx(p, x, e);
  const CAFrame f = ca_frame(c.p, 5, c.x.cb1 - 2);
  for (long long k = 0; k < f.total; ++k) {
    int j, i;
    if (ca_frame_cell(c.p, f, (int)(reverse ? f.total - 1 - k : k), j, i)) swe_ca_tend_cell(c, j, i);
  }
}
void emu_ca_fric_frame(const B2SweParams* p, const B2SweCA* x, const EmuStep* e, int reverse) {
  const CACtx c = make_ctx(p, x, e);
  const CAFrame f = ca_frame(c.p, 3, c.x.cb1);
  const long long n = f.total + ca_ext_total(c.p);
  for (long long k = 0; k < n; ++k) swe_ca_fric_task(c, f, e->u_o, e->v_o, reverse ? n - 1 - k : k);
}

// swe_ca_bulk_step with `rows` rows per segment: warps one after the other (`reverse`: backwards), the
// 32 lanes of a warp in lockstep, every phase of a row as a loop over the lanes; the lane exchange is
// __shfl_up_sync / __shfl_down_sync by one lane (a lane without a partner gets its own value)
void emu_ca_bulk_step(const B2SweParams* p, const EmuStep* e, int rows, int reverse) {
  CABulkArgs a = bulk_args(p, rows);
  a.h = e->h; a.u = e->u; a.v = e->v; a.du = e->du; a.dv = e->dv;
  a.h_o = e->h_o; a.u_o = e->u_o; a.v_o = e->v_o; a.du_o = e->du_o; a.dv_o = e->dv_o;
  a.dh = e->dh;
  const long long nw = ca_bulk_warps(a);
  static CABulkLane L[32];
  for (long long k = 0; k < nw; ++k) {
    const int w = (int)(reverse ? nw - 1 - k : k);
    int s, en;
    ca_bulk_rows(a, w / a.wcols, s, en);
    for (int l = 0; l < 32; ++l) {
      L[l].store = ca_bulk_lane(a, w % a.wcols, l, L[l].i0);
      ca_bulk_begin(a, L[l], s);
    }
    for (int t = s - 2; t <= en; ++t) {
      float uw2[32], uw3[32], ue[32], ve[32];
      for (int l = 0; l < 32; ++l) ca_bulk_tend(a, L[l], t, t >= s && t < en);
      for (int l = 0; l < 32; ++l) {
        const int lw = l > 0 ? l - 1 : l, le = l < 31 ? l + 1 : l;
        uw2[l] = L[lw].upn[2]; uw3[l] = L[lw].upn[3];
        ue[l] = L[le].upn[0]; ve[l] = L[le].vpn[0];
      }
      for (int l = 0; l < 32; ++l) ca_bulk_fric(a, L[l], t, uw2[l], uw3[l], ue[l], ve[l], t == s, t > s);
    }
  }
}

// which interior cells do the bulk kernel (`rows` rows per segment) and the frame kernels WRITE?
// marks[j * nx + i]: +1 frame (kernel D's cells = kernel A's full updates), +16 bulk (per store),
// +256 kernel A's u' / v' band
void emu_ca_marks(const B2SweParams* p, int rows, int* marks) {
  const int cb1 = swe_ca_cb1(*p);
  const CAFrame fd = ca_frame(*p, 3, cb1), fa = ca_frame(*p, 5, cb1 - 2);
  int j, i;
  for (long long t = 0; t < fd.total; ++t)
    if (ca_frame_cell(*p, fd, (int)t, j, i)) marks[j * p->nx + i] += 1;
  for (long long t = 0; t < fa.total; ++t)
    if (ca_frame_cell(*p, fa, (int)t, j, i)) marks[j * p->nx + i] += 256;
  const CABulkArgs a = bulk_args(p, rows);
  for (long long w = 0; w < ca_bulk_warps(a); ++w) {
    int s, e;
    ca_bulk_rows(a, (int)(w / a.wcols), s, e);
    for (int l = 0; l < 32; ++l) {
      int i0;
      if (!ca_bulk_lane(a, (int)(w % a.wcols), l, i0)) continue;
      for (j = s; j < e; ++j)
        for (int k = 0; k < 4; ++k) marks[j * p->nx + i0 + k] += 16;
    }
  }
}

// the message that lands on `side` of the receiver: read from the sender's arrays exactly as the push
// loop of fz_exchange (b2_halo_ll.cuh) does, received exactly as its poll loop hands it to the receive
// rule of b2_k_halo_ca (emu_ca_deliver) or of b2_k_halo_ll (emu_halo_deliver); no transport in between
void emu_ca_deliver(int ny, int nx, int pitch, int epitch, int side, int recv_has_south, int recv_has_north,
                    float* const* send_field, float* const* recv_field, float* const* recv_ext) {
  const int jlo = recv_has_south ? 1 : 0, jhi = recv_has_north ? ny - 1 : ny;
  for (int e = 0; e < ca_msg_count(ny, nx, side); ++e) {
    int f, js, is, jr, ir, layer;
    ca_msg_elem(ny, nx, side, e, f, js, is, jr, ir, layer);
    ca_scatter(ny, nx, (size_t)pitch, epitch, side, e, jlo, jhi, send_field[f][(size_t)js * pitch + is], recv_field,
               recv_ext);
  }
}
void emu_halo_deliver(int ny, int nx, int pitch, int nf, const int* kind, int side, int recv_has_south,
                      int recv_has_north, int uwall, int vwall, float* const* send_field, float* const* recv_field) {
  const int jlo = recv_has_south ? 1 : 0, jhi = recv_has_north ? ny - 1 : ny;
  for (int e = 0; e < halo_msg_count(nf, 1, ny, nx, side); ++e) {
    int f, js, is, jr, ir, layer;
    halo_msg_elem(1, ny, nx, side, e, f, js, is, jr, ir, layer);
    halo_recv_walls(ny, nx, (size_t)pitch, side, e, jlo, jhi, uwall != 0, vwall != 0,
                    send_field[f][(size_t)js * pitch + is], recv_field, kind);
  }
}
// b2_k_halo_ll's closing wall pass, one thread
void emu_halo_wall_pass(int ny, int nx, int pitch, int nf, const int* kind, int has_west, int has_east, int has_south,
                        int has_north, int uwall, int vwall, float* const* field) {
  halo_wall_pass(ny, nx, (size_t)pitch, nf, has_south ? 1 : 0, has_north ? ny - 1 : ny, has_west ? 1 : 0,
                 has_east ? nx - 1 : nx, uwall != 0, vwall != 0, field, kind, 0, 1);
}

// swe_ca_init_ext
void emu_ca_init_ext(const B2SweParams* p, const B2SweCA* x, const float* u, const float* v) {
  int j, i;
  for (long long t = 0; t < ca_ext_total(*p); ++t)
    if (ca_ext_cell(*p, t, j, i)) {
      const size_t e = ca_e(*x, j, i);
      x->uppx[e] = x->upx[e];
      x->vppx[e] = x->vpx[e];
    }
  for (j = 1; j <= p->ny - 2; ++j)
    for (i = 1; i <= p->nx - 2; ++i)
      if (j == 1 || j == p->ny - 2 || i == 1 || i == p->nx - 2) {
        x->upx[ca_e(*x, j, i)] = u[ca_m(*p, j, i)];
        x->vpx[ca_e(*x, j, i)] = v[ca_m(*p, j, i)];
      }
}

}  // extern "C"
