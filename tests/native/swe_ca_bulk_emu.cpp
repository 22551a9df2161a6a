// Host emulation of the communication-avoiding step as b2_swe_multistep_ca launches it: the one-pass
// bulk kernel swe_ca_bulk_step (csrc/b2_swe_k12_body.cuh) with its 32 lanes in lockstep, and the frame
// kernels with ping-pong storage.  Builds on swe_host_emu.cpp (same compiler setup, exchange geometry).
// Build: g++ -O1 -ffp-contract=off -shared -fPIC -I csrc -I $CUDA/include tests/native/swe_ca_bulk_emu.cpp
#include "swe_host_emu.cpp"

struct EmuStepPP {    // one rank's arrays for one step, B2SweState roles of b2_swe_multistep_ca
  const float *h, *u, *v, *du, *dv;            // this step
  float *h_o, *u_o, *v_o, *du_o, *dv_o;        // the next step (ping-pong partners)
  float *dh, *upf, *vpf;
};

static CACtx make_ctx_pp(const B2SweParams* p, const B2SweCA* x, const EmuStepPP* e) {
  CACtx c;
  c.p = *p; c.x = *x; c.x.cb1 = swe_ca_cb1(*p);
  c.h = e->h; c.hn = e->h_o; c.ua = e->u; c.va = e->v; c.dh = e->dh;
  c.du = const_cast<float*>(e->du); c.dv = const_cast<float*>(e->dv);
  c.dub = c.dvb = nullptr; c.du_o = e->du_o; c.dv_o = e->dv_o;
  c.upf = e->upf; c.vpf = e->vpf;
  return c;
}

static CABulkArgs bulk_args(const B2SweParams* p, const EmuStepPP* e, int rows) {
  CABulkArgs a;
  a.p = *p;
  ca_bulk_geometry(*p, swe_ca_cb1(*p), rows, a);
  a.h = e->h; a.u = e->u; a.v = e->v; a.du = e->du; a.dv = e->dv;
  a.h_o = e->h_o; a.u_o = e->u_o; a.v_o = e->v_o; a.du_o = e->du_o; a.dv_o = e->dv_o;
  a.dh = e->dh;
  return a;
}

extern "C" {

// kernel A / kernel D (ping-pong layout); `reverse` walks the tasks backwards
void emu_pp_tend_frame(const B2SweParams* p, const B2SweCA* x, const EmuStepPP* e, int reverse) {
  const CACtx c = make_ctx_pp(p, x, e);
  const CAFrame f = ca_frame(c.p, 5, c.x.cb1 - 2);
  for (long long k = 0; k < f.total; ++k) {
    int j, i;
    if (ca_frame_cell(c.p, f, (int)(reverse ? f.total - 1 - k : k), j, i)) swe_ca_tend_cell(c, j, i);
  }
}
void emu_pp_fric_frame(const B2SweParams* p, const B2SweCA* x, const EmuStepPP* e, int reverse) {
  const CACtx c = make_ctx_pp(p, x, e);
  const CAFrame f = ca_frame(c.p, 3, c.x.cb1);
  const long long n = f.total + ca_ext_total(c.p);
  for (long long k = 0; k < n; ++k) swe_ca_fric_task(c, f, e->u_o, e->v_o, reverse ? n - 1 - k : k);
}

// swe_ca_bulk_step with `rows` rows per segment: warps one after the other (`reverse`: backwards), the
// 32 lanes of a warp in lockstep, every phase of a row as a loop over the lanes; the lane exchange is
// __shfl_up_sync / __shfl_down_sync by one lane (a lane without a partner gets its own value)
void emu_ca_bulk_step(const B2SweParams* p, const EmuStepPP* e, int rows, int reverse) {
  const CABulkArgs a = bulk_args(p, e, rows);
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

// how often swe_ca_bulk_step stores each interior cell: counts[j * nx + i]
void emu_ca_bulk_step_counts(const B2SweParams* p, int rows, int* counts) {
  CABulkArgs a;
  a.p = *p;
  ca_bulk_geometry(*p, swe_ca_cb1(*p), rows, a);
  for (long long w = 0; w < ca_bulk_warps(a); ++w) {
    int s, e;
    ca_bulk_rows(a, (int)(w / a.wcols), s, e);
    for (int l = 0; l < 32; ++l) {
      int i0;
      if (!ca_bulk_lane(a, (int)(w % a.wcols), l, i0)) continue;
      for (int j = s; j < e; ++j)
        for (int k = 0; k < 4; ++k) counts[j * p->nx + i0 + k] += 1;
    }
  }
}

}  // extern "C"
