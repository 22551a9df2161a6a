// Host emulation of the pair schedule of the communication-avoiding shallow-water step
// (csrc/b2_swe_ca.cu: swe_ca_bulk_pair, the ring launches, the frame kernels with dh moved between
// buffers): the kernels' own source compiled by g++, as in swe_host_emu.cpp, whose entry points this
// library also exports.  The two warps of a pair run round by round with their lanes in lockstep, the
// shared-memory row ring is a host array indexed as on the device.
// Build: g++ -O1 -ffp-contract=off -shared -fPIC -I csrc -I $CUDA/include tests/native/swe_pair_emu.cpp
#include "swe_host_emu.cpp"

struct EmuIO {        // one launch's arrays: every field read from one buffer and written to another
  const float *h, *u, *v, *du, *dv;
  float *h_o, *u_o, *v_o, *du_o, *dv_o;
  const float* dh_src;                         // null: dh is updated in place
  float *dh, *upf, *vpf;
};

static void set_io(CABulkArgs& a, const EmuIO* e) {
  a.h = e->h; a.u = e->u; a.v = e->v; a.du = e->du; a.dv = e->dv;
  a.h_o = e->h_o; a.u_o = e->u_o; a.v_o = e->v_o; a.du_o = e->du_o; a.dv_o = e->dv_o;
  a.dh = e->dh; a.dh_src = e->dh_src;
}
static CACtx make_ctx_io(const B2SweParams* p, const B2SweCA* x, const EmuIO* e) {
  CACtx c;
  c.p = *p; c.x = *x; c.x.cb1 = swe_ca_cb1(*p);
  c.h = e->h; c.hn = e->h_o; c.ua = e->u; c.va = e->v;
  c.dh = e->dh; c.dh_src = e->dh_src;
  c.du = e->du; c.dv = e->dv; c.du_o = e->du_o; c.dv_o = e->dv_o;
  c.upf = e->upf; c.vpf = e->vpf;
  return c;
}

// the geometry b2_swe_multistep_ca gives its bulk launches: w = 0 the whole bulk (`rows` per segment),
// 1 the pair kernel's inner bulk (`rows`), 2 .. 5 the ring launches
static CABulkArgs window(const B2SweParams* p, int w, int rows) {
  const int cb1 = swe_ca_cb1(*p), ng = (cb1 >> 2) - 1, ny = p->ny;
  CABulkArgs a = {};
  a.p = *p;
  if (w == 0) ca_bulk_geometry(*p, cb1, rows, a);
  else if (w == 1) ca_bulk_window(cb1, 8, ny - 7, 1, ng - 1, 3, rows, a);
  else if (w == 2) ca_bulk_window(cb1, 4, 8, 0, ng, 1, 2, a);
  else if (w == 3) ca_bulk_window(cb1, ny - 7, ny - 4, 0, ng, 1, 2, a);
  else if (w == 4) ca_bulk_window(cb1, 8, ny - 7, 0, 1, 1, 2, a);
  else ca_bulk_window(cb1, 8, ny - 7, ng - 1, ng, 1, 2, a);
  return a;
}

// one round of a warp's walk (swe_ca_bulk_step's loop body) with its 32 lanes in lockstep
template <bool IN_RING, bool OUT_RING>
static void warp_row(const CABulkArgs& a, CABulkLane* L, int t, int s, int e, float* ring, const bool* hbm_t,
                     const bool* hbm_r) {
  float uw2[32], uw3[32], ue[32], ve[32];
  for (int l = 0; l < 32; ++l) ca_bulk_tend<IN_RING, OUT_RING>(a, L[l], t, t >= s && t < e, ring, hbm_t[l]);
  for (int l = 0; l < 32; ++l) {
    const int lw = l > 0 ? l - 1 : l, le = l < 31 ? l + 1 : l;
    uw2[l] = L[lw].upn[2]; uw3[l] = L[lw].upn[3];
    ue[l] = L[le].upn[0]; ve[l] = L[le].vpn[0];
  }
  for (int l = 0; l < 32; ++l)
    ca_bulk_fric<OUT_RING>(a, L[l], t, uw2[l], uw3[l], ue[l], ve[l], t == s, t > s, ring, hbm_r[l]);
}

extern "C" {

int emu_ca_pairs(const B2SweParams* p) { return p->ny - 7 > 8 && (swe_ca_cb1(*p) >> 2) - 1 >= 3 ? 1 : 0; }

void emu_ca_tend_frame_io(const B2SweParams* p, const B2SweCA* x, const EmuIO* e, int reverse) {
  const CACtx c = make_ctx_io(p, x, e);
  const CAFrame f = ca_frame(c.p, 5, c.x.cb1 - 2);
  for (long long k = 0; k < f.total; ++k) {
    int j, i;
    if (ca_frame_cell(c.p, f, (int)(reverse ? f.total - 1 - k : k), j, i)) swe_ca_tend_cell(c, j, i);
  }
}
void emu_ca_fric_frame_io(const B2SweParams* p, const B2SweCA* x, const EmuIO* e, int reverse) {
  const CACtx c = make_ctx_io(p, x, e);
  const CAFrame f = ca_frame(c.p, 3, c.x.cb1);
  const long long n = f.total + ca_ext_total(c.p);
  for (long long k = 0; k < n; ++k) swe_ca_fric_task(c, f, e->u_o, e->v_o, reverse ? n - 1 - k : k);
}

// swe_ca_bulk_step as launch `w` (see window()) runs it
void emu_ca_window(const B2SweParams* p, const EmuIO* e, int w, int rows, int reverse) {
  CABulkArgs a = window(p, w, rows);
  set_io(a, e);
  static CABulkLane L[32];
  bool yes[32];
  for (int l = 0; l < 32; ++l) yes[l] = true;
  const long long nw = ca_bulk_warps(a);
  for (long long k = 0; k < nw; ++k) {
    const int wi = (int)(reverse ? nw - 1 - k : k);
    int s, en;
    ca_bulk_rows(a, wi / a.wcols, s, en);
    for (int l = 0; l < 32; ++l) {
      L[l].store = ca_bulk_lane(a, wi % a.wcols, l, L[l].i0);
      ca_bulk_begin(a, L[l], s);
    }
    for (int t = s - 2; t <= en; ++t) warp_row<false, false>(a, L, t, s, en, nullptr, yes, yes);
  }
}

// swe_ca_bulk_pair: step 1 (state t from `e1`, band of state t+1 to its outputs) and step 2 (state
// t+2 to the outputs of `e2`) of each pair in the kernel's rounds, the ring a host array
void emu_ca_pair(const B2SweParams* p, const EmuIO* e1, const EmuIO* e2, int rows, int reverse) {
  CABulkArgs a = window(p, 0, 16), b = window(p, 1, rows);
  set_io(a, e1);
  set_io(b, e2);
  static CABulkLane L1[32], L2[32];
  static float ring[CA_RING_FLOATS];
  CAPairBand band[32];
  bool yes[32], hbm_t[32], hbm_r[32];
  for (int l = 0; l < 32; ++l) yes[l] = true;
  const long long nw = ca_bulk_warps(b);
  for (long long k = 0; k < nw; ++k) {
    const int w = (int)(reverse ? nw - 1 - k : k), seg = w / b.wcols, wc = w % b.wcols;
    for (int i = 0; i < CA_RING_FLOATS; ++i) ring[i] = NAN;       // (a fresh CTA's shared memory)
    int s, e;
    ca_bulk_rows(b, seg, s, e);
    const int s1 = s - 4, e1r = e + 3;
    for (int l = 0; l < 32; ++l) {
      const bool own = ca_bulk_lane(b, wc, l, L1[l].i0);
      L2[l].i0 = L1[l].i0;
      L1[l].ic = L2[l].ic = 4 + 4 * l;
      L2[l].store = own;
      band[l] = ca_pair_band(b, seg, wc, l, own, L1[l]);
      ca_bulk_begin(a, L1[l], s1);
    }
    for (int r = s1 - 2; r <= e + 4; ++r) {
      if (r <= e1r) {
        for (int l = 0; l < 32; ++l) {
          hbm_t[l] = ca_pair_hbm(band[l], p->ny, r);
          hbm_r[l] = ca_pair_hbm(band[l], p->ny, r - 1);
        }
        warp_row<false, true>(a, L1, r, s1, e1r, ring, hbm_t, hbm_r);
      }
      const int t = r - 4;
      if (r == s + 1)
        for (int l = 0; l < 32; ++l) ca_bulk_begin<true>(b, L2[l], s, ring);
      else if (t >= s - 2)
        warp_row<true, false>(b, L2, t, s, e, ring, yes, yes);
    }
  }
}

// the pair schedule's stores: marks1 (state t+1) gets +16 per cell S2's step 1 stores to the arrays,
// marks2 (state t+2) +16 per cell S2's step 2 stores and +4096 per cell a ring launch stores
void emu_ca_pair_marks(const B2SweParams* p, int rows, int* marks1, int* marks2) {
  const CABulkArgs b = window(p, 1, rows);
  for (long long w = 0; w < ca_bulk_warps(b); ++w) {
    const int seg = (int)(w / b.wcols), wc = (int)(w % b.wcols);
    int s, e;
    ca_bulk_rows(b, seg, s, e);
    for (int l = 0; l < 32; ++l) {
      CABulkLane L;
      const bool own = ca_bulk_lane(b, wc, l, L.i0);
      const CAPairBand band = ca_pair_band(b, seg, wc, l, own, L);
      for (int j = s - 4; j < e + 3; ++j)
        if (L.store && ca_pair_hbm(band, p->ny, j))
          for (int k = 0; k < 4; ++k) marks1[j * p->nx + L.i0 + k] += 16;
      if (own)
        for (int j = s; j < e; ++j)
          for (int k = 0; k < 4; ++k) marks2[j * p->nx + L.i0 + k] += 16;
    }
  }
  for (int r = 2; r < 6; ++r) {
    const CABulkArgs a = window(p, r, 2);
    for (long long w = 0; w < ca_bulk_warps(a); ++w) {
      int s, e, i0;
      ca_bulk_rows(a, (int)(w / a.wcols), s, e);
      for (int l = 0; l < 32; ++l)
        if (ca_bulk_lane(a, (int)(w % a.wcols), l, i0))
          for (int j = s; j < e; ++j)
            for (int k = 0; k < 4; ++k) marks2[j * p->nx + i0 + k] += 4096;
    }
  }
}

}  // extern "C"
