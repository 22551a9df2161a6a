// mpi4jax_b200 -- communication-avoiding shallow-water step: kernels and the two-stream schedule.
// Design, storage and the "views" that keep the reference's discrete system: b2_swe_ca_body.cuh.
//
// One model step (the reference's shallow_water_step, examples/shallow_water.py:270-403):
//
//   stream s  (bulk) :  S  flux + tendency + friction of the bulk, one pass ---------------> next step
//   stream s2 (frame):  A (tendencies, frame band) -> X (deep halo exchange) -> D (friction, frame + ext)
//
// S writes only bulk cells, A / X / D own the frame.  h, u, v, du and dv are ping-pong pairs: every
// kernel reads this step's buffers and writes the next step's, and dh is updated cell by cell by the
// kernel that owns the cell.  So the streams meet only at the step boundary: S(t+1) reads what D(t)
// wrote next to the bulk, A(t+1) what S(t) wrote next to the frame.  Seven arrays are read once and
// written once per step (12 array passes instead of the stand-alone path's 32; at 8 GPUs, 2 M cells
// per rank, the step's working set is larger than the 50 MB L2 of an H100, so passes are HBM traffic),
// one exchange instead of three, and the NVLink round of X is hidden behind S.  Under CUDA-graph
// capture (mpi4jax_b200.jit) the event fork / join becomes graph edges.

#include "b2_device.cuh"
#include "b2_halo_ll.cuh"
#include "b2_runtime.h"
#include "b2_swe_ca_body.cuh"
#include "b2_swe_k12_body.cuh"

#define CA_THREADS 256

// Optional device-side timeline (MPI4JAX_B200_SWE_TIMELINE=1, scripts/swe_timeline.py): every CTA folds
// its entry / exit %globaltimer into the [first start, last end] pair of its kernel's slot.  Unlike a
// profiler, which serialises the launches, this shows how the two streams actually overlap inside a
// CUDA-graph replay.  Null pointer = off (the default): one predictable branch per CTA.
struct CAStamp {
  unsigned long long* slot;      // {min start, max end} or null
};
__device__ __forceinline__ void ca_stamp_begin(const CAStamp& s) {
  if (s.slot != nullptr && threadIdx.x == 0) atomicMin(s.slot, b2_gtime());
}
__device__ __forceinline__ void ca_stamp_end(const CAStamp& s) {
  if (s.slot != nullptr && threadIdx.x == 0) atomicMax(s.slot + 1, b2_gtime());
}

// ---- frame kernels -------------------------------------------------------------------------------
// The frame is a few thousand cells and sits on the step's critical path: latency, not throughput.
// A thread per cell would evaluate 14 flux quantities (kernel A) or 3 friction stencils (kernel D) one
// after the other -- ~4000 dependent-issue instructions on the critical path.  Instead a CTA takes 32 cells
// and one WARP per kind of quantity: warp w evaluates the fluxes of kind w (fe / fn / q / ke; u'' of
// the cell / its west / its south neighbour in kernel D) for the 32 cells -- no divergence inside a
// warp --, the values meet in shared memory, warp 0 finishes the cells.
#define CA_CELLS 32
#define CA_TEND_WARPS 4          // one warp per flux KIND (fe, fn, q, ke): slots 0-3, 4-7, 8-10, 11-13
__global__ void __launch_bounds__(CA_CELLS * CA_TEND_WARPS)
swe_ca_tend_frame(const __grid_constant__ CACtx c, const CAFrame f, const CAStamp ts) {
  ca_stamp_begin(ts);
  __shared__ float fl[CA_NSLOT][CA_CELLS];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  int j, i;
  const bool ok = ca_frame_cell(c.p, f, (int)blockIdx.x * CA_CELLS + lane, j, i);
  if (ok) {
    float r[4];
    if (w == 0) ca_flux_kind<0>(c, j, i, r);
    else if (w == 1) ca_flux_kind<1>(c, j, i, r);
    else if (w == 2) ca_flux_kind<2>(c, j, i, r);
    else ca_flux_kind<3>(c, j, i, r);
    const int s0 = ca_slot_base(w), n = ca_slot_count(w);
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if (k < n) fl[s0 + k][lane] = r[k];
  }
  __syncthreads();
  if (ok && w == 0) {
    float v[CA_NSLOT];
#pragma unroll
    for (int s = 0; s < CA_NSLOT; ++s) v[s] = fl[s][lane];
    swe_ca_tend_finish(c, j, i, v);
  }
  ca_stamp_end(ts);
}

// friction on the frame cells (u', v' -> ua_out, va_out) and u'' / v'' of the neighbours' cells
__global__ void __launch_bounds__(CA_CELLS * 3) swe_ca_fric_frame(const CACtx c, const CAFrame f,
                                                                  float* __restrict__ ua_out,
                                                                  float* __restrict__ va_out, const CAStamp ts) {
  ca_stamp_begin(ts);
  __shared__ float up[3][CA_CELLS];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  int j, i;
  bool ext;
  const bool ok = ca_fric_task(c.p, f, (long long)blockIdx.x * CA_CELLS + lane, j, i, ext);
  if (ok && (w == 0 || ca_needs_vpp(c.p, j, i))) up[w][lane] = ca_upp_slot(c, j, i, w);
  __syncthreads();
  if (ok && w == 0) {
    const float v[3] = {up[0][lane], up[1][lane], up[2][lane]};
    if (ext) swe_ca_fric_ext_finish(c, ua_out, va_out, j, i, v);
    else swe_ca_fric_finish(c, ua_out, va_out, j, i, v);
  }
  ca_stamp_end(ts);
}

// after (re)initialising the state: no friction step has happened yet, so the "fresh" values of
// the neighbours' cells are the exchanged ones, and the stale mirror of the ring is u, v itself
__global__ void __launch_bounds__(CA_THREADS) swe_ca_init_ext(const B2SweParams p, const B2SweCA x,
                                                              const float* __restrict__ u,
                                                              const float* __restrict__ v) {
  const long long t = (long long)blockIdx.x * CA_THREADS + threadIdx.x;
  const long long next = ca_ext_total(p);
  int j, i;
  if (t < next) {
    if (!ca_ext_cell(p, t, j, i)) return;
    const size_t e = ca_e(x, j, i);
    x.uppx[e] = x.upx[e];
    x.vppx[e] = x.vpx[e];
  } else {
    const long long r = t - next;            // ring cells: rows 1, ny-2 and columns 1, nx-2
    const int nrow = 2 * (p.nx - 2);
    if (r < nrow) { j = r < p.nx - 2 ? 1 : p.ny - 2; i = 1 + (int)(r % (p.nx - 2)); }
    else {
      const long long q = r - nrow;
      if (q >= 2LL * (p.ny - 2)) return;
      j = 1 + (int)(q >> 1); i = (q & 1) ? p.nx - 2 : 1;
    }
    const size_t e = ca_e(x, j, i), off = ca_m(p, j, i);
    x.upx[e] = u[off];
    x.vpx[e] = v[off];
  }
}

// ---- S: the bulk, one pass per step (b2_swe_k12_body.cuh) ---------------------------------------
__global__ void __launch_bounds__(CA_BULK_WARPS * 32)
swe_ca_bulk_step(const CABulkArgs a, const CAStamp ts) {
  ca_stamp_begin(ts);
  const int w = (int)blockIdx.x * CA_BULK_WARPS + (int)(threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (w < ca_bulk_warps(a)) {                          // (whole warps: the lane exchange needs all 32)
    int s, e;
    ca_bulk_rows(a, w / a.wcols, s, e);
    CABulkLane L;
    L.store = ca_bulk_lane(a, w % a.wcols, lane, L.i0);
    ca_bulk_begin(a, L, s);
    for (int t = s - 2; t <= e; ++t) {
      ca_bulk_tend(a, L, t, t >= s && t < e);
      const float uw2 = __shfl_up_sync(0xffffffffu, L.upn[2], 1), uw3 = __shfl_up_sync(0xffffffffu, L.upn[3], 1);
      const float ue = __shfl_down_sync(0xffffffffu, L.upn[0], 1), ve = __shfl_down_sync(0xffffffffu, L.vpn[0], 1);
      ca_bulk_fric(a, L, t, uw2, uw3, ue, ve, t == s, t > s);
    }
  }
  ca_stamp_end(ts);
}

// ---- X: three layers of (h', u', v') to all eight neighbours, flag-in-data (b2_halo_ll.cuh) -----
// Pushes go straight from the arrays into the neighbours' receive buffers; the receiver polls the
// data itself and scatters it into the ext arrays (all layers) and the main arrays' halo (layer 1).
struct CAExt3 { float* a[CA_NF]; };

__global__ void __launch_bounds__(CA_THREADS) b2_k_halo_ca(const B2DevComm c, const B2HaloDesc d,
                                                           const CAExt3 ext, const int epitch, const CAStamp ts) {
  ca_stamp_begin(ts);
  __shared__ unsigned s_rx[FS_NSIDES], s_tx[FS_NSIDES];
  __shared__ int s_cnt[FS_NSIDES + 1];
  const int gt = blockIdx.x * blockDim.x + threadIdx.x, gn = gridDim.x * blockDim.x;
  const int ny = d.ny, nx = d.nx;
  const size_t pitch = (size_t)d.pitch;
  const int nb[FS_NSIDES] = {d.west, d.east, d.south, d.north, d.sw, d.se, d.nw, d.ne};
  const int opp[FS_NSIDES] = {CA_E, CA_W, CA_N, CA_S, CA_NE, CA_NW, CA_SE, CA_SW};
  if (threadIdx.x < FS_NSIDES) {
    s_rx[threadIdx.x] = b2_ld_volatile(c.ticket + TK_RX + threadIdx.x);
    s_tx[threadIdx.x] = b2_ld_volatile(c.ticket + TK_TX + threadIdx.x);
  }
  if (threadIdx.x == 0) {
    int acc = 0;
    for (int k = 0; k < FS_NSIDES; ++k) {
      s_cnt[k] = acc;
      if (nb[k] >= 0) acc += ca_msg_count(ny, nx, k);     // |message towards k| == |message landing on k|
    }
    s_cnt[FS_NSIDES] = acc;
  }
  __syncthreads();
  const int total = s_cnt[FS_NSIDES];
  // ---------------- push ----------------
  for (int k = gt; k < total; k += gn) {
    int s = 0;
    while (k >= s_cnt[s + 1]) ++s;
    const int e = k - s_cnt[s], land = opp[s];
    int f, js, is, jr, ir, layer;
    ca_msg_elem(ny, nx, land, e, f, js, is, jr, ir, layer);
    fz_put(fz_buf(c, nb[s], s_tx[s] & 1u, land) + e, d.field[f][(size_t)js * pitch + is], s_tx[s] + 1u);
  }
  // ---------------- poll + scatter ----------------
  const int jlo = (d.south >= 0) ? 1 : 0, jhi = (d.north >= 0) ? ny - 1 : ny;
  for (int k = gt; k < total; k += gn) {
    int s = 0;
    while (k >= s_cnt[s + 1]) ++s;
    const int e = k - s_cnt[s];
    const float val = fz_get(c, fz_buf(c, c.rank, s_rx[s] & 1u, s) + e, s_rx[s] + 1u, s);
    ca_scatter(ny, nx, pitch, epitch, s, e, jlo, jhi, val, d.field, ext.a);
  }
  fz_finish(c, nb, s_rx, s_tx);
  ca_stamp_end(ts);
}

// ---- host side --------------------------------------------------------------------------------------
static cudaStream_t g_side = nullptr;
static cudaEvent_t g_ev[3];

static int ca_streams() {
  if (g_side) return 0;
  // highest priority: the frame kernels are tiny and on the critical path, their CTAs must not queue
  // behind the thousands of CTAs of the bulk kernel running next to them
  int lo = 0, hi = 0;
  cudaDeviceGetStreamPriorityRange(&lo, &hi);
  if (cudaStreamCreateWithPriority(&g_side, cudaStreamNonBlocking, hi) != cudaSuccess) {
    b2_set_error("swe_ca: cudaStreamCreate failed");
    g_side = nullptr;
    return 1;
  }
  for (int k = 0; k < 3; ++k)
    if (cudaEventCreateWithFlags(&g_ev[k], cudaEventDisableTiming) != cudaSuccess) {
      b2_set_error("swe_ca: cudaEventCreate failed");
      return 1;
    }
  return 0;
}

static unsigned ca_blocks(long long tasks, int threads) { return (unsigned)((tasks + threads - 1) / threads); }

static int ca_check(B2Comm* c, const B2SweParams& p, const B2SweCA& x) {
  if (p.pitch % 4 != 0 || p.pitch < p.nx) {
    b2_set_error("swe_ca: the row pitch must be a multiple of 4 floats and >= nx");
    return B2_ERR_BAD_ARG;
  }
  if (x.epitch < p.nx + 4 || !x.hx || !x.upx || !x.vpx || !x.uppx || !x.vppx) {
    b2_set_error("swe_ca: ext arrays missing or too narrow (epitch %d < nx + 4)", x.epitch);
    return B2_ERR_BAD_ARG;
  }
  const size_t need = (size_t)CA_NF * CA_L * (size_t)(p.ny > p.nx ? p.ny : p.nx) * sizeof(uint2);
  if (need > c->dev.lay.halo_ll_cap) {
    b2_set_error("swe_ca: halo buffers too small (%zu > %zu); raise MPI4JAX_B200_HALO_BYTES", need,
                 c->dev.lay.halo_ll_cap);
    return B2_ERR_BAD_ARG;
  }
  return 0;
}

// timeline buffer: [step][kernel 0 = A, 1 = S, 2 = X, 3 = D][start, end]
static unsigned long long* g_stamps = nullptr;
static int g_stamp_steps = 0;
static CAStamp ca_slot(int step, int kernel) {
  CAStamp s;
  s.slot = (g_stamps != nullptr && step >= 0 && step < g_stamp_steps) ? g_stamps + ((size_t)step * 4 + kernel) * 2 : nullptr;
  return s;
}

// Rows per segment of the bulk kernel: about two waves of warps on this GPU, so that the frame chain's
// CTAs find free slots while the bulk runs, and at least 16 rows (a segment evaluates the tendencies of
// three rows beyond its own).
static int ca_bulk_rows_per_segment(const B2SweParams& p, int cb1) {
  static int slot_warps = 0;
  if (slot_warps == 0) {
    int dev = 0, sms = 0, per_sm = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, swe_ca_bulk_step, CA_BULK_WARPS * 32, 0);
    slot_warps = sms * per_sm * CA_BULK_WARPS;
    if (slot_warps <= 0) slot_warps = 132 * 16;
  }
  CABulkArgs g;
  g.p = p;
  ca_bulk_geometry(p, cb1, 1, g);
  const int nseg = (2 * slot_warps) / g.wcols > 1 ? (2 * slot_warps) / g.wcols : 1;
  const int rows = (p.ny - 8 + nseg - 1) / nseg;
  return rows < 16 ? 16 : rows;
}

static int ca_exchange(B2Comm* c, const B2HaloDesc& topo, const B2SweParams& p, const B2SweCA& x, float* f0,
                       float* f1, float* f2, cudaStream_t s, CAStamp ts = CAStamp{nullptr}) {
  B2HaloDesc d = topo;
  d.ny = p.ny; d.nx = p.nx; d.pitch = p.pitch;
  d.nfields = CA_NF;
  d.field[0] = f0; d.kind[0] = 0;
  d.field[1] = f1; d.kind[1] = 1;
  d.field[2] = f2; d.kind[2] = 2;
  CAExt3 ext;
  ext.a[0] = x.hx; ext.a[1] = x.upx; ext.a[2] = x.vpx;
  long long total = 0;
  const int nb[8] = {d.west, d.east, d.south, d.north, d.sw, d.se, d.nw, d.ne};
  for (int k = 0; k < 8; ++k) {
    if (nb[k] < -1 || nb[k] >= c->dev.size) {
      b2_set_error("swe_ca: invalid neighbour rank %d", nb[k]);
      return B2_ERR_BAD_ARG;
    }
    if (nb[k] >= 0) total += ca_msg_count(p.ny, p.nx, k);
  }
  unsigned ctas = ca_blocks(total, CA_THREADS);          // pure latency: about one element per thread
  if (ctas < 8) ctas = 8;
  if (ctas > 120) ctas = 120;                            // all co-resident next to the bulk kernel's CTAs
  b2_k_halo_ca<<<ctas, CA_THREADS, 0, s>>>(c->dev, d, ext, x.epitch, ts);
  return b2_launched(c, "halo_ca");
}

extern "C" {

// Debug timeline: `buf` holds nsteps * 4 * 2 u64 (device memory, start slots preset to ~0, end slots to 0);
// pass null to switch it off again.  Applies to multistep calls (and graphs captured) afterwards.
void b2_swe_ca_timeline(unsigned long long* buf, int nsteps) {
  g_stamps = buf;
  g_stamp_steps = buf ? nsteps : 0;
}

// Fill the ext arrays from a state whose main arrays are complete (after reset / load_state):
// deep exchange of (h, u, v), then fresh := exchanged and the ring mirror.  Collective.
int b2_swe_ca_init(B2Comm* c, const B2SweParams* p0, const B2SweState* st, const B2SweCA* x0,
                   const B2HaloDesc* topo, cudaStream_t s) {
  B2SweParams p = *p0;
  B2SweCA x = *x0;
  if (!swe_ca_supported(p)) return 0;
  x.cb1 = swe_ca_cb1(p);
  if (int rc = ca_check(c, p, x)) return rc;
  if (int rc = ca_streams()) return rc;       // (here, never inside a stream capture: reset / load_state are eager)
  if (int rc = ca_exchange(c, *topo, p, x, st->h0, st->u, st->v, s)) return rc;
  const long long tasks = ca_ext_total(p) + 2LL * (p.nx - 2) + 2LL * (p.ny - 2);
  swe_ca_init_ext<<<ca_blocks(tasks, CA_THREADS), CA_THREADS, 0, s>>>(p, x, st->u, st->v);
  return b2_launched(c, "swe_ca_init_ext");
}

int b2_swe_multistep_ca(B2Comm* c, const B2SweParams* p0, const B2SweState* st, const B2SweCA* x0,
                        const B2HaloDesc* topo, int nsteps, int first_step, cudaStream_t s) {
  // blocks too small for the bulk / frame split, or no friction step: the stand-alone kernels
  if (!swe_ca_supported(*p0) || !(p0->viscosity > 0.f))
    return b2_swe_multistep(c, p0, st, topo, nsteps, first_step, s);
  B2SweParams p = *p0;
  B2SweCA x = *x0;
  x.cb1 = swe_ca_cb1(p);
  if (int rc = ca_check(c, p, x)) return rc;
  if (int rc = ca_streams()) return rc;
  const cudaStream_t s2 = g_side;
  const cudaEvent_t e0 = g_ev[0], eS = g_ev[1], eD = g_ev[2];
  // ping-pong pairs: [cur] = this step's, [nxt] = the next step's; the flux arrays of the stand-alone
  // path are free here: fe / fn hold u', v' of the frame band between kernels A, X and D
  float* H[2] = {st->h0, st->h1};
  float* U[2] = {st->u, st->u1};
  float* V[2] = {st->v, st->v1};
  float* DU[2] = {st->du, st->du1};
  float* DV[2] = {st->dv, st->dv1};
  float* const upf = st->fe;
  float* const vpf = st->fn;
  CABulkArgs sa;
  sa.p = p;
  ca_bulk_geometry(p, x.cb1, ca_bulk_rows_per_segment(p, x.cb1), sa);
  const unsigned bulk_blocks = ca_blocks(ca_bulk_warps(sa), CA_BULK_WARPS);
  const CAFrame fa = ca_frame(p, 5, x.cb1 - 2), fd = ca_frame(p, 3, x.cb1);
  const unsigned tend_blocks = ca_blocks(fa.total, CA_CELLS);
  const unsigned fric_blocks = ca_blocks(fd.total + ca_ext_total(p), CA_CELLS);
  int rc = 0;
#define CA_RT(call) \
  if (rc == 0) rc = b2_cuda_check((call), "swe_multistep_ca: %s failed", #call);
  CA_RT(cudaEventRecord(e0, s));
  CA_RT(cudaStreamWaitEvent(s2, e0, 0));
  int cur = 0;
  for (int it = 0; it < nsteps && rc == 0; ++it) {
    const int nxt = cur ^ 1;
    p.first_step = (first_step && it == 0) ? 1 : 0;
    // ---- frame stream: needs the bulk kernel of the previous step (u'', v'', h next to the frame);
    // enqueued before this step's bulk kernel re-records eS
    if (it > 0) CA_RT(cudaStreamWaitEvent(s2, eS, 0));
    // ---- bulk stream: needs D of the previous step (u'', v'' of the frame, the arrays' halos)
    if (it > 0) CA_RT(cudaStreamWaitEvent(s, eD, 0));
    if (rc) break;
    sa.p = p;
    sa.h = H[cur]; sa.u = U[cur]; sa.v = V[cur]; sa.du = DU[cur]; sa.dv = DV[cur];
    sa.h_o = H[nxt]; sa.u_o = U[nxt]; sa.v_o = V[nxt]; sa.du_o = DU[nxt]; sa.dv_o = DV[nxt];
    sa.dh = st->dh;
    swe_ca_bulk_step<<<bulk_blocks, CA_BULK_WARPS * 32, 0, s>>>(sa, ca_slot(it, 1));
    if ((rc = b2_launched(c, "swe_ca_bulk_step"))) break;
    CA_RT(cudaEventRecord(eS, s));
    CACtx ctx;
    ctx.p = p; ctx.x = x;
    ctx.h = H[cur]; ctx.hn = H[nxt];
    ctx.ua = U[cur]; ctx.va = V[cur];
    ctx.dh = st->dh; ctx.du = DU[cur]; ctx.dv = DV[cur];
    ctx.dub = ctx.dvb = nullptr; ctx.du_o = DU[nxt]; ctx.dv_o = DV[nxt];
    ctx.upf = upf; ctx.vpf = vpf;
    swe_ca_tend_frame<<<tend_blocks, CA_CELLS * CA_TEND_WARPS, 0, s2>>>(ctx, fa, ca_slot(it, 0));
    if ((rc = b2_launched(c, "swe_ca_tend_frame"))) break;
    if ((rc = ca_exchange(c, *topo, p, x, H[nxt], upf, vpf, s2, ca_slot(it, 2)))) break;
    swe_ca_fric_frame<<<fric_blocks, CA_CELLS * 3, 0, s2>>>(ctx, fd, U[nxt], V[nxt], ca_slot(it, 3));
    if ((rc = b2_launched(c, "swe_ca_fric_frame"))) break;
    CA_RT(cudaEventRecord(eD, s2));
    cur = nxt;
  }
  CA_RT(cudaStreamWaitEvent(s, eD, 0));           // join (also required to end a stream capture)
  // odd step count: the state goes back to its home buffers
  const size_t bytes = (size_t)p.ny * p.pitch * sizeof(float);
  if (cur != 0)
    for (int k = 0; k < 5 && rc == 0; ++k) {
      float* const pair[5][2] = {{H[0], H[1]}, {U[0], U[1]}, {V[0], V[1]}, {DU[0], DU[1]}, {DV[0], DV[1]}};
      CA_RT(cudaMemcpyAsync(pair[k][0], pair[k][1], bytes, cudaMemcpyDeviceToDevice, s));
    }
#undef CA_RT
  return rc;
}

}  // extern "C"
