// mpi4jax_b200 -- communication-avoiding shallow-water step: kernels and the two-stream schedule.
// Design, storage and the "views" that keep the reference's discrete system: b2_swe_ca_body.cuh.
//
// One model step (the reference's shallow_water_step, examples/shallow_water.py:270-403):
//
//   stream s  (bulk) :  S  flux + tendency + friction of the bulk, one pass ---------------> next step
//   stream s2 (frame):  A (tendencies, frame band) -> X (deep halo exchange) -> D (friction, frame + ext)
//
// S writes only bulk cells, A / X / D own the frame.  Every kernel reads this step's buffer set and
// writes the next step's.  So the streams meet only at the step boundary: S(t+1) reads what D(t)
// wrote next to the bulk, A(t+1) what S(t) wrote next to the frame.  Seven arrays are read once and
// written once per step (12 array passes instead of the stand-alone path's 32; at 8 GPUs, 2 M cells
// per rank, the step's working set is larger than the 50 MB L2 of an H100, so passes are HBM traffic),
// one exchange instead of three, and the NVLink round of X is hidden behind S.  Pairs of steps advance
// the bulk twice per pass (S2, see b2_swe_multistep_ca).  Under CUDA-graph
// capture (mpi4jax_b200.jit) the event fork / join becomes graph edges.

#include "b2_device.cuh"
#include "b2_halo_ll.cuh"
#include "b2_runtime.h"
#include "b2_swe_ca_body.cuh"
#include "b2_swe_ca_bulk.cuh"

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

// ---- S: the bulk, one pass per step (b2_swe_ca_bulk.cuh) ----------------------------------------
// Also the ring launch of the pair schedule: the same kernel over the four narrower store windows in one
// launch.  blockIdx.y picks the window of `win` (the whole bulk: a table of one); `a`'s own window is not
// used.
#define CA_MAX_WINDOWS 4
struct CAWindows {
  CAWin w[CA_MAX_WINDOWS];
};
__global__ void __launch_bounds__(CA_BULK_WARPS * 32)
swe_ca_bulk_step(const CABulkArgs a, const __grid_constant__ CAWindows win, const CAStamp ts) {
  ca_stamp_begin(ts);
  const CAWin& g = win.w[blockIdx.y];
  const int w = (int)blockIdx.x * CA_BULK_WARPS + (int)(threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (w < ca_bulk_warps(g)) {                          // (whole warps: the lane exchange needs all 32)
    int s, e;
    ca_bulk_rows(g, w / g.wcols, s, e);
    CABulkLane L;
    L.store = ca_bulk_lane(g, w % g.wcols, lane, L.i0);
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

// ---- S2: two steps of the bulk in one pass (b2_swe_ca_bulk.cuh) ---------------------------------
// A PAIR of warps owns a strip of the inner bulk (`b`: rows [8, ny-7) x groups [1, ng-1)) and a segment
// of its rows [s, e).  The step-1 warp walks rows [s-4, e+3) of step t exactly as swe_ca_bulk_step does
// (`a`: state t in, state t+1 out) and puts its rows of state t+1 into the pair's shared-memory row
// ring; the step-2 warp walks rows [s, e) of step t+1 four rows behind it, reading state t+1 from the
// ring and writing state t+2.  One step's dependency cone is 4 rows south (row s-4 feeds the fluxes of
// row s-2), 3 north (row e+2 feeds the u' of row e) and 3 columns (one lane either side, each of which
// needs its own neighbour lanes for the friction), so step 2 needs nothing the frame kernels write.
//
// Lanes: step-1 friction is valid on lanes 1..30 (lanes 0, 31 lack a neighbour's u'); step-2 reads
// the ring columns of its lane and both neighbour lanes, so its tendency is valid on lanes 2..29 and its
// friction on 3..28: a strip stores 26 groups (`halo` 3).
// Lockstep: round k runs step-1 row k and step-2 row k-4, then the pair meets at a named barrier.  Row
// k-4 of step 2 needs rows up to k-1 of step 1 (its tendency reads row k-2, whose u'' is finished by
// step-1 row k-1); in round k step 2 reads ring rows k-5 .. k-2 and step 1 writes rows k-1, k, so eight
// ring slots leave every row in place until it has been read.
// Step 1 also stores state t+1 to the arrays where the ring launch and the frame kernels of step t+1
// read it (ca_pair_band).
#define CA_PAIR_WARPS 4              // warps per CTA: two pairs
#define CA_PAIR_CTAS 3               // CTAs per SM: 6 pairs, 3 x 2 rings of shared memory
#define CA_PAIR_SMEM (2 * CA_RING_FLOATS * (int)sizeof(float))
__global__ void __launch_bounds__(CA_PAIR_WARPS * 32, CA_PAIR_CTAS)
swe_ca_bulk_pair(const CABulkArgs a, const CABulkArgs b, const CAStamp ts) {
  ca_stamp_begin(ts);
  extern __shared__ float4 ca_ring_mem[];
  const int pair = (int)(threadIdx.x >> 6), lane = threadIdx.x & 31;
  const bool second = (threadIdx.x >> 5) & 1;
  float* const ring = reinterpret_cast<float*>(ca_ring_mem) + pair * CA_RING_FLOATS;
  const int w = (int)blockIdx.x * (CA_PAIR_WARPS / 2) + pair;
  if (w < ca_bulk_warps(b)) {                          // (whole pairs: both warps meet at every barrier)
    const int seg = w / b.wcols, wc = w % b.wcols;
    int s, e;
    ca_bulk_rows(b, seg, s, e);
    CABulkLane L;
    const bool own = ca_bulk_lane(b, wc, lane, L.i0);
    L.ic = 4 + 4 * lane;
    const int s1 = s - 4, e1 = e + 3;
    if (!second) {
      const CAPairBand band = ca_pair_band(b, seg, wc, lane, own, L);
      ca_bulk_begin(a, L, s1);
      for (int k = s1 - 2; k <= e + 4; ++k) {
        if (k <= e1) {
          ca_bulk_tend<false, true>(a, L, k, k >= s1 && k < e1, ring, ca_pair_hbm(band, a.p.ny, k));
          const float uw2 = __shfl_up_sync(0xffffffffu, L.upn[2], 1), uw3 = __shfl_up_sync(0xffffffffu, L.upn[3], 1);
          const float ue = __shfl_down_sync(0xffffffffu, L.upn[0], 1), ve = __shfl_down_sync(0xffffffffu, L.vpn[0], 1);
          ca_bulk_fric<true>(a, L, k, uw2, uw3, ue, ve, k == s1, k > s1, ring, ca_pair_hbm(band, a.p.ny, k - 1));
        }
        asm volatile("bar.sync %0, 64;" ::"r"(1 + pair) : "memory");
      }
    } else {
      L.store = own;
      for (int k = s1 - 2; k <= e + 4; ++k) {
        const int t = k - 4;
        if (k == s + 1) {
          ca_bulk_begin<true>(b, L, s, ring);
        } else if (t >= s - 2) {
          ca_bulk_tend<true, false>(b, L, t, t >= s && t < e, ring);
          const float uw2 = __shfl_up_sync(0xffffffffu, L.upn[2], 1), uw3 = __shfl_up_sync(0xffffffffu, L.upn[3], 1);
          const float ue = __shfl_down_sync(0xffffffffu, L.upn[0], 1), ve = __shfl_down_sync(0xffffffffu, L.vpn[0], 1);
          ca_bulk_fric(b, L, t, uw2, uw3, ue, ve, t == s, t > s);
        }
        asm volatile("bar.sync %0, 64;" ::"r"(1 + pair) : "memory");
      }
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

// Rows per segment of a bulk launch: about two waves of warps (pairs) on this GPU, so that the frame
// chain's CTAs find free slots while the bulk runs, and at least 16 rows (a segment evaluates the
// tendencies of three rows beyond its own, the pair kernel's step 1 of seven).
static int ca_rows_per_segment(int slots, int wcols, int rows_total) {
  const int nseg = (2 * slots) / wcols > 1 ? (2 * slots) / wcols : 1;
  const int rows = (rows_total + nseg - 1) / nseg;
  return rows < 16 ? 16 : rows;
}
static int ca_slots(const void* kernel, int threads, int smem, int per_cta) {
  int dev = 0, sms = 0, per_sm = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, smem);
  return sms * per_sm * per_cta > 0 ? sms * per_sm * per_cta : 132 * per_cta;
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

// Schedule.  A step is the bulk kernel S on stream s next to the frame chain A -> X -> D on stream s2.
// Pairs of steps (t, t+1) after the first (Euler) step advance the bulk twice per pass over the arrays:
//
//   s :  S2 (step t on the bulk, t+1 on the inner bulk) ------------> ring (t+1) ----------> next
//   s2:  A X D (t) ----------------------------------------------> A X D (t+1) ------------> next
//                                   (ring waits for D (t), A X D (t+1) for S2)
//
// The ring launch is swe_ca_bulk_step on the four windows around the inner bulk, one window per
// blockIdx.y: rows [4, 8) and [ny-7, ny-4), groups 0 and ng-1 between them; it is the only part of step t+1
// that needs the frame's state t+1.  An odd step left over runs the one-step schedule.  h, u, v, du and dv rotate through three
// buffer sets: a step reads one and writes another; S2 reads set c (state t), stores the band of state
// t+1 into set n, where A X D (t) write the frame's, and state t+2 into set m (a segment's step 1 reads
// rows that a neighbouring segment's step 2 overwrites, so ping-pong is not enough).  dh stays in place
// through a one-step launch and moves to another of its three buffers with a pair, for the same reason.
// Each launch picks its output sets so that the call ends in the home buffers (`target`).
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
  // [k] = buffer set k; the flux arrays of the stand-alone path are free here: fe / fn hold u', v' of
  // the frame band between kernels A, X and D
  float* const H[3] = {st->h0, st->h1, st->h2};
  float* const U[3] = {st->u, st->u1, st->u2};
  float* const V[3] = {st->v, st->v1, st->v2};
  float* const DU[3] = {st->du, st->du1, st->du2};
  float* const DV[3] = {st->dv, st->dv1, st->dv2};
  float* const DH[3] = {st->dh, st->dh1, st->dh2};
  float* const upf = st->fe;
  float* const vpf = st->fn;
  static int slot_warps = 0, slot_pairs = 0;
  if (slot_warps == 0) {
    if (int rc = b2_cuda_check(cudaFuncSetAttribute(swe_ca_bulk_pair, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                    CA_PAIR_SMEM), "swe_multistep_ca: shared memory of the pair kernel"))
      return rc;
    slot_warps = ca_slots((const void*)swe_ca_bulk_step, CA_BULK_WARPS * 32, 0, CA_BULK_WARPS);
    slot_pairs = ca_slots((const void*)swe_ca_bulk_pair, CA_PAIR_WARPS * 32, CA_PAIR_SMEM, CA_PAIR_WARPS / 2);
  }
  const int ng = (x.cb1 >> 2) - 1, ny = p.ny;
  CABulkArgs sa = {};                                   // one step, whole bulk
  ca_bulk_geometry(p, x.cb1, 1, sa);
  ca_bulk_geometry(p, x.cb1, ca_rows_per_segment(slot_warps, sa.wcols, ny - 8), sa);
  // pairs: S2's inner bulk (step 1 walks its segments), the ring's four windows; two rows per segment
  // there: the ring launch is exposed and moves little data, so a warp's walk (its rows + 3 tendency
  // rows, each a round trip to HBM) is kept short
  const bool pairs = ny - 7 > 8 && ng >= 3;
  CAWindows whole = {}, ring = {};
  whole.w[0] = sa;
  const unsigned whole_blocks = ca_blocks(ca_bulk_warps(sa), CA_BULK_WARPS);
  CABulkArgs pa = {}, pb = {}, ra = {};
  unsigned ring_blocks = 0;
  if (pairs) {
    ca_bulk_window(x.cb1, 8, ny - 7, 1, ng - 1, 3, 1, pb);
    ca_bulk_window(x.cb1, 8, ny - 7, 1, ng - 1, 3, ca_rows_per_segment(slot_pairs, pb.wcols, ny - 15), pb);
    pa.ng = pb.ng;
    ca_bulk_window(x.cb1, 4, 8, 0, ng, 1, 2, ring.w[0]);
    ca_bulk_window(x.cb1, ny - 7, ny - 4, 0, ng, 1, 2, ring.w[1]);
    ca_bulk_window(x.cb1, 8, ny - 7, 0, 1, 1, 2, ring.w[2]);
    ca_bulk_window(x.cb1, 8, ny - 7, ng - 1, ng, 1, 2, ring.w[3]);
    for (const CAWin& g : ring.w)
      if (ca_blocks(ca_bulk_warps(g), CA_BULK_WARPS) > ring_blocks) ring_blocks = ca_blocks(ca_bulk_warps(g), CA_BULK_WARPS);
  }
  const CAFrame fa = ca_frame(p, 5, x.cb1 - 2), fd = ca_frame(p, 3, x.cb1);
  const unsigned tend_blocks = ca_blocks(fa.total, CA_CELLS);
  const unsigned fric_blocks = ca_blocks(fd.total + ca_ext_total(p), CA_CELLS);
  int rc = 0;
#define CA_RT(call) \
  if (rc == 0) rc = b2_cuda_check((call), "swe_multistep_ca: %s failed", #call);
  // sets `in` -> `out`; dh from dh_in (null: in place) to dh_out
  auto io = [&](CABulkArgs& a, int in, int out, const float* dh_in, float* dh_out) {
    a.p = p;
    a.h = H[in]; a.u = U[in]; a.v = V[in]; a.du = DU[in]; a.dv = DV[in];
    a.h_o = H[out]; a.u_o = U[out]; a.v_o = V[out]; a.du_o = DU[out]; a.dv_o = DV[out];
    a.dh = dh_out; a.dh_src = dh_in;
  };
  auto frame = [&](int it, int in, int out, const float* dh_in, float* dh_out) -> int {
    CACtx ctx;
    ctx.p = p; ctx.x = x;
    ctx.h = H[in]; ctx.hn = H[out];
    ctx.ua = U[in]; ctx.va = V[in];
    ctx.dh = dh_out; ctx.dh_src = dh_in;
    ctx.du = DU[in]; ctx.dv = DV[in];
    ctx.du_o = DU[out]; ctx.dv_o = DV[out];
    ctx.upf = upf; ctx.vpf = vpf;
    swe_ca_tend_frame<<<tend_blocks, CA_CELLS * CA_TEND_WARPS, 0, s2>>>(ctx, fa, ca_slot(it, 0));
    if (int r = b2_launched(c, "swe_ca_tend_frame")) return r;
    if (int r = ca_exchange(c, *topo, p, x, H[out], upf, vpf, s2, ca_slot(it, 2))) return r;
    swe_ca_fric_frame<<<fric_blocks, CA_CELLS * 3, 0, s2>>>(ctx, fd, U[out], V[out], ca_slot(it, 3));
    if (int r = b2_launched(c, "swe_ca_fric_frame")) return r;
    return b2_cuda_check(cudaEventRecord(eD, s2), "swe_multistep_ca: cudaEventRecord failed");
  };
  // h .. dv move to another set with every one-step or pair launch, dh with every pair launch; the last
  // move goes to the home set and the one before it elsewhere, so only a call of a single move (of dh:
  // a single pair) ends with copies
  const int lead = (first_step && nsteps > 0) ? 1 : 0;
  const int npairs = pairs ? (nsteps - lead) / 2 : 0;
  const int moves = nsteps - npairs;
  auto target = [](int mv, int n, int cur) {
    if (mv == n - 1 && cur != 0) return 0;
    return mv == n - 2 ? (cur == 1 ? 2 : 1) : (cur + 1) % 3;
  };
  CA_RT(cudaEventRecord(e0, s));
  CA_RT(cudaStreamWaitEvent(s2, e0, 0));
  int cur = 0, dc = 0;
  for (int it = 0, mv = 0, pv = 0; it < nsteps && rc == 0; ++mv) {
    p.first_step = (first_step && it == 0) ? 1 : 0;
    const bool pair = pairs && !p.first_step && nsteps - it >= 2;
    // single step: cur -> nxt; pair: cur -> nxt (band of step t+1, frame) -> third
    const int third = target(mv, moves, cur), nxt = pair ? 3 - cur - third : third;
    // ---- frame stream: needs the bulk launches of the previous step (state next to the frame);
    // enqueued before this step's bulk kernel re-records eS
    if (it > 0) CA_RT(cudaStreamWaitEvent(s2, eS, 0));
    // ---- bulk stream: needs D of the previous step (u'', v'' of the frame, the arrays' halos)
    if (it > 0) CA_RT(cudaStreamWaitEvent(s, eD, 0));
    if (rc) break;
    if (!pair) {
      io(sa, cur, nxt, nullptr, DH[dc]);
      swe_ca_bulk_step<<<whole_blocks, CA_BULK_WARPS * 32, 0, s>>>(sa, whole, ca_slot(it, 1));
      if ((rc = b2_launched(c, "swe_ca_bulk_step"))) break;
      CA_RT(cudaEventRecord(eS, s));
      if (rc || (rc = frame(it, cur, nxt, nullptr, DH[dc]))) break;
      cur = nxt;
      ++it;
      continue;
    }
    const int dm = target(pv++, npairs, dc), dn = 3 - dc - dm;
    io(pa, cur, nxt, DH[dc], DH[dn]);
    io(pb, nxt, third, nullptr, DH[dm]);
    swe_ca_bulk_pair<<<ca_blocks(ca_bulk_warps(pb), CA_PAIR_WARPS / 2), CA_PAIR_WARPS * 32, CA_PAIR_SMEM, s>>>(
        pa, pb, ca_slot(it, 1));
    if ((rc = b2_launched(c, "swe_ca_bulk_pair"))) break;
    CA_RT(cudaEventRecord(eS, s));
    if (rc || (rc = frame(it, cur, nxt, DH[dc], DH[dn]))) break;
    // ring (t+1): needs D (t); A X D (t+1): needs S2 (eS, recorded before the ring re-records it)
    CA_RT(cudaStreamWaitEvent(s, eD, 0));
    CA_RT(cudaStreamWaitEvent(s2, eS, 0));
    if (rc) break;
    io(ra, nxt, third, DH[dn], DH[dm]);
    swe_ca_bulk_step<<<dim3(ring_blocks, CA_MAX_WINDOWS), CA_BULK_WARPS * 32, 0, s>>>(ra, ring, ca_slot(it + 1, 1));
    if ((rc = b2_launched(c, "swe_ca_bulk_step"))) break;
    if ((rc = frame(it + 1, nxt, third, DH[dn], DH[dm]))) break;
    CA_RT(cudaEventRecord(eS, s));
    cur = third;
    dc = dm;
    it += 2;
  }
  CA_RT(cudaStreamWaitEvent(s, eD, 0));           // join (also required to end a stream capture)
  // the state goes back to its home buffers
  const size_t bytes = (size_t)p.ny * p.pitch * sizeof(float);
  if (cur != 0) {
    float* const* set[5] = {H, U, V, DU, DV};
    for (int k = 0; k < 5 && rc == 0; ++k)
      CA_RT(cudaMemcpyAsync(set[k][0], set[k][cur], bytes, cudaMemcpyDeviceToDevice, s));
  }
  if (dc != 0) CA_RT(cudaMemcpyAsync(DH[0], DH[dc], bytes, cudaMemcpyDeviceToDevice, s));
#undef CA_RT
  return rc;
}

}  // extern "C"
