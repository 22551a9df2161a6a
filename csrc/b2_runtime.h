// mpi4jax_b200 -- host-side runtime objects and the C ABI.
//
// B2Seg   : one symmetric-memory segment (same size on every rank), backed by
//           the CUDA VMM API (cuMemCreate + POSIX fd export) or, as a fallback,
//           by cudaMalloc + cudaIpc handles.  Peers' segments are mapped into
//           this process' address space; file descriptors / IPC handles are
//           exchanged by the Python control plane (unix sockets / gloo).
// B2Mc    : an NVLS multicast object bound to a segment on every rank
//           (multimem.ld_reduce / multimem.st address space).
// B2Comm  : a communicator: rank/size, control segment (flags, p2p rings, LL
//           buffers, halo buffers), growable staging segment, local counters.
//
// This is the H100-native counterpart of the reference's native bridge layer
// (mpi4jax/_src/xla_bridge/mpi_xla_bridge_cuda.cpp + mpi_ops_common.h); the
// reference hands device pointers to a CUDA-aware MPI, we own the transport.
#pragma once

#include <cuda.h>
#include <cuda_runtime.h>

#include "b2_common.h"

struct B2Seg {
  int mode;                 // 0 = VMM, 1 = cudaIpc
  int device;
  int nranks;
  int rank;
  size_t bytes;             // rounded-up size
  CUmemGenericAllocationHandle handle;      // local physical allocation (VMM)
  CUmemGenericAllocationHandle peer_handle[B2_MAX_RANKS];
  void* ptr[B2_MAX_RANKS];  // mapped address of every rank's segment (ptr[rank] = local)
  int export_fd;
};

struct B2Mc {
  CUmemGenericAllocationHandle handle;
  size_t bytes;
  int device;
  void* ptr;                // mapped multicast VA
  int export_fd;
  int bound;
};

struct B2Comm {
  B2DevComm dev;
  int device;
  int sm_count;
  B2Seg* ctl;
  B2Seg* stage;
  B2Mc* stage_mc;
  // algorithm thresholds (bytes); tunable from Python (measured table)
  size_t ll_max;
  size_t oneshot_max;
  size_t nvls_min;
  size_t bcast_mc_min;          // bcast: root multimem.st from this size on
  int nvls_pipeline;            // software-pipelined NVLS allreduce (default on)
  int gemm_raster;              // tile order of the persistent GEMM: -1 = compile-time default, 0 = row-major, G = bands
  int p2p_anysource_scan;       // ANY_SOURCE + tag receives scan every source's window (default off, b2_p2p.cu)
  unsigned long long* trace;    // device buffer for the phase timeline of CTA 0 (scripts/allreduce_phases.py)
  int trace_cap;
  int max_blocks;
  B2ErrorRecord* err_host;      // host pointer of the mapped error record
  int launches;                 // kernels launched through this communicator
};

#ifdef __cplusplus
extern "C" {
#endif

// --- library / logging -------------------------------------------------------
const char* b2_version(void);
const char* b2_last_error(void);
void b2_set_logging(int enable);
int b2_get_logging(void);
typedef void (*b2_print_fn)(const char*);
void b2_set_print_callback(b2_print_fn fn);
int b2_launch_count(void);

// --- device / driver ---------------------------------------------------------
int b2_init(int device);
int b2_multicast_supported(int device);
int b2_vmm_supported(int device);
size_t b2_granularity(int device, int for_multicast);

// --- segments ----------------------------------------------------------------
B2Seg* b2_seg_create(int device, int rank, int nranks, size_t bytes, int mode);
int b2_seg_export_fd(B2Seg* s);                       // VMM: fd to send to peers
int b2_seg_import_fd(B2Seg* s, int peer, int fd);     // VMM: map a peer's allocation
int b2_seg_ipc_handle(B2Seg* s, void* out64);         // IPC: 64-byte handle
int b2_seg_import_ipc(B2Seg* s, int peer, const void* handle64);
void* b2_seg_ptr(B2Seg* s, int peer);
size_t b2_seg_bytes(B2Seg* s);
int b2_seg_destroy(B2Seg* s);

// --- multicast ---------------------------------------------------------------
B2Mc* b2_mc_create(int device, int nranks, size_t bytes);      // rank 0
int b2_mc_export_fd(B2Mc* m);
B2Mc* b2_mc_import(int device, int fd, size_t bytes);           // other ranks
int b2_mc_add_device(B2Mc* m);
int b2_mc_bind(B2Mc* m, B2Seg* s);
void* b2_mc_ptr(B2Mc* m);
int b2_mc_destroy(B2Mc* m);

// --- communicator ------------------------------------------------------------
size_t b2_layout_bytes(int nranks, size_t slot_bytes, size_t ll_cap, size_t halo_cap);
B2Comm* b2_comm_create(int device, int rank, int nranks, B2Seg* ctl, size_t slot_bytes,
                       size_t ll_cap, size_t halo_cap, double timeout_s);
int b2_comm_set_stage(B2Comm* c, B2Seg* stage, B2Mc* mc);
size_t b2_comm_stage_half(B2Comm* c);
// keys: "ll_max", "oneshot_max", "nvls_min" (bytes), "max_blocks", "bcast_mc_min", "nvls_pipeline",
// "gemm_raster", "p2p_anysource_scan", "trace_ptr", "trace_cap"; get_option also reads "sm_count" and
// "p2p_slot_bytes" (the p2p ring's slot size, as rounded up at creation)
int b2_comm_set_option(B2Comm* c, const char* key, long long value);
long long b2_comm_get_option(B2Comm* c, const char* key);
int b2_comm_check_error(B2Comm* c, char* buf, int buflen);     // 0 = ok
int b2_comm_destroy(B2Comm* c);
size_t b2_stage_need(int opcode, int nranks, size_t blk_bytes); // staging half needed by an op

// Layout of a non-contiguous input (elements, innermost dimension last); nd == 0: contiguous.
// Dimension 0 of an alltoall / scatter input (the per-peer blocks) is described separately.
struct B2Strided {
  int nd;
  int esize;                 // element size in bytes: 1, 2, 4, 8 or 16
  long long shape[4];
  long long stride[4];       // in elements
  long long blk_stride;      // elements between consecutive blocks
};

// --- collectives (all enqueue on `stream`, never synchronise the host) --------
int b2_barrier(B2Comm* c, cudaStream_t stream);
int b2_allreduce(B2Comm* c, const void* in, void* out, size_t count, int dtype, int op, int algo,
                 cudaStream_t stream);
int b2_allreduce_sym(B2Comm* c, void* mc, size_t count, int dtype, cudaStream_t stream);
int b2_reduce(B2Comm* c, const void* in, void* out, size_t count, int dtype, int op, int root,
              cudaStream_t stream);
int b2_scan(B2Comm* c, const void* in, void* out, size_t count, int dtype, int op,
            cudaStream_t stream);
// `in`: nranks blocks of `count` elements each; `out`: this rank's reduced block (`count` elements)
int b2_reduce_scatter(B2Comm* c, const void* in, void* out, size_t count, int dtype, int op,
                      cudaStream_t stream);
// `lay` (may be null = contiguous) describes a strided input; the pack is fused into the staging copy
int b2_allgather(B2Comm* c, const void* in, void* out, size_t blk_bytes, const B2Strided* lay,
                 cudaStream_t stream);
int b2_alltoall(B2Comm* c, const void* in, void* out, size_t blk_bytes, const B2Strided* lay,
                cudaStream_t stream);
int b2_bcast(B2Comm* c, const void* in, void* out, size_t nbytes, int root, const B2Strided* lay,
             cudaStream_t stream);
int b2_gather(B2Comm* c, const void* in, void* out, size_t blk_bytes, int root, const B2Strided* lay,
              cudaStream_t stream);
int b2_scatter(B2Comm* c, const void* in, void* out, size_t blk_bytes, int root, const B2Strided* lay,
               cudaStream_t stream);
// Variable-count all-to-all whose counts stay on the device.  `in`: in_rows rows of row_bytes bytes
// (contiguous); `send_counts`, `recv_counts`: [nranks] int64 device arrays.  Forward (place_counts
// null): rows sent to each rank are clamped in rank order to the rows that exist, received segments
// are packed in source order and clipped to out_rows.  Reverse (place_counts = the send counts of a
// forward call, out_rows = its in_rows): the segment from rank q lands at the sum of place_counts[p]
// over p < q.  Output rows that receive nothing are zeroed; recv_counts holds the rows written.
int b2_alltoallv(B2Comm* c, const void* in, void* out, size_t row_bytes, size_t in_rows, size_t out_rows,
                 const long long* send_counts, long long* recv_counts, const long long* place_counts,
                 cudaStream_t stream);
// Variable-count allgather whose counts stay on the device.  `in`: in_rows rows of row_bytes bytes
// (contiguous, in_rows the same on every rank); `count`: one int64 on the device, clamped to
// [0, in_rows]; `recv_counts`: [nranks] int64.  Forward (place_counts null): the segments of all ranks
// are packed in rank order and clipped to out_rows.  Reverse (place_counts: [nranks] int64, the send
// counts of a reduce_scatterv): the segment from rank q lands at the sum of place_counts[p] over p < q,
// at most place_counts[q] rows of it, all clamped in rank order to out_rows.  Output rows that receive
// nothing are zeroed; recv_counts holds the rows written from each rank.
int b2_allgatherv(B2Comm* c, const void* in, void* out, size_t row_bytes, size_t in_rows, size_t out_rows,
                  const long long* count, long long* recv_counts, const long long* place_counts,
                  cudaStream_t stream);
// Variable-count gather whose counts stay on the device: b2_allgatherv with output rows on `root` only
// (`out` and `place_counts` are read there only; the other ranks' recv_counts become zeros).  max_rows
// bounds the rows any rank stages and must be the same on every rank: it sizes the staging and the
// chunks; in_rows may differ.
int b2_gatherv(B2Comm* c, const void* in, void* out, size_t row_bytes, size_t in_rows, size_t out_rows,
               size_t max_rows, const long long* count, long long* recv_counts, const long long* place_counts,
               int root, cudaStream_t stream);
// Variable-count scatter whose counts stay on the device.  On `root`, `in` holds in_rows rows and
// `send_counts` [nranks] int64, clamped in rank order to min(in_rows, max_rows); neither is read on the
// other ranks.  Rank q receives its segment, packed from row 0 and clipped to its out_rows, zeros after
// it; `recv_count`: one int64, the rows written.  max_rows: as for b2_gatherv.
int b2_scatterv(B2Comm* c, const void* in, void* out, size_t row_bytes, size_t in_rows, size_t out_rows,
                size_t max_rows, const long long* send_counts, long long* recv_count, int root,
                cudaStream_t stream);
// Variable-count reduce-scatter whose counts stay on the device.  `in`: in_rows rows of row_bytes bytes
// (contiguous; in_rows may differ between ranks); `send_counts`: [nranks] int64, clamped in rank order
// to in_rows; out_rows (N) must be the same on every rank.  Row i of `out` is `op` folded in rank order
// over the ranks q whose segment for this rank has more than i rows (at most N), rows past the longest
// segment are zeroed; `recv_counts`: [nranks] int64, min(send_counts_q[rank], N).
int b2_reduce_scatterv(B2Comm* c, const void* in, void* out, size_t row_bytes, size_t in_rows, size_t out_rows,
                       const long long* send_counts, long long* recv_counts, int dtype, int op,
                       cudaStream_t stream);
// MAXLOC / MINLOC (op) of (value, index) pairs for the reduction collective `opcode` (B2_OPC_ALLREDUCE,
// _REDUCE, _SCAN or _REDUCE_SCATTER).  `in_val`: count pairs' values of dtype val_dtype (f32, f64, f16, bf16,
// i16, i32 or i64), `in_idx`: their indices, idx_bytes 4 (int32) or 8 (int64); reduce-scatter: nranks blocks of
// count pairs each.  `out_val` / `out_idx` (count pairs, the same dtypes) receive the winning pair, which is
// always one of the inputs; reduce writes them on `root` only.  Pairs fold in rank order (see b2_reduce_loc.cu).
int b2_reduce_loc(B2Comm* c, const void* in_val, const void* in_idx, void* out_val, void* out_idx, size_t count,
                  int val_dtype, int idx_bytes, int op, int opcode, int root, cudaStream_t stream);
// Top-k expert dispatch (b2_moe.cu).  `order` [n_pairs] int64: the pair (t * k + j) at each position of this
// rank's pairs sorted by expert; `send_counts` [num_experts] int64: the sorted pairs of each expert, clamped in
// expert order to n_pairs (the pairs past their sum go nowhere).  Sorted pair s carries row order[s] / k of `in`
// (k = 1: row order[s], the pair mode).  Expert e lives on rank e / L (L = num_experts / nranks); rank r's
// out_rows rows hold, for l = 0..L-1 and then q = 0..nranks-1, the pairs rank q sends to expert r L + l, cut
// at out_rows, then zeros.  recv_counts [L x nranks], pos and dest [n_pairs] (this rank's pairs: the row and
// rank they landed in, -1 if dropped) are written unless null.  n_pairs, row_bytes, num_experts and out_rows
// must be the same on every rank.
int b2_moe_dispatch(B2Comm* c, const void* in, void* out, size_t row_bytes, size_t n_pairs, int k,
                    const long long* order, const long long* send_counts, int num_experts, size_t out_rows,
                    long long* recv_counts, long long* pos, long long* dest, cudaStream_t stream);
// Top-k expert combine (b2_moe.cu): token t of `out` (tokens rows of row_bytes) is the fold over its k pairs,
// slot order, of weights[t k + j] * (row pos[t k + j] of rank dest[t k + j]'s `in`), pairs with dest -1
// skipped: fp32 (f64 for f64) products and sums, rounded once, +0 for a token with none.  `weights` null:
// unit weights.  pairs != 0: out holds the tokens x k pair rows unfolded and unweighted (zeros where dropped).
// Each rank stages the first sum(recv_counts[0..n_counts)) of its in_rows rows; in_rows, row_bytes, tokens, k
// and dtype (f32, f64, f16 or bf16) must be the same on every rank.
int b2_moe_combine(B2Comm* c, const void* in, void* out, size_t row_bytes, size_t in_rows, size_t tokens, int k,
                   const long long* pos, const long long* dest, const float* weights, const long long* recv_counts,
                   int n_counts, int dtype, int pairs, cudaStream_t stream);

// --- point to point ----------------------------------------------------------
// source/tag may be -1 (ANY).  `status` is a host-mapped B2StatusRecord or null.
B2StatusRecord* b2_status_alloc(void);
void b2_status_free(B2StatusRecord* s);
int b2_send(B2Comm* c, const void* buf, size_t nbytes, int dest, int tag, cudaStream_t stream);
int b2_recv(B2Comm* c, void* buf, size_t nbytes, int source, int tag, B2StatusRecord* status,
            cudaStream_t stream);
int b2_sendrecv(B2Comm* c, const void* sendbuf, size_t send_bytes, int dest, int sendtag,
                void* recvbuf, size_t recv_bytes, int source, int recvtag, B2StatusRecord* status,
                cudaStream_t stream);

// --- tensor-parallel linear: wgmma GEMM + in-switch allreduce in one kernel (b2_gemm.cu) ---
int b2_gemm_allreduce(B2Comm* c, const void* A, const void* B, void* out, int M, int N, int K,
                      cudaStream_t stream);
// ... and its sequence-parallel twin: GEMM + reduce-scatter over the rows (M % size == 0), this rank's
// (M / size) x N shard of the sum; pull-and-fold epilogue, no multicast
int b2_gemm_reduce_scatter(B2Comm* c, const void* A, const void* B, void* out, int M, int N, int K,
                           cudaStream_t stream);
// ... and the column-parallel layer before it (b2_gemm_ag.cu): out (size m x N) = the (m x K) x_local of
// every rank, gathered in rank order, @ w^T (w: N x K); m and K the same on every rank, N may differ.  The
// shards are pushed into the staging while the GEMM runs; no multicast
int b2_gemm_allgather(B2Comm* c, const void* x_local, const void* w, void* out, int m, int N, int K,
                      cudaStream_t stream);
// ... and their scaled float8 twins (b2_gemm_f8.cu): e4m3 operands, K a multiple of 128, bf16 output; each
// rank's partial (i, j) is rn_bf16(S[i, j] * (sx[i * sx_inc] * sw[j * sw_inc])), fp32 scales read on the device
// (inc 0: one per tensor, 1: one per row of A / x_local, one per column of the output)
int b2_gemm_allreduce_f8(B2Comm* c, const void* A, const void* B, void* out, int M, int N, int K, const float* sx,
                         int sx_inc, const float* sw, int sw_inc, cudaStream_t stream);
int b2_gemm_reduce_scatter_f8(B2Comm* c, const void* A, const void* B, void* out, int M, int N, int K,
                              const float* sx, int sx_inc, const float* sw, int sw_inc, cudaStream_t stream);
int b2_gemm_allgather_f8(B2Comm* c, const void* x_local, const void* w, void* out, int m, int N, int K,
                         const float* sx, int sx_inc, const float* sw, int sw_inc, cudaStream_t stream);

// --- fused halo exchange + shallow-water stencils (see b2_halo.cu, b2_swe.cu) --
struct B2HaloDesc {
  int nfields;
  float* field[B2_HALO_MAX_FIELDS];   // (ny, nx) row-major fp32 arrays with a 1-cell halo
  int kind[B2_HALO_MAX_FIELDS];       // 0 = "h", 1 = "u", 2 = "v"  (wall conditions)
  int ny, nx;
  int pitch;                          // row pitch in floats (>= nx)
  int west, east, south, north;       // neighbour ranks, -1 = wall
  int sw, se, nw, ne;                 // diagonal neighbours (-1 where south/north is a wall)
  int periodic_x;
  int at_east_wall;                   // last column of processes (u wall, non-periodic only)
  int at_north_wall;                  // last row of processes (v wall)
};
int b2_halo_exchange(B2Comm* c, const B2HaloDesc* d, cudaStream_t stream);

struct B2SweParams {
  int ny, nx, pitch;
  float dx, dy, dt, gravity, viscosity;
  float rdx, rdy;             // 1/dx, 1/dy: x * (1/dx) instead of x / dx (<= 1 ulp apart, ~8x cheaper)
  float ab_a, ab_b;           // Adams-Bashforth weights
  int first_step;
  int south_wall, north_wall; // this rank touches the y walls (hc edge padding)
  const float* coriolis;      // [ny]
  // folded constants (fp32 products formed on the host, models/shallow_water.py)
  float c_gx, c_gy;           // -gravity / dx, -gravity / dy
  float c_nux, c_nuy;         // viscosity / dx, viscosity / dy
  float c_fx, c_fy;           // dt * viscosity / dx^2, dt * viscosity / dy^2
};

// Device pointers of a model's fields (mirrored by ctypes in _src/native/__init__.py; the layout
// is part of the ABI checked at import).  h0/h1, u/u1, v/v1, du/du1 and dv/dv1 are ping-pong pairs;
// the first of each holds the state between calls.  The communication-avoiding step rotates three
// sets (h0, u, v, dh, du, dv), (h1, u1, ..., dh1, ...) and (h2, u2, ..., dh2, ...).
struct B2SweState {
  float *h0, *h1, *u, *v, *dh, *du, *dv, *fe, *fn, *q, *ke, *fe2, *fn2;
  float* u1;
  float* v1;
  float* du1;
  float* dv1;
  float *h2, *u2, *v2, *dh1, *dh2, *du2, *dv2;
};

// "ext" arrays of the communication-avoiding step (b2_swe_ca_body.cuh): [(ny + 4) x epitch] floats,
// cell (j, i) at (j + 2) * epitch + (i + 2); only cells beyond the interior (and the ring mirror) are used
struct B2SweCA {
  float *hx, *upx, *vpx, *uppx, *vppx;
  int epitch;
  int cb1;            // first column of the east frame: a multiple of 4, <= nx - 4 (filled in natively)
};

int b2_swe_multistep(B2Comm* c, const B2SweParams* p0, const B2SweState* st, const B2HaloDesc* topo,
                     int nsteps, int first_step, cudaStream_t s);
// struct sizes for the import-time ABI check (mpi4jax_b200/_src/native/__init__.py)
int b2_abi_info(int* out, int n);

// --- internal: shared by the translation units, not called from Python --------
void b2_set_error(const char* fmt, ...) __attribute__((format(printf, 1, 2)));
// 0 if `e` is cudaSuccess; otherwise sets the last error to "<fmt...>: <CUDA error string>" and returns 1000 + e
int b2_cuda_check(cudaError_t e, const char* fmt, ...) __attribute__((format(printf, 2, 3)));
// after a kernel launch: counts it (b2_launch_count), then b2_cuda_check(cudaGetLastError(), "<name>: kernel launch failed")
int b2_launched(B2Comm* c, const char* name);
// the staging check and launch geometry of a staged kernel (b2_collectives.cu)
int b2_plan_staged(B2Comm* c, int opcode, size_t blk_bytes, const void* kernel, const char* name, size_t* chunk,
                   int* grid);
// argument checks shared by the halo exchanges (b2_halo.cu): 0, or B2_ERR_BAD_ARG with the error "<what>: ..."
int b2_halo_check_ranks(B2Comm* c, const B2HaloDesc* d, const char* what);
int b2_halo_check_cap(B2Comm* c, int nfields, int depth, int ny, int nx, const char* what);
// per-call debug log (b2_logging.cpp): `fmt` (may be null) formats the details only when logging is on
struct B2DebugScope;
B2DebugScope* b2_debug_begin(B2Comm* c, const char* opname, cudaStream_t stream, const char* fmt, ...)
    __attribute__((format(printf, 4, 5)));
void b2_debug_end(B2DebugScope* s, int code);
int b2_tensor_map_2d_bf16(CUtensorMap* out, const void* ptr, unsigned long long rows, unsigned long long cols,
                          unsigned box_rows, unsigned box_cols);
int b2_tensor_map_2d_u8(CUtensorMap* out, const void* ptr, unsigned long long rows, unsigned long long cols,
                        unsigned box_rows, unsigned box_cols);

#ifdef __cplusplus
}
#endif
