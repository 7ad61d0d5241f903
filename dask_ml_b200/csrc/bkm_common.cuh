// bkm_common.cuh — shared definitions for the KMeans hot-path kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stddef.h>
#include <atomic>
#include "../../include/bkm_b200.h"

#define BKM_CUDA_TRY(expr)                                  \
  do {                                                      \
    cudaError_t _e = (expr);                                \
    if (_e != cudaSuccess) { (void)cudaGetLastError(); return (int)_e; } \
  } while (0)

namespace bkm {

// Counts kernel launches enqueued by the library (bench.py reports it as gpu_launches).
extern std::atomic<long long> g_launches;
inline void note_launch(int n = 1) { g_launches.fetch_add(n, std::memory_order_relaxed); }

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

static const int kDefaultSMs = 132;     // H100 SXM: sizing when no device is visible

// SM count of the current device, cached per device (defined in bkm_api.cu)
int sm_count(int* out);
// ... or kDefaultSMs when there is no device: for the *_workspace_bytes sizing, which must answer without one
static inline int sm_count_or_default() {
  int sms = 0;
  if (sm_count(&sms) != 0 || sms <= 0) sms = kDefaultSMs;
  return sms;
}

// the dense input dtypes of the row-chunk passes, and their element sizes
static inline bool dtype_ok(int t) { return t == BKM_F32 || t == BKM_F64 || t == BKM_BF16; }
static inline size_t elem_size(int t) { return t == BKM_F64 ? 8 : (t == BKM_F32 ? 4 : 2); }

// Last-CTA election of a deterministic fold.  Every CTA calls it after writing its partial; the one that arrives last
// of `arrivals` gets true (block-uniform) and, after the fences, sees every other CTA's partial.  The caller folds the
// partials in its own fixed order and resets the ticket.  The second barrier carries the result to every thread, so the
// election needs no shared memory.
__device__ __forceinline__ bool last_block(unsigned* ticket, unsigned arrivals) {
  __threadfence();
  __syncthreads();
  const bool mine = threadIdx.x == 0 && atomicAdd(ticket, 1u) == arrivals - 1;
  const bool last = __syncthreads_or(mine);
  if (last) __threadfence();
  return last;
}

// last_block for one warp (warp-uniform): every lane fences its own writes before lane 0 takes the ticket.
__device__ __forceinline__ bool last_warp(unsigned* ticket, unsigned arrivals) {
  __threadfence();
  __syncwarp();
  int last = 0;
  if ((threadIdx.x & 31) == 0) last = atomicAdd(ticket, 1u) == arrivals - 1;
  last = __shfl_sync(0xffffffffu, last, 0);
  if (last) __threadfence();
  return last;
}

// Workspace of a one-ticket last_block fold: `grid` CTA partials of `per_cta` doubles, then 256 bytes for the ticket
static inline size_t partials_bytes(long long grid, size_t per_cta) {
  return align_up((size_t)grid * per_cta * 8, 256) + 256;
}
// ... carved from `ws` of `bytes` = partials_bytes(...) bytes, the ticket zeroed on the stream
static inline cudaError_t carve_partials(void* ws, size_t bytes, double** part, unsigned** ticket, cudaStream_t s) {
  *part = reinterpret_cast<double*>(ws);
  *ticket = reinterpret_cast<unsigned*>(reinterpret_cast<unsigned char*>(ws) + bytes - 256);
  return cudaMemsetAsync(*ticket, 0, 4, s);
}

// Column record of the signed arg-max epilogues (bkm_project_chunk, bkm_csr_panel_chunk): the largest |t|, its lowest
// global row, the signed value, and a lock word.  Ordered by (|t| descending, row ascending): every update order ends
// on the same record.
struct ColMax {
  double absmax;
  long long row;
  double value;
  unsigned long long lock;
};

__device__ __forceinline__ bool colmax_beats(double a, long long ra, double b, long long rb) {
  return a > b || (a == b && ra < rb);
}

// one CTA's best candidate of a column folded into its global record under the record's lock
__device__ __forceinline__ void colmax_fold(ColMax* rec, double a, long long row, double v) {
  while (atomicCAS(&rec->lock, 0ull, 1ull) != 0ull) { }
  __threadfence();
  volatile ColMax* vr = rec;
  if (colmax_beats(a, row, vr->absmax, vr->row)) { vr->absmax = a; vr->row = row; vr->value = v; }
  __threadfence();
  atomicExch(&rec->lock, 0ull);
}

// ---------------------------------------------------------------------------------------
// Geometry of the large-shape tensor path (bkm_tc2.cu): the k centres are cut into S slices of NS <= 256 (one slice
// per CTA, resident in shared memory), the features into KB blocks of 64 16-bit values (one 128-byte swizzle atom).
// The label-indexed row pass (bkm_rowpass.cu) cuts the clusters into DS slices so that (k/DS)*d fp32 sums fit one CTA.
// ---------------------------------------------------------------------------------------
struct Tc2Geom { int S, NS, KB, kp2, dk2, DS; };
static inline Tc2Geom tc2_geom(int k, int d) {
  Tc2Geom g;
  g.S = (k + 255) / 256;
  const int per = (k + g.S - 1) / g.S;
  g.NS = (per + 15) / 16 * 16;
  g.kp2 = g.S * g.NS;
  g.KB = (d + 63) / 64;
  g.dk2 = g.KB * 64;
  // label-indexed M-step (bkm_rowpass.cu): DS cluster slices so that the (k / DS) x d_padded fp32 sums of one slice
  // (+ counts + two staged label tiles) fit one CTA
  const int dpad = d <= 32 ? 32 : (d <= 64 ? 64 : 128);
  g.DS = 1;
  while ((size_t)((k + g.DS - 1) / g.DS) * dpad * 4 + (size_t)((k + g.DS - 1) / g.DS) * 4 + 40 * 1024 > 210 * 1024) g.DS <<= 1;      // a power of two
  return g;
}
// bf16 input of any k / d <= 128 (BASELINE config C5: 128 features, k = 1024)
static inline bool tc2_shape(int d, int k, int dtype) {
  return dtype == BKM_BF16 && d >= 1 && d <= 128 && k >= 1 && k <= 4096;      // <= 16 cluster slices in the M-step row pass
}

// fp32 input with d <= 64 and k <= 256: the tensor-core kernel of bkm_tc.cu (implemented there)
bool tc_supported(int d, int k, int dtype);

// ---------------------------------------------------------------------------------------
// Centre pack: one device buffer holding every layout of the (k,d) centres the kernels use.
// Built from the float64 centres (reference keeps centres in f64: dask_ml/cluster/k_means.py:551-552) by
// bkm_pack_centers / bkm_finalize_step (bkm_aux.cu, which lists the layouts).  A shape's pack holds the layouts of the
// kernels that can read it: every shape has the four plain ones, tc_supported shapes the family-1 operands and
// tc2_shape shapes the family-3 operands.
// ---------------------------------------------------------------------------------------
struct PackLayout {
  int k, d, dtype;
  int d4;      // d rounded up to a multiple of 4 (SIMT row pitch, zero padded)
  int kp;      // k rounded up to a multiple of 16 (MMA N granularity)
  bool tc;     // family-1 operands present (tc_supported)
  bool tc2;    // family-3 operands present (tc2_shape)
  int kp2, dk2;  // family-3 operand tiles: rows (all centre slices) x 16-bit columns (Tc2Geom)
  size_t esz;  // sizeof(T)
  size_t off_cT, off_cnT, off_c64, off_cn64, total;
  // family 1: fp16 (hi, lo) operand tiles [kp][64], s^2 ||c||^2 [kp] fp32, float64 centres transposed [d][kp]
  size_t off_bhi, off_blo, off_cns, off_c64T;
  // family 3: bf16 (hi, lo) operand tiles [kp2][dk2], ||c||^2 [kp2] fp32, float64 centres transposed [d][kp2]
  size_t off_b2hi, off_b2lo, off_cn2, off_c64T2;
};

static inline PackLayout pack_layout(int k, int d, int dtype) {
  PackLayout L;
  L.k = k; L.d = d; L.dtype = dtype;
  L.d4 = (d + 3) / 4 * 4;
  L.kp = (k + 15) / 16 * 16;
  L.tc = tc_supported(d, k, dtype);
  L.tc2 = tc2_shape(d, k, dtype);
  L.esz = dtype == BKM_F64 ? 8 : 4;                // bf16 input: the fp32 layouts (the kernels widen the rows)
  size_t o = 256;  // header
  L.off_cT = o;   o = align_up(o + (size_t)k * L.d4 * L.esz, 256);
  L.off_cnT = o;  o = align_up(o + (size_t)k * L.esz, 256);
  L.off_c64 = o;  o = align_up(o + (size_t)k * d * 8, 256);
  L.off_cn64 = o; o = align_up(o + (size_t)k * 8, 256);
  L.off_bhi = L.off_blo = L.off_cns = L.off_c64T = o;
  if (L.tc) {
    L.off_bhi = o;  o = align_up(o + (size_t)L.kp * 64 * 2, 256);    // 64 halves = one 128-byte swizzle atom per row
    L.off_blo = o;  o = align_up(o + (size_t)L.kp * 64 * 2, 256);
    L.off_cns = o;  o = align_up(o + (size_t)L.kp * 4, 256);
    L.off_c64T = o; o = align_up(o + (size_t)d * L.kp * 8, 256);     // float64 re-check, coalesced over centres
  }
  L.kp2 = L.dk2 = 0;
  L.off_b2hi = L.off_b2lo = L.off_cn2 = L.off_c64T2 = o;
  if (L.tc2) {
    const Tc2Geom g = tc2_geom(k, d);
    L.kp2 = g.kp2; L.dk2 = g.dk2;
    L.off_b2hi = o;  o = align_up(o + (size_t)g.kp2 * g.dk2 * 2, 1024);
    L.off_b2lo = o;  o = align_up(o + (size_t)g.kp2 * g.dk2 * 2, 1024);
    L.off_cn2 = o;   o = align_up(o + (size_t)g.kp2 * 4, 256);
    L.off_c64T2 = o; o = align_up(o + (size_t)d * g.kp2 * 8, 256);
  }
  L.total = o;
  return L;
}

// Header at the start of the pack (device memory).
struct PackHeader {
  int k, d, dtype, pad;
  double cn_max;   // max_j ||c_j||^2 (float64) — used by the near-tie margin bound
  float scale;     // power of two s with s * max|c_ji| in [2^9, 2^10): the tensor path multiplies X and C by s
  float pad2;      // before the fp16 split, so that both fit fp16's range (exact: only exponents change)
};

// Magnitude window of the unscaled fp32 / bf16 distance arithmetic (families 0, 2 and 3): a row whose fp32
// ||x||^2 + max ||c||^2 lies outside [2^-100, 2^100] is decided in float64 like a near-tie.  Below the window the
// products fall into fp32's subnormals, whose absolute rounding (2^-149) exceeds the near-tie bound; above it they
// overflow.  NaN fails the test too.
__device__ __forceinline__ bool fp32_norm_in_window(float v) {
  return v >= 7.888609052210118e-31f && v <= 1.2676506002282294e30f;      // 2^-100, 2^100
}

// ---------------------------------------------------------------------------------------
// Workspace for one chunk call: per-CTA partials.  Sized for the largest grid we launch.
// ---------------------------------------------------------------------------------------
// Per-CTA partial sums: one [k*d] slot per CTA of the largest grid a CUDA-core kernel launches (8 CTAs per SM),
// fewer when a slot is large (a kernel whose per-CTA sums occupy most of the shared memory runs 1-2 CTAs per SM), and a
// single slot when k*d cannot be CTA-resident at all (generic kernel's GLOBAL mode: float64 atomics into slot 0, so the
// psum area always holds at least k*d doubles).
struct WsLayout {
  size_t off_bal, off_psum, off_pcnt, off_pin, off_flag, off_defer, off_rec, off_lab, off_bin, off_binoff, total;
  size_t psum_esz;
  int psum_slots;     // capacity of off_psum in [k*d] slots
  int part_slots;     // capacity of off_pcnt / off_pin (per-CTA counts / distance sums): the largest grid
};
static inline WsLayout ws_layout(long long n, int d, int k, int dtype, int sm_count = kDefaultSMs) {
  WsLayout W;
  if (sm_count <= 0) sm_count = kDefaultSMs;
  W.psum_esz = dtype == BKM_F64 ? 8 : 4;
  const size_t slot = (size_t)k * d * W.psum_esz;
  W.part_slots = sm_count * 8;
  const bool tc2 = tc2_shape(d, k, dtype);
  if (tc2) {
    // label-indexed row pass: one [k][d] slot per row block (sm_count / DS CTAs own the same row block)
    const Tc2Geom g = tc2_geom(k, d);
    W.psum_slots = sm_count / g.DS > 0 ? sm_count / g.DS : 1;
  } else if (2 * slot > 227 * 1024) W.psum_slots = 1;          // cannot be CTA-resident: global accumulation
  else {
    size_t per_sm = (227 * 1024) / (2 * slot);                  // CTAs per SM that could hold centres + sums
    if (per_sm > 8) per_sm = 8;
    if (per_sm < 1) per_sm = 1;
    W.psum_slots = (int)(sm_count * per_sm);
  }
  size_t o = 0;
  // FIXED offset (independent of n): the cluster -> warp balance table of the label-indexed M-step pass survives from one
  // chunk call to the next (16-byte header {magic, k, cluster slices} + one byte per cluster, k <= 4096)
  W.off_bal = o; o = align_up(o + 16 + 4096, 256);
  const size_t psum_bytes = (size_t)W.psum_slots * slot, global_bytes = (size_t)k * d * 8;
  W.off_psum = o; o = align_up(o + (psum_bytes > global_bytes ? psum_bytes : global_bytes), 256);
  W.off_pcnt = o; o = align_up(o + (size_t)W.part_slots * k * 4, 256);
  W.off_pin = o;  o = align_up(o + (size_t)W.part_slots * 8, 256);
  W.off_flag = o; o = align_up(o + 256, 256);          // [0] = deferred-row counter
  W.off_defer = o; o = align_up(o + (size_t)(n > 0 ? n : 0) * 4, 256);
  // large-shape tensor path with more than one centre slice: per (slice, row) partial arg-min records (16 B)
  W.off_rec = o;
  if (tc2 && tc2_geom(k, d).S > 1) o = align_up(o + (size_t)tc2_geom(k, d).S * (size_t)(n > 0 ? n : 0) * 16, 256);
  // ... and a label buffer for callers that do not want the labels (the row passes are driven by them)
  W.off_lab = o;
  if (tc2) o = align_up(o + (size_t)(n > 0 ? n : 0) * 4, 256);
  // ... and the per-tile bins of the M-step row pass: 4 B per row (tiles of 4096 rows) + 257 offsets per tile
  W.off_bin = W.off_binoff = o;
  if (tc2) {
    const size_t ntile = (size_t)((n > 0 ? n : 0) + 4095) / 4096;
    W.off_bin = o;    o = align_up(o + ntile * 4096 * 4, 256);
    W.off_binoff = o; o = align_up(o + ntile * 257 * 4, 256);
  }
  W.total = o;
  return W;
}

// Arguments shared by the fused chunk kernels (passed by value as one struct).
struct ChunkArgs {
  const void* X;
  long long n;
  int d;
  long long ldx;
  const unsigned char* pack;
  PackLayout L;
  int k;
  int* labels;        // nullable
  void* min_out;      // nullable; x-dtype
  int squared;        // 1: min_out/dist_sum are d^2 ; 0: sqrt(d^2)
  void* psum;         // [grid][k][d] partial sums (M-step only)
  int* pcnt;          // [grid][k]
  double* pin;        // [grid] partial sum of min distances
  float tau;          // near-tie margin coefficient (0 disables the f64 re-check)
  int want_sum;       // caller wants the summed min distance (inertia / cost)
  int* defer_cnt;     // tensor paths: number of rows deferred to the float64 re-check kernel
  int* defer_idx;     // [n] their row indices
  int psum_slots;     // capacity of psum in [k*d] slots (grid clamp of the kernels that keep per-CTA sums)
  int part_slots;     // capacity of pcnt / pin
  float4* rec;        // large-shape tensor path: [S][n] partial arg-min records {m1, m2, label bits, ||x||^2}
  void* bin_list;     // ... M-step row pass: per-tile row bins (4 B per row) and their bucket offsets
  int* bin_off;
  unsigned char* bal;  // ... and its persistent balance table (WsLayout::off_bal)
  float* xf_out;      // transform variants: output block (rows x k), row pitch xf_ld floats; mode 0 sqrt / 1 squared / 2 rbf
  long long xf_ld;
  int xf_mode;
  double xf_gamma;    // float64: the tensor path applies it as gamma / s^2, which an fp32 gamma could not carry
  const int* skip;    // nullable: device word (LoopState::done); non-zero -> every kernel of the call returns at once
  int first_chunk;    // reduce_partials overwrites the accumulators (first chunk of an iteration) instead of adding
  int counts_f64;     // the counts accumulator is float64 (one float64 buffer for the all-reduce) instead of int64
  double* out_sums;   // final accumulators (the re-check kernel adds the deferred rows' contributions)
  long long* out_counts;
  double* out_dist_sum;
};

// Device-resident state of a Lloyd loop (bkm_loop_reset / bkm_finalize_step): the stop test of
// dask_ml/cluster/k_means.py:555-559 runs on the device, iterations enqueued after convergence are no-ops.
struct LoopState {
  int done;          // set by the iteration whose shift < tol (its centre update is NOT applied: Q3)
  int n_iter;        // iterations executed (including the converging one)
  int hist_cap;
  int pad;
  double tol;
  double shift;      // shift of the last executed iteration
  double* hist;      // nullable: shift of iteration i at hist[i] (i < hist_cap)
};

// The end of one iteration's step (bkm_finalize_step, bkm_sparse_finalize_step), by one thread after every CTA of the
// step has read st->done and st->tol: record the shift, count the iteration, and stop the loop once it converged.
__device__ __forceinline__ void loop_commit(LoopState* st, double shift, bool converged) {
  st->pad = 0;
  st->shift = shift;
  if (st->hist && st->n_iter < st->hist_cap) st->hist[st->n_iter] = shift;
  st->n_iter += 1;
  __threadfence();
  if (converged) st->done = 1;
}

// implemented in bkm_simt.cu
int launch_simt(const ChunkArgs& a, bool mstep, int dtype, int sm_count, int* grid_out, cudaStream_t s);
int simt_layout(int d, int k, int dtype, bool mstep, int* out13);
// implemented in bkm_tc.cu
int launch_tc(const ChunkArgs& a, bool mstep, int sm_count, int* grid_out, cudaStream_t s);
int launch_tc_recheck(const ChunkArgs& a, bool mstep, int sm_count, cudaStream_t s);
int launch_tc_transform(const ChunkArgs& a, int sm_count, cudaStream_t s);
int launch_tc_colsum(const ChunkArgs& a, double* part, size_t part_bytes, int sm_count, int* parts_out, cudaStream_t s);
int launch_tc_embed(const ChunkArgs& a, const float* W, int kw, int sm_count, cudaStream_t s);
int tc_trace(long long* out, int n);
// implemented in bkm_stream.cu
bool stream_supported(int d, int k, int dtype);
int launch_stream(const ChunkArgs& a, bool mstep, int sm_count, int* grid_out, cudaStream_t s);
int stream_layout(int d, int k, long long ldx, int* out13);
// implemented in bkm_tc2.cu / bkm_rowpass.cu
int launch_tc2(const ChunkArgs& a, bool mstep, int sm_count, int* grid_out, cudaStream_t s);
int launch_rowpass_mstep(const ChunkArgs& a, int x_dtype, int sm_count, int* parts_out, cudaStream_t s);
int launch_rowpass_dist(const ChunkArgs& a, int x_dtype, int sm_count, int* parts_out, cudaStream_t s);
int rowpass_layout(int k, int d, long long n, int sm_count, int* out9);
// implemented in bkm_aux.cu
int launch_reduce_partials(const ChunkArgs& a, int sum_parts, int cnt_parts, int pin_parts, bool mstep, int psum_dtype,
                           double* sums, long long* counts, double* dist_sum, cudaStream_t s);

}  // namespace bkm
