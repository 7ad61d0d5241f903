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

// ---------------------------------------------------------------------------------------
// Centre pack: one device buffer holding every layout of the (k,d) centres the kernels use.
// Built by pack_centers_kernel from the float64 centres (reference keeps centres in f64:
// dask_ml/cluster/k_means.py:551-552).
// ---------------------------------------------------------------------------------------
struct PackLayout {
  int k, d, dtype;
  int d4;      // d rounded up to a multiple of 4 (SIMT row pitch, zero padded)
  int kp;      // k rounded up to a multiple of 16 (MMA N granularity)
  int dk;      // d rounded up to a multiple of 32 (one 128-byte swizzle atom of fp32 per K-block)
  int dh;      // row length of the fp16 MMA operand tiles: 64 halves = one 128-byte swizzle atom (d <= 64)
  size_t esz;  // sizeof(T)
  size_t off_cT, off_cnT, off_c64, off_cn64, off_bhi, off_blo, off_cn32, off_bcn, off_c64T, total;
  // large-shape tensor path (tc2_shape): fp16 (hi, lo) operand tiles [kp2][dk2], ||c||^2 operand rows [kp2][8] tf32,
  // float64 centres transposed [d][kp2]
  size_t off_b2hi, off_b2lo, off_bcn2, off_c64T2;
};

static inline PackLayout pack_layout(int k, int d, int dtype) {
  PackLayout L;
  L.k = k; L.d = d; L.dtype = dtype;
  L.d4 = (d + 3) / 4 * 4;
  L.kp = (k + 15) / 16 * 16;
  L.dk = (d + 31) / 32 * 32;
  L.dh = 64;
  L.esz = dtype == BKM_F64 ? 8 : 4;                // bf16 input: the fp32 layouts (the kernels widen the rows)
  size_t o = 256;  // header
  L.off_cT = o;   o = align_up(o + (size_t)k * L.d4 * L.esz, 256);
  L.off_cnT = o;  o = align_up(o + (size_t)k * L.esz, 256);
  L.off_c64 = o;  o = align_up(o + (size_t)k * d * 8, 256);
  L.off_cn64 = o; o = align_up(o + (size_t)k * 8, 256);
  L.off_bhi = o;  o = align_up(o + (size_t)L.kp * L.dh * 2, 256);   // fp16 tiles (tensor path, d <= 64)
  L.off_blo = o;  o = align_up(o + (size_t)L.kp * L.dh * 2, 256);
  L.off_cn32 = o; o = align_up(o + (size_t)L.kp * 4, 256);
  L.off_bcn = o;  o = align_up(o + (size_t)L.kp * 32, 256);   // ||c||^2 as an MMA operand tile (see bkm_tc.cu)
  // float64 centres transposed [d][kp] for the float64 re-check of the tensor path (coalesced over centres)
  L.off_c64T = o; if (dtype == BKM_F32 && d <= 64 && k <= 256) o = align_up(o + (size_t)d * L.kp * 8, 256);
  L.off_b2hi = L.off_b2lo = L.off_bcn2 = L.off_c64T2 = o;
  if (tc2_shape(d, k, dtype)) {
    const Tc2Geom g = tc2_geom(k, d);
    L.off_b2hi = o;  o = align_up(o + (size_t)g.kp2 * g.dk2 * 2, 1024);
    L.off_b2lo = o;  o = align_up(o + (size_t)g.kp2 * g.dk2 * 2, 1024);
    L.off_bcn2 = o;  o = align_up(o + (size_t)g.kp2 * 32, 256);
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

// ---------------------------------------------------------------------------------------
// Workspace for one chunk call: per-CTA partials.  Sized for the largest grid we launch.
// ---------------------------------------------------------------------------------------
// Per-CTA partial sums: one [k*d] slot per CTA of the largest grid a CUDA-core kernel launches (8 CTAs per SM),
// fewer when a slot is large (a kernel whose per-CTA sums occupy most of the shared memory runs 1-2 CTAs per SM), and a
// single slot when k*d cannot be CTA-resident at all (generic kernel's GLOBAL mode: atomics into slot 0).
static const int kDefaultSMs = 132;     // H100 SXM: sizing when no device is visible

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
  W.off_psum = o; o = align_up(o + (size_t)W.psum_slots * slot, 256);
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
  float xf_gamma;
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

// implemented in bkm_simt.cu
int launch_simt(const ChunkArgs& a, bool mstep, int dtype, int sm_count, int* grid_out, cudaStream_t s);
// implemented in bkm_tc.cu
bool tc_supported(int d, int k, int dtype);
int launch_tc(const ChunkArgs& a, bool mstep, int sm_count, int* grid_out, cudaStream_t s);
int launch_tc_recheck(const ChunkArgs& a, bool mstep, int sm_count, cudaStream_t s);
int launch_tc_transform(const ChunkArgs& a, int sm_count, cudaStream_t s);
int tc_trace(long long* out, int n);
// implemented in bkm_stream.cu
bool stream_supported(int d, int k, int dtype);
int launch_stream(const ChunkArgs& a, bool mstep, int sm_count, int* grid_out, cudaStream_t s);
// implemented in bkm_tc2.cu / bkm_rowpass.cu
int launch_tc2(const ChunkArgs& a, bool mstep, int sm_count, int* grid_out, cudaStream_t s);
int launch_rowpass_mstep(const ChunkArgs& a, int x_dtype, int sm_count, int* parts_out, cudaStream_t s);
int launch_rowpass_dist(const ChunkArgs& a, int x_dtype, int sm_count, int* parts_out, cudaStream_t s);
// implemented in bkm_aux.cu
int launch_reduce_partials(const ChunkArgs& a, int sum_parts, int cnt_parts, int pin_parts, bool mstep, int dtype,
                           double* sums, long long* counts, double* dist_sum, cudaStream_t s);

}  // namespace bkm
