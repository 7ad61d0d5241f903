// bkm_aux.cu — small kernels around the fused chunk kernel: centre packing, deterministic
// reduction of per-CTA partials, centre update + shift, k-means|| sampling, transform, NaN scan.
#include "bkm_common.cuh"
#include <math_constants.h>
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <atomic>

namespace bkm {

std::atomic<long long> g_launches{0};

// ---------------------------------------------------------------------------------------
// Centre pack: float64 centres [k][d] -> every layout the kernels read (offsets: pack_layout, bkm_common.cuh).
//   header     PackHeader: cn_max = max_j ||c_j||^2 and the scale s
//   cT   [k][d4] x-dtype (bf16 rows: fp32), zero padded      cnT  [k] the same dtype: ||c||^2
//   c64  [k][d]  float64 copy                                 cn64 [k] float64 ||c||^2
// family 1 (tc_supported, bkm_tc.cu):
//   bhi / blo [kp][64] fp16: rn(-2 s c), rn(-2 s c - bhi)     cns  [kp] fp32: rn(s^2 ||c||^2), 3e38 beyond k
//   c64T [d][kp] float64 (re-check)
// family 3 (tc2_shape, bkm_tc2.cu):
//   b2hi / b2lo [kp2][dk2] bf16: rn(-2 c), rn(-2 c - b2hi)    cn2  [kp2] fp32: rn(||c||^2), 3e38 beyond k
//   c64T2 [d][kp2] float64 (re-check)
// Tile entries beyond (k, d) are zero.  ||c||^2 is computed once, in float64 (pack_norms); every layout rounds that.
// The writers take the centres from a source: `C(i)` yields element i of the row-major (k, d) float64 centres.
// ---------------------------------------------------------------------------------------
struct CentreFromMemory {
  const double* p;
  __device__ __forceinline__ double operator()(size_t i) const { return p[i]; }
};

// scale = 2^(9 - floor(log2 max|c|)): s * max|c| in [2^9, 2^10), so -2 s c fits fp16 with a 32x margin and
// rows of X up to ~64x the largest centre component convert without overflow (larger ones are deferred to
// the float64 path by the kernel).  The exponent is clamped to [-126, 126], so that s and 1/s are normal floats: the
// transform epilogue divides by s twice in fp32.  So the rule holds whenever max|c| >= 2^-117.
__device__ __forceinline__ int pack_scale_exp(double max_abs_c) {
  int e = 0;
  if (max_abs_c > 0.0 && max_abs_c < CUDART_INF) e = 9 - ilogb(max_abs_c);
  return e > 126 ? 126 : (e < -126 ? -126 : e);
}

// maximum of v over the CTA, in every thread
__device__ __forceinline__ double block_max(double v) {
  __shared__ double red[32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  v = red[0];
  for (int w = 1; w < (int)(blockDim.x >> 5); ++w) v = fmax(v, red[w]);
  __syncthreads();
  return v;
}

// ||c_j||^2 -> cn[j] for the centres j = w, w + nw, ... of warp w (of nw): lane-strided fma, then the xor-shuffle tree
template <typename Src>
__device__ __forceinline__ void pack_norms(Src C, const PackLayout& L, double* cn, int w, int nw) {
  const int lane = threadIdx.x & 31;
  for (int j = w; j < L.k; j += nw) {
    double s = 0.0;
    for (int i = lane; i < L.d; i += 32) { const double v = C((size_t)j * L.d + i); s = fma(v, v, s); }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) cn[j] = s;
  }
}

// max |c| over one CTA (coalesced; on the one-kernel path it also brings the centres into L1 for pack_norms)
template <typename Src>
__device__ __forceinline__ double pack_max_abs(Src C, const PackLayout& L) {
  double m = 0.0;
#pragma unroll 8
  for (int i = threadIdx.x; i < L.k * L.d; i += blockDim.x) m = fmax(m, fabs(C(i)));
  return block_max(m);
}

// One CTA, after every cn[j] is written: the scale from max |c| (returned) and cn_max; CTA 0 writes the header.
__device__ __forceinline__ double pack_header(unsigned char* pack, const PackLayout& L, double max_abs,
                                              const double* cn) {
  const double sc = scalbn(1.0, pack_scale_exp(max_abs));
  double cm = 0.0;
  for (int j = threadIdx.x; j < L.k; j += blockDim.x) cm = fmax(cm, cn[j]);
  cm = block_max(cm);
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    PackHeader* h = reinterpret_cast<PackHeader*>(pack);
    h->k = L.k; h->d = L.d; h->dtype = L.dtype; h->pad = 0; h->cn_max = cm; h->scale = (float)sc; h->pad2 = 0.f;
  }
  return sc;
}

// cT and cnT in the element type T of the rows' layouts
template <typename T, typename Src>
__device__ __forceinline__ void pack_rows(Src C, unsigned char* pack, const PackLayout& L, const double* cn, int gt,
                                          int nth) {
  T* cT = reinterpret_cast<T*>(pack + L.off_cT);
  T* cnT = reinterpret_cast<T*>(pack + L.off_cnT);
  for (int i = gt; i < L.k * L.d4; i += nth) {
    const int r = i / L.d4, c = i - r * L.d4;
    cT[i] = c < L.d ? (T)C((size_t)r * L.d + c) : T(0);
  }
  for (int j = gt; j < L.k; j += nth) cnT[j] = (T)cn[j];
}

// 16-bit (hi, lo) pair of v: hi + lo carries 22 (fp16) or 16 (bf16) significant bits
__device__ __forceinline__ void split16(double v, __half& hi, __half& lo) {
  hi = __double2half(v);
  lo = __double2half(v - (double)__half2float(hi));
}
__device__ __forceinline__ void split16(double v, __nv_bfloat16& hi, __nv_bfloat16& lo) {
  hi = __double2bfloat16(v);
  lo = __double2bfloat16(v - (double)__bfloat162float(hi));
}

// MMA operand tiles [rows][cols] of f * C: row r = centre r, column c = feature c
template <typename H, typename Src>
__device__ __forceinline__ void pack_split_tiles(Src C, const PackLayout& L, H* hi, H* lo, int rows, int cols, double f,
                                                 int gt, int nth) {
  for (int i = gt; i < rows * cols; i += nth) {
    const int r = i / cols, c = i - r * cols;
    H h, l;
    split16(r < L.k && c < L.d ? f * C((size_t)r * L.d + c) : 0.0, h, l);
    hi[i] = h; lo[i] = l;
  }
}

// float64 centres transposed [d][cols] (coalesced over centres for the re-check kernels)
template <typename Src>
__device__ __forceinline__ void pack_transposed(Src C, const PackLayout& L, double* out, int cols, int gt, int nth) {
  for (int i = gt; i < L.d * cols; i += nth) {
    const int f = i / cols, j = i - f * cols;
    out[i] = j < L.k ? C((size_t)j * L.d + f) : 0.0;
  }
}

// Every layout but the header, grid-strided, from the norms cn and the scale sc.
template <typename Src>
__device__ __forceinline__ void pack_layouts(Src C, unsigned char* pack, const PackLayout& L, const double* cn,
                                             double sc) {
  const int k = L.k, gt = blockIdx.x * blockDim.x + threadIdx.x, nth = gridDim.x * blockDim.x;
  double* c64 = reinterpret_cast<double*>(pack + L.off_c64);
  double* cn64 = reinterpret_cast<double*>(pack + L.off_cn64);
  for (int i = gt; i < k * L.d; i += nth) c64[i] = C(i);
  if (cn != cn64)                                   // the large path's pack_norms_kernel wrote them in place
    for (int j = gt; j < k; j += nth) cn64[j] = cn[j];
  if (L.dtype == BKM_F64) pack_rows<double>(C, pack, L, cn, gt, nth);
  else pack_rows<float>(C, pack, L, cn, gt, nth);
  if (L.tc) {                                       // the tensor path works on s X and s C
    pack_split_tiles(C, L, reinterpret_cast<__half*>(pack + L.off_bhi), reinterpret_cast<__half*>(pack + L.off_blo),
                     L.kp, 64, -2.0 * sc, gt, nth);
    float* cns = reinterpret_cast<float*>(pack + L.off_cns);
    for (int j = gt; j < L.kp; j += nth) cns[j] = j < k ? (float)(cn[j] * sc * sc) : 3.0e38f;
    pack_transposed(C, L, reinterpret_cast<double*>(pack + L.off_c64T), L.kp, gt, nth);
  }
  if (L.tc2) {                                      // bf16 has fp32's range: no scale
    pack_split_tiles(C, L, reinterpret_cast<__nv_bfloat16*>(pack + L.off_b2hi),
                     reinterpret_cast<__nv_bfloat16*>(pack + L.off_b2lo), L.kp2, L.dk2, -2.0, gt, nth);
    float* cn2 = reinterpret_cast<float*>(pack + L.off_cn2);
    for (int j = gt; j < L.kp2; j += nth) cn2[j] = j < k ? (float)cn[j] : 3.0e38f;
    pack_transposed(C, L, reinterpret_cast<double*>(pack + L.off_c64T2), L.kp2, gt, nth);
  }
}

// Every CTA of one kernel computes the norms and the header quantities (k*d is a few thousand elements), then writes
// its share of the layouts: dependent launches cost more than the repeated work.  In shared memory: cn_s [k].
template <typename Src>
__device__ __forceinline__ void pack_small(Src C, unsigned char* pack, const PackLayout& L, double* cn_s) {
  const double m = pack_max_abs(C, L);
  pack_norms(C, L, cn_s, threadIdx.x >> 5, blockDim.x >> 5);
  __syncthreads();
  pack_layouts(C, pack, L, cn_s, pack_header(pack, L, m, cn_s));
}

__global__ void __launch_bounds__(1024)
pack_small_kernel(const double* __restrict__ C, unsigned char* pack, PackLayout L) {
  extern __shared__ double cn_s[];        // [k]
  pack_small(CentreFromMemory{C}, pack, L, cn_s);
}

// Large shapes: pack_norms_kernel writes the norms to the pack's cn64, then pack_layouts_kernel the rest; its CTA 0
// also the header.  The layouts do not wait for the scale: only family-1 layouts use it, and those shapes are small.
// st (nullable): the Lloyd loop of bkm_finalize_step; once it is done, its pack stays as it is.
__global__ void __launch_bounds__(256)
pack_norms_kernel(const double* __restrict__ C, unsigned char* pack, PackLayout L, const LoopState* st) {
  if (st && st->done) return;
  pack_norms(CentreFromMemory{C}, L, reinterpret_cast<double*>(pack + L.off_cn64),
             (blockIdx.x * blockDim.x + threadIdx.x) >> 5, (gridDim.x * blockDim.x) >> 5);
}

__global__ void __launch_bounds__(1024)
pack_layouts_kernel(const double* __restrict__ C, unsigned char* pack, PackLayout L, const LoopState* st) {
  if (st && st->done) return;
  const double* cn64 = reinterpret_cast<const double*>(pack + L.off_cn64);
  if (blockIdx.x == 0) pack_header(pack, L, pack_max_abs(CentreFromMemory{C}, L), cn64);
  pack_layouts(CentreFromMemory{C}, pack, L, cn64, 0.0);
}

// ---------------------------------------------------------------------------------------
// One Lloyd iteration's tail:
//   C' = sums / max(counts, 1)  (k_means.py:548-551, empty cluster -> zero vector)
//   shift = ||C - C'||_F^2      (k_means.py:555)        -> LoopState.shift, hist[n_iter], n_iter += 1
//   if shift < tol: LoopState.done = 1, C' is NOT taken over (k_means.py:558-560: break before the assignment) and
//   the pack is left as it is
//   else: c_out = C', and the centre pack for the NEXT iteration is built from C'.
// Every CTA recomputes the shift (fixed order -> the same value and the same decision everywhere); centres are read
// from c_in and written to c_out (two buffers: no CTA reads what another one writes).  red = [k*d sums | k counts as
// float64 | inertia] is the all-reduced buffer of the step.
// LAYOUTS (small shapes): the whole pack too (pack_small).  Otherwise (large shapes, one CTA) pack_norms_kernel and
// pack_layouts_kernel follow, reading c_out.
// ---------------------------------------------------------------------------------------
struct CentreFromSums {
  const double* red;
  int kd, d;
  __device__ __forceinline__ double operator()(size_t i) const {
    const double c = red[kd + (int)(i / (size_t)d)];
    return red[i] / (c > 1.0 ? c : 1.0);
  }
};

// STAGED: every CTA first evaluates C' = sums / max(counts, 1) ONCE into shared memory (k*d float64: 128 KB at C2) and
// all later passes (shift, norms, header, layouts) read that copy instead of repeating the float64 division per access — the
// same quotient, computed once (44 -> ~15 us at k*d = 16384).
template <bool STAGED, bool LAYOUTS>
__global__ void __launch_bounds__(1024)
finalize_step_kernel(const double* __restrict__ red, const double* __restrict__ c_in, double* __restrict__ c_out,
                     LoopState* st, unsigned char* pack, PackLayout L) {
  extern __shared__ double cn_s[];        // LAYOUTS: [k] (+ [k*d] staged centres)
  __shared__ double sred[32];
  if (st->done) return;
  const int k = L.k, d = L.d, kd = k * d, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const CentreFromSums cfs{red, kd, d};
  double* cs = cn_s + k;
  if (STAGED) {
    for (int i = tid; i < kd; i += 1024) cs[i] = cfs(i);
    __syncthreads();
  }
  const CentreFromMemory cmem{cs};
  double acc = 0.0;
  for (int i = tid; i < kd; i += 1024) { const double df = c_in[i] - (STAGED ? cmem(i) : cfs(i)); acc = fma(df, df, acc); }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) sred[wid] = acc;
  __syncthreads();
  double shift = 0.0;
  for (int w = 0; w < 32; ++w) shift += sred[w];
  __syncthreads();
  const bool converged = shift < st->tol;
  if (!converged) {
    for (int i = blockIdx.x * 1024 + tid; i < kd; i += gridDim.x * 1024) c_out[i] = STAGED ? cmem(i) : cfs(i);
    if (LAYOUTS && STAGED) pack_small(cmem, pack, L, cn_s);
    else if (LAYOUTS) pack_small(cfs, pack, L, cn_s);
  }
  // the state is written last, by one thread of the last CTA to get here (every CTA has read st->done / st->tol)
  __shared__ bool last;
  __threadfence();
  __syncthreads();
  if (tid == 0) last = atomicAdd(reinterpret_cast<unsigned int*>(&st->pad), 1u) == gridDim.x - 1;
  __syncthreads();
  if (last && tid == 0) {
    st->pad = 0;
    st->shift = shift;
    if (st->hist && st->n_iter < st->hist_cap) st->hist[st->n_iter] = shift;
    st->n_iter += 1;
    __threadfence();
    if (converged) st->done = 1;
  }
}

__global__ void loop_reset_kernel(LoopState* st, double tol, double* hist, int hist_cap) {
  st->done = 0; st->n_iter = 0; st->hist_cap = hist_cap; st->pad = 0;
  st->tol = tol; st->shift = CUDART_INF; st->hist = hist;
}

int launch_loop_reset(void* state, double tol, double* hist, int hist_cap, cudaStream_t s) {
  loop_reset_kernel<<<1, 1, 0, s>>>(reinterpret_cast<LoopState*>(state), tol, hist, hist_cap);
  note_launch();
  BKM_CUDA_TRY(cudaGetLastError());
  return 0;
}

// The one-kernel path: k*d up to 64 K elements (every shape of the fused chunk kernels).
static bool pack_in_one_kernel(const PackLayout& L) { return L.k <= 2048 && (long long)L.k * L.d <= 65536; }

// CTAs of a layouts pass: one per `per` elements of the largest layout, at most `cap`
static int pack_grid(const PackLayout& L, int per, int cap) {
  size_t n = (size_t)L.k * L.d4;
  if (L.tc && (size_t)L.kp * 64 > n) n = (size_t)L.kp * 64;
  if (L.tc2 && (size_t)L.kp2 * L.dk2 > n) n = (size_t)L.kp2 * L.dk2;
  const size_t nb = (n + per - 1) / per;
  return nb < 1 ? 1 : (nb > (size_t)cap ? cap : (int)nb);
}

int launch_pack(const double* C, int k, int d, int dtype, void* pack, cudaStream_t s) {
  const PackLayout L = pack_layout(k, d, dtype);
  unsigned char* p = (unsigned char*)pack;
  if (pack_in_one_kernel(L)) {
    pack_small_kernel<<<pack_grid(L, 2048, 16), 1024, (size_t)k * 8, s>>>(C, p, L);
    note_launch();
  } else {
    pack_norms_kernel<<<(k + 7) / 8 < 132 ? (k + 7) / 8 : 132, 256, 0, s>>>(C, p, L, nullptr);
    pack_layouts_kernel<<<pack_grid(L, 1024, 132), 1024, 0, s>>>(C, p, L, nullptr);
    note_launch(2);
  }
  BKM_CUDA_TRY(cudaGetLastError());
  return 0;
}

int launch_finalize_step(const double* red, const double* c_in, double* c_out, void* state, int k, int d, int dtype,
                         void* pack, cudaStream_t s) {
  const PackLayout L = pack_layout(k, d, dtype);
  LoopState* st = reinterpret_cast<LoopState*>(state);
  unsigned char* p = (unsigned char*)pack;
  if (pack_in_one_kernel(L)) {
    const int nb = pack_grid(L, 2048, 16);
    const size_t staged_bytes = ((size_t)k + (size_t)k * d) * 8;
    if (staged_bytes <= 200 * 1024) {
      if (staged_bytes > 48 * 1024)
        BKM_CUDA_TRY(cudaFuncSetAttribute(finalize_step_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          (int)staged_bytes));
      finalize_step_kernel<true, true><<<nb, 1024, staged_bytes, s>>>(red, c_in, c_out, st, p, L);
    } else {
      finalize_step_kernel<false, true><<<nb, 1024, (size_t)k * 8, s>>>(red, c_in, c_out, st, p, L);
    }
    note_launch();
  } else {
    finalize_step_kernel<false, false><<<1, 1024, 0, s>>>(red, c_in, c_out, st, p, L);
    pack_norms_kernel<<<(k + 7) / 8 < 132 ? (k + 7) / 8 : 132, 256, 0, s>>>(c_out, p, L, st);
    pack_layouts_kernel<<<pack_grid(L, 1024, 132), 1024, 0, s>>>(c_out, p, L, st);
    note_launch(3);
  }
  BKM_CUDA_TRY(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------------------
// One mini-batch step (scikit-learn's _minibatch_update_dense, sklearn/cluster/_k_means_minibatch.pyx), after the fused
// E+M pass over the batch left red = [k*d sums S | k counts n as float64 | inertia]:
//   c_out[j] = (c_in[j] * w_in[j] + S[j]) * (1 / (w_in[j] + n[j]))   where n[j] > 0, else c_in[j]
//   w_out[j] = w_in[j] + n[j]
// and the centre pack of c_out.  The products and sums are explicit round-to-nearest intrinsics: the expression is
// scikit-learn's, evaluated in float64 without FMA contraction.  Centres and weight sums are read from the *_in
// buffers and written to the *_out ones (ping-pong), so no CTA reads what another one writes.
// LAYOUTS (small shapes): every CTA also builds the whole pack (pack_small).  Otherwise pack_norms_kernel and
// pack_layouts_kernel follow, reading c_out.
// ---------------------------------------------------------------------------------------
struct CentreFromMinibatch {
  const double* red;
  const double* c;
  const double* w;
  int kd, d;
  __device__ __forceinline__ double operator()(size_t i) const {
    const int j = (int)(i / (size_t)d);
    const double n = red[kd + j];
    if (!(n > 0.0)) return c[i];
    const double alpha = __ddiv_rn(1.0, __dadd_rn(w[j], n));
    return __dmul_rn(__dadd_rn(__dmul_rn(c[i], w[j]), red[i]), alpha);
  }
};

// STAGED: every CTA evaluates the new centres once into shared memory ([k] norms + [k*d] centres), as
// finalize_step_kernel does; the pack passes then read that copy.
template <bool STAGED, bool LAYOUTS>
__global__ void __launch_bounds__(1024)
minibatch_step_kernel(const double* __restrict__ red, const double* __restrict__ c_in, const double* __restrict__ w_in,
                      double* __restrict__ c_out, double* __restrict__ w_out, unsigned char* pack, PackLayout L) {
  extern __shared__ double cn_s[];        // LAYOUTS: [k] (+ [k*d] staged centres)
  const int k = L.k, kd = k * L.d, tid = threadIdx.x;
  const CentreFromMinibatch cmb{red, c_in, w_in, kd, L.d};
  double* cs = cn_s + k;
  if (STAGED) {
    for (int i = tid; i < kd; i += blockDim.x) cs[i] = cmb(i);
    __syncthreads();
  }
  const CentreFromMemory cmem{cs};
  const int gt = blockIdx.x * blockDim.x + tid, nth = gridDim.x * blockDim.x;
  for (int i = gt; i < kd; i += nth) c_out[i] = STAGED ? cmem(i) : cmb(i);
  for (int j = gt; j < k; j += nth) w_out[j] = __dadd_rn(w_in[j], red[kd + j]);
  if (LAYOUTS && STAGED) pack_small(cmem, pack, L, cn_s);
  else if (LAYOUTS) pack_small(cmb, pack, L, cn_s);
}

int launch_minibatch_step(const double* red, const double* c_in, const double* w_in, double* c_out, double* w_out,
                          int k, int d, int dtype, void* pack, cudaStream_t s) {
  const PackLayout L = pack_layout(k, d, dtype);
  unsigned char* p = (unsigned char*)pack;
  if (pack_in_one_kernel(L)) {
    const int nb = pack_grid(L, 2048, 16);
    const size_t staged_bytes = ((size_t)k + (size_t)k * d) * 8;
    if (staged_bytes <= 200 * 1024) {
      if (staged_bytes > 48 * 1024)
        BKM_CUDA_TRY(cudaFuncSetAttribute(minibatch_step_kernel<true, true>,
                                          cudaFuncAttributeMaxDynamicSharedMemorySize, (int)staged_bytes));
      minibatch_step_kernel<true, true><<<nb, 1024, staged_bytes, s>>>(red, c_in, w_in, c_out, w_out, p, L);
    } else {
      minibatch_step_kernel<false, true><<<nb, 1024, (size_t)k * 8, s>>>(red, c_in, w_in, c_out, w_out, p, L);
    }
    note_launch();
  } else {
    const long long kd = (long long)k * d;
    const int nb = (int)((kd + 1023) / 1024 < 132 ? (kd + 1023) / 1024 : 132);
    minibatch_step_kernel<false, false><<<nb, 1024, 0, s>>>(red, c_in, w_in, c_out, w_out, p, L);
    pack_norms_kernel<<<(k + 7) / 8 < 132 ? (k + 7) / 8 : 132, 256, 0, s>>>(c_out, p, L, nullptr);
    pack_layouts_kernel<<<pack_grid(L, 1024, 132), 1024, 0, s>>>(c_out, p, L, nullptr);
    note_launch(3);
  }
  BKM_CUDA_TRY(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------------------
// reduce_partials: fold the per-CTA partials of one chunk into the float64 accumulators in a
// FIXED order (CTA 0,1,2,...), so a chunk's contribution is bit-reproducible run to run.
// ---------------------------------------------------------------------------------------
template <typename PS>
__global__ void reduce_partials_kernel(const PS* __restrict__ psum, const int* __restrict__ pcnt,
                                       const double* __restrict__ pin, int cnt_parts, int pin_parts, int sum_parts,
                                       int kd, int k, bool mstep,
                                       double* sums, long long* counts, double* dist_sum,
                                       const int* skip, int first, int counts_f64) {
  if (skip && *skip) return;
  const int tid = blockIdx.x * blockDim.x + threadIdx.x;
  const int nth = gridDim.x * blockDim.x;
  // The additions run in CTA order (that is what makes a chunk's contribution reproducible); the loads of a
  // batch are independent, so 16 of them are in flight at a time instead of one.
  if (mstep) {
    // sums: thread (x, y) of a 32 x 8 block adds the partials y, y + 8, ... of output 32 * block + x (coalesced across
    // x, 8 independent chains per output instead of one), then the 8 chain sums are added in order y = 0..7: a fixed
    // order, so a chunk's contribution is bit-reproducible run to run.
    __shared__ double part_s[8][33];
    const int x = threadIdx.x & 31, y = threadIdx.x >> 5;
    for (int i0 = blockIdx.x * 32; i0 < kd; i0 += gridDim.x * 32) {
      const int i = i0 + x;
      double s = 0.0;
      if (i < kd) {
        int g = y;
        for (; g + 24 < sum_parts; g += 32) {
          const PS v0 = psum[(size_t)g * kd + i], v1 = psum[(size_t)(g + 8) * kd + i];
          const PS v2 = psum[(size_t)(g + 16) * kd + i], v3 = psum[(size_t)(g + 24) * kd + i];
          s += (double)v0; s += (double)v1; s += (double)v2; s += (double)v3;
        }
        for (; g < sum_parts; g += 8) s += (double)psum[(size_t)g * kd + i];
      }
      part_s[y][x] = s;
      __syncthreads();
      if (y == 0 && i < kd) {
        double t = part_s[0][x];
#pragma unroll
        for (int q = 1; q < 8; ++q) t += part_s[q][x];
        sums[i] = first ? t : sums[i] + t;
      }
      __syncthreads();
    }
    // counts: the last CTAs take them (the first ones already carry the tail of the sums loop)
    for (int i = nth - 1 - tid; i < k; i += nth) {
      long long c = 0;
      int g = 0;
      for (; g + 16 <= cnt_parts; g += 16) {
        int v[16];
#pragma unroll
        for (int q = 0; q < 16; ++q) v[q] = pcnt[(size_t)(g + q) * k + i];
#pragma unroll
        for (int q = 0; q < 16; ++q) c += v[q];
      }
      for (; g < cnt_parts; ++g) c += pcnt[(size_t)g * k + i];
      if (counts_f64) { double* cf = reinterpret_cast<double*>(counts); cf[i] = first ? (double)c : cf[i] + (double)c; }
      else counts[i] = first ? c : counts[i] + c;
    }
  }
  if (blockIdx.x == 0 && threadIdx.x < 32 && dist_sum) {
    // lane l adds CTAs l, l+32, ... in order, then a fixed shuffle tree: reproducible
    double s = 0.0;
    for (int g = threadIdx.x; g < pin_parts; g += 32) s += pin[g];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (threadIdx.x == 0) *dist_sum = first ? s : *dist_sum + s;
  }
}

// sum_parts / cnt_parts / pin_parts: how many partial slots the chunk kernel(s) wrote of the sums, the counts and the
// distance sums (one per CTA for the fused kernels; 1 sums slot in the generic kernel's GLOBAL mode; row blocks and
// distance-pass CTAs for the large-shape path).  psum_dtype: BKM_F64 when the partial sums are float64 (float64 rows, and
// the generic kernel's GLOBAL slot whatever the rows are), else they are fp32.
int launch_reduce_partials(const ChunkArgs& a, int sum_parts, int cnt_parts, int pin_parts, bool mstep, int psum_dtype,
                           double* sums, long long* counts, double* dist_sum, cudaStream_t s) {
  const int kd = a.k * a.d;
  int nb = (kd + 31) / 32; if (nb > 592) nb = 592; if (nb < 1) nb = 1;      // blocks of 32 outputs x 8 partial chains
  if (psum_dtype != BKM_F64)
    reduce_partials_kernel<float><<<nb, 256, 0, s>>>((const float*)a.psum, a.pcnt, a.pin, cnt_parts, pin_parts, sum_parts,
                                                     kd, a.k, mstep, sums, counts, dist_sum, a.skip, a.first_chunk, a.counts_f64);
  else
    reduce_partials_kernel<double><<<nb, 256, 0, s>>>((const double*)a.psum, a.pcnt, a.pin, cnt_parts, pin_parts, sum_parts,
                                                      kd, a.k, mstep, sums, counts, dist_sum, a.skip, a.first_chunk, a.counts_f64);
  note_launch();
  BKM_CUDA_TRY(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------------------
// finalize: C' = sums / max(counts,1) ; shift = ||C - C'||_F^2   (k_means.py:548-555)
// up to 64 CTAs; the last one to finish adds the per-CTA parts in CTA order -> deterministic shift.
// The per-launch scratch is one of 32 slots handed out round-robin by the host (an atomic counter), so finalize calls
// of different estimators / streams / host threads in flight at the same time never share one.
// ---------------------------------------------------------------------------------------
static const int kFinSlots = 32;
__device__ double g_fin_part[kFinSlots][64];
__device__ unsigned int g_fin_done[kFinSlots];
static std::atomic<unsigned int> g_fin_seq{0};

__global__ void __launch_bounds__(1024)
finalize_kernel(const double* __restrict__ sums, const long long* __restrict__ counts,
                const double* __restrict__ Cold, double* __restrict__ Cnew,
                double* shift, int k, int d, int slot) {
  __shared__ double sm[32];
  __shared__ bool last;
  double acc = 0.0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < k * d; i += gridDim.x * blockDim.x) {
    int j = i / d;
    long long c = counts[j];
    double cn = sums[i] / (double)(c > 1 ? c : 1);
    Cnew[i] = cn;
    double df = Cold[i] - cn;
    acc = fma(df, df, acc);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += sm[w];
    g_fin_part[slot][blockIdx.x] = s;
    __threadfence();
    last = atomicAdd(&g_fin_done[slot], 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (last && threadIdx.x == 0) {
    // the last CTA to finish adds the per-CTA parts in CTA order: deterministic shift
    __threadfence();
    double s = 0.0;
    for (int b = 0; b < (int)gridDim.x; ++b) s += *(volatile double*)&g_fin_part[slot][b];
    *shift = s;
    g_fin_done[slot] = 0;
  }
}

int launch_finalize(const double* sums, const long long* counts, const double* Cold, double* Cnew,
                    double* shift, int k, int d, cudaStream_t s) {
  int nb = (k * d + 1023) / 1024; if (nb > 64) nb = 64; if (nb < 1) nb = 1;
  const int slot = (int)(g_fin_seq.fetch_add(1u) % kFinSlots);
  finalize_kernel<<<nb, 1024, 0, s>>>(sums, counts, Cold, Cnew, shift, k, d, slot);
  note_launch();
  BKM_CUDA_TRY(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------------------
// k-means|| Bernoulli sampling (k_means.py:472-491).  U_i = Philox4x32-10 keyed by `seed`,
// counter = global row index; the first 32-bit output word / 2^32 is the uniform draw.
// The same generator is restated in numpy under tests/ so the draw sequence is pinned.
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t philox_first_word(uint64_t seed, uint64_t ctr) {
  uint32_t c0 = (uint32_t)ctr, c1 = (uint32_t)(ctr >> 32), c2 = 0u, c3 = 0u;
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return c0;
}

template <typename T>
__global__ void sample_kernel(const T* __restrict__ d2, long long n, double ell_over_phi,
                              uint64_t seed, uint64_t row_offset, long long* picked, long long cap,
                              int* n_picked) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x) {
    double p = ell_over_phi * (double)d2[i];
    double u = (double)philox_first_word(seed, row_offset + (uint64_t)i) * (1.0 / 4294967296.0);
    if (p > u) {
      int slot = atomicAdd(n_picked, 1);
      if (slot < cap) picked[slot] = (long long)(row_offset + (uint64_t)i);
    }
  }
}

int launch_sample(const void* d2, long long n, int dtype, double eop, uint64_t seed, uint64_t off,
                  long long* picked, long long cap, int* n_picked, cudaStream_t s) {
  if (n == 0) return 0;
  long long nb = (n + 255) / 256; if (nb > 132 * 8) nb = 132 * 8;
  if (dtype == BKM_F32)
    sample_kernel<float><<<(int)nb, 256, 0, s>>>((const float*)d2, n, eop, seed, off, picked, cap, n_picked);
  else
    sample_kernel<double><<<(int)nb, 256, 0, s>>>((const double*)d2, n, eop, seed, off, picked, cap, n_picked);
  note_launch();
  BKM_CUDA_TRY(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------------------
// transform: out[i][j] = sqrt(max(||x_i||^2 - 2 x_i.c_j + ||c_j||^2, 0))   (pairwise.py:79-97)
// computed in the dtype of X like the reference does.  Output-bandwidth bound: each CTA stages
// 64 rows, every thread produces (row, 4 centres) micro-tiles, results go out through smem so
// the global stores are coalesced along k.
// ---------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256)
transform_kernel(const T* __restrict__ X, long long n, int d, long long ldx,
                 const unsigned char* __restrict__ pack, PackLayout L, T* __restrict__ out, long long ld_out, int mode,
                 double gamma, int TR) {
  extern __shared__ __align__(16) unsigned char smem[];   // TR rows per tile: 64, fewer for very wide rows
  const int k = L.k, d4 = L.d4;
  T* xs = reinterpret_cast<T*>(smem);                // [TR][d4+1]
  T* xn = xs + TR * (d4 + 1);                        // [TR]
  const T* C = reinterpret_cast<const T*>(pack + L.off_cT);
  const T* cn = reinterpret_cast<const T*>(pack + L.off_cnT);
  const int tid = threadIdx.x;
  const long long ntiles = (n + TR - 1) / TR;
  for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const long long r0 = tile * TR;
    const int rows = (int)min((long long)TR, n - r0);
    __syncthreads();
    for (int e = tid; e < rows * d; e += 256) {
      int r = e / d, c = e - r * d;
      xs[r * (d4 + 1) + c] = X[(r0 + r) * ldx + c];
    }
    __syncthreads();
    if (tid < rows) {
      T s = T(0);
      for (int i = 0; i < d; ++i) { T v = xs[tid * (d4 + 1) + i]; s = fma(v, v, s); }
      xn[tid] = s;
    }
    __syncthreads();
    // thread -> (centre j fastest, row) so that stores are coalesced along k
    for (long long e = tid; e < (long long)rows * k; e += 256) {
      int r = (int)(e / k), j = (int)(e - (long long)r * k);
      const T* xr = xs + r * (d4 + 1);
      const T* cr = C + (size_t)j * d4;
      T acc = T(0);
      for (int i = 0; i < d; ++i) acc = fma(xr[i], cr[i], acc);
      T v = xn[r] + cn[j] - T(2) * acc;
      v = v > T(0) ? v : T(0);
      out[(r0 + r) * ld_out + j] = mode == 0 ? sqrt(v) : (mode == 1 ? v : (T)exp(-(T)gamma * v));
    }
  }
}

int launch_transform(const void* X, long long n, int d, long long ldx, int dtype,
                     const void* pack, int k, void* out, long long ld_out, int mode, double gamma, int sm_count,
                     cudaStream_t s) {
  if (n == 0) return 0;
  PackLayout L = pack_layout(k, d, dtype);
  size_t esz = dtype == BKM_F64 ? 8 : 4;
  int TR = 64;                                   // rows per tile; wide rows (d in the hundreds / thousands) take fewer
  while (TR > 1 && (size_t)TR * (L.d4 + 1) * esz + TR * esz + 16 > 200 * 1024) TR >>= 1;
  size_t smem = (size_t)TR * (L.d4 + 1) * esz + TR * esz + 16;
  if (smem > 227 * 1024) return BKM_EUNSUPPORTED;
  long long ntiles = (n + TR - 1) / TR;
  long long grid = (long long)sm_count * 4; if (grid > ntiles) grid = ntiles;
  if (dtype == BKM_F32) {
    BKM_CUDA_TRY(cudaFuncSetAttribute(transform_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    transform_kernel<float><<<(int)grid, 256, smem, s>>>((const float*)X, n, d, ldx, (const unsigned char*)pack, L, (float*)out, ld_out, mode, gamma, TR);
  } else {
    BKM_CUDA_TRY(cudaFuncSetAttribute(transform_kernel<double>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    transform_kernel<double><<<(int)grid, 256, smem, s>>>((const double*)X, n, d, ldx, (const unsigned char*)pack, L, (double*)out, ld_out, mode, gamma, TR);
  }
  note_launch();
  BKM_CUDA_TRY(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------------------
// Nystrom passes of SpectralClustering (spectral.py:237-282) on the CUDA cores, any shape, computed in the dtype of X:
//   COLSUM (mode 0): part[cta][j] = sum over the CTA's rows of exp(-gamma y_ij),  y_ij = max(||x_i||^2 - 2 x_i.c_j
//                    + ||c_j||^2, 0), accumulated in float64 (colsum_fold adds the CTAs in order), for the keep rows
//                    j0 <= j < j0 + lb of one launch (the host launches one per block of lb keep rows)
//   EMBED  (mode 1): out_i = e_i / ||e_i||,  e_i = sum_j exp(-gamma (y_ij - m_i)) W_j,  m_i = min_j y_ij; NaN where
//                    gamma m_i > 745.13 (the float64 reference's kernel row is 0 there).  The l kernel values go through
//                    shared memory lb at a time; when l > lb, a first sweep finds m_i and the second recomputes y.
// One warp per row (rows in a fixed order per warp); lane j handles keep rows j, j + 32, ...  Per warp in shared
// memory: the row, lb kernel values and kw outputs; COLSUM adds the warp's float64 column sums [lb].  Every sum runs
// over j (rows) in the same order whatever lb is, so the results do not depend on the blocking.
// ---------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256)
nystrom_kernel(const T* __restrict__ X, long long n, int d, long long ldx, const unsigned char* __restrict__ pack,
               PackLayout L, double gamma, int mode, const T* __restrict__ W, int kw, T* __restrict__ out,
               long long ld_out, double* __restrict__ part, int j0, int lb) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int l = L.k, d4 = L.d4, lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const size_t per_warp = ((size_t)(d4 + lb + kw) * sizeof(T) + 15) / 16 * 16;
  double* cacc = reinterpret_cast<double*>(smem);                                           // [nw][lb] (COLSUM)
  unsigned char* wbase = smem + (mode == 0 ? ((size_t)nw * lb * 8 + 15) / 16 * 16 : 0) + wid * per_warp;
  T* xw = reinterpret_cast<T*>(wbase);                // [d4]
  T* vw = xw + d4;                                    // [lb]
  T* ew = vw + lb;                                    // [kw]
  const T* C = reinterpret_cast<const T*>(pack + L.off_cT);
  const T* cn = reinterpret_cast<const T*>(pack + L.off_cnT);
  const T g = (T)gamma;
  const bool one = l <= lb;                           // EMBED: every kernel value of a row fits at once
  if (mode == 0)
    for (int j = lane; j < lb; j += 32) cacc[wid * lb + j] = 0.0;
  for (long long row = (long long)blockIdx.x * nw + wid; row < n; row += (long long)gridDim.x * nw) {
    __syncwarp();
    for (int i = lane; i < d; i += 32) xw[i] = X[row * ldx + i];
    __syncwarp();
    T xn = T(0);
    for (int i = lane; i < d; i += 32) xn = fma(xw[i], xw[i], xn);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) xn += __shfl_xor_sync(0xffffffffu, xn, o);   // the same value in every lane
    auto y_of = [&](int j) {
      const T* cr = C + (size_t)j * d4;
      T acc = T(0);
      for (int i = 0; i < d; ++i) acc = fma(xw[i], cr[i], acc);
      const T y = xn + cn[j] - T(2) * acc;
      return y > T(0) ? y : T(0);
    };
    if (mode == 0) {
      for (int j = lane; j < lb; j += 32) cacc[wid * lb + j] += (double)exp(-g * y_of(j0 + j));
      continue;
    }
    T m = T(CUDART_INF);
    for (int j = lane; j < l; j += 32) {
      const T y = y_of(j);
      if (one) vw[j] = y;
      m = y < m ? y : m;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { const T v = __shfl_xor_sync(0xffffffffu, m, o); m = v < m ? v : m; }
    for (int o = lane; o < kw; o += 32) ew[o] = T(0);
    for (int b0 = 0; b0 < l; b0 += lb) {
      const int nb = min(lb, l - b0);
      for (int j = lane; j < nb; j += 32) vw[j] = exp(-g * ((one ? vw[j] : y_of(b0 + j)) - m));
      __syncwarp();
      for (int o = lane; o < kw; o += 32) {
        T e = ew[o];
        for (int j = 0; j < nb; ++j) e = fma(vw[j], W[(size_t)(b0 + j) * kw + o], e);
        ew[o] = e;
      }
      __syncwarp();
    }
    T nrm = T(0);
    for (int o = lane; o < kw; o += 32) nrm = fma(ew[o], ew[o], nrm);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) nrm += __shfl_xor_sync(0xffffffffu, nrm, o);
    const T f = ((double)m * gamma > 745.13) ? T(CUDART_NAN) : T(1) / sqrt(nrm);
    for (int o = lane; o < kw; o += 32) out[row * ld_out + o] = ew[o] * f;
  }
  if (mode != 0) return;
  __syncthreads();
  for (int j = threadIdx.x; j < lb; j += blockDim.x) {
    double s = 0.0;
    for (int w = 0; w < nw; ++w) s += cacc[w * lb + j];
    part[(size_t)blockIdx.x * l + j0 + j] = s;
  }
}

// colsum[j] (+)= sum of the partial slots p = 0, 1, ... in order (first: overwrite)
__global__ void colsum_fold_kernel(const double* __restrict__ part, int parts, int l, double* colsum, int first) {
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < l; j += gridDim.x * blockDim.x) {
    double s = 0.0;
    for (int p = 0; p < parts; ++p) s += part[(size_t)p * l + j];
    colsum[j] = first ? s : colsum[j] + s;
  }
}

int launch_colsum_fold(const double* part, int parts, int l, double* colsum, int first, cudaStream_t s) {
  colsum_fold_kernel<<<(l + 255) / 256, 256, 0, s>>>(part, parts, l, colsum, first);
  note_launch();
  BKM_CUDA_TRY(cudaGetLastError());
  return 0;
}

// mode 0: column sums into part ([grid][l] float64, *parts_out = grid); mode 1: embedding rows into out.
// Shared memory decides the warps per CTA (8 down to 1) and the block of keep rows lb (l down to 32).
int launch_nystrom(const void* X, long long n, int d, long long ldx, int dtype, const void* pack, int l, double gamma,
                   int mode, const void* W, int kw, void* out, long long ld_out, double* part, size_t part_bytes,
                   int sm_count, int* parts_out, cudaStream_t s) {
  PackLayout L = pack_layout(l, d, dtype);
  const size_t esz = dtype == BKM_F64 ? 8 : 4;
  auto smem_of = [&](int w, int b) {
    return (mode == 0 ? align_up((size_t)w * b * 8, 16) : 0) + (size_t)w * align_up((size_t)(L.d4 + b + kw) * esz, 16);
  };
  int nw = 8, lb = l;
  while (smem_of(nw, lb) > 200 * 1024) {
    if (lb > 1024) lb = (lb / 2 + 31) / 32 * 32;
    else if (nw > 1) nw >>= 1;
    else if (lb > 32) lb = (lb / 2 + 31) / 32 * 32;
    else break;
  }
  const size_t smem = smem_of(nw, lb);
  if (smem > 227 * 1024) return BKM_EUNSUPPORTED;      // a row of X plus k outputs alone exceed shared memory
  long long grid = (n + nw - 1) / nw;
  if (grid > (long long)sm_count * 4) grid = (long long)sm_count * 4;
  if (grid < 1) grid = 1;
  if (mode == 0) {
    if ((size_t)grid * l * 8 > part_bytes) return BKM_EWORKSPACE;
    *parts_out = (int)grid;
  }
  if (dtype == BKM_F32)
    BKM_CUDA_TRY(cudaFuncSetAttribute(nystrom_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  else
    BKM_CUDA_TRY(cudaFuncSetAttribute(nystrom_kernel<double>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  // COLSUM: one launch per block of lb keep rows; EMBED: one launch (the kernel walks the blocks itself)
  for (int j0 = 0; j0 < l; j0 += lb) {
    const int nb = mode == 0 ? (l - j0 < lb ? l - j0 : lb) : lb;
    if (dtype == BKM_F32)
      nystrom_kernel<float><<<(int)grid, nw * 32, smem, s>>>((const float*)X, n, d, ldx, (const unsigned char*)pack, L,
                                                             gamma, mode, (const float*)W, kw, (float*)out, ld_out, part,
                                                             j0, nb);
    else
      nystrom_kernel<double><<<(int)grid, nw * 32, smem, s>>>((const double*)X, n, d, ldx, (const unsigned char*)pack, L,
                                                              gamma, mode, (const double*)W, kw, (double*)out, ld_out,
                                                              part, j0, nb);
    note_launch();
    BKM_CUDA_TRY(cudaGetLastError());
    if (mode != 0) break;
  }
  return 0;
}

// ---------------------------------------------------------------------------------------
// k-means|| rounds (k_means.py:423-431 / 466-469): the reference re-evaluates the distances to ALL candidates every
// round; min_j d(x, c_j) over a growing set is the running minimum of the per-round minima.  This kernel folds the
// minima of the new candidates into the running minimum and sums the result (the cost phi) in one pass, with a fixed
// reduction order (per-CTA partial -> last CTA adds them in CTA order), so phi is reproducible.
// ---------------------------------------------------------------------------------------
static const int kFoldSlots = 32;
__device__ double g_fold_part[kFoldSlots][1024];
__device__ unsigned int g_fold_done[kFoldSlots];
static std::atomic<unsigned int> g_fold_seq{0};

template <typename T>
__global__ void __launch_bounds__(256)
min_fold_kernel(T* __restrict__ run_min, const T* __restrict__ new_min, long long n, double* phi_acc, int slot) {
  __shared__ double sm[8];
  __shared__ bool last;
  double acc = 0.0;
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
    T v = run_min[i];
    if (new_min) { const T w = new_min[i]; v = w < v ? w : v; run_min[i] = v; }
    acc += (double)v;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int w = 0; w < 8; ++w) s += sm[w];
    g_fold_part[slot][blockIdx.x] = s;
    __threadfence();
    last = atomicAdd(&g_fold_done[slot], 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (last && threadIdx.x == 0) {
    __threadfence();
    double s = 0.0;
    for (int b = 0; b < (int)gridDim.x; ++b) s += *(volatile double*)&g_fold_part[slot][b];
    if (phi_acc) *phi_acc += s;
    g_fold_done[slot] = 0;
  }
}

int launch_min_fold(void* run_min, const void* new_min, long long n, int dtype, double* phi_acc, int sm_count, cudaStream_t s) {
  if (n == 0) return 0;
  long long nb = (n + 2047) / 2048;
  if (nb > 1024) nb = 1024;
  if (nb > (long long)sm_count * 4) nb = (long long)sm_count * 4;
  const int slot = (int)(g_fold_seq.fetch_add(1u) % kFoldSlots);
  if (dtype == BKM_F64) min_fold_kernel<double><<<(int)nb, 256, 0, s>>>((double*)run_min, (const double*)new_min, n, phi_acc, slot);
  else min_fold_kernel<float><<<(int)nb, 256, 0, s>>>((float*)run_min, (const float*)new_min, n, phi_acc, slot);
  note_launch();
  BKM_CUDA_TRY(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------------------
// Device generator for datasets.make_blobs blocks (dask_ml/datasets.py:178-189: every block is generated on its own
// from (centres, cluster_std, seed = block index)).  Row i of the block: label = floor(U_i * k) from one Philox stream,
// features = centre[label] + std[label] * N(0, 1) with Box-Muller normals from a second Philox stream keyed by the same
// seed; counters are (row, feature pair), so a block is reproducible whatever GPU / grid generates it.
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ void philox_two_words(uint64_t seed, uint64_t ctr, uint32_t& w0, uint32_t& w1) {
  uint32_t c0 = (uint32_t)ctr, c1 = (uint32_t)(ctr >> 32), c2 = 0u, c3 = 0u;
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  w0 = c0; w1 = c1;
}

template <typename T>
__global__ void make_blobs_kernel(T* __restrict__ X, long long* __restrict__ y, long long n, int d, long long ldx,
                                  const double* __restrict__ centers, const double* __restrict__ stds, int k,
                                  uint64_t seed) {
  const int pairs = (d + 1) / 2;
  const long long total = n * pairs;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const long long row = e / pairs;
    const int p = (int)(e - row * pairs);
    const uint32_t lw = philox_first_word(seed ^ 0x5bd1e995a5a5a5a5ull, (uint64_t)row);
    int lab = (int)(((unsigned long long)lw * (unsigned long long)k) >> 32);
    if (lab >= k) lab = k - 1;
    uint32_t w0, w1;
    philox_two_words(seed, (uint64_t)e, w0, w1);
    const double u1 = ((double)w0 + 1.0) * (1.0 / 4294967296.0);          // (0, 1]
    const double u2 = (double)w1 * (1.0 / 4294967296.0);
    const double rad = sqrt(-2.0 * log(u1));
    double sn, cs;
    sincospi(2.0 * u2, &sn, &cs);
    const double sd = stds[lab];
    const int f0 = 2 * p, f1 = 2 * p + 1;
    X[row * ldx + f0] = (T)(centers[(size_t)lab * d + f0] + sd * rad * cs);
    if (f1 < d) X[row * ldx + f1] = (T)(centers[(size_t)lab * d + f1] + sd * rad * sn);
    if (p == 0 && y) y[row] = lab;
  }
}

int launch_make_blobs(void* X, long long* y, long long n, int d, long long ldx, int dtype, const double* centers,
                      const double* stds, int k, uint64_t seed, int sm_count, cudaStream_t s) {
  if (n == 0) return 0;
  long long nb = (n * ((d + 1) / 2) + 255) / 256; if (nb > (long long)sm_count * 16) nb = (long long)sm_count * 16;
  if (dtype == BKM_F32) make_blobs_kernel<float><<<(int)nb, 256, 0, s>>>((float*)X, y, n, d, ldx, centers, stds, k, seed);
  else make_blobs_kernel<double><<<(int)nb, 256, 0, s>>>((double*)X, y, n, d, ldx, centers, stds, k, seed);
  note_launch();
  BKM_CUDA_TRY(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------------------
// NaN / inf scan (k_means.py:179-180)
// ---------------------------------------------------------------------------------------
template <typename T> __device__ __forceinline__ double cf_to_double(T v) { return (double)v; }
template <> __device__ __forceinline__ double cf_to_double<__nv_bfloat16>(__nv_bfloat16 v) { return (double)__bfloat162float(v); }

template <typename T>
__global__ void check_finite_kernel(const T* __restrict__ X, long long n, int d, long long ldx, int* flag) {
  bool bad = false;
  if (ldx == d) {
    const long long tot = n * d;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < tot;
         i += (long long)gridDim.x * blockDim.x) {
      T v = X[i];
      bad |= !(fabs(cf_to_double<T>(v)) <= 1.7976931348623157e308);
    }
  } else {
    for (long long r = blockIdx.x; r < n; r += gridDim.x)
      for (int c = threadIdx.x; c < d; c += blockDim.x) {
        T v = X[r * ldx + c];
        bad |= !(fabs(cf_to_double<T>(v)) <= 1.7976931348623157e308);
      }
  }
  if (__syncthreads_or(bad) && threadIdx.x == 0) atomicOr(flag, 1);
}

int launch_check_finite(const void* X, long long n, int d, long long ldx, int dtype, int* flag,
                        int sm_count, cudaStream_t s) {
  if (n == 0) return 0;
  int grid = sm_count * 8;
  if (dtype == BKM_F32) check_finite_kernel<float><<<grid, 256, 0, s>>>((const float*)X, n, d, ldx, flag);
  else if (dtype == BKM_BF16) check_finite_kernel<__nv_bfloat16><<<grid, 256, 0, s>>>((const __nv_bfloat16*)X, n, d, ldx, flag);
  else check_finite_kernel<double><<<grid, 256, 0, s>>>((const double*)X, n, d, ldx, flag);
  note_launch();
  BKM_CUDA_TRY(cudaGetLastError());
  return 0;
}

}  // namespace bkm
