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
// pack_centers: float64 centres [k][d] -> every layout the kernels read (see PackLayout).
//   cT   [k][d4]  x-dtype, zero padded          cnT  [k] x-dtype   ||c||^2 (computed in f64)
//   c64  [k][d]   float64 copy                  cn64 [k] float64
//   bhi  [kp][64] fp16: rn(-2 s c)              blo  [kp][64] fp16: rn(-2 s c - bhi)   (s = header scale)
//   cn32 [kp]     fp32 ||c||^2, +inf for padded centres
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ float to_tf32_rna(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}

__global__ void pack_centers_kernel(const double* __restrict__ C, unsigned char* pack, PackLayout L) {
  const int k = L.k, d = L.d;
  const int tid = blockIdx.x * blockDim.x + threadIdx.x;
  const int nth = gridDim.x * blockDim.x;
  double* c64 = reinterpret_cast<double*>(pack + L.off_c64);
  for (int i = tid; i < k * d; i += nth) c64[i] = C[i];
  if (L.dtype != BKM_F64) {
    float* cT = reinterpret_cast<float*>(pack + L.off_cT);
    for (int i = tid; i < k * L.d4; i += nth) {
      int r = i / L.d4, c = i - r * L.d4;
      cT[i] = c < d ? (float)C[(size_t)r * d + c] : 0.f;
    }
    // tensor-core operands: B = -2 s C as an fp16 pair (hi + lo carries 22 significant bits); rows/columns
    // beyond (k, d) are zero.  Only shapes the tensor path takes (d <= 64) have room in the pack.
    if (d <= L.dh) {
      const double sc = (double)reinterpret_cast<const PackHeader*>(pack)->scale;
      __half* bhi = reinterpret_cast<__half*>(pack + L.off_bhi);
      __half* blo = reinterpret_cast<__half*>(pack + L.off_blo);
      for (int i = tid; i < L.kp * L.dh; i += nth) {
        int r = i / L.dh, c = i - r * L.dh;
        __half hi = __float2half_rn(0.f), lo = hi;
        if (r < k && c < d) {
          const double v = -2.0 * sc * C[(size_t)r * d + c];
          hi = __double2half(v);
          lo = __double2half(v - (double)__half2float(hi));
        }
        bhi[i] = hi; blo[i] = lo;
      }
    }
  } else {
    double* cT = reinterpret_cast<double*>(pack + L.off_cT);
    for (int i = tid; i < k * L.d4; i += nth) {
      int r = i / L.d4, c = i - r * L.d4;
      cT[i] = c < d ? C[(size_t)r * d + c] : 0.0;
    }
  }
}

// one warp per centre: ||c||^2 in float64, then block 0 computes the max.
__global__ void pack_norms_kernel(const double* __restrict__ C, unsigned char* pack, PackLayout L) {
  const int k = L.k, d = L.d;
  const int lane = threadIdx.x & 31;
  const int wid = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nw = (gridDim.x * blockDim.x) >> 5;
  double* cn64 = reinterpret_cast<double*>(pack + L.off_cn64);
  float* cn32 = reinterpret_cast<float*>(pack + L.off_cn32);
  for (int j = wid; j < L.kp; j += nw) {
    double s = 0.0;
    if (j < k) for (int i = lane; i < d; i += 32) { double v = C[(size_t)j * d + i]; s = fma(v, v, s); }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) {
      if (j < k) {
        cn64[j] = s;
        if (L.dtype != BKM_F64) reinterpret_cast<float*>(pack + L.off_cnT)[j] = (float)s;
        else reinterpret_cast<double*>(pack + L.off_cnT)[j] = s;
      }
      if (L.dtype != BKM_F64) {
        cn32[j] = j < k ? (float)s : CUDART_INF_F;
        // ||c_j||^2 as a K=8 tf32 operand row [hi, mid, lo, 0...] (hi+mid+lo == fp32 value exactly) in the
        // canonical no-swizzle K-major layout: 8-row groups of 256 B = [8 rows x 16 B | 8 rows x 16 B].
        float* bcn = reinterpret_cast<float*>(pack + L.off_bcn) + (j >> 3) * 64 + (j & 7) * 4;
        float hi = 3.0e38f, mid = 0.f, lo = 0.f;
        if (j < k) {
          const double sc = (double)reinterpret_cast<const PackHeader*>(pack)->scale;
          const float cf = (float)(s * sc * sc);          // the tensor path works on s X and s C
          hi = to_tf32_rna(cf);
          const float r1 = cf - hi;
          mid = to_tf32_rna(r1);
          lo = r1 - mid;
        }
        bcn[0] = hi; bcn[1] = mid; bcn[2] = lo; bcn[3] = 0.f;
        bcn[32] = 0.f; bcn[33] = 0.f; bcn[34] = 0.f; bcn[35] = 0.f;
      }
    }
  }
}

// scale = 2^(9 - floor(log2 max|c|)): s * max|c| in [2^9, 2^10), so -2 s c fits fp16 with a 32x margin and
// rows of X up to ~64x the largest centre component convert without overflow (larger ones are deferred to
// the float64 path by the kernel).  Runs first: the other pack kernels read it.
__global__ void pack_scale_kernel(const double* __restrict__ C, unsigned char* pack, PackLayout L) {
  __shared__ double sm[32];
  double m = 0.0;
  for (int i = threadIdx.x; i < L.k * L.d; i += blockDim.x) m = fmax(m, fabs(C[i]));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) m = fmax(m, sm[w]);
    int e = 0;
    if (m > 0.0 && m < CUDART_INF) e = 9 - ilogb(m);
    e = e > 100 ? 100 : (e < -100 ? -100 : e);
    PackHeader* h = reinterpret_cast<PackHeader*>(pack);
    h->scale = (float)scalbn(1.0, e);
    h->pad2 = 0.f;
  }
}

__global__ void pack_header_kernel(unsigned char* pack, PackLayout L) {
  const double* cn64 = reinterpret_cast<const double*>(pack + L.off_cn64);
  __shared__ double sm[32];
  double m = 0.0;
  for (int j = threadIdx.x; j < L.k; j += blockDim.x) m = fmax(m, cn64[j]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) m = fmax(m, sm[w]);
    PackHeader* h = reinterpret_cast<PackHeader*>(pack);
    h->k = L.k; h->d = L.d; h->dtype = L.dtype; h->pad = 0; h->cn_max = m;
  }
}

// Small (k, d) — every shape the tensor path takes — are packed by ONE kernel: each CTA recomputes the two
// global quantities (max |c| -> scale, all ||c||^2 -> cn_max; k*d is a few thousand elements) and then writes
// its share of every layout.  Four dependent launches cost more than the work itself.
// The body is shared by pack_fused_kernel (centres read from memory) and finalize_step_fused_kernel (centres computed
// on the fly from the reduced sums and counts): `C(i)` yields element i of the row-major (k, d) float64 centres.
template <typename Src>
__device__ __forceinline__ void pack_fused_body(Src C, unsigned char* pack, const PackLayout& L, double* cn_s) {
  __shared__ double red[32];
  const int k = L.k, d = L.d, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  // ---- max |c| -> scale
  double m = 0.0;
#pragma unroll 8
  for (int i = tid; i < k * d; i += 1024) m = fmax(m, fabs(C(i)));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
  if (lane == 0) red[wid] = m;
  __syncthreads();
  m = red[0];
  for (int w = 1; w < 32; ++w) m = fmax(m, red[w]);
  int e = 0;
  if (m > 0.0 && m < CUDART_INF) e = 9 - ilogb(m);
  e = e > 100 ? 100 : (e < -100 ? -100 : e);
  const double sc = scalbn(1.0, e);
  __syncthreads();
  // ---- ||c_j||^2 (one warp per centre, same summation order as pack_norms_kernel) and their maximum
  for (int j = wid; j < k; j += 32) {
    double s = 0.0;
    for (int i = lane; i < d; i += 32) { double v = C((size_t)j * d + i); s = fma(v, v, s); }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) cn_s[j] = s;
  }
  __syncthreads();
  double cm = 0.0;
  for (int j = tid; j < k; j += 1024) cm = fmax(cm, cn_s[j]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) cm = fmax(cm, __shfl_xor_sync(0xffffffffu, cm, o));
  if (lane == 0) red[wid] = cm;
  __syncthreads();
  if (blockIdx.x == 0 && tid == 0) {
    cm = red[0];
    for (int w = 1; w < 32; ++w) cm = fmax(cm, red[w]);
    PackHeader* h = reinterpret_cast<PackHeader*>(pack);
    h->k = k; h->d = d; h->dtype = L.dtype; h->pad = 0; h->cn_max = cm; h->scale = (float)sc; h->pad2 = 0.f;
  }
  // ---- this CTA's share of the layouts
  const int gt = blockIdx.x * 1024 + tid, nth = gridDim.x * 1024;
  double* c64 = reinterpret_cast<double*>(pack + L.off_c64);
  for (int i = gt; i < k * d; i += nth) c64[i] = C(i);
  double* cn64 = reinterpret_cast<double*>(pack + L.off_cn64);
  if (L.dtype != BKM_F64) {
    float* cT = reinterpret_cast<float*>(pack + L.off_cT);
    for (int i = gt; i < k * L.d4; i += nth) {
      int r = i / L.d4, c = i - r * L.d4;
      cT[i] = c < d ? (float)C((size_t)r * d + c) : 0.f;
    }
    if (d <= L.dh) {
      __half* bhi = reinterpret_cast<__half*>(pack + L.off_bhi);
      __half* blo = reinterpret_cast<__half*>(pack + L.off_blo);
      for (int i = gt; i < L.kp * L.dh; i += nth) {
        int r = i / L.dh, c = i - r * L.dh;
        __half hi = __float2half_rn(0.f), lo = hi;
        if (r < k && c < d) {
          const double v = -2.0 * sc * C((size_t)r * d + c);
          hi = __double2half(v);
          lo = __double2half(v - (double)__half2float(hi));
        }
        bhi[i] = hi; blo[i] = lo;
      }
    }
    if (L.off_c64T != L.total) {
      double* cTT = reinterpret_cast<double*>(pack + L.off_c64T);
      for (int i = gt; i < d * L.kp; i += nth) {
        int f = i / L.kp, j = i - f * L.kp;
        cTT[i] = j < k ? C((size_t)j * d + f) : 0.0;
      }
    }
    float* cn32 = reinterpret_cast<float*>(pack + L.off_cn32);
    for (int j = gt; j < L.kp; j += nth) {
      const double s = j < k ? cn_s[j] : 0.0;
      if (j < k) { cn64[j] = s; reinterpret_cast<float*>(pack + L.off_cnT)[j] = (float)s; }
      cn32[j] = j < k ? (float)s : CUDART_INF_F;
      float* bcn = reinterpret_cast<float*>(pack + L.off_bcn) + (j >> 3) * 64 + (j & 7) * 4;
      float hi = 3.0e38f, mid = 0.f, lo = 0.f;
      if (j < k) {
        const float cf = (float)(s * sc * sc);          // the tensor path works on s X and s C
        hi = to_tf32_rna(cf);
        const float r1 = cf - hi;
        mid = to_tf32_rna(r1);
        lo = r1 - mid;
      }
      bcn[0] = hi; bcn[1] = mid; bcn[2] = lo; bcn[3] = 0.f;
      bcn[32] = 0.f; bcn[33] = 0.f; bcn[34] = 0.f; bcn[35] = 0.f;
    }
  } else {
    double* cT = reinterpret_cast<double*>(pack + L.off_cT);
    for (int i = gt; i < k * L.d4; i += nth) {
      int r = i / L.d4, c = i - r * L.d4;
      cT[i] = c < d ? C((size_t)r * d + c) : 0.0;
    }
    for (int j = gt; j < k; j += nth) { cn64[j] = cn_s[j]; reinterpret_cast<double*>(pack + L.off_cnT)[j] = cn_s[j]; }
  }
}

struct CentreFromMemory {
  const double* p;
  __device__ __forceinline__ double operator()(size_t i) const { return p[i]; }
};

__global__ void __launch_bounds__(1024)
pack_fused_kernel(const double* __restrict__ C, unsigned char* pack, PackLayout L) {
  extern __shared__ double cn_s[];        // [k]
  pack_fused_body(CentreFromMemory{C}, pack, L, cn_s);
}

// ---------------------------------------------------------------------------------------
// One Lloyd iteration's tail in ONE kernel (small k*d, i.e. every shape of the fused chunk kernels):
//   C' = sums / max(counts, 1)  (k_means.py:548-551, empty cluster -> zero vector)
//   shift = ||C - C'||_F^2      (k_means.py:555)        -> LoopState.shift, hist[n_iter], n_iter += 1
//   if shift < tol: LoopState.done = 1, C' is NOT taken over (k_means.py:558-560: break before the assignment)
//   else: c_out = C', and the centre pack for the NEXT iteration is built from C' right here.
// Every CTA recomputes the shift (fixed order -> the same value and the same decision everywhere) and the two global
// quantities of the pack; centres are read from c_in and written to c_out (two buffers: no CTA reads what another one
// writes).  red = [k*d sums | k counts as float64 | inertia] is the all-reduced buffer of the step.
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
// all later passes (shift, max |c|, norms, the five layouts) read that copy instead of repeating the float64 division
// per access — the same quotient, computed once (44 -> ~15 us at k*d = 16384).
template <bool STAGED>
__global__ void __launch_bounds__(1024)
finalize_step_fused_kernel(const double* __restrict__ red, const double* __restrict__ c_in, double* __restrict__ c_out,
                           LoopState* st, unsigned char* pack, PackLayout L) {
  extern __shared__ double cn_s[];        // [k] (+ [k*d] staged centres)
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
    if (STAGED) pack_fused_body(cmem, pack, L, cn_s);
    else pack_fused_body(cfs, pack, L, cn_s);
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

// Large k*d: single-CTA state update (shift, stop test, centre hand-over); the pack follows as separate kernels.
__global__ void __launch_bounds__(1024)
finalize_state_kernel(const double* __restrict__ red, const double* __restrict__ c_in, double* __restrict__ c_out,
                      LoopState* st, int k, int d) {
  __shared__ double sred[32];
  if (st->done) return;
  const int kd = k * d, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const CentreFromSums cnew{red, kd, d};
  double acc = 0.0;
  for (int i = tid; i < kd; i += 1024) { const double df = c_in[i] - cnew(i); acc = fma(df, df, acc); }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) sred[wid] = acc;
  __syncthreads();
  double shift = 0.0;
  for (int w = 0; w < 32; ++w) shift += sred[w];
  const bool converged = shift < st->tol;
  // on convergence c_out = c_in, so that the pack kernels that follow (and the host) always read c_out
  for (int i = tid; i < kd; i += 1024) c_out[i] = converged ? c_in[i] : cnew(i);
  __syncthreads();
  if (tid == 0) {
    st->shift = shift;
    if (st->hist && st->n_iter < st->hist_cap) st->hist[st->n_iter] = shift;
    st->n_iter += 1;
    __threadfence();
    if (converged) st->done = 2;       // 2: converged in THIS iteration (bkm_finalize_step's pack still runs once)
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

// Layouts of the large-shape tensor path (bkm_tc2.cu), written after the float64 norms:
//   b2hi / b2lo [kp2][dk2] bf16: rn(-2 c), rn(-2 c - hi)          (row j = centre j; rows >= k and columns >= d: zero)
//   bcn2 [kp2] rows [hi, mid, lo, 0 | 0 0 0 0] tf32 of ||c_j||^2 in the no-swizzle K-major operand layout; rows >= k: 3e38
//   c64T2 [d][kp2] float64 (re-check)
__global__ void pack_tc2_kernel(const double* __restrict__ C, unsigned char* pack, PackLayout L, Tc2Geom g) {
  const int k = L.k, d = L.d;
  const int gt = blockIdx.x * blockDim.x + threadIdx.x, nth = gridDim.x * blockDim.x;
  const double* cn64 = reinterpret_cast<const double*>(pack + L.off_cn64);
  __nv_bfloat16* bhi = reinterpret_cast<__nv_bfloat16*>(pack + L.off_b2hi);
  __nv_bfloat16* blo = reinterpret_cast<__nv_bfloat16*>(pack + L.off_b2lo);
  for (int i = gt; i < g.kp2 * g.dk2; i += nth) {
    const int r = i / g.dk2, c = i - r * g.dk2;
    __nv_bfloat16 hi = __float2bfloat16_rn(0.f), lo = hi;
    if (r < k && c < d) {
      const double v = -2.0 * C[(size_t)r * d + c];
      hi = __double2bfloat16(v);
      lo = __double2bfloat16(v - (double)__bfloat162float(hi));
    }
    bhi[i] = hi; blo[i] = lo;
  }
  for (int j = gt; j < g.kp2; j += nth) {
    float* bcn = reinterpret_cast<float*>(pack + L.off_bcn2) + (j >> 3) * 64 + (j & 7) * 4;
    float hi = 3.0e38f, mid = 0.f, lo = 0.f;
    if (j < k) {
      const float cf = (float)cn64[j];
      hi = to_tf32_rna(cf);
      const float r1 = cf - hi;
      mid = to_tf32_rna(r1);
      lo = r1 - mid;
    }
    bcn[0] = hi; bcn[1] = mid; bcn[2] = lo; bcn[3] = 0.f;
    bcn[32] = 0.f; bcn[33] = 0.f; bcn[34] = 0.f; bcn[35] = 0.f;
  }
  double* cTT = reinterpret_cast<double*>(pack + L.off_c64T2);
  for (int i = gt; i < d * g.kp2; i += nth) {
    const int f = i / g.kp2, j = i - f * g.kp2;
    cTT[i] = j < k ? C[(size_t)j * d + f] : 0.0;
  }
}

static int launch_pack_tc2(const double* C, const PackLayout& L, void* pack, cudaStream_t s) {
  if (!tc2_shape(L.d, L.k, L.dtype)) return 0;
  const Tc2Geom g = tc2_geom(L.k, L.d);
  int nb = (g.kp2 * g.dk2 + 1023) / 1024; if (nb > 296) nb = 296; if (nb < 1) nb = 1;
  pack_tc2_kernel<<<nb, 256, 0, s>>>(C, (unsigned char*)pack, L, g);
  note_launch();
  BKM_CUDA_TRY(cudaGetLastError());
  return 0;
}

int launch_pack(const double* C, int k, int d, int dtype, void* pack, cudaStream_t s) {
  PackLayout L = pack_layout(k, d, dtype);
  if (k <= 2048 && (long long)k * d <= 65536) {
    int nb = (L.kp * L.dk + 2047) / 2048; if (nb > 16) nb = 16; if (nb < 1) nb = 1;
    pack_fused_kernel<<<nb, 1024, (size_t)k * 8, s>>>(C, (unsigned char*)pack, L);
    note_launch();
    BKM_CUDA_TRY(cudaGetLastError());
    return launch_pack_tc2(C, L, pack, s);
  }
  int nb = (L.kp * L.dk + 255) / 256; if (nb > 296) nb = 296; if (nb < 1) nb = 1;
  pack_scale_kernel<<<1, 1024, 0, s>>>(C, (unsigned char*)pack, L);
  pack_centers_kernel<<<nb, 256, 0, s>>>(C, (unsigned char*)pack, L);
  int nb2 = (L.kp + 7) / 8; if (nb2 > 132) nb2 = 132;
  pack_norms_kernel<<<nb2, 256, 0, s>>>(C, (unsigned char*)pack, L);
  pack_header_kernel<<<1, 256, 0, s>>>((unsigned char*)pack, L);
  note_launch(4);
  BKM_CUDA_TRY(cudaGetLastError());
  return launch_pack_tc2(C, L, pack, s);
}

int launch_finalize_step(const double* red, const double* c_in, double* c_out, void* state, int k, int d, int dtype,
                         void* pack, cudaStream_t s) {
  PackLayout L = pack_layout(k, d, dtype);
  LoopState* st = reinterpret_cast<LoopState*>(state);
  if (k <= 2048 && (long long)k * d <= 65536 && !tc2_shape(d, k, dtype)) {
    int nb = (L.kp * L.dk + 2047) / 2048; if (nb > 16) nb = 16; if (nb < 1) nb = 1;
    const size_t staged_bytes = ((size_t)k + (size_t)k * d) * 8;
    if (staged_bytes <= 200 * 1024) {
      if (staged_bytes > 48 * 1024)
        BKM_CUDA_TRY(cudaFuncSetAttribute(finalize_step_fused_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          (int)staged_bytes));
      finalize_step_fused_kernel<true><<<nb, 1024, staged_bytes, s>>>(red, c_in, c_out, st, (unsigned char*)pack, L);
    } else {
      finalize_step_fused_kernel<false><<<nb, 1024, (size_t)k * 8, s>>>(red, c_in, c_out, st, (unsigned char*)pack, L);
    }
    note_launch();
    BKM_CUDA_TRY(cudaGetLastError());
    return 0;
  }
  finalize_state_kernel<<<1, 1024, 0, s>>>(red, c_in, c_out, st, k, d);
  note_launch();
  BKM_CUDA_TRY(cudaGetLastError());
  return launch_pack(c_out, k, d, dtype, pack, s);
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
// distance-pass CTAs for the large-shape path)
int launch_reduce_partials(const ChunkArgs& a, int sum_parts, int cnt_parts, int pin_parts, bool mstep, int dtype,
                           double* sums, long long* counts, double* dist_sum, cudaStream_t s) {
  const int kd = a.k * a.d;
  int nb = (kd + 31) / 32; if (nb > 592) nb = 592; if (nb < 1) nb = 1;      // blocks of 32 outputs x 8 partial chains
  if (dtype != BKM_F64)
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
