// bkm_glm.cu — the fused pass of the generalised linear models (LogisticRegression, LinearRegression,
// PoissonRegression) over one row chunk, in float64 arithmetic (sm_90a).
//
//   eta_i = x_i . beta[0:d] + beta[d]                       (rows widened to float64, as in the Gram pass)
//   family  mu                loss_i                        r_i = c (mu - y)      Newton weight w_i
//   0 logistic  sigmoid(eta)  softplus(eta) - y eta         mu - y                mu (1 - mu)
//   1 normal    eta           (y - eta)^2                   2 (mu - y)            2
//   2 poisson   exp(eta)      exp(eta) - y eta              mu - y                mu
//
//   gradient mode: grad = [sum r_i x_i (d) | sum r_i | sum loss_i]
//   Newton mode:   the same, plus w_i per row and hrow = [sum w_i x_i (d) | sum w_i] (the intercept row of the
//                  Hessian; the (d, d) block comes from bkm_gram_weighted_chunk with these w_i)
//   predict modes: out_i = mu_i (float64) or mu_i > 0.5 (uint8); nothing is accumulated.
//
// A CTA walks tiles of TR rows.  Phase A: each warp takes TR / 8 rows, the lanes split the features, and a butterfly
// shuffle gives every lane the same eta; lane q < RW evaluates the family for the warp's row q, keeps r_i and w_i in
// shared memory and adds loss, r and w to its own registers (the lanes are added in lane order at the end).
// Phase B: the threads split the features into column groups and the tile rows into row groups, sum r_i x_ij (and
// w_i x_ij) over their rows in order, and the row groups are added in order into the CTA's partial in the workspace
// (one owner per element).  After the last tile the warps are added in order, and the last CTA to finish (a ticket counter) adds the CTA partials in CTA order.  So every sum has a fixed order: two calls
// with the same inputs give the same bits, and there are no float atomics.
//
// Phase A reads rows whose base, pitch and width are multiples of 16 bytes with 16-byte vector loads (lane l takes
// the 16-byte segments l, l + 32, ...); other rows are read with element loads, so every base address and row pitch
// works.  Phase B re-reads the tile with element loads; it is still in L1 / L2.
//
// exp(eta) above 709.78 is +inf (no clamp): the loss and the gradient become +inf, which the caller sees (the host
// solvers reject such a step and halve it).  The softplus is max(eta, 0) + log1p(exp(-|eta|)) and the sigmoid is
// evaluated on the side where exp does not overflow, so every finite eta gives a finite logistic loss and a mu in [0, 1].
#include "bkm_common.cuh"
#include <cuda_bf16.h>

namespace bkm {
namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int TR = 32;                 // rows per tile
constexpr int RW = TR / kWarps;        // rows per warp in phase A

enum { GLM_GRAD = 0, GLM_NEWTON = 1, GLM_PREDICT = 2, GLM_LABEL = 3 };

__device__ __forceinline__ double to_f64(float v) { return (double)v; }
__device__ __forceinline__ double to_f64(double v) { return v; }
__device__ __forceinline__ double to_f64(__nv_bfloat16 v) { return (double)__bfloat162float(v); }

// element v of a 16-byte segment, widened to float64 (v is a compile-time constant after unrolling)
__device__ __forceinline__ unsigned word(const uint4& u, int k) { return k == 0 ? u.x : k == 1 ? u.y : k == 2 ? u.z : u.w; }
template <typename T> __device__ __forceinline__ double lane_elem(const uint4& u, int v);
template <> __device__ __forceinline__ double lane_elem<float>(const uint4& u, int v) {
  return (double)__uint_as_float(word(u, v));
}
template <> __device__ __forceinline__ double lane_elem<double>(const uint4& u, int v) {
  return __hiloint2double((int)word(u, 2 * v + 1), (int)word(u, 2 * v));
}
template <> __device__ __forceinline__ double lane_elem<__nv_bfloat16>(const uint4& u, int v) {
  return (double)__uint_as_float(((word(u, v >> 1) >> (16 * (v & 1))) & 0xffffu) << 16);
}

struct GlmArgs {
  const void* X;
  long long n;
  int d;
  long long ldx;
  const double* y;
  const double* beta;     // [d + 1]: coefficients, then the intercept
  int family, mode;
  double* grad;           // [d + 2]
  double* hrow;           // [d + 1]   (Newton)
  double* w;              // [n]       (Newton)
  void* out;              // [n]       (predict)
  double* part;           // [grid][P] CTA partials, P = 2 d + 3: [r x (d) | r | loss | w x (d) | w]
  unsigned int* ticket;
  int first;
  int vec;                // rows are 16-byte aligned: phase A uses vector loads
};

// (mu, loss, r, w) of one row
__device__ __forceinline__ void family_terms(int family, double eta, double y, double& mu, double& loss, double& r,
                                             double& w) {
  if (family == 0) {
    const double e = exp(-fabs(eta));                     // in (0, 1]: never overflows
    mu = eta >= 0.0 ? 1.0 / (1.0 + e) : e / (1.0 + e);
    loss = (fmax(eta, 0.0) + log1p(e)) - y * eta;
    r = mu - y;
    w = mu * (1.0 - mu);
  } else if (family == 1) {
    mu = eta;
    const double t = y - eta;
    loss = t * t;
    r = 2.0 * (eta - y);
    w = 2.0;
  } else {
    mu = exp(eta);
    loss = mu - y * eta;
    r = mu - y;
    w = mu;
  }
}

template <typename T>
__global__ void __launch_bounds__(kThreads, 3) glm_pass_kernel(GlmArgs a) {
  __shared__ double s_r[TR], s_w[TR];
  __shared__ double s_fold[kThreads * 2];
  __shared__ double s_warp[kWarps][RW][3];

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int d = a.d;
  const int P = 2 * d + 3;
  const T* X = reinterpret_cast<const T*>(a.X);
  const bool accumulate = a.mode == GLM_GRAD || a.mode == GLM_NEWTON;
  const bool newton = a.mode == GLM_NEWTON;
  const double b0 = a.beta[d];
  double* part = a.part + (size_t)blockIdx.x * P;
  // phase B geometry: CB columns per pass (a multiple of 32, at most kThreads), G = kThreads / CB row groups
  const int CB = min(kThreads, (d + 31) / 32 * 32);
  const int G = kThreads / CB;
  const int bc = tid % CB, bg = tid / CB;

  if (accumulate)
    for (int j = tid; j < P; j += kThreads) part[j] = 0.0;
  double wl = 0.0, wr = 0.0, ww = 0.0;        // lane q < RW: loss, r and w sums of the warp's rows q, in tile order

  const long long ntiles = (a.n + TR - 1) / TR;
#pragma unroll 1
  for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const long long r0 = tile * TR;
    const int rows = (int)min((long long)TR, a.n - r0);
    // ---- phase A: eta of this warp's RW rows, the features split over the lanes ----
    double dot[RW];
#pragma unroll
    for (int q = 0; q < RW; ++q) dot[q] = 0.0;
    if (a.vec) {
      constexpr int V = 16 / sizeof(T);
#pragma unroll 1
      for (int j0 = lane * V; j0 < d; j0 += 32 * V) {
        uint4 raw[RW];
#pragma unroll
        for (int q = 0; q < RW; ++q) {
          const int r = warp * RW + q;
          if (r < rows) raw[q] = *reinterpret_cast<const uint4*>(X + (r0 + r) * a.ldx + j0);
        }
#pragma unroll
        for (int q = 0; q < RW; ++q) {
          if (warp * RW + q < rows) {
#pragma unroll
            for (int v = 0; v < V; ++v) dot[q] = fma(lane_elem<T>(raw[q], v), __ldg(a.beta + j0 + v), dot[q]);
          }
        }
      }
    } else {
#pragma unroll 2
      for (int j = lane; j < d; j += 32) {
        const double bj = a.beta[j];
#pragma unroll
        for (int q = 0; q < RW; ++q) {
          const int r = warp * RW + q;
          if (r < rows) dot[q] = fma(to_f64(X[(r0 + r) * a.ldx + j]), bj, dot[q]);
        }
      }
    }
#pragma unroll
    for (int q = 0; q < RW; ++q) {
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) dot[q] += __shfl_xor_sync(0xffffffffu, dot[q], off);
    }
    if (lane < RW) {
      const int q = lane;
      double dq = dot[0];
#pragma unroll
      for (int k = 1; k < RW; ++k)
        if (q == k) dq = dot[k];
      {
        const int r = warp * RW + q;
        double rr = 0.0, w = 0.0;
        if (r < rows) {
          const long long i = r0 + r;
          const double eta = dq + b0;
          const double y = accumulate ? a.y[i] : 0.0;
          double mu, loss;
          family_terms(a.family, eta, y, mu, loss, rr, w);
          if (a.mode == GLM_PREDICT) reinterpret_cast<double*>(a.out)[i] = mu;
          else if (a.mode == GLM_LABEL) reinterpret_cast<unsigned char*>(a.out)[i] = mu > 0.5 ? 1 : 0;
          if (accumulate) {
            wl += loss;
            wr += rr;
            if (newton) {
              ww += w;
              a.w[i] = w;
            }
          }
        }
        s_r[r] = rr;
        s_w[r] = w;
      }
    }
    if (!accumulate) continue;
    __syncthreads();
    // ---- phase B: sum r_i x_i (and w_i x_i) over the tile, CB columns per pass, row groups added in order ----
    const int rpg = (rows + G - 1) / G;
    const int rb = bg * rpg, re = min(rows, rb + rpg);
#pragma unroll 1
    for (int j0 = 0; j0 < d; j0 += CB) {
      const int j = j0 + bc;
      double sr = 0.0, sw = 0.0;
      if (j < d) {
#pragma unroll 4
        for (int r = rb; r < re; ++r) {
          const double x = to_f64(X[(r0 + r) * a.ldx + j]);
          sr = fma(s_r[r], x, sr);
          if (newton) sw = fma(s_w[r], x, sw);
        }
      }
      if (G > 1) {
        s_fold[tid] = sr;
        s_fold[kThreads + tid] = sw;
        __syncthreads();
        if (bg == 0) {
          for (int g = 1; g < G; ++g) {
            sr += s_fold[g * CB + bc];
            sw += s_fold[kThreads + g * CB + bc];
          }
        }
        __syncthreads();
      }
      if (bg == 0 && j < d) {
        part[j] += sr;
        if (newton) part[d + 2 + j] += sw;
      }
    }
    __syncthreads();                            // s_r / s_w are rewritten by the next tile
  }
  if (!accumulate) return;

  // ---- the scalar sums of the warps and their lanes, in order, then the ticket ----
  if (lane < RW) {
    s_warp[warp][lane][0] = wr;
    s_warp[warp][lane][1] = wl;
    s_warp[warp][lane][2] = ww;
  }
  __syncthreads();
  if (tid == 0) {
    double sr = 0.0, sl = 0.0, sw = 0.0;
    for (int k = 0; k < kWarps; ++k)
      for (int q = 0; q < RW; ++q) {
        sr += s_warp[k][q][0];
        sl += s_warp[k][q][1];
        sw += s_warp[k][q][2];
      }
    part[d] = sr;
    part[d + 1] = sl;
    part[2 * d + 2] = sw;
  }
  if (!last_block(a.ticket, gridDim.x)) return;

  // ---- the last CTA: the CTA partials in CTA order ----
  const int m = newton ? P : d + 2;
  for (int e = tid; e < m; e += kThreads) {
    double v = 0.0;
#pragma unroll 8
    for (unsigned c = 0; c < gridDim.x; ++c) v += __ldcg(a.part + (size_t)c * P + e);
    double* dst = e < d + 2 ? a.grad + e : a.hrow + (e - (d + 2));
    *dst = a.first ? v : *dst + v;
  }
  if (tid == 0) *a.ticket = 0u;
}

static int glm_grid(long long n, int sms) {
  const long long tiles = (n + TR - 1) / TR;
  long long g = 3LL * sms;                      // three CTAs per SM: all resident at once (launch bounds)
  if (g > tiles) g = tiles;
  if (g < 1) g = 1;
  return (int)g;
}

static size_t glm_ws(long long n, int d, int sms) { return partials_bytes(glm_grid(n, sms), 2 * (size_t)d + 3); }

template <typename T>
static int launch_glm(const GlmArgs& a, int grid, cudaStream_t s) {
  glm_pass_kernel<T><<<grid, kThreads, 0, s>>>(a);
  BKM_CUDA_TRY(cudaGetLastError());
  note_launch();
  return 0;
}

}  // namespace
}  // namespace bkm

using namespace bkm;

extern "C" int bkm_glm_workspace_bytes(int64_t n, int d, size_t* out) {
  if (!out || n < 0 || d <= 0) return BKM_EINVAL;
  *out = glm_ws(n, d, sm_count_or_default());
  return 0;
}

extern "C" int bkm_glm_pass_chunk(const void* X, int64_t n, int d, int64_t ldx, int x_dtype, const double* y,
                                  const double* beta, int family, int mode, double* grad, double* hrow, double* w,
                                  void* out, void* workspace, size_t ws_bytes, int flags, void* stream) {
  if (n < 0 || d <= 0 || ldx < d || !beta || family < 0 || family > 2 || mode < GLM_GRAD || mode > GLM_LABEL)
    return BKM_EINVAL;
  if (n > 0 && !X) return BKM_EINVAL;
  if (!dtype_ok(x_dtype)) return BKM_EDTYPE;
  const bool accumulate = mode == GLM_GRAD || mode == GLM_NEWTON;
  if (accumulate && (!grad || !workspace || (n > 0 && !y))) return BKM_EINVAL;
  if (mode == GLM_NEWTON && (!hrow || (n > 0 && !w))) return BKM_EINVAL;
  if (!accumulate && n > 0 && !out) return BKM_EINVAL;
  if (!accumulate && n == 0) return 0;
  int sms = 0;
  const int rc = sm_count(&sms);
  if (rc) return rc;
  const int grid = glm_grid(n, sms);
  cudaStream_t s = (cudaStream_t)stream;
  GlmArgs a;
  a.X = X; a.n = n; a.d = d; a.ldx = ldx; a.y = y; a.beta = beta; a.family = family; a.mode = mode;
  a.grad = grad; a.hrow = hrow; a.w = w; a.out = out;
  a.first = (flags & BKM_FLAG_FIRST_CHUNK) ? 1 : 0;
  const size_t es = elem_size(x_dtype);
  a.vec = n > 0 && ((uintptr_t)X % 16 == 0) && ((ldx * es) % 16 == 0) && ((d * es) % 16 == 0);
  a.part = nullptr;
  a.ticket = nullptr;
  if (accumulate) {
    const size_t need = glm_ws(n, d, sms);
    if (ws_bytes < need) return BKM_EWORKSPACE;
    BKM_CUDA_TRY(carve_partials(workspace, need, &a.part, &a.ticket, s));
  }
  if (x_dtype == BKM_F32) return launch_glm<float>(a, grid, s);
  if (x_dtype == BKM_F64) return launch_glm<double>(a, grid, s);
  return launch_glm<__nv_bfloat16>(a, grid, s);
}
