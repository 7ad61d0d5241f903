// bkm_datasets.cu — one block of make_classification / make_regression / make_counts on the device (sm_90a).
//
// The stream (include/bkm_b200.h, "datasets.make_classification / make_regression / make_counts"):
//   w = Philox4x32-10(key, counter = (row lo, row hi, j, tag)), row = the GLOBAL row index
//   tag 0  X:         j = feature pair p; Box-Muller of (w0, w1) gives x[2p] = r cospi(2 u2), x[2p + 1] = r sinpi(2 u2)
//                     with u1 = (w0 + 1) / 2^32, u2 = w1 / 2^32, r = sqrt(-2 log u1)  (the normals of make_blobs_kernel)
//   tag 1  response:  j = attempt; U = ((w0 >> 5) 2^26 + (w1 >> 6)) / 2^53, V = the same of (w2, w3)
//   tag 2  noise:     j = target; the cosine normal of (w0, w1)
//
// One launch writes X and y.  The first loop gives every thread one feature pair of a row (consecutive threads take
// consecutive pairs, so the stores are coalesced) and writes the two normals once, in X's dtype.  The second loop gives
// every thread one row: it recomputes the m informative normals from their counters instead of reading X back or
// reducing across the threads that wrote the row, rounds each to X's dtype, and sums z in list order with correctly
// rounded float64 steps (no FMA contraction), so the host restatement in datasets.py gives the same bits.  Then:
//   family 0 logistic:  y = U < 1 / (1 + exp(-z))                          int64
//   family 1 normal:    y[t] = z[t] + bias (+ noise * N)                    float64 [n][n_targets]
//   family 2 poisson:   y ~ Poisson(exp(z)) by numpy's legacy algorithm     int64
// A Poisson rate that numpy's RandomState.poisson rejects (NaN or above its lam maximum) sets *flag and writes 0.
#include "bkm_common.cuh"

namespace bkm {
namespace {

constexpr int kThreads = 256;
constexpr uint32_t kTagX = 0, kTagResponse = 1, kTagNoise = 2;
constexpr double kPoissonLamMax = 9.223372006484771e18;   // numpy's POISSON_LAM_MAX: int64 max - 10 sqrt(int64 max)

struct W4 { uint32_t w0, w1, w2, w3; };

__device__ __forceinline__ W4 philox4(uint64_t key, uint64_t row, uint32_t j, uint32_t tag) {
  uint32_t c0 = (uint32_t)row, c1 = (uint32_t)(row >> 32), c2 = j, c3 = tag;
  uint32_t k0 = (uint32_t)key, k1 = (uint32_t)(key >> 32);
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return W4{c0, c1, c2, c3};
}

__device__ __forceinline__ double u53(uint32_t a, uint32_t b) {
  return ((double)(a >> 5) * 67108864.0 + (double)(b >> 6)) * (1.0 / 9007199254740992.0);
}

// the Box-Muller pair of (w0, w1)
__device__ __forceinline__ void normal_pair(uint32_t w0, uint32_t w1, double& n0, double& n1) {
  const double u1 = ((double)w0 + 1.0) * (1.0 / 4294967296.0);          // (0, 1]
  const double u2 = (double)w1 * (1.0 / 4294967296.0);
  const double rad = sqrt(-2.0 * log(u1));
  double sn, cs;
  sincospi(2.0 * u2, &sn, &cs);
  n0 = __dmul_rn(rad, cs);
  n1 = __dmul_rn(rad, sn);
}

// numpy's random_loggam (legacy distributions)
__device__ double loggam(double x) {
  const double a[10] = {8.333333333333333e-02, -2.777777777777778e-03, 7.936507936507937e-04,
                        -5.952380952380952e-04, 8.417508417508418e-04, -1.917526917526918e-03,
                        6.410256410256410e-03, -2.955065359477124e-02, 1.796443723749843e-01,
                        -1.39243221690590e+00};
  if (x == 1.0 || x == 2.0) return 0.0;
  const long long n = x < 7.0 ? (long long)(7.0 - x) : 0;
  double x0 = __dadd_rn(x, (double)n);
  const double r = __ddiv_rn(1.0, x0);
  const double x2 = __dmul_rn(r, r);
  double gl0 = a[9];
  for (int k = 8; k >= 0; --k) gl0 = __dadd_rn(__dmul_rn(gl0, x2), a[k]);
  double gl = __dadd_rn(__dadd_rn(__dadd_rn(__ddiv_rn(gl0, x0), 0.5 * 1.8378770664093453e+00),
                                  __dmul_rn(__dsub_rn(x0, 0.5), log(x0))), -x0);
  for (long long k = 1; k <= n; ++k) {
    gl = __dsub_rn(gl, log(__dsub_rn(x0, 1.0)));
    x0 = __dsub_rn(x0, 1.0);
  }
  return gl;
}

// numpy's legacy random_poisson with the response uniforms of `row`: attempt j reads counter (row, j, tag 1)
__device__ long long poisson_draw(double lam, uint64_t key, uint64_t row) {
  if (lam == 0.0) return 0;
  uint32_t att = 0;
  if (lam < 10.0) {                                   // multiplication method
    const double enlam = exp(-lam);
    long long X = 0;
    double prod = 1.0;
    while (true) {
      const W4 w = philox4(key, row, att++, kTagResponse);
      prod = __dmul_rn(prod, u53(w.w0, w.w1));
      if (prod > enlam) X += 1;
      else return X;
    }
  }
  // PTRS (Hörmann 1993)
  const double slam = sqrt(lam), loglam = log(lam);
  const double b = __dadd_rn(0.931, __dmul_rn(2.53, slam));
  const double a = __dadd_rn(-0.059, __dmul_rn(0.02483, b));
  const double invalpha = __dadd_rn(1.1239, __ddiv_rn(1.1328, __dsub_rn(b, 3.4)));
  const double vr = __dsub_rn(0.9277, __ddiv_rn(3.6224, __dsub_rn(b, 2.0)));
  while (true) {
    const W4 w = philox4(key, row, att++, kTagResponse);
    const double U = __dsub_rn(u53(w.w0, w.w1), 0.5);
    const double V = u53(w.w2, w.w3);
    const double us = __dsub_rn(0.5, fabs(U));
    const double t = __dadd_rn(__dadd_rn(__dmul_rn(__dadd_rn(__ddiv_rn(2.0 * a, us), b), U), lam), 0.43);
    const long long k = (long long)floor(t);
    if (us >= 0.07 && V <= vr) return k;
    if (k < 0 || (us < 0.013 && V > us)) continue;
    const double lhs = __dsub_rn(__dadd_rn(log(V), log(invalpha)),
                                 log(__dadd_rn(__ddiv_rn(a, __dmul_rn(us, us)), b)));
    const double rhs = __dsub_rn(__dadd_rn(-lam, __dmul_rn((double)k, loglam)), loggam((double)k + 1.0));
    if (lhs <= rhs) return k;
  }
}

template <typename T> __device__ __forceinline__ void store_pair(T* p, double a, double b, bool both, bool vec);
template <> __device__ __forceinline__ void store_pair<float>(float* p, double a, double b, bool both, bool vec) {
  if (vec) *reinterpret_cast<float2*>(p) = make_float2((float)a, (float)b);
  else { p[0] = (float)a; if (both) p[1] = (float)b; }
}
template <> __device__ __forceinline__ void store_pair<double>(double* p, double a, double b, bool both, bool vec) {
  if (vec) *reinterpret_cast<double2*>(p) = make_double2(a, b);
  else { p[0] = a; if (both) p[1] = b; }
}

struct GenArgs {
  void* X; void* y; long long n; int d; long long ldx; long long row0;
  const double* info; int m; int nt; double bias; double noise; uint64_t key; int* flag; bool vec;
};

template <typename T, int FAMILY>
__global__ void __launch_bounds__(kThreads) make_glm_kernel(const GenArgs a) {
  T* __restrict__ X = reinterpret_cast<T*>(a.X);
  const int pairs = (a.d + 1) / 2;
  const long long total = a.n * pairs;
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long tid = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  for (long long e = tid; e < total; e += stride) {
    const long long r = e / pairs;
    const int p = (int)(e - r * pairs);
    const W4 w = philox4(a.key, (uint64_t)(a.row0 + r), (uint32_t)p, kTagX);
    double n0, n1;
    normal_pair(w.w0, w.w1, n0, n1);
    store_pair<T>(X + r * a.ldx + 2 * p, n0, n1, 2 * p + 1 < a.d, a.vec);
  }
  const int ld_info = 1 + a.nt;
  for (long long r = tid; r < a.n; r += stride) {
    const uint64_t row = (uint64_t)(a.row0 + r);
    if (FAMILY == 1) {
      double* __restrict__ y = reinterpret_cast<double*>(a.y) + r * a.nt;
      for (int t = 0; t < a.nt; ++t) {
        double z = 0.0;
        for (int q = 0; q < a.m; ++q) {
          const int f = (int)a.info[q * ld_info];
          const W4 w = philox4(a.key, row, (uint32_t)(f >> 1), kTagX);
          double n0, n1;
          normal_pair(w.w0, w.w1, n0, n1);
          const double x = (double)(T)((f & 1) ? n1 : n0);
          z = __dadd_rn(z, __dmul_rn(x, a.info[q * ld_info + 1 + t]));
        }
        z = __dadd_rn(z, a.bias);
        if (a.noise > 0.0) {
          const W4 w = philox4(a.key, row, (uint32_t)t, kTagNoise);
          double n0, n1;
          normal_pair(w.w0, w.w1, n0, n1);
          z = __dadd_rn(z, __dmul_rn(a.noise, n0));
        }
        y[t] = z;
      }
    } else {
      double z = 0.0;
      for (int q = 0; q < a.m; ++q) {
        const int f = (int)a.info[q * ld_info];
        const W4 w = philox4(a.key, row, (uint32_t)(f >> 1), kTagX);
        double n0, n1;
        normal_pair(w.w0, w.w1, n0, n1);
        const double x = (double)(T)((f & 1) ? n1 : n0);
        z = __dadd_rn(z, __dmul_rn(x, a.info[q * ld_info + 1]));
      }
      long long* __restrict__ y = reinterpret_cast<long long*>(a.y);
      if (FAMILY == 0) {
        const W4 w = philox4(a.key, row, 0u, kTagResponse);
        const double pr = __ddiv_rn(1.0, __dadd_rn(1.0, exp(-z)));
        y[r] = u53(w.w0, w.w1) < pr ? 1 : 0;
      } else {
        const double lam = exp(z);
        if (!(lam <= kPoissonLamMax)) {
          atomicOr(a.flag, 1);
          y[r] = 0;
        } else {
          y[r] = poisson_draw(lam, a.key, row);
        }
      }
    }
  }
}

template <typename T>
int launch_gen(const GenArgs& a, int family, int grid, cudaStream_t s) {
  if (family == 0) make_glm_kernel<T, 0><<<grid, kThreads, 0, s>>>(a);
  else if (family == 1) make_glm_kernel<T, 1><<<grid, kThreads, 0, s>>>(a);
  else make_glm_kernel<T, 2><<<grid, kThreads, 0, s>>>(a);
  BKM_CUDA_TRY(cudaGetLastError());
  note_launch();
  return 0;
}

}  // namespace
}  // namespace bkm

using namespace bkm;

extern "C" int bkm_make_glm_chunk(void* X, void* y, int64_t n, int d, int64_t ldx, int x_dtype, int64_t row0,
                                  int family, const double* info, int m, int n_targets, double bias, double noise,
                                  uint64_t key, int* flag, void* stream) {
  if (n < 0 || d <= 0 || ldx < d || row0 < 0 || family < 0 || family > 2 || m < 0 || n_targets <= 0) return BKM_EINVAL;
  if (family != 1 && n_targets != 1) return BKM_EINVAL;
  if (x_dtype != BKM_F32 && x_dtype != BKM_F64) return BKM_EDTYPE;
  if (n == 0) return 0;
  if (!X || !y || (m > 0 && !info) || (family == 2 && !flag)) return BKM_EINVAL;
  const int pairs = (d + 1) / 2;
  int sms = 0;
  const int rc = sm_count(&sms);
  if (rc) return rc;
  long long grid = (n * pairs + kThreads - 1) / kThreads;
  if (grid > (long long)sms * 16) grid = (long long)sms * 16;
  GenArgs a;
  a.X = X; a.y = y; a.n = n; a.d = d; a.ldx = ldx; a.row0 = row0; a.info = info; a.m = m; a.nt = n_targets;
  a.bias = bias; a.noise = noise; a.key = key; a.flag = flag;
  const size_t es = elem_size(x_dtype);
  a.vec = (d % 2 == 0) && (ldx % 2 == 0) && ((uintptr_t)X % (2 * es) == 0);
  if (x_dtype == BKM_F32) return launch_gen<float>(a, family, (int)grid, (cudaStream_t)stream);
  return launch_gen<double>(a, family, (int)grid, (cudaStream_t)stream);
}
