// bkm_scale.cu — the passes of the feature scalers (StandardScaler, MinMaxScaler, RobustScaler) over row chunks
// (sm_90a).
//
//   bkm_colstats_chunk     per column, in float64 and in one read of X: sum (x - s) and sum (x - s)^2 over the finite
//                          x, min and max over the non-NaN x, and the counts of NaN, +inf and -inf.  A column_reduce
//                          pass (bkm_select.cuh): two calls with the same inputs give the same bits.
//   bkm_radix_hist_chunk   one round of an exact radix select: every value maps to an order-preserving unsigned key
//                          (16 bits for bf16, 32 for fp32, 64 for fp64); for each (column, target) it counts the next
//                          8-bit digit of the keys that carry the target's prefix.  Targets with equal prefixes share
//                          one histogram slot (prefixes of one length are disjoint, so a key matches at most one slot).
//                          The CTA counts in shared memory and adds its non-zero bins to the float64 histogram with
//                          atomics: the counts are integers below 2^53, so the sums are exact in any order.
//   bkm_radix_select_step  one thread per column walks the bins of each target's slot, appends the digit that holds the
//                          target's rank to its prefix and keeps the rank within that digit.  Round 0 first derives the
//                          ranks from the number of non-NaN values (numpy's 'linear' virtual index, floor and floor + 1).
//   bkm_affine_chunk       out = op2(op1(x, a), b), each operation rounded once in the output's dtype (__fsub_rn,
//                          __fdiv_rn, __dmul_rn, ...): no FMA contraction, so the result equals numpy's two-step
//                          expression bit for bit.
#include "bkm_select.cuh"
#include <math_constants.h>

namespace bkm {
namespace {

constexpr int kMaxTargets = 6;

// ============================================ column statistics ============================================
enum { ST_SUM = 0, ST_SQ, ST_NAN, ST_PINF, ST_NINF, ST_MIN, ST_MAX, ST_N };

struct StatsArgs {
  const void* X;
  long long n;
  int d;
  long long ldx;
  const double* shift;     // [d], nullable
  double* acc;             // [5][d]: sums | squares | NaN | +inf | -inf
  double* minmax;          // [2][d]: min | max
  double* part;            // [grid][ST_N][d]
  unsigned int* ticket;
  int first;
};

template <typename T>
struct StatsRows {
  const StatsArgs& a;
  __device__ __forceinline__ void operator()(double (&f)[ST_N], int j, long long r0, long long re, int G) const {
    const T* X = reinterpret_cast<const T*>(a.X);
    const double s = a.shift ? a.shift[j] : 0.0;
    constexpr int U = 8;
#pragma unroll 1
    for (long long r = r0; r < re; r += (long long)G * U) {
      T v[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const long long rr = r + (long long)u * G;
        if (rr < re) v[u] = X[rr * a.ldx + j];
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (r + (long long)u * G < re) {
          const double x = widen(v[u]);
          if (x != x) {
            f[ST_NAN] += 1.0;
          } else {
            f[ST_MIN] = fmin(f[ST_MIN], x);
            f[ST_MAX] = fmax(f[ST_MAX], x);
            if (isinf(x)) {
              if (x > 0) f[ST_PINF] += 1.0; else f[ST_NINF] += 1.0;
            } else {
              const double t = x - s;
              f[ST_SUM] += t;
              f[ST_SQ] = fma(t, t, f[ST_SQ]);
            }
          }
        }
      }
    }
  }
};

// sums for the first five statistics, min and max for the last two, which go to minmax
struct StatsFold {
  const StatsArgs& a;
  static constexpr int live = ST_N;
  __device__ __forceinline__ static double identity(int k) {
    return k == ST_MIN ? CUDART_INF : (k == ST_MAX ? -CUDART_INF : 0.0);
  }
  __device__ __forceinline__ static double combine(int k, double v, double p) {
    return k == ST_MIN ? fmin(v, p) : (k == ST_MAX ? fmax(v, p) : v + p);
  }
  __device__ __forceinline__ void store(int k, int j, double v) const {
    double* dst = k < ST_MIN ? a.acc + (size_t)k * a.d + j : a.minmax + (size_t)(k - ST_MIN) * a.d + j;
    *dst = a.first ? v : combine(k, *dst, v);
  }
};

template <typename T>
__global__ void __launch_bounds__(kThreads) colstats_kernel(StatsArgs a) {
  column_reduce<ST_N>(StatsRows<T>{a}, StatsFold{a}, a.n, a.d, col_block(a.d), a.part, a.ticket);
}

// ============================================ radix select ============================================
struct HistArgs {
  const void* X;
  long long n;
  int d;
  long long ldx;
  const SelState* state;   // [d][T]
  int T;
  int slots;               // histogram slots held in shared memory: 1 in round 0 (every prefix is empty), else T
  int shift;               // bit position of this round's digit
  int round;
  double* hist;            // [d][T][256]
};

template <typename T>
__global__ void __launch_bounds__(kThreads) radix_hist_kernel(HistArgs a) {
  extern __shared__ unsigned s_hist[];                       // [CS][slots][256]
  constexpr int CS = 32 / sizeof(T);                         // columns per CTA: one 32-byte sector of a row
  constexpr int RL = kThreads / CS;                          // row lanes
  __shared__ unsigned long long s_pref[CS][kMaxTargets];
  __shared__ int s_slot[CS][kMaxTargets];
  __shared__ int s_nu[CS];
  const int tid = threadIdx.x;
  const int S = a.slots;
  const int jb = blockIdx.y * CS;
  for (int e = tid; e < CS * S * 256; e += kThreads) s_hist[e] = 0u;
  if (tid < CS) {
    const int j = jb + tid;
    int nu = 0;
    if (j < a.d) {
      for (int t = 0; t < a.T; ++t) {
        const SelState st = a.state[(size_t)j * a.T + t];
        if (a.round == 0 ? t == 0 : st.slot == t) {       // round 0 runs before the state is initialised
          s_pref[tid][nu] = a.round > 0 ? st.prefix : 0ull;
          s_slot[tid][nu] = a.round > 0 ? t : 0;
          ++nu;
        }
      }
    }
    s_nu[tid] = nu;
  }
  __syncthreads();

  const int c = tid % CS, rl = tid / CS;
  const int j = jb + c;
  const T* X = reinterpret_cast<const T*>(a.X);
  const long long per = (a.n + gridDim.x - 1) / gridDim.x;
  const long long rb = (long long)blockIdx.x * per, re = min(a.n, rb + per);
  const int nu = s_nu[c];
  const int sh = a.shift;
  constexpr int U = 16;
  if (j < a.d && nu > 0) {
#pragma unroll 1
    for (long long r = rb + rl; r < re; r += (long long)RL * U) {
      T v[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const long long rr = r + (long long)u * RL;
        if (rr < re) v[u] = X[rr * a.ldx + j];
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (r + (long long)u * RL < re && !is_nan(v[u])) {
          const unsigned long long key = radix_key(v[u]);
          const unsigned digit = (unsigned)(key >> sh) & 255u;
          const unsigned long long high = a.round == 0 ? 0ull : key >> (sh + 8);
          for (int q = 0; q < nu; ++q) {
            if (high == s_pref[c][q]) {
              atomicAdd(&s_hist[(c * S + s_slot[c][q]) * 256 + digit], 1u);
              break;
            }
          }
        }
      }
    }
  }
  __syncthreads();
  for (int e = tid; e < CS * S * 256; e += kThreads) {
    const unsigned cnt = s_hist[e];
    const int cc = e / (S * 256);
    if (cnt && jb + cc < a.d) atomicAdd(&a.hist[(size_t)(jb + cc) * a.T * 256 + (e - cc * S * 256)], (double)cnt);
  }
}

struct SelectArgs {
  double* hist;            // [d][T][256]
  SelState* state;         // [d][T]
  int d, T, round, bits;
  double qf[kMaxTargets / 2];
};

__global__ void radix_select_kernel(SelectArgs a) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= a.d) return;
  SelState* st = a.state + (size_t)j * a.T;
  const double* h = a.hist + (size_t)j * a.T * 256;
  if (a.round == 0) {
    double nv = 0.0;
    for (int b = 0; b < 256; ++b) nv += h[b];
    for (int t = 0; t < a.T; ++t) {
      // numpy's 'linear' method: virtual index (n - 1) q; floor, and floor + 1; at or above n - 1 both take the
      // last value, below 0 both the first
      const double vi = __dmul_rn(nv - 1.0, a.qf[t >> 1]);
      double idx = floor(vi) + (double)(t & 1);
      if (vi >= nv - 1.0) idx = nv - 1.0;
      if (vi < 0.0) idx = 0.0;
      st[t].rank = nv > 0.0 ? idx : 0.0;
      st[t].nvalid = nv;
      st[t].prefix = 0ull;
      st[t].slot = 0;
    }
  }
  for (int t = 0; t < a.T; ++t) {
    const double* hs = h + (size_t)st[t].slot * 256;
    double rank = st[t].rank, cum = 0.0;
    int digit = 255;
    for (int b = 0; b < 256; ++b) {
      const double c = hs[b];
      if (rank < cum + c) {
        digit = b;
        break;
      }
      cum += c;
    }
    if (st[t].nvalid > 0.0) {
      st[t].rank = rank - cum;
      st[t].prefix = (st[t].prefix << 8) | (unsigned long long)digit;
    }
  }
  for (int t = 0; t < a.T; ++t) {
    int s = t;
    for (int u = 0; u < t; ++u)
      if (st[u].prefix == st[t].prefix) {
        s = u;
        break;
      }
    st[t].slot = s;
  }
}

// ============================================ affine ============================================
enum { OP1_NONE = 0, OP1_SUB = 1, OP1_MUL = 2 };
enum { OP2_NONE = 0, OP2_DIV = 1, OP2_ADD = 2 };

struct AffineArgs {
  const void* X;
  long long n;
  int d;
  long long ldx;
  const double* a;
  const double* b;
  int op1, op2;
  void* out;
  long long ldo;
};

__device__ __forceinline__ float to_compute(float v, float) { return v; }
__device__ __forceinline__ float to_compute(__nv_bfloat16 v, float) { return __bfloat162float(v); }
__device__ __forceinline__ double to_compute(float v, double) { return (double)v; }
__device__ __forceinline__ double to_compute(double v, double) { return v; }
__device__ __forceinline__ double to_compute(__nv_bfloat16 v, double) { return (double)__bfloat162float(v); }

__device__ __forceinline__ float op_sub(float x, float y) { return __fsub_rn(x, y); }
__device__ __forceinline__ float op_mul(float x, float y) { return __fmul_rn(x, y); }
__device__ __forceinline__ float op_div(float x, float y) { return __fdiv_rn(x, y); }
__device__ __forceinline__ float op_add(float x, float y) { return __fadd_rn(x, y); }
__device__ __forceinline__ double op_sub(double x, double y) { return __dsub_rn(x, y); }
__device__ __forceinline__ double op_mul(double x, double y) { return __dmul_rn(x, y); }
__device__ __forceinline__ double op_div(double x, double y) { return __ddiv_rn(x, y); }
__device__ __forceinline__ double op_add(double x, double y) { return __dadd_rn(x, y); }

template <typename T, typename C>
__global__ void __launch_bounds__(kThreads) affine_kernel(AffineArgs p) {
  const int tid = threadIdx.x;
  const int d = p.d;
  const int CB = col_block(d), G = kThreads / CB;
  const int bc = tid % CB, bg = tid / CB;
  const T* X = reinterpret_cast<const T*>(p.X);
  C* out = reinterpret_cast<C*>(p.out);
  const long long per = (p.n + gridDim.x - 1) / gridDim.x;
  const long long rb = (long long)blockIdx.x * per, re = min(p.n, rb + per);
  constexpr int U = 8;
#pragma unroll 1
  for (int j0 = 0; j0 < d; j0 += CB) {
    const int j = j0 + bc;
    if (bg >= G || j >= d) continue;         // the 256 mod CB spare threads: their rows belong to row group 0
    const C a = p.op1 != OP1_NONE ? (C)p.a[j] : (C)0;
    const C b = p.op2 != OP2_NONE ? (C)p.b[j] : (C)0;
#pragma unroll 1
    for (long long r = rb + bg; r < re; r += (long long)G * U) {
      T v[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const long long rr = r + (long long)u * G;
        if (rr < re) v[u] = X[rr * p.ldx + j];
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const long long rr = r + (long long)u * G;
        if (rr < re) {
          C x = to_compute(v[u], C());
          if (p.op1 == OP1_SUB) x = op_sub(x, a);
          else if (p.op1 == OP1_MUL) x = op_mul(x, a);
          if (p.op2 == OP2_DIV) x = op_div(x, b);
          else if (p.op2 == OP2_ADD) x = op_add(x, b);
          out[rr * p.ldo + j] = x;
        }
      }
    }
  }
}

template <typename T, typename C>
static int launch_affine(const AffineArgs& p, int grid, cudaStream_t s) {
  affine_kernel<T, C><<<grid, kThreads, 0, s>>>(p);
  BKM_CUDA_TRY(cudaGetLastError());
  note_launch();
  return 0;
}

template <typename T>
static int launch_hist(const HistArgs& a, int sms, cudaStream_t s) {
  constexpr int CS = 32 / sizeof(T);
  const size_t smem = (size_t)CS * a.slots * 256 * 4;
  BKM_CUDA_TRY(cudaFuncSetAttribute(radix_hist_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int gy = (a.d + CS - 1) / CS;
  const int per_sm = smem <= 24 * 1024 ? 8 : (smem <= 48 * 1024 ? 4 : 2);
  long long gx = ((long long)per_sm * sms + gy - 1) / gy;
  const long long most = (a.n + (kThreads / CS) * 16 - 1) / ((kThreads / CS) * 16);   // >= 16 rows per thread
  if (gx > most) gx = most;
  if (gx < 1) gx = 1;
  radix_hist_kernel<T><<<dim3((unsigned)gx, (unsigned)gy), kThreads, smem, s>>>(a);
  BKM_CUDA_TRY(cudaGetLastError());
  note_launch();
  return 0;
}

}  // namespace
}  // namespace bkm

using namespace bkm;

extern "C" int bkm_colstats_workspace_bytes(int64_t n, int d, size_t* out) {
  if (!out || n < 0 || d <= 0) return BKM_EINVAL;
  *out = partials_bytes(reduce_grid(n, kThreads / col_block(d), 4, sm_count_or_default()), ST_N * (size_t)d);
  return 0;
}

extern "C" int bkm_colstats_chunk(const void* X, int64_t n, int d, int64_t ldx, int x_dtype, const double* shift,
                                  double* acc, double* minmax, void* workspace, size_t ws_bytes, int flags,
                                  void* stream) {
  if (n < 0 || d <= 0 || ldx < d || !acc || !minmax || !workspace) return BKM_EINVAL;
  if (n > 0 && !X) return BKM_EINVAL;
  if (!dtype_ok(x_dtype)) return BKM_EDTYPE;
  int sms = 0;
  const int rc = sm_count(&sms);
  if (rc) return rc;
  const int grid = reduce_grid(n, kThreads / col_block(d), 4, sms);
  const size_t need = partials_bytes(grid, ST_N * (size_t)d);
  if (ws_bytes < need) return BKM_EWORKSPACE;
  cudaStream_t s = (cudaStream_t)stream;
  StatsArgs a;
  a.X = X; a.n = n; a.d = d; a.ldx = ldx; a.shift = shift; a.acc = acc; a.minmax = minmax;
  a.first = (flags & BKM_FLAG_FIRST_CHUNK) ? 1 : 0;
  BKM_CUDA_TRY(carve_partials(workspace, need, &a.part, &a.ticket, s));
  if (x_dtype == BKM_F32) colstats_kernel<float><<<grid, kThreads, 0, s>>>(a);
  else if (x_dtype == BKM_F64) colstats_kernel<double><<<grid, kThreads, 0, s>>>(a);
  else colstats_kernel<__nv_bfloat16><<<grid, kThreads, 0, s>>>(a);
  BKM_CUDA_TRY(cudaGetLastError());
  note_launch();
  return 0;
}

extern "C" int bkm_radix_state_bytes(int d, int T, size_t* out) {
  if (!out || d <= 0 || T <= 0 || T > kMaxTargets) return BKM_EINVAL;
  *out = (size_t)d * T * sizeof(SelState);
  return 0;
}

extern "C" int bkm_radix_hist_chunk(const void* X, int64_t n, int d, int64_t ldx, int x_dtype, const void* state,
                                    int T, int round, double* hist, int flags, void* stream) {
  if (n < 0 || d <= 0 || ldx < d || !state || !hist || T <= 0 || T > kMaxTargets || round < 0) return BKM_EINVAL;
  if (n > 0 && !X) return BKM_EINVAL;
  if (!dtype_ok(x_dtype)) return BKM_EDTYPE;
  const int bits = (int)elem_size(x_dtype) * 8;
  if (round >= bits / 8) return BKM_EINVAL;
  cudaStream_t s = (cudaStream_t)stream;
  if (flags & BKM_FLAG_FIRST_CHUNK) BKM_CUDA_TRY(cudaMemsetAsync(hist, 0, (size_t)d * T * 256 * 8, s));
  if (n == 0) return 0;
  int sms = 0;
  const int rc = sm_count(&sms);
  if (rc) return rc;
  HistArgs a;
  a.X = X; a.n = n; a.d = d; a.ldx = ldx; a.state = reinterpret_cast<const SelState*>(state); a.T = T;
  a.slots = round == 0 ? 1 : T;
  a.shift = bits - 8 * (round + 1);
  a.round = round;
  a.hist = hist;
  if (x_dtype == BKM_F32) return launch_hist<float>(a, sms, s);
  if (x_dtype == BKM_F64) return launch_hist<double>(a, sms, s);
  return launch_hist<__nv_bfloat16>(a, sms, s);
}

extern "C" int bkm_radix_select_step(double* hist, void* state, int d, int T, int round, int x_dtype,
                                     const double* q_host, void* stream) {
  if (!hist || !state || !q_host || d <= 0 || T <= 0 || T > kMaxTargets || (T & 1) || round < 0) return BKM_EINVAL;
  if (!dtype_ok(x_dtype)) return BKM_EDTYPE;
  const int bits = (int)elem_size(x_dtype) * 8;
  if (round >= bits / 8) return BKM_EINVAL;
  SelectArgs a;
  a.hist = hist; a.state = reinterpret_cast<SelState*>(state); a.d = d; a.T = T; a.round = round; a.bits = bits;
  for (int i = 0; i < kMaxTargets / 2; ++i) a.qf[i] = i < T / 2 ? q_host[i] : 0.0;
  radix_select_kernel<<<(d + 127) / 128, 128, 0, (cudaStream_t)stream>>>(a);
  BKM_CUDA_TRY(cudaGetLastError());
  note_launch();
  return 0;
}

extern "C" int bkm_affine_chunk(const void* X, int64_t n, int d, int64_t ldx, int x_dtype, const double* a,
                                const double* b, int op1, int op2, void* out, int64_t ld_out, int out_dtype,
                                void* stream) {
  if (n < 0 || d <= 0 || ldx < d || ld_out < d || op1 < OP1_NONE || op1 > OP1_MUL || op2 < OP2_NONE || op2 > OP2_ADD)
    return BKM_EINVAL;
  if ((op1 != OP1_NONE && !a) || (op2 != OP2_NONE && !b)) return BKM_EINVAL;
  if (n > 0 && (!X || !out)) return BKM_EINVAL;
  if (!dtype_ok(x_dtype) || (out_dtype != BKM_F32 && out_dtype != BKM_F64)) return BKM_EDTYPE;
  if (x_dtype == BKM_F64 && out_dtype == BKM_F32) return BKM_EDTYPE;   // the output dtype never narrows the input
  if (n == 0) return 0;
  int sms = 0;
  const int rc = sm_count(&sms);
  if (rc) return rc;
  AffineArgs p;
  p.X = X; p.n = n; p.d = d; p.ldx = ldx; p.a = a; p.b = b; p.op1 = op1; p.op2 = op2; p.out = out; p.ldo = ld_out;
  const int grid = col_pass_grid(n, d, sms);
  cudaStream_t s = (cudaStream_t)stream;
  if (out_dtype == BKM_F32) {
    if (x_dtype == BKM_F32) return launch_affine<float, float>(p, grid, s);
    return launch_affine<__nv_bfloat16, float>(p, grid, s);
  }
  if (x_dtype == BKM_F32) return launch_affine<float, double>(p, grid, s);
  if (x_dtype == BKM_F64) return launch_affine<double, double>(p, grid, s);
  return launch_affine<__nv_bfloat16, double>(p, grid, s);
}
