// bkm_impute.cu — the passes of SimpleImputer over row chunks (sm_90a).  The mode's count pass, best entry and
// multi-rank merge are the per-column key tables of bkm_keys.cu.
//
//   bkm_impute_stats_chunk   per column, in float64 and in one read of X: the missing count, the NaN and inf counts and
//                            sum (x - s) over the non-missing finite x.  The layout and fold of column_reduce
//                            (bkm_select.cuh), so two calls give the same bits.
//   bkm_impute_chunk         one read of X, one write of the output: kept columns with missing elements replaced by
//                            their statistic, then 0 / 1 indicator columns; NaN / inf counted on the way for validation.
//                            The inverse writes the missing value where an indicator is 1.
#include "bkm_select.cuh"
#include <math_constants.h>

namespace bkm {
namespace {

// ============================================ statistics ============================================
enum { IS_MISS = 0, IS_NAN, IS_INF, IS_SUM, IS_N };

struct IStatsArgs {
  const void* X;
  long long n;
  int d;
  long long ldx;
  Miss miss;
  const double* shift;     // [d], nullable
  double* acc;             // [IS_N][d]
  double* part;            // [grid][IS_N][d]
  unsigned int* ticket;
  int first;
};

// column_reduce's layout and fold (bkm_select.cuh), written out: with this row loop passed to column_reduce, ptxas
// gives the float64 kernel 70 registers instead of 54, so 3 CTAs per SM are resident instead of 4 and the kernel took
// 28 % longer on 10M x 64 float64 rows (H100 80GB HBM3, 700 W).
template <typename T>
__global__ void __launch_bounds__(kThreads) impute_stats_kernel(IStatsArgs a) {
  __shared__ double s_fold[IS_N][kThreads];
  const int tid = threadIdx.x;
  const int d = a.d;
  const int CB = col_block(d), G = kThreads / CB;
  const int bc = tid % CB, bg = tid / CB;
  const T* X = reinterpret_cast<const T*>(a.X);
  const long long per = (a.n + gridDim.x - 1) / gridDim.x;
  const long long rb = (long long)blockIdx.x * per, re = min(a.n, rb + per);
  double* part = a.part + (size_t)blockIdx.x * IS_N * d;
  constexpr int U = 8;

#pragma unroll 1
  for (int j0 = 0; j0 < d; j0 += CB) {
    const int j = j0 + bc;
    const bool on = bg < G && j < d;
    const double s = (on && a.shift) ? a.shift[j] : 0.0;
    double f[IS_N] = {0.0, 0.0, 0.0, 0.0};
    if (on) {
#pragma unroll 1
      for (long long r = rb + bg; r < re; r += (long long)G * U) {
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
            if (x != x) f[IS_NAN] += 1.0;
            else if (isinf(x)) f[IS_INF] += 1.0;
            if (is_missing(v[u], a.miss)) f[IS_MISS] += 1.0;
            else if (isfinite(x)) f[IS_SUM] += x - s;
          }
        }
      }
    }
    if (G > 1) {
#pragma unroll
      for (int k = 0; k < IS_N; ++k) s_fold[k][tid] = f[k];
      __syncthreads();
      if (bg == 0 && on) {
        for (int g = 1; g < G; ++g) {
#pragma unroll
          for (int k = 0; k < IS_N; ++k) f[k] += s_fold[k][g * CB + bc];
        }
#pragma unroll
        for (int k = 0; k < IS_N; ++k) part[(size_t)k * d + j] = f[k];
      }
      __syncthreads();
    } else if (on) {
#pragma unroll
      for (int k = 0; k < IS_N; ++k) part[(size_t)k * d + j] = f[k];
    }
  }

  if (!last_block(a.ticket, gridDim.x)) return;
  for (int e = tid; e < IS_N * d; e += kThreads) {
    double v = 0.0;
    for (unsigned c = 0; c < gridDim.x; ++c) v += __ldcg(a.part + (size_t)c * IS_N * d + e);
    a.acc[e] = a.first ? v : a.acc[e] + v;
  }
  if (tid == 0) *a.ticket = 0u;
}

// ============================================ fill ============================================
struct FillArgs {
  const void* X;
  long long n;
  int d;                   // input columns
  long long ldx;
  Miss miss;
  const double* stats;     // [d] forward: per input column, values of the output dtype
  const int* cols;         // forward: [n_keep + n_ind + n_check] source columns; inverse: [2 d_out] (-1: none)
  int n_keep, n_ind, n_check;
  int inverse;
  int d_out;
  void* out;
  long long ldo;
  double* invalid;         // [2] (+)= NaN count, inf count of the elements read; nullable
};

template <typename C, typename T> __device__ __forceinline__ C to_out(T v) { return (C)widen(v); }
template <> __device__ __forceinline__ float to_out<float, float>(float v) { return v; }
template <> __device__ __forceinline__ float to_out<float, __nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }

template <typename T, typename C>
__global__ void __launch_bounds__(kThreads) impute_fill_kernel(FillArgs p) {
  __shared__ double s_bad[2];
  const int tid = threadIdx.x;
  const int tasks = p.inverse ? p.d_out : p.n_keep + p.n_ind + p.n_check;
  const int CB = col_block(tasks), G = kThreads / CB;
  const int bc = tid % CB, bg = tid / CB;
  const T* X = reinterpret_cast<const T*>(p.X);
  C* out = reinterpret_cast<C*>(p.out);
  const long long per = (p.n + gridDim.x - 1) / gridDim.x;
  const long long rb = (long long)blockIdx.x * per, re = min(p.n, rb + per);
  if (tid < 2) s_bad[tid] = 0.0;
  __syncthreads();
  double nan_c = 0.0, inf_c = 0.0;
  const C mv = (C)p.miss.value;
  constexpr int U = 8;
#pragma unroll 1
  for (int o0 = 0; o0 < tasks; o0 += CB) {
    const int o = o0 + bc;
    if (bg >= G || o >= tasks) continue;     // the spare threads would count row group 0's rows in invalid again
    int src, kind;                 // kind 0: filled column, 1: indicator, 2: validation only, 3: inverse
    int isrc = -1;
    C fill = (C)0;
    if (p.inverse) {
      kind = 3;
      src = p.cols[o];
      isrc = p.cols[p.d_out + o];
    } else {
      src = p.cols[o];
      kind = o < p.n_keep ? 0 : (o < p.n_keep + p.n_ind ? 1 : 2);
      if (kind == 0) fill = (C)p.stats[src];
    }
#pragma unroll 1
    for (long long r = rb + bg; r < re; r += (long long)G * U) {
      T v[U], iv[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const long long rr = r + (long long)u * G;
        if (rr < re) {
          if (src >= 0) v[u] = X[rr * p.ldx + src];
          if (isrc >= 0) iv[u] = X[rr * p.ldx + isrc];
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const long long rr = r + (long long)u * G;
        if (rr >= re) continue;
        if (kind == 3) {
          C y = src >= 0 ? to_out<C>(v[u]) : (C)0;
          if (isrc >= 0 && widen(iv[u]) != 0.0) y = mv;
          out[rr * p.ldo + o] = y;
          continue;
        }
        const double x = widen(v[u]);
        if (kind != 1) {
          if (x != x) nan_c += 1.0;
          else if (isinf(x)) inf_c += 1.0;
        }
        const bool m = is_missing(v[u], p.miss);
        if (kind == 0) out[rr * p.ldo + o] = m ? fill : to_out<C>(v[u]);
        else if (kind == 1) out[rr * p.ldo + o] = m ? (C)1 : (C)0;
      }
    }
  }
  if (p.invalid && (nan_c > 0.0 || inf_c > 0.0)) {
    atomicAdd(&s_bad[0], nan_c);
    atomicAdd(&s_bad[1], inf_c);
  }
  __syncthreads();
  if (p.invalid && tid < 2 && s_bad[tid] > 0.0) atomicAdd(p.invalid + tid, s_bad[tid]);
}

template <typename T, typename C>
static int launch_fill(const FillArgs& p, int sms, cudaStream_t s) {
  const int tasks = p.inverse ? p.d_out : p.n_keep + p.n_ind + p.n_check;
  impute_fill_kernel<T, C><<<col_pass_grid(p.n, tasks, sms), kThreads, 0, s>>>(p);
  BKM_CUDA_TRY(cudaGetLastError());
  note_launch();
  return 0;
}

}  // namespace
}  // namespace bkm

using namespace bkm;

extern "C" int bkm_impute_stats_workspace_bytes(int64_t n, int d, size_t* out) {
  if (!out || n < 0 || d <= 0) return BKM_EINVAL;
  *out = partials_bytes(reduce_grid(n, kThreads / col_block(d), 4, sm_count_or_default()), IS_N * (size_t)d);
  return 0;
}

extern "C" int bkm_impute_stats_chunk(const void* X, int64_t n, int d, int64_t ldx, int x_dtype, int miss_is_nan,
                                      double miss_value, const double* shift, double* acc, void* workspace,
                                      size_t ws_bytes, int flags, void* stream) {
  if (n < 0 || d <= 0 || ldx < d || !acc || !workspace || !miss_ok(miss_is_nan, miss_value)) return BKM_EINVAL;
  if (n > 0 && !X) return BKM_EINVAL;
  if (!dtype_ok(x_dtype)) return BKM_EDTYPE;
  int sms = 0;
  const int rc = sm_count(&sms);
  if (rc) return rc;
  const int grid = reduce_grid(n, kThreads / col_block(d), 4, sms);
  const size_t need = partials_bytes(grid, IS_N * (size_t)d);
  if (ws_bytes < need) return BKM_EWORKSPACE;
  cudaStream_t s = (cudaStream_t)stream;
  IStatsArgs a;
  a.X = X; a.n = n; a.d = d; a.ldx = ldx; a.miss.is_nan = miss_is_nan; a.miss.value = miss_value; a.shift = shift;
  a.acc = acc; a.first = (flags & BKM_FLAG_FIRST_CHUNK) ? 1 : 0;
  BKM_CUDA_TRY(carve_partials(workspace, need, &a.part, &a.ticket, s));
  if (x_dtype == BKM_F32) impute_stats_kernel<float><<<grid, kThreads, 0, s>>>(a);
  else if (x_dtype == BKM_F64) impute_stats_kernel<double><<<grid, kThreads, 0, s>>>(a);
  else impute_stats_kernel<__nv_bfloat16><<<grid, kThreads, 0, s>>>(a);
  BKM_CUDA_TRY(cudaGetLastError());
  note_launch();
  return 0;
}

extern "C" int bkm_impute_chunk(const void* X, int64_t n, int d, int64_t ldx, int x_dtype, int miss_is_nan,
                                double miss_value, const double* stats, const int* cols, int n_keep, int n_ind,
                                int n_check, int inverse, void* out, int64_t ld_out, int out_dtype, double* invalid,
                                void* stream) {
  if (n < 0 || d <= 0 || ldx < d || !cols || n_keep < 0 || n_ind < 0 || n_check < 0 || (inverse != 0 && inverse != 1))
    return BKM_EINVAL;
  if (!miss_ok(miss_is_nan, miss_value)) return BKM_EINVAL;
  if (inverse && (n_keep <= 0 || n_ind != n_keep || n_check != 0)) return BKM_EINVAL;
  if (!inverse && (n_keep + n_ind + n_check <= 0 || (n_keep > 0 && !stats))) return BKM_EINVAL;
  const int d_out = inverse ? n_keep : n_keep + n_ind;
  if (ld_out < d_out || (d_out > 0 && n > 0 && !out)) return BKM_EINVAL;
  if (n > 0 && !X) return BKM_EINVAL;
  if (!dtype_ok(x_dtype) || (out_dtype != BKM_F32 && out_dtype != BKM_F64)) return BKM_EDTYPE;
  if ((x_dtype == BKM_F64) != (out_dtype == BKM_F64)) return BKM_EDTYPE;     // X's dtype (float32 for bf16 rows)
  if (n == 0) return 0;
  int sms = 0;
  const int rc = sm_count(&sms);
  if (rc) return rc;
  FillArgs p;
  p.X = X; p.n = n; p.d = d; p.ldx = ldx; p.miss.is_nan = miss_is_nan; p.miss.value = miss_value; p.stats = stats;
  p.cols = cols; p.n_keep = n_keep; p.n_ind = n_ind; p.n_check = n_check; p.inverse = inverse; p.d_out = d_out;
  p.out = out; p.ldo = ld_out; p.invalid = invalid;
  cudaStream_t s = (cudaStream_t)stream;
  if (x_dtype == BKM_F32) return launch_fill<float, float>(p, sms, s);
  if (x_dtype == BKM_F64) return launch_fill<double, double>(p, sms, s);
  return launch_fill<__nv_bfloat16, float>(p, sms, s);
}
