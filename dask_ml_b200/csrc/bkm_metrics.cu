// bkm_metrics.cu — the reduction pass of the scoring metrics over a pair of row chunks (sm_90a).
//
//   bkm_metric_chunk   one read of both operands, float64 arithmetic, at most four sums per output column:
//                        EQ       one output column: [sum w [row of a == row of b] | sum w]
//                        ERR      m output columns:  [sum (b - a)^2 | sum |b - a| | sum (a - s_j) | sum (a - s_j)^2]
//                        LOGLOSS  one output column: [sum -w log(q[a] / sum_j q_j) | sum w], q = clip(p, eps, 1 - eps)
//                      A column_reduce pass (bkm_select.cuh), same inputs, same bits: ERR with CB = min(m, 256) output
//                      columns, so that the CTA's loads are contiguous whatever m is; EQ / LOGLOSS with CB = 1, a thread
//                      owns whole rows.
//                      The operands' element types are run-time codes: the pass is bound by memory, and a uniform
//                      switch per load costs nothing next to it, where a template over both types would be 49 kernels.
#include "bkm_select.cuh"
#include <cuda_fp16.h>
#include <math_constants.h>

namespace bkm {
namespace {

constexpr int kStats = 4;

struct MetricArgs {
  const void* a;
  const void* b;
  int a_dt, b_dt;
  const double* w;         // [n], nullable
  long long n;
  int m, mode;
  const double* shift;     // [m], nullable (ERR)
  double eps;
  double* acc;             // [kStats][cols] (ERR) or [2]
  double* part;            // [grid][kStats][cols]
  unsigned int* ticket;
  int first;
};

__device__ __forceinline__ double load_f64(const void* p, int dt, long long i) {
  switch (dt) {
    case BKM_F32: return (double)reinterpret_cast<const float*>(p)[i];
    case BKM_F64: return reinterpret_cast<const double*>(p)[i];
    case BKM_BF16: return (double)__bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p)[i]);
    case BKM_M_F16: return (double)__half2float(reinterpret_cast<const __half*>(p)[i]);
    case BKM_M_I32: return (double)reinterpret_cast<const int*>(p)[i];
    case BKM_M_I64: return (double)reinterpret_cast<const long long*>(p)[i];
    default: return (double)reinterpret_cast<const unsigned char*>(p)[i];
  }
}

__device__ __forceinline__ long long load_i64(const void* p, int dt, long long i) {
  switch (dt) {
    case BKM_M_I32: return reinterpret_cast<const int*>(p)[i];
    case BKM_M_I64: return reinterpret_cast<const long long*>(p)[i];
    default: return reinterpret_cast<const unsigned char*>(p)[i];
  }
}

__host__ __device__ __forceinline__ bool is_int_code(int dt) { return dt == BKM_M_I32 || dt == BKM_M_I64 || dt == BKM_M_U8; }
static bool metric_dtype_ok(int dt) { return dt >= BKM_F32 && dt <= BKM_M_U8; }

__host__ __device__ __forceinline__ int metric_cols(int m, int mode) { return mode == BKM_METRIC_ERR ? m : 1; }

// at most 8 CTAs per SM
static int metric_grid(long long n, int m, int mode, int sms) {
  const int cols = metric_cols(m, mode);
  return reduce_grid(n, kThreads / (cols < kThreads ? cols : kThreads), 8, sms);
}

// NaN stays NaN, as in np.clip
__device__ __forceinline__ double clip(double p, double lo, double hi) { return p < lo ? lo : (p > hi ? hi : p); }

struct MetricRows {
  const MetricArgs& a;
  bool both_int;
  double hi;
  __device__ __forceinline__ void operator()(double (&f)[kStats], int j, long long r0, long long re, int G) const {
    const int m = a.m;
    if (a.mode == BKM_METRIC_ERR) {
      const double s = a.shift ? a.shift[j] : 0.0;
#pragma unroll 4
      for (long long r = r0; r < re; r += G) {
        const double x = load_f64(a.a, a.a_dt, r * m + j), y = load_f64(a.b, a.b_dt, r * m + j);
        const double dl = y - x, t = x - s;
        f[0] = fma(dl, dl, f[0]);
        f[1] += fabs(dl);
        f[2] += t;
        f[3] = fma(t, t, f[3]);
      }
    } else if (a.mode == BKM_METRIC_EQ) {
#pragma unroll 2
      for (long long r = r0; r < re; r += G) {
        bool eq = true;
        for (int q = 0; q < m; ++q) {
          const long long e = r * m + q;
          eq = eq && (both_int ? load_i64(a.a, a.a_dt, e) == load_i64(a.b, a.b_dt, e)
                               : load_f64(a.a, a.a_dt, e) == load_f64(a.b, a.b_dt, e));
        }
        const double wt = a.w ? a.w[r] : 1.0;
        f[0] += eq ? wt : wt * 0.0;          // a NaN or infinite weight reaches the sum as numpy's w * [eq] does
        f[1] += wt;
      }
    } else {
#pragma unroll 2
      for (long long r = r0; r < re; r += G) {
        const long long cls = load_i64(a.a, a.a_dt, r);
        double sum, pick;
        if (m == 1) {
          const double p1 = clip(load_f64(a.b, a.b_dt, r), a.eps, hi), p0 = 1.0 - p1;
          sum = p0 + p1;
          pick = cls == 1 ? p1 : (cls == 0 ? p0 : CUDART_NAN);
        } else {
          sum = 0.0;
          pick = CUDART_NAN;
          for (int q = 0; q < m; ++q) {
            const double p = clip(load_f64(a.b, a.b_dt, r * m + q), a.eps, hi);
            sum += p;
            if (q == cls) pick = p;
          }
        }
        const double wt = a.w ? a.w[r] : 1.0;
        f[0] -= wt * log(pick / sum);
        f[1] += wt;
      }
    }
  }
};

// ERR writes its four rows, EQ and LOGLOSS their first two
__global__ void __launch_bounds__(kThreads) metric_kernel(MetricArgs a) {
  const int cols = metric_cols(a.m, a.mode);
  const MetricRows rows{a, is_int_code(a.a_dt) && is_int_code(a.b_dt), 1.0 - a.eps};
  const SumFold fold{a.acc, cols, a.mode == BKM_METRIC_ERR ? kStats : 2, a.first};
  column_reduce<kStats>(rows, fold, a.n, cols, min(cols, kThreads), a.part, a.ticket);
}

}  // namespace
}  // namespace bkm

using namespace bkm;

extern "C" int bkm_metric_workspace_bytes(int64_t n, int m, int mode, size_t* out) {
  if (!out || n < 0 || m <= 0 || mode < BKM_METRIC_EQ || mode > BKM_METRIC_LOGLOSS) return BKM_EINVAL;
  *out = partials_bytes(metric_grid(n, m, mode, sm_count_or_default()), kStats * (size_t)metric_cols(m, mode));
  return 0;
}

extern "C" int bkm_metric_chunk(const void* a, int a_dtype, const void* b, int b_dtype, const double* w, int64_t n,
                                int m, int mode, const double* shift, double eps, double* acc, void* workspace,
                                size_t ws_bytes, int flags, void* stream) {
  if (n < 0 || m <= 0 || mode < BKM_METRIC_EQ || mode > BKM_METRIC_LOGLOSS || !acc || !workspace) return BKM_EINVAL;
  if (n > 0 && (!a || !b)) return BKM_EINVAL;
  if (!metric_dtype_ok(a_dtype) || !metric_dtype_ok(b_dtype)) return BKM_EDTYPE;
  if (mode == BKM_METRIC_LOGLOSS) {
    if (a_dtype != BKM_M_I32 || is_int_code(b_dtype)) return BKM_EDTYPE;
    if (!(eps >= 0.0 && eps < 0.5)) return BKM_EINVAL;
  }
  int sms = 0;
  const int rc = sm_count(&sms);
  if (rc) return rc;
  const int grid = metric_grid(n, m, mode, sms);
  const size_t need = partials_bytes(grid, kStats * (size_t)metric_cols(m, mode));
  if (ws_bytes < need) return BKM_EWORKSPACE;
  cudaStream_t s = (cudaStream_t)stream;
  MetricArgs g;
  g.a = a; g.b = b; g.a_dt = a_dtype; g.b_dt = b_dtype; g.w = mode == BKM_METRIC_ERR ? nullptr : w;
  g.n = n; g.m = m; g.mode = mode; g.shift = shift; g.eps = eps; g.acc = acc;
  g.first = (flags & BKM_FLAG_FIRST_CHUNK) ? 1 : 0;
  BKM_CUDA_TRY(carve_partials(workspace, need, &g.part, &g.ticket, s));
  metric_kernel<<<grid, kThreads, 0, s>>>(g);
  BKM_CUDA_TRY(cudaGetLastError());
  note_launch();
  return 0;
}
