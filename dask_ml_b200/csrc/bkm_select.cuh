// bkm_select.cuh — pieces shared by the scaler passes (bkm_scale.cu), the QuantileTransformer passes
// (bkm_quantile.cu), SimpleImputer (bkm_impute.cu), the encoders (bkm_encode.cu) and the per-column key tables
// (bkm_keys.cu) and the scoring metrics (bkm_metrics.cu): the element helpers, the column-pass geometry, the
// deterministic column reduction, the missing-value test, the order-preserving keys of the exact radix selection and the
// keys of the key tables.
#pragma once
#include "bkm_common.cuh"
#include <cuda_bf16.h>

namespace bkm {
namespace {

constexpr int kThreads = 256;

__device__ __forceinline__ double widen(float v) { return (double)v; }
__device__ __forceinline__ double widen(double v) { return v; }
__device__ __forceinline__ double widen(__nv_bfloat16 v) { return (double)__bfloat162float(v); }

// column-pass geometry shared by the stats and affine kernels: CB columns per pass (a multiple of 32, at most
// kThreads), G = kThreads / CB interleaved row groups
__host__ __device__ __forceinline__ int col_block(int d) { return min(kThreads, (d + 31) / 32 * 32); }

// Grid of the element passes (bkm_affine_chunk, bkm_impute_chunk) over `cols` columns: at least 8 rows per thread, at
// most 8 CTAs per SM
static int col_pass_grid(long long n, int cols, int sms) {
  const int G = kThreads / col_block(cols);
  long long g = (n + 8LL * G - 1) / (8LL * G);
  if (g > 8LL * sms) g = 8LL * sms;
  if (g < 1) g = 1;
  return (int)g;
}

// Grid of a column_reduce pass with G row groups: at least 16 rows per thread, at most cap_per_sm CTAs per SM.  Its
// workspace is partials_bytes(grid, N * cols).
static int reduce_grid(long long n, int G, int cap_per_sm, int sms) {
  long long g = (n + 16LL * G - 1) / (16LL * G);
  if (g > (long long)cap_per_sm * sms) g = (long long)cap_per_sm * sms;
  if (g < 1) g = 1;
  return (int)g;
}

// The deterministic column reduction of the statistics passes (bkm_colstats_chunk, bkm_metric_chunk; written out in
// bkm_impute_stats_chunk): N float64 statistics of each of `cols` columns over the n rows, with the same bits from two calls
// with the same inputs and no float atomics.
//   - The threads split into G = kThreads / CB interleaved row groups of CB columns.  The CTA takes a contiguous range
//     of rows; for each column, a thread starts f[N] at Fold::identity and runs rows(f, j, first row, end, G), which
//     adds its rows in row order.
//   - The row groups are combined in order through shared memory, and each CTA writes its partial [N][cols] to `part`.
//   - The last CTA to finish (last_block) combines the partials in CTA order and hands row k < fold.live of the
//     result to fold.store(k, j, v).
// Fold::combine is the fold rule: a sum, or a min / max.
template <int N, typename Rows, typename Fold>
__device__ __forceinline__ void column_reduce(const Rows& rows, const Fold& fold, long long n, int cols, int CB,
                                              double* part, unsigned* ticket) {
  __shared__ double s_fold[N][kThreads];
  const int tid = threadIdx.x;
  const int G = kThreads / CB;
  const int bc = tid % CB, bg = tid / CB;
  const long long per = (n + gridDim.x - 1) / gridDim.x;
  const long long rb = (long long)blockIdx.x * per, re = min(n, rb + per);
  double* mine = part + (size_t)blockIdx.x * N * cols;

#pragma unroll 1
  for (int j0 = 0; j0 < cols; j0 += CB) {
    const int j = j0 + bc;
    const bool on = bg < G && j < cols;
    double f[N];
#pragma unroll
    for (int k = 0; k < N; ++k) f[k] = Fold::identity(k);
    if (on) rows(f, j, rb + bg, re, G);
    // the row groups, in order
    if (G > 1) {
#pragma unroll
      for (int k = 0; k < N; ++k) s_fold[k][tid] = f[k];
      __syncthreads();
      if (bg == 0 && on) {
        for (int g = 1; g < G; ++g) {
#pragma unroll
          for (int k = 0; k < N; ++k) f[k] = Fold::combine(k, f[k], s_fold[k][g * CB + bc]);
        }
#pragma unroll
        for (int k = 0; k < N; ++k) mine[(size_t)k * cols + j] = f[k];
      }
      __syncthreads();
    } else if (on) {
#pragma unroll
      for (int k = 0; k < N; ++k) mine[(size_t)k * cols + j] = f[k];
    }
  }

  if (!last_block(ticket, gridDim.x)) return;
  // ---- the last CTA: the CTA partials in CTA order ----
  for (int e = tid; e < fold.live * cols; e += kThreads) {
    const int k = e / cols, j = e - k * cols;
    double v = Fold::identity(k);
    for (unsigned c = 0; c < gridDim.x; ++c) v = Fold::combine(k, v, __ldcg(part + (size_t)c * N * cols + e));
    fold.store(k, j, v);
  }
  if (tid == 0) *ticket = 0u;
}

// The fold rule of statistics that are all sums: row k of the result goes to acc[k][cols], written over on the first
// chunk and added to after it.  Rows from `live` on are not written.
struct SumFold {
  double* acc;
  int cols, live, first;
  __device__ __forceinline__ static double identity(int) { return 0.0; }
  __device__ __forceinline__ static double combine(int, double v, double p) { return v + p; }
  __device__ __forceinline__ void store(int k, int j, double v) const {
    double* dst = acc + (size_t)k * cols + j;
    *dst = first ? v : *dst + v;
  }
};

static bool enc_dtype_ok(int t) {
  return t == BKM_F32 || t == BKM_F64 || t == BKM_BF16 || t == BKM_M_I32 || t == BKM_M_I64 || t == BKM_M_U8;
}

// Per (column, target) state of a radix selection, 32 bytes; the host reads `prefix` (the full key after the last
// round) and `nvalid`.
struct SelState {
  unsigned long long prefix;
  double rank;             // the target's rank among the keys that carry `prefix`
  double nvalid;           // non-NaN values of the column (set by round 0)
  int slot;                // the histogram slot this target reads
  int pad;
};

// Order-preserving unsigned keys: a < b as values (-0.0 before +0.0, NaN excluded) iff key(a) < key(b).
__device__ __forceinline__ unsigned long long radix_key(float v) {
  const unsigned u = __float_as_uint(v);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ unsigned long long radix_key(double v) {
  const unsigned long long u = (unsigned long long)__double_as_longlong(v);
  return (u & 0x8000000000000000ull) ? ~u : (u | 0x8000000000000000ull);
}
__device__ __forceinline__ unsigned long long radix_key(__nv_bfloat16 v) {
  const unsigned u = (unsigned)__bfloat16_as_ushort(v);
  return (u & 0x8000u) ? (~u & 0xffffu) : (u | 0x8000u);
}
__device__ __forceinline__ bool is_nan(float v) { return v != v; }
__device__ __forceinline__ bool is_nan(double v) { return v != v; }
__device__ __forceinline__ bool is_nan(__nv_bfloat16 v) { return __hisnan(v); }

// The missing value of SimpleImputer's passes
struct Miss {
  int is_nan;              // 1: NaN is the missing value; 0: x == value (compared after widening to float64)
  double value;
};

template <typename T>
__device__ __forceinline__ bool is_missing(T v, const Miss& m) {
  return m.is_nan ? is_nan(v) : widen(v) == m.value;
}

static bool miss_ok(int is_nan_flag, double v) { return (is_nan_flag == 0 || is_nan_flag == 1) && (is_nan_flag || v == v); }

// The keys of the per-column key tables (bkm_keys.cu) and of the encoders' sorted category lists (bkm_encode.cu):
// order-preserving, floats the radix keys with -0.0 folded to +0.0 and every NaN one key (the canonical quiet NaN's,
// the largest); int32 / int64 the value with its sign bit flipped; uint8 the value.
__device__ __forceinline__ unsigned long long enc_key(float v) {
  if (v != v) return 0xFFC00000ull;
  return v == 0.0f ? 0x80000000ull : radix_key(v);
}
__device__ __forceinline__ unsigned long long enc_key(double v) {
  if (v != v) return 0xFFF8000000000000ull;
  return v == 0.0 ? 0x8000000000000000ull : radix_key(v);
}
__device__ __forceinline__ unsigned long long enc_key(__nv_bfloat16 v) {
  if (__hisnan(v)) return 0xFFC0ull;
  return __bfloat162float(v) == 0.0f ? 0x8000ull : radix_key(v);
}
__device__ __forceinline__ unsigned long long enc_key(int v) { return (unsigned long long)((unsigned)v ^ 0x80000000u); }
__device__ __forceinline__ unsigned long long enc_key(long long v) {
  return (unsigned long long)v ^ 0x8000000000000000ull;
}
__device__ __forceinline__ unsigned long long enc_key(unsigned char v) { return (unsigned long long)v; }

// The key tables' empty slot marker (a NaN pattern for float keys; the key of INT64_MAX for int64 keys) and slot hash
constexpr unsigned long long kEmpty = ~0ull;
constexpr int kTileRows = 256;     // rows of X a CTA stages per tile

__device__ __forceinline__ unsigned long long mix64(unsigned long long k) {
  k ^= k >> 33;
  k *= 0xff51afd7ed558ccdull;
  k ^= k >> 33;
  k *= 0xc4ceb9fe1a85ec53ull;
  k ^= k >> 33;
  return k;
}

}  // namespace
}  // namespace bkm
