// bkm_select.cuh — pieces shared by the scaler passes (bkm_scale.cu), the QuantileTransformer passes
// (bkm_quantile.cu), SimpleImputer (bkm_impute.cu), the encoders (bkm_encode.cu) and the per-column key tables
// (bkm_keys.cu): the element helpers, the column-pass geometry, the missing-value test, the order-preserving keys of
// the exact radix selection and the keys of the key tables.
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

static int sm_count(int* out) {
  int dev = 0;
  BKM_CUDA_TRY(cudaGetDevice(&dev));
  BKM_CUDA_TRY(cudaDeviceGetAttribute(out, cudaDevAttrMultiProcessorCount, dev));
  return 0;
}

static bool dtype_ok(int t) { return t == BKM_F32 || t == BKM_F64 || t == BKM_BF16; }
static bool enc_dtype_ok(int t) {
  return t == BKM_F32 || t == BKM_F64 || t == BKM_BF16 || t == BKM_M_I32 || t == BKM_M_I64 || t == BKM_M_U8;
}
static size_t elem_size(int t) { return t == BKM_F64 ? 8 : (t == BKM_F32 ? 4 : 2); }

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
