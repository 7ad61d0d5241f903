// bkm_select.cuh — pieces shared by the scaler passes (bkm_scale.cu) and the QuantileTransformer passes
// (bkm_quantile.cu): the element helpers, the column-pass geometry and the order-preserving keys of the exact radix
// selection.
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

// Open-addressing key tables of the mode (bkm_impute.cu) and distinct-value (bkm_encode.cu) passes: the empty slot
// marker (a NaN pattern for float keys; the key of INT64_MAX for int64 keys) and the slot hash.
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
