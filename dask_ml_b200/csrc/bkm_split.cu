// bkm_split.cu — the two passes of train_test_split / ShuffleSplit over one row block (sm_90a).
//
//   bkm_split_indices_chunk  idx_out[i] = offset + pi_seed(start + i): the block's keyed permutation (bkm_b200.h,
//                            "the split permutation") evaluated per position.  Each thread derives the round keys once,
//                            keeps them in registers and walks its positions; nothing is read from memory.
//   bkm_gather_rows_chunk    out row i = src row idx[i] - idx_offset, rows as bytes.  The copy unit V is the widest of
//                            16, 8, 4, 2, 1 bytes that divides both base addresses, both row pitches and the row size.
//                            A row of nv = row_bytes / V units is copied by a lane group of lpr = min(32, 2^ceil(log2 nv))
//                            lanes, so a warp carries 32 / lpr rows at once (32 rows of a 1-D int64 y), and every lane
//                            group keeps kRowsInFlight rows in flight: the index loads, then the row loads, then the
//                            stores.
#include "bkm_common.cuh"
#include <assert.h>

namespace bkm {
namespace {

constexpr int kThreads = 256;
constexpr int kRounds = BKM_SPLIT_ROUNDS;

// ============================================ the permutation ============================================
struct SplitKeys { uint32_t k0[kRounds], k1[kRounds]; };

__device__ __forceinline__ SplitKeys split_keys(unsigned long long seed) {
  SplitKeys K;
#pragma unroll
  for (int r = 0; r < kRounds; ++r) {
    unsigned long long z = seed + (unsigned long long)(r + 1) * BKM_SPLIT_KEY_STEP;
    z = (z ^ (z >> 30)) * BKM_SPLIT_KEY_MUL1;
    z = (z ^ (z >> 27)) * BKM_SPLIT_KEY_MUL2;
    z ^= z >> 31;
    K.k0[r] = (uint32_t)z;
    K.k1[r] = (uint32_t)(z >> 32);
  }
  return K;
}

__device__ __forceinline__ unsigned long long split_permute(const SplitKeys& K, int w, unsigned long long c,
                                                            unsigned long long v) {
  const uint32_t mask = (uint32_t)((1ull << w) - 1ull);
  do {
    uint32_t L = (uint32_t)(v >> w), R = (uint32_t)v & mask;
#pragma unroll
    for (int r = 0; r < kRounds; ++r) {
      const uint32_t x = R ^ K.k0[r];
      uint32_t f = __umulhi(x, BKM_SPLIT_ROUND_MUL) ^ (x * BKM_SPLIT_ROUND_MUL) ^ K.k1[r];
      f = (f ^ (f >> 16)) * BKM_SPLIT_ROUND_MIX;
      f ^= f >> 15;
      const uint32_t t = L ^ (f >> (32 - w));
      L = R;
      R = t;
    }
    v = ((unsigned long long)L << w) | R;
  } while (v >= c);          // cycle walking: the cycle through a value below c comes back below c
  return v;
}

__global__ void __launch_bounds__(kThreads) split_indices_kernel(unsigned long long seed, unsigned long long c, int w,
                                                                  long long start, long long count, long long offset,
                                                                  long long* __restrict__ out) {
  const SplitKeys K = split_keys(seed);
  const long long stride = (long long)gridDim.x * kThreads;
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < count; i += stride)
    out[i] = offset + (long long)split_permute(K, w, c, (unsigned long long)(start + i));
}

// ============================================ the row gather ============================================
constexpr int kRowsInFlight = 4;

struct GatherArgs {
  const unsigned char* src;
  long long n_src;
  long long ld_src, ld_out;      // row pitches in units of V bytes
  int nv;                        // units per row
  int lpr;                       // lanes per row: a power of two <= 32
  const long long* idx;
  long long idx_offset, count;
  unsigned char* out;
};

template <typename VT>
__global__ void __launch_bounds__(kThreads) gather_rows_kernel(GatherArgs a) {
  const VT* __restrict__ src = reinterpret_cast<const VT*>(a.src);
  VT* __restrict__ out = reinterpret_cast<VT*>(a.out);
  const int lane = threadIdx.x & 31;
  const int sub = lane & (a.lpr - 1), grp = lane / a.lpr, rpw = 32 / a.lpr;
  const long long warp = ((long long)blockIdx.x * kThreads + threadIdx.x) >> 5;
  const long long step = ((long long)gridDim.x * kThreads >> 5) * rpw * kRowsInFlight;
  for (long long base = warp * rpw * kRowsInFlight; base < a.count; base += step) {
    long long row[kRowsInFlight];
#pragma unroll
    for (int u = 0; u < kRowsInFlight; ++u) {
      const long long i = base + (long long)u * rpw + grp;
      row[u] = i < a.count ? __ldg(a.idx + i) - a.idx_offset : -1;
#ifdef BKM_DEBUG
      assert(i >= a.count || (row[u] >= 0 && row[u] < a.n_src));
#endif
    }
    if (a.nv <= a.lpr) {
      VT v[kRowsInFlight];
#pragma unroll
      for (int u = 0; u < kRowsInFlight; ++u)
        if (row[u] >= 0 && sub < a.nv) v[u] = __ldg(src + row[u] * a.ld_src + sub);
#pragma unroll
      for (int u = 0; u < kRowsInFlight; ++u)
        if (row[u] >= 0 && sub < a.nv) out[(base + (long long)u * rpw + grp) * a.ld_out + sub] = v[u];
    } else {
#pragma unroll
      for (int u = 0; u < kRowsInFlight; ++u) {
        if (row[u] < 0) continue;
        const VT* s = src + row[u] * a.ld_src;
        VT* o = out + (base + (long long)u * rpw + grp) * a.ld_out;
        for (int q = sub; q < a.nv; q += a.lpr) o[q] = __ldg(s + q);
      }
    }
  }
}

static int grid_for(long long work_items, int per_thread) {
  const int sms = sm_count_or_default();
  long long g = (work_items + (long long)kThreads * per_thread - 1) / ((long long)kThreads * per_thread);
  if (g > 16LL * sms) g = 16LL * sms;
  return (int)(g < 1 ? 1 : g);
}

}  // namespace
}  // namespace bkm

using namespace bkm;

extern "C" int bkm_split_indices_chunk(uint64_t seed, int64_t c, int64_t start, int64_t count, int64_t offset,
                                       int64_t* idx_out, void* stream) {
  if (c < 1 || c > (1LL << 31) || start < 0 || count < 0 || start + count > c) return BKM_EINVAL;
  if (count == 0) return 0;
  if (!idx_out) return BKM_EINVAL;
  int bits = 0;
  while ((1LL << bits) < c) ++bits;
  const int w = bits < 2 ? 1 : (bits + 1) / 2;
  split_indices_kernel<<<grid_for(count, 4), kThreads, 0, (cudaStream_t)stream>>>(
      seed, (unsigned long long)c, w, start, count, offset, reinterpret_cast<long long*>(idx_out));
  BKM_CUDA_TRY(cudaGetLastError());
  note_launch();
  return 0;
}

extern "C" int bkm_gather_rows_chunk(const void* src, int64_t n_src, int64_t row_bytes, int64_t ld_src_bytes,
                                     const int64_t* idx, int64_t idx_offset, int64_t count, void* out,
                                     int64_t ld_out_bytes, void* stream) {
  if (n_src < 0 || count < 0 || row_bytes <= 0 || ld_src_bytes < row_bytes || ld_out_bytes < row_bytes)
    return BKM_EINVAL;
  if (count == 0) return 0;
  if (!src || !idx || !out || n_src == 0) return BKM_EINVAL;
  const uintptr_t bits = (uintptr_t)src | (uintptr_t)out | (uintptr_t)row_bytes | (uintptr_t)ld_src_bytes |
                         (uintptr_t)ld_out_bytes;
  int V = 16;
  while (bits & (uintptr_t)(V - 1)) V >>= 1;
  if (row_bytes / V > (1LL << 30)) return BKM_EUNSUPPORTED;
  GatherArgs a;
  a.src = reinterpret_cast<const unsigned char*>(src);
  a.n_src = n_src;
  a.ld_src = ld_src_bytes / V;
  a.ld_out = ld_out_bytes / V;
  a.nv = (int)(row_bytes / V);
  a.lpr = 1;
  while (a.lpr < 32 && a.lpr < a.nv) a.lpr <<= 1;
  a.idx = reinterpret_cast<const long long*>(idx);
  a.idx_offset = idx_offset;
  a.count = count;
  a.out = reinterpret_cast<unsigned char*>(out);
  const int grid = grid_for(count * a.lpr, kRowsInFlight);
  cudaStream_t s = (cudaStream_t)stream;
  switch (V) {
    case 16: gather_rows_kernel<uint4><<<grid, kThreads, 0, s>>>(a); break;
    case 8: gather_rows_kernel<uint2><<<grid, kThreads, 0, s>>>(a); break;
    case 4: gather_rows_kernel<uint32_t><<<grid, kThreads, 0, s>>>(a); break;
    case 2: gather_rows_kernel<uint16_t><<<grid, kThreads, 0, s>>>(a); break;
    default: gather_rows_kernel<uint8_t><<<grid, kThreads, 0, s>>>(a); break;
  }
  BKM_CUDA_TRY(cudaGetLastError());
  note_launch();
  return 0;
}
