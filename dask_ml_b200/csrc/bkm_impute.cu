// bkm_impute.cu — the passes of SimpleImputer over row chunks (sm_90a).
//
//   bkm_impute_stats_chunk   per column, in float64 and in one read of X: the missing count, the NaN and inf counts and
//                            sum (x - s) over the non-missing finite x.  Same geometry and fold as bkm_colstats_chunk:
//                            threads add their rows in row order, row groups and then CTA partials are added in a fixed
//                            order (a ticket counter elects the last CTA), so two calls give the same bits.
//   bkm_mode_count_chunk     per column, the count of every distinct non-missing value: the order-preserving radix key
//                            of bkm_select.cuh (-0.0 folded to +0.0) is counted in an open-addressing table in global
//                            memory (linear probing, atomicCAS on the key, atomicAdd on the count).  A CTA stages a tile
//                            of 256 rows x one 32-byte sector of columns in shared memory; a warp then takes 32 values
//                            of one column and lanes holding equal keys are merged with __match_any_sync, so a column of
//                            few distinct values costs one atomic per distinct key per warp.  A table's capacity is a
//                            power of two >= 2 x the values it can receive: it never fills.
//   bkm_mode_best            per column the entry of largest count, the smallest key among equal counts (a total order:
//                            the result depends neither on the table layout nor on scheduling), and the distinct count:
//                            up to 128 CTAs per column reduce slices of its table into partials, folded per column.
//   bkm_mode_compact         the occupied entries of the tables as float64 rows {column, key >> 32, key & 0xffffffff,
//                            count} (integers below 2^53: a sum all-reduce of per-rank slices is an exact all-gather).
//   bkm_mode_merge           the tables rebuilt from such rows, each inserted with its count.
//   bkm_impute_chunk         one read of X, one write of the output: kept columns with missing elements replaced by
//                            their statistic, then 0 / 1 indicator columns; NaN / inf counted on the way for validation.
//                            The inverse writes the missing value where an indicator is 1.
#include "bkm_select.cuh"
#include <math_constants.h>

namespace bkm {
namespace {

struct Miss {
  int is_nan;              // 1: NaN is the missing value; 0: x == value (compared after widening to float64)
  double value;
};

template <typename T>
__device__ __forceinline__ bool is_missing(T v, const Miss& m) {
  return m.is_nan ? is_nan(v) : widen(v) == m.value;
}

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

static int istats_grid(long long n, int d, int sms) {
  const int G = kThreads / col_block(d);
  long long g = (n + 16LL * G - 1) / (16LL * G);
  if (g > 4LL * sms) g = 4LL * sms;
  if (g < 1) g = 1;
  return (int)g;
}

static size_t istats_ws(long long n, int d, int sms) {
  return align_up((size_t)istats_grid(n, d, sms) * IS_N * (size_t)d * 8, 256) + 256;
}

template <typename T>
__global__ void __launch_bounds__(kThreads) impute_stats_kernel(IStatsArgs a) {
  __shared__ double s_fold[IS_N][kThreads];
  __shared__ int s_last;
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
    const bool on = j < d;
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

  __threadfence();
  __syncthreads();
  if (tid == 0) s_last = atomicAdd(a.ticket, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  for (int e = tid; e < IS_N * d; e += kThreads) {
    double v = 0.0;
    for (unsigned c = 0; c < gridDim.x; ++c) v += __ldcg(a.part + (size_t)c * IS_N * d + e);
    a.acc[e] = a.first ? v : a.acc[e] + v;
  }
  if (tid == 0) *a.ticket = 0u;
}

// ============================================ mode ============================================
// add `cnt` to the entry of `key` in the table keys / counts [cap] (cap a power of two, never full)
__device__ __forceinline__ void table_add(unsigned long long* keys, unsigned long long* counts, long long cap,
                                          unsigned long long key, unsigned long long cnt) {
  unsigned long long h = mix64(key) & (unsigned long long)(cap - 1);
  while (true) {
    unsigned long long cur = __ldcg(keys + h);
    if (cur == kEmpty) cur = atomicCAS(keys + h, kEmpty, key);
    if (cur == kEmpty || cur == key) {
      atomicAdd(counts + h, cnt);
      return;
    }
    h = (h + 1) & (unsigned long long)(cap - 1);
  }
}

template <typename T>
__device__ __forceinline__ unsigned long long mode_key(T v) {
  if (widen(v) == 0.0) return 1ull << (8 * sizeof(T) - 1);      // the key of +0.0, for both zeros
  return radix_key(v);
}

struct ModeArgs {
  const void* X;
  long long n;
  int g;                   // columns of the group
  long long ldx;
  Miss miss;
  unsigned long long* keys;
  unsigned long long* counts;
  const long long* off;    // [g + 1] slot offsets: column j owns [off[j], off[j + 1]), a power of two (or 0) slots
};

template <typename T>
__global__ void __launch_bounds__(kThreads) mode_count_kernel(ModeArgs a) {
  constexpr int CS = 32 / sizeof(T);                         // columns per CTA: one 32-byte sector of a row
  __shared__ T s_tile[kTileRows * CS];
  __shared__ long long s_off[CS + 1];
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const T* X = reinterpret_cast<const T*>(a.X);
  const long long tiles = (a.n + kTileRows - 1) / kTileRows;
  const long long per = (tiles + gridDim.x - 1) / gridDim.x;
  const long long tb = (long long)blockIdx.x * per, te = min(tiles, tb + per);
#pragma unroll 1
  for (int jb = blockIdx.y * CS; jb < a.g; jb += gridDim.y * CS) {
    const int nc = min(CS, a.g - jb);
    __syncthreads();
    if (tid <= CS) s_off[tid] = a.off[min(jb + tid, a.g)];
#pragma unroll 1
    for (long long t = tb; t < te; ++t) {
      const long long r0 = t * kTileRows;
      __syncthreads();
      for (int e = tid; e < kTileRows * CS; e += kThreads) {
        const int r = e / CS, c = e - r * CS;
        if (r0 + r < a.n && c < nc) s_tile[e] = X[(r0 + r) * a.ldx + jb + c];
      }
      __syncthreads();
      // tasks: (column c, 32 rows), warp-uniform
      for (int task = w; task < CS * (kTileRows / 32); task += kThreads / 32) {
        const int c = task % CS, rs = (task / CS) * 32;
        if (c >= nc) continue;
        const long long cap = s_off[c + 1] - s_off[c];
        if (cap == 0) continue;
        const long long r = r0 + rs + lane;
        const T v = s_tile[(rs + lane) * CS + c];
        const bool ok = r < a.n && !is_nan(v) && !is_missing(v, a.miss);
        const unsigned act = __ballot_sync(0xffffffffu, ok);
        if (ok) {
          const unsigned long long key = mode_key(v);
          const unsigned peers = __match_any_sync(act, key);
          if ((peers & ((1u << lane) - 1u)) == 0u)
            table_add(a.keys + s_off[c], a.counts + s_off[c], cap, key, (unsigned long long)__popc(peers));
        }
      }
    }
  }
}

struct BestPart {                  // one CTA's reduction of a slice of one column's table
  unsigned long long count, key, distinct;
};

struct BestArgs {
  const unsigned long long* keys;
  const unsigned long long* counts;
  const long long* off;
  int g;
  int parts;                       // CTAs per column
  BestPart* part;                  // [g][parts]
  unsigned long long* best_key;    // [g]
  double* best_count;              // [g] (0: no value)
  double* distinct;                // [g]
};

// (count descending, key ascending): true when (c1, k1) comes first
__device__ __forceinline__ bool better(unsigned long long c1, unsigned long long k1, unsigned long long c2,
                                      unsigned long long k2) {
  return c1 > c2 || (c1 == c2 && c1 > 0 && k1 < k2);
}

// grid (parts, <= 65535): CTA x of a column reduces slots [x cap / parts, (x + 1) cap / parts) of its table
__global__ void __launch_bounds__(kThreads) mode_best_part_kernel(BestArgs a) {
  __shared__ unsigned long long s_c[kThreads / 32], s_k[kThreads / 32], s_n[kThreads / 32];
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
#pragma unroll 1
  for (int j = blockIdx.y; j < a.g; j += gridDim.y) {
    const long long o = a.off[j], cap = a.off[j + 1] - o;
    const long long s0 = cap * blockIdx.x / a.parts, s1 = cap * (blockIdx.x + 1) / a.parts;
    unsigned long long bc = 0, bk = kEmpty, nd = 0;
    for (long long s = s0 + tid; s < s1; s += kThreads) {
      const unsigned long long k = a.keys[o + s];
      if (k == kEmpty) continue;
      const unsigned long long c = a.counts[o + s];
      ++nd;
      if (better(c, k, bc, bk)) { bc = c; bk = k; }
    }
#pragma unroll
    for (int sh = 16; sh > 0; sh >>= 1) {
      const unsigned long long c = __shfl_xor_sync(0xffffffffu, bc, sh), k = __shfl_xor_sync(0xffffffffu, bk, sh);
      nd += __shfl_xor_sync(0xffffffffu, nd, sh);
      if (better(c, k, bc, bk)) { bc = c; bk = k; }
    }
    __syncthreads();
    if (lane == 0) { s_c[w] = bc; s_k[w] = bk; s_n[w] = nd; }
    __syncthreads();
    if (tid == 0) {
      for (int i = 1; i < kThreads / 32; ++i) {
        nd += s_n[i];
        if (better(s_c[i], s_k[i], bc, bk)) { bc = s_c[i]; bk = s_k[i]; }
      }
      BestPart p;
      p.count = bc; p.key = bk; p.distinct = nd;
      a.part[(size_t)j * a.parts + blockIdx.x] = p;
    }
  }
}

// one thread per column folds its partials in CTA order (the order is total, the counts integers: any order gives the
// same result)
__global__ void __launch_bounds__(kThreads) mode_best_fold_kernel(BestArgs a) {
  const int j = blockIdx.x * kThreads + threadIdx.x;
  if (j >= a.g) return;
  unsigned long long bc = 0, bk = kEmpty, nd = 0;
  for (int x = 0; x < a.parts; ++x) {
    const BestPart p = a.part[(size_t)j * a.parts + x];
    nd += p.distinct;
    if (better(p.count, p.key, bc, bk)) { bc = p.count; bk = p.key; }
  }
  a.best_key[j] = bk;
  a.best_count[j] = (double)bc;
  a.distinct[j] = (double)nd;
}

// CTAs per column of the best-entry reduction: about 16 slots per thread, at most 128 (the widest table, 2^26 slots,
// then takes 128 CTAs)
static int best_parts(int g, long long total_slots) {
  long long per_col = g > 0 ? total_slots / g : 0;
  long long p = per_col / (16LL * kThreads);
  if (p > 128) p = 128;
  if (p < 1) p = 1;
  return (int)p;
}

struct CompactArgs {
  const unsigned long long* keys;
  const unsigned long long* counts;
  const long long* off;
  double* entries;                 // [*][4]
  unsigned long long* cursor;
  int g;
};

__global__ void __launch_bounds__(kThreads) mode_compact_kernel(CompactArgs a) {
#pragma unroll 1
  for (int j = blockIdx.y; j < a.g; j += gridDim.y) {
    const long long o = a.off[j], cap = a.off[j + 1] - o;
    for (long long s = (long long)blockIdx.x * kThreads + threadIdx.x; s < cap; s += (long long)gridDim.x * kThreads) {
      const unsigned long long k = a.keys[o + s];
      if (k == kEmpty) continue;
      const unsigned long long p = atomicAdd(a.cursor, 1ull);
      double* e = a.entries + p * 4;
      e[0] = (double)j;
      e[1] = (double)(k >> 32);
      e[2] = (double)(k & 0xffffffffull);
      e[3] = (double)a.counts[o + s];
    }
  }
}

struct MergeArgs {
  const double* entries;
  long long n_entries;
  unsigned long long* keys;
  unsigned long long* counts;
  const long long* off;
  int g;
};

__global__ void __launch_bounds__(kThreads) mode_merge_kernel(MergeArgs a) {
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < a.n_entries;
       i += (long long)gridDim.x * kThreads) {
    const double* e = a.entries + i * 4;
    const double cnt = e[3];
    const int j = (int)e[0];
    if (!(cnt > 0.0) || j < 0 || j >= a.g) continue;          // zero rows: the padding of the gathered slices
    const long long o = a.off[j], cap = a.off[j + 1] - o;
    if (cap == 0) continue;
    const unsigned long long k = ((unsigned long long)e[1] << 32) | (unsigned long long)e[2];
    table_add(a.keys + o, a.counts + o, cap, k, (unsigned long long)cnt);
  }
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
    if (o >= tasks) continue;
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

template <typename T>
static int launch_mode_count(const ModeArgs& a, int sms, cudaStream_t s) {
  constexpr int CS = 32 / sizeof(T);
  const int gy = (a.g + CS - 1) / CS < 65535 ? (a.g + CS - 1) / CS : 65535;
  const long long tiles = (a.n + kTileRows - 1) / kTileRows;
  long long gx = ((long long)8 * sms + gy - 1) / gy;
  if (gx > tiles) gx = tiles;
  if (gx < 1) gx = 1;
  mode_count_kernel<T><<<dim3((unsigned)gx, (unsigned)gy), kThreads, 0, s>>>(a);
  BKM_CUDA_TRY(cudaGetLastError());
  note_launch();
  return 0;
}

template <typename T, typename C>
static int launch_fill(const FillArgs& p, int sms, cudaStream_t s) {
  const int tasks = p.inverse ? p.d_out : p.n_keep + p.n_ind + p.n_check;
  const int G = kThreads / col_block(tasks);
  long long g = (p.n + 8LL * G - 1) / (8LL * G);
  if (g > 8LL * sms) g = 8LL * sms;
  if (g < 1) g = 1;
  impute_fill_kernel<T, C><<<(unsigned)g, kThreads, 0, s>>>(p);
  BKM_CUDA_TRY(cudaGetLastError());
  note_launch();
  return 0;
}

static bool miss_ok(int is_nan_flag, double v) { return (is_nan_flag == 0 || is_nan_flag == 1) && (is_nan_flag || v == v); }

}  // namespace
}  // namespace bkm

using namespace bkm;

extern "C" int bkm_impute_stats_workspace_bytes(int64_t n, int d, size_t* out) {
  if (!out || n < 0 || d <= 0) return BKM_EINVAL;
  int sms = 0;
  if (sm_count(&sms) != 0 || sms <= 0) sms = kDefaultSMs;
  *out = istats_ws(n, d, sms);
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
  if (ws_bytes < istats_ws(n, d, sms)) return BKM_EWORKSPACE;
  cudaStream_t s = (cudaStream_t)stream;
  IStatsArgs a;
  a.X = X; a.n = n; a.d = d; a.ldx = ldx; a.miss.is_nan = miss_is_nan; a.miss.value = miss_value; a.shift = shift;
  a.acc = acc; a.first = (flags & BKM_FLAG_FIRST_CHUNK) ? 1 : 0;
  unsigned char* ws = reinterpret_cast<unsigned char*>(workspace);
  a.part = reinterpret_cast<double*>(ws);
  a.ticket = reinterpret_cast<unsigned int*>(ws + istats_ws(n, d, sms) - 256);
  BKM_CUDA_TRY(cudaMemsetAsync(a.ticket, 0, 4, s));
  const int grid = istats_grid(n, d, sms);
  if (x_dtype == BKM_F32) impute_stats_kernel<float><<<grid, kThreads, 0, s>>>(a);
  else if (x_dtype == BKM_F64) impute_stats_kernel<double><<<grid, kThreads, 0, s>>>(a);
  else impute_stats_kernel<__nv_bfloat16><<<grid, kThreads, 0, s>>>(a);
  BKM_CUDA_TRY(cudaGetLastError());
  note_launch();
  return 0;
}

extern "C" int bkm_mode_count_chunk(const void* X, int64_t n, int g, int64_t ldx, int x_dtype, int miss_is_nan,
                                    double miss_value, unsigned long long* keys, unsigned long long* counts,
                                    const int64_t* slot_off, int64_t total_slots, int flags, void* stream) {
  if (n < 0 || g <= 0 || ldx < g || total_slots < 0 || !slot_off || !miss_ok(miss_is_nan, miss_value)) return BKM_EINVAL;
  if (total_slots > 0 && (!keys || !counts)) return BKM_EINVAL;
  if (n > 0 && !X) return BKM_EINVAL;
  if (!dtype_ok(x_dtype)) return BKM_EDTYPE;
  cudaStream_t s = (cudaStream_t)stream;
  if ((flags & BKM_FLAG_FIRST_CHUNK) && total_slots > 0) {
    BKM_CUDA_TRY(cudaMemsetAsync(keys, 0xff, (size_t)total_slots * 8, s));
    BKM_CUDA_TRY(cudaMemsetAsync(counts, 0, (size_t)total_slots * 8, s));
  }
  if (n == 0 || total_slots == 0) return 0;
  int sms = 0;
  const int rc = sm_count(&sms);
  if (rc) return rc;
  ModeArgs a;
  a.X = X; a.n = n; a.g = g; a.ldx = ldx; a.miss.is_nan = miss_is_nan; a.miss.value = miss_value; a.keys = keys;
  a.counts = counts; a.off = reinterpret_cast<const long long*>(slot_off);
  if (x_dtype == BKM_F32) return launch_mode_count<float>(a, sms, s);
  if (x_dtype == BKM_F64) return launch_mode_count<double>(a, sms, s);
  return launch_mode_count<__nv_bfloat16>(a, sms, s);
}

extern "C" int bkm_mode_best_workspace_bytes(int g, int64_t total_slots, size_t* out) {
  if (!out || g <= 0 || total_slots < 0) return BKM_EINVAL;
  *out = (size_t)g * best_parts(g, total_slots) * sizeof(BestPart);
  return 0;
}

extern "C" int bkm_mode_best(const unsigned long long* keys, const unsigned long long* counts, const int64_t* slot_off,
                             int g, int64_t total_slots, unsigned long long* best_key, double* best_count,
                             double* distinct, void* workspace, size_t ws_bytes, void* stream) {
  if (g <= 0 || total_slots < 0 || !slot_off || !best_key || !best_count || !distinct || !workspace) return BKM_EINVAL;
  if (total_slots > 0 && (!keys || !counts)) return BKM_EINVAL;
  const int parts = best_parts(g, total_slots);
  if (ws_bytes < (size_t)g * parts * sizeof(BestPart)) return BKM_EWORKSPACE;
  BestArgs a;
  a.keys = keys; a.counts = counts; a.off = reinterpret_cast<const long long*>(slot_off); a.g = g; a.parts = parts;
  a.part = reinterpret_cast<BestPart*>(workspace); a.best_key = best_key; a.best_count = best_count;
  a.distinct = distinct;
  cudaStream_t s = (cudaStream_t)stream;
  mode_best_part_kernel<<<dim3((unsigned)parts, (unsigned)(g < 65535 ? g : 65535)), kThreads, 0, s>>>(a);
  BKM_CUDA_TRY(cudaGetLastError());
  mode_best_fold_kernel<<<(unsigned)((g + kThreads - 1) / kThreads), kThreads, 0, s>>>(a);
  BKM_CUDA_TRY(cudaGetLastError());
  note_launch(2);
  return 0;
}

extern "C" int bkm_mode_compact(const unsigned long long* keys, const unsigned long long* counts,
                                const int64_t* slot_off, int g, double* entries, unsigned long long* cursor,
                                void* stream) {
  if (g <= 0 || !slot_off || !entries || !cursor) return BKM_EINVAL;
  cudaStream_t s = (cudaStream_t)stream;
  BKM_CUDA_TRY(cudaMemsetAsync(cursor, 0, 8, s));
  int sms = 0;
  const int rc = sm_count(&sms);
  if (rc) return rc;
  CompactArgs a;
  a.keys = keys; a.counts = counts; a.off = reinterpret_cast<const long long*>(slot_off); a.entries = entries;
  a.cursor = cursor; a.g = g;
  unsigned gx = (unsigned)((4 * sms + g - 1) / g);
  mode_compact_kernel<<<dim3(gx < 1 ? 1 : gx, (unsigned)(g < 65535 ? g : 65535)), kThreads, 0, s>>>(a);
  BKM_CUDA_TRY(cudaGetLastError());
  note_launch();
  return 0;
}

extern "C" int bkm_mode_merge(const double* entries, int64_t n_entries, unsigned long long* keys,
                              unsigned long long* counts, const int64_t* slot_off, int g, int64_t total_slots,
                              void* stream) {
  if (g <= 0 || !slot_off || n_entries < 0 || total_slots < 0) return BKM_EINVAL;
  if ((n_entries > 0 && !entries) || (total_slots > 0 && (!keys || !counts))) return BKM_EINVAL;
  cudaStream_t s = (cudaStream_t)stream;
  if (total_slots > 0) {
    BKM_CUDA_TRY(cudaMemsetAsync(keys, 0xff, (size_t)total_slots * 8, s));
    BKM_CUDA_TRY(cudaMemsetAsync(counts, 0, (size_t)total_slots * 8, s));
  }
  if (n_entries == 0 || total_slots == 0) return 0;
  int sms = 0;
  const int rc = sm_count(&sms);
  if (rc) return rc;
  MergeArgs a;
  a.entries = entries; a.n_entries = n_entries; a.keys = keys; a.counts = counts;
  a.off = reinterpret_cast<const long long*>(slot_off); a.g = g;
  long long gx = (n_entries + kThreads - 1) / kThreads;
  if (gx > 8LL * sms) gx = 8LL * sms;
  mode_merge_kernel<<<(unsigned)gx, kThreads, 0, s>>>(a);
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
