// bkm_keys.cu — the per-column key tables of SimpleImputer's mode and of the encoders' categories (sm_90a).
//
// A group of g columns owns keys / counts [total_slots] uint64; column j owns slots [off[j], off[j + 1]), a power of
// two (or 0).  An empty slot holds kEmpty.  A key (enc_key of bkm_select.cuh) is placed by mix64 and linear probing,
// an empty slot claimed with atomicCAS.  A table's content is a set of keys with integer counts: every result read
// from it (the best entry, the compacted entries up to their order, the distinct counts) is independent of the slot
// layout and of scheduling.
//
//   bkm_mode_count_chunk     per column, the count of every distinct non-missing value.  A table's capacity is a
//                            power of two >= 2 x the values it can receive: it never fills.
//   bkm_distinct_chunk       per column, every distinct key (count 1).  Tables start small: a column whose occupancy
//                            passes half its capacity, or whose probe chain passes kMaxProbe, is flagged and the host
//                            grows it and runs the group again.  With BKM_FLAG_FULL_PROBE the bound is the capacity: a
//                            table sized so that it can never pass half full then never overflows: a chain longer than
//                            kMaxProbe is walked, not grown away.  Before it probes global memory, the leader looks the
//                            key up in a per-CTA, per-column direct-mapped cache of keys already in the table (shared
//                            memory): a column of few distinct values costs about one global lookup per value per CTA.
//                            INT64_MAX, whose key is kEmpty, is carried as a per-column flag.
//     Both are one sector scan: a CTA stages a tile of 256 rows x one 32-byte sector of columns in shared memory; a
//     warp then takes 32 values of one column and lanes holding equal keys are merged with __match_any_sync, so a
//     column of few distinct values costs one probe per distinct key per warp.
//   bkm_mode_best            per column the entry of largest count, the smallest key among equal counts (a total order),
//                            and the distinct count: up to 128 CTAs per column reduce slices of its table into
//                            partials, folded per column.
//   bkm_mode_compact         the occupied entries of the tables as float64 rows {column, key >> 32, key & 0xffffffff,
//                            count} (integers below 2^53: a sum all-reduce of per-rank slices is an exact all-gather).
//   bkm_mode_merge           the tables rebuilt from such rows, each inserted with its count.
#include "bkm_select.cuh"

namespace bkm {
namespace {

constexpr int kMaxProbe = 1024;          // probe chain bound of the distinct tables
constexpr int kFilterSlots = 4096;       // per CTA, shared between the columns of a sector

enum { ST_OVERFLOW = 1, ST_MARKER = 2 };

// The slot of `key` in the table keys [cap] (cap a power of two), found or claimed within `bound` probes, or -1.
// CLAIM: *claimed is set when this call stored the key, and a found key and a claimed slot leave the loop by separate
// returns.  Without CLAIM both leave by one return.  Each shape is the faster one for its callers: on an H100 80GB HBM3
// at a 700 W power limit the shared exit made the distinct pass on 10^4-key fp32 columns 1.5x slower, and separate
// exits made the count pass on 16-value bf16 columns 8 % slower.
template <bool CLAIM>
__device__ __forceinline__ long long probe(unsigned long long* keys, long long cap, long long bound,
                                           unsigned long long key, bool* claimed) {
  const unsigned long long mask = (unsigned long long)(cap - 1);
  unsigned long long h = mix64(key) & mask;
  for (long long p = 0; p < bound; ++p) {
    unsigned long long cur = __ldcg(keys + h);
    if (cur == kEmpty) {
      cur = atomicCAS(keys + h, kEmpty, key);
      if (CLAIM && cur == kEmpty) {
        *claimed = true;
        return (long long)h;
      }
    }
    if (cur == key || (!CLAIM && cur == kEmpty)) {
      if (CLAIM) *claimed = false;
      return (long long)h;
    }
    h = (h + 1) & mask;
  }
  return -1;
}

// ============================================ sector scan ============================================
struct ScanArgs {
  const void* X;
  long long n;
  int g;                           // columns of the group
  long long ldx;
  Miss miss;                       // COUNT
  unsigned long long* keys;
  unsigned long long* counts;
  const long long* off;            // [g + 1]
  unsigned long long* occupied;    // !COUNT: [g]
  unsigned long long* status;      // !COUNT: [g]
  int full_probe;                  // !COUNT: probe bound the capacity instead of min(capacity, kMaxProbe)
};

// COUNT: add each non-missing, non-NaN value's multiplicity to its key's count.  !COUNT: record each key (count 1),
// with the occupancy, the overflow flag and the INT64_MAX marker.
template <typename T, bool COUNT>
__global__ void __launch_bounds__(kThreads) key_scan_kernel(ScanArgs a) {
  constexpr int CS = 32 / sizeof(T);                         // columns per CTA: one 32-byte sector of a row
  constexpr int FS = kFilterSlots / CS;                      // !COUNT: cache slots per column
  __shared__ T s_tile[kTileRows * CS];
  __shared__ long long s_off[CS + 1];
  unsigned long long* s_cache = nullptr;
  if constexpr (!COUNT) {
    __shared__ unsigned long long s_filter[kFilterSlots];
    s_cache = s_filter;
  }
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
    if constexpr (!COUNT)
      for (int e = tid; e < kFilterSlots; e += kThreads) s_cache[e] = kEmpty;
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
        const int j = jb + c;
        const long long o = s_off[c], cap = s_off[c + 1] - o;
        unsigned long long st = 0ull;
        if constexpr (!COUNT) {
          st = lane == 0 ? __ldcg(a.status + j) : 0ull;
          st = __shfl_sync(0xffffffffu, st, 0);
        }
        if (cap == 0 || (st & ST_OVERFLOW)) continue;                     // !COUNT: an overflowed group runs again
        const T v = s_tile[(rs + lane) * CS + c];
        bool ok = r0 + rs + lane < a.n;
        if constexpr (COUNT) ok = ok && !is_nan(v) && !is_missing(v, a.miss);
        const unsigned act = __ballot_sync(0xffffffffu, ok);
        if (!ok) continue;
        const unsigned long long key = enc_key(v);
        const unsigned peers = __match_any_sync(act, key);
        if ((peers & ((1u << lane) - 1u)) != 0u) continue;               // one leader per key
        if constexpr (COUNT) {
          const long long h = probe<false>(a.keys + o, cap, cap, key, nullptr);
          if (h >= 0) atomicAdd(a.counts + o + h, (unsigned long long)__popc(peers));   // -1: a full, undersized table
        } else {
          if (key == kEmpty) {                               // INT64_MAX: the table's empty marker, kept as a flag
            if (!(__ldcg(a.status + j) & ST_MARKER)) atomicOr(a.status + j, (unsigned long long)ST_MARKER);
            continue;
          }
          volatile unsigned long long* slot = s_cache + c * FS + (int)((mix64(key) >> 40) & (FS - 1));
          if (*slot == key) continue;
          bool claimed = false;
          const long long h = probe<true>(a.keys + o, cap, a.full_probe || cap < kMaxProbe ? cap : kMaxProbe, key,
                                            &claimed);
          if (h < 0) {
            atomicOr(a.status + j, (unsigned long long)ST_OVERFLOW);
            continue;
          }
          if (claimed) {
            a.counts[o + h] = 1ull;
            const unsigned long long occ = atomicAdd(a.occupied + j, 1ull) + 1ull;
            if (2 * occ > (unsigned long long)cap) atomicOr(a.status + j, (unsigned long long)ST_OVERFLOW);
          }
          *slot = key;
        }
      }
    }
  }
}

template <typename T, bool COUNT>
static int launch_key_scan(const ScanArgs& a, int sms, cudaStream_t s) {
  constexpr int CS = 32 / sizeof(T);
  const int gy = (a.g + CS - 1) / CS < 65535 ? (a.g + CS - 1) / CS : 65535;
  const long long tiles = (a.n + kTileRows - 1) / kTileRows;
  long long gx = ((long long)8 * sms + gy - 1) / gy;
  if (gx > tiles) gx = tiles;
  if (gx < 1) gx = 1;
  key_scan_kernel<T, COUNT><<<dim3((unsigned)gx, (unsigned)gy), kThreads, 0, s>>>(a);
  BKM_CUDA_TRY(cudaGetLastError());
  note_launch();
  return 0;
}

// ============================================ best entry ============================================
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

// ============================================ compact / merge ============================================
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
    const long long h = probe<false>(a.keys + o, cap, cap, k, nullptr);
    if (h >= 0) atomicAdd(a.counts + o + h, (unsigned long long)cnt);
  }
}

}  // namespace
}  // namespace bkm

using namespace bkm;

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
  ScanArgs a = {};
  a.X = X; a.n = n; a.g = g; a.ldx = ldx; a.miss.is_nan = miss_is_nan; a.miss.value = miss_value; a.keys = keys;
  a.counts = counts; a.off = reinterpret_cast<const long long*>(slot_off);
  if (x_dtype == BKM_F32) return launch_key_scan<float, true>(a, sms, s);
  if (x_dtype == BKM_F64) return launch_key_scan<double, true>(a, sms, s);
  return launch_key_scan<__nv_bfloat16, true>(a, sms, s);
}

extern "C" int bkm_distinct_chunk(const void* X, int64_t n, int g, int64_t ldx, int x_dtype, unsigned long long* keys,
                                  unsigned long long* counts, const int64_t* slot_off, int64_t total_slots,
                                  unsigned long long* state, int flags, void* stream) {
  if (n < 0 || g <= 0 || ldx < g || total_slots < 0 || !slot_off || !state) return BKM_EINVAL;
  if (total_slots > 0 && (!keys || !counts)) return BKM_EINVAL;
  if (n > 0 && !X) return BKM_EINVAL;
  if (!enc_dtype_ok(x_dtype)) return BKM_EDTYPE;
  cudaStream_t s = (cudaStream_t)stream;
  if (flags & BKM_FLAG_FIRST_CHUNK) {
    if (total_slots > 0) {
      BKM_CUDA_TRY(cudaMemsetAsync(keys, 0xff, (size_t)total_slots * 8, s));
      BKM_CUDA_TRY(cudaMemsetAsync(counts, 0, (size_t)total_slots * 8, s));
    }
    BKM_CUDA_TRY(cudaMemsetAsync(state, 0, (size_t)g * 16, s));
  }
  if (n == 0 || total_slots == 0) return 0;
  int sms = 0;
  const int rc = sm_count(&sms);
  if (rc) return rc;
  ScanArgs a = {};
  a.X = X; a.n = n; a.g = g; a.ldx = ldx; a.keys = keys; a.counts = counts;
  a.off = reinterpret_cast<const long long*>(slot_off); a.occupied = state; a.status = state + g;
  a.full_probe = (flags & BKM_FLAG_FULL_PROBE) ? 1 : 0;
  switch (x_dtype) {
    case BKM_F32: return launch_key_scan<float, false>(a, sms, s);
    case BKM_F64: return launch_key_scan<double, false>(a, sms, s);
    case BKM_BF16: return launch_key_scan<__nv_bfloat16, false>(a, sms, s);
    case BKM_M_I32: return launch_key_scan<int, false>(a, sms, s);
    case BKM_M_I64: return launch_key_scan<long long, false>(a, sms, s);
    default: return launch_key_scan<unsigned char, false>(a, sms, s);
  }
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
