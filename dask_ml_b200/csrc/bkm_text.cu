// bkm_text.cu — the passes of HashingVectorizer over one block of ASCII documents (sm_90a).
//
//   bkm_text_tokens_chunk  token starts (one stream compaction over the bytes), each document's first token (a binary
//                          search per document) and its n-gram count, scanned into pair offsets
//   bkm_text_hash_chunk    one thread per token hashes the token and the n-grams it starts (MurmurHash3 x86_32 fed
//                          incrementally, so an n-gram costs the bytes it adds), giving a (column, sign) key per n-gram;
//                          a segmented sort orders each document's keys; one warp per document counts its columns and
//                          the l1 / l2 sum of its values, scanned into indptr
//   bkm_text_write_chunk   one warp per document writes indices and data, binary and norm applied
//
// A key is 2 column + (1 when the n-gram's sign is negative), so that one document's sorted keys hold each column's
// positive n-grams, then its negative ones: a column's value is their difference, found by two binary searches from
// the first key of its run.
#include "bkm_select.cuh"
#include <cub/device/device_scan.cuh>
#include <cub/device/device_segmented_sort.cuh>
#include <cub/device/device_select.cuh>
#include <thrust/iterator/counting_iterator.h>
#include <limits.h>

namespace bkm {
namespace {

__device__ __forceinline__ bool is_word(unsigned char c) {
  return (c >= '0' && c <= '9') || (c >= 'A' && c <= 'Z') || (c >= 'a' && c <= 'z') || c == '_';
}

// a token starts at i: a run of at least two word bytes begins there
struct TokenStart {
  const unsigned char* b;
  long long n;
  __device__ __forceinline__ bool operator()(long long i) const {
    return is_word(b[i]) && i + 1 < n && is_word(b[i + 1]) && (i == 0 || !is_word(b[i - 1]));
  }
};

// first position in a[lo, hi) whose value is >= v
template <typename T, typename V>
__device__ __forceinline__ long long lower_bound(const T* a, long long lo, long long hi, V v) {
  while (lo < hi) {
    const long long m = (lo + hi) >> 1;
    if ((V)a[m] < v) lo = m + 1;
    else hi = m;
  }
  return lo;
}

// n-grams of a document of t tokens with min_n <= n <= max_n
__device__ __forceinline__ long long ngram_count(long long t, int min_n, int max_n) {
  const long long hi = t < max_n ? t : max_n;
  if (hi < min_n) return 0;
  const long long m = hi - min_n + 1;
  return m * (t + 1) - (min_n + hi) * m / 2;
}

__global__ void __launch_bounds__(kThreads) doc_tokens_kernel(const long long* tok_start, const long long* n_tokens,
                                                              const long long* doc_off, long long n, int min_n,
                                                              int max_n, long long* tok_off, long long* pcount) {
  const long long d = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (d > n) return;
  const long long T = *n_tokens;
  const long long t0 = lower_bound(tok_start, 0, T, doc_off[d]);
  tok_off[d] = t0;
  if (d == n) {
    pcount[d] = 0;
    return;
  }
  const long long t1 = lower_bound(tok_start, t0, T, doc_off[d + 1]);
  pcount[d] = ngram_count(t1 - t0, min_n, max_n);
}

// MurmurHash3 x86_32 (seed 0) over a byte stream
struct Murmur {
  unsigned h, k, len;
  int nt;
  __device__ __forceinline__ void init() { h = 0; k = 0; len = 0; nt = 0; }
  __device__ __forceinline__ static unsigned scramble(unsigned k) {
    k *= 0xcc9e2d51u;
    k = (k << 15) | (k >> 17);
    return k * 0x1b873593u;
  }
  __device__ __forceinline__ void feed(unsigned c) {
    k |= c << (8 * nt);
    ++len;
    if (++nt == 4) {
      h ^= scramble(k);
      h = (h << 13) | (h >> 19);
      h = h * 5u + 0xe6546b64u;
      k = 0;
      nt = 0;
    }
  }
  __device__ __forceinline__ int finish() const {
    unsigned x = h;
    if (nt) x ^= scramble(k);
    x ^= len;
    x ^= x >> 16;
    x *= 0x85ebca6bu;
    x ^= x >> 13;
    x *= 0xc2b2ae35u;
    x ^= x >> 16;
    return (int)x;
  }
};

__device__ __forceinline__ void feed_token(Murmur& m, const unsigned char* b, long long p, long long n_bytes,
                                           bool lower) {
  for (; p < n_bytes; ++p) {
    unsigned c = b[p];
    if (!is_word((unsigned char)c)) break;
    if (lower && c >= 'A' && c <= 'Z') c += 32;
    m.feed(c);
  }
}

struct HashArgs {
  const unsigned char* buf;
  long long n_bytes;
  const long long* tok_start;
  const long long* tok_off;
  const long long* pair_off;
  long long n_docs, n_tokens, n_features;
  int min_n, max_n, lower, alternate_sign;
  unsigned* keys;
};

// scikit-learn's column and sign of a signed 32-bit hash (_hashing_fast.pyx)
__device__ __forceinline__ unsigned hash_key(int h, long long nf, int alternate_sign) {
  const long long col = h == INT_MIN ? (2147483647LL - (nf - 1)) % nf : (long long)(h < 0 ? -h : h) % nf;
  return (unsigned)(2 * col) + (alternate_sign && h < 0 ? 1u : 0u);
}

__global__ void __launch_bounds__(kThreads) hash_kernel(HashArgs a) {
  const long long k = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (k >= a.n_tokens) return;
  // the document of token k: the last d with tok_off[d] <= k
  long long lo = 0, hi = a.n_docs;
  while (lo < hi) {
    const long long m = (lo + hi + 1) >> 1;
    if (a.tok_off[m] <= k) lo = m;
    else hi = m - 1;
  }
  const long long d = lo, t = k - a.tok_off[d], T = a.tok_off[d + 1] - a.tok_off[d];
  long long pos = a.pair_off[d] + t;          // the n-grams of length n start at the sum of the counts of shorter ones
  Murmur m;
  m.init();
  feed_token(m, a.buf, a.tok_start[k], a.n_bytes, a.lower);
  for (int n = 1; n <= a.max_n; ++n) {
    if (n > 1) {
      if (t + n > T) break;
      m.feed(' ');
      feed_token(m, a.buf, a.tok_start[k + n - 1], a.n_bytes, a.lower);
    }
    if (n >= a.min_n) {
      a.keys[pos] = hash_key(m.finish(), a.n_features, a.alternate_sign);
      pos += T - n + 1;
    }
  }
}

// One warp per document over its sorted keys [pair_off[d], pair_off[d + 1]).  For each run of one column the first
// lane of the run computes the column's value.  RowPass 0 counts the columns and folds the norm's sum into scale[d]
// (0: leave the row alone); RowPass 1 writes indices and data at indptr[d].
template <typename T, int PASS>
__global__ void __launch_bounds__(kThreads) rows_kernel(const unsigned* keys, const long long* pair_off, long long n,
                                                        int binary, int norm, long long* count, double* scale,
                                                        const long long* indptr, long long* indices, T* data) {
  const long long d = ((long long)blockIdx.x * kThreads + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (d >= n) return;
  const long long a = pair_off[d], e = pair_off[d + 1];
  long long nnz = PASS == 1 ? indptr[d] : 0;
  double acc = 0.0;
  const double s = PASS == 1 ? scale[d] : 0.0;
  for (long long p0 = a; p0 < e; p0 += 32) {
    const long long p = p0 + lane;
    bool start = false;
    unsigned col = 0;
    if (p < e) {
      const unsigned key = keys[p];
      col = key >> 1;
      start = p == a || (keys[p - 1] >> 1) != col;
    }
    const unsigned ball = __ballot_sync(0xffffffffu, start);
    if (start) {
      long long v = 1;
      if (!binary) {
        const long long q = lower_bound(keys, p, e, 2ull * col + 1);
        const long long r = lower_bound(keys, q, e, 2ull * col + 2);
        v = (q - p) - (r - q);
      }
      const T vt = (T)v;
      if (PASS == 0) {
        if (norm == 1) acc = __dadd_rn(acc, fabs((double)vt));
        else if (norm == 2) acc = __dadd_rn(acc, (double)(sizeof(T) == 4 ? (T)__fmul_rn((float)vt, (float)vt)
                                                                          : (T)__dmul_rn((double)vt, (double)vt)));
      } else {
        const long long o = nnz + __popc(ball & ((1u << lane) - 1u));
        indices[o] = col;
        T out = vt;
        if (s != 0.0) {
          const double q = __ddiv_rn((double)vt, s);
          out = sizeof(T) == 4 ? (T)__double2float_rn(q) : (T)q;
        }
        data[o] = out;
      }
    }
    nnz += __popc(ball);
  }
  if constexpr (PASS == 0) {
    // the terms are integers (or float32 roundings of integer squares) whose sum stays below 2^53: exact in any order
    for (int o = 16; o; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) {
      count[d] = nnz;
      scale[d] = acc == 0.0 ? 0.0 : (norm == 2 ? __dsqrt_rn(acc) : acc);
    }
  }
}

// ------------------------------------------------ workspace ------------------------------------------------
constexpr size_t kAlign = 256;

struct TextWs {
  size_t counts;      // (n + 1) int64 per-document counts before their scan
  size_t keys;        // n_pairs uint32 unsorted keys
  size_t temp;        // CUB scratch
  size_t temp_bytes;
  size_t total;
};

static int text_ws(long long n_bytes, long long n, long long n_pairs, TextWs* w) {
  size_t sel = 0, scan = 0, sort = 0;
  thrust::counting_iterator<long long> it(0);
  BKM_CUDA_TRY(cub::DeviceSelect::If(nullptr, sel, it, (long long*)nullptr, (long long*)nullptr,
                                     (int64_t)(n_bytes > 0 ? n_bytes : 1), TokenStart{nullptr, 0}));
  BKM_CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, scan, (long long*)nullptr, (long long*)nullptr, (int)(n + 1)));
  if (n_pairs > 0)
    BKM_CUDA_TRY(cub::DeviceSegmentedSort::SortKeys(nullptr, sort, (const unsigned*)nullptr, (unsigned*)nullptr,
                                                    (int)n_pairs, (int)n, (const long long*)nullptr,
                                                    (const long long*)nullptr));
  w->counts = 0;
  w->keys = align_up((size_t)(n + 1) * 8, kAlign);
  w->temp = w->keys + align_up((size_t)n_pairs * 4, kAlign);
  size_t t = sel > scan ? sel : scan;
  w->temp_bytes = t > sort ? t : sort;
  w->total = w->temp + align_up(w->temp_bytes, kAlign);
  return 0;
}

}  // namespace
}  // namespace bkm

using namespace bkm;

extern "C" int bkm_text_workspace_bytes(int64_t n_bytes, int64_t n_docs, int64_t n_pairs, size_t* out) {
  if (!out || n_bytes < 0 || n_docs < 0 || n_docs >= INT_MAX || n_pairs < 0) return BKM_EINVAL;
  if (n_pairs > INT_MAX) return BKM_EUNSUPPORTED;
  TextWs w;
  const int rc = text_ws(n_bytes, n_docs, n_pairs, &w);
  if (rc) return rc;
  *out = w.total;
  return 0;
}

extern "C" int bkm_text_tokens_chunk(const uint8_t* buf, int64_t n_bytes, const int64_t* doc_off, int64_t n_docs,
                                     int min_n, int max_n, int64_t* tok_start, int64_t tok_cap, int64_t* tok_off,
                                     int64_t* pair_off, int64_t* totals, void* workspace, size_t ws_bytes,
                                     void* stream) {
  if (n_bytes < 0 || n_docs < 0 || n_docs >= INT_MAX || min_n < 1 || max_n < min_n) return BKM_EINVAL;
  if (!doc_off || !tok_off || !pair_off || !totals || !workspace) return BKM_EINVAL;
  if (n_bytes > 0 && (!buf || !tok_start)) return BKM_EINVAL;
  if (tok_cap < n_bytes / 3 + 1) return BKM_EINVAL;
  TextWs w;
  int rc = text_ws(n_bytes, n_docs, 0, &w);
  if (rc) return rc;
  if (ws_bytes < w.total) return BKM_EWORKSPACE;
  cudaStream_t s = (cudaStream_t)stream;
  unsigned char* ws = reinterpret_cast<unsigned char*>(workspace);
  long long* T = reinterpret_cast<long long*>(totals);
  size_t tb = w.temp_bytes;
  if (n_bytes > 0) {
    BKM_CUDA_TRY(cub::DeviceSelect::If(ws + w.temp, tb, thrust::counting_iterator<long long>(0),
                                       reinterpret_cast<long long*>(tok_start), T, (int64_t)n_bytes,
                                       TokenStart{buf, n_bytes}, s));
    note_launch();
  } else {
    BKM_CUDA_TRY(cudaMemsetAsync(T, 0, 8, s));
  }
  long long* pc = reinterpret_cast<long long*>(ws + w.counts);
  doc_tokens_kernel<<<(unsigned)((n_docs + kThreads) / kThreads), kThreads, 0, s>>>(
      reinterpret_cast<const long long*>(tok_start), T, reinterpret_cast<const long long*>(doc_off), n_docs, min_n,
      max_n, reinterpret_cast<long long*>(tok_off), pc);
  BKM_CUDA_TRY(cudaGetLastError());
  note_launch();
  tb = w.temp_bytes;
  BKM_CUDA_TRY(cub::DeviceScan::ExclusiveSum(ws + w.temp, tb, pc, reinterpret_cast<long long*>(pair_off),
                                             (int)(n_docs + 1), s));
  note_launch();
  BKM_CUDA_TRY(cudaMemcpyAsync(T + 1, pair_off + n_docs, 8, cudaMemcpyDeviceToDevice, s));
  return 0;
}

extern "C" int bkm_text_hash_chunk(const uint8_t* buf, int64_t n_bytes, const int64_t* tok_start,
                                   const int64_t* tok_off, const int64_t* pair_off, int64_t n_docs, int64_t n_tokens,
                                   int64_t n_pairs, int min_n, int max_n, int lowercase, int64_t n_features,
                                   int alternate_sign, int binary, int norm, int out_dtype, uint32_t* keys,
                                   int64_t* indptr, double* scale, int64_t* totals, void* workspace, size_t ws_bytes,
                                   void* stream) {
  if (n_bytes < 0 || n_docs < 0 || n_docs >= INT_MAX || n_tokens < 0 || n_pairs < 0 || min_n < 1 || max_n < min_n)
    return BKM_EINVAL;
  if (n_features < 1 || n_features > INT_MAX || norm < 0 || norm > 2) return BKM_EINVAL;
  if (!tok_off || !pair_off || !indptr || !scale || !totals || !workspace) return BKM_EINVAL;
  if (n_tokens > 0 && (!buf || !tok_start)) return BKM_EINVAL;
  if (n_pairs > 0 && !keys) return BKM_EINVAL;
  if (out_dtype != BKM_F32 && out_dtype != BKM_F64) return BKM_EDTYPE;
  if (n_pairs > INT_MAX) return BKM_EUNSUPPORTED;
  TextWs w;
  int rc = text_ws(n_bytes, n_docs, n_pairs, &w);
  if (rc) return rc;
  if (ws_bytes < w.total) return BKM_EWORKSPACE;
  cudaStream_t s = (cudaStream_t)stream;
  unsigned char* ws = reinterpret_cast<unsigned char*>(workspace);
  const long long* poff = reinterpret_cast<const long long*>(pair_off);
  if (n_tokens > 0) {
    HashArgs a;
    a.buf = buf; a.n_bytes = n_bytes; a.tok_start = reinterpret_cast<const long long*>(tok_start);
    a.tok_off = reinterpret_cast<const long long*>(tok_off); a.pair_off = poff; a.n_docs = n_docs;
    a.n_tokens = n_tokens; a.n_features = n_features; a.min_n = min_n; a.max_n = max_n; a.lower = lowercase != 0;
    a.alternate_sign = alternate_sign != 0; a.keys = reinterpret_cast<unsigned*>(ws + w.keys);
    hash_kernel<<<(unsigned)((n_tokens + kThreads - 1) / kThreads), kThreads, 0, s>>>(a);
    BKM_CUDA_TRY(cudaGetLastError());
    note_launch();
  }
  size_t tb = w.temp_bytes;
  if (n_pairs > 0) {
    BKM_CUDA_TRY(cub::DeviceSegmentedSort::SortKeys(ws + w.temp, tb, reinterpret_cast<const unsigned*>(ws + w.keys),
                                                    reinterpret_cast<unsigned*>(keys), (int)n_pairs, (int)n_docs, poff,
                                                    poff + 1, s));
    note_launch();
  }
  long long* cnt = reinterpret_cast<long long*>(ws + w.counts);
  BKM_CUDA_TRY(cudaMemsetAsync(cnt + n_docs, 0, 8, s));
  if (n_docs > 0) {
    const unsigned grid = (unsigned)((n_docs * 32 + kThreads - 1) / kThreads);
    if (out_dtype == BKM_F32)
      rows_kernel<float, 0><<<grid, kThreads, 0, s>>>(reinterpret_cast<const unsigned*>(keys), poff, n_docs,
                                                      binary != 0, norm, cnt, scale, nullptr, nullptr, nullptr);
    else
      rows_kernel<double, 0><<<grid, kThreads, 0, s>>>(reinterpret_cast<const unsigned*>(keys), poff, n_docs,
                                                       binary != 0, norm, cnt, scale, nullptr, nullptr, nullptr);
    BKM_CUDA_TRY(cudaGetLastError());
    note_launch();
  }
  tb = w.temp_bytes;
  BKM_CUDA_TRY(cub::DeviceScan::ExclusiveSum(ws + w.temp, tb, cnt, reinterpret_cast<long long*>(indptr),
                                             (int)(n_docs + 1), s));
  note_launch();
  BKM_CUDA_TRY(cudaMemcpyAsync(totals + 2, indptr + n_docs, 8, cudaMemcpyDeviceToDevice, s));
  return 0;
}

extern "C" int bkm_text_write_chunk(const uint32_t* keys, const int64_t* pair_off, const int64_t* indptr,
                                    const double* scale, int64_t n_docs, int binary, int64_t* indices, void* data,
                                    int out_dtype, void* stream) {
  if (n_docs < 0 || n_docs >= INT_MAX || !pair_off || !indptr || !scale) return BKM_EINVAL;
  if (out_dtype != BKM_F32 && out_dtype != BKM_F64) return BKM_EDTYPE;
  if (n_docs == 0) return 0;
  cudaStream_t s = (cudaStream_t)stream;
  const unsigned grid = (unsigned)((n_docs * 32 + kThreads - 1) / kThreads);
  const long long* poff = reinterpret_cast<const long long*>(pair_off);
  const long long* ip = reinterpret_cast<const long long*>(indptr);
  long long* idx = reinterpret_cast<long long*>(indices);
  if (out_dtype == BKM_F32)
    rows_kernel<float, 1><<<grid, kThreads, 0, s>>>(keys, poff, n_docs, binary != 0, 0, nullptr,
                                                    const_cast<double*>(scale), ip, idx, reinterpret_cast<float*>(data));
  else
    rows_kernel<double, 1><<<grid, kThreads, 0, s>>>(keys, poff, n_docs, binary != 0, 0, nullptr,
                                                     const_cast<double*>(scale), ip, idx,
                                                     reinterpret_cast<double*>(data));
  BKM_CUDA_TRY(cudaGetLastError());
  note_launch();
  return 0;
}
