// bkm_encode.cu — the passes of LabelEncoder and OneHotEncoder over row chunks (sm_90a).  The categories come from the
// per-column key tables of bkm_keys.cu (bkm_distinct_chunk).
//
//   bkm_encode_chunk     one read of X: each element's key is looked up by binary search in its column's sorted key
//                        list (staged in shared memory when every list fits, else read through L2) and written as a
//                        code (CODES), a CSR index and one (CSR), or a one-hot row (DENSE: the CTA's tile of rows is
//                        written once, zeros and ones together, in 16-byte stores).  Unknown keys are counted and a few
//                        per column kept for the error message.
//   bkm_decode_chunk     codes -> category values, a typeless gather of 1, 2, 4 or 8-byte elements; codes outside
//                        [0, K) counted and kept as for unknown keys.
#include "bkm_select.cuh"
#include <type_traits>

namespace bkm {
namespace {

constexpr int kDenseRowsMax = 256;       // rows per tile of the one-hot writer
constexpr int kPosInts = 2048;           // the tile's positions (rows x d ints) in shared memory

// ============================================ encode ============================================
struct EncodeArgs {
  const void* X;
  long long n;
  int d;
  long long ldx;
  const unsigned long long* cat_keys;   // [n_cats], global
  const long long* cat_off;             // [d + 1], global
  long long n_cats;
  int layout;
  int stage;                            // 1: keys and offsets staged in shared memory
  int rows;                             // rows per tile
  void* out;
  long long ld_out;
  long long* indices;
  unsigned long long* unknown;          // [1 + d + d * BKM_ENCODE_KEEP]
};

__device__ __forceinline__ void note_unknown(unsigned long long* unknown, int d, int j, unsigned long long key) {
  atomicAdd(unknown, 1ull);
  const unsigned long long p = atomicAdd(unknown + 1 + j, 1ull);
  if (p < BKM_ENCODE_KEEP) unknown[1 + d + (size_t)j * BKM_ENCODE_KEEP + p] = key;
}

// position of `key` in keys[lo, hi) (sorted), or -1
__device__ __forceinline__ long long find_key(const unsigned long long* keys, long long lo, long long hi,
                                              unsigned long long key) {
  long long b = lo, e = hi;
  while (b < e) {
    const long long m = (b + e) >> 1;
    if (keys[m] < key) b = m + 1;
    else e = m;
  }
  return (b < hi && keys[b] == key) ? b : -1;
}

template <typename C> __device__ __forceinline__ C one_of(bool v) { return v ? (C)1 : (C)0; }

template <typename T, typename C>
__global__ void __launch_bounds__(kThreads) encode_kernel(EncodeArgs a) {
  extern __shared__ __align__(16) unsigned char s_raw[];
  const int tid = threadIdx.x, d = a.d;
  long long* s_off = reinterpret_cast<long long*>(s_raw);
  unsigned long long* s_keys = reinterpret_cast<unsigned long long*>(s_raw + (size_t)(d + 1) * 8);
  int* s_pos = reinterpret_cast<int*>(s_raw + (a.stage ? (size_t)(d + 1 + a.n_cats) * 8 : 0));
  const long long* off = a.cat_off;
  const unsigned long long* keys = a.cat_keys;
  if (a.stage) {
    for (int i = tid; i <= d; i += kThreads) s_off[i] = a.cat_off[i];
    for (long long i = tid; i < a.n_cats; i += kThreads) s_keys[i] = a.cat_keys[i];
    __syncthreads();
    off = s_off;
    keys = s_keys;
  }
  const T* X = reinterpret_cast<const T*>(a.X);
  const int R = a.rows;
  const long long tiles = (a.n + R - 1) / R;
  const long long W = a.n_cats;
#pragma unroll 1
  for (long long t = blockIdx.x; t < tiles; t += gridDim.x) {
    const long long r0 = t * R;
    const int rt = (int)min((long long)R, a.n - r0);
    for (int e = tid; e < rt * d; e += kThreads) {
      const int r = e / d, j = e - r * d;
      const unsigned long long key = enc_key(X[(r0 + r) * a.ldx + j]);
      const long long lo = off[j];
      const long long p = find_key(keys, lo, off[j + 1], key);
      if (p < 0) note_unknown(a.unknown, d, j, key);
      if (a.layout == BKM_ENCODE_CODES) {
        reinterpret_cast<long long*>(a.out)[(r0 + r) * a.ld_out + j] = p < 0 ? -1 : p - lo;
      } else if (a.layout == BKM_ENCODE_CSR) {
        const long long i = (r0 + r) * d + j;
        a.indices[i] = p;
        reinterpret_cast<C*>(a.out)[i] = (C)1;
      } else {
        s_pos[e] = (int)p;
      }
    }
    if (a.layout != BKM_ENCODE_DENSE) continue;
    __syncthreads();
    // the tile's rows are the contiguous elements [r0 W, (r0 + rt) W) of out: 16-byte stores in the aligned middle,
    // single elements at the two ends; element (r, c) is 1 iff c is the position of row r's value of the input column
    // whose output columns hold c
    constexpr int V = 16 / sizeof(C);
    C* out = reinterpret_cast<C*>(a.out);
    const long long e0 = r0 * W, e1 = (r0 + rt) * W;
    const long long v0 = (e0 + V - 1) / V, v1 = e1 / V;
    auto value = [&](long long e, int& j) -> C {
      const long long r = e / W - r0, c = e - (e / W) * W;
      if (j < 0 || c < off[j] || c >= off[j + 1]) {               // find the input column of c (upper bound - 1)
        int b = 0, f = d;
        while (b < f) {
          const int m = (b + f) >> 1;
          if (off[m + 1] <= c) b = m + 1;
          else f = m;
        }
        j = b;
      }
      return one_of<C>(s_pos[r * d + j] == c);
    };
    if (v0 < v1) {
      for (long long v = v0 + tid; v < v1; v += kThreads) {
        union { uint4 u; C c[V]; } pack;
        int j = -1;
#pragma unroll
        for (int i = 0; i < V; ++i) pack.c[i] = value(v * V + i, j);
        reinterpret_cast<uint4*>(out)[v] = pack.u;
      }
      for (long long e = e0 + tid; e < v0 * V; e += kThreads) { int j = -1; out[e] = value(e, j); }
      for (long long e = v1 * V + tid; e < e1; e += kThreads) { int j = -1; out[e] = value(e, j); }
    } else {
      for (long long e = e0 + tid; e < e1; e += kThreads) { int j = -1; out[e] = value(e, j); }
    }
    __syncthreads();
  }
}

template <typename T, typename C>
static int launch_encode(EncodeArgs& a, int sms, cudaStream_t s) {
  const size_t keys_bytes = (size_t)(a.d + 1 + a.n_cats) * 8;
  const size_t pos_bytes = a.layout == BKM_ENCODE_DENSE ? (size_t)a.rows * a.d * 4 : 0;
  a.stage = keys_bytes + pos_bytes <= 40 * 1024;
  const size_t smem = (a.stage ? keys_bytes : 0) + pos_bytes;
  const long long tiles = (a.n + a.rows - 1) / a.rows;
  long long g = tiles < 8LL * sms ? tiles : 8LL * sms;
  if (g < 1) g = 1;
  encode_kernel<T, C><<<(unsigned)g, kThreads, smem, s>>>(a);
  BKM_CUDA_TRY(cudaGetLastError());
  note_launch();
  return 0;
}

template <typename T>
static int dispatch_out(EncodeArgs& a, int out_dtype, int sms, cudaStream_t s) {
  if (a.layout == BKM_ENCODE_CODES) return launch_encode<T, long long>(a, sms, s);
  switch (out_dtype) {
    case BKM_F64: return launch_encode<T, double>(a, sms, s);
    case BKM_F32: return launch_encode<T, float>(a, sms, s);
    case BKM_M_I64: return launch_encode<T, long long>(a, sms, s);
    case BKM_M_I32: return launch_encode<T, int>(a, sms, s);
    default: return launch_encode<T, unsigned char>(a, sms, s);
  }
}

// ============================================ decode ============================================
struct DecodeArgs {
  const void* codes;
  int code_dtype;
  long long n;
  int d;
  long long ldc;
  const unsigned char* vals;
  const long long* cat_off;
  int elem;
  unsigned char* out;
  long long ld_out;
  unsigned long long* unknown;
};

template <int E>
__global__ void __launch_bounds__(kThreads) decode_kernel(DecodeArgs a) {
  using U = typename std::conditional<E == 8, unsigned long long,
            typename std::conditional<E == 4, unsigned, typename std::conditional<E == 2, unsigned short,
                                                                                   unsigned char>::type>::type>::type;
  const U* vals = reinterpret_cast<const U*>(a.vals);
  U* out = reinterpret_cast<U*>(a.out);
  const long long total = a.n * a.d;
  for (long long e = (long long)blockIdx.x * kThreads + threadIdx.x; e < total; e += (long long)gridDim.x * kThreads) {
    const long long r = e / a.d;
    const int j = (int)(e - r * a.d);
    const long long code = a.code_dtype == BKM_M_I64 ? reinterpret_cast<const long long*>(a.codes)[r * a.ldc + j]
                                                     : (long long)reinterpret_cast<const int*>(a.codes)[r * a.ldc + j];
    const long long lo = __ldg(a.cat_off + j), k = __ldg(a.cat_off + j + 1) - lo;
    U v = 0;
    if (code >= 0 && code < k) v = vals[lo + code];
    else note_unknown(a.unknown, a.d, j, (unsigned long long)code);
    out[r * a.ld_out + j] = v;
  }
}

}  // namespace
}  // namespace bkm

using namespace bkm;

extern "C" int bkm_encode_chunk(const void* X, int64_t n, int d, int64_t ldx, int x_dtype,
                                const unsigned long long* cat_keys, const int64_t* cat_off, int64_t n_cats, int layout,
                                void* out, int64_t ld_out, int out_dtype, int64_t* indices, unsigned long long* unknown,
                                void* stream) {
  if (n < 0 || d <= 0 || ldx < d || n_cats < 0 || !cat_off || !unknown) return BKM_EINVAL;
  if (n_cats > 0 && !cat_keys) return BKM_EINVAL;
  if (layout != BKM_ENCODE_CODES && layout != BKM_ENCODE_DENSE && layout != BKM_ENCODE_CSR) return BKM_EINVAL;
  if (layout == BKM_ENCODE_CODES && ld_out < d) return BKM_EINVAL;
  if (layout == BKM_ENCODE_DENSE && (ld_out != n_cats || n_cats > 0x7fffffffLL)) return BKM_EINVAL;
  if (layout == BKM_ENCODE_CSR && n > 0 && !indices) return BKM_EINVAL;
  if (n > 0 && (!X || (!out && !(layout == BKM_ENCODE_DENSE && n_cats == 0)))) return BKM_EINVAL;
  if (!enc_dtype_ok(x_dtype)) return BKM_EDTYPE;
  if (layout != BKM_ENCODE_CODES && out_dtype != BKM_F64 && out_dtype != BKM_F32 && out_dtype != BKM_M_I64 &&
      out_dtype != BKM_M_I32 && out_dtype != BKM_M_U8)
    return BKM_EDTYPE;
  if (layout == BKM_ENCODE_DENSE && ((uintptr_t)out & 15)) return BKM_EALIGN;
  if (n == 0 || (layout == BKM_ENCODE_DENSE && n_cats == 0)) return 0;
  int sms = 0;
  const int rc = sm_count(&sms);
  if (rc) return rc;
  EncodeArgs a;
  a.X = X; a.n = n; a.d = d; a.ldx = ldx; a.cat_keys = cat_keys; a.cat_off = reinterpret_cast<const long long*>(cat_off);
  a.n_cats = n_cats; a.layout = layout; a.out = out; a.ld_out = ld_out; a.indices = reinterpret_cast<long long*>(indices);
  a.unknown = unknown; a.stage = 0;
  a.rows = layout == BKM_ENCODE_DENSE ? (kPosInts / d < kDenseRowsMax ? kPosInts / d : kDenseRowsMax) : kThreads * 4 / d;
  if (a.rows < 1) a.rows = 1;
  if (layout == BKM_ENCODE_DENSE && (long long)a.rows * d > kPosInts) return BKM_EUNSUPPORTED;   // d > 2048
  cudaStream_t s = (cudaStream_t)stream;
  switch (x_dtype) {
    case BKM_F32: return dispatch_out<float>(a, out_dtype, sms, s);
    case BKM_F64: return dispatch_out<double>(a, out_dtype, sms, s);
    case BKM_BF16: return dispatch_out<__nv_bfloat16>(a, out_dtype, sms, s);
    case BKM_M_I32: return dispatch_out<int>(a, out_dtype, sms, s);
    case BKM_M_I64: return dispatch_out<long long>(a, out_dtype, sms, s);
    default: return dispatch_out<unsigned char>(a, out_dtype, sms, s);
  }
}

extern "C" int bkm_decode_chunk(const void* codes, int64_t n, int d, int64_t ldc, int code_dtype, const void* cat_vals,
                                const int64_t* cat_off, int elem_bytes, void* out, int64_t ld_out,
                                unsigned long long* unknown, void* stream) {
  if (n < 0 || d <= 0 || ldc < d || ld_out < d || !cat_off || !unknown) return BKM_EINVAL;
  if (elem_bytes != 1 && elem_bytes != 2 && elem_bytes != 4 && elem_bytes != 8) return BKM_EINVAL;
  if (n > 0 && (!codes || !out || !cat_vals)) return BKM_EINVAL;
  if (code_dtype != BKM_M_I32 && code_dtype != BKM_M_I64) return BKM_EDTYPE;
  if (n == 0) return 0;
  int sms = 0;
  const int rc = sm_count(&sms);
  if (rc) return rc;
  DecodeArgs a;
  a.codes = codes; a.code_dtype = code_dtype; a.n = n; a.d = d; a.ldc = ldc;
  a.vals = reinterpret_cast<const unsigned char*>(cat_vals); a.cat_off = reinterpret_cast<const long long*>(cat_off);
  a.elem = elem_bytes; a.out = reinterpret_cast<unsigned char*>(out); a.ld_out = ld_out; a.unknown = unknown;
  long long g = (n * d + kThreads - 1) / kThreads;
  if (g > 8LL * sms) g = 8LL * sms;
  cudaStream_t s = (cudaStream_t)stream;
  if (elem_bytes == 8) decode_kernel<8><<<(unsigned)g, kThreads, 0, s>>>(a);
  else if (elem_bytes == 4) decode_kernel<4><<<(unsigned)g, kThreads, 0, s>>>(a);
  else if (elem_bytes == 2) decode_kernel<2><<<(unsigned)g, kThreads, 0, s>>>(a);
  else decode_kernel<1><<<(unsigned)g, kThreads, 0, s>>>(a);
  BKM_CUDA_TRY(cudaGetLastError());
  note_launch();
  return 0;
}
