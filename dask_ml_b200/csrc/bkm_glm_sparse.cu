// bkm_glm_sparse.cu — the passes of the generalised linear models over one sparse CSR block (sm_90a): the CSR twin of
// bkm_glm_pass_chunk, the block's transpose (CSC) built once per fit, the column pass X^T v over that transpose, and
// the weighted Gram sum_i w_i x_i x_i^T of a Newton step.
//
// Every value is widened to float64 from the block's dtype (float32 or float64); every sum runs in a fixed order and
// no float atomics are used, so two calls with the same inputs give the same bits.
//
//   row pass     rows are handled by groups of G lanes (G = 4, 8, 16 or 32 from the block's mean entries per row): the
//                lanes sum val_k beta[col_k] lane-strided, a shuffle tree of fixed shape adds them, and the group's
//                first lane evaluates the family (the table of bkm_glm.cu).  The per-row [r | loss | w] sums are added
//                by a fixed shuffle tree per warp, the warps in order per CTA, and the CTA partials in CTA order by the
//                last CTA to finish (a ticket counter).
//   transpose    each entry's row is expanded, a stable radix sort on the column keeps the rows of a column ascending,
//                and the column pointers are the boundaries of the sorted keys.  The same call checks the block: a
//                column index outside [0, d) or not strictly above its predecessor in the row sets a flag.  It also
//                cuts every column into segments of at most SEG entries (the plan below), for the two passes after it.
//   column pass  one warp per segment sums v[row] val lane-strided, then a fixed shuffle tree; a column of one
//                segment is written directly, the segments of a longer column are written to slots and the last
//                segment to finish (a ticket per column) adds the slots in segment order.
//   Gram         one CTA per run of GS segments of column j keeps Gram row j in shared memory, one copy per warp; each
//                warp walks a contiguous part of the run in row order and, for each entry (i, x_ij), its lanes add
//                (w_i x_ij) x_ik over row i's entries k (the columns of a row are distinct: one writer per address per
//                step).  The warp copies are added in warp order; a column of several runs goes through slots folded
//                in run order by the last run to finish.
#include "bkm_common.cuh"
#include "bkm_csc_plan.cuh"
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

namespace bkm {
namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr long long GS = 32;           // segments per Gram run: a Gram CTA walks up to 64 Ki entries of its column
constexpr int kGramSmem = 96 * 1024;   // shared memory of a Gram CTA: the warps' copies of one Gram row

enum { GLM_GRAD = 0, GLM_NEWTON = 1, GLM_PREDICT = 2, GLM_LABEL = 3 };

__device__ __forceinline__ double to_f64(float v) { return (double)v; }
__device__ __forceinline__ double to_f64(double v) { return v; }

// (mu, loss, r, w) of one row: the families of bkm_glm.cu
__device__ __forceinline__ void family_terms(int family, double eta, double y, double& mu, double& loss, double& r,
                                             double& w) {
  if (family == 0) {
    const double e = exp(-fabs(eta));
    mu = eta >= 0.0 ? 1.0 / (1.0 + e) : e / (1.0 + e);
    loss = (fmax(eta, 0.0) + log1p(e)) - y * eta;
    r = mu - y;
    w = mu * (1.0 - mu);
  } else if (family == 1) {
    mu = eta;
    const double t = y - eta;
    loss = t * t;
    r = 2.0 * (eta - y);
    w = 2.0;
  } else {
    mu = exp(eta);
    loss = mu - y * eta;
    r = mu - y;
    w = mu;
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// row pass
// ---------------------------------------------------------------------------------------------------------------------
struct RowArgs {
  const long long* crow;
  const long long* col;
  const void* val;
  long long n;
  int d;
  const double* y;
  const double* beta;
  int family, mode;
  double* r;         // [n] (modes 0, 1)
  double* w;         // [n] (mode 1)
  double* grad;      // [d + 2]: [d] and [d + 1] written here
  double* hrow;      // [d + 1]: [d] written here (mode 1)
  void* out;         // [n] (modes 2, 3)
  double* part;      // [grid][3]
  unsigned int* ticket;
  int first;
};

template <typename T, int G>
__global__ void __launch_bounds__(kThreads, 4) csr_row_kernel(RowArgs a) {
  __shared__ double s_warp[kWarps][3];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int sub = lane & (G - 1);
  const T* val = reinterpret_cast<const T*>(a.val);
  const bool accumulate = a.mode == GLM_GRAD || a.mode == GLM_NEWTON;
  const double b0 = a.beta[a.d];
  constexpr int GPW = 32 / G;                                    // groups per warp
  const long long stride = (long long)gridDim.x * kWarps * GPW;
  double sr = 0.0, sl = 0.0, sw = 0.0;
  // the loop bound is uniform over the warp, so the shuffles below are convergent
#pragma unroll 1
  for (long long base = ((long long)blockIdx.x * kWarps + warp) * GPW; base < a.n; base += stride) {
    const long long i = base + lane / G;
    double acc = 0.0;
    if (i < a.n) {
      const long long k1 = a.crow[i + 1];
#pragma unroll 4
      for (long long k = a.crow[i] + sub; k < k1; k += G) {
        const long long c = a.col[k];
        if ((unsigned long long)c < (unsigned long long)a.d) acc = fma(to_f64(val[k]), __ldg(a.beta + c), acc);
      }
    }
#pragma unroll
    for (int off = G / 2; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
    if (sub == 0 && i < a.n) {
      const double eta = acc + b0;
      const double y = accumulate ? a.y[i] : 0.0;
      double mu, loss, rr, ww;
      family_terms(a.family, eta, y, mu, loss, rr, ww);
      if (a.mode == GLM_PREDICT) reinterpret_cast<double*>(a.out)[i] = mu;
      else if (a.mode == GLM_LABEL) reinterpret_cast<unsigned char*>(a.out)[i] = mu > 0.5 ? 1 : 0;
      else {
        a.r[i] = rr;
        sr += rr;
        sl += loss;
        if (a.mode == GLM_NEWTON) {
          a.w[i] = ww;
          sw += ww;
        }
      }
    }
  }
  if (!accumulate) return;

#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    sr += __shfl_xor_sync(0xffffffffu, sr, off);
    sl += __shfl_xor_sync(0xffffffffu, sl, off);
    sw += __shfl_xor_sync(0xffffffffu, sw, off);
  }
  if (lane == 0) {
    s_warp[warp][0] = sr;
    s_warp[warp][1] = sl;
    s_warp[warp][2] = sw;
  }
  __syncthreads();
  if (tid < 3) {
    double v = 0.0;
    for (int k = 0; k < kWarps; ++k) v += s_warp[k][tid];
    a.part[(size_t)blockIdx.x * 3 + tid] = v;
  }
  if (!last_block(a.ticket, gridDim.x)) return;
  if (tid < 3 && (tid < 2 || a.mode == GLM_NEWTON)) {
    double v = 0.0;
    for (unsigned c = 0; c < gridDim.x; ++c) v += __ldcg(a.part + (size_t)c * 3 + tid);
    double* dst = tid == 0 ? a.grad + a.d : tid == 1 ? a.grad + a.d + 1 : a.hrow + a.d;
    *dst = a.first ? v : *dst + v;
  }
  if (tid == 0) *a.ticket = 0u;
}

static int row_grid(long long n, int G, int sms) {
  const long long rows_per_cta = (long long)kWarps * (32 / G);
  long long g = (n + rows_per_cta - 1) / rows_per_cta;
  if (g > 4LL * sms) g = 4LL * sms;              // four CTAs per SM are resident (launch bounds)
  if (g < 1) g = 1;
  return (int)g;
}

static int row_group(long long n, long long nnz) {
  const double mean = n > 0 ? (double)nnz / (double)n : 0.0;
  return mean <= 6.0 ? 4 : mean <= 12.0 ? 8 : mean <= 24.0 ? 16 : 32;
}

static size_t row_ws(int sms) { return partials_bytes(4LL * sms, 3); }

template <typename T>
static int launch_row(const RowArgs& a, int G, int grid, cudaStream_t s) {
  switch (G) {
    case 4: csr_row_kernel<T, 4><<<grid, kThreads, 0, s>>>(a); break;
    case 8: csr_row_kernel<T, 8><<<grid, kThreads, 0, s>>>(a); break;
    case 16: csr_row_kernel<T, 16><<<grid, kThreads, 0, s>>>(a); break;
    default: csr_row_kernel<T, 32><<<grid, kThreads, 0, s>>>(a); break;
  }
  BKM_CUDA_TRY(cudaGetLastError());
  note_launch();
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------------
// transpose
// ---------------------------------------------------------------------------------------------------------------------
// one warp per row: each entry's row, its sort key and index; the checks of the block
__global__ void __launch_bounds__(kThreads) expand_kernel(const long long* crow, const long long* col, long long n,
                                                          int d, long long nnz, int* erow, unsigned* key, int* idx,
                                                          long long* status) {
  const long long warp0 = ((long long)blockIdx.x * kThreads + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const long long nw = ((long long)gridDim.x * kThreads) >> 5;
  int bad = 0;
  for (long long i = warp0; i < n; i += nw) {
    long long k0 = crow[i], k1 = crow[i + 1];
    if (k0 < 0 || k1 < k0 || k1 > nnz) {
      bad = 1;
      continue;
    }
    if (i == 0 && k0 != 0) bad = 1;
    if (i == n - 1 && k1 != nnz) bad = 1;
    for (long long k = k0 + lane; k < k1; k += 32) {
      const long long c = col[k];
      const bool ok = (unsigned long long)c < (unsigned long long)d;
      if (!ok || (k + 1 < k1 && col[k + 1] <= c)) bad = 1;
      erow[k] = (int)i;
      key[k] = ok ? (unsigned)c : 0u;
      idx[k] = (int)k;
    }
  }
  if (bad) atomicOr(reinterpret_cast<unsigned long long*>(status + ST_BAD), 1ull);
}

// rows / vals in sorted order; colptr[c] = the first sorted position whose key is >= c
template <typename T>
__global__ void __launch_bounds__(kThreads) gather_kernel(const unsigned* key_s, const int* perm, const int* erow,
                                                          const T* val, long long nnz, int d, long long* colptr,
                                                          int* rows, T* vals) {
  for (long long k = (long long)blockIdx.x * kThreads + threadIdx.x; k <= nnz; k += (long long)gridDim.x * kThreads) {
    if (k < nnz) {
      const int p = perm[k];
      rows[k] = erow[p];
      vals[k] = val[p];
    }
    const long long prev = k == 0 ? -1 : (long long)key_s[k - 1];
    const long long cur = k == nnz ? (long long)d : (long long)key_s[k];
    for (long long c = prev + 1; c <= cur; ++c) colptr[c] = k;
  }
}

// per column: its segments, its Gram runs when they are more than one (slots), the longest column
__global__ void __launch_bounds__(kThreads) count_kernel(const long long* colptr, int d, long long* nseg,
                                                         long long* nslot, long long* status) {
  const int j = blockIdx.x * kThreads + threadIdx.x;
  if (j > d) return;
  if (j == d) {
    nseg[d] = 0;
    nslot[d] = 0;
    return;
  }
  const long long len = colptr[j + 1] - colptr[j];
  const long long s = len > SEG ? (len + SEG - 1) / SEG : 1;
  nseg[j] = s;
  nslot[j] = s > GS ? (s + GS - 1) / GS : 0;
  atomicMax(reinterpret_cast<unsigned long long*>(status + ST_MAXLEN), (unsigned long long)len);
}

__global__ void __launch_bounds__(kThreads) fill_kernel(const long long* seg_off, const long long* gseg_off, int d,
                                                        int* seg_col, long long* status) {
  const int j = blockIdx.x * kThreads + threadIdx.x;
  if (j == 0) {
    status[ST_SEGS] = seg_off[d];
    status[ST_SLOTS] = gseg_off[d];
  }
  if (j >= d) return;
  for (long long t = seg_off[j]; t < seg_off[j + 1]; ++t) seg_col[t] = j;
}

struct TransposeWs {
  size_t erow, key, key_s, idx, perm, nseg, nslot, temp, temp_bytes, total;
};

static int transpose_ws(long long nnz, int d, TransposeWs* w) {
  size_t sort_b = 0, scan_b = 0;
  const int m = (int)(nnz > 0 ? nnz : 1);
  BKM_CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, sort_b, (const unsigned*)nullptr, (unsigned*)nullptr,
                                               (const int*)nullptr, (int*)nullptr, m));
  BKM_CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, scan_b, (long long*)nullptr, (long long*)nullptr, d + 1));
  size_t o = 0;
  const size_t e4 = align_up((size_t)m * 4, 256);
  w->erow = o; o += e4;
  w->key = o; o += e4;
  w->key_s = o; o += e4;
  w->idx = o; o += e4;
  w->perm = o; o += e4;
  w->nseg = o; o = align_up(o + (size_t)(d + 1) * 8, 256);
  w->nslot = o; o = align_up(o + (size_t)(d + 1) * 8, 256);
  w->temp = o;
  w->temp_bytes = align_up(sort_b > scan_b ? sort_b : scan_b, 256);
  o += w->temp_bytes;
  w->total = o;
  return 0;
}

static size_t plan_bytes(int d, long long nnz) {
  return (size_t)(ST_N + 2 * ((size_t)d + 1)) * 8 + (size_t)seg_cap(d, nnz) * 4;
}

static int grid_for(long long work, int per_cta, int cap) {
  long long g = (work + per_cta - 1) / per_cta;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

// ---------------------------------------------------------------------------------------------------------------------
// column pass
// ---------------------------------------------------------------------------------------------------------------------
struct ColArgs {
  const long long* colptr;
  const int* rows;
  const void* vals;
  int d;
  const long long* plan;
  const double* v1;
  const double* v2;    // or null
  double* out1;        // [d]
  double* out2;        // [d] (with v2)
  double* slot;        // [seg_cap][2]
  unsigned* ticket;    // [d], zero
  int first;
};

template <typename T>
__global__ void __launch_bounds__(kThreads) csc_matvec_kernel(ColArgs a) {
  const int lane = threadIdx.x & 31;
  const long long* seg_off = a.plan + ST_N;
  const int* seg_col = reinterpret_cast<const int*>(a.plan + ST_N + 2 * ((long long)a.d + 1));
  const long long T_ = a.plan[ST_SEGS];
  const T* vals = reinterpret_cast<const T*>(a.vals);
  const bool two = a.v2 != nullptr;
  const long long nw = ((long long)gridDim.x * kThreads) >> 5;
#pragma unroll 1
  for (long long t = ((long long)blockIdx.x * kThreads + threadIdx.x) >> 5; t < T_; t += nw) {
    const int j = seg_col[t];
    const long long s0 = seg_off[j], ns = seg_off[j + 1] - s0;
    const long long e0 = a.colptr[j] + (t - s0) * SEG;
    const long long e1 = min(a.colptr[j + 1], e0 + SEG);
    double p1 = 0.0, p2 = 0.0;
#pragma unroll 4
    for (long long e = e0 + lane; e < e1; e += 32) {
      const int r = a.rows[e];
      const double x = to_f64(vals[e]);
      p1 = fma(a.v1[r], x, p1);
      if (two) p2 = fma(a.v2[r], x, p2);
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      p1 += __shfl_xor_sync(0xffffffffu, p1, off);
      p2 += __shfl_xor_sync(0xffffffffu, p2, off);
    }
    if (ns > 1) {
      if (lane == 0) {
        a.slot[2 * t] = p1;
        a.slot[2 * t + 1] = p2;
      }
      if (!last_warp(a.ticket + j, (unsigned)ns)) continue;
      p1 = p2 = 0.0;                                 // the slots of column j in segment order: lane-strided, then the tree
      for (long long u = lane; u < ns; u += 32) {
        p1 += __ldcg(a.slot + 2 * (s0 + u));
        p2 += __ldcg(a.slot + 2 * (s0 + u) + 1);
      }
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) {
        p1 += __shfl_xor_sync(0xffffffffu, p1, off);
        p2 += __shfl_xor_sync(0xffffffffu, p2, off);
      }
      if (lane == 0) a.ticket[j] = 0u;
    }
    if (lane == 0) {
      a.out1[j] = a.first ? p1 : a.out1[j] + p1;
      if (two) a.out2[j] = a.first ? p2 : a.out2[j] + p2;
    }
  }
}

static size_t matvec_ws(int d, long long nnz) {
  return align_up((size_t)seg_cap(d, nnz) * 16, 256) + align_up((size_t)d * 4, 256);
}

// ---------------------------------------------------------------------------------------------------------------------
// Gram
// ---------------------------------------------------------------------------------------------------------------------
struct GramArgs {
  const long long* crow;
  const long long* col;
  const void* val;
  const long long* colptr;
  const int* rows;
  const void* vals;
  int d;
  const long long* plan;
  const double* w;
  double* gram;      // [d][d]
  double* slot;      // [slots][d]
  unsigned* ticket;  // [d], zero
  int first;
};

template <typename T>
__global__ void __launch_bounds__(kThreads) gram_csr_kernel(GramArgs a) {
  extern __shared__ double s_row[];              // [warps][d]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, W = blockDim.x >> 5;
  const int d = a.d;
  const long long* seg_off = a.plan + ST_N;
  const long long* gseg_off = seg_off + d + 1;
  const int* seg_col = reinterpret_cast<const int*>(gseg_off + d + 1);
  const long long T_ = a.plan[ST_SEGS];
  const T* val = reinterpret_cast<const T*>(a.val);
  const T* vals = reinterpret_cast<const T*>(a.vals);
  double* mine = s_row + (size_t)warp * d;
#pragma unroll 1
  for (long long t = blockIdx.x; t < T_; t += gridDim.x) {
    const int j = seg_col[t];
    const long long s0 = seg_off[j], ns = seg_off[j + 1] - s0, s = t - s0;
    if (s % GS) continue;                        // uniform over the CTA: t is
    for (int k = tid; k < W * d; k += blockDim.x) s_row[k] = 0.0;
    __syncthreads();
    const long long a0 = a.colptr[j] + s * SEG;
    const long long a1 = min(a.colptr[j + 1], a0 + GS * SEG);
    const long long per = (a1 - a0 + W - 1) / W;
    const long long w0 = a0 + warp * per, w1 = min(a1, w0 + per);
#pragma unroll 1
    for (long long e0 = w0; e0 < w1; e0 += 32) {
      // lane l loads entry e0 + l; the warp then takes the entries one by one, in row order
      long long k0 = 0, k1 = 0;
      double c = 0.0;
      if (e0 + lane < w1) {
        const int i = a.rows[e0 + lane];
        c = a.w[i] * to_f64(vals[e0 + lane]);
        k0 = a.crow[i];
        k1 = a.crow[i + 1];
      }
      const int m = (int)min(32LL, w1 - e0);
      for (int q = 0; q < m; ++q) {
        const double cq = __shfl_sync(0xffffffffu, c, q);
        const long long b0 = __shfl_sync(0xffffffffu, k0, q), b1 = __shfl_sync(0xffffffffu, k1, q);
        for (long long k = b0 + lane; k < b1; k += 32) {
          const long long cc = a.col[k];
          if ((unsigned long long)cc < (unsigned long long)d) mine[cc] += cq * to_f64(val[k]);
        }
        __syncwarp();
      }
    }
    __syncthreads();
    const bool split = ns > GS;
    double* dst = split ? a.slot + (size_t)(gseg_off[j] + s / GS) * d : a.gram + (size_t)j * d;
    for (int k = tid; k < d; k += blockDim.x) {
      double v = 0.0;
      for (int q = 0; q < W; ++q) v += s_row[(size_t)q * d + k];
      dst[k] = (split || a.first) ? v : dst[k] + v;
    }
    if (split) {
      const long long runs = (ns + GS - 1) / GS;
      if (last_block(a.ticket + j, (unsigned)runs)) {
        const double* src = a.slot + (size_t)gseg_off[j] * d;
        double* g = a.gram + (size_t)j * d;
        for (int k = tid; k < d; k += blockDim.x) {
          double v = 0.0;
          for (long long u = 0; u < runs; ++u) v += __ldcg(src + (size_t)u * d + k);
          g[k] = a.first ? v : g[k] + v;
        }
        if (tid == 0) a.ticket[j] = 0u;
      }
    }
    __syncthreads();                             // s_row is cleared for the next run
  }
}

static int gram_warps(int d) {
  int w = kGramSmem / (d * 8);
  return w > kWarps ? kWarps : w;
}

static size_t gram_ws(int d, long long slots) {
  return align_up((size_t)slots * d * 8, 256) + align_up((size_t)d * 4, 256);
}

}  // namespace
}  // namespace bkm

using namespace bkm;

static bool val_dtype_ok(int t) { return t == BKM_F32 || t == BKM_F64; }

extern "C" int bkm_glm_csr_workspace_bytes(int64_t n, size_t* out) {
  if (!out || n < 0) return BKM_EINVAL;
  *out = row_ws(sm_count_or_default());
  return 0;
}

extern "C" int bkm_glm_csr_pass_chunk(const int64_t* crow, const int64_t* col, const void* val, int val_dtype,
                                      int64_t n, int d, int64_t nnz, const double* y, const double* beta, int family,
                                      int mode, double* r, double* w, double* grad, double* hrow, void* out,
                                      void* workspace, size_t ws_bytes, int flags, void* stream) {
  if (n < 0 || d <= 0 || nnz < 0 || !beta || !crow || family < 0 || family > 2 || mode < GLM_GRAD ||
      mode > GLM_LABEL)
    return BKM_EINVAL;
  if (nnz > 0 && (!col || !val)) return BKM_EINVAL;
  if (!val_dtype_ok(val_dtype)) return BKM_EDTYPE;
  const bool accumulate = mode == GLM_GRAD || mode == GLM_NEWTON;
  if (accumulate && (!grad || !workspace || (n > 0 && (!y || !r)))) return BKM_EINVAL;
  if (mode == GLM_NEWTON && (!hrow || (n > 0 && !w))) return BKM_EINVAL;
  if (!accumulate && n > 0 && !out) return BKM_EINVAL;
  if (!accumulate && n == 0) return 0;
  const int sms = sm_count_or_default();
  const int G = row_group(n, nnz);
  const int grid = row_grid(n, G, sms);
  cudaStream_t s = (cudaStream_t)stream;
  RowArgs a;
  a.crow = reinterpret_cast<const long long*>(crow);
  a.col = reinterpret_cast<const long long*>(col);
  a.val = val; a.n = n; a.d = d; a.y = y; a.beta = beta; a.family = family; a.mode = mode;
  a.r = r; a.w = w; a.grad = grad; a.hrow = hrow; a.out = out;
  a.first = (flags & BKM_FLAG_FIRST_CHUNK) ? 1 : 0;
  a.part = nullptr;
  a.ticket = nullptr;
  if (accumulate) {
    const size_t need = row_ws(sms);
    if (ws_bytes < need) return BKM_EWORKSPACE;
    BKM_CUDA_TRY(carve_partials(workspace, need, &a.part, &a.ticket, s));
  }
  if (val_dtype == BKM_F32) return launch_row<float>(a, G, grid, s);
  return launch_row<double>(a, G, grid, s);
}

extern "C" int bkm_csr_transpose_workspace_bytes(int64_t n, int d, int64_t nnz, size_t* ws_bytes,
                                                 size_t* plan_bytes_out) {
  if (!ws_bytes || !plan_bytes_out || n < 0 || d <= 0 || nnz < 0) return BKM_EINVAL;
  if (n >= INT32_MAX || nnz >= INT32_MAX) return BKM_EUNSUPPORTED;
  TransposeWs w;
  const int rc = transpose_ws(nnz, d, &w);
  if (rc) return rc;
  *ws_bytes = w.total;
  *plan_bytes_out = plan_bytes(d, nnz);
  return 0;
}

extern "C" int bkm_csr_transpose_chunk(const int64_t* crow, const int64_t* col, const void* val, int val_dtype,
                                       int64_t n, int d, int64_t nnz, int64_t* colptr, int32_t* rows, void* vals,
                                       int64_t* plan, size_t plan_bytes_, void* workspace, size_t ws_bytes,
                                       void* stream) {
  if (n < 0 || d <= 0 || nnz < 0 || !crow || !colptr || !plan || !workspace) return BKM_EINVAL;
  if (nnz > 0 && (!col || !val || !rows || !vals)) return BKM_EINVAL;
  if (n == 0 && nnz != 0) return BKM_EINVAL;
  if (!val_dtype_ok(val_dtype)) return BKM_EDTYPE;
  if (n >= INT32_MAX || nnz >= INT32_MAX) return BKM_EUNSUPPORTED;
  if (plan_bytes_ < plan_bytes(d, nnz)) return BKM_EWORKSPACE;
  TransposeWs w;
  int rc = transpose_ws(nnz, d, &w);
  if (rc) return rc;
  if (ws_bytes < w.total) return BKM_EWORKSPACE;
  cudaStream_t s = (cudaStream_t)stream;
  unsigned char* ws = reinterpret_cast<unsigned char*>(workspace);
  int* erow = reinterpret_cast<int*>(ws + w.erow);
  unsigned* key = reinterpret_cast<unsigned*>(ws + w.key);
  unsigned* key_s = reinterpret_cast<unsigned*>(ws + w.key_s);
  int* idx = reinterpret_cast<int*>(ws + w.idx);
  int* perm = reinterpret_cast<int*>(ws + w.perm);
  long long* nseg = reinterpret_cast<long long*>(ws + w.nseg);
  long long* nslot = reinterpret_cast<long long*>(ws + w.nslot);
  long long* status = reinterpret_cast<long long*>(plan);
  long long* seg_off = status + ST_N;
  long long* gseg_off = seg_off + d + 1;
  int* seg_col = reinterpret_cast<int*>(gseg_off + d + 1);
  const long long* cr = reinterpret_cast<const long long*>(crow);
  const int sms = sm_count_or_default();
  BKM_CUDA_TRY(cudaMemsetAsync(status, 0, ST_N * 8, s));
  if (n > 0) {
    expand_kernel<<<grid_for(n, kWarps, 16 * sms), kThreads, 0, s>>>(cr, reinterpret_cast<const long long*>(col), n, d,
                                                                      nnz, erow, key, idx, status);
    BKM_CUDA_TRY(cudaGetLastError());
    note_launch();
  }
  if (nnz > 0) {
    int bits = 1;
    while (bits < 32 && (1LL << bits) < (long long)d) ++bits;
    size_t tb = w.temp_bytes;
    BKM_CUDA_TRY(cub::DeviceRadixSort::SortPairs(ws + w.temp, tb, key, key_s, idx, perm, (int)nnz, 0, bits, s));
    note_launch();
  }
  const int gg = grid_for(nnz + 1, kThreads, 16 * sms);
  if (val_dtype == BKM_F32)
    gather_kernel<float><<<gg, kThreads, 0, s>>>(key_s, perm, erow, reinterpret_cast<const float*>(val), nnz, d,
                                                 reinterpret_cast<long long*>(colptr), rows,
                                                 reinterpret_cast<float*>(vals));
  else
    gather_kernel<double><<<gg, kThreads, 0, s>>>(key_s, perm, erow, reinterpret_cast<const double*>(val), nnz, d,
                                                  reinterpret_cast<long long*>(colptr), rows,
                                                  reinterpret_cast<double*>(vals));
  BKM_CUDA_TRY(cudaGetLastError());
  const int gd = (d + kThreads) / kThreads;
  count_kernel<<<gd, kThreads, 0, s>>>(reinterpret_cast<const long long*>(colptr), d, nseg, nslot, status);
  BKM_CUDA_TRY(cudaGetLastError());
  size_t tb = w.temp_bytes;
  BKM_CUDA_TRY(cub::DeviceScan::ExclusiveSum(ws + w.temp, tb, nseg, seg_off, d + 1, s));
  tb = w.temp_bytes;
  BKM_CUDA_TRY(cub::DeviceScan::ExclusiveSum(ws + w.temp, tb, nslot, gseg_off, d + 1, s));
  fill_kernel<<<gd, kThreads, 0, s>>>(seg_off, gseg_off, d, seg_col, status);
  BKM_CUDA_TRY(cudaGetLastError());
  note_launch(5);
  return 0;
}

extern "C" int bkm_csc_matvec_workspace_bytes(int d, int64_t nnz, size_t* out) {
  if (!out || d <= 0 || nnz < 0) return BKM_EINVAL;
  *out = matvec_ws(d, nnz);
  return 0;
}

extern "C" int bkm_csc_matvec_chunk(const int64_t* colptr, const int32_t* rows, const void* vals, int val_dtype, int d,
                                    int64_t nnz, const int64_t* plan, const double* v1, const double* v2,
                                    double* out1, double* out2, void* workspace, size_t ws_bytes, int flags,
                                    void* stream) {
  if (d <= 0 || nnz < 0 || !colptr || !plan || !out1 || !workspace) return BKM_EINVAL;
  if (nnz > 0 && (!rows || !vals || !v1)) return BKM_EINVAL;
  if (!val_dtype_ok(val_dtype)) return BKM_EDTYPE;
  if (ws_bytes < matvec_ws(d, nnz)) return BKM_EWORKSPACE;
  cudaStream_t s = (cudaStream_t)stream;
  unsigned char* ws = reinterpret_cast<unsigned char*>(workspace);
  ColArgs a;
  a.colptr = reinterpret_cast<const long long*>(colptr);
  a.rows = rows; a.vals = vals; a.d = d; a.plan = reinterpret_cast<const long long*>(plan);
  a.v1 = v1; a.v2 = v2; a.out1 = out1; a.out2 = out2;
  a.slot = reinterpret_cast<double*>(ws);
  a.ticket = reinterpret_cast<unsigned*>(ws + align_up((size_t)seg_cap(d, nnz) * 16, 256));
  a.first = (flags & BKM_FLAG_FIRST_CHUNK) ? 1 : 0;
  BKM_CUDA_TRY(cudaMemsetAsync(a.ticket, 0, (size_t)d * 4, s));
  const int grid = grid_for(seg_cap(d, nnz), kWarps, 16 * sm_count_or_default());
  if (val_dtype == BKM_F32) csc_matvec_kernel<float><<<grid, kThreads, 0, s>>>(a);
  else csc_matvec_kernel<double><<<grid, kThreads, 0, s>>>(a);
  BKM_CUDA_TRY(cudaGetLastError());
  note_launch();
  return 0;
}

extern "C" int bkm_gram_weighted_csr_workspace_bytes(int d, int64_t n_slots, size_t* out) {
  if (!out || d <= 0 || n_slots < 0) return BKM_EINVAL;
  if (gram_warps(d) < 1) return BKM_EUNSUPPORTED;
  *out = gram_ws(d, n_slots);
  return 0;
}

extern "C" int bkm_gram_weighted_csr_chunk(const int64_t* crow, const int64_t* col, const void* val, int val_dtype,
                                           int64_t n, int d, int64_t nnz, const int64_t* colptr, const int32_t* rows,
                                           const void* vals, const int64_t* plan, int64_t n_slots, const double* w,
                                           double* gram, void* workspace, size_t ws_bytes, int flags, void* stream) {
  if (n < 0 || d <= 0 || nnz < 0 || n_slots < 0 || !crow || !colptr || !plan || !gram || !workspace ||
      (n > 0 && !w))
    return BKM_EINVAL;
  if (nnz > 0 && (!col || !val || !rows || !vals)) return BKM_EINVAL;
  if (!val_dtype_ok(val_dtype)) return BKM_EDTYPE;
  const int W = gram_warps(d);
  if (W < 1) return BKM_EUNSUPPORTED;
  if (ws_bytes < gram_ws(d, n_slots)) return BKM_EWORKSPACE;
  cudaStream_t s = (cudaStream_t)stream;
  unsigned char* ws = reinterpret_cast<unsigned char*>(workspace);
  GramArgs a;
  a.crow = reinterpret_cast<const long long*>(crow);
  a.col = reinterpret_cast<const long long*>(col);
  a.val = val;
  a.colptr = reinterpret_cast<const long long*>(colptr);
  a.rows = rows; a.vals = vals; a.d = d; a.plan = reinterpret_cast<const long long*>(plan);
  a.w = w; a.gram = gram;
  a.slot = reinterpret_cast<double*>(ws);
  a.ticket = reinterpret_cast<unsigned*>(ws + align_up((size_t)n_slots * d * 8, 256));
  a.first = (flags & BKM_FLAG_FIRST_CHUNK) ? 1 : 0;
  BKM_CUDA_TRY(cudaMemsetAsync(a.ticket, 0, (size_t)d * 4, s));
  const int sms = sm_count_or_default();
  const int per_sm = (228 * 1024) / (W * d * 8 + 1024);
  const int grid = grid_for(seg_cap(d, nnz), 1, (per_sm < 1 ? 1 : per_sm) * sms);
  const size_t smem = (size_t)W * d * 8;
  if (val_dtype == BKM_F32) {
    BKM_CUDA_TRY(cudaFuncSetAttribute(gram_csr_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    gram_csr_kernel<float><<<grid, W * 32, smem, s>>>(a);
  } else {
    BKM_CUDA_TRY(cudaFuncSetAttribute(gram_csr_kernel<double>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    gram_csr_kernel<double><<<grid, W * 32, smem, s>>>(a);
  }
  BKM_CUDA_TRY(cudaGetLastError());
  note_launch();
  return 0;
}
