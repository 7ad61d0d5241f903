// bkm_quantile.cu — the passes of QuantileTransformer over row chunks (sm_90a).
//
//   bkm_quantile_hist_chunk + bkm_quantile_select_step   exact order statistics at thousands of target ranks per
//       column (two per reference quantile: floor and floor + 1 of numpy's 'linear' virtual index).  Values map to
//       the order-preserving keys of bkm_select.cuh and are selected 8 bits per round, as for RobustScaler, but the
//       selection works on the column's sorted DISTINCT ranks, whose prefixes after round r form a sorted,
//       duplicate-free "live" list of L_r <= min(T, 256^r) entries:
//         round 0      one 256-bin histogram per column, counted in shared memory;
//         round r >= 1 a CTA takes one 32-byte sector of columns over a row range, stages each column's live list in
//                      shared memory (or reads it from global memory when it does not fit), finds a key's slot by
//                      binary search of key >> (shift + 8) and counts the digit into the global [d][L][256] float64
//                      histogram with an atomic add (integer counts below 2^53: exact in any order).  Keys whose
//                      prefix is not live are skipped.
//         select step one CTA per column: a warp-level scan of each live slot's 256 bins, a binary search per rank
//                      for its digit, the extended prefix, and the next live list by adjacent-unique compaction (the
//                      ranks are sorted, so their prefixes are).  Round 0 first derives the ranks from the column's
//                      non-NaN count and merges the floor / floor + 1 lists into the distinct sorted ranks.
//   bkm_quantile_hist_masked_chunk   the same count with the values equal to a numeric missing value skipped too, so
//       the non-NaN count the select step derives in round 0 is the non-missing count (SimpleImputer's median).
//   bkm_quantile_transform_chunk   per element, in float64: numpy's interp (restated branch by branch, every operation
//       rounded once: no FMA contraction), the reference's +-1e-7 bounds test in X's dtype, then the output
//       distribution's ppf and the clip (forward), or its cdf first (inverse).  A CTA stages one sector of columns'
//       quantiles and the references in shared memory when they fit, else searches them in global memory.
#include "bkm_select.cuh"
#include <math_constants.h>

namespace bkm {
namespace {

// ============================================ selection state ============================================
// Per column: a 16-byte header, then T = 2 n_q records of SelState (the distinct ranks in ascending order; `slot` is
// the rank's index in the live list), then T uint64 live prefixes.  Round 0 uses the live array as scratch for the
// merged rank list.
struct QHead {
  double nvalid;           // non-NaN values of the column
  int R;                   // distinct target ranks
  int L;                   // live prefixes (0: nothing left to count in this column)
};

__host__ __device__ __forceinline__ size_t qstate_stride(int nq) { return 16 + (size_t)2 * nq * 40; }
__host__ __device__ __forceinline__ long long live_cap(int nq, int round) {
  long long c = 1;
  for (int r = 0; r < round && c < 2LL * nq; ++r) c *= 256;
  return c < 2LL * nq ? c : 2LL * nq;
}

struct QCol {
  QHead* head;
  SelState* rec;
  unsigned long long* live;
};
__device__ __forceinline__ QCol qcol(void* state, int nq, int j) {
  unsigned char* b = reinterpret_cast<unsigned char*>(state) + (size_t)j * qstate_stride(nq);
  QCol c;
  c.head = reinterpret_cast<QHead*>(b);
  c.rec = reinterpret_cast<SelState*>(b + 16);
  c.live = reinterpret_cast<unsigned long long*>(b + 16 + (size_t)2 * nq * 32);
  return c;
}

template <typename T> struct KeyOf { typedef unsigned type; };
template <> struct KeyOf<double> { typedef unsigned long long type; };

struct QHistArgs {
  const void* X;
  long long n;
  int d;
  long long ldx;
  const void* state;
  int nq;
  int round;
  int shift;               // bit position of this round's digit
  long long cap;           // slots per column of the histogram: live_cap(nq, round)
  int stage;               // round >= 1: the CTA's live lists are staged in shared memory
  double* hist;            // [d][cap][256]
  double miss;             // MASKED: values equal to it (after widening to float64) are skipped
};

// the index of `v` in the sorted, duplicate-free list[0, L), or -1
template <typename K, typename P>
__device__ __forceinline__ int find_live(P list, int L, K v) {
  int lo = 0, hi = L;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if ((K)list[mid] < v) lo = mid + 1;
    else hi = mid;
  }
  return (lo < L && (K)list[lo] == v) ? lo : -1;
}

template <typename T, bool MASKED>
__global__ void __launch_bounds__(kThreads) quantile_hist_kernel(QHistArgs a) {
  typedef typename KeyOf<T>::type K;
  extern __shared__ __align__(16) unsigned char q_smem[];
  constexpr int CS = 32 / sizeof(T);                         // columns per CTA: one 32-byte sector of a row
  constexpr int RL = kThreads / CS;                          // row lanes
  __shared__ int s_L[CS];
  const int tid = threadIdx.x;
  const int jb = blockIdx.y * CS;
  unsigned* s_hist = reinterpret_cast<unsigned*>(q_smem);   // round 0: [CS][256]
  K* s_live = reinterpret_cast<K*>(q_smem);                 // round >= 1, staged: [CS][cap]
  if (a.round == 0) {
    for (int e = tid; e < CS * 256; e += kThreads) s_hist[e] = 0u;
    if (tid < CS) s_L[tid] = 1;
  } else {
    if (tid < CS) s_L[tid] = jb + tid < a.d ? qcol(const_cast<void*>(a.state), a.nq, jb + tid).head->L : 0;
    __syncthreads();
    if (a.stage) {
      for (int c = 0; c < CS; ++c) {
        if (jb + c >= a.d) break;
        const unsigned long long* g = qcol(const_cast<void*>(a.state), a.nq, jb + c).live;
        for (int e = tid; e < s_L[c]; e += kThreads) s_live[(size_t)c * a.cap + e] = (K)g[e];
      }
    }
  }
  __syncthreads();

  const int c = tid % CS, rl = tid / CS;
  const int j = jb + c;
  const T* X = reinterpret_cast<const T*>(a.X);
  const long long per = (a.n + gridDim.x - 1) / gridDim.x;
  const long long rb = (long long)blockIdx.x * per, re = min(a.n, rb + per);
  const int L = s_L[c];
  const int sh = a.shift;
  const K* my_s = s_live + (size_t)c * a.cap;
  const unsigned long long* my_g = (a.round > 0 && j < a.d) ? qcol(const_cast<void*>(a.state), a.nq, j).live : nullptr;
  double* H = a.hist + (size_t)j * a.cap * 256;
  constexpr int U = 8;
  if (j < a.d && L > 0) {
#pragma unroll 1
    for (long long r = rb + rl; r < re; r += (long long)RL * U) {
      T v[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const long long rr = r + (long long)u * RL;
        if (rr < re) v[u] = X[rr * a.ldx + j];
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (r + (long long)u * RL < re && !is_nan(v[u]) && !(MASKED && widen(v[u]) == a.miss)) {
          const unsigned long long key = radix_key(v[u]);
          const unsigned digit = (unsigned)(key >> sh) & 255u;
          if (a.round == 0) {
            atomicAdd(&s_hist[c * 256 + digit], 1u);
          } else {
            const K high = (K)(key >> (sh + 8));
            const int s = a.stage ? find_live<K>(my_s, L, high) : find_live<K>(my_g, L, high);
            if (s >= 0) atomicAdd(&H[(size_t)s * 256 + digit], 1.0);
          }
        }
      }
    }
  }
  if (a.round == 0) {
    __syncthreads();
    for (int e = tid; e < CS * 256; e += kThreads) {
      const unsigned cnt = s_hist[e];
      const int cc = e >> 8;
      if (cnt && jb + cc < a.d) atomicAdd(&a.hist[(size_t)(jb + cc) * 256 + (e & 255)], (double)cnt);
    }
  }
}

struct QSelectArgs {
  double* hist;            // [d][cap][256]
  void* state;
  const double* qf;        // [nq] ascending quantiles in [0, 1]
  int d, nq, round;
  long long cap;
};

// numpy's 'linear' method: virtual index (m - 1) q; floor, and floor + 1; at or above m - 1 both take the last value
__device__ __forceinline__ double rank_lo(const double* qf, int i, double nv) {
  const double vi = __dmul_rn(nv - 1.0, qf[i]);
  double idx = floor(vi);
  if (vi >= nv - 1.0) idx = nv - 1.0;
  if (vi < 0.0) idx = 0.0;
  return nv > 0.0 ? idx : 0.0;
}
__device__ __forceinline__ double rank_hi(const double* qf, int i, double nv) {
  const double vi = __dmul_rn(nv - 1.0, qf[i]);
  double idx = floor(vi) + 1.0;
  if (vi >= nv - 1.0) idx = nv - 1.0;
  if (vi < 0.0) idx = 0.0;
  return nv > 0.0 ? idx : 0.0;
}

// Position of each thread's flag among the CTA's set flags (exclusive), and their total.  Every thread calls it.
__device__ __forceinline__ int block_flag_rank(bool f, int* s_warp, int* total) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const unsigned b = __ballot_sync(0xffffffffu, f);
  if (lane == 0) s_warp[w] = __popc(b);
  __syncthreads();
  int off = 0, tot = 0;
  for (int i = 0; i < nw; ++i) {
    const int c = s_warp[i];
    off += i < w ? c : 0;
    tot += c;
  }
  __syncthreads();
  *total = tot;
  return off + __popc(b & ((1u << lane) - 1u));
}

__global__ void __launch_bounds__(kThreads) quantile_select_kernel(QSelectArgs a) {
  __shared__ int s_warp[kThreads / 32];
  __shared__ double s_red[kThreads / 32];
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int j = blockIdx.x;
  QCol col = qcol(a.state, a.nq, j);
  double* h = a.hist + (size_t)j * a.cap * 256;
  const int T = 2 * a.nq;

  if (a.round == 0) {
    // the column's non-NaN count: the sum of its 256 bins (integers, exact in any order)
    double v = h[tid];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) s_red[w] = v;
    __syncthreads();
    double nv = 0.0;
    for (int i = 0; i < kThreads / 32; ++i) nv += s_red[i];
    // merge the floor list A and the floor + 1 list B (both ascending) into the scratch, ties A first
    double* merged = reinterpret_cast<double*>(col.live);
    for (int t = tid; t < T; t += kThreads) {
      const int i = t >> 1;
      const bool is_b = t & 1;
      const double r = is_b ? rank_hi(a.qf, i, nv) : rank_lo(a.qf, i, nv);
      int lo = 0, hi = a.nq;       // A: count B_k < r; B: count A_k <= r
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        const bool left = is_b ? rank_lo(a.qf, mid, nv) <= r : rank_hi(a.qf, mid, nv) < r;
        if (left) lo = mid + 1;
        else hi = mid;
      }
      merged[i + lo] = r;
    }
    __syncthreads();
    int R = 0;
    for (int base = 0; base < T; base += kThreads) {
      const int t = base + tid;
      const bool f = t < T && (t == 0 || merged[t] != merged[t - 1]);
      const double r = t < T ? merged[t] : 0.0;
      int tot;
      const int pos = block_flag_rank(f, s_warp, &tot);      // synchronises: every read above precedes the writes
      if (f) {
        SelState s;
        s.prefix = 0ull; s.rank = r; s.nvalid = nv; s.slot = 0; s.pad = 0;
        col.rec[R + pos] = s;
      }
      R += tot;
    }
    if (tid == 0) {
      col.head->nvalid = nv;
      col.head->R = R;
      col.head->L = nv > 0.0 ? 1 : 0;
    }
    __syncthreads();
  }

  const QHead hd = *col.head;
  __syncthreads();
  if (hd.L == 0) return;

  // inclusive scan of each live slot's 256 bins: a warp per slot, 8 bins per lane
  for (int s = w; s < hd.L; s += kThreads / 32) {
    double* hs = h + (size_t)s * 256 + lane * 8;
    double v[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = hs[k];
#pragma unroll
    for (int k = 1; k < 8; ++k) v[k] += v[k - 1];
    double run = v[7];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const double up = __shfl_up_sync(0xffffffffu, run, o);
      if (lane >= o) run += up;
    }
    const double before = run - v[7];
#pragma unroll
    for (int k = 0; k < 8; ++k) hs[k] = v[k] + before;
  }
  __syncthreads();

  // each distinct rank: the first bin whose inclusive count exceeds it holds the rank's digit
  for (int i = tid; i < hd.R; i += kThreads) {
    SelState s = col.rec[i];
    const double* c = h + (size_t)s.slot * 256;
    int lo = 0, hi = 255;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (c[mid] > s.rank) hi = mid;
      else lo = mid + 1;
    }
    s.rank -= lo > 0 ? c[lo - 1] : 0.0;
    s.prefix = (s.prefix << 8) | (unsigned long long)lo;
    col.rec[i] = s;
  }
  __syncthreads();

  // the next live list: the distinct prefixes, in order (equal prefixes are adjacent: the ranks are sorted)
  int L = 0;
  for (int base = 0; base < hd.R; base += kThreads) {
    const int i = base + tid;
    const unsigned long long p = i < hd.R ? col.rec[i].prefix : 0ull;
    const bool f = i < hd.R && (i == 0 || p != col.rec[i - 1].prefix);
    int tot;
    const int pos = block_flag_rank(f, s_warp, &tot);
    if (i < hd.R) {
      // the slot of a rank is the index of its run's first entry: the number of run starts up to it, minus one
      const int incl = L + pos + (f ? 1 : 0);
      col.rec[i].slot = incl - 1;
      if (f) col.live[incl - 1] = p;
    }
    L += tot;
  }
  if (tid == 0) col.head->L = L;
}

// ============================================ transform ============================================
enum { QT_UNIFORM = 0, QT_NORMAL = 1 };

struct QTransformArgs {
  const void* X;
  long long n;
  int d;
  long long ldx;
  const double* qT;        // [d][nq] the quantiles of each column, ascending
  const double* ref;       // [nq] the references
  int nq;
  int inverse, dist;
  double clip_lo, clip_hi;
  double* out;
  long long ldo;
};

// numpy's interp(x, xp, fp) for one x (numpy/_core/src/multiarray/compiled_base.c, arr_interp): left / right take
// fp[0] / fp[n - 1]; one knot compares; otherwise j = the last knot <= x, the last knot and an exact match return
// fp[j], else slope (x - xp[j]) + fp[j], retried from the right knot when that is NaN, and fp[j] when it is still NaN
// and fp[j] == fp[j + 1].  With REV the knots are -xp[n - 1 - k] and the values -fp[n - 1 - k] (exact negations: the
// descending interpolation of the reference on the same arrays).
template <bool REV, typename P>
__device__ __forceinline__ double np_interp(double x, P xp, P fp, int n) {
#define XP(k) (REV ? -xp[n - 1 - (k)] : xp[(k)])
#define FP(k) (REV ? -fp[n - 1 - (k)] : fp[(k)])
  if (n == 1) return FP(0);           // left, right and the knot's value are all fp[0], for NaN x too
  if (x != x) return x;
  if (x > XP(n - 1)) return FP(n - 1);
  if (x < XP(0)) return FP(0);
  int lo = 0, hi = n;                 // the last k with xp[k] <= x (0 when the knots are NaN, as numpy's search gives
  while (lo < hi) {                   // an interior index there)
    const int mid = (lo + hi) >> 1;
    if (x >= XP(mid)) lo = mid + 1;
    else hi = mid;
  }
  int k = lo - 1;
  if (k < 0) k = 0;
  if (k == n - 1) return FP(k);
  const double xk = XP(k);
  if (xk == x) return FP(k);
  const double xk1 = XP(k + 1), fk = FP(k), fk1 = FP(k + 1);
  const double slope = __ddiv_rn(__dsub_rn(fk1, fk), __dsub_rn(xk1, xk));
  double r = __dadd_rn(__dmul_rn(slope, __dsub_rn(x, xk)), fk);
  if (r != r) {
    r = __dadd_rn(__dmul_rn(slope, __dsub_rn(x, xk1)), fk1);
    if (r != r && fk == fk1) r = fk;
  }
  return r;
#undef XP
#undef FP
}

// the bounds test of the reference in X's dtype: x - 1e-7 < lo, x + 1e-7 > hi (float32 arithmetic for fp32 / bf16
// rows, compared in float64)
__device__ __forceinline__ void bounds(float x, double lo, double hi, bool* below, bool* above) {
  *below = (double)__fsub_rn(x, 1e-7f) < lo;
  *above = (double)__fadd_rn(x, 1e-7f) > hi;
}
__device__ __forceinline__ void bounds(double x, double lo, double hi, bool* below, bool* above) {
  *below = __dsub_rn(x, 1e-7) < lo;
  *above = __dadd_rn(x, 1e-7) > hi;
}
__device__ __forceinline__ float narrow_bounds(float v) { return v; }
__device__ __forceinline__ double narrow_bounds(double v) { return v; }
__device__ __forceinline__ float narrow_bounds(__nv_bfloat16 v) { return __bfloat162float(v); }

// scipy.stats.uniform / norm .ppf and .cdf with loc 0, scale 1 (rv_continuous: the support's ends are placed exactly,
// points outside it give NaN (ppf) or 0 / 1 (cdf))
__device__ __forceinline__ double dist_ppf(int dist, double y) {
  if (!(y >= 0.0 && y <= 1.0)) return CUDART_NAN;
  if (dist == QT_UNIFORM) return y == 0.0 ? 0.0 : y;
  if (y == 0.0) return -CUDART_INF;
  if (y == 1.0) return CUDART_INF;
  return normcdfinv(y);
}
__device__ __forceinline__ double dist_cdf(int dist, double x) {
  if (x != x) return x;
  if (dist == QT_UNIFORM) return x <= 0.0 ? 0.0 : (x >= 1.0 ? 1.0 : x);
  if (x == -CUDART_INF) return 0.0;
  if (x == CUDART_INF) return 1.0;
  return normcdf(x);
}

template <typename T, typename P>
__device__ __forceinline__ double quantile_one(const QTransformArgs& p, T v, P q, P ref) {
  const int nq = p.nq;
  const double x = widen(v);
  if (!p.inverse) {
    bool below, above;
    bounds(narrow_bounds(v), q[0], q[nq - 1], &below, &above);
    const double up = np_interp<false>(x, q, ref, nq);
    const double dn = np_interp<true>(-x, q, ref, nq);
    double y = __dmul_rn(0.5, __dsub_rn(up, dn));
    if (above) y = 1.0;
    if (below) y = 0.0;
    y = dist_ppf(p.dist, y);
    y = y < p.clip_lo ? p.clip_lo : y;               // np.clip: NaN stays NaN
    return y > p.clip_hi ? p.clip_hi : y;
  }
  const double c = dist_cdf(p.dist, x);
  bool below, above;
  bounds(c, 0.0, 1.0, &below, &above);
  double y = np_interp<false>(c, ref, q, nq);
  if (above) y = q[nq - 1];
  if (below) y = q[0];
  return y;
}

template <typename T> struct TCols { static constexpr int value = 32 / sizeof(T) < 8 ? 32 / sizeof(T) : 8; };

template <typename T, bool STAGED>
__global__ void __launch_bounds__(kThreads) quantile_transform_kernel(QTransformArgs p) {
  extern __shared__ __align__(16) unsigned char q_smem[];
  constexpr int CS = TCols<T>::value;                        // columns per CTA
  constexpr int RL = kThreads / CS;
  const int tid = threadIdx.x;
  const int jb = blockIdx.x * CS;                            // the column groups of one row range run side by side
  const int nq = p.nq;
  double* s_ref = reinterpret_cast<double*>(q_smem);         // staged: [nq] references, then [CS][nq] quantiles
  double* s_q = s_ref + nq;
  if (STAGED) {
    for (int e = tid; e < nq; e += kThreads) s_ref[e] = p.ref[e];
    for (int c = 0; c < CS && jb + c < p.d; ++c)
      for (int e = tid; e < nq; e += kThreads) s_q[(size_t)c * nq + e] = p.qT[(size_t)(jb + c) * nq + e];
    __syncthreads();
  }
  const int c = tid % CS, rl = tid / CS;
  const int j = jb + c;
  if (j >= p.d) return;
  const double* q = STAGED ? s_q + (size_t)c * nq : p.qT + (size_t)j * nq;
  const double* ref = STAGED ? s_ref : p.ref;
  const T* X = reinterpret_cast<const T*>(p.X);
  const long long per = (p.n + gridDim.y - 1) / gridDim.y;
  const long long rb = (long long)blockIdx.y * per, re = min(p.n, rb + per);
  constexpr int U = 4;
#pragma unroll 1
  for (long long r = rb + rl; r < re; r += (long long)RL * U) {
    T v[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const long long rr = r + (long long)u * RL;
      if (rr < re) v[u] = X[rr * p.ldx + j];
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const long long rr = r + (long long)u * RL;
      if (rr < re) p.out[rr * p.ldo + j] = quantile_one(p, v[u], q, ref);
    }
  }
}

constexpr size_t kStageBytes = 96 * 1024;    // two CTAs per SM

template <typename T, bool MASKED>
static int launch_qhist(QHistArgs a, int sms, cudaStream_t s) {
  constexpr int CS = 32 / sizeof(T);
  typedef typename KeyOf<T>::type K;
  size_t smem = a.round == 0 ? (size_t)CS * 256 * 4 : 0;
  a.stage = 0;
  if (a.round > 0 && (size_t)CS * a.cap * sizeof(K) <= kStageBytes) {
    a.stage = 1;
    smem = (size_t)CS * a.cap * sizeof(K);
  }
  BKM_CUDA_TRY(cudaFuncSetAttribute(quantile_hist_kernel<T, MASKED>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    (int)kStageBytes));
  const int gy = (a.d + CS - 1) / CS;
  const int per_sm = smem <= 24 * 1024 ? 8 : (smem <= 48 * 1024 ? 4 : 2);
  long long gx = ((long long)per_sm * sms + gy - 1) / gy;
  const long long most = (a.n + (kThreads / CS) * 16 - 1) / ((kThreads / CS) * 16);   // >= 16 rows per thread
  if (gx > most) gx = most;
  if (gx < 1) gx = 1;
  quantile_hist_kernel<T, MASKED><<<dim3((unsigned)gx, (unsigned)gy), kThreads, smem, s>>>(a);
  BKM_CUDA_TRY(cudaGetLastError());
  note_launch();
  return 0;
}

template <typename T>
static int launch_qtransform(const QTransformArgs& p, int sms, cudaStream_t s) {
  constexpr int CS = TCols<T>::value;
  const size_t smem = (size_t)(CS + 1) * p.nq * 8;
  const unsigned gx = (unsigned)((p.d + CS - 1) / CS);
  const bool staged = smem <= kStageBytes;
  const int per_sm = staged ? (smem <= 24 * 1024 ? 8 : (smem <= 48 * 1024 ? 4 : 2)) : 8;
  long long gy = ((long long)per_sm * sms + gx - 1) / gx;
  const long long most = (p.n + (kThreads / CS) * 8 - 1) / ((kThreads / CS) * 8);    // >= 8 rows per thread
  if (gy > most) gy = most;
  if (gy > 65535) gy = 65535;
  if (gy < 1) gy = 1;
  if (staged) {
    BKM_CUDA_TRY(cudaFuncSetAttribute(quantile_transform_kernel<T, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)kStageBytes));
    quantile_transform_kernel<T, true><<<dim3(gx, (unsigned)gy), kThreads, smem, s>>>(p);
  } else {
    quantile_transform_kernel<T, false><<<dim3(gx, (unsigned)gy), kThreads, 0, s>>>(p);
  }
  BKM_CUDA_TRY(cudaGetLastError());
  note_launch();
  return 0;
}

}  // namespace
}  // namespace bkm

using namespace bkm;

extern "C" int bkm_quantile_state_bytes(int d, int n_q, size_t* out) {
  if (!out || d <= 0 || n_q <= 0) return BKM_EINVAL;
  *out = (size_t)d * qstate_stride(n_q);
  return 0;
}

static int quantile_hist(const void* X, int64_t n, int d, int64_t ldx, int x_dtype, const void* state, int n_q,
                         int round, double* hist, int flags, void* stream, bool masked, double miss) {
  if (n < 0 || d <= 0 || ldx < d || !state || !hist || n_q <= 0 || round < 0) return BKM_EINVAL;
  if (n > 0 && !X) return BKM_EINVAL;
  if (!dtype_ok(x_dtype)) return BKM_EDTYPE;
  const int bits = (int)elem_size(x_dtype) * 8;
  if (round >= bits / 8) return BKM_EINVAL;
  cudaStream_t s = (cudaStream_t)stream;
  const long long cap = live_cap(n_q, round);
  if (flags & BKM_FLAG_FIRST_CHUNK) BKM_CUDA_TRY(cudaMemsetAsync(hist, 0, (size_t)d * cap * 256 * 8, s));
  if (n == 0) return 0;
  int sms = 0;
  const int rc = sm_count(&sms);
  if (rc) return rc;
  QHistArgs a;
  a.X = X; a.n = n; a.d = d; a.ldx = ldx; a.state = state; a.nq = n_q; a.round = round;
  a.shift = bits - 8 * (round + 1);
  a.cap = cap;
  a.stage = 0;
  a.hist = hist;
  a.miss = miss;
  if (masked) {
    if (x_dtype == BKM_F32) return launch_qhist<float, true>(a, sms, s);
    if (x_dtype == BKM_F64) return launch_qhist<double, true>(a, sms, s);
    return launch_qhist<__nv_bfloat16, true>(a, sms, s);
  }
  if (x_dtype == BKM_F32) return launch_qhist<float, false>(a, sms, s);
  if (x_dtype == BKM_F64) return launch_qhist<double, false>(a, sms, s);
  return launch_qhist<__nv_bfloat16, false>(a, sms, s);
}

extern "C" int bkm_quantile_hist_chunk(const void* X, int64_t n, int d, int64_t ldx, int x_dtype, const void* state,
                                       int n_q, int round, double* hist, int flags, void* stream) {
  return quantile_hist(X, n, d, ldx, x_dtype, state, n_q, round, hist, flags, stream, false, 0.0);
}

extern "C" int bkm_quantile_hist_masked_chunk(const void* X, int64_t n, int d, int64_t ldx, int x_dtype,
                                              double miss_value, const void* state, int n_q, int round, double* hist,
                                              int flags, void* stream) {
  if (miss_value != miss_value) return BKM_EINVAL;          // NaN is skipped by bkm_quantile_hist_chunk already
  return quantile_hist(X, n, d, ldx, x_dtype, state, n_q, round, hist, flags, stream, true, miss_value);
}

extern "C" int bkm_quantile_select_step(double* hist, void* state, int d, int n_q, int round, int x_dtype,
                                        const double* qf, void* stream) {
  if (!hist || !state || !qf || d <= 0 || n_q <= 0 || round < 0) return BKM_EINVAL;
  if (!dtype_ok(x_dtype)) return BKM_EDTYPE;
  const int bits = (int)elem_size(x_dtype) * 8;
  if (round >= bits / 8) return BKM_EINVAL;
  QSelectArgs a;
  a.hist = hist; a.state = state; a.qf = qf; a.d = d; a.nq = n_q; a.round = round; a.cap = live_cap(n_q, round);
  quantile_select_kernel<<<d, kThreads, 0, (cudaStream_t)stream>>>(a);
  BKM_CUDA_TRY(cudaGetLastError());
  note_launch();
  return 0;
}

extern "C" int bkm_quantile_transform_chunk(const void* X, int64_t n, int d, int64_t ldx, int x_dtype,
                                            const double* quantiles, const double* references, int n_q, int inverse,
                                            int distribution, double clip_lo, double clip_hi, double* out,
                                            int64_t ld_out, void* stream) {
  if (n < 0 || d <= 0 || ldx < d || ld_out < d || n_q <= 0 || !quantiles || !references) return BKM_EINVAL;
  if ((inverse != 0 && inverse != 1) || (distribution != QT_UNIFORM && distribution != QT_NORMAL)) return BKM_EINVAL;
  if (n > 0 && (!X || !out)) return BKM_EINVAL;
  if (!dtype_ok(x_dtype)) return BKM_EDTYPE;
  if (n == 0) return 0;
  int sms = 0;
  const int rc = sm_count(&sms);
  if (rc) return rc;
  QTransformArgs p;
  p.X = X; p.n = n; p.d = d; p.ldx = ldx; p.qT = quantiles; p.ref = references; p.nq = n_q; p.inverse = inverse;
  p.dist = distribution; p.clip_lo = clip_lo; p.clip_hi = clip_hi; p.out = out; p.ldo = ld_out;
  cudaStream_t s = (cudaStream_t)stream;
  if (x_dtype == BKM_F32) return launch_qtransform<float>(p, sms, s);
  if (x_dtype == BKM_F64) return launch_qtransform<double>(p, sms, s);
  return launch_qtransform<__nv_bfloat16>(p, sms, s);
}
