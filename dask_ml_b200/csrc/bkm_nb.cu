// bkm_nb.cu — the passes of GaussianNB over row chunks (sm_90a).
//
//   bkm_class_moments_chunk  mode 0: sums[c][j] (+)= sum_{i: y_i = c} x_ij,  counts[c] (+)= #{i: y_i = c}
//                            mode 1: sums[c][j] (+)= sum_{i: y_i = c} (x_ij - theta_cj)^2
//   bkm_nb_jll_chunk         jll_ic = logc_c - 1/2 sum_j (x_ij - theta_cj)^2 w_cj, then per row either the arg-max
//                            (labels) or jll - logsumexp(jll) (float64 log-probabilities, optionally exponentiated)
//
// and the dense passes of PartialMultinomialNB / PartialBernoulliNB:
//
//   bkm_class_counts_chunk   FC[c][j] (+)= sum_{i: y_i = c} w_i f(x_ij),  CC[c] (+)= sum_{i: y_i = c} w_i  (w_i = 1 without
//                            weights; f the identity, or x > t when binarising): the moments kernel's mode 0
//   bkm_nb_linear_jll_chunk  jll_ic = b_c + sum_j f(x_ij) W_cj in float64 on the fp64 tensor cores, then per row the
//                            arg-max (labels) and / or jll, jll - logsumexp(jll) or its exp (float64, any row pitch)
//
// Moments.  A CTA owns one row split and one (class slice x feature slice) of the accumulators.  Its threads are
// `groups` row groups of `fs` feature lanes; every group has its own float64 accumulator copy in shared memory, so the
// lane of feature j in group g is the only writer of acc[g][c][j]: no atomics, and the order of its additions is the
// row order.  Each 256-row tile is first compacted to the rows whose class lies in the CTA's slice (a ballot in row
// order); group g then takes members g, g + groups, ...  Classes beyond one slice's budget go to further slices: a
// slice CTA reads only the class indices of rows outside it, so X is still read once.  At the end the groups are added
// in group order into the split's partial, and a second launch adds the split partials in split order.  Two calls with
// the same inputs therefore give the same bits.
//
// Log-likelihood.  One thread per row, 128-row tiles.  The tile's rows are staged in shared memory (converted to the
// compute type: fp32 for fp32 / bf16 rows, float64 for float64 rows) and, for d <= 64, held in registers.  theta and w
// are staged as (theta, w) pairs: all K classes at once while they fit (resident for the CTA's lifetime), otherwise
// class blocks re-staged per tile.  For d > 64 the features go in 32-wide chunks with per-class partial sums in shared
// memory.  Each thread walks the classes in index order and the features in index order, so the arithmetic does not
// depend on the blocking.  The sum is taken in direct form, fma((x - theta) w, x - theta, acc), never expanded.
// fp32 rows whose best class is not ahead of every other class by more than the error bound E (DESIGN.md, A21) are
// re-decided in float64 by the same thread, with the float64 path's exact arithmetic.
//
// Linear log-likelihood.  One CTA owns a 64-row tile and all K classes; it walks the classes in blocks of 16, 32 or 64
// columns (chosen from K as bkm_project_chunk chooses them, so a small K pads no columns).  For each block the rows
// and W are staged 32 features at a time, widened to float64 (f(x) applied) in shared memory, and multiplied with
// DMMA.16x8x16 as in bkm_project_chunk: the products of fp32 and bf16 rows are exact, and 0 (-inf) stays NaN as in
// numpy's BLAS product.  After each block, b is added and thread r folds row r's block into its running arg-max (the
// first maximum, the first NaN, as np.argmax) and running logsumexp, in class order.  The raw block goes out at once;
// normalised outputs are rewritten by the CTA after the tile's last block (directly from shared memory when K fits one
// block).
#include "bkm_common.cuh"
#include "bkm_ptx.cuh"
#include <cuda_bf16.h>

namespace bkm {
namespace {

// ------------------------------------------------------------------------------------------------------- moments
constexpr int MT = 256;                       // threads per CTA
constexpr int MR = 256;                       // rows per member tile
constexpr size_t MBUDGET = 96 * 1024;         // accumulator bytes per CTA (two CTAs per SM)

__device__ __forceinline__ double to_f64(float v) { return (double)v; }
__device__ __forceinline__ double to_f64(double v) { return v; }
__device__ __forceinline__ double to_f64(__nv_bfloat16 v) { return (double)__bfloat162float(v); }

struct MomGeom {
  int fs, nf;                 // feature slice width and count
  int groups;                 // row groups per CTA
  int ks, nk;                 // class slice size and count
  int splits;                 // row splits
  long long rows_per_split;   // a multiple of MR
  size_t smem;
  size_t off_part, off_cpart, total;
};

static MomGeom mom_geom(long long n, int d, int K, int sms) {
  MomGeom g;
  g.fs = d < MT ? d : MT;
  g.nf = (d + g.fs - 1) / g.fs;
  g.groups = MT / g.fs;
  long long ks = (long long)(MBUDGET / ((size_t)g.groups * (g.fs + 1) * 8));
  if (ks < 1) ks = 1;
  g.ks = (int)(ks < K ? ks : K);
  g.nk = (K + g.ks - 1) / g.ks;
  const long long tiles = (n + MR - 1) / MR;
  const long long slices = (long long)g.nk * g.nf;
  long long s = (2LL * sms + slices - 1) / slices;   // about two CTAs per SM in all
  if (s > tiles) s = tiles;
  if (s < 1) s = 1;
  g.rows_per_split = ((tiles + s - 1) / s) * MR;
  if (g.rows_per_split < MR) g.rows_per_split = MR;
  g.splits = n > 0 ? (int)((n + g.rows_per_split - 1) / g.rows_per_split) : 0;
  g.smem = (size_t)g.groups * g.ks * (g.fs + 1) * 8 + (size_t)MR * sizeof(int2);
  const size_t sp = g.splits > 0 ? (size_t)g.splits : 1;
  size_t o = 0;
  g.off_part = o;  o = align_up(o + sp * K * d * 8, 256);
  g.off_cpart = o; o = align_up(o + sp * K * 8, 256);
  g.total = o;
  return g;
}

struct MomArgs {
  const void* X;
  long long n;
  int d;
  long long ldx;
  const int32_t* cls;
  int K;
  int mode;
  const double* theta;
  double* part;
  double* cpart;
  int fs, groups, ks, nk;
  long long rows_per_split;
  const double* w;          // COUNTS: the row weights [n], nullable
  double thr;               // COUNTS with bin: f(x) = x > thr
  int bin;
};

// COUNTS (bkm_class_counts_chunk): mode 0 with f(x) w_i in place of x and w_i in place of 1
template <typename T, bool COUNTS = false>
__global__ void __launch_bounds__(MT) moments_kernel(MomArgs a) {
  extern __shared__ __align__(16) unsigned char smem[];
  __shared__ int wcount[MT / 32];
  const int G = a.groups, KS = a.ks, FS = a.fs;
  double* acc = reinterpret_cast<double*>(smem);                      // [G][KS][FS]
  double* cnt = acc + (size_t)G * KS * FS;                            // [G][KS]
  int2* mem = reinterpret_cast<int2*>(cnt + (size_t)G * KS);          // [MR] (row in tile, class - k0)

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int split = blockIdx.x;
  const int ksl = blockIdx.y % a.nk, fsl = blockIdx.y / a.nk;
  const int k0 = ksl * KS, kw = min(KS, a.K - k0);
  const int f0 = fsl * FS, fw = min(FS, a.d - f0);
  const int g = tid / FS, f = tid - g * FS;
  const bool act = g < G && f < fw;
  const bool counter = a.mode == 0 && fsl == 0;

  for (int e = tid; e < G * KS * FS; e += MT) acc[e] = 0.0;
  for (int e = tid; e < G * KS; e += MT) cnt[e] = 0.0;

  const long long rb = (long long)split * a.rows_per_split;
  const long long re = min(a.n, rb + a.rows_per_split);
  const T* X = reinterpret_cast<const T*>(a.X);
  double* A = acc + (size_t)g * KS * FS + f;
  double* C = cnt + (size_t)g * KS;

#pragma unroll 1
  for (long long r0 = rb; r0 < re; r0 += MR) {
    const int rows = (int)min((long long)MR, re - r0);
    int c = -1;
    if (tid < rows) c = a.cls[r0 + tid] - k0;
    const bool in = tid < rows && c >= 0 && c < kw;
    const unsigned b = __ballot_sync(0xffffffffu, in);
    __syncthreads();                            // the previous tile's members are consumed
    if (lane == 0) wcount[warp] = __popc(b);
    __syncthreads();
    int base = 0, total = 0;
#pragma unroll
    for (int w = 0; w < MT / 32; ++w) {
      const int v = wcount[w];
      base += w < warp ? v : 0;
      total += v;
    }
    if (in) mem[base + __popc(b & ((1u << lane) - 1u))] = make_int2(tid, c);
    __syncthreads();
    if (act) {
#pragma unroll 4
      for (int m = g; m < total; m += G) {
        const int2 e = mem[m];
        const double x = to_f64(X[(r0 + e.x) * a.ldx + f0 + f]);
        double v = x;
        if (COUNTS) {
          if (a.bin) v = x > a.thr ? 1.0 : 0.0;
          const double wi = a.w ? __ldg(a.w + r0 + e.x) : 1.0;
          A[e.y * FS] += v * wi;
          if (counter && f == 0) C[e.y] += wi;
          continue;
        }
        if (a.mode != 0) {
          const double t = x - __ldg(a.theta + (size_t)(k0 + e.y) * a.d + f0 + f);
          v = t * t;
        }
        A[e.y * FS] += v;
        if (counter && f == 0) C[e.y] += 1.0;
      }
    }
  }
  __syncthreads();

  // ---- this CTA's slice of the split partial: the groups added in group order ----
  double* P = a.part + (size_t)split * a.K * a.d;
  for (int e = tid; e < kw * fw; e += MT) {
    const int cc = e / fw, ff = e - cc * fw;
    double v = 0.0;
    for (int q = 0; q < G; ++q) v += acc[((size_t)q * KS + cc) * FS + ff];
    P[(size_t)(k0 + cc) * a.d + f0 + ff] = v;
  }
  if (counter) {
    for (int cc = tid; cc < kw; cc += MT) {
      double v = 0.0;
      for (int q = 0; q < G; ++q) v += cnt[(size_t)q * KS + cc];
      a.cpart[(size_t)split * a.K + k0 + cc] = v;
    }
  }
}

// the split partials added in split order; overwrite (first) or accumulate
__global__ void __launch_bounds__(256) moments_fold_kernel(const double* part, const double* cpart, int splits, int K,
                                                           int d, int mode, double* sums, double* counts, int first) {
  const long long kd = (long long)K * d;
  const long long total = kd + (mode == 0 ? K : 0);
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total;
       e += (long long)gridDim.x * blockDim.x) {
    double v = 0.0;
    if (e < kd) {
      for (int s = 0; s < splits; ++s) v += part[(size_t)s * kd + e];
      sums[e] = first ? v : sums[e] + v;
    } else {
      const long long c = e - kd;
      for (int s = 0; s < splits; ++s) v += cpart[(size_t)s * K + c];
      counts[c] = first ? v : counts[c] + v;
    }
  }
}

// ------------------------------------------------------------------------------------------- log-likelihood
constexpr int JT = 128;                       // threads = rows per tile
constexpr int JC = 32;                        // feature chunk of the d > 64 path
constexpr size_t JBUDGET = 100 * 1024;        // shared memory per CTA

template <typename TC> struct Pair;
template <> struct Pair<float> { using type = float2; };
template <> struct Pair<double> { using type = double2; };

__device__ __forceinline__ float to_tc(float v, float) { return v; }
__device__ __forceinline__ float to_tc(__nv_bfloat16 v, float) { return __bfloat162float(v); }
__device__ __forceinline__ double to_tc(double v, double) { return v; }

// acc + (x - t)^2 w in direct form; explicit rounding so that no contraction differs between call sites
__device__ __forceinline__ float term(float acc, float x, float t, float w) {
  const float u = __fsub_rn(x, t);
  return __fmaf_rn(__fmul_rn(u, w), u, acc);
}
__device__ __forceinline__ double term(double acc, double x, double t, double w) {
  const double u = __dsub_rn(x, t);
  return __fma_rn(__dmul_rn(u, w), u, acc);
}

struct JllArgs {
  const void* X;
  long long n;
  int d;
  long long ldx;
  const double* theta;      // [K][d]
  const double* w;          // [K][d]
  const double* logc;       // [K]
  int K;
  int kb;                   // classes per block (K: resident)
  int dp;                   // staged row width of theta / w (FC for d <= 64, JC otherwise)
  int32_t* labels;          // nullable
  double* out;              // nullable
  long long ldo;
  int exp_out;
  int* n_deferred;          // nullable
  int recheck;
  float tau;                // (d + 8) 2^-25
};

// float64 arg-max of one row with the float64 path's arithmetic (features, then classes, in index order)
template <typename T>
__device__ __noinline__ int recheck_row(const T* xr, int d, const double* theta, const double* w, const double* logc, int K) {
  double best = -INFINITY;
  int bi = 0, nani = -1;
  for (int k = 0; k < K; ++k) {
    double s = 0.0;
    const double* tk = theta + (size_t)k * d;
    const double* wk = w + (size_t)k * d;
    for (int j = 0; j < d; ++j) s = term(s, to_f64(xr[j]), __ldg(tk + j), __ldg(wk + j));
    const double v = __fma_rn(-0.5, s, __ldg(logc + k));
    if (isnan(v)) {
      if (nani < 0) nani = k;
    } else if (v > best) {
      best = v;
      bi = k;
    }
  }
  return nani >= 0 ? nani : bi;
}

struct JllSmem {
  size_t off_tw, off_big, off_c, off_xs, off_sacc, off_ob, off_lse, total;
};

template <typename TC>
static JllSmem jll_smem(int kb, int dp, int fc, bool ch, bool out) {
  JllSmem L;
  size_t o = 0;
  L.off_tw = o;   o = align_up(o + (size_t)kb * dp * 2 * sizeof(TC), 16);
  L.off_big = o;  o = align_up(o + (size_t)kb * 4, 16);
  L.off_c = o;    o = align_up(o + (size_t)kb * 8, 16);
  L.off_xs = o;   o = align_up(o + (size_t)JT * (fc + 1) * sizeof(TC), 16);
  L.off_sacc = o; o = align_up(o + (ch ? (size_t)kb * JT * sizeof(TC) : 0), 16);
  L.off_ob = o;   o = align_up(o + (out ? (size_t)JT * (kb + 1) * 8 : 0), 16);
  L.off_lse = o;  o = align_up(o + (out ? (size_t)JT * 8 : 0), 16);
  L.total = o;
  return L;
}

// FC: features held in registers per pass; CH: d > FC, features in FC-wide chunks with partial sums in shared memory
template <typename T, typename TC, int FC, bool CH>
__global__ void __launch_bounds__(JT, 4) jll_kernel(JllArgs a, JllSmem L) {
  using P2 = typename Pair<TC>::type;
  constexpr bool F32 = sizeof(TC) == 4;
  extern __shared__ __align__(16) unsigned char smem[];
  P2* tw = reinterpret_cast<P2*>(smem + L.off_tw);          // [kb][dp] (theta, w)
  float* big = reinterpret_cast<float*>(smem + L.off_big);  // [kb] sum_j w theta^2 (fp32 bound)
  double* cs = reinterpret_cast<double*>(smem + L.off_c);   // [kb] logc
  TC* xs = reinterpret_cast<TC*>(smem + L.off_xs);          // [JT][FC + 1]
  TC* sacc = reinterpret_cast<TC*>(smem + L.off_sacc);      // [kb][JT]
  double* ob = reinterpret_cast<double*>(smem + L.off_ob);  // [JT][kb + 1]
  double* lse_s = reinterpret_cast<double*>(smem + L.off_lse);

  const int tid = threadIdx.x;
  const int d = a.d, K = a.K, KB = a.kb, dp = a.dp;
  const int nblk = (K + KB - 1) / KB;
  const bool resident = nblk == 1;
  const int nch = CH ? (d + FC - 1) / FC : 1;
  const T* X = reinterpret_cast<const T*>(a.X);
  const long long ntiles = (a.n + JT - 1) / JT;
  const bool want_lab = a.labels != nullptr, want_out = a.out != nullptr;

  // stage classes [kb0, kb0 + kw) and features [f0, f0 + dp) of theta / w (zero beyond d), logc, and the fp32 bound's
  // sum_j w theta^2 (over all d features, computed in float64)
  auto stage_classes = [&](int kb0, int f0, bool consts) {
    const int kw = min(KB, K - kb0);
    for (int e = tid; e < KB * dp; e += JT) {
      const int k = e / dp, j = e - k * dp;
      P2 p;
      p.x = 0; p.y = 0;
      if (k < kw && f0 + j < d) {
        p.x = (TC)a.theta[(size_t)(kb0 + k) * d + f0 + j];
        p.y = (TC)a.w[(size_t)(kb0 + k) * d + f0 + j];
      }
      tw[e] = p;
    }
    if (consts) {
      for (int k = tid; k < KB; k += JT) {
        double c = 0.0, bg = 0.0;
        if (k < kw) {
          c = a.logc[kb0 + k];
          if (F32 && want_lab)
            for (int j = 0; j < d; ++j) {
              const double t = a.theta[(size_t)(kb0 + k) * d + j];
              bg += a.w[(size_t)(kb0 + k) * d + j] * t * t;
            }
        }
        cs[k] = c;
        big[k] = (float)bg;
      }
    }
  };
  auto stage_rows = [&](long long r0, int rows, int f0) {
#pragma unroll 4
    for (int e = tid; e < JT * FC; e += JT) {
      const int r = e / FC, j = e - r * FC;
      TC v = 0;
      if (r < rows && f0 + j < d) v = to_tc(X[(r0 + r) * a.ldx + f0 + j], TC());
      xs[r * (FC + 1) + j] = v;
    }
  };

  if (resident && !CH) {
    stage_classes(0, 0, true);
  }

#pragma unroll 1
  for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const long long r0 = tile * JT;
    const int rows = (int)min((long long)JT, a.n - r0);
    const bool live = tid < rows;

    // per-row state: arg-max, the fp32 margin test, the running logsumexp
    double best = -INFINITY, Eb = 0.0, U1 = -INFINITY, U2 = -INFINITY;
    int bi = 0, U1i = -1, nani = -1;
    bool defer = false, anynan = false;
    double m = -INFINITY, ssum = 0.0;

    TC xr[FC];
    if (!CH) {
      __syncthreads();                          // the previous tile is done with xs
      stage_rows(r0, rows, 0);
      __syncthreads();
#pragma unroll
      for (int j = 0; j < FC; ++j) xr[j] = xs[tid * (FC + 1) + j];
    }

#pragma unroll 1
    for (int blk = 0; blk < nblk; ++blk) {
      const int kb0 = blk * KB, kw = min(KB, K - kb0);
#pragma unroll 1
      for (int ch = 0; ch < nch; ++ch) {
        if (CH || !resident) {
          __syncthreads();                      // the previous block / chunk is done with tw, xs, ob
          stage_classes(kb0, ch * FC, ch == 0);
          if (CH) stage_rows(r0, rows, ch * FC);
          __syncthreads();
          if (CH) {
#pragma unroll
            for (int j = 0; j < FC; ++j) xr[j] = xs[tid * (FC + 1) + j];
          }
        }
        const bool last = ch == nch - 1;
#pragma unroll 1
        for (int k = 0; k < kw; ++k) {
          const P2* tk = tw + (size_t)k * dp;
          TC s = (CH && ch > 0) ? sacc[k * JT + tid] : (TC)0;
#pragma unroll
          for (int j = 0; j < FC; ++j) {
            const P2 p = tk[j];
            s = term(s, xr[j], p.x, p.y);
          }
          if (!last) {
            sacc[k * JT + tid] = s;
            continue;
          }
          // ---- epilogue of class kb0 + k ----
          const int kk = kb0 + k;
          const double ck = cs[k];
          const double v = __fma_rn(-0.5, (double)s, ck);
          if (want_lab) {
            if (isnan(v)) {
              if (!F32 || isnan(ck)) {
                if (nani < 0) nani = kk;
              } else {
                defer = true;                   // NaN from the fp32 sum (x not finite, or an fp32 overflow)
              }
            } else {
              if (F32) {
                const float sf = (float)s;
                if (!(fabsf(sf) < INFINITY)) defer = true;
                const double E = (double)(a.tau * (sf + sqrtf(sf * big[k]))) + 0x1p-50 * fabs(v);
                const double U = v + E;
                if (v > best) { best = v; bi = kk; Eb = E; }
                if (U > U1) { U2 = U1; U1 = U; U1i = kk; } else if (U > U2) { U2 = U; }
              } else if (v > best) {
                best = v;
                bi = kk;
              }
            }
          }
          if (want_out) {
            if (isnan(v)) {
              anynan = true;
            } else if (v > m) {
              ssum = ssum * exp(m - v) + 1.0;
              m = v;
            } else if (v != -INFINITY) {
              ssum += exp(v - m);
            }
            ob[tid * (KB + 1) + k] = v;
          }
        }
      }
      if (want_out && nblk > 1) {               // the raw block goes out now; it is normalised after the last block
        __syncthreads();
        for (int e = tid; e < rows * kw; e += JT) {
          const int r = e / kw, k = e - r * kw;
          a.out[(r0 + r) * a.ldo + kb0 + k] = ob[r * (KB + 1) + k];
        }
      }
    }

    // ---- labels ----
    if (want_lab && live) {
      int lab = nani >= 0 ? nani : bi;
      if (F32 && !defer && nani < 0) {
        const double Uo = (U1i == bi) ? U2 : U1;
        if (!(best - Eb > Uo)) defer = true;
      }
      if (F32) {
        const unsigned dm = __ballot_sync(__activemask(), defer);
        if (a.n_deferred && defer && (__ffs(dm) - 1) == (tid & 31)) atomicAdd(a.n_deferred, __popc(dm));
        if (defer && a.recheck) lab = recheck_row(X + (r0 + tid) * a.ldx, d, a.theta, a.w, a.logc, K);
      }
      a.labels[r0 + tid] = lab;
    }

    // ---- log-probabilities: jll - (log sum exp(jll - max) + max), as the reference's logsumexp ----
    if (want_out) {
      const double lse = (anynan || !(fabs(m) < INFINITY)) ? (double)NAN : log(ssum) + m;
      lse_s[tid] = lse;
      __syncthreads();
      if (nblk == 1) {
        for (int e = tid; e < rows * K; e += JT) {
          const int r = e / K, k = e - r * K;
          double o = ob[r * (KB + 1) + k] - lse_s[r];
          if (a.exp_out) o = exp(o);
          a.out[(r0 + r) * a.ldo + k] = o;
        }
      } else {
        for (int e = tid; e < rows * K; e += JT) {
          const int r = e / K, k = e - r * K;
          double* p = a.out + (r0 + r) * a.ldo + k;
          double o = *p - lse_s[r];
          if (a.exp_out) o = exp(o);
          *p = o;
        }
      }
    }
  }
}

template <typename T, bool COUNTS = false>
static int launch_moments(const MomArgs& a, const MomGeom& G, cudaStream_t s) {
  BKM_CUDA_TRY(cudaFuncSetAttribute(moments_kernel<T, COUNTS>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    (int)G.smem));
  moments_kernel<T, COUNTS><<<dim3(G.splits, G.nk * G.nf), MT, G.smem, s>>>(a);
  BKM_CUDA_TRY(cudaGetLastError());
  note_launch();
  return 0;
}

template <typename T, typename TC, int FC, bool CH>
static int launch_jll_fc(JllArgs a, int sms, cudaStream_t s) {
  constexpr size_t es = sizeof(TC);
  const bool out = a.out != nullptr;
  a.dp = FC;
  // classes per block: all K while they fit the budget, else as many as fit
  auto fits = [&](int kb) { return jll_smem<TC>(kb, FC, FC, CH, out).total <= JBUDGET; };
  int kb = a.K;
  if (!fits(kb)) {
    const size_t fixed = jll_smem<TC>(0, FC, FC, CH, out).total + 64;
    const size_t per = (size_t)FC * 2 * es + 12 + (CH ? JT * es : 0) + (out ? JT * 8 : 0);
    kb = (int)((JBUDGET - fixed) / per);
    if (kb < 1) kb = 1;
    while (kb > 1 && !fits(kb)) --kb;
  }
  a.kb = kb;
  const JllSmem L = jll_smem<TC>(kb, FC, FC, CH, out);
  auto kern = jll_kernel<T, TC, FC, CH>;
  BKM_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)L.total));
  int per_sm = 0;
  BKM_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, JT, L.total));
  if (per_sm < 1) per_sm = 1;
  const long long ntiles = (a.n + JT - 1) / JT;
  long long gx = (long long)per_sm * sms;
  if (gx > ntiles) gx = ntiles;
  kern<<<(unsigned)gx, JT, L.total, s>>>(a, L);
  BKM_CUDA_TRY(cudaGetLastError());
  note_launch();
  return 0;
}

template <typename T>
static int launch_jll_f32(const JllArgs& a, int sms, cudaStream_t s) {
  if (a.d <= 8) return launch_jll_fc<T, float, 8, false>(a, sms, s);
  if (a.d <= 16) return launch_jll_fc<T, float, 16, false>(a, sms, s);
  if (a.d <= 32) return launch_jll_fc<T, float, 32, false>(a, sms, s);
  if (a.d <= 64) return launch_jll_fc<T, float, 64, false>(a, sms, s);
  return launch_jll_fc<T, float, JC, true>(a, sms, s);
}

static int launch_jll_f64(const JllArgs& a, int sms, cudaStream_t s) {
  if (a.d <= 8) return launch_jll_fc<double, double, 8, false>(a, sms, s);
  if (a.d <= 16) return launch_jll_fc<double, double, 16, false>(a, sms, s);
  if (a.d <= 32) return launch_jll_fc<double, double, 32, false>(a, sms, s);
  return launch_jll_fc<double, double, JC, true>(a, sms, s);
}

// ------------------------------------------------------------------------------------- linear log-likelihood
constexpr int LT = 256;                       // threads
constexpr int LR = 64;                        // rows per tile
constexpr int LF = 32;                        // features per staged step
constexpr int LP = LF + 4;                    // float64 operand pitch (as bkm_project_chunk's)

struct LinArgs {
  const void* X;
  long long n;
  int d;
  long long ldx;
  int bin;
  double thr;
  const double* W;          // [K][d]
  const double* b;          // [K]
  int K;
  int32_t* labels;          // nullable
  double* out;              // nullable
  long long ldo;
  int out_mode;             // BKM_NB_JLL, BKM_NB_LOG_PROBA, BKM_NB_PROBA
};

template <int NT>
static size_t lin_smem() {
  constexpr int CW = 2 * NT * 8;
  return (size_t)(LR + CW) * LP * 8 + (size_t)LR * (CW + 1) * 8 + (size_t)LR * 8;
}

template <typename T, int NT>
__global__ void __launch_bounds__(LT) linear_jll_kernel(LinArgs a) {
  using namespace ptx;
  constexpr int CW = 2 * NT * 8;                // classes per block
  extern __shared__ __align__(16) unsigned char smem[];
  double* Xs = reinterpret_cast<double*>(smem);           // [LR][LP]
  double* Ws = Xs + LR * LP;                              // [CW][LP]
  double* ob = Ws + CW * LP;                              // [LR][CW + 1]
  double* lse_s = ob + LR * (CW + 1);                     // [LR]

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, tq = lane & 3;
  const int mb = warp & 3, nh = warp >> 2;
  const int d = a.d, K = a.K;
  const int nblk = (K + CW - 1) / CW;
  const T* X = reinterpret_cast<const T*>(a.X);
  const long long ntiles = (a.n + LR - 1) / LR;
  const bool want_lab = a.labels != nullptr, want_out = a.out != nullptr;
  const bool norm = want_out && a.out_mode != BKM_NB_JLL;

#pragma unroll 1
  for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const long long r0 = tile * LR;
    const int rows = (int)min((long long)LR, a.n - r0);
    // row tid's running arg-max and logsumexp (threads tid < rows)
    double best = -INFINITY, m = -INFINITY, ssum = 0.0;
    int bi = 0, nani = -1;
    bool anynan = false;

#pragma unroll 1
    for (int blk = 0; blk < nblk; ++blk) {
      const int c0 = blk * CW, kw = min(CW, K - c0);
      double acc[NT][4];
#pragma unroll
      for (int nt = 0; nt < NT; ++nt)
#pragma unroll
        for (int q = 0; q < 4; ++q) acc[nt][q] = 0.0;
#pragma unroll 1
      for (int f0 = 0; f0 < d; f0 += LF) {
        __syncthreads();                        // the previous step's MMAs (and block's epilogue) are done
        const int f = tid & (LF - 1);
        const bool fin = f0 + f < d;
#pragma unroll 4
        for (int e = tid; e < LR * LF; e += LT) {
          const int r = e >> 5;
          double v = 0.0;
          if (r < rows && fin) {
            v = to_f64(X[(r0 + r) * a.ldx + f0 + f]);
            if (a.bin) v = v > a.thr ? 1.0 : 0.0;
          }
          Xs[r * LP + f] = v;
        }
        for (int e = tid; e < CW * LF; e += LT) {
          const int c = e >> 5;
          Ws[c * LP + f] = (c < kw && fin) ? a.W[(size_t)(c0 + c) * d + f0 + f] : 0.0;
        }
        __syncthreads();
#pragma unroll
        for (int ks = 0; ks < LF / 16; ++ks) {
          const int k0 = ks * 16;
          double af[8];
#pragma unroll
          for (int i = 0; i < 8; ++i) af[i] = Xs[(mb * 16 + g + 8 * (i & 1)) * LP + k0 + tq + 4 * (i >> 1)];
#pragma unroll
          for (int nt = 0; nt < NT; ++nt) {
            double bf[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) bf[i] = Ws[(nh * NT * 8 + nt * 8 + g) * LP + k0 + tq + 4 * i];
            dmma16816(acc[nt], af, bf);
          }
        }
      }
      // ---- the block's jll into shared memory, then row tid's fold in class order ----
#pragma unroll
      for (int nt = 0; nt < NT; ++nt)
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int r = mb * 16 + g + 8 * (q >> 1), c = nh * NT * 8 + nt * 8 + 2 * tq + (q & 1);
          if (c < kw) ob[r * (CW + 1) + c] = acc[nt][q] + __ldg(a.b + c0 + c);
        }
      __syncthreads();
      if (tid < rows && (want_lab || norm)) {
#pragma unroll 1
        for (int c = 0; c < kw; ++c) {
          const double v = ob[tid * (CW + 1) + c];
          if (isnan(v)) {
            if (nani < 0) nani = c0 + c;
            anynan = true;
          } else {
            if (v > best) { best = v; bi = c0 + c; }
            if (norm) {
              if (v > m) {
                ssum = ssum * exp(m - v) + 1.0;
                m = v;
              } else if (v != -INFINITY) {
                ssum += exp(v - m);
              }
            }
          }
        }
      }
      if (want_out && (!norm || nblk > 1)) {    // the raw block goes out now
        for (int e = tid; e < rows * kw; e += LT) {
          const int r = e / kw, c = e - r * kw;
          a.out[(r0 + r) * a.ldo + c0 + c] = ob[r * (CW + 1) + c];
        }
      }
    }

    if (want_lab && tid < rows) a.labels[r0 + tid] = nani >= 0 ? nani : bi;
    if (norm) {
      // jll - (log sum exp(jll - max) + max), NaN throughout for a row with a NaN or without a finite maximum
      if (tid < LR) lse_s[tid] = (anynan || !(fabs(m) < INFINITY)) ? (double)NAN : log(ssum) + m;
      __syncthreads();
      const bool ex = a.out_mode == BKM_NB_PROBA;
      for (int e = tid; e < rows * K; e += LT) {
        const int r = e / K, c = e - r * K;
        double* p = a.out + (r0 + r) * a.ldo + c;
        double o = (nblk == 1 ? ob[r * (CW + 1) + c] : *p) - lse_s[r];
        if (ex) o = exp(o);
        *p = o;
      }
    }
  }
}

template <typename T, int NT>
static int launch_linear_nt(const LinArgs& a, int sms, cudaStream_t s) {
  const size_t sm = lin_smem<NT>();
  auto kern = linear_jll_kernel<T, NT>;
  BKM_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
  int per_sm = 0;
  BKM_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, LT, sm));
  if (per_sm < 1) per_sm = 1;
  const long long ntiles = (a.n + LR - 1) / LR;
  long long gx = (long long)per_sm * sms;
  if (gx > ntiles) gx = ntiles;
  kern<<<(unsigned)gx, LT, sm, s>>>(a);
  BKM_CUDA_TRY(cudaGetLastError());
  note_launch();
  return 0;
}

template <typename T>
static int launch_linear(const LinArgs& a, int sms, cudaStream_t s) {
  if (a.K <= 16) return launch_linear_nt<T, 1>(a, sms, s);
  if (a.K <= 32) return launch_linear_nt<T, 2>(a, sms, s);
  return launch_linear_nt<T, 4>(a, sms, s);
}

static int moments_run(const void* X, int64_t n, int d, int64_t ldx, int x_dtype, const int32_t* cls, int K, int mode,
                       const double* theta, bool counts_pass, const double* w, int bin, double thr, double* sums,
                       double* counts, void* workspace, size_t ws_bytes, int flags, void* stream) {
  int sms = 0;
  const int rc = sm_count(&sms);
  if (rc) return rc;
  const MomGeom G = mom_geom(n, d, K, sms);
  if (ws_bytes < G.total) return BKM_EWORKSPACE;
  cudaStream_t s = (cudaStream_t)stream;
  unsigned char* ws = reinterpret_cast<unsigned char*>(workspace);
  MomArgs a;
  a.X = X; a.n = n; a.d = d; a.ldx = ldx; a.cls = cls; a.K = K; a.mode = mode; a.theta = theta;
  a.part = reinterpret_cast<double*>(ws + G.off_part);
  a.cpart = reinterpret_cast<double*>(ws + G.off_cpart);
  a.fs = G.fs; a.groups = G.groups; a.ks = G.ks; a.nk = G.nk; a.rows_per_split = G.rows_per_split;
  a.w = w; a.thr = thr; a.bin = bin ? 1 : 0;
  if (G.splits > 0) {
    int r = 0;
    if (counts_pass) {
      if (x_dtype == BKM_F32) r = launch_moments<float, true>(a, G, s);
      else if (x_dtype == BKM_F64) r = launch_moments<double, true>(a, G, s);
      else r = launch_moments<__nv_bfloat16, true>(a, G, s);
    } else {
      if (x_dtype == BKM_F32) r = launch_moments<float>(a, G, s);
      else if (x_dtype == BKM_F64) r = launch_moments<double>(a, G, s);
      else r = launch_moments<__nv_bfloat16>(a, G, s);
    }
    if (r) return r;
  }
  const long long total = (long long)K * d + (mode == 0 ? K : 0);
  long long blocks = (total + 255) / 256;
  if (blocks > 4LL * sms) blocks = 4LL * sms;
  moments_fold_kernel<<<(unsigned)blocks, 256, 0, s>>>(a.part, a.cpart, G.splits, K, d, mode, sums,
                                                       mode == 0 ? counts : nullptr,
                                                       (flags & BKM_FLAG_FIRST_CHUNK) ? 1 : 0);
  BKM_CUDA_TRY(cudaGetLastError());
  note_launch();
  return 0;
}

}  // namespace
}  // namespace bkm

using namespace bkm;

extern "C" int bkm_nb_workspace_bytes(int64_t n, int d, int K, size_t* out) {
  if (!out || n < 0 || d <= 0 || K <= 0) return BKM_EINVAL;
  *out = mom_geom(n, d, K, sm_count_or_default()).total;
  return 0;
}

extern "C" int bkm_class_moments_chunk(const void* X, int64_t n, int d, int64_t ldx, int x_dtype, const int32_t* cls,
                                       int K, int mode, const double* theta, double* sums, double* counts,
                                       void* workspace, size_t ws_bytes, int flags, void* stream) {
  if (n < 0 || d <= 0 || K <= 0 || ldx < d || !sums || !workspace) return BKM_EINVAL;
  if (n > 0 && (!X || !cls)) return BKM_EINVAL;
  if (mode == 0 ? !counts : (mode != 1 || !theta)) return BKM_EINVAL;
  if (!dtype_ok(x_dtype)) return BKM_EDTYPE;
  return moments_run(X, n, d, ldx, x_dtype, cls, K, mode, theta, false, nullptr, 0, 0.0, sums, counts, workspace,
                     ws_bytes, flags, stream);
}

extern "C" int bkm_class_counts_chunk(const void* X, int64_t n, int d, int64_t ldx, int x_dtype, const int32_t* cls,
                                      int K, const double* w, int binarize, double threshold, double* fc, double* cc,
                                      void* workspace, size_t ws_bytes, int flags, void* stream) {
  if (n < 0 || d <= 0 || K <= 0 || ldx < d || !fc || !cc || !workspace) return BKM_EINVAL;
  if (n > 0 && (!X || !cls)) return BKM_EINVAL;
  if (!dtype_ok(x_dtype)) return BKM_EDTYPE;
  return moments_run(X, n, d, ldx, x_dtype, cls, K, 0, nullptr, true, w, binarize, threshold, fc, cc, workspace,
                     ws_bytes, flags, stream);
}

extern "C" int bkm_nb_jll_chunk(const void* X, int64_t n, int d, int64_t ldx, int x_dtype, const double* theta,
                                const double* inv_sigma, const double* logc, int K, int32_t* labels, double* out,
                                int64_t ldo, int exp_out, int* n_deferred, int flags, void* stream) {
  if (n < 0 || d <= 0 || K <= 0 || ldx < d || !theta || !inv_sigma || !logc) return BKM_EINVAL;
  if (!dtype_ok(x_dtype)) return BKM_EDTYPE;
  if (n == 0) return 0;                         // nothing to write (zero-size outputs may be null)
  if (!X || (!labels && !out)) return BKM_EINVAL;
  if (out && ldo < K) return BKM_EINVAL;
  int sms = 0;
  const int rc = sm_count(&sms);
  if (rc) return rc;
  JllArgs a;
  a.X = X; a.n = n; a.d = d; a.ldx = ldx; a.theta = theta; a.w = inv_sigma; a.logc = logc; a.K = K;
  a.kb = K; a.dp = 0; a.labels = labels; a.out = out; a.ldo = ldo; a.exp_out = exp_out ? 1 : 0;
  a.n_deferred = n_deferred; a.recheck = (flags & BKM_FLAG_NO_RECHECK) ? 0 : 1;
  a.tau = (float)((d + 8) * 0x1p-25);
  cudaStream_t s = (cudaStream_t)stream;
  if (x_dtype == BKM_F32) return launch_jll_f32<float>(a, sms, s);
  if (x_dtype == BKM_BF16) return launch_jll_f32<__nv_bfloat16>(a, sms, s);
  return launch_jll_f64(a, sms, s);
}

extern "C" int bkm_nb_linear_jll_chunk(const void* X, int64_t n, int d, int64_t ldx, int x_dtype, int binarize,
                                       double threshold, const double* W, const double* b, int K, int32_t* labels,
                                       double* out, int64_t ldo, int out_mode, int flags, void* stream) {
  (void)flags;
  if (n < 0 || d <= 0 || K <= 0 || ldx < d || !W || !b) return BKM_EINVAL;
  if (out_mode != BKM_NB_JLL && out_mode != BKM_NB_LOG_PROBA && out_mode != BKM_NB_PROBA) return BKM_EINVAL;
  if (!dtype_ok(x_dtype)) return BKM_EDTYPE;
  if (n == 0) return 0;
  if (!X || (!labels && !out)) return BKM_EINVAL;
  if (out && ldo < K) return BKM_EINVAL;
  int sms = 0;
  const int rc = sm_count(&sms);
  if (rc) return rc;
  LinArgs a;
  a.X = X; a.n = n; a.d = d; a.ldx = ldx; a.bin = binarize ? 1 : 0; a.thr = threshold; a.W = W; a.b = b; a.K = K;
  a.labels = labels; a.out = out; a.ldo = ldo; a.out_mode = out_mode;
  cudaStream_t s = (cudaStream_t)stream;
  if (x_dtype == BKM_F32) return launch_linear<float>(a, sms, s);
  if (x_dtype == BKM_F64) return launch_linear<double>(a, sms, s);
  return launch_linear<__nv_bfloat16>(a, sms, s);
}
