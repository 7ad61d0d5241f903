// bkm_kmeans_sparse.cu — the passes of KMeans on sparse CSR blocks (sm_90a): the E-step over the rows, the M-step sums
// over the block's transpose, and the centre update on the transposed centres.
//
//   bkm_sparse_pack_centers   C [k][p] float64 -> the sparse pack [CT (p x k) | cn (k)], CT the transposed centres and
//                             cn_j = ||c_j||^2
//   bkm_csr_assign_chunk      d2_ij = max(||x_i||^2 - 2 x_i.c_j + cn_j, 0) for one CSR block against a sparse pack:
//                             the arg-min epilogue (labels, min, distance sum, counts) or the full (n x k) block
//   bkm_csc_label_sums_chunk  sumsT (p x k) (+)= X^T onehot(labels) over the block's transpose
//   bkm_sparse_finalize_step  bkm_finalize_step on the transposed layout: C' = sums / max(counts, 1), the shift, the stop
//                             test, and the next iteration's sparse pack
//   bkm_csr_kernel_colsum_chunk  colsum_j (+)= sum_i exp(-gamma d2_ij) against the sparse pack of the l keep rows: the
//                             first Nystrom pass of SpectralClustering (the COLSUM epilogue of the assign kernel)
//   bkm_csr_nystrom_embed_chunk  out_i = e_i / ||e_i||, e_i = sum_j exp(-gamma (d2_ij - m_i)) W_j, m_i = min_j d2_ij:
//                             the second Nystrom pass (the EMBED epilogue of the assign kernel)
//   bkm_sparse_minibatch_step bkm_minibatch_step on the transposed layout: scikit-learn's _minibatch_update_sparse on the
//                             reduced [p k sumsT | k counts | inertia], the weight sums, and the next sparse pack
//   bkm_csc_class_counts_chunk  FC^T (p x K) (+)= X^T (w * onehot(labels)) with the entries optionally binarised (x > t):
//                             the class counts of PartialMultinomialNB / PartialBernoulliNB (the label sums' kernel)
//   bkm_nb_csr_jll_chunk      jll_ic = b_c + sum_j f(x_ij) W^T[j][c] and the arg-max / log-softmax epilogues of the
//                             discrete naive Bayes models (the row body of bkm_csr_panel_chunk)
//
// Every value is widened to float64 from the block's dtype; every sum runs in a fixed order and no float atomics are
// used, so two calls with the same inputs give the same bits.
//
//   assign        one warp per row, the row body of bkm_csr_panel_chunk (csr_row_gather): its lanes walk the centres in
//                 tiles of 32 C and gather the CT rows of the row's entries for each tile.  Each lane keeps its best
//                 (d2, j) over its centres, the warp folds them (ties to the lowest j).  Counts are integer atomics;
//                 the distance sums are folded per warp in row order, per CTA in warp order and over the CTAs in CTA
//                 order by the last CTA, which also adds the counts to the float64 output.
//   label sums    one warp per column segment of the transpose's plan (rows ascending) with a k-wide float64
//                 accumulator in shared memory: entry (row, v) adds v to acc[labels[row]], the lane that owns
//                 labels[row] mod 32 doing the add, so every (column, cluster) sum runs in row order.  Columns of several
//                 segments use the segment-and-ticket fold of bkm_csc_plan.cuh.
//   colsum        each warp adds exp(-gamma d2) of its rows, in row order, into a per-warp float64 row of shared
//                 memory (a lane owns the keep rows c0 + lane + 32 j of each tile); the CTA adds its warps in warp order
//                 into its partial row, and colsum_fold adds the CTA partials in CTA order.  At most 3200 keep rows per
//                 launch (the shared rows of 8 warps in 200 KB): more are split into windows of keep rows.
//   embed         per row, m_i first (one tile: from the tile's distances; several tiles: a first sweep over every
//                 tile), then per tile the kernel values go through a per-warp row of shared memory and the lanes own
//                 the outputs o = lane + 32 t, each adding the tile's keep rows in order by fma.  NaN where
//                 gamma m_i > 745.13, the rule of bkm_nystrom_embed_chunk.
//   nb jll        one warp per row; its lanes walk the classes in tiles of 32 C and gather the W^T rows of the row's
//                 entries (csr_row_gather, stored entries only).  Each lane keeps the first maximum / first NaN and a
//                 running logsumexp of its classes; the warp folds them in a fixed butterfly order.  Raw jll goes out per
//                 tile; normalised outputs are written from registers when K fits one tile, else rewritten by the
//                 lanes that wrote them.
//   pack / step   column_reduce (bkm_select.cuh) over the p rows of CT: each element of C' (from the centres or from the
//                 reduced sums) is written to CT, and per cluster the CTA-ordered sums of (C - C')^2 and of C'^2 give the
//                 shift terms and cn.  The step adds the k shift terms in cluster order.  One kernel writes every pack.
#include <climits>
#include <math_constants.h>
#include "bkm_select.cuh"
#include "bkm_csc_plan.cuh"
#include "bkm_csr_rows.cuh"

namespace bkm {
namespace {

constexpr int kWarps = kThreads / 32;

// ---------------------------------------------------------------------------------------------------------------------
// assign
// ---------------------------------------------------------------------------------------------------------------------
struct AssignArgs {
  const long long* crow;
  const long long* col;
  const void* val;
  long long n;
  int p;
  const double* CT;    // [p][k]
  const double* cn;    // [k]
  int k;
  int mode;            // BKM_SPARSE_ARGMIN / _DIST / _DIST2
  int* labels;         // nullable
  double* min_out;     // nullable
  int squared;
  void* out;           // full modes: [n][ldo]
  long long ldo;
  int out_dtype;
  double* dist_sum;    // nullable, accumulated
  double* counts;      // nullable, accumulated
  int first;
  const int* skip;     // nullable: LoopState::done
  double* part;        // [grid] CTA partial distance sums (COLSUM: [grid][k] partial column sums)
  unsigned long long* cnt;  // [k] integer counts of this call, zero at launch
  unsigned* ticket;
  double gamma;        // COLSUM / EMBED
  int j0, jn;          // COLSUM: the keep rows [j0, j0 + jn) of this launch
  const double* W;     // EMBED: [k][kw]
  int kw;
};

// the epilogues of csr_assign_kernel: the E-step (arg-min or the full distance block), the Nystrom passes
enum CsrEpi { CSR_EPI_ASSIGN = 0, CSR_EPI_COLSUM = 1, CSR_EPI_EMBED = 2 };
constexpr int kColsumWindow = 3200;    // keep rows of one COLSUM launch: kWarps rows of float64 in 200 KB

// One tile of row i: the lanes own the centres c0 + lane + 32 j below `hi` (own[j]); y[j] = d2 to each (CUDART_INF
// where not owned).
template <typename T, int C>
__device__ __forceinline__ void csr_row_tile(const AssignArgs& a, const T* val, long long i, int c0, int hi,
                                             bool (&own)[C], double (&y)[C]) {
  const int lane = threadIdx.x & 31;
  double acc[C];
#pragma unroll
  for (int j = 0; j < C; ++j) { own[j] = c0 + lane + 32 * j < hi; acc[j] = 0.0; }
  double xn = 0.0;
  csr_row_gather<T, C, true>(a.crow, a.col, val, i, a.p, a.CT, a.k, c0, own, acc, xn);
#pragma unroll
  for (int j = 0; j < C; ++j)
    y[j] = own[j] ? fmax(fma(-2.0, acc[j], xn) + a.cn[c0 + lane + 32 * j], 0.0) : CUDART_INF;
}

// EMBED: row i of the embedding.  vw [32 C] and ew [kw] are the warp's rows of shared memory.
template <typename T, int C>
__device__ __forceinline__ void embed_row(const AssignArgs& a, const T* val, long long i, double* vw, double* ew) {
  constexpr int CW = 32 * C;
  const int lane = threadIdx.x & 31, l = a.k, kw = a.kw;
  const bool one = l <= CW;
  bool own[C];
  double y[C];
  double m = CUDART_INF;
#pragma unroll 1
  for (int c0 = 0; c0 < l; c0 += CW) {                  // one tile: its distances stay in y for the second sweep
    csr_row_tile<T, C>(a, val, i, c0, l, own, y);
#pragma unroll
    for (int j = 0; j < C; ++j) m = fmin(m, y[j]);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmin(m, __shfl_xor_sync(0xffffffffu, m, o));
  for (int o = lane; o < kw; o += 32) ew[o] = 0.0;
#pragma unroll 1
  for (int c0 = 0; c0 < l; c0 += CW) {
    if (!one) csr_row_tile<T, C>(a, val, i, c0, l, own, y);
    __syncwarp();
#pragma unroll
    for (int j = 0; j < C; ++j)
      if (own[j]) vw[lane + 32 * j] = exp(-a.gamma * (y[j] - m));
    __syncwarp();
    const int nb = min(CW, l - c0);
    const double* w = a.W + (size_t)c0 * kw;
    for (int o = lane; o < kw; o += 32) {
      double e = ew[o];
      for (int j = 0; j < nb; ++j) e = fma(vw[j], __ldg(w + (size_t)j * kw + o), e);
      ew[o] = e;
    }
  }
  double nrm = 0.0;
  for (int o = lane; o < kw; o += 32) nrm = fma(ew[o], ew[o], nrm);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) nrm += __shfl_xor_sync(0xffffffffu, nrm, o);
  const double f = m * a.gamma > 745.13 ? CUDART_NAN : 1.0 / sqrt(nrm);
  for (int o = lane; o < kw; o += 32) {
    const double v = ew[o] * f;
    if (a.out_dtype == BKM_F64) reinterpret_cast<double*>(a.out)[i * a.ldo + o] = v;
    else reinterpret_cast<float*>(a.out)[i * a.ldo + o] = (float)v;
  }
}

// The Nystrom epilogues ask for 3 CTAs per SM: without a minimum, ptxas holds them to 48 registers and spills.  The
// E-step keeps its bounds (and registers).
template <typename T, int C, int EPI = CSR_EPI_ASSIGN>
__global__ void __launch_bounds__(kThreads, EPI == CSR_EPI_ASSIGN ? 0 : 3) csr_assign_kernel(AssignArgs a) {
  constexpr int CW = 32 * C;
  __shared__ double s_sum[kWarps];
  extern __shared__ double s_dyn[];    // COLSUM: [kWarps][jn] column sums; EMBED: [kWarps][CW + kw] vw, ew
  if (a.skip && *a.skip) return;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const T* val = reinterpret_cast<const T*>(a.val);
  const bool argmin = a.mode == BKM_SPARSE_ARGMIN;
  double wsum = 0.0;
  const long long nw = (long long)gridDim.x * kWarps;
  if constexpr (EPI == CSR_EPI_COLSUM) {
    for (int j = lane; j < a.jn; j += 32) s_dyn[warp * a.jn + j] = 0.0;
    __syncwarp();
  }
#pragma unroll 1
  for (long long i = (long long)blockIdx.x * kWarps + warp; i < a.n; i += nw) {
    if constexpr (EPI == CSR_EPI_EMBED) {
      double* vw = s_dyn + (size_t)warp * (CW + a.kw);
      embed_row<T, C>(a, val, i, vw, vw + CW);
      continue;
    } else if constexpr (EPI == CSR_EPI_COLSUM) {
      double* cs = s_dyn + (size_t)warp * a.jn - a.j0;
#pragma unroll 1
      for (int c0 = a.j0; c0 < a.j0 + a.jn; c0 += CW) {
        bool own[C];
        double y[C];
        csr_row_tile<T, C>(a, val, i, c0, a.j0 + a.jn, own, y);
#pragma unroll
        for (int j = 0; j < C; ++j)
          if (own[j]) cs[c0 + lane + 32 * j] += exp(-a.gamma * y[j]);
      }
      continue;
    }
    double best = CUDART_INF;
    int bj = 0x7fffffff;
#pragma unroll 1
    for (int c0 = 0; c0 < a.k; c0 += CW) {
      bool own[C];
      double acc[C];
#pragma unroll
      for (int j = 0; j < C; ++j) { own[j] = c0 + lane + 32 * j < a.k; acc[j] = 0.0; }
      double xn = 0.0;
      csr_row_gather<T, C, true>(a.crow, a.col, val, i, a.p, a.CT, a.k, c0, own, acc, xn);
#pragma unroll
      for (int j = 0; j < C; ++j) {
        if (!own[j]) continue;
        const int cc = c0 + lane + 32 * j;
        const double d2 = fmax(fma(-2.0, acc[j], xn) + a.cn[cc], 0.0);
        if (argmin) {
          if (d2 < best) { best = d2; bj = cc; }           // a lane's centres ascend: ties keep the lowest
        } else {
          const double v = a.mode == BKM_SPARSE_DIST2 ? d2 : sqrt(d2);
          if (a.out_dtype == BKM_F64) reinterpret_cast<double*>(a.out)[i * a.ldo + cc] = v;
          else reinterpret_cast<float*>(a.out)[i * a.ldo + cc] = (float)v;
        }
      }
    }
    if (!argmin) continue;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const double ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int oj = __shfl_xor_sync(0xffffffffu, bj, o);
      if (ob < best || (ob == best && oj < bj)) { best = ob; bj = oj; }
    }
    if (bj >= a.k) bj = 0;                                // every distance infinite
    if (lane == 0) {
      const double m = a.squared ? best : sqrt(best);
      if (a.labels) a.labels[i] = bj;
      if (a.min_out) a.min_out[i] = m;
      wsum += m;
      if (a.counts) atomicAdd(a.cnt + bj, 1ull);
    }
  }
  if constexpr (EPI == CSR_EPI_COLSUM) {
    // ---- the CTA's partial: its warps in order ----
    __syncthreads();
    for (int j = tid; j < a.jn; j += kThreads) {
      double v = 0.0;
      for (int w = 0; w < kWarps; ++w) v += s_dyn[w * a.jn + j];
      a.part[(size_t)blockIdx.x * a.k + a.j0 + j] = v;
    }
    return;
  }
  if constexpr (EPI != CSR_EPI_ASSIGN) return;
  if (!argmin || (!a.dist_sum && !a.counts)) return;

  // ---- the fold: warps in order, CTAs in order by the last CTA, which also publishes the counts ----
  if (lane == 0) s_sum[warp] = wsum;
  __syncthreads();
  if (tid == 0) {
    double v = 0.0;
    for (int w = 0; w < kWarps; ++w) v += s_sum[w];
    a.part[blockIdx.x] = v;
  }
  if (!last_block(a.ticket, gridDim.x)) return;
  if (a.dist_sum && tid == 0) {
    double v = 0.0;
    for (unsigned c = 0; c < gridDim.x; ++c) v += __ldcg(a.part + c);
    *a.dist_sum = a.first ? v : *a.dist_sum + v;
  }
  if (a.counts) {
    for (int j = tid; j < a.k; j += kThreads) {
      const double c = (double)__ldcg(a.cnt + j);
      a.counts[j] = a.first ? c : a.counts[j] + c;
    }
  }
  if (tid == 0) *a.ticket = 0u;
}

static int grid_for(long long work, int per_cta, long long cap) {
  long long g = (work + per_cta - 1) / per_cta;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

static int assign_grid(long long n, int sms) { return grid_for(n, kWarps, 8LL * sms); }
static size_t assign_ws(long long n, int k, int sms) {
  return align_up((size_t)assign_grid(n, sms) * 8, 256) + align_up((size_t)k * 8, 256) + 256;
}

// dynamic shared memory of an epilogue launch
template <int C, int EPI>
static size_t assign_smem(const AssignArgs& a) {
  if (EPI == CSR_EPI_COLSUM) return (size_t)kWarps * a.jn * 8;
  if (EPI == CSR_EPI_EMBED) return (size_t)kWarps * (32 * C + a.kw) * 8;
  return 0;
}

template <typename T, int C, int EPI>
static int launch_assign(const AssignArgs& a, int grid, cudaStream_t s) {
  const size_t smem = assign_smem<C, EPI>(a);
  if (smem > 200 * 1024) return BKM_EUNSUPPORTED;
  if (smem > 48 * 1024)
    BKM_CUDA_TRY(cudaFuncSetAttribute(csr_assign_kernel<T, C, EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)smem));
  csr_assign_kernel<T, C, EPI><<<grid, kThreads, smem, s>>>(a);
  BKM_CUDA_TRY(cudaGetLastError());
  note_launch();
  return 0;
}

template <typename T, int EPI = CSR_EPI_ASSIGN>
static int assign(const AssignArgs& a, int grid, cudaStream_t s) {
  if (a.k <= 32) return launch_assign<T, 1, EPI>(a, grid, s);
  if (a.k <= 64) return launch_assign<T, 2, EPI>(a, grid, s);
  return launch_assign<T, 4, EPI>(a, grid, s);
}

template <int EPI>
static int assign_dt(const AssignArgs& a, int val_dtype, int grid, cudaStream_t s) {
  return val_dtype == BKM_F32 ? assign<float, EPI>(a, grid, s) : assign<double, EPI>(a, grid, s);
}

// ---------------------------------------------------------------------------------------------------------------------
// label sums
// ---------------------------------------------------------------------------------------------------------------------
struct LabelSumArgs {
  const long long* colptr;
  const int* rows;
  const void* vals;
  int p;
  const long long* plan;
  const int* labels;   // [n]
  int k;
  double* out;         // [p][k]
  double* slot;
  unsigned* ticket;    // [p], zero
  int first;
  const int* skip;
  const double* w;     // WB: the row weights [n], nullable
  double thr;          // WB with bin: entries count as val > thr
  int bin;
};

// WB (bkm_csc_class_counts_chunk): entry (row, v) adds f(v) w[row] in place of v
template <typename T, bool WB = false>
__global__ void __launch_bounds__(kThreads) csc_label_sums_kernel(LabelSumArgs a) {
  extern __shared__ double s_acc[];        // [warps][k]
  if (a.skip && *a.skip) return;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, warps = blockDim.x >> 5, k = a.k;
  double* acc = s_acc + (size_t)warp * k;
  const long long T_ = a.plan[ST_SEGS];
  const T* vals = reinterpret_cast<const T*>(a.vals);
  const long long nw = (long long)gridDim.x * warps;
#pragma unroll 1
  for (long long t = (long long)blockIdx.x * warps + warp; t < T_; t += nw) {
    const SegSpan sp = seg_span(a.plan, a.colptr, a.p, t);
    for (int c = lane; c < k; c += 32) acc[c] = 0.0;
    __syncwarp();
#pragma unroll 1
    for (long long eb = sp.e0; eb < sp.e1; eb += 32) {
      int lab = -1;
      double v = 0.0;
      if (eb + lane < sp.e1) {
        if (WB) {
          const int r = a.rows[eb + lane];
          lab = a.labels[r];
          v = to_f64(vals[eb + lane]);
          if (a.bin) v = v > a.thr ? 1.0 : 0.0;
          if (a.w) v *= __ldg(a.w + r);
        } else {
          lab = a.labels[a.rows[eb + lane]];
          v = to_f64(vals[eb + lane]);
        }
      }
      const int m = (int)min(32LL, sp.e1 - eb);
#pragma unroll 4
      for (int q = 0; q < m; ++q) {
        const int lq = __shfl_sync(0xffffffffu, lab, q);
        const double vq = __shfl_sync(0xffffffffu, v, q);
        if ((unsigned)lq < (unsigned)k && (lq & 31) == lane) acc[lq] += vq;
      }
    }
    __syncwarp();
    if (sp.ns > 1) {
      double* slot = seg_slot(a.slot, sp, t, k);
      for (int c = lane; c < k; c += 32) slot[c] = acc[c];
      seg_fold(sp, a.slot, a.ticket, a.out, k, a.first);
    } else {
      double* o = a.out + (size_t)sp.j * k;
      for (int c = lane; c < k; c += 32) o[c] = a.first ? acc[c] : o[c] + acc[c];
    }
    __syncwarp();
  }
}

// warps per CTA of the label sums: as many k-wide accumulators as fit 200 KB of shared memory (k <= 25600), at most 8
static int label_sums_warps(int k) {
  const long long w = (200LL * 1024) / ((long long)k * 8);
  return w > kWarps ? kWarps : (int)w;
}

template <typename T, bool WB>
static int launch_label_sums(const LabelSumArgs& a, long long nnz, cudaStream_t s) {
  const int warps = label_sums_warps(a.k);
  const size_t smem = (size_t)warps * a.k * 8;
  if (smem > 48 * 1024)
    BKM_CUDA_TRY(cudaFuncSetAttribute(csc_label_sums_kernel<T, WB>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)smem));
  const int grid = grid_for(seg_cap(a.p, nnz), warps, 16LL * sm_count_or_default());
  csc_label_sums_kernel<T, WB><<<grid, warps * 32, smem, s>>>(a);
  BKM_CUDA_TRY(cudaGetLastError());
  note_launch();
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------------
// naive Bayes log-likelihood
// ---------------------------------------------------------------------------------------------------------------------
struct NbJllArgs {
  const long long* crow;
  const long long* col;
  const void* val;
  long long n;
  int p;
  const double* WT;    // [p][K]
  const double* b;     // [K]
  int K;
  int bin;
  double thr;
  int32_t* labels;     // nullable
  double* out;         // [n][ldo], nullable
  long long ldo;
  int out_mode;
};

template <typename T, int C, bool BIN>
__global__ void __launch_bounds__(kThreads) csr_nb_jll_kernel(NbJllArgs a) {
  constexpr int CW = 32 * C;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int K = a.K;
  const bool one = K <= CW;
  const bool norm = a.out && a.out_mode != BKM_NB_JLL;
  const T* val = reinterpret_cast<const T*>(a.val);
  const long long nw = (long long)gridDim.x * kWarps;
#pragma unroll 1
  for (long long i = (long long)blockIdx.x * kWarps + warp; i < a.n; i += nw) {
    double best = -INFINITY, m = -INFINITY, ssum = 0.0;
    int bi = INT_MAX, nani = INT_MAX;
    double acc[C];
    bool own[C];
#pragma unroll 1
    for (int c0 = 0; c0 < K; c0 += CW) {
#pragma unroll
      for (int j = 0; j < C; ++j) {
        own[j] = c0 + lane + 32 * j < K;
        acc[j] = 0.0;
      }
      double xn = 0.0;
      csr_row_gather<T, C, false, BIN>(a.crow, a.col, val, i, a.p, a.WT, K, c0, own, acc, xn, a.thr);
#pragma unroll
      for (int j = 0; j < C; ++j) {
        if (!own[j]) continue;
        const int cc = c0 + lane + 32 * j;
        const double v = acc[j] + __ldg(a.b + cc);
        acc[j] = v;
        if (isnan(v)) {
          if (nani == INT_MAX) nani = cc;
        } else {
          if (bi == INT_MAX || v > best) { best = v; bi = cc; }
          if (v > m) {
            ssum = ssum * exp(m - v) + 1.0;
            m = v;
          } else if (v != -INFINITY) {
            ssum += exp(v - m);
          }
        }
        if (a.out && (!norm || !one)) a.out[i * a.ldo + cc] = v;
      }
    }
    // ---- the warp's fold: first NaN, else the first maximum; the logsumexp terms by a fixed butterfly ----
    nani = __reduce_min_sync(0xffffffffu, nani);
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      const double ob = __shfl_xor_sync(0xffffffffu, best, off);
      const int obi = __shfl_xor_sync(0xffffffffu, bi, off);
      if (obi != INT_MAX && (bi == INT_MAX || ob > best || (ob == best && obi < bi))) { best = ob; bi = obi; }
      const double om = __shfl_xor_sync(0xffffffffu, m, off);
      const double os = __shfl_xor_sync(0xffffffffu, ssum, off);
      const double M = fmax(m, om);
      // rounded products: the two lanes of a pair get the same bits
      if (M != -INFINITY)
        ssum = __dadd_rn(m == -INFINITY ? 0.0 : __dmul_rn(ssum, exp(m - M)), om == -INFINITY ? 0.0 : __dmul_rn(os, exp(om - M)));
      m = M;
    }
    if (a.labels && lane == 0) a.labels[i] = nani != INT_MAX ? nani : (bi == INT_MAX ? 0 : bi);
    if (!norm) continue;
    const double lse = (nani != INT_MAX || !(fabs(m) < INFINITY)) ? (double)NAN : log(ssum) + m;
    const bool ex = a.out_mode == BKM_NB_PROBA;
    if (one) {
#pragma unroll
      for (int j = 0; j < C; ++j) {
        if (!own[j]) continue;
        double o = acc[j] - lse;
        if (ex) o = exp(o);
        a.out[i * a.ldo + lane + 32 * j] = o;
      }
    } else {
      for (int cc = lane; cc < K; cc += 32) {          // the lane that wrote each raw value rewrites it
        double* q = a.out + i * a.ldo + cc;
        double o = *q - lse;
        if (ex) o = exp(o);
        *q = o;
      }
    }
  }
}

template <typename T, int C, bool BIN>
static int launch_nb_jll(const NbJllArgs& a, int sms, cudaStream_t s) {
  csr_nb_jll_kernel<T, C, BIN><<<assign_grid(a.n, sms), kThreads, 0, s>>>(a);
  BKM_CUDA_TRY(cudaGetLastError());
  note_launch();
  return 0;
}

template <typename T, bool BIN>
static int nb_jll(const NbJllArgs& a, int sms, cudaStream_t s) {
  if (a.K <= 32) return launch_nb_jll<T, 1, BIN>(a, sms, s);
  if (a.K <= 64) return launch_nb_jll<T, 2, BIN>(a, sms, s);
  return launch_nb_jll<T, 4, BIN>(a, sms, s);
}

// ---------------------------------------------------------------------------------------------------------------------
// pack / step
// ---------------------------------------------------------------------------------------------------------------------
// C'[f][j] from the float64 centres C [k][p]
struct FromCentres {
  const double* C;
  int p;
  __device__ __forceinline__ double operator()(long long f, int j) const { return C[(size_t)j * p + f]; }
};
// ... from the reduced buffer [p k sumsT | k counts | inertia]: sums / max(counts, 1)
struct FromSums {
  const double* red;
  long long pk;
  int k;
  __device__ __forceinline__ double operator()(long long f, int j) const {
    const double c = red[pk + j];
    return red[(size_t)f * k + j] / (c > 1.0 ? c : 1.0);
  }
};

// ... from the reduced buffer and the current pack and weight sums: scikit-learn's _minibatch_update_sparse,
// C' = (C w + S) (1 / (w + n)) where n > 0, else C, with the explicit round-to-nearest intrinsics of
// CentreFromMinibatch (bkm_aux.cu).  The element of row 0 of each cluster also writes w' = w + n.
struct FromMinibatch {
  const double* red;
  const double* ct;    // the current CT [p][k]
  const double* w_in;
  double* w_out;
  long long pk;
  int k;
  __device__ __forceinline__ double operator()(long long f, int j) const {
    const double n = red[pk + j];
    if (f == 0) w_out[j] = __dadd_rn(w_in[j], n);
    const double c = ct[(size_t)f * k + j];
    if (!(n > 0.0)) return c;
    const double alpha = __ddiv_rn(1.0, __dadd_rn(w_in[j], n));
    return __dmul_rn(__dadd_rn(__dmul_rn(c, w_in[j]), red[(size_t)f * k + j]), alpha);
  }
};

template <typename Src>
struct PackRows {
  Src src;
  const double* ct_in;   // nullable: the current CT (the step's shift)
  double* ct_out;
  int k;
  __device__ __forceinline__ void operator()(double (&f)[2], int j, long long r0, long long re, int G) const {
    for (long long r = r0; r < re; r += G) {
      const double c = src(r, j);
      ct_out[(size_t)r * k + j] = c;
      if (ct_in) { const double df = ct_in[(size_t)r * k + j] - c; f[0] = fma(df, df, f[0]); }
      f[1] = fma(c, c, f[1]);
    }
  }
};

struct PackFold {
  double* shift_col;     // [k]
  double* cn;            // [k]
  int* last;             // shared: set by the CTA that folds
  int live;
  __device__ __forceinline__ static double identity(int) { return 0.0; }
  __device__ __forceinline__ static double combine(int, double v, double p) { return v + p; }
  __device__ __forceinline__ void store(int s, int j, double v) const {
    if (s == 0) shift_col[j] = v;
    else cn[j] = v;
    *last = 1;
  }
};

template <typename Src>
__global__ void __launch_bounds__(kThreads)
sparse_pack_kernel(Src src, const double* ct_in, double* ct_out, double* cn_out, int p, int k, LoopState* st,
                   double* part, unsigned* ticket, double* shift_col) {
  __shared__ int s_last;
  if (st && st->done) return;
  if (threadIdx.x == 0) s_last = 0;
  __syncthreads();
  const PackRows<Src> rows{src, ct_in, ct_out, k};
  const PackFold fold{shift_col, cn_out, &s_last, 2};
  column_reduce<2>(rows, fold, p, k, col_block(k), part, ticket);
  if (!st) return;
  __syncthreads();
  if (s_last && threadIdx.x == 0) {
    double shift = 0.0;
    for (int j = 0; j < k; ++j) shift += shift_col[j];
    loop_commit(st, shift, shift < st->tol);
  }
}

static int pack_grid_sparse(int p, int k, int sms) { return reduce_grid(p, kThreads / col_block(k), 4, sms); }
static size_t pack_ws(int p, int k, int sms) {
  return align_up((size_t)k * 8, 256) + partials_bytes(pack_grid_sparse(p, k, sms), 2 * (size_t)k);
}

template <typename Src>
static int launch_pack(const Src& src, const double* ct_in, double* pack_out, int p, int k, LoopState* st,
                       void* ws, size_t ws_bytes, cudaStream_t s) {
  const int sms = sm_count_or_default();
  const int grid = pack_grid_sparse(p, k, sms);
  double* shift_col = reinterpret_cast<double*>(ws);
  const size_t off = align_up((size_t)k * 8, 256);
  double* part;
  unsigned* ticket;
  BKM_CUDA_TRY(carve_partials(reinterpret_cast<unsigned char*>(ws) + off, ws_bytes - off, &part, &ticket, s));
  double* ct_out = pack_out;
  double* cn_out = pack_out + (size_t)p * k;
  sparse_pack_kernel<Src><<<grid, kThreads, 0, s>>>(src, ct_in, ct_out, cn_out, p, k, st, part, ticket, shift_col);
  BKM_CUDA_TRY(cudaGetLastError());
  note_launch();
  return 0;
}

}  // namespace

int launch_colsum_fold(const double* part, int parts, int l, double* colsum, int first, cudaStream_t s);
}  // namespace bkm

using namespace bkm;

extern "C" int bkm_csr_assign_workspace_bytes(int64_t n, int k, size_t* out) {
  if (!out || n < 0 || k <= 0) return BKM_EINVAL;
  *out = assign_ws(n, k, sm_count_or_default());
  return 0;
}

extern "C" int bkm_csr_assign_chunk(const int64_t* crow, const int64_t* col, const void* val, int val_dtype, int64_t n,
                                    int p, int64_t nnz, const double* pack, int k, int mode, int32_t* labels,
                                    double* min_out, int squared, double* dist_sum, double* counts, void* out,
                                    int64_t ldo, int out_dtype, void* workspace, size_t ws_bytes, int flags,
                                    const void* loop_state, void* stream) {
  if (n < 0 || p <= 0 || nnz < 0 || k <= 0 || !crow || !pack) return BKM_EINVAL;
  if (nnz > 0 && (!col || !val)) return BKM_EINVAL;
  if (val_dtype != BKM_F32 && val_dtype != BKM_F64) return BKM_EDTYPE;
  if (mode != BKM_SPARSE_ARGMIN && mode != BKM_SPARSE_DIST && mode != BKM_SPARSE_DIST2) return BKM_EINVAL;
  if (mode != BKM_SPARSE_ARGMIN && (!out || ldo < k || (out_dtype != BKM_F32 && out_dtype != BKM_F64)))
    return BKM_EINVAL;
  const bool fold = mode == BKM_SPARSE_ARGMIN && (dist_sum || counts);
  const int sms = sm_count_or_default();
  if (fold && (!workspace || ws_bytes < assign_ws(n, k, sms))) return BKM_EWORKSPACE;
  if (mode != BKM_SPARSE_ARGMIN && n == 0) return 0;
  if (mode == BKM_SPARSE_ARGMIN && !fold && (n == 0 || (!labels && !min_out))) return 0;
  cudaStream_t s = (cudaStream_t)stream;
  AssignArgs a;
  a.crow = reinterpret_cast<const long long*>(crow);
  a.col = reinterpret_cast<const long long*>(col);
  a.val = val; a.n = n; a.p = p; a.CT = pack; a.cn = pack + (size_t)p * k; a.k = k; a.mode = mode;
  a.labels = labels; a.min_out = min_out; a.squared = squared ? 1 : 0;
  a.out = out; a.ldo = ldo; a.out_dtype = out_dtype; a.dist_sum = dist_sum; a.counts = counts;
  a.first = (flags & BKM_FLAG_FIRST_CHUNK) ? 1 : 0;
  a.skip = loop_state ? &reinterpret_cast<const LoopState*>(loop_state)->done : nullptr;
  a.part = nullptr; a.cnt = nullptr; a.ticket = nullptr;
  const int grid = assign_grid(n, sms);
  if (fold) {
    unsigned char* ws = reinterpret_cast<unsigned char*>(workspace);
    const size_t o1 = align_up((size_t)grid * 8, 256), o2 = o1 + align_up((size_t)k * 8, 256);
    a.part = reinterpret_cast<double*>(ws);
    a.cnt = reinterpret_cast<unsigned long long*>(ws + o1);
    a.ticket = reinterpret_cast<unsigned*>(ws + o2);
    BKM_CUDA_TRY(cudaMemsetAsync(ws + o1, 0, o2 - o1 + 256, s));
  }
  return assign_dt<CSR_EPI_ASSIGN>(a, val_dtype, grid, s);
}

// AssignArgs of the Nystrom epilogues: the block against the sparse pack of the l keep rows
static AssignArgs nystrom_args(const int64_t* crow, const int64_t* col, const void* val, int64_t n, int p,
                               const double* pack, int l, double gamma) {
  AssignArgs a = {};
  a.crow = reinterpret_cast<const long long*>(crow);
  a.col = reinterpret_cast<const long long*>(col);
  a.val = val; a.n = n; a.p = p; a.CT = pack; a.cn = pack + (size_t)p * l; a.k = l;
  a.gamma = gamma;
  return a;
}

extern "C" int bkm_csr_kernel_colsum_workspace_bytes(int64_t n, int l, size_t* out) {
  if (!out || n < 0 || l <= 0) return BKM_EINVAL;
  *out = align_up((size_t)assign_grid(n, sm_count_or_default()) * l * 8, 256);
  return 0;
}

extern "C" int bkm_csr_kernel_colsum_chunk(const int64_t* crow, const int64_t* col, const void* val, int val_dtype,
                                           int64_t n, int p, int64_t nnz, const double* pack, int l, double gamma,
                                           double* colsum, void* workspace, size_t ws_bytes, int flags, void* stream) {
  if (n < 0 || p <= 0 || nnz < 0 || l <= 0 || !crow || !pack || !colsum) return BKM_EINVAL;
  if (nnz > 0 && (!col || !val)) return BKM_EINVAL;
  if (val_dtype != BKM_F32 && val_dtype != BKM_F64) return BKM_EDTYPE;
  cudaStream_t s = (cudaStream_t)stream;
  const int first = (flags & BKM_FLAG_FIRST_CHUNK) ? 1 : 0;
  if (n == 0) {
    if (first) BKM_CUDA_TRY(cudaMemsetAsync(colsum, 0, (size_t)l * sizeof(double), s));
    return 0;
  }
  const int sms = sm_count_or_default();
  const int grid = assign_grid(n, sms);
  if (!workspace || ws_bytes < align_up((size_t)grid * l * 8, 256)) return BKM_EWORKSPACE;
  AssignArgs a = nystrom_args(crow, col, val, n, p, pack, l, gamma);
  a.part = reinterpret_cast<double*>(workspace);
  for (int j0 = 0; j0 < l; j0 += kColsumWindow) {
    a.j0 = j0;
    a.jn = min(kColsumWindow, l - j0);
    const int rc = assign_dt<CSR_EPI_COLSUM>(a, val_dtype, grid, s);
    if (rc) return rc;
  }
  return launch_colsum_fold(a.part, grid, l, colsum, first, s);
}

extern "C" int bkm_csr_nystrom_embed_chunk(const int64_t* crow, const int64_t* col, const void* val, int val_dtype,
                                           int64_t n, int p, int64_t nnz, const double* pack, int l, double gamma,
                                           const double* W, int k, void* out, int64_t ldo, int out_dtype, int flags,
                                           void* stream) {
  (void)flags;
  if (n < 0 || p <= 0 || nnz < 0 || l <= 0 || k <= 0 || ldo < k || !crow || !pack || !W) return BKM_EINVAL;
  if (nnz > 0 && (!col || !val)) return BKM_EINVAL;
  if (val_dtype != BKM_F32 && val_dtype != BKM_F64) return BKM_EDTYPE;
  if (out_dtype != BKM_F32 && out_dtype != BKM_F64) return BKM_EDTYPE;
  if (n == 0) return 0;
  if (!out) return BKM_EINVAL;
  AssignArgs a = nystrom_args(crow, col, val, n, p, pack, l, gamma);
  a.W = W; a.kw = k; a.out = out; a.ldo = ldo; a.out_dtype = out_dtype;
  return assign_dt<CSR_EPI_EMBED>(a, val_dtype, assign_grid(n, sm_count_or_default()), (cudaStream_t)stream);
}

extern "C" int bkm_csc_label_sums_workspace_bytes(int p, int64_t nnz, int k, size_t* out) {
  if (!out || p <= 0 || nnz < 0 || k <= 0) return BKM_EINVAL;
  *out = seg_fold_ws(p, nnz, k);
  return 0;
}

extern "C" int bkm_csc_label_sums_chunk(const int64_t* colptr, const int32_t* rows, const void* vals, int val_dtype,
                                        int p, int64_t nnz, const int64_t* plan, const int32_t* labels, int k,
                                        double* sumsT, void* workspace, size_t ws_bytes, int flags,
                                        const void* loop_state, void* stream) {
  if (p <= 0 || nnz < 0 || k <= 0 || !colptr || !plan || !sumsT || !workspace) return BKM_EINVAL;
  if (nnz > 0 && (!rows || !vals || !labels)) return BKM_EINVAL;
  if (val_dtype != BKM_F32 && val_dtype != BKM_F64) return BKM_EDTYPE;
  const int warps = label_sums_warps(k);
  if (warps < 1) return BKM_EINVAL;
  if (ws_bytes < seg_fold_ws(p, nnz, k)) return BKM_EWORKSPACE;
  cudaStream_t s = (cudaStream_t)stream;
  unsigned char* ws = reinterpret_cast<unsigned char*>(workspace);
  LabelSumArgs a;
  a.colptr = reinterpret_cast<const long long*>(colptr);
  a.rows = rows; a.vals = vals; a.p = p; a.plan = reinterpret_cast<const long long*>(plan);
  a.labels = labels; a.k = k; a.out = sumsT;
  a.slot = reinterpret_cast<double*>(ws);
  a.ticket = reinterpret_cast<unsigned*>(ws + seg_slots_bytes(nnz, k));
  a.first = (flags & BKM_FLAG_FIRST_CHUNK) ? 1 : 0;
  a.skip = loop_state ? &reinterpret_cast<const LoopState*>(loop_state)->done : nullptr;
  a.w = nullptr; a.thr = 0.0; a.bin = 0;
  BKM_CUDA_TRY(cudaMemsetAsync(a.ticket, 0, (size_t)p * 4, s));
  if (val_dtype == BKM_F32) return launch_label_sums<float, false>(a, nnz, s);
  return launch_label_sums<double, false>(a, nnz, s);
}

extern "C" int bkm_csc_class_counts_chunk(const int64_t* colptr, const int32_t* rows, const void* vals, int val_dtype,
                                          int p, int64_t nnz, const int64_t* plan, const int32_t* labels, int k,
                                          const double* w, int binarize, double threshold, double* fcT,
                                          void* workspace, size_t ws_bytes, int flags, void* stream) {
  if (p <= 0 || nnz < 0 || k <= 0 || !colptr || !plan || !fcT || !workspace) return BKM_EINVAL;
  if (nnz > 0 && (!rows || !vals || !labels)) return BKM_EINVAL;
  if (val_dtype != BKM_F32 && val_dtype != BKM_F64) return BKM_EDTYPE;
  if (label_sums_warps(k) < 1) return BKM_EINVAL;
  if (ws_bytes < seg_fold_ws(p, nnz, k)) return BKM_EWORKSPACE;
  cudaStream_t s = (cudaStream_t)stream;
  unsigned char* ws = reinterpret_cast<unsigned char*>(workspace);
  LabelSumArgs a;
  a.colptr = reinterpret_cast<const long long*>(colptr);
  a.rows = rows; a.vals = vals; a.p = p; a.plan = reinterpret_cast<const long long*>(plan);
  a.labels = labels; a.k = k; a.out = fcT;
  a.slot = reinterpret_cast<double*>(ws);
  a.ticket = reinterpret_cast<unsigned*>(ws + seg_slots_bytes(nnz, k));
  a.first = (flags & BKM_FLAG_FIRST_CHUNK) ? 1 : 0;
  a.skip = nullptr;
  a.w = w; a.thr = threshold; a.bin = binarize ? 1 : 0;
  BKM_CUDA_TRY(cudaMemsetAsync(a.ticket, 0, (size_t)p * 4, s));
  if (val_dtype == BKM_F32) return launch_label_sums<float, true>(a, nnz, s);
  return launch_label_sums<double, true>(a, nnz, s);
}

extern "C" int bkm_nb_csr_jll_chunk(const int64_t* crow, const int64_t* col, const void* val, int val_dtype, int64_t n,
                                    int p, int64_t nnz, int binarize, double threshold, const double* WT,
                                    const double* b, int K, int32_t* labels, double* out, int64_t ldo, int out_mode,
                                    int flags, void* stream) {
  (void)flags;
  if (n < 0 || p <= 0 || nnz < 0 || K <= 0 || !crow || !WT || !b) return BKM_EINVAL;
  if (nnz > 0 && (!col || !val)) return BKM_EINVAL;
  if (val_dtype != BKM_F32 && val_dtype != BKM_F64) return BKM_EDTYPE;
  if (out_mode != BKM_NB_JLL && out_mode != BKM_NB_LOG_PROBA && out_mode != BKM_NB_PROBA) return BKM_EINVAL;
  if (out && ldo < K) return BKM_EINVAL;
  if (n == 0 || (!labels && !out)) return 0;
  NbJllArgs a;
  a.crow = reinterpret_cast<const long long*>(crow);
  a.col = reinterpret_cast<const long long*>(col);
  a.val = val; a.n = n; a.p = p; a.WT = WT; a.b = b; a.K = K; a.bin = binarize ? 1 : 0; a.thr = threshold;
  a.labels = labels; a.out = out; a.ldo = ldo; a.out_mode = out_mode;
  const int sms = sm_count_or_default();
  cudaStream_t s = (cudaStream_t)stream;
  if (val_dtype == BKM_F32) return a.bin ? nb_jll<float, true>(a, sms, s) : nb_jll<float, false>(a, sms, s);
  return a.bin ? nb_jll<double, true>(a, sms, s) : nb_jll<double, false>(a, sms, s);
}

extern "C" int bkm_sparse_pack_workspace_bytes(int k, int p, size_t* out) {
  if (!out || k <= 0 || p <= 0) return BKM_EINVAL;
  *out = pack_ws(p, k, sm_count_or_default());
  return 0;
}

extern "C" int bkm_sparse_pack_centers(const double* centers64, int k, int p, double* pack, void* workspace,
                                       size_t ws_bytes, void* stream) {
  if (!centers64 || !pack || !workspace || k <= 0 || p <= 0) return BKM_EINVAL;
  if (ws_bytes < pack_ws(p, k, sm_count_or_default())) return BKM_EWORKSPACE;
  return launch_pack(FromCentres{centers64, p}, nullptr, pack, p, k, nullptr, workspace, ws_bytes,
                     (cudaStream_t)stream);
}

extern "C" int bkm_sparse_finalize_step(const double* reduced, const double* pack_in, double* pack_out,
                                        void* loop_state, int k, int p, void* workspace, size_t ws_bytes,
                                        void* stream) {
  if (!reduced || !pack_in || !pack_out || !loop_state || !workspace || k <= 0 || p <= 0) return BKM_EINVAL;
  if (pack_in == pack_out) return BKM_EINVAL;
  if (ws_bytes < pack_ws(p, k, sm_count_or_default())) return BKM_EWORKSPACE;
  return launch_pack(FromSums{reduced, (long long)p * k, k}, pack_in, pack_out, p, k,
                     reinterpret_cast<LoopState*>(loop_state), workspace, ws_bytes, (cudaStream_t)stream);
}

extern "C" int bkm_sparse_minibatch_step(const double* reduced, const double* pack_in, const double* weights_in,
                                         double* pack_out, double* weights_out, int k, int p, void* workspace,
                                         size_t ws_bytes, void* stream) {
  if (!reduced || !pack_in || !weights_in || !pack_out || !weights_out || !workspace || k <= 0 || p <= 0)
    return BKM_EINVAL;
  if (pack_in == pack_out || weights_in == weights_out) return BKM_EINVAL;
  if (ws_bytes < pack_ws(p, k, sm_count_or_default())) return BKM_EWORKSPACE;
  const FromMinibatch src{reduced, pack_in, weights_in, weights_out, (long long)p * k, k};
  return launch_pack(src, nullptr, pack_out, p, k, nullptr, workspace, ws_bytes, (cudaStream_t)stream);
}
