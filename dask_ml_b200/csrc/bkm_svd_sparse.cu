// bkm_svd_sparse.cu — the products of a sparse CSR block with a dense float64 panel (sm_90a): the two passes of
// TruncatedSVD's randomized power iterator on sparse X, and its projection pass.
//
//   bkm_csr_panel_chunk  out (n x l) = X W           W (p x l) float64 row-major, out float32 / float64, any row pitch,
//                        with an optional signed arg-max epilogue per column (the ColMax records of bkm_project_chunk)
//   bkm_csc_panel_chunk  out (p x l) (+)= X^T P      P (n x l) float64 row-major, over the block's transpose
//
// Every value is widened to float64 from the block's dtype; every sum runs in a fixed order and no float atomics are
// used, so two calls with the same inputs give the same bits.
//
//   row panel     one warp per row; its lanes own 32 C consecutive output columns (blockIdx.y picks the column tile).
//                 The warp loads 32 entries of the row at a time and takes them one by one in stored (ascending column)
//                 order: each entry gathers the W row's l * 8 contiguous bytes and every lane adds val W[col][c] to its
//                 columns by fma.  With the epilogue, each lane keeps the best (|t|, row) of its columns over its rows;
//                 the warps of a CTA are folded in shared memory and each CTA folds its candidate into the record under
//                 the record's lock.  The order (|t| descending, row ascending) is total, so the result does not depend
//                 on the order of the folds.
//   column panel  one warp per column segment of the transpose's plan (at most 2048 entries, rows ascending); its lanes
//                 walk the column tiles of 32 C columns in turn and add val P[row][c] in row order.  A column of one
//                 segment is written directly; the segments of a longer column write slots and the last segment to
//                 finish (a ticket per column) adds them in segment order.
#include "bkm_common.cuh"
#include "bkm_csc_plan.cuh"
#include "bkm_csr_rows.cuh"

namespace bkm {
namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;

// ---------------------------------------------------------------------------------------------------------------------
// row panel
// ---------------------------------------------------------------------------------------------------------------------
struct RowPanelArgs {
  const long long* crow;
  const long long* col;
  const void* val;
  long long n;
  int p;
  const double* W;     // [p][l]
  int l;
  void* out;           // [n][ldo], nullable
  long long ldo;
  int out_dtype;
  ColMax* colmax;      // [l], nullable
  long long row_offset;
};

template <typename T, int C>
__global__ void __launch_bounds__(kThreads) csr_panel_kernel(RowPanelArgs a) {
  constexpr int CW = 32 * C;                     // columns per CTA
  __shared__ double r_abs[kWarps][CW];
  __shared__ long long r_row[kWarps][CW];
  __shared__ double r_val[kWarps][CW];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int c0 = blockIdx.y * CW;
  const T* val = reinterpret_cast<const T*>(a.val);
  bool own[C];
#pragma unroll
  for (int j = 0; j < C; ++j) own[j] = c0 + lane + 32 * j < a.l;
  double babs[C], bval[C];
  long long brow[C];
#pragma unroll
  for (int j = 0; j < C; ++j) { babs[j] = -1.0; brow[j] = 0x7fffffffffffffffLL; bval[j] = 0.0; }

  const long long nw = (long long)gridDim.x * kWarps;
#pragma unroll 1
  for (long long i = (long long)blockIdx.x * kWarps + warp; i < a.n; i += nw) {
    double acc[C];
#pragma unroll
    for (int j = 0; j < C; ++j) acc[j] = 0.0;
    double xn = 0.0;
    csr_row_gather<T, C, false>(a.crow, a.col, val, i, a.p, a.W, a.l, c0, own, acc, xn);
    const long long grow = a.row_offset + i;
#pragma unroll
    for (int j = 0; j < C; ++j) {
      if (!own[j]) continue;
      const int cc = c0 + lane + 32 * j;
      if (a.out) {
        if (a.out_dtype == BKM_F64) reinterpret_cast<double*>(a.out)[i * a.ldo + cc] = acc[j];
        else reinterpret_cast<float*>(a.out)[i * a.ldo + cc] = (float)acc[j];
      }
      if (a.colmax && colmax_beats(fabs(acc[j]), grow, babs[j], brow[j])) {
        babs[j] = fabs(acc[j]); brow[j] = grow; bval[j] = acc[j];
      }
    }
  }
  if (!a.colmax) return;

  // ---- CTA fold: the warps in shared memory, then one locked update of the global record per column ----
#pragma unroll
  for (int j = 0; j < C; ++j) {
    r_abs[warp][lane + 32 * j] = babs[j];
    r_row[warp][lane + 32 * j] = brow[j];
    r_val[warp][lane + 32 * j] = bval[j];
  }
  __syncthreads();
  for (int cc = tid; cc < CW && c0 + cc < a.l; cc += kThreads) {
    double ba = r_abs[0][cc], bv = r_val[0][cc];
    long long br = r_row[0][cc];
    for (int w = 1; w < kWarps; ++w)
      if (colmax_beats(r_abs[w][cc], r_row[w][cc], ba, br)) { ba = r_abs[w][cc]; br = r_row[w][cc]; bv = r_val[w][cc]; }
    if (ba >= 0.0) colmax_fold(a.colmax + c0 + cc, ba, br, bv);
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// column panel
// ---------------------------------------------------------------------------------------------------------------------
struct ColPanelArgs {
  const long long* colptr;
  const int* rows;
  const void* vals;
  int p;
  const long long* plan;
  const double* P;     // [n][l]
  int l;
  double* out;         // [p][l]
  double* slot;        // [2 (nnz / SEG + 1)][l]
  unsigned* ticket;    // [p], zero
  int first;
};

template <typename T, int C>
__global__ void __launch_bounds__(kThreads) csc_panel_kernel(ColPanelArgs a) {
  constexpr int CW = 32 * C;
  const int lane = threadIdx.x & 31;
  const long long T_ = a.plan[ST_SEGS];
  const T* vals = reinterpret_cast<const T*>(a.vals);
  const int l = a.l;
  const long long nw = ((long long)gridDim.x * kThreads) >> 5;
#pragma unroll 1
  for (long long t = ((long long)blockIdx.x * kThreads + threadIdx.x) >> 5; t < T_; t += nw) {
    const SegSpan sp = seg_span(a.plan, a.colptr, a.p, t);
    const int j = sp.j;
    const long long ns = sp.ns, e0 = sp.e0, e1 = sp.e1;
    double* slot = seg_slot(a.slot, sp, t, l);
#pragma unroll 1
    for (int c0 = 0; c0 < l; c0 += CW) {
      const int lim = l - c0 - lane;                 // this lane's columns c0 + lane + 32 u with 32 u < lim
      double acc[C];
#pragma unroll
      for (int q = 0; q < C; ++q) acc[q] = 0.0;
#pragma unroll 1
      for (long long eb = e0; eb < e1; eb += 32) {
        int r = 0;
        double v = 0.0;
        if (eb + lane < e1) {
          r = a.rows[eb + lane];
          v = to_f64(vals[eb + lane]);
        }
        const int m = (int)min(32LL, e1 - eb);
#pragma unroll 2
        for (int q = 0; q < m; ++q) {
          const int rq = __shfl_sync(0xffffffffu, r, q);
          const double vq = __shfl_sync(0xffffffffu, v, q);
          const double* pp = a.P + (size_t)rq * l + c0 + lane;
#pragma unroll
          for (int u = 0; u < C; ++u)
            if (32 * u < lim) acc[u] = fma(vq, __ldg(pp + 32 * u), acc[u]);
        }
      }
#pragma unroll
      for (int u = 0; u < C; ++u) {
        if (32 * u >= lim) continue;
        const int cc = c0 + lane + 32 * u;
        if (ns > 1) slot[cc] = acc[u];
        else a.out[(size_t)j * l + cc] = a.first ? acc[u] : a.out[(size_t)j * l + cc] + acc[u];
      }
    }
    if (ns > 1) seg_fold(sp, a.slot, a.ticket, a.out, l, a.first);
  }
}


static int grid_for(long long work, int per_cta, long long cap) {
  long long g = (work + per_cta - 1) / per_cta;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

template <typename T, int C>
static int launch_row_panel(const RowPanelArgs& a, int sms, cudaStream_t s) {
  constexpr int CW = 32 * C;
  const int gy = (a.l + CW - 1) / CW;
  const int gx = grid_for(a.n, kWarps, (8LL * sms + gy - 1) / gy);
  csr_panel_kernel<T, C><<<dim3((unsigned)gx, (unsigned)gy), kThreads, 0, s>>>(a);
  BKM_CUDA_TRY(cudaGetLastError());
  note_launch();
  return 0;
}

template <typename T>
static int row_panel(const RowPanelArgs& a, int sms, cudaStream_t s) {
  if (a.l <= 32) return launch_row_panel<T, 1>(a, sms, s);
  if (a.l <= 64) return launch_row_panel<T, 2>(a, sms, s);
  return launch_row_panel<T, 4>(a, sms, s);
}

template <typename T, int C>
static int launch_col_panel(const ColPanelArgs& a, long long nnz, int sms, cudaStream_t s) {
  const int grid = grid_for(seg_cap(a.p, nnz), kWarps, 16LL * sms);
  csc_panel_kernel<T, C><<<grid, kThreads, 0, s>>>(a);
  BKM_CUDA_TRY(cudaGetLastError());
  note_launch();
  return 0;
}

template <typename T>
static int col_panel(const ColPanelArgs& a, long long nnz, int sms, cudaStream_t s) {
  if (a.l <= 32) return launch_col_panel<T, 1>(a, nnz, sms, s);
  if (a.l <= 64) return launch_col_panel<T, 2>(a, nnz, sms, s);
  return launch_col_panel<T, 4>(a, nnz, sms, s);
}

}  // namespace
}  // namespace bkm

using namespace bkm;

extern "C" int bkm_csr_panel_chunk(const int64_t* crow, const int64_t* col, const void* val, int val_dtype, int64_t n,
                                   int p, int64_t nnz, const double* W, int l, void* out, int64_t ldo, int out_dtype,
                                   void* colmax, int64_t row_offset, void* stream) {
  if (n < 0 || p <= 0 || nnz < 0 || l <= 0 || !crow || !W) return BKM_EINVAL;
  if (nnz > 0 && (!col || !val)) return BKM_EINVAL;
  if (val_dtype != BKM_F32 && val_dtype != BKM_F64) return BKM_EDTYPE;
  if (out && (ldo < l || (out_dtype != BKM_F32 && out_dtype != BKM_F64))) return BKM_EINVAL;
  if (n == 0 || (!out && !colmax)) return 0;
  RowPanelArgs a;
  a.crow = reinterpret_cast<const long long*>(crow);
  a.col = reinterpret_cast<const long long*>(col);
  a.val = val; a.n = n; a.p = p; a.W = W; a.l = l; a.out = out; a.ldo = ldo; a.out_dtype = out_dtype;
  a.colmax = reinterpret_cast<ColMax*>(colmax); a.row_offset = row_offset;
  const int sms = sm_count_or_default();
  cudaStream_t s = (cudaStream_t)stream;
  if (val_dtype == BKM_F32) return row_panel<float>(a, sms, s);
  return row_panel<double>(a, sms, s);
}

extern "C" int bkm_csc_panel_workspace_bytes(int p, int64_t nnz, int l, size_t* out) {
  if (!out || p <= 0 || nnz < 0 || l <= 0) return BKM_EINVAL;
  *out = seg_fold_ws(p, nnz, l);
  return 0;
}

extern "C" int bkm_csc_panel_chunk(const int64_t* colptr, const int32_t* rows, const void* vals, int val_dtype, int p,
                                   int64_t nnz, const int64_t* plan, const double* P, int l, double* out,
                                   void* workspace, size_t ws_bytes, int flags, void* stream) {
  if (p <= 0 || nnz < 0 || l <= 0 || !colptr || !plan || !out || !workspace) return BKM_EINVAL;
  if (nnz > 0 && (!rows || !vals || !P)) return BKM_EINVAL;
  if (val_dtype != BKM_F32 && val_dtype != BKM_F64) return BKM_EDTYPE;
  if (ws_bytes < seg_fold_ws(p, nnz, l)) return BKM_EWORKSPACE;
  cudaStream_t s = (cudaStream_t)stream;
  unsigned char* ws = reinterpret_cast<unsigned char*>(workspace);
  ColPanelArgs a;
  a.colptr = reinterpret_cast<const long long*>(colptr);
  a.rows = rows; a.vals = vals; a.p = p; a.plan = reinterpret_cast<const long long*>(plan);
  a.P = P; a.l = l; a.out = out;
  a.slot = reinterpret_cast<double*>(ws);
  a.ticket = reinterpret_cast<unsigned*>(ws + seg_slots_bytes(nnz, l));
  a.first = (flags & BKM_FLAG_FIRST_CHUNK) ? 1 : 0;
  BKM_CUDA_TRY(cudaMemsetAsync(a.ticket, 0, (size_t)p * 4, s));
  const int sms = sm_count_or_default();
  if (val_dtype == BKM_F32) return col_panel<float>(a, nnz, sms, s);
  return col_panel<double>(a, nnz, sms, s);
}
