// bkm_pca.cu — the two passes of PCA / TruncatedSVD over row chunks, in float64 on the fp64 tensor cores (sm_90a).
//
//   bkm_gram_chunk     m (+)= sum_i (x_i - s),  G (+)= sum_i (x_i - s)(x_i - s)^T          (d, d) float64, symmetric
//   bkm_project_chunk  out = (x - s) W^T cast to out_dtype, and per column the signed arg-max of |out| (svd_flip)
//
// Both convert the rows to float64 (minus the shift) in shared memory and multiply with
// mma.sync.aligned.m16n8k16.row.col.f64 (DMMA.16x8x16): for fp32 and bf16 rows the products are exact float64 products
// of the shifted rows, so the results differ from a float64 numpy computation only by the order of the sums.
//
// Gram: the features are cut into 64-wide blocks; one CTA column per block pair (bi <= bj, the tiles on or above the
// diagonal) and S row splits per pair.  Each CTA streams its rows in 32-row tiles: the two feature segments of every row
// are bulk-copied (cp.async.bulk, one mbarrier per stage, double-buffered) into shared memory, then widened to float64
// and shifted into the operand tiles.  Rows that cannot be bulk-copied (a pitch, base or width that is not a multiple
// of 16 bytes) are read with plain loads by the same conversion step.  Every CTA writes its 64x64 partial (and, on
// the diagonal, its 64 column sums) to the workspace; the last CTA of a pair to finish (a ticket counter) adds the S
// partials in split order and writes the tile and its mirror.  The sums therefore have a fixed order: two calls with
// the same inputs give the same bits.
#include "bkm_common.cuh"
#include "bkm_ptx.cuh"
#include <cuda_bf16.h>

namespace bkm {
namespace {

using namespace ptx;

constexpr int kThreads = 256;
constexpr int GB = 64;          // gram: feature block (tile edge)
constexpr int GR = 32;          // gram: rows per staged tile
constexpr int GP = GB + 4;      // float64 operand pitch: lanes (t, g) read word t*GP + g, conflict-free per half-warp
constexpr int PR = 64;          // project: rows per tile
constexpr int PF = 32;          // project: features per staged step
constexpr int PP = PF + 4;      // project operand pitch

__device__ __forceinline__ double to_f64(float v) { return (double)v; }
__device__ __forceinline__ double to_f64(double v) { return v; }
__device__ __forceinline__ double to_f64(__nv_bfloat16 v) { return (double)__bfloat162float(v); }

// D = A B + D, A 16x16 (row), B 16x8 (col), float64.  Fragments (g = lane / 4, t = lane % 4):
//   a[i] = A[g + 8 (i & 1)][t + 4 (i >> 1)],  b[i] = B[t + 4 i][g],  c = {(g, 2t), (g, 2t+1), (g+8, 2t), (g+8, 2t+1)}
__device__ __forceinline__ void dmma16816(double (&c)[4], const double (&a)[8], const double (&b)[4]) {
  asm("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, "
      "{%12,%13,%14,%15}, {%0,%1,%2,%3};"
      : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
      : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]),
        "d"(b[0]), "d"(b[1]), "d"(b[2]), "d"(b[3]));
}

// ------------------------------------------------------------------------------------------------------------ gram
struct GramGeom {
  int nb;                  // feature blocks
  int pairs;               // nb (nb + 1) / 2 upper tiles
  int splits;              // row splits per tile
  long long rows_per_split;  // a multiple of GR
  size_t off_part, off_cpart, off_ticket, total;
};

static GramGeom gram_geom(long long n, int d, int sm_count) {
  GramGeom g;
  g.nb = (d + GB - 1) / GB;
  g.pairs = g.nb * (g.nb + 1) / 2;
  const long long tiles = (n + GR - 1) / GR;
  long long s = (2LL * sm_count + g.pairs - 1) / g.pairs;        // about two CTAs per SM in all
  if (s > tiles) s = tiles;
  if (s < 1) s = 1;
  g.rows_per_split = ((tiles + s - 1) / s) * GR;
  if (g.rows_per_split < GR) g.rows_per_split = GR;
  g.splits = (int)((n + g.rows_per_split - 1) / g.rows_per_split);
  if (g.splits < 1) g.splits = 1;
  size_t o = 0;
  g.off_part = o;   o = align_up(o + (size_t)g.pairs * g.splits * GB * GB * 8, 256);
  g.off_cpart = o;  o = align_up(o + (size_t)g.nb * g.splits * GB * 8, 256);
  g.off_ticket = o; o = align_up(o + (size_t)g.pairs * 4, 256);
  g.total = o;
  return g;
}

struct GramArgs {
  const void* X;
  long long n;
  int d;
  long long ldx;
  const double* shift;
  double* colsum;
  double* gram;
  double* part;
  double* cpart;
  unsigned int* ticket;
  int nb, splits;
  long long rows_per_split;
  int first;
  int bulk;
  const double* w;         // WEIGHTED: the row weights [n]
};

template <typename T>
static size_t gram_smem_bytes() {
  return (size_t)2 * GR * GP * 8            // float64 operand tiles (block i, block j)
         + (size_t)2 * 2 * GR * GB * sizeof(T)  // raw rows: 2 stages x 2 blocks
         + 4 * GB * 8                        // column-sum partials of the diagonal tiles
         + 16;                               // two mbarriers
}

// WEIGHTED: G (+)= sum_i w_i x_i x_i^T, no shift and no column sums.  The weight scales the block-j operand tile as it
// is widened, so the diagonal tiles convert their one staged block twice (block i plain, block j weighted).
template <typename T, bool WEIGHTED = false>
__global__ void __launch_bounds__(kThreads) gram_kernel(GramArgs a) {
  extern __shared__ __align__(128) unsigned char smem[];
  double* Fi = reinterpret_cast<double*>(smem);
  T* raw = reinterpret_cast<T*>(smem + 2 * GR * GP * 8);
  double* cred = reinterpret_cast<double*>(smem + 2 * GR * GP * 8 + 2 * 2 * GR * GB * sizeof(T));
  const uint32_t bar0 = smem_u32(cred + 4 * GB);

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int d = a.d;
  const int pair = blockIdx.x, split = blockIdx.y;
  int bi = 0, rem = pair;
  while (rem >= a.nb - bi) { rem -= a.nb - bi; ++bi; }
  const int bj = bi + rem;
  const bool diag = bi == bj;
  const int f0i = bi * GB, f0j = bj * GB;
  const int wi = min(GB, d - f0i), wj = min(GB, d - f0j);
  double* Fj = (diag && !WEIGHTED) ? Fi : Fi + GR * GP;
  const int nblk = diag ? 1 : 2;
  const int ncvt = WEIGHTED ? 2 : nblk;         // operand tiles converted per staged tile

  const long long rb = (long long)split * a.rows_per_split;
  const long long re = min(a.n, rb + a.rows_per_split);
  const long long ntile = re > rb ? (re - rb + GR - 1) / GR : 0;
  const T* X = reinterpret_cast<const T*>(a.X);

  if (a.bulk && tid == 0) {
    mbar_init(bar0, 1);
    mbar_init(bar0 + 8, 1);
    mbar_fence_init();
  }
  __syncthreads();

  // warp 0 issues the copies of tile t into stage t & 1: one bulk copy per row and feature block
  auto issue = [&](long long t) {
    const int st = (int)(t & 1);
    const long long r0 = rb + t * GR;
    const int rows = (int)min((long long)GR, re - r0);
    const uint32_t bar = bar0 + 8u * st;
    if (lane == 0) mbar_expect_tx(bar, (uint32_t)(rows * (wi + (diag ? 0 : wj)) * sizeof(T)));
    __syncwarp();
    if (lane < rows) {
      for (int b = 0; b < nblk; ++b) {
        const int f0 = b ? f0j : f0i, w = b ? wj : wi;
        T* dst = raw + ((size_t)(st * 2 + b) * GR + lane) * GB;
        bulk_g2s(smem_u32(dst), X + (r0 + lane) * a.ldx + f0, (uint32_t)(w * sizeof(T)), bar);
      }
    }
  };
  if (a.bulk && warp == 0) {
    if (ntile > 0) issue(0);
    if (ntile > 1) issue(1);
  }

  const int g = lane >> 2, tq = lane & 3;
  const int mb = warp & 3, nh = warp >> 2;     // warp tile: rows mb*16.. of block i, columns nh*32.. of block j
  const bool mact = mb * 16 < wi;
  double acc[4][4];
#pragma unroll
  for (int nt = 0; nt < 4; ++nt)
#pragma unroll
    for (int q = 0; q < 4; ++q) acc[nt][q] = 0.0;
  double csum = 0.0;                            // diagonal tiles: column tid % 64, rows tid / 64 + 4 q
  const int cf = tid & (GB - 1);

#pragma unroll 1
  for (long long t = 0; t < ntile; ++t) {
    const int st = (int)(t & 1);
    const long long r0 = rb + t * GR;
    const int rows = (int)min((long long)GR, re - r0);
    if (a.bulk) mbar_wait(bar0 + 8u * st, (uint32_t)((t >> 1) & 1));
    __syncthreads();                            // the previous tile's MMAs are done with Fi / Fj
#pragma unroll 1
    for (int b = 0; b < ncvt; ++b) {
      double* F = b ? Fj : Fi;
      const int f0 = b ? f0j : f0i, w = b ? wj : wi;
      const T* rs = raw + (size_t)(st * 2 + (WEIGHTED && diag ? 0 : b)) * GR * GB;
      const double sh = WEIGHTED ? 0.0 : (cf < w ? a.shift[f0 + cf] : 0.0);
#pragma unroll 4
      for (int e = tid; e < GR * GB; e += kThreads) {
        const int r = e >> 6;
        double v = 0.0;
        if (r < rows && cf < w) {
          const T x = a.bulk ? rs[r * GB + cf] : X[(r0 + r) * a.ldx + f0 + cf];
          v = to_f64(x) - sh;
          if (WEIGHTED && b) v *= a.w[r0 + r];
        }
        F[r * GP + cf] = v;
        if (diag && !WEIGHTED) csum += v;
      }
    }
    __syncthreads();
    if (a.bulk && warp == 0 && t + 2 < ntile) {
      fence_proxy_async();                      // the generic reads of this stage precede the async writes
      issue(t + 2);
    }
    if (mact) {
#pragma unroll
      for (int ks = 0; ks < GR / 16; ++ks) {
        const int k0 = ks * 16;
        double af[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) af[i] = Fi[(k0 + tq + 4 * (i >> 1)) * GP + mb * 16 + g + 8 * (i & 1)];
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
          if (nh * 32 + nt * 8 < wj) {
            double bf[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) bf[i] = Fj[(k0 + tq + 4 * i) * GP + nh * 32 + nt * 8 + g];
            dmma16816(acc[nt], af, bf);
          }
        }
      }
    }
  }

  // ---- this CTA's partial tile and column sums ----
  const size_t tile_elems = (size_t)GB * GB;
  double* P = a.part + ((size_t)pair * a.splits + split) * tile_elems;
#pragma unroll
  for (int nt = 0; nt < 4; ++nt) {
    const int r = mb * 16 + g, c = nh * 32 + nt * 8 + 2 * tq;
    P[r * GB + c] = acc[nt][0];
    P[r * GB + c + 1] = acc[nt][1];
    P[(r + 8) * GB + c] = acc[nt][2];
    P[(r + 8) * GB + c + 1] = acc[nt][3];
  }
  if (diag && !WEIGHTED) {
    cred[(tid >> 6) * GB + cf] = csum;
    __syncthreads();
    if (tid < GB)
      a.cpart[((size_t)bi * a.splits + split) * GB + tid] = ((cred[tid] + cred[GB + tid]) + cred[2 * GB + tid]) + cred[3 * GB + tid];
  }
  if (!last_block(&a.ticket[pair], (unsigned)a.splits)) return;

  // ---- the last CTA of the tile: the splits in order, then the tile and its mirror ----
  const double* P0 = a.part + (size_t)pair * a.splits * tile_elems;
  for (int e = tid; e < GB * GB; e += kThreads) {
    const int r = e >> 6, c = e & (GB - 1);
    const int I = f0i + r, J = f0j + c;
    if (r >= wi || c >= wj || I > J) continue;
    double v = 0.0;
    for (int s = 0; s < a.splits; ++s) v += __ldcg(P0 + (size_t)s * tile_elems + e);
    double* gij = a.gram + (size_t)I * d + J;
    double* gji = a.gram + (size_t)J * d + I;
    if (a.first) {
      *gij = v;
      *gji = v;
    } else {
      const double u = *gij + v;
      *gij = u;
      *gji = u;
    }
  }
  if (diag && !WEIGHTED && tid < wi) {
    double v = 0.0;
    for (int s = 0; s < a.splits; ++s) v += __ldcg(a.cpart + ((size_t)bi * a.splits + s) * GB + tid);
    a.colsum[f0i + tid] = a.first ? v : a.colsum[f0i + tid] + v;
  }
  if (tid == 0) a.ticket[pair] = 0u;
}

// ------------------------------------------------------------------------------------------------------- project
// The arg-max epilogue folds into ColMax records (bkm_common.cuh).
struct ProjArgs {
  const void* X;
  long long n;
  int d;
  long long ldx;
  const double* shift;     // nullable
  const double* W;         // [k][d]
  int k;
  void* out;               // nullable
  long long ldo;
  int out_dtype;
  ColMax* colmax;          // nullable
  long long row_offset;
};

template <typename T, int NT>
__global__ void __launch_bounds__(kThreads) project_kernel(ProjArgs a) {
  constexpr int CW = 2 * NT * 8;                // columns per CTA
  __shared__ __align__(16) double Xs[PR * PP];
  __shared__ __align__(16) double Ws[CW * PP];
  __shared__ double r_abs[4][CW];
  __shared__ long long r_row[4][CW];
  __shared__ double r_val[4][CW];

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, tq = lane & 3;
  const int mb = warp & 3, nh = warp >> 2;
  const int d = a.d;
  const int c0 = blockIdx.y * CW;
  const int kw = min(CW, a.k - c0);
  const T* X = reinterpret_cast<const T*>(a.X);
  const long long ntiles = (a.n + PR - 1) / PR;

  double babs[NT][2], bval[NT][2];
  long long brow[NT][2];
#pragma unroll
  for (int nt = 0; nt < NT; ++nt)
#pragma unroll
    for (int j = 0; j < 2; ++j) { babs[nt][j] = -1.0; brow[nt][j] = 0x7fffffffffffffffLL; bval[nt][j] = 0.0; }

#pragma unroll 1
  for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const long long r0 = tile * PR;
    const int rows = (int)min((long long)PR, a.n - r0);
    double acc[NT][4];
#pragma unroll
    for (int nt = 0; nt < NT; ++nt)
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[nt][q] = 0.0;
#pragma unroll 1
    for (int f0 = 0; f0 < d; f0 += PF) {
      __syncthreads();
      const int f = tid & (PF - 1);
      const bool fin = f0 + f < d;
      const double sh = (fin && a.shift) ? a.shift[f0 + f] : 0.0;
#pragma unroll 4
      for (int e = tid; e < PR * PF; e += kThreads) {
        const int r = e >> 5;
        Xs[r * PP + f] = (r < rows && fin) ? to_f64(X[(r0 + r) * a.ldx + f0 + f]) - sh : 0.0;
      }
      for (int e = tid; e < CW * PF; e += kThreads) {
        const int c = e >> 5;
        Ws[c * PP + f] = (c < kw && fin) ? a.W[(size_t)(c0 + c) * d + f0 + f] : 0.0;
      }
      __syncthreads();
#pragma unroll
      for (int ks = 0; ks < PF / 16; ++ks) {
        const int k0 = ks * 16;
        double af[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) af[i] = Xs[(mb * 16 + g + 8 * (i & 1)) * PP + k0 + tq + 4 * (i >> 1)];
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) {
          double bf[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) bf[i] = Ws[(nh * NT * 8 + nt * 8 + g) * PP + k0 + tq + 4 * i];
          dmma16816(acc[nt], af, bf);
        }
      }
    }
    // ---- epilogue: the cast output and the running arg-max of every column this thread holds ----
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = mb * 16 + g + 8 * h;
        if (r >= rows) continue;
        const long long grow = a.row_offset + r0 + r;
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int c = nh * NT * 8 + nt * 8 + 2 * tq + j;
          if (c >= kw) continue;
          const double v = acc[nt][2 * h + j];
          if (a.out) {
            if (a.out_dtype == BKM_F64)
              reinterpret_cast<double*>(a.out)[(r0 + r) * a.ldo + c0 + c] = v;
            else
              reinterpret_cast<float*>(a.out)[(r0 + r) * a.ldo + c0 + c] = (float)v;
          }
          if (a.colmax && colmax_beats(fabs(v), grow, babs[nt][j], brow[nt][j])) {
            babs[nt][j] = fabs(v); brow[nt][j] = grow; bval[nt][j] = v;
          }
        }
      }
    }
  }
  if (!a.colmax) return;

  // ---- CTA fold: the 8 row groups of a warp (shuffles), then the 4 warps of a column half (shared), then one locked
  // update of the global record per column ----
#pragma unroll
  for (int nt = 0; nt < NT; ++nt)
#pragma unroll
    for (int j = 0; j < 2; ++j) {
#pragma unroll
      for (int off = 4; off < 32; off <<= 1) {
        const double oa = __shfl_xor_sync(0xffffffffu, babs[nt][j], off);
        const long long orow = __shfl_xor_sync(0xffffffffu, brow[nt][j], off);
        const double ov = __shfl_xor_sync(0xffffffffu, bval[nt][j], off);
        if (colmax_beats(oa, orow, babs[nt][j], brow[nt][j])) { babs[nt][j] = oa; brow[nt][j] = orow; bval[nt][j] = ov; }
      }
      if (g == 0) {
        const int c = nh * NT * 8 + nt * 8 + 2 * tq + j;
        r_abs[mb][c] = babs[nt][j]; r_row[mb][c] = brow[nt][j]; r_val[mb][c] = bval[nt][j];
      }
    }
  __syncthreads();
  if (tid < kw) {
    double ba = r_abs[0][tid], bv = r_val[0][tid];
    long long br = r_row[0][tid];
    for (int m = 1; m < 4; ++m)
      if (colmax_beats(r_abs[m][tid], r_row[m][tid], ba, br)) { ba = r_abs[m][tid]; br = r_row[m][tid]; bv = r_val[m][tid]; }
    if (ba >= 0.0) colmax_fold(a.colmax + c0 + tid, ba, br, bv);
  }
}

template <typename T, bool WEIGHTED = false>
static int launch_gram(const GramArgs& a, int pairs, int splits, cudaStream_t s) {
  const size_t sm = gram_smem_bytes<T>();
  BKM_CUDA_TRY(cudaFuncSetAttribute(gram_kernel<T, WEIGHTED>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
  gram_kernel<T, WEIGHTED><<<dim3(pairs, splits), kThreads, sm, s>>>(a);
  BKM_CUDA_TRY(cudaGetLastError());
  note_launch();
  return 0;
}

template <typename T, int NT>
static int launch_project_nt(const ProjArgs& a, int sms, cudaStream_t s) {
  constexpr int CW = 2 * NT * 8;
  const int gy = (a.k + CW - 1) / CW;
  const long long ntiles = (a.n + PR - 1) / PR;
  long long gx = (4LL * sms + gy - 1) / gy;
  if (gx > ntiles) gx = ntiles;
  if (gx < 1) gx = 1;
  project_kernel<T, NT><<<dim3((unsigned)gx, gy), kThreads, 0, s>>>(a);
  BKM_CUDA_TRY(cudaGetLastError());
  note_launch();
  return 0;
}

template <typename T>
static int launch_project(const ProjArgs& a, int sms, cudaStream_t s) {
  if (a.k <= 16) return launch_project_nt<T, 1>(a, sms, s);
  if (a.k <= 32) return launch_project_nt<T, 2>(a, sms, s);
  return launch_project_nt<T, 4>(a, sms, s);
}

template <bool WEIGHTED>
static int gram_run(const void* X, int64_t n, int d, int64_t ldx, int x_dtype, const double* shift, double* colsum,
                    double* gram, const double* w, const GramGeom& G, void* workspace, int flags, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  unsigned char* ws = reinterpret_cast<unsigned char*>(workspace);
  BKM_CUDA_TRY(cudaMemsetAsync(ws + G.off_ticket, 0, (size_t)G.pairs * 4, s));
  const size_t es = elem_size(x_dtype);
  GramArgs a;
  a.X = X; a.n = n; a.d = d; a.ldx = ldx; a.shift = shift; a.colsum = colsum; a.gram = gram; a.w = w;
  a.part = reinterpret_cast<double*>(ws + G.off_part);
  a.cpart = reinterpret_cast<double*>(ws + G.off_cpart);
  a.ticket = reinterpret_cast<unsigned int*>(ws + G.off_ticket);
  a.nb = G.nb; a.splits = G.splits; a.rows_per_split = G.rows_per_split;
  a.first = (flags & BKM_FLAG_FIRST_CHUNK) ? 1 : 0;
  // bulk copies need 16-byte aligned sources and sizes: base, row pitch and (for the last block) the row width
  a.bulk = n > 0 && ((uintptr_t)X % 16 == 0) && ((ldx * es) % 16 == 0) && ((d * es) % 16 == 0);
  if (x_dtype == BKM_F32) return launch_gram<float, WEIGHTED>(a, G.pairs, G.splits, s);
  if (x_dtype == BKM_F64) return launch_gram<double, WEIGHTED>(a, G.pairs, G.splits, s);
  return launch_gram<__nv_bfloat16, WEIGHTED>(a, G.pairs, G.splits, s);
}

}  // namespace
}  // namespace bkm

using namespace bkm;

extern "C" int bkm_gram_workspace_bytes(int64_t n, int d, size_t* out) {
  if (!out || n < 0 || d <= 0) return BKM_EINVAL;
  *out = gram_geom(n, d, sm_count_or_default()).total;
  return 0;
}

extern "C" int bkm_gram_chunk(const void* X, int64_t n, int d, int64_t ldx, int x_dtype, const double* shift,
                              double* colsum, double* gram, void* workspace, size_t ws_bytes, int flags, void* stream) {
  if (n < 0 || d <= 0 || ldx < d || !shift || !colsum || !gram || !workspace) return BKM_EINVAL;
  if (n > 0 && !X) return BKM_EINVAL;
  if (!dtype_ok(x_dtype)) return BKM_EDTYPE;
  int sms = 0;
  const int rc = sm_count(&sms);
  if (rc) return rc;
  const GramGeom G = gram_geom(n, d, sms);
  if (ws_bytes < G.total) return BKM_EWORKSPACE;
  return gram_run<false>(X, n, d, ldx, x_dtype, shift, colsum, gram, nullptr, G, workspace, flags, stream);
}

extern "C" int bkm_gram_weighted_chunk(const void* X, int64_t n, int d, int64_t ldx, int x_dtype, const double* w,
                                       double* gram, void* workspace, size_t ws_bytes, int flags, void* stream) {
  if (n < 0 || d <= 0 || ldx < d || !gram || !workspace) return BKM_EINVAL;
  if (n > 0 && (!X || !w)) return BKM_EINVAL;
  if (!dtype_ok(x_dtype)) return BKM_EDTYPE;
  int sms = 0;
  const int rc = sm_count(&sms);
  if (rc) return rc;
  const GramGeom G = gram_geom(n, d, sms);
  if (ws_bytes < G.total) return BKM_EWORKSPACE;
  return gram_run<true>(X, n, d, ldx, x_dtype, nullptr, nullptr, gram, w, G, workspace, flags, stream);
}

extern "C" int bkm_project_chunk(const void* X, int64_t n, int d, int64_t ldx, int x_dtype, const double* shift,
                                 const double* W, int k, void* out, int64_t ldo, int out_dtype, void* colmax,
                                 int64_t row_offset, int flags, void* stream) {
  (void)flags;
  if (n < 0 || d <= 0 || k <= 0 || ldx < d || !W) return BKM_EINVAL;
  if (n > 0 && !X) return BKM_EINVAL;
  if (!dtype_ok(x_dtype)) return BKM_EDTYPE;
  if (out && (ldo < k || (out_dtype != BKM_F32 && out_dtype != BKM_F64))) return BKM_EINVAL;
  int sms = 0;
  const int rc = sm_count(&sms);
  if (rc) return rc;
  ProjArgs a;
  a.X = X; a.n = n; a.d = d; a.ldx = ldx; a.shift = shift; a.W = W; a.k = k; a.out = out; a.ldo = ldo;
  a.out_dtype = out_dtype; a.colmax = reinterpret_cast<ColMax*>(colmax); a.row_offset = row_offset;
  cudaStream_t s = (cudaStream_t)stream;
  if (x_dtype == BKM_F32) return launch_project<float>(a, sms, s);
  if (x_dtype == BKM_F64) return launch_project<double>(a, sms, s);
  return launch_project<__nv_bfloat16>(a, sms, s);
}
