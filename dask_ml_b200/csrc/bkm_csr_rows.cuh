// bkm_csr_rows.cuh — the row body of the CSR panel passes: one warp gathers a dense float64 panel's rows for the entries
// of one CSR row.  Used by bkm_csr_panel_chunk (bkm_svd_sparse.cu), bkm_csr_assign_chunk and bkm_nb_csr_jll_chunk
// (bkm_kmeans_sparse.cu).
#pragma once

namespace bkm {
namespace {

__device__ __forceinline__ double to_f64(float v) { return (double)v; }
__device__ __forceinline__ double to_f64(double v) { return v; }

// Row i of the block against W [p][l] float64 row-major: the lanes own the columns c0 + lane + 32 j (own[j]) and add
// val W[col][c] to acc[j] by fma.  The warp loads 32 entries of the row at a time and takes them one by one in stored
// (ascending column) order, so each entry gathers l * 8 contiguous bytes of W.  An entry whose column is outside [0, p)
// is skipped.  With NORM every lane also adds val^2 to xn in the same order (the row's squared norm).  With BIN the
// entries are binarised as scikit-learn binarises a sparse matrix: an entry with val > thr counts as 1, any other is
// dropped (it adds nothing, not 0 W).
template <typename T, int C, bool NORM, bool BIN = false>
__device__ __forceinline__ void csr_row_gather(const long long* __restrict__ crow, const long long* __restrict__ col,
                                               const T* __restrict__ val, long long i, int p,
                                               const double* __restrict__ W, int l, int c0, const bool (&own)[C],
                                               double (&acc)[C], double& xn, double thr = 0.0) {
  const int lane = threadIdx.x & 31;
  const long long k0 = crow[i], k1 = crow[i + 1];
#pragma unroll 1
  for (long long e0 = k0; e0 < k1; e0 += 32) {
    long long c = -1;
    double v = 0.0;
    if (e0 + lane < k1) {
      c = col[e0 + lane];
      v = to_f64(val[e0 + lane]);
    }
    const int m = (int)min(32LL, k1 - e0);
#pragma unroll 4
    for (int q = 0; q < m; ++q) {
      const long long cq = __shfl_sync(0xffffffffu, c, q);
      double vq = __shfl_sync(0xffffffffu, v, q);
      if ((unsigned long long)cq >= (unsigned long long)p) continue;      // uniform over the warp
      if (BIN) {
        if (!(vq > thr)) continue;                                        // uniform over the warp
        vq = 1.0;
      }
      if (NORM) xn = fma(vq, vq, xn);
      const double* w = W + (size_t)cq * l + c0 + lane;
#pragma unroll
      for (int j = 0; j < C; ++j)
        if (own[j]) acc[j] = fma(vq, __ldg(w + 32 * j), acc[j]);
    }
  }
}

}  // namespace
}  // namespace bkm
