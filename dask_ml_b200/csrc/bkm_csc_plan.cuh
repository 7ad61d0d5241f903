// bkm_csc_plan.cuh — the segment plan of a sparse block's transpose, written by bkm_csr_transpose_chunk
// (bkm_glm_sparse.cu) and read by the column passes there, in bkm_svd_sparse.cu and in bkm_kmeans_sparse.cu; and the
// segment-and-ticket fold of the column passes whose per-column result is a row of l float64 values.
#pragma once

namespace bkm {
namespace {

constexpr long long SEG = 2048;        // entries per column segment (column passes)
// plan layout (int64): [status (4) | seg_off (d + 1) | gseg_off (d + 1) | seg_col (int32, seg_cap(d, nnz))]
// status = [non-canonical flag | segments T | Gram slots | longest column]
enum { ST_BAD = 0, ST_SEGS = 1, ST_SLOTS = 2, ST_MAXLEN = 3, ST_N = 4 };

// an upper bound of the segments T: one per column, plus one per further SEG entries of a longer column
static inline long long seg_cap(int d, long long nnz) { return (long long)d + nnz / SEG + 1; }

#ifdef __CUDACC__
// Segment t of the plan: its column j, the column's first segment s0 and segment count ns, and its entry range
// [e0, e1) of the transpose (at most SEG entries, rows ascending).
struct SegSpan {
  int j;
  long long s0, ns, e0, e1;
};

__device__ __forceinline__ SegSpan seg_span(const long long* plan, const long long* colptr, int d, long long t) {
  const long long* seg_off = plan + ST_N;
  const int* seg_col = reinterpret_cast<const int*>(plan + ST_N + 2 * ((long long)d + 1));
  SegSpan s;
  s.j = seg_col[t];
  s.s0 = seg_off[s.j];
  s.ns = seg_off[s.j + 1] - s.s0;
  s.e0 = colptr[s.j] + (t - s.s0) * SEG;
  s.e1 = min(colptr[s.j + 1], s.e0 + SEG);
  return s;
}

// The slot row (l float64) of segment t of a multi-segment column.  s0 - j is the number of segments beyond the first
// of every column before j, so the slots 2 (s0 - j) + (t - s0) of different segments do not overlap and stay below
// 2 (nnz / SEG + 1).
__device__ __forceinline__ double* seg_slot(double* slots, const SegSpan& s, long long t, int l) {
  return slots + (size_t)(2 * (s.s0 - s.j) + (t - s.s0)) * l;
}

// Called by the warp of every segment of a multi-segment column after it wrote its slot: the last one to finish (a
// ticket per column, reset here) adds the column's slots in segment order into out[j][0..l), written over when `first`
// and added to otherwise.
__device__ __forceinline__ void seg_fold(const SegSpan& s, const double* slots, unsigned* ticket, double* out, int l,
                                         int first) {
  if (!last_warp(ticket + s.j, (unsigned)s.ns)) return;
  const int lane = threadIdx.x & 31;
  const double* src = slots + (size_t)(2 * (s.s0 - s.j)) * l;
  for (int cc = lane; cc < l; cc += 32) {
    double v = 0.0;
    for (long long u = 0; u < s.ns; ++u) v += __ldcg(src + (size_t)u * l + cc);
    out[(size_t)s.j * l + cc] = first ? v : out[(size_t)s.j * l + cc] + v;
  }
  if (lane == 0) ticket[s.j] = 0u;
}

// Workspace of a seg_fold pass: the slots, then one ticket per column (zeroed at launch)
static size_t seg_slots_bytes(long long nnz, int l) { return align_up((size_t)2 * (nnz / SEG + 1) * l * 8, 256); }
static size_t seg_fold_ws(int d, long long nnz, int l) { return seg_slots_bytes(nnz, l) + align_up((size_t)d * 4, 256); }
#endif

}  // namespace
}  // namespace bkm
