// bkm_csc_plan.cuh — the segment plan of a sparse block's transpose, written by bkm_csr_transpose_chunk
// (bkm_glm_sparse.cu) and read by the column passes there and in bkm_svd_sparse.cu.
#pragma once

namespace bkm {
namespace {

constexpr long long SEG = 2048;        // entries per column segment (column passes)
// plan layout (int64): [status (4) | seg_off (d + 1) | gseg_off (d + 1) | seg_col (int32, seg_cap(d, nnz))]
// status = [non-canonical flag | segments T | Gram slots | longest column]
enum { ST_BAD = 0, ST_SEGS = 1, ST_SLOTS = 2, ST_MAXLEN = 3, ST_N = 4 };

// an upper bound of the segments T: one per column, plus one per further SEG entries of a longer column
static inline long long seg_cap(int d, long long nnz) { return (long long)d + nnz / SEG + 1; }

}  // namespace
}  // namespace bkm
