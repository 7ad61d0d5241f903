"""Canonical CSR blocks built to reach the limits of the sparse passes, and a numpy restatement of the transpose's plan
and of the plain-add column passes, in the kernels' order.

The plan (bkm_csc_plan.cuh, written by bkm_csr_transpose_chunk in bkm_glm_sparse.cu) cuts each column into segments of
SEG entries; the segments of a column of more than one write slots 2 (s0 - j) + (t - s0) that the last segment folds in
segment order.  The weighted CSR Gram walks runs of GS segments, and a column of more than one run has Gram slots
gseg_off[j] + s / GS.  The row passes load a row 32 entries at a time (bkm_csr_rows.cuh) and walk column tiles of 32 C;
the GLM row pass sums a row with G lanes.  The small host rules that pick those shapes are restated below with the
source lines they follow, so a test can assert which limits a case reaches."""
import types

import numpy as np
import scipy.sparse as sp

SEG = 2048               # entries per column segment: bkm_csc_plan.cuh:9
GS = 32                  # segments per Gram run: bkm_glm_sparse.cu:35
KWARPS = 8               # warps of a 256-thread CTA
COLSUM_WINDOW = 3200     # keep rows per colsum launch: bkm_kmeans_sparse.cu:95
MAX_LABEL_SUM_K = 25600  # the largest k with one k-wide accumulator in 200 KB: bkm_kmeans_sparse.cu:390-393

# the widths the GPU tests run each pass at (tests/test_gpu_sparse_plan.py), checked for their reach on the CPU
L_PANEL = [1, 32, 33, 65, 129, 257]              # csr_panel / csc_panel: C = 1, 2, 4, and up to 3 blockIdx.y tiles
K_ASSIGN = [1, 33, 65, 129, 257]                 # csr_assign
K_LABEL = [1, 32, 33, 3200, 3201, 25600]         # csc_label_sums: 8, 7 and 1 warps
K_NB = [2, 33, 129]                              # nb_csr_jll
L_COLSUM = [3200, 3201, 6401]                    # csr_kernel_colsum: 1, 2 and 3 windows
L_EMBED = [129, 257]                             # csr_nystrom_embed: several tiles of 128 keep rows
GRAM_D = [18, 1536, 1537, 4096]                  # gram_weighted_csr: 8, 8, 7 and 3 warps

# the column lengths of the edge case: every segment and Gram-run edge, long columns next to empty ones
EDGE_LENGTHS = [3 * 65536 + 1, 0, 0, 1, 2, 2047, 0, 2048, 2049, 0, 4097, 65535, 0, 65536, 65537, 0, 0, 131073]


# ---------------------------------------------------------------------------------------------------------------------
# host rules
# ---------------------------------------------------------------------------------------------------------------------
def seg_cap(d, nnz):
    """The bound of the plan's segments: bkm_csc_plan.cuh:15."""
    return d + nnz // SEG + 1


def row_group(n, nnz):
    """Lanes per row of the GLM row pass: bkm_glm_sparse.cu:169-172."""
    mean = nnz / n if n > 0 else 0.0
    return 4 if mean <= 6.0 else 8 if mean <= 12.0 else 16 if mean <= 24.0 else 32


def gram_warps(d):
    """Warps of a Gram CTA (one d-wide float64 row each in 96 KB): bkm_glm_sparse.cu:466-469."""
    return min(KWARPS, (96 * 1024) // (d * 8))


def label_sums_warps(k):
    """Warps of a label-sum CTA (one k-wide float64 accumulator each in 200 KB): bkm_kmeans_sparse.cu:390-393."""
    return min(KWARPS, (200 * 1024) // (k * 8))


def col_tile(l):
    """C of the 32 C column tiles of the row-gather passes: bkm_svd_sparse.cu:196-200 (and 211-216),
    bkm_kmeans_sparse.cu:305-309 and 520-524."""
    return 1 if l <= 32 else 2 if l <= 64 else 4


def col_tiles(l):
    """blockIdx.y tiles of bkm_csr_panel_chunk: bkm_svd_sparse.cu:187."""
    cw = 32 * col_tile(l)
    return (l + cw - 1) // cw


def colsum_windows(l):
    """Launches of bkm_csr_kernel_colsum_chunk: bkm_kmeans_sparse.cu:724-729."""
    return (l + COLSUM_WINDOW - 1) // COLSUM_WINDOW


# ---------------------------------------------------------------------------------------------------------------------
# builders
# ---------------------------------------------------------------------------------------------------------------------
def _values(rng, size, values):
    """'int': small nonzero integers (every sum of them is exact); 'rand': standard normal."""
    if values == "int":
        return (rng.randint(1, 5, size) * rng.choice([-1.0, 1.0], size)).astype(np.float64)
    return rng.standard_normal(size)


def _distinct(rng, n, L):
    """L distinct values of [0, n) in random order."""
    if 4 * L > n:
        return rng.permutation(n)[:L]
    u = np.unique(rng.randint(0, n, 2 * L + 8))
    while len(u) < L:
        u = np.unique(np.concatenate([u, rng.randint(0, n, L)]))
    return rng.choice(u, L, replace=False)


def _csr(r, c, n, d, dtype, seed, values):
    rng = np.random.RandomState(seed + 7919)
    m = sp.csr_matrix((_values(rng, len(r), values).astype(dtype), (r, c)), shape=(n, d))
    m.sum_duplicates()
    m.sort_indices()
    assert m.nnz == len(r)            # no coordinate was drawn twice
    return m


def columns(lengths, n, dtype=np.float64, seed=0, values="int"):
    """n x len(lengths): column j holds exactly lengths[j] entries in distinct random rows."""
    rng = np.random.RandomState(seed)
    r = [_distinct(rng, n, L) for L in lengths]
    c = [np.full(L, j, np.int64) for j, L in enumerate(lengths)]
    return _csr(np.concatenate(r), np.concatenate(c), n, len(lengths), dtype, seed, values)


def packed_multiseg(d, n=2100, dtype=np.float64, seed=0, values="int", length=SEG + 1):
    """Every column of SEG + 1 entries: two segments each, the densest packing of the slot formula (the slots of
    consecutive columns touch)."""
    return columns([length] * d, n, dtype, seed, values)


def rows_at(lengths, d, dtype=np.float64, seed=0, values="int"):
    """len(lengths) x d: row i holds exactly lengths[i] entries in distinct random columns."""
    rng = np.random.RandomState(seed)
    c = [np.sort(_distinct(rng, d, L)) for L in lengths]
    r = [np.full(L, i, np.int64) for i, L in enumerate(lengths)]
    return _csr(np.concatenate(r), np.concatenate(c), len(lengths), d, dtype, seed, values)


def skewed(n, mean, heavy_row_len, d, dtype=np.float64, seed=0, values="int"):
    """One row of heavy_row_len entries (row n // 2) among short rows of 0 .. 2 (mean - 1) entries, about ``mean``
    entries per row in all: the mean picks a small lane group while one row is 10^5 entries long."""
    rng = np.random.RandomState(seed)
    short = max(0.0, (mean * n - heavy_row_len) / (n - 1))
    lens = rng.randint(0, int(2 * short) + 1, n)
    lens[n // 2] = heavy_row_len
    return rows_at(lens, d, dtype, seed, values)


def mean_at(t, side, n=1000, d=100, dtype=np.float64, seed=0, values="int"):
    """n rows of t entries but one of t + side: a mean of t + side / n entries per row, on one side of a G threshold."""
    lens = np.full(n, t, np.int64)
    lens[n // 3] = t + side
    return rows_at(lens, d, dtype, seed, values)


# ---------------------------------------------------------------------------------------------------------------------
# the plan
# ---------------------------------------------------------------------------------------------------------------------
def plan(m, d):
    """The transpose of CSR ``m`` and its segment plan, restated from expand_kernel / the stable radix sort /
    gather_kernel / count_kernel / fill_kernel (bkm_glm_sparse.cu:193-263):

    colptr, rows, vals   the CSC, rows ascending within each column
    seg_off, gseg_off    exclusive scans of the segments per column and of the Gram slots per column
    seg_col              the column of each segment
    status               [non-canonical flag, segments T, Gram slots, longest column]
    seg_e0, seg_e1       each segment's entry range
    seg_slot             each segment's slot 2 (s0 - j) + (t - s0) (-1 for a column of one segment)
    run_seg, run_slot    the first segment of each Gram run (s % GS == 0) and its slot gseg_off[j] + s / GS (-1 for a
                         column of one run)"""
    m = sp.csr_matrix(m)
    col = m.indices.astype(np.int64)
    erow = np.repeat(np.arange(m.shape[0], dtype=np.int64), np.diff(m.indptr))
    perm = np.argsort(col, kind="stable")            # the radix sort is stable: rows stay ascending
    lens = np.bincount(col, minlength=d).astype(np.int64)
    colptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    nseg = np.where(lens > SEG, (lens + SEG - 1) // SEG, 1)
    nslot = np.where(nseg > GS, (nseg + GS - 1) // GS, 0)
    seg_off = np.concatenate([[0], np.cumsum(nseg)]).astype(np.int64)
    gseg_off = np.concatenate([[0], np.cumsum(nslot)]).astype(np.int64)
    T = int(seg_off[-1])
    seg_col = np.repeat(np.arange(d, dtype=np.int64), nseg)
    t = np.arange(T, dtype=np.int64)
    s0 = seg_off[seg_col]
    s = t - s0
    seg_e0 = colptr[seg_col] + s * SEG
    seg_e1 = np.minimum(colptr[seg_col + 1], seg_e0 + SEG)
    seg_slot = np.where(nseg[seg_col] > 1, 2 * (s0 - seg_col) + s, -1)
    run = np.nonzero(s % GS == 0)[0]
    run_slot = np.where(nseg[seg_col[run]] > GS, gseg_off[seg_col[run]] + s[run] // GS, -1)
    status = np.array([0, T, int(gseg_off[-1]), int(lens.max(initial=0))], np.int64)
    return types.SimpleNamespace(
        d=d, nnz=int(m.nnz), colptr=colptr, rows=erow[perm].astype(np.int32), vals=m.data[perm], lens=lens,
        nseg=nseg, nslot=nslot, seg_off=seg_off, gseg_off=gseg_off, seg_col=seg_col.astype(np.int32), status=status,
        seg_e0=seg_e0, seg_e1=seg_e1, seg_slot=seg_slot, run_seg=run, run_slot=run_slot,
        words=np.concatenate([status, seg_off, gseg_off]))


def slot_rows(P):
    """Rows of the slot area of a seg_fold pass: bkm_csc_plan.cuh:61."""
    return 2 * (P.nnz // SEG + 1)


# ---------------------------------------------------------------------------------------------------------------------
# the plain-add column passes
# ---------------------------------------------------------------------------------------------------------------------
def label_sums(P, labels, k, w=None, binarize=None, prev=None):
    """sumsT (d, k) of bkm_csc_label_sums_chunk (w and binarize None) or bkm_csc_class_counts_chunk, in the kernel's
    order (csc_label_sums_kernel, bkm_kmeans_sparse.cu:339-387, and seg_fold, bkm_csc_plan.cuh:47-58):

    * per segment, acc[label] = 0.0, then acc[label] += f(v) w[row] entry by entry in row order; a label outside
      [0, k) adds nothing;
    * per column, 0.0 plus its segments' accumulators in segment order (one segment: its accumulator itself);
    * ``prev`` None writes that (a first call), else it is added to ``prev``.

    np.add.at applies its adds one by one in index order, which is that order (np.sum would add pairwise)."""
    labels = np.asarray(labels, np.int64)
    d = P.d
    seg = np.repeat(np.arange(len(P.seg_col), dtype=np.int64), P.seg_e1 - P.seg_e0)
    lab = labels[P.rows]
    v = P.vals.astype(np.float64)
    if binarize is not None:
        v = (v > binarize).astype(np.float64)
    if w is not None:
        v = v * np.asarray(w, np.float64)[P.rows]
    keep = (lab >= 0) & (lab < k)
    key = seg[keep] * k + lab[keep]
    uniq, inv = np.unique(key, return_inverse=True)
    acc = np.zeros(len(uniq))
    np.add.at(acc, inv, v[keep])                       # within a segment, in row order
    out = np.zeros(d * k)
    np.add.at(out, P.seg_col[uniq // k].astype(np.int64) * k + uniq % k, acc)   # per column, in segment order
    out = out.reshape(d, k)
    return out if prev is None else prev + out


def onehot(labels, k, w=None):
    """(n, k) sparse one-hot of labels in [0, k) (others dropped), weighted by w."""
    labels = np.asarray(labels, np.int64)
    keep = np.nonzero((labels >= 0) & (labels < k))[0]
    vals = np.ones(len(keep)) if w is None else np.asarray(w, np.float64)[keep]
    return sp.csr_matrix((vals, (keep, labels[keep])), shape=(len(labels), k))


# ---------------------------------------------------------------------------------------------------------------------
# the cases
# ---------------------------------------------------------------------------------------------------------------------
def column_cases(dtype=np.float64, values="int"):
    """The blocks of the column passes, by name: each a pair of blocks of the same width with different plans (a first
    call and an accumulating call)."""
    E = EDGE_LENGTHS
    trail = [0, 1, 131073, 2049, 0, 65537, 2048, 4097, 65536, 2047, 65535, 3 * 65536 + 1, 2, 0, 0, 0, 0, 0]
    kw = dict(dtype=dtype, values=values)
    return {
        "edges": lambda: (columns(E, 200000, seed=1, **kw), columns(trail, 200000, seed=2, **kw)),
        "packed": lambda: (packed_multiseg(40, seed=3, **kw), packed_multiseg(40, n=4200, seed=4, length=2 * SEG + 1,
                                                                              **kw)),
        "gram1536": lambda: (gram_block(1536, 5, **kw), gram_block(1536, 6, **kw)),
        "gram1537": lambda: (gram_block(1537, 7, **kw), gram_block(1537, 8, **kw)),
        "gram4096": lambda: (gram_block(4096, 9, **kw), gram_block(4096, 10, **kw)),
    }


def gram_block(d, seed, dtype=np.float64, values="int"):
    """d columns of 0 .. 40 entries with columns of 1, 2, 3 and 4 Gram runs at j = 0, d // 2, d // 3 and d - 1."""
    rng = np.random.RandomState(seed)
    lens = rng.randint(0, 41, d)
    lens[:3] = 0
    lens[0], lens[d // 3], lens[d // 2], lens[d - 1] = 3 * 65536 + 1, 65536, 65537, 131073
    lens[d - 2] = 2049
    return columns(list(lens), 200000, dtype, seed, values)


def row_cases(dtype=np.float64, values="int"):
    """The blocks of the row passes, by name, as pairs of the same width."""
    kw = dict(dtype=dtype, values=values)
    batch = list(range(66)) * 2 + [1024, 1025, 2048, 31, 32, 33, 64, 65]
    cases = {
        "rows": lambda: (rows_at(batch, 2100, seed=11, **kw), rows_at(batch[::-1], 2100, seed=12, **kw)),
        "skewed": lambda: (skewed(50000, 5.0, 100000, 131072, seed=13, **kw),
                           skewed(20000, 3.0, 50000, 131072, seed=14, **kw)),
        "edges": lambda: column_cases(dtype, values)["edges"](),
    }
    for t in (6, 12, 24):
        for side in (0, 1):
            cases["mean%d%+d" % (t, side)] = (lambda t=t, side=side: (mean_at(t, side, seed=t + side, **kw),
                                                                       mean_at(t, -side, seed=t - side + 50, **kw)))
    return cases
