"""The sparse intake shared by the estimators that take sparse X (the linear models, TruncatedSVD, KMeans): a
ChunkedArray of torch sparse CSR blocks, one torch CSR tensor or any scipy.sparse matrix becomes ``_SparseData``, the
blocks on the device with each block's transpose built once on first use."""
import numpy as np
import scipy.sparse
import torch

from .chunked import ChunkedArray, _is_torch, is_sparse_csr_block


class _SparseData(object):
    """Sparse CSR row blocks on the device: ``blocks`` = [(crow int64, col int64, val float32 / float64, n)], with what
    ``_y_chunks`` and the passes read of ``DeviceData``.  ``transposes()`` builds each block's CSC once."""

    def __init__(self, blocks, d, backend, comm=None):
        from .engine import Comm

        self.blocks, self.d, self.backend = blocks, int(d), backend
        self.comm = comm or Comm()
        self.chunk_rows = [int(b[3]) for b in blocks]
        self.n_local = int(sum(self.chunk_rows))
        self.chunk_offsets = np.cumsum([0] + self.chunk_rows)
        self._csc = None
        self.n_slots = None

    def global_layout(self):
        """(global row of this rank's first row, rows over every rank): one gather across ranks."""
        sizes = [int(v) for v in self.comm.allgather_obj(self.n_local)]
        return int(sum(sizes[: self.comm.rank])), int(sum(sizes))

    # -- what KMeans reads besides the blocks ------------------------------------------------
    @property
    def dtype(self):
        """The values' dtype (float32 or float64)."""
        return self.blocks[0][2].dtype if self.blocks else torch.float64

    @property
    def np_dtype(self):
        return np.dtype("float32") if self.dtype == torch.float32 else np.dtype("float64")

    def _layout(self):
        if getattr(self, "_row_offset", None) is None:
            self._row_offset, self._n_global = self.global_layout()
        return self._row_offset, self._n_global

    @property
    def row_offset(self):
        """Global row of this rank's first row (one gather across ranks on first use)."""
        return self._layout()[0]

    @property
    def n_global(self):
        return self._layout()[1]

    def check_finite(self):
        """ValueError on every rank when a value of any rank is NaN or infinite: the values scanned as one column."""
        from .cluster.k_means import _NONFINITE_MSG

        be = self.backend
        vals = [b[2].view(-1, 1) for b in self.blocks if b[2].numel() > 0]
        flag = be.check_finite(vals).to(torch.float64) if vals else torch.zeros(1, dtype=torch.float64,
                                                                                 device=be.device)
        self.comm.allreduce_sum_(flag)
        if float(flag.item()) != 0.0:
            raise ValueError(_NONFINITE_MSG)

    def _local_csr(self, local_idx):
        """The rows of LOCAL indices ``local_idx`` (in that order) as a host scipy CSR: one gather per block."""
        local_idx = np.asarray(local_idx, dtype=np.int64)
        dt = self.np_dtype
        parts = [None] * len(local_idx)
        which = np.searchsorted(self.chunk_offsets, local_idx, side="right") - 1
        for w in np.unique(which):
            pos = np.nonzero(which == w)[0]
            crow, col, val, _n = self.blocks[w]
            rel = torch.as_tensor(local_idx[pos] - self.chunk_offsets[w], dtype=torch.int64, device=crow.device)
            start, stop = crow[rel], crow[rel + 1]
            lens = stop - start
            # the entries of each chosen row, in the chosen order
            base = torch.repeat_interleave(start - torch.cumsum(lens, 0) + lens, lens)
            e = base + torch.arange(int(lens.sum().item()), dtype=torch.int64, device=crow.device)
            ln = lens.cpu().numpy()
            c = col[e].cpu().numpy()
            v = val[e].cpu().numpy().astype(dt, copy=False)
            off = np.concatenate([[0], np.cumsum(ln)])
            for t, q in enumerate(pos):
                parts[q] = (c[off[t]:off[t + 1]], v[off[t]:off[t + 1]])
        return self._assemble(parts)

    def _assemble(self, parts):
        lens = np.array([len(p[0]) for p in parts], dtype=np.int64)
        indptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
        cols = np.concatenate([p[0] for p in parts]) if parts else np.zeros(0, np.int64)
        vals = np.concatenate([p[1] for p in parts]) if parts else np.zeros(0, self.np_dtype)
        return scipy.sparse.csr_matrix((vals.astype(self.np_dtype, copy=False), cols, indptr),
                                       shape=(len(parts), self.d))

    def global_rows(self, global_idx):
        """Rows by GLOBAL index (any rank's rows) as a host scipy CSR, on every rank, in the given order."""
        global_idx = np.asarray(global_idx, dtype=np.int64)
        lo = self.row_offset
        mine = np.nonzero((global_idx >= lo) & (global_idx < lo + self.n_local))[0]
        rows = self._local_csr(global_idx[mine] - lo)
        if self.comm.world == 1:
            return rows
        parts = [None] * len(global_idx)
        for pos, r in self.comm.allgather_obj((mine, rows)):
            for t, q in enumerate(pos):
                parts[q] = (r.indices[r.indptr[t]:r.indptr[t + 1]], r.data[r.indptr[t]:r.indptr[t + 1]])
        return self._assemble(parts)

    def to_host(self):
        """All LOCAL rows as one host scipy CSR (the in-memory k-means++ init)."""
        blocks = [scipy.sparse.csr_matrix((v.cpu().numpy(), c.cpu().numpy(), r.cpu().numpy()), shape=(int(n), self.d))
                  for r, c, v, n in self.blocks]
        return scipy.sparse.vstack(blocks, format="csr").astype(self.np_dtype, copy=False)

    def transposes(self):
        """The blocks' transposes, built on first use.  Their checks are read here, once: a block whose column indices
        are not strictly increasing within each row (or not in [0, d)) raises ValueError on every rank."""
        if self._csc is None:
            be = self.backend
            csc = [be.csr_transpose_chunk(b, self.d) for b in self.blocks]
            status = torch.stack([c[3][:4] for c in csc]).cpu().numpy()
            bad = [i for i in range(len(csc)) if status[i, 0] != 0]
            flag = torch.tensor([float(len(bad))], dtype=torch.float64, device=be.device)
            self.comm.allreduce_sum_(flag)
            if float(flag.item()) != 0.0:
                where = ("block %d" % bad[0]) if bad else "a block of another rank"
                raise ValueError("Sparse input must be canonical CSR: the column indices of %s are not strictly "
                                 "increasing within each row, or not in [0, %d)" % (where, self.d))
            self.n_slots = [int(v) for v in status[:, 2]]
            self._csc = csc
        return self._csc


# The label-sum pass over a block's transpose (bkm_csc_label_sums_chunk, bkm_csc_class_counts_chunk) keeps one k-wide
# float64 accumulator per warp in 200 KB of shared memory, so it takes at most this many clusters or classes.
MAX_LABEL_SUM_CLASSES = 25600


def check_label_sum_classes(k, what):
    """ValueError at intake when sparse X would need the label-sum pass for more than MAX_LABEL_SUM_CLASSES values of
    ``what`` ("clusters" or "classes")."""
    if int(k) > MAX_LABEL_SUM_CLASSES:
        raise ValueError("Sparse input supports at most %d %s, got %d: the label-sum pass keeps a float64 sum for "
                         "each of them in shared memory" % (MAX_LABEL_SUM_CLASSES, what, int(k)))


def _sparse_values(v):
    """float32 / float64 values as they are; integer and bool values widened once to float64."""
    if v.dtype in (torch.float32, torch.float64):
        return v
    if v.dtype == torch.bool or not (v.dtype.is_floating_point or v.dtype.is_complex):
        return v.to(torch.float64)
    raise TypeError("Sparse input values of dtype %s are not supported: use float32, float64, an integer type or "
                    "bool" % (v.dtype,))


def _csr_block(m, device):
    """One canonical host scipy CSR as a (crow, col, val, n) block on ``device``."""
    m = scipy.sparse.csr_matrix(m, copy=True)
    m.sum_duplicates()
    m.sort_indices()
    return (torch.from_numpy(m.indptr.astype(np.int64)).to(device), torch.from_numpy(m.indices.astype(np.int64)).to(device),
            _sparse_values(torch.from_numpy(np.ascontiguousarray(m.data))).to(device), int(m.shape[0]))


def _sparse_data(X):
    """Sparse X -> ``_SparseData``, or None for every other input.  Accepted: a ChunkedArray whose blocks are all torch
    sparse CSR tensors (device or host), one torch sparse CSR tensor, or a scipy.sparse matrix of any format (made
    canonical CSR on the host and uploaded as one block)."""
    if isinstance(X, ChunkedArray):
        sp = [is_sparse_csr_block(b) for b in X.blocks]
        if not any(sp):
            return None
        if not all(sp):
            raise TypeError("A ChunkedArray that mixes dense and sparse CSR blocks is not supported")
        blocks = X.blocks
    elif _is_torch(X) and X.layout == torch.sparse_csr:
        blocks = [X]
    elif scipy.sparse.issparse(X):
        m = scipy.sparse.csr_matrix(X, copy=True)
        m.sum_duplicates()
        m.sort_indices()
        v = torch.from_numpy(np.ascontiguousarray(m.data))
        blocks = [(torch.from_numpy(m.indptr.astype(np.int64)), torch.from_numpy(m.indices.astype(np.int64)), v,
                   m.shape)]
    else:
        return None
    from .cluster import k_means as _km

    be = _km._get_backend()
    out = []
    for b in blocks:
        if isinstance(b, tuple):
            crow, col, val, shape = b
        else:
            crow, col, val, shape = b.crow_indices(), b.col_indices(), b.values(), tuple(b.shape)
        if len(shape) != 2:
            raise ValueError("Expected a 2-D sparse matrix, got shape %s" % (tuple(shape),))
        val = _sparse_values(val)
        crow = crow.to(device=be.device, dtype=torch.int64).contiguous()
        col = col.to(device=be.device, dtype=torch.int64).contiguous()
        out.append((crow, col, val.to(device=be.device).contiguous(), int(shape[0])))
    return _SparseData(out, int(shape[1]), be)
