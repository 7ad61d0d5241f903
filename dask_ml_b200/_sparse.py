"""The sparse intake shared by the estimators that take sparse X (the linear models, TruncatedSVD): a ChunkedArray of
torch sparse CSR blocks, one torch CSR tensor or any scipy.sparse matrix becomes ``_SparseData``, the blocks on the device
with each block's transpose built once on first use."""
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


def _sparse_values(v):
    """float32 / float64 values as they are; integer and bool values widened once to float64."""
    if v.dtype in (torch.float32, torch.float64):
        return v
    if v.dtype == torch.bool or not (v.dtype.is_floating_point or v.dtype.is_complex):
        return v.to(torch.float64)
    raise TypeError("Sparse input values of dtype %s are not supported: use float32, float64, an integer type or "
                    "bool" % (v.dtype,))


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
