"""Minimal row-chunked array: the stand-in for ``dask.array`` on the KMeans path.

dask is not a dependency of the engine (and is not installable in the build image).  The
reference only ever uses arrays chunked along axis 0 with a single block on axis 1
(dask_ml/utils.py:128-135); ``ChunkedArray`` models exactly that: a list of row blocks.
Blocks may be numpy arrays or torch tensors (CPU or CUDA).  Real dask arrays are accepted by
``as_chunked`` when dask is importable.
"""
import numpy as np

try:  # torch is required for the engine, optional for the container type itself
    import torch
except Exception:  # pragma: no cover
    torch = None


def _is_torch(x):
    return torch is not None and isinstance(x, torch.Tensor)


_TORCH_TO_NP = {}
if torch is not None:
    _TORCH_TO_NP = {
        torch.float32: np.dtype("float32"), torch.float64: np.dtype("float64"),
        torch.float16: np.dtype("float16"), torch.int32: np.dtype("int32"),
        torch.int64: np.dtype("int64"), torch.bool: np.dtype("bool"), torch.uint8: np.dtype("uint8"),
        torch.int8: np.dtype("int8"), torch.int16: np.dtype("int16"), torch.uint16: np.dtype("uint16"),
        torch.uint32: np.dtype("uint32"),
        # numpy has no bfloat16: a bf16 block presents itself as float32 to numpy consumers (it is widened on
        # the way out) and stays bf16 on the device (the large-shape tensor path multiplies the rows as stored)
        torch.bfloat16: np.dtype("float32"),
    }


def block_dtype(b):
    return _TORCH_TO_NP[b.dtype] if _is_torch(b) else np.dtype(b.dtype)


def is_sparse_csr_block(b):
    return _is_torch(b) and b.layout == torch.sparse_csr


def block_to_numpy(b):
    """A block as numpy; a torch sparse CSR block (OneHotEncoder's sparse output) as a scipy.sparse.csr_matrix."""
    if is_sparse_csr_block(b):
        import scipy.sparse

        b = b.detach().cpu()
        vals = b.values()
        vals = (vals.float() if vals.dtype == torch.bfloat16 else vals).numpy()
        return scipy.sparse.csr_matrix((vals, b.col_indices().numpy(), b.crow_indices().numpy()), shape=tuple(b.shape))
    if _is_torch(b):
        b = b.detach()
        if b.dtype == torch.bfloat16:
            b = b.float()
        return b.cpu().numpy()
    return np.asarray(b)


def is_bf16_block(b):
    return _is_torch(b) and b.dtype == torch.bfloat16


class ChunkedArray(object):
    """A 1-D or 2-D array stored as a list of row blocks (chunks on axis 0 only)."""

    def __init__(self, blocks):
        blocks = list(blocks)
        if not blocks:
            raise ValueError("ChunkedArray needs at least one block")
        nd = blocks[0].ndim
        if nd not in (1, 2):
            raise ValueError("blocks must be 1-D or 2-D")
        for b in blocks:
            if b.ndim != nd:
                raise ValueError("all blocks must have the same number of dimensions")
            if nd == 2 and b.shape[1] != blocks[0].shape[1]:
                raise ValueError("all blocks must have the same number of columns")
            if block_dtype(b) != block_dtype(blocks[0]):
                raise ValueError("all blocks must share one dtype")
        self.blocks = blocks

    # -- dask.array-like metadata ------------------------------------------------------
    @property
    def ndim(self):
        return self.blocks[0].ndim

    @property
    def dtype(self):
        return block_dtype(self.blocks[0])

    @property
    def chunks(self):
        rows = tuple(int(b.shape[0]) for b in self.blocks)
        if self.ndim == 1:
            return (rows,)
        return (rows, (int(self.blocks[0].shape[1]),))

    @property
    def numblocks(self):
        return (len(self.blocks),) if self.ndim == 1 else (len(self.blocks), 1)

    @property
    def shape(self):
        n = sum(int(b.shape[0]) for b in self.blocks)
        return (n,) if self.ndim == 1 else (n, int(self.blocks[0].shape[1]))

    def __len__(self):
        return self.shape[0]

    # -- materialisation ---------------------------------------------------------------
    def compute(self):
        parts = [block_to_numpy(b) for b in self.blocks]
        if len(parts) == 1:
            return parts[0]
        if any(is_sparse_csr_block(b) for b in self.blocks):
            import scipy.sparse

            return scipy.sparse.vstack(parts, format="csr")
        return np.concatenate(parts, axis=0)

    def __array__(self, dtype=None, copy=None):
        a = self.compute()
        return a.astype(dtype) if dtype is not None else a

    def astype(self, dtype):
        dtype = np.dtype(dtype)
        out = []
        for b in self.blocks:
            if _is_torch(b):
                tdt = {v: k for k, v in _TORCH_TO_NP.items() if k != torch.bfloat16}[dtype]
                out.append(b.to(tdt))
            else:
                out.append(np.asarray(b).astype(dtype))
        return ChunkedArray(out)

    def rows(self, idx):
        """Gather rows by global index (sorted or not) into a numpy array."""
        idx = np.asarray(idx, dtype=np.int64)
        bounds = np.cumsum([0] + list(self.chunks[0]))
        which = np.searchsorted(bounds, idx, side="right") - 1
        out = np.empty((len(idx),) + tuple(self.shape[1:]), dtype=self.dtype)
        for p, (i, w) in enumerate(zip(idx, which)):
            b = self.blocks[w]
            r = b[int(i - bounds[w])]
            out[p] = block_to_numpy(r)
        return out

    def __getitem__(self, key):
        a = self.compute()
        return a[key]

    def __repr__(self):
        return "ChunkedArray<shape=%s, dtype=%s, chunks=%s>" % (self.shape, self.dtype, self.chunks)

    @classmethod
    def from_array(cls, x, chunks):
        """Split a 1-D/2-D array into row blocks of ``chunks`` rows (int) or explicit sizes."""
        n = x.shape[0]
        if isinstance(chunks, (tuple, list)) and len(chunks) and isinstance(chunks[0], (tuple, list)):
            sizes = list(chunks[0])
        else:
            c = int(chunks[0] if isinstance(chunks, (tuple, list)) else chunks)
            c = max(1, c)
            sizes = [c] * (n // c) + ([n % c] if n % c else [])
            if not sizes:
                sizes = [0]
        out, s = [], 0
        for m in sizes:
            out.append(x[s:s + m])
            s += m
        return cls(out)


def is_dask_array(x):
    t = type(x)
    return t.__module__.startswith("dask.array") and t.__name__ == "Array"


def is_dask_dataframe(x):
    t = type(x)
    return t.__module__.startswith("dask.dataframe") or t.__module__.startswith("dask_expr")


def as_chunked(x):
    """dask array -> ChunkedArray (blocks computed one at a time); ChunkedArray passes through."""
    if isinstance(x, ChunkedArray):
        return x
    if is_dask_array(x):
        if any(np.isnan(c) for c in x.chunks[0]):
            raise TypeError("Cannot operate on Dask array with unknown chunk sizes.")
        if x.ndim > 1 and len(x.chunks[1]) > 1:
            raise TypeError(
                "Chunking is only allowed on the first axis. "
                "Use 'array.rechunk({1: array.shape[1]})' to "
                "rechunk to a single block along the second axis."
            )
        blocks = [np.asarray(b.compute()) for b in x.to_delayed().flatten().tolist()]
        return ChunkedArray(blocks)
    raise TypeError("not a chunked array: %r" % type(x))


def _y_flat(y, who="GaussianNB.fit"):
    """y (numpy, torch on any device, ChunkedArray or dask array, any chunking) -> one flat numpy array or tensor."""
    if y is None:
        raise ValueError("%s needs the labels y; got None" % who)
    if isinstance(y, ChunkedArray):
        blocks = y.blocks
    elif is_dask_array(y):
        blocks = as_chunked(y).blocks
    else:
        blocks = [y]
    if all(_is_torch(b) for b in blocks):
        flat = [b.detach().reshape(-1) for b in blocks]
        return flat[0] if len(flat) == 1 else torch.cat([f.to(flat[0].device) for f in flat])
    flat = [np.asarray(block_to_numpy(b) if _is_torch(b) else b).reshape(-1) for b in blocks]
    return flat[0] if len(flat) == 1 else np.concatenate(flat)
