"""ShuffleSplit, KFold and train_test_split with the dask_ml.model_selection API, executed block-wise on the device.

Mirrors dask_ml/model_selection/_split.py:24-318 and :321-465 (reference @ 0310a90).  ShuffleSplit: every row block
is permuted on its own and cut into a test part (positions [0, n_test) of the block's permutation) and a train part (the
next n_train positions), so no row leaves its block, its device or its rank.  Per block of c rows

    seeds     check_random_state(random_state).randint(0, 2**32 - 1, size=n_blocks, dtype="u8")   (the reference's draw)
    sizes     scikit-learn's _validate_shuffle_split(c, test_size, train_size)
    indices   offset + pi_seed(p), p = 0 .. n_test + n_train - 1      bkm_split_indices_chunk, one launch
    rows      out[i] = block[idx[i] - offset] for every array          bkm_gather_rows_chunk, one launch per array and part

The one deviation (DESIGN.md A26): the block's permutation pi_seed is not numpy's Mersenne-Twister Fisher-Yates, which is
serial, but the keyed bijection defined in include/bkm_b200.h ("the split permutation"), which any thread evaluates for
one position without memory.  ``permutation_indices`` restates it in numpy; host blocks are split with it and are never
uploaded, and the device kernel is tested against it bit for bit, so a split depends on ``random_state`` and the row
chunks only: not on the device, on torch, or on which array of the call is being split.
"""
import itertools
import logging
import numbers

import numpy as np
from sklearn.model_selection._split import BaseCrossValidator, _validate_shuffle_split
from sklearn.utils import check_random_state

from ..chunked import ChunkedArray, _is_torch, as_chunked, is_dask_array, is_dask_dataframe

logger = logging.getLogger(__name__)

# ---- the split permutation: include/bkm_b200.h restated ------------------------------------------------------------
SPLIT_ROUNDS = 12
_KEY_STEP = np.uint64(0x9E3779B97F4A7C15)
_KEY_MUL1 = np.uint64(0xBF58476D1CE4E5B9)
_KEY_MUL2 = np.uint64(0x94D049BB133111EB)
_ROUND_MUL = np.uint64(0xD2511F53)
_ROUND_MIX = np.uint64(0x7FEB352D)
_LOW32 = np.uint64(0xFFFFFFFF)
MAX_BLOCK_ROWS = 1 << 31


def _half_width(c):
    """w: the Feistel network permutes [0, 4^w), the smallest such domain that holds [0, c)."""
    bits = max(int(c) - 1, 0).bit_length()
    return max(1, (bits + 1) // 2)


def _round_keys(seed, rounds):
    """(k0, k1) of every round, each the low / high word of splitmix64's finaliser of seed + (r + 1) * step."""
    seed = np.asarray(seed, dtype=np.uint64)
    keys = []
    with np.errstate(over="ignore"):
        for r in range(rounds):
            z = seed + np.uint64(r + 1) * _KEY_STEP
            z = (z ^ (z >> np.uint64(30))) * _KEY_MUL1
            z = (z ^ (z >> np.uint64(27))) * _KEY_MUL2
            z = z ^ (z >> np.uint64(31))
            keys.append((z & _LOW32, z >> np.uint64(32)))
    return keys


def permutation_indices(seed, c, positions, rounds=SPLIT_ROUNDS):
    """pi_seed(p) for every p of ``positions`` (values in [0, c)): int64, the shape of ``positions`` broadcast with
    ``seed`` (a seed per position is allowed: the uniformity tests evaluate one position under many seeds)."""
    c = int(c)
    if not 1 <= c <= MAX_BLOCK_ROWS:
        raise ValueError("a block must have between 1 and 2**31 rows; got %d" % c)
    seed = np.atleast_1d(np.asarray(seed, dtype=np.uint64))
    pos = np.atleast_1d(np.asarray(positions))
    if pos.size and (pos.min() < 0 or pos.max() >= c):
        raise ValueError("positions must lie in [0, %d)" % c)
    seed, pos = np.broadcast_arrays(seed, pos.astype(np.uint64))
    v = pos.copy()
    w = np.uint64(_half_width(c))
    mask = np.uint64((1 << int(w)) - 1)
    up = np.uint64(32) - w
    todo = np.ones(v.shape, dtype=bool)
    with np.errstate(over="ignore"):
        while todo.any():                                   # cycle walking: re-apply where the value is >= c
            x = v[todo]
            keys = _round_keys(seed[todo], rounds)
            L, R = x >> w, x & mask
            for k0, k1 in keys:
                t = (R ^ k0) & _LOW32
                p = t * _ROUND_MUL
                f = ((p >> np.uint64(32)) ^ p ^ k1) & _LOW32
                f = ((f ^ (f >> np.uint64(16))) * _ROUND_MIX) & _LOW32
                f = f ^ (f >> np.uint64(15))
                L, R = R, L ^ (f >> up)
            x = (L << w) | R
            v[todo] = x
            todo[todo] = x >= np.uint64(c)
    return v.astype(np.int64)


# ---- validation ----------------------------------------------------------------------------------------------------
def _check_blockwise(blockwise):
    if blockwise not in {True, False}:
        raise ValueError("Expected a boolean for 'blockwise but got {} instead".format(blockwise))
    return blockwise


def _validate_shuffle_split_init(test_size, train_size):
    """The constructor checks of scikit-learn < 0.24's helper of this name, which the reference calls."""
    if test_size is None and train_size is None:
        raise ValueError("test_size and train_size can not both be None")
    for name, size in (("test_size", test_size), ("train_size", train_size)):
        if size is None:
            continue
        kind = np.asarray(size).dtype.kind
        if kind == "f":
            if size >= 1.0:
                raise ValueError("{}={} should be smaller than 1.0 or be an integer".format(name, size))
        elif kind != "i":
            raise ValueError("Invalid value for {}: {!r}".format(name, size))
    if (train_size is not None and test_size is not None and np.asarray(train_size).dtype.kind == "f"
            and np.asarray(test_size).dtype.kind == "f" and train_size + test_size > 1.0):
        raise ValueError("The sum of test_size and train_size = {}, should be smaller than 1.0. Reduce test_size "
                         "and/or train_size.".format(train_size + test_size))


def _maybe_normalize_split_sizes(train_size, test_size):
    if train_size is None and test_size is None:
        raise ValueError("test_size and train_size can not both be None")
    elif any(isinstance(x, numbers.Integral) for x in (train_size, test_size)):
        raise ValueError("Dask-ML does not support absolute sizes for 'train_size' and 'test_size'. Use floats between "
                         "0 and 1 to specify the fraction of each block that should go to the train and test set.")
    if train_size is not None:
        if train_size < 0 or train_size > 1:
            raise ValueError("'train_size' must be between 0 and 1. Got {}".format(train_size))
        if test_size is None:
            test_size = 1 - train_size
    if test_size is not None:
        if test_size < 0 or test_size > 1:
            raise ValueError("'test_size' be between 0 and 1. Got {}".format(test_size))
        if train_size is None:
            train_size = 1 - test_size
    if abs(1 - (train_size + test_size)) > 0.001:
        raise ValueError("The sum of 'train_size' and 'test_size' must be 1. train_size: {} test_size: {}"
                         .format(train_size, test_size))
    return train_size, test_size


# ---- intake --------------------------------------------------------------------------------------------------------
def _is_plain(a):
    """numpy / pandas / list input: nothing chunked, nothing on a device."""
    return not (isinstance(a, ChunkedArray) or _is_torch(a) or is_dask_array(a) or is_dask_dataframe(a))


def _as_blocks(a):
    """ChunkedArray, dask array, torch tensor or numpy array (one block each) -> ChunkedArray."""
    if is_dask_dataframe(a):
        raise TypeError("dask DataFrames are not supported; pass row-chunked arrays")
    if isinstance(a, ChunkedArray) or is_dask_array(a):
        return as_chunked(a)
    if _is_torch(a):
        return ChunkedArray([a.detach()])
    return ChunkedArray([np.asarray(a)])


def _check_matching_blocks(arrays):
    chunks = arrays[0].chunks[0]
    for a in arrays[1:]:
        if a.chunks[0] != chunks:
            raise ValueError("Mismatched chunks. {} != {}".format(chunks, a.chunks[0]))


def _cuda_device(block):
    return block.device if _is_torch(block) and block.is_cuda else None


_BACKENDS = {}


def _backend(device):
    from ..engine import CudaBackend

    be = _BACKENDS.get(device)
    if be is None:
        be = _BACKENDS[device] = CudaBackend(device)
    return be


def _block_seeds(random_state, n_blocks):
    """The reference's per-block seed draw.  With torch.distributed the seeds of the blocks of all ranks are drawn in
    rank order and a rank keeps its own, so equal integer seeds on every rank never give two blocks one seed."""
    from ..engine import Comm

    comm = Comm()
    counts = comm.allgather_obj(int(n_blocks))
    rng = check_random_state(random_state)
    seeds = rng.randint(0, 2 ** 32 - 1, size=int(sum(counts)), dtype="u8")
    lo = int(sum(counts[:comm.rank]))
    return seeds[lo:lo + n_blocks]


class ShuffleSplit(BaseCrossValidator):
    """Random permutation cross-validator over row blocks (API of dask_ml.model_selection.ShuffleSplit).

    Every block is shuffled internally and cut into a train and a test part; rows are not shuffled between blocks.
    ``split`` yields ``(train_idx, test_idx)``: int64 ChunkedArrays of global row indices with one block per block of
    X, each on the device (or host) that block of X is on.  As in the reference the block seeds are drawn from
    ``random_state`` anew at every split, so an integer ``random_state`` gives ``n_splits`` equal splits.

    Parameters
    ----------
    n_splits : int, default 10
    test_size, train_size : float in [0, 1] or None
        The fraction of each block that goes to the test / train part; None is the complement of the other.
    blockwise : bool, default True.  ``False`` is not implemented.
    random_state : int, RandomState instance or None
    """

    def __init__(self, n_splits=10, test_size=0.1, train_size=None, blockwise=True, random_state=None):
        _validate_shuffle_split_init(test_size, train_size)
        self.n_splits = n_splits
        self.test_size = test_size
        self.train_size = train_size
        self.random_state = random_state
        self.blockwise = _check_blockwise(blockwise)

    def split(self, X, y=None, groups=None):
        X = _as_blocks(X)
        for _ in range(self.n_splits):
            if self.blockwise:
                yield self._split_blockwise(X)
            else:
                yield self._split(X)

    def _split_blockwise(self, X):
        chunks = X.chunks[0]
        seeds = _block_seeds(self.random_state, len(chunks))
        train_pct, test_pct = _maybe_normalize_split_sizes(self.train_size, self.test_size)
        sizes = [_validate_shuffle_split(c, test_pct, train_pct) for c in chunks]
        offsets = np.hstack([0, np.cumsum(chunks)])
        train, test = [], []
        for b, c, seed, (n_train, n_test), off in zip(X.blocks, chunks, seeds, sizes, offsets):
            n_train, n_test, off = int(n_train), int(n_test), int(off)
            dev = _cuda_device(b)
            if dev is not None:
                idx = _backend(dev).split_indices_chunk(int(seed), c, 0, n_test + n_train, off)
            else:
                idx = permutation_indices(seed, c, np.arange(n_test + n_train)) + off
            test.append(idx[:n_test])
            train.append(idx[n_test:])
        return ChunkedArray(train), ChunkedArray(test)

    def _split(self, X):
        raise NotImplementedError("ShuffleSplit with `blockwise=False` has not been implemented yet.")

    def get_n_splits(self, X=None, y=None, groups=None):
        return self.n_splits


def _rank_layout(chunks):
    """(n, lo): the global number of rows, and the global position of this rank's first row (rank order, then block
    order).  One ``allgather_obj`` with torch.distributed, none without."""
    from ..engine import Comm

    comm = Comm()
    counts = comm.allgather_obj(int(sum(chunks)))
    return int(sum(counts)), int(sum(counts[:comm.rank]))


class KFold(BaseCrossValidator):
    """K-Folds cross-validator over row blocks (API of dask_ml.model_selection.KFold).

    The global rows, in rank order and then block order, are cut into ``n_splits`` consecutive windows (the first
    ``n % n_splits`` one row longer); fold f tests window f and trains on the rest.  ``split`` yields
    ``(train_idx, test_idx)``: int64 ChunkedArrays of row indices (rank-local, as ``ShuffleSplit``'s), made of index
    pieces in the reference's order: per block of X, the train piece before the window, the test piece, the train
    piece after it, each piece non-empty and on the device (or host) its block of X is on.  A rank none of whose
    blocks meets a part holds one 0-row block there.

    ``shuffle=True`` draws one seed per block once per ``split`` call (``ShuffleSplit``'s draw), so every fold sees
    the same permutation of each block and the test parts partition the rows; positions [a, b) of a block hold
    ``offset + pi_seed(p)`` for p in [a, b), the split permutation of DESIGN.md A26, one ``bkm_split_indices_chunk``
    launch per piece of a device block.  Rows never leave their block.  ``random_state`` is ignored without
    ``shuffle``, as in the reference.
    """

    def __init__(self, n_splits=5, shuffle=False, random_state=None):
        if not isinstance(n_splits, numbers.Integral) or isinstance(n_splits, bool):
            raise ValueError("The number of folds must be of Integral type. %r of type %s was passed."
                             % (n_splits, type(n_splits)))
        if n_splits < 2:
            raise ValueError("k-fold cross-validation requires at least one train/test split by setting n_splits=2 "
                             "or more, got n_splits={0}.".format(n_splits))
        if not isinstance(shuffle, bool):
            raise TypeError("shuffle must be True or False; got {0}".format(shuffle))
        self.n_splits = int(n_splits)
        self.shuffle = shuffle
        self.random_state = random_state

    def _windows(self, chunks):
        """Per fold, (train, test): lists of (block, start, stop) positions within this rank's blocks."""
        n, lo = _rank_layout(chunks)
        if self.n_splits > n:
            raise ValueError("Cannot have number of splits n_splits={0} greater than the number of samples: "
                             "n_samples={1}.".format(self.n_splits, n))
        sizes = np.full(self.n_splits, n // self.n_splits, dtype=np.int64)
        sizes[: n % self.n_splits] += 1
        stops = np.cumsum(sizes)
        starts = stops - sizes
        folds = []
        for t0, t1 in zip(starts, stops):
            train, test = [], []
            start = lo
            for i, c in enumerate(chunks):
                stop = start + c
                a, b = max(int(t0), start), min(int(t1), stop)
                if min(a, stop) > start:
                    train.append((i, 0, min(a, stop) - start))
                if a < b:
                    test.append((i, a - start, b - start))
                if max(b, start) < stop:
                    train.append((i, max(b, start) - start, c))
                start = stop
            folds.append((train, test))
        return folds

    def split(self, X, y=None, groups=None):
        X = _as_blocks(X)
        chunks = X.chunks[0]
        folds = self._windows(chunks)
        seeds = _block_seeds(self.random_state, len(chunks)) if self.shuffle else None
        offsets = np.hstack([0, np.cumsum(chunks)])
        for train, test in folds:
            yield tuple(ChunkedArray(self._indices(X, part, seeds, offsets)) for part in (train, test))

    def _indices(self, X, pieces, seeds, offsets):
        out = []
        for i, a, b in pieces:
            blk, c, off = X.blocks[i], int(X.chunks[0][i]), int(offsets[i])
            dev = _cuda_device(blk)
            if dev is not None:
                import torch

                if seeds is None:
                    out.append(torch.arange(off + a, off + b, dtype=torch.int64, device=dev))
                else:
                    out.append(_backend(dev).split_indices_chunk(int(seeds[i]), c, a, b - a, off))
            elif seeds is None:
                out.append(np.arange(off + a, off + b, dtype=np.int64))
            else:
                out.append(permutation_indices(seeds[i], c, np.arange(a, b)) + off)
        return out or [_empty_like_rows(X.blocks[0], np.int64)]

    def get_n_splits(self, X=None, y=None, groups=None):
        return self.n_splits


def _empty_like_rows(b, dtype=None):
    """A 0-row block on the device (or host) of ``b``: of ``b``'s trailing shape and dtype, or 1-D of ``dtype``."""
    if dtype is None:
        return b[:0]
    if _is_torch(b):
        import torch

        return torch.empty(0, dtype=torch.int64, device=b.device)
    return np.empty(0, dtype=dtype)


def _gather(b, ix, off, validate):
    """Rows ``ix - off`` of block ``b``, where ``b`` is: the row-gather kernel for a device block, numpy on the host."""
    n = int(b.shape[0])
    dev = _cuda_device(b)
    if dev is not None:
        import torch

        ix = ix if _is_torch(ix) else torch.as_tensor(np.ascontiguousarray(ix))
        ix = ix.to(device=dev, dtype=torch.int64)
        if validate and ix.numel():
            lo, hi = (int(v) for v in torch.aminmax(ix))
            if lo < off or hi >= off + n:
                raise IndexError("index block holds rows outside its block [%d, %d)" % (off, off + n))
        return _backend(dev).gather_rows_chunk(b, ix, off)
    ix = ix.cpu().numpy() if _is_torch(ix) else np.asarray(ix)
    if validate and ix.size and (ix.min() < off or ix.max() >= off + n):
        raise IndexError("index block holds rows outside its block [%d, %d)" % (off, off + n))
    if _is_torch(b):
        import torch

        return b[torch.as_tensor(ix - off)]
    return np.asarray(b)[ix - off]


def _blockwise_slice(arr, idx, validate=True):
    """Slice an array that is blockwise-aligned with idx: block i of the result is ``arr`` block i at the rows
    ``idx`` block i names (global indices, each within block i), on the device (or host) ``arr`` block i is on.

    Device blocks go through the row-gather kernel, whatever their dtype; host blocks through numpy.  ``validate``
    checks the index range (the kernel does not); ``train_test_split`` skips it for indices it has just generated."""
    offsets = np.hstack([0, np.cumsum(arr.chunks[0])[:-1]])
    return ChunkedArray([_gather(b, ix, int(off), validate) for b, ix, off in zip(arr.blocks, idx.blocks, offsets)])


def _take(arr, idx):
    """``arr[idx]`` for index blocks that need not match ``arr``'s blocks: KFold's pieces, ShuffleSplit's parts, or the
    one host array of indices a scikit-learn splitter returns.  Each index block is cut where its values cross a
    boundary of ``arr``'s blocks (a binary search on the block offsets) and every cut is gathered from its one source
    block as ``_blockwise_slice`` gathers, so the result has one block per cut, where its source block is.  A host
    index block is grouped by source block first (stably, so sorted indices keep their order); a device index block
    must lie inside one block of ``arr`` (IndexError otherwise), which KFold's and ShuffleSplit's do.  Index values
    are rank-local, as the splitters give them."""
    bounds = np.hstack([0, np.cumsum(arr.chunks[0])])
    n = int(bounds[-1])
    out = []
    for ix in idx.blocks:
        if _is_torch(ix) and ix.is_cuda:
            if not ix.numel():
                continue
            import torch

            lo, hi = (int(v) for v in torch.aminmax(ix))
            k = int(np.searchsorted(bounds, lo, side="right")) - 1
            if lo < 0 or hi >= n or hi >= bounds[k + 1]:
                raise IndexError("a device index block must name rows of one block of the array; it spans [%d, %d]"
                                 % (lo, hi))
            out.append(_gather(arr.blocks[k], ix, int(bounds[k]), validate=False))
            continue
        ix = np.asarray(ix.cpu().numpy() if _is_torch(ix) else ix)
        if ix.dtype == bool:
            ix = np.flatnonzero(ix)
        ix = ix.astype(np.int64, copy=False)
        if ix.size and (ix.min() < 0 or ix.max() >= n):
            raise IndexError("index out of range for %d rows" % n)
        which = np.searchsorted(bounds, ix, side="right") - 1
        if np.any(which[1:] < which[:-1]):
            order = np.argsort(which, kind="stable")
            ix, which = ix[order], which[order]
        cuts = np.flatnonzero(np.diff(which)) + 1
        for part, k in zip(np.split(ix, cuts), which[np.hstack([0, cuts]).astype(np.int64)] if ix.size else []):
            out.append(_gather(arr.blocks[int(k)], part, int(bounds[k]), validate=False))
    return ChunkedArray(out or [_empty_like_rows(arr.blocks[0])])


def train_test_split(*arrays, **options):
    """Split arrays into random train and test subsets, block by block (API of dask_ml.model_selection.train_test_split).

    Parameters
    ----------
    *arrays : ChunkedArray (numpy or torch blocks, host or CUDA), torch tensor (one block) or row-chunked dask array,
        1-D or 2-D, any block dtype, all with the same row chunks
    test_size, train_size : float in [0, 1], optional.  With neither, ``test_size=0.1``.
    random_state : int, RandomState instance or None
    shuffle : bool, default True.  ``False`` is not supported.
    blockwise : bool, optional.  Only ``True`` (the default) is implemented.

    Returns
    -------
    list of ChunkedArray, ``[a_train, a_test, b_train, b_test, ...]``: output block i holds rows of input block i only,
    in permutation order, where input block i was.  Arrays that are all plain numpy / pandas go to scikit-learn.
    """
    test_size = options.pop("test_size", None)
    train_size = options.pop("train_size", None)
    random_state = options.pop("random_state", None)
    shuffle = options.pop("shuffle", True)
    blockwise = options.pop("blockwise", None)

    if train_size is None and test_size is None:
        test_size = 0.1
    if options:
        raise TypeError("Unexpected options {}".format(options))
    if not shuffle:
        raise NotImplementedError("'shuffle=False' is not currently supported.")

    if not arrays or all(_is_plain(a) for a in arrays):
        import sklearn.model_selection as ms

        logger.warning("Mixture of types in 'arrays'. Falling back to scikit-learn.")
        return ms.train_test_split(*arrays, test_size=test_size, train_size=train_size, random_state=random_state,
                                   shuffle=shuffle)

    if blockwise is None:
        blockwise = True
    arrays = [_as_blocks(a) for a in arrays]
    _check_matching_blocks(arrays)
    splitter = ShuffleSplit(n_splits=1, test_size=test_size, train_size=train_size, blockwise=blockwise,
                            random_state=random_state)
    train_idx, test_idx = next(splitter.split(arrays[0]))
    pairs = ((_blockwise_slice(a, train_idx, validate=False), _blockwise_slice(a, test_idx, validate=False))
             for a in arrays)
    return list(itertools.chain.from_iterable(pairs))
