"""The block-wise partial-fit plumbing shared by the SGD family (``linear_model/_sgd.py``) and the discrete naive Bayes
pair (``naive_bayes.py``).

Mirrors dask_ml/_partial.py (reference @ 0310a90): a scikit-learn estimator with the reference's constructor (the
``_init_kwargs`` it requires), FutureWarning and ``_get_param_names``, whose ``fit`` calls ``partial_fit`` once per row
block, in the order ``check_random_state(None).shuffle`` gives.  Here the blocks stay where they are (device
ChunkedArrays, ``host_resident`` streams, numpy, CSR blocks from torch, scipy or HashingVectorizer); the input checks
run once over all of X before the first block, and each ``partial_fit`` takes a pre-validated ``_Batch``.  A model
keeps its state on the device and copies it to its numpy attributes (``_publish``) after every user-level
``partial_fit`` and once at the end of ``fit``.
"""
import warnings

import numpy as np
import torch
from sklearn.base import _fit_context
from sklearn.utils import check_random_state
from sklearn.utils.validation import _assert_all_finite

from ._sparse import _SparseData
from .chunked import ChunkedArray, _is_torch, _y_flat
from .cluster import k_means as _km
from .engine import StreamedChunks, single_process as _single_process

_partial_deprecation = (
    "'{cls.__name__}' is deprecated. Use "
    "'dask_ml.wrappers.Incremental({base.__name__}(), **kwargs)' "
    "instead."
)


def _sklearn_base(cls):
    for base in cls.mro():
        if base.__module__.startswith("sklearn"):
            return base


def _copy_partial_doc(cls):
    """The reference's docstring header and deprecation note, then the family's note (``cls._partial_doc``), over the
    scikit-learn class's documentation."""
    base = _sklearn_base(cls)
    lines = (base.__doc__ or "").split("\n")
    insert = """

    .. deprecated:: 0.6.0 (in dask-ml)
       Use the :class:`dask_ml.wrappers.Incremental` meta-estimator instead.
""" + cls._partial_doc.format(classname=base.__name__)
    cls.__doc__ = "\n".join([lines[0] + insert] + lines[1:])
    return cls


def _block_data(X):
    """Input -> ``DeviceData`` or ``_SparseData`` (the forms the GLMs take); ``_checked`` tests the values."""
    return _km._to_device_data(X, check_finite=False)


def _y_ndim_check(y):
    """scikit-learn's ``column_or_1d`` refusal of a 2-D y with more than one column."""
    first = y.blocks[0] if isinstance(y, ChunkedArray) else y
    shape = tuple(getattr(first, "shape", ()))
    if len(shape) == 2 and shape[1] != 1:
        n = int(y.shape[0]) if hasattr(y, "shape") else shape[0]
        raise ValueError("y should be a 1d array, got an array of shape {} instead.".format((n, shape[1])))


def _flags(t):
    """float64 [any NaN, any inf] of a float tensor, on its device (no host read)."""
    return torch.stack([torch.isnan(t).any(), torch.isinf(t).any()]).to(torch.float64)


def _checked(who, X, y, negative=False):
    """(``DeviceData`` / ``_SparseData``, flat y, any negative value in X) after scikit-learn's input checks, with their
    messages: a 2-D y, inconsistent lengths, NaN / inf in X or y, and (sparse X) rows whose columns are not strictly
    increasing or out of range.  With ``negative`` X is also tested for negative values (MultinomialNB refuses them; the
    caller raises where scikit-learn does), else the third value is False.  The value checks are one device pass and
    one host read."""
    Xd = _block_data(X)
    _y_ndim_check(y)
    yf = _y_flat(y, who)
    if int(yf.shape[0]) != Xd.n_local:
        raise ValueError("Found input variables with inconsistent numbers of samples: [%d, %d]"
                         % (Xd.n_local, int(yf.shape[0])))
    dev = Xd.backend.device
    flags = torch.zeros(6 if negative else 5, dtype=torch.float64, device=dev)
    if isinstance(Xd, _SparseData):
        for crow, col, val, n in Xd.blocks:
            flags[:2] += _flags(val).to(dev)
            if negative:
                flags[5] += (val < 0).any().to(torch.float64).to(dev)
            if col.numel():
                rows = torch.repeat_interleave(torch.arange(int(n), device=col.device), crow[1:] - crow[:-1])
                bad = ((col[1:] <= col[:-1]) & (rows[1:] == rows[:-1])).any() | (col < 0).any() | (col >= Xd.d).any()
                flags[4] += bad.to(torch.float64).to(dev)
    else:
        parts = Xd.chunks.parts if isinstance(Xd.chunks, StreamedChunks) else Xd.chunks
        for c in parts:
            flags[:2] += _flags(c).to(dev)
            if negative:
                flags[5] += (c < 0).any().to(torch.float64).to(dev)
    if _is_torch(yf) and yf.is_floating_point():
        flags[2:4] += _flags(yf).to(dev)
    elif not _is_torch(yf) and np.asarray(yf).dtype.kind in "fc":
        yh = np.asarray(yf)
        flags[2:4] += torch.tensor([float(np.isnan(yh).any()), float(np.isinf(yh).any())], device=dev)
    h = flags.cpu().numpy()
    for off, name in ((0, "X"), (2, "y")):
        if h[off] or h[off + 1]:
            _assert_all_finite(np.array([np.nan if h[off] else np.inf]), input_name=name, estimator_name=who)
    if h[4]:
        raise ValueError("Sparse input must be canonical CSR: the column indices of a row are not strictly "
                         "increasing, or not in [0, %d)" % Xd.d)
    return Xd, yf, bool(negative and h[5])


def _one_block(X):
    """The rows of X as one block: a dense device tensor, or a CSR (crow, col, val, n) tuple."""
    if isinstance(X, _SparseData):
        if len(X.blocks) == 1:
            return X.blocks[0]
        crows, cols, vals, base = [], [], [], 0
        for i, (crow, col, val, n) in enumerate(X.blocks):
            crows.append(crow[(0 if i == 0 else 1):] + base)
            cols.append(col)
            vals.append(val)
            base += int(col.numel())
        return torch.cat(crows), torch.cat(cols), torch.cat(vals), X.n_local
    chunks = list(X.chunks.parts) if isinstance(X.chunks, StreamedChunks) else X.chunks
    if len(chunks) == 1:
        return X.backend.to_device(chunks[0], chunks[0].dtype) if not chunks[0].is_cuda and \
            X.backend.device.type == "cuda" else chunks[0]
    return torch.cat([c.to(X.backend.device) for c in chunks])


class _Batch(object):
    """One pre-validated batch: the block, its labels and what ``partial_fit`` reads of it (``negative``: X has a
    negative value, when the model asked ``_checked`` for that test)."""

    def __init__(self, backend, block, d, sparse, np_dtype, y, negative=False):
        self.backend, self.block, self.d, self.sparse, self.np_dtype, self.y = backend, block, d, sparse, np_dtype, y
        self.negative = negative
        self.n = int(block[3]) if sparse else int(block.shape[0])


class _PartialMixin(object):
    """The reference's constructor, deprecation, ``_get_param_names`` and block-order ``fit``.  A model names the
    attribute that holds its device state (``_state_attr``), defines ``_publish(np_dtype)``, and may ask for the
    negative-value test (``_check_negative``)."""

    _init_kwargs = []
    _fit_kwargs = []
    _state_attr = None
    _check_negative = False

    def __init__(self, **kwargs):
        self._deprecated()
        missing = set(self._init_kwargs) - set(kwargs)
        if missing:
            raise TypeError("{} requires the keyword arguments {}".format(type(self), missing))
        for kwarg in self._init_kwargs:
            setattr(self, kwarg, kwargs.pop(kwarg))
        super(_PartialMixin, self).__init__(**kwargs)

    @classmethod
    def _deprecated(cls):
        warnings.warn(_partial_deprecation.format(cls=cls, base=_sklearn_base(cls)), FutureWarning)

    @classmethod
    def _get_param_names(cls):
        return list(cls._init_kwargs) + list(_sklearn_base(cls)._get_param_names())

    @_fit_context(prefer_skip_nested_validation=True)
    def fit(self, X, y=None, compute=True):
        """One ``partial_fit`` per row block of X, in the order ``check_random_state(None).shuffle`` gives (the global
        numpy RNG), continuing from the state already learned.  The learned attributes are copied from the device once,
        at the end."""
        if not compute:
            raise NotImplementedError("compute=False: %s.fit runs eagerly, there is no lazy result"
                                      % type(self).__name__)
        _single_process(type(self).__name__)
        Xd, yf, neg = _checked(type(self).__name__, X, y, self._check_negative)
        sparse = isinstance(Xd, _SparseData)
        order = list(range(len(Xd.chunk_rows)))
        check_random_state(None).shuffle(order)
        if sparse:
            blocks = (Xd.blocks[i] for i in order)
        elif isinstance(Xd.chunks, StreamedChunks):
            blocks = Xd.chunks.iter_order(order)
        else:
            blocks = (Xd.chunks[i] for i in order)
        kwargs = {k: getattr(self, k) for k in self._fit_kwargs}
        self._defer_publish = True
        try:
            for i, blk in zip(order, blocks):
                off, n = int(Xd.chunk_offsets[i]), int(Xd.chunk_rows[i])
                if n == 0:
                    continue
                batch = _Batch(Xd.backend, blk, Xd.d, sparse, Xd.np_dtype, yf[off:off + n], neg)
                self.partial_fit(batch, None, **kwargs)
        finally:
            self._defer_publish = False
        if getattr(self, self._state_attr, None) is not None:
            self._publish(Xd.np_dtype)
        return self

    def _batch(self, X, y):
        if isinstance(X, _Batch):
            return X
        Xd = _block_data(X)
        if Xd.n_local == 0:
            raise ValueError("Found array with 0 sample(s) (shape=(0, %d)) while a minimum of 1 is required by %s."
                             % (Xd.d, type(self).__name__))
        Xd, yf, neg = _checked(type(self).__name__, Xd, y, self._check_negative)
        return _Batch(Xd.backend, _one_block(Xd), Xd.d, isinstance(Xd, _SparseData), Xd.np_dtype, yf, neg)

    def _check_features(self, b, first_call):
        if first_call:
            self.n_features_in_ = b.d
        elif b.d != self.n_features_in_:
            raise ValueError("X has {} features, but {} is expecting {} features as input.".format(
                b.d, type(self).__name__, self.n_features_in_))


def _accuracy(est, X, y, sample_weight=None):
    """Mean accuracy of ``est.predict(X)`` against y, computed in float64 (on the device for numeric labels)."""
    if sample_weight is not None:
        raise NotImplementedError("sample_weight is not supported by score")
    pred = est.predict(X)
    p = torch.cat(list(pred.blocks)) if isinstance(pred, ChunkedArray) else pred
    yf = _y_flat(y, type(est).__name__ + ".score")
    if _is_torch(p) and _is_torch(yf):
        return float((p.to(torch.float64) == yf.to(p.device, torch.float64)).to(torch.float64).mean())
    ph = p.cpu().numpy() if _is_torch(p) else np.asarray(p)
    yh = yf.cpu().numpy() if _is_torch(yf) else np.asarray(yf)
    return float(np.mean(ph == yh))
