"""OneHotEncoder with the dask_ml.preprocessing API, executed by the H100 engine.

Mirrors dask_ml/preprocessing/_encoders.py:18-244 (reference @ 0310a90): the reference's constructor, checks and
messages, with numeric arrays (numpy, torch on any device, ChunkedArray, dask arrays) encoded on the device
(``_encode``).  ``categories_`` equal scikit-learn's for the same numpy input (NaN is a category and sorts last; a zero
category is +0.0), ``sparse=True`` gives a ChunkedArray of device ``torch.sparse_csr_tensor`` blocks whose ``.compute()``
is scikit-learn's ``csr_matrix``, ``sparse=False`` a dense device ChunkedArray in ``dtype``.  Non-numeric input goes to
scikit-learn's OneHotEncoder and its learned attributes are copied.  ``inverse_transform`` of device outputs is not
implemented.
"""
import numpy as np
import sklearn.preprocessing
import torch
from sklearn.preprocessing._encoders import _check_unknown
from sklearn.utils.validation import check_is_fitted

from .. import _lib
from ..chunked import ChunkedArray
from . import _encode

# the one-hot dtypes the pass writes
_OUT = {np.dtype("float64"): torch.float64, np.dtype("float32"): torch.float32, np.dtype("int64"): torch.int64,
        np.dtype("int32"): torch.int32, np.dtype("uint8"): torch.uint8, np.dtype("bool"): torch.bool}


class OneHotEncoder(sklearn.preprocessing.OneHotEncoder):
    """Encode categorical integer features as a one-hot numeric array, on the device for numeric arrays.

    Parameters
    ----------
    n_values, categorical_features : accepted and ignored, as in the reference
    categories : 'auto' or a list of sorted arrays of values, one per feature
    sparse : bool, default True
        A ChunkedArray of device CSR blocks if True, else of dense device blocks.
    dtype : number type, default np.float64
        float64, float32, int64, int32, uint8 or bool on the device.
    handle_unknown : 'error'
        'ignore' is not implemented, as in the reference.

    Attributes
    ----------
    categories_ : list of arrays
        The categories of each feature, in X's dtype (float32 for bfloat16 input).
    dtypes_ : list of None
    """

    _legacy_mode = False
    feature_name_combiner = "concat"

    def __init__(self, n_values=None, categorical_features=None, categories="auto", sparse=True, dtype=np.float64,
                 handle_unknown="error"):
        self.n_values = n_values
        self.categorical_features = categorical_features
        self.categories = categories
        self.sparse = sparse
        self.dtype = dtype
        self.handle_unknown = handle_unknown

    def _sklearn_encoder(self):
        return sklearn.preprocessing.OneHotEncoder(categories=self.categories, sparse_output=self.sparse,
                                                   dtype=self.dtype, handle_unknown=self.handle_unknown)

    def fit(self, X, y=None):
        if self.handle_unknown == "ignore":
            raise NotImplementedError("handle_unkown='ignore' is not implemented yet.")
        if self.handle_unknown != "error":
            msg = "handle_unknown must be 'error'." "got {0}.".format(self.handle_unknown)
            raise ValueError(msg)
        self._sk = None
        if not _encode.device_input(X):
            self._sk = self._sklearn_encoder().fit(X)
            for a in ("categories_", "drop_idx_", "_drop_idx_after_grouping", "_infrequent_enabled",
                      "_n_features_outs", "n_features_in_", "feature_names_in_"):
                if hasattr(self._sk, a):
                    setattr(self, a, getattr(self._sk, a))
            self.dtypes_ = [None] * len(self.categories_)
            return self
        data, hdt = _encode.intake(X, 2)
        d = data.d
        if self.categories != "auto":
            for cats in self.categories:
                if not np.all(np.sort(cats) == np.array(cats)):
                    raise ValueError("Unsorted categories are not yet supported")
            if len(self.categories) != d:
                raise ValueError("Shape mismatch: if n_values is an array, it has to be of shape (n_features,).")
        keys, counts = _encode.fit_keys(data)
        found = _encode.categories_from_keys(keys, counts, data.dtype, hdt)
        if self.categories == "auto":
            cats = found
        else:
            cats = []
            for i in range(d):
                c = np.array(self.categories[i], dtype=hdt)
                diff = _check_unknown(found[i], c)
                if diff:
                    raise ValueError("Found unknown categories {0} in column {1} during fit".format(diff, i))
                cats.append(c)
        self.categories_ = cats
        self.dtypes_ = [None] * d
        self.n_features_in_ = d
        self.drop_idx_ = None
        self._drop_idx_after_grouping = None
        self._infrequent_enabled = False
        self._n_features_outs = [len(c) for c in cats]
        self._fit_dtype = data.dtype
        return self

    def transform(self, X):
        check_is_fitted(self, "categories_")
        if getattr(self, "_sk", None) is not None or not _encode.device_input(X):
            if getattr(self, "_sk", None) is None:
                raise ValueError("this OneHotEncoder was fitted on numeric input; transform takes numeric input")
            return self._sk.transform(X)
        out_np = np.dtype(self.dtype)
        if out_np not in _OUT:
            raise ValueError("dtype %s is not supported on the device; use one of %s" % (out_np, sorted(map(str, _OUT))))
        data, _ = _encode.intake(X, 2)
        d = data.d
        if d != len(self.categories_):
            raise ValueError("X has %d features, but OneHotEncoder is expecting %d features as input."
                             % (d, len(self.categories_)))
        layout = _lib.ENCODE_CSR if self.sparse else _lib.ENCODE_DENSE
        blocks, unknown, W = _encode.encode(data, self.categories_, self._fit_dtype, layout, _OUT[out_np])
        if unknown is not None:
            j = next(i for i, u in enumerate(unknown) if len(u))
            raise ValueError("Found unknown categories {0} in column {1} during transform"
                             .format(list(unknown[j]), j))
        if self.sparse:
            blocks = [_encode.csr_block(idx, val, int(val.shape[0]) // d, d, W) for idx, val in blocks]
        return ChunkedArray(blocks)

    def fit_transform(self, X, y=None):
        return self.fit(X).transform(X)

    def inverse_transform(self, X):
        if getattr(self, "_sk", None) is not None:
            return self._sk.inverse_transform(X)
        raise NotImplementedError("inverse_transform of the device one-hot output is not implemented")
