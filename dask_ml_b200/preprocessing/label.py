"""LabelEncoder with the dask_ml.preprocessing API, executed by the H100 engine.

Mirrors dask_ml/preprocessing/label.py:14-188 (reference @ 0310a90), a subclass of scikit-learn's.  Numeric y (numpy,
torch on any device, ChunkedArray, dask arrays, numeric pandas Series) runs on the device (``_encode``): ``classes_``
is ``np.unique(y)`` in y's dtype (NaN last), ``transform`` returns a device ChunkedArray of int64 codes with y's row
blocks and ``inverse_transform`` a device ChunkedArray of values.  A pandas categorical Series keeps the reference's
categorical branch; strings and objects go to scikit-learn.  Unseen labels raise ValueError on every path (the
reference's numpy branch maps them silently through ``np.searchsorted``: a documented deviation).
"""
import numpy as np
import pandas as pd
import sklearn.preprocessing
from sklearn.utils.validation import check_is_fitted

from .. import _lib
from ..chunked import ChunkedArray
from . import _encode


def _is_categorical(y):
    return isinstance(y, pd.Series) and isinstance(y.dtype, pd.CategoricalDtype)


def _unseen(values):
    return ValueError("y contains previously unseen values {}".format(list(np.asarray(values).tolist())))


class LabelEncoder(sklearn.preprocessing.LabelEncoder):
    """Encode labels with value between 0 and n_classes-1, on the device for numeric labels.

    Parameters
    ----------
    use_categorical : bool, default True
        Whether to use the categorical dtype information when `y` is a pandas Series with a categorical dtype.

    Attributes
    ----------
    classes_ : array of shape (n_class,)
        Holds the label for each class (``np.unique(y)``: sorted, NaN last, y's dtype; float32 for bfloat16 labels).
    dtype_ : Optional CategoricalDtype
        For categorical `y`, the dtype is stored here.
    """

    def __init__(self, use_categorical=True):
        self.use_categorical = use_categorical
        super().__init__()

    def _check_array(self, y):
        if isinstance(y, pd.DataFrame):
            y = y.squeeze()
            if y.ndim > 1:
                raise ValueError("Expected a 1-D array or Series.")
        if isinstance(y, pd.Series) and not (self.use_categorical and _is_categorical(y)):
            y = np.asarray(y)
        return y

    def _fit_device(self, y):
        Y, hdt = _encode.intake(y, 1)
        keys, counts = _encode.fit_keys(Y)
        self.classes_ = _encode.categories_from_keys(keys, counts, Y.dtype, hdt)[0]
        self.dtype_ = None
        return Y

    def fit(self, y):
        y = self._check_array(y)
        if _is_categorical(y):
            self.classes_ = np.asarray(y.cat.categories)
            self.dtype_ = y.dtype
            return self
        if _encode.device_input(y):
            self._fit_device(y)
            return self
        self.dtype_ = None
        return super().fit(y)

    def fit_transform(self, y):
        y = self._check_array(y)
        if _is_categorical(y):
            self.classes_ = np.asarray(y.cat.categories)
            self.dtype_ = y.dtype
            return y.cat.codes
        if _encode.device_input(y):
            return self._transform_device(self._fit_device(y))
        self.dtype_ = None
        return super().fit_transform(y)

    def _transform_device(self, Y):
        tdt = _encode.device_dtype(self.classes_.dtype)
        blocks, unknown, _ = _encode.encode(Y, [self.classes_], tdt, _lib.ENCODE_CODES)
        if unknown is not None:
            raise _unseen(unknown[0])
        return ChunkedArray([b.view(-1) for b in blocks])

    def transform(self, y):
        check_is_fitted(self, "classes_")
        y = self._check_array(y)
        if _is_categorical(y):
            assert y.dtype.categories.equals(self.dtype_.categories)
            return y.cat.codes.values
        if _encode.device_input(y) and _encode.device_dtype(np.asarray(self.classes_).dtype) is not None:
            return self._transform_device(_encode.intake(y, 1)[0])
        y = np.asarray(y)
        diff = np.setdiff1d(y, self.classes_)
        if len(diff):
            raise _unseen(diff)
        return super().transform(y)

    def inverse_transform(self, y):
        check_is_fitted(self, "classes_")
        y = self._check_array(y)
        if getattr(self, "dtype_", None):
            return pd.Series(pd.Categorical.from_codes(np.asarray(y), categories=self.dtype_.categories,
                                                       ordered=self.dtype_.ordered))
        if _encode.device_dtype(np.asarray(self.classes_).dtype) is None or not _encode.device_input(y):
            return super().inverse_transform(np.asarray(y))
        blocks, bad = _encode.decode(y, [self.classes_])
        if bad is not None:
            raise ValueError("y contains previously unseen labels: %s" % str(list(bad[0].tolist())))
        return ChunkedArray([b.view(-1) for b in blocks])
