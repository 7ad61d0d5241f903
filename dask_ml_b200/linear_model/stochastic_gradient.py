"""PartialSGDClassifier and PartialSGDRegressor (dask_ml/linear_model/stochastic_gradient.py), executed by the H100
engine through the shared driver in ``_sgd.py``."""
from sklearn.linear_model import SGDClassifier as _SGDClassifier
from sklearn.linear_model import SGDRegressor as _SGDRegressor

from ._sgd import _copy_partial_doc, _PartialSGDClassifierMixin, _PartialSGDRegressorMixin


@_copy_partial_doc
class PartialSGDClassifier(_PartialSGDClassifierMixin, _SGDClassifier):
    _init_kwargs = ["classes"]
    _fit_kwargs = ["classes"]


@_copy_partial_doc
class PartialSGDRegressor(_PartialSGDRegressorMixin, _SGDRegressor):
    pass
