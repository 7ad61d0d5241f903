"""PartialPassiveAggressiveClassifier and PartialPassiveAggressiveRegressor
(dask_ml/linear_model/passive_aggressive.py), executed by the H100 engine through ``_sgd.py``."""
from sklearn import linear_model as _lm

from ._sgd import _copy_partial_doc, _PartialSGDClassifierMixin, _PartialSGDRegressorMixin


@_copy_partial_doc
class PartialPassiveAggressiveClassifier(_PartialSGDClassifierMixin, _lm.PassiveAggressiveClassifier):
    _init_kwargs = _fit_kwargs = ["classes"]


@_copy_partial_doc
class PartialPassiveAggressiveRegressor(_PartialSGDRegressorMixin, _lm.PassiveAggressiveRegressor):
    pass
