"""PartialPerceptron (dask_ml/linear_model/perceptron.py), executed by the H100 engine through ``_sgd.py``."""
from sklearn.linear_model import Perceptron as _Perceptron

from ._sgd import _copy_partial_doc, _PartialSGDClassifierMixin


@_copy_partial_doc
class PartialPerceptron(_PartialSGDClassifierMixin, _Perceptron):
    _init_kwargs = ["classes"]
    _fit_kwargs = ["classes"]
