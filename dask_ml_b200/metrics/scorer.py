"""Scorers over the package's metrics (API of dask_ml/metrics/scorer.py): ``scorer(estimator, X, y) -> float``.

A scorer calls the estimator's ``predict`` (or ``predict_proba``) and hands the result to the device metric as it is,
so device blocks stay on the device and a ``(n,)`` class-1 probability column (``LogisticRegression.predict_proba``) is
scored as the metric scores it.  scikit-learn's ``make_scorer`` is not used: its response handling converts the
output with numpy.
"""
from . import accuracy_score, log_loss, mean_absolute_error, mean_squared_error, r2_score


class _Scorer(object):
    def __init__(self, name, metric, sign=1, response="predict"):
        self.name = name
        self.metric = metric
        self.sign = sign
        self.response = response

    def __call__(self, estimator, X, y):
        return self.sign * float(self.metric(y, getattr(estimator, self.response)(X)))

    def __repr__(self):
        return "make_scorer(%s%s%s)" % (self.metric.__name__, ", greater_is_better=False" if self.sign < 0 else "",
                                        ", response_method=%r" % self.response if self.response != "predict" else "")


SCORERS = dict(
    accuracy=_Scorer("accuracy", accuracy_score),
    neg_mean_squared_error=_Scorer("neg_mean_squared_error", mean_squared_error, -1),
    neg_mean_absolute_error=_Scorer("neg_mean_absolute_error", mean_absolute_error, -1),
    r2=_Scorer("r2", r2_score),
    neg_log_loss=_Scorer("neg_log_loss", log_loss, -1, "predict_proba"),
)


def get_scorer(scoring, compute=True):
    """The scorer named ``scoring`` in ``SCORERS``; a callable is returned as it is."""
    if isinstance(scoring, str):
        try:
            return SCORERS[scoring]
        except KeyError:
            raise ValueError("{} is not a valid scoring value. Valid options are {}".format(scoring, sorted(SCORERS)))
    return scoring


def _passthrough_score(estimator, X, y=None):
    return estimator.score(X, y)


def check_scoring(estimator, scoring=None):
    """The scorer a search uses: ``estimator.score`` for None (TypeError when there is none), ``SCORERS[scoring]``
    for a name, a callable as it is.  A metric function of this package passed as ``scoring`` is a ValueError: a
    scorer takes the estimator first."""
    if not hasattr(estimator, "fit"):
        raise TypeError("estimator should be an estimator implementing 'fit' method, %r was passed" % estimator)
    if scoring is None:
        if not hasattr(estimator, "score"):
            raise TypeError("If no scoring is specified, the estimator passed should have a 'score' method. The "
                            "estimator %r does not." % estimator)
        return _passthrough_score
    if isinstance(scoring, str):
        return get_scorer(scoring)
    if not callable(scoring):
        raise ValueError("scoring value should either be a callable, string or None. %r was passed" % scoring)
    module = getattr(scoring, "__module__", None)
    if (isinstance(module, str) and module.startswith(__package__ + ".")
            and not module.startswith(__name__) and not module.startswith(__package__ + ".tests.")):
        raise ValueError("scoring value %r looks like it is a metric function rather than a scorer. A scorer should "
                         "require an estimator as its first parameter. Please use `make_scorer` to convert a metric "
                         "to a scorer." % scoring)
    return scoring
