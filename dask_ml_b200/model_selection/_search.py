"""GridSearchCV and RandomizedSearchCV with the dask_ml.model_selection API (dask_ml/model_selection/_search.py,
methods.py), run split by split on the blocks' devices.

For each split X and y are materialised once for train and for test, then every candidate is cloned, set, fitted and
scored on them, one after another on the device stream; the split's rows are released before the next split is built,
so at most one split's copies are resident.  How a split is materialised depends on the splitter:

    KFold(shuffle=False)        row-slice views of the blocks of X and y: no copy, no launch
    KFold(shuffle=True),        the index pieces gathered by ``_split._take`` (one ``bkm_gather_rows_chunk`` per piece
    ShuffleSplit                of a device block, numpy for a host block)
    a scikit-learn splitter,    run on the host, on y and groups copied to the host and an (n, 0) placeholder for X
    an iterable of index pairs  (scikit-learn's splitters read only its length); its indices go through ``_take``

y is cut into the same pieces as X, so the metrics see aligned ``(y, prediction)`` blocks.  Host input (numpy, a host
ChunkedArray) is split on the host and every fit receives host blocks.  With torch.distributed every rank runs the same
candidates on its own rows; the estimators and metrics all-reduce, so every rank computes the same scores and the same
``cv_results_`` apart from the timings.  Pipelines and FeatureUnions are opaque estimators: cloned and fitted whole.
"""
import numbers
import warnings
from collections import defaultdict
from collections.abc import Sequence
from multiprocessing import cpu_count
from timeit import default_timer

import numpy as np
from numpy.ma import MaskedArray
from scipy.stats import rankdata
from sklearn import model_selection
from sklearn.base import BaseEstimator, MetaEstimatorMixin, clone, is_classifier
from sklearn.exceptions import FitFailedWarning, NotFittedError
from sklearn.model_selection._split import (
    BaseShuffleSplit,
    LeaveOneGroupOut,
    LeaveOneOut,
    LeavePGroupsOut,
    LeavePOut,
    PredefinedSplit,
    StratifiedKFold,
    _BaseKFold,
    _CVIterableWrapper,
)
from sklearn.utils._available_if import available_if
from sklearn.utils.multiclass import type_of_target
from sklearn.utils.validation import check_is_fitted

from ..chunked import ChunkedArray, _is_torch, block_to_numpy
from ..metrics.scorer import check_scoring
from ._split import KFold, ShuffleSplit, _as_blocks, _empty_like_rows, _take

__all__ = ["GridSearchCV", "RandomizedSearchCV", "check_cv", "compute_n_splits"]


# ------------ #
# CV splitting #
# ------------ #
def _is_chunked(a):
    return a is not None and not isinstance(a, np.ndarray) and (isinstance(a, ChunkedArray) or _is_torch(a)
                                                                  or hasattr(a, "chunks"))


def _host(a):
    """A 1-D label or group array on the host (the only host copies a search makes, and only where asked for)."""
    if a is None:
        return None
    blocks = _as_blocks(a).blocks
    return np.concatenate([np.asarray(block_to_numpy(b) if _is_torch(b) else b) for b in blocks])


def check_cv(cv=3, y=None, classifier=False):
    """The splitter a search uses (dask_ml.model_selection.check_cv).  None means 3; an integer is this package's
    ``KFold``, or scikit-learn's ``StratifiedKFold`` for a classifier whose y is binary or multiclass (the type is read
    from y on the host); a splitter passes through and an iterable of (train, test) pairs is wrapped, as in
    scikit-learn."""
    if cv is None:
        cv = 3
    if isinstance(cv, numbers.Integral):
        if classifier and y is not None and type_of_target(_host(y)) in ("binary", "multiclass"):
            return StratifiedKFold(cv)
        return KFold(cv)
    return model_selection.check_cv(cv, None, classifier=classifier)


def compute_n_splits(cv, X, y=None, groups=None):
    """The number of splits ``cv`` makes of X (dask_ml.model_selection.compute_n_splits)."""
    if not any(_is_chunked(a) for a in (X, y, groups)):
        return cv.get_n_splits(X, y, groups)
    if isinstance(cv, (KFold, ShuffleSplit, _BaseKFold, BaseShuffleSplit)):
        return cv.n_splits
    if isinstance(cv, PredefinedSplit):
        return len(cv.unique_folds)
    if isinstance(cv, _CVIterableWrapper):
        return len(cv.cv)
    if isinstance(cv, (LeaveOneOut, LeavePOut)):
        return cv.get_n_splits(np.zeros((len(_as_blocks(X)), 0)))
    return cv.get_n_splits(np.zeros((len(_as_blocks(X)), 0)), _host(y), _host(groups))


def _rows_like(y, chunks):
    """y as a ChunkedArray with the row chunks of X: as it is when they agree, else re-cut (views of one flat copy,
    made on y's device when every block of y is a tensor)."""
    if y is None:
        return None
    Y = _as_blocks(y)
    if Y.chunks[0] == tuple(chunks):
        return Y
    if all(_is_torch(b) for b in Y.blocks):
        import torch

        flat = torch.cat([b.to(Y.blocks[0].device) for b in Y.blocks])
    else:
        flat = np.concatenate([np.asarray(block_to_numpy(b) if _is_torch(b) else b) for b in Y.blocks])
    if int(flat.shape[0]) != int(sum(chunks)):
        raise ValueError("Found input variables with inconsistent numbers of samples: [%d, %d]"
                         % (int(sum(chunks)), int(flat.shape[0])))
    return ChunkedArray.from_array(flat, (tuple(chunks),))


def _views(a, pieces):
    """The rows (block, start, stop) of ``pieces`` as views of ``a``'s blocks, one block per piece."""
    if a is None:
        return None
    return ChunkedArray([a.blocks[i][s:e] for i, s, e in pieces] or [_empty_like_rows(a.blocks[0])])


def _splits(cv, X, y, groups):
    """(X_train, y_train, X_test, y_test) of every split, built when asked for."""
    if isinstance(cv, KFold) and not cv.shuffle:
        for train, test in cv._windows(X.chunks[0]):
            yield _views(X, train), _views(y, train), _views(X, test), _views(y, test)
        return
    if isinstance(cv, (KFold, ShuffleSplit)):
        pairs = cv.split(X, y, groups)
    else:
        from ..engine import Comm

        if Comm().world > 1:
            raise NotImplementedError("%s runs on the host over all rows, which one process holds only with a single "
                                      "rank; use dask_ml_b200.model_selection.KFold or ShuffleSplit with "
                                      "torch.distributed" % type(cv).__name__)
        placeholder = np.zeros((len(X), 0))
        pairs = ((ChunkedArray([np.asarray(tr)]), ChunkedArray([np.asarray(te)]))
                 for tr, te in cv.split(placeholder, _host(y), _host(groups)))
    for train, test in pairs:
        yield (_take(X, train), None if y is None else _take(y, train),
               _take(X, test), None if y is None else _take(y, test))


def _normalize_n_jobs(n_jobs):
    if not isinstance(n_jobs, int):
        raise TypeError("n_jobs should be an int, got %s" % n_jobs)
    if n_jobs == -1:
        return None
    if n_jobs < -1:
        return cpu_count() + 1 + n_jobs
    return n_jobs


def _check_param_grid(param_grid):
    """The checks scikit-learn < 1.1's helper of this name made, which the reference calls."""
    if hasattr(param_grid, "items"):
        param_grid = [param_grid]
    for p in param_grid:
        for name, v in p.items():
            if isinstance(v, np.ndarray) and v.ndim > 1:
                raise ValueError("Parameter array should be one-dimensional.")
            if isinstance(v, str) or not isinstance(v, (np.ndarray, Sequence)):
                raise ValueError("Parameter values for parameter ({0}) need to be a sequence(but not a string) or "
                                 "np.ndarray.".format(name))
            if len(v) == 0:
                raise ValueError("Parameter values for parameter ({0}) need to be a non-empty sequence."
                                 .format(name))


# ------------------- #
# fitting and scoring #
# ------------------- #
def _check_multimetric_scoring(estimator, scoring):
    """({name: scorer}, multimetric): one scorer named "score", or the scorers of a list / tuple / set of names or a
    dict of names to scorers."""
    if scoring is None or isinstance(scoring, str) or callable(scoring):
        return {"score": check_scoring(estimator, scoring)}, False
    if isinstance(scoring, (list, tuple, set)):
        keys = list(scoring)
        if not keys:
            raise ValueError("The list/tuple elements must be unique strings of predefined scorers. Empty list was "
                             "given. %r was passed" % (scoring,))
        if len(set(keys)) < len(keys):
            raise ValueError("The list/tuple elements must be unique strings of predefined scorers. Duplicate "
                             "elements were found in the given list. %r" % (scoring,))
        if not all(isinstance(k, str) for k in keys):
            raise ValueError("The list/tuple elements must be unique strings of predefined scorers. One or more of "
                             "the elements were callables. Use a dict of score name mapped to the scorer callable. "
                             "Got %r" % (scoring,))
        return {k: check_scoring(estimator, k) for k in keys}, True
    if isinstance(scoring, dict):
        if not scoring:
            raise ValueError("An empty dict was passed. %r" % (scoring,))
        if not all(isinstance(k, str) for k in scoring):
            raise ValueError("Non-string types were found in the keys of the given dict. scoring=%r" % (scoring,))
        return {k: check_scoring(estimator, v) for k, v in scoring.items()}, True
    raise ValueError("scoring value should either be a callable, string or None. %r was passed" % (scoring,))


def _score(est, X, y, scorers):
    return {k: float(s(est, X) if y is None else s(est, X, y)) for k, s in scorers.items()}


def _fit_and_score(estimator, params, parts, scorers, error_score, fit_params, return_train_score):
    """(fit time, score time, {name: test score}, {name: train score} or None) of one candidate on one split."""
    X_train, y_train, X_test, y_test = parts
    start = default_timer()
    try:
        est = clone(estimator).set_params(**params)
        est.fit(X_train, y_train, **fit_params)
    except Exception as e:
        if error_score == "raise":
            raise
        warnings.warn("Classifier fit failed. The score on this train-test partition for these parameters will be "
                      "set to %f. Details: \n%r" % (error_score, e), FitFailedWarning)
        failed = {k: error_score for k in scorers}
        return default_timer() - start, 0.0, failed, failed if return_train_score else None
    fit_time = default_timer() - start
    start = default_timer()
    try:
        test = _score(est, X_test, y_test, scorers)
    except Exception:
        if error_score == "raise":
            raise
        failed = {k: error_score for k in scorers}
        return fit_time, default_timer() - start, failed, failed if return_train_score else None
    score_time = default_timer() - start
    train = _score(est, X_train, y_train, scorers) if return_train_score else None
    return fit_time, score_time, test, train


def _store(results, key_name, array, weights=None, splits=False, rank=False):
    """Scores or times of shape (n_splits, n_candidates) into ``cv_results_`` (methods.py:328-356)."""
    array = np.asarray(array, dtype=np.float64).T
    if splits:
        for i in range(array.shape[1]):
            results["split%d_%s" % (i, key_name)] = array[:, i]
    means = np.average(array, axis=1, weights=weights)
    results["mean_%s" % key_name] = means
    results["std_%s" % key_name] = np.sqrt(np.average((array - means[:, None]) ** 2, axis=1, weights=weights))
    if rank:
        if np.isnan(means).all():
            ranks = np.ones(len(means), dtype=np.int32)
        else:                                        # a candidate whose mean is NaN ranks last, as in scikit-learn
            means = np.where(np.isnan(means), np.nanmin(means) - 1, means)
            ranks = rankdata(-means, method="min").astype(np.int32)
        results["rank_%s" % key_name] = ranks


def _estimator_has(attr):
    def check(self):
        return hasattr(getattr(self, "best_estimator_", self.estimator), attr)
    return check


class DaskBaseSearchCV(BaseEstimator, MetaEstimatorMixin):
    """Base class of the hyper-parameter searches with cross-validation."""

    def __init__(self, estimator, scoring=None, iid=True, refit=True, cv=None, error_score="raise",
                 return_train_score=True, scheduler=None, n_jobs=-1, cache_cv=True):
        self.scoring = scoring
        self.estimator = estimator
        self.iid = iid
        self.refit = refit
        self.cv = cv
        self.error_score = error_score
        self.return_train_score = return_train_score
        self.scheduler = scheduler
        self.n_jobs = n_jobs
        self.cache_cv = cache_cv

    def _check_if_refit(self, attr):
        if not self.refit:
            raise AttributeError("'{}' is not a valid attribute with 'refit=False'.".format(attr))

    @property
    def best_params_(self):
        check_is_fitted(self, "cv_results_")
        self._check_if_refit("best_params_")
        return self.cv_results_["params"][self.best_index_]

    @property
    def best_score_(self):
        check_is_fitted(self, "cv_results_")
        self._check_if_refit("best_score_")
        key = self.refit if self.multimetric_ else "score"
        return self.cv_results_["mean_test_{}".format(key)][self.best_index_]

    def _check_is_fitted(self, method_name):
        if not self.refit:
            raise NotFittedError("This {0} instance was initialized with refit=False. {1} is available only after "
                                 "refitting on the best parameters.".format(type(self).__name__, method_name))
        check_is_fitted(self, "best_estimator_")

    @property
    def classes_(self):
        self._check_is_fitted("classes_")
        return self.best_estimator_.classes_

    @available_if(_estimator_has("predict"))
    def predict(self, X):
        self._check_is_fitted("predict")
        return self.best_estimator_.predict(X)

    @available_if(_estimator_has("predict_proba"))
    def predict_proba(self, X):
        self._check_is_fitted("predict_proba")
        return self.best_estimator_.predict_proba(X)

    @available_if(_estimator_has("predict_log_proba"))
    def predict_log_proba(self, X):
        self._check_is_fitted("predict_log_proba")
        return self.best_estimator_.predict_log_proba(X)

    @available_if(_estimator_has("decision_function"))
    def decision_function(self, X):
        self._check_is_fitted("decision_function")
        return self.best_estimator_.decision_function(X)

    @available_if(_estimator_has("transform"))
    def transform(self, X):
        self._check_is_fitted("transform")
        return self.best_estimator_.transform(X)

    @available_if(_estimator_has("inverse_transform"))
    def inverse_transform(self, Xt):
        self._check_is_fitted("inverse_transform")
        return self.best_estimator_.inverse_transform(Xt)

    def score(self, X, y=None):
        """The refit scorer (``scoring``, or the estimator's ``score``) of ``best_estimator_`` on X and y."""
        self._check_is_fitted("score")
        scorer = self.scorer_[self.refit] if self.multimetric_ else self.scorer_
        return scorer(self.best_estimator_, X) if y is None else scorer(self.best_estimator_, X, y)

    def fit(self, X, y=None, groups=None, **fit_params):
        """Fit and score every candidate on every split, then refit the best candidate on all of X and y.

        ``fit_params`` go unchanged to every fit (no estimator of this package takes per-row fit parameters)."""
        estimator = self.estimator
        scorers, multimetric = _check_multimetric_scoring(estimator, self.scoring)
        if multimetric and self.refit is not False and (not isinstance(self.refit, str) or self.refit not in scorers):
            raise ValueError("For multi-metric scoring, the parameter refit must be set to a scorer key to refit an "
                             "estimator with the best parameter setting on the whole data and make the best_* "
                             "attributes available for that metric. If this is not needed, refit should be set to "
                             "False explicitly. %r was passed." % (self.refit,))
        self.multimetric_ = multimetric
        self.scorer_ = scorers if multimetric else scorers["score"]
        error_score = self.error_score
        if not (isinstance(error_score, numbers.Number) or error_score == "raise"):
            raise ValueError("error_score must be the string 'raise' or a numeric value.")
        _normalize_n_jobs(self.n_jobs)

        candidates = list(self._get_param_iterator())
        Xc = _as_blocks(X)
        yc = _rows_like(y, Xc.chunks[0])
        cv = check_cv(self.cv, y, is_classifier(estimator))
        n_splits = compute_n_splits(cv, Xc, yc, groups)
        self.n_splits_ = n_splits

        shape = (n_splits, len(candidates))
        fit_times, score_times = np.zeros(shape), np.zeros(shape)
        test = {k: np.zeros(shape) for k in scorers}
        train = {k: np.zeros(shape) for k in scorers} if self.return_train_score else None
        test_rows = []
        s = -1
        for s, parts in enumerate(_splits(cv, Xc, yc, groups)):
            if s >= n_splits:
                break
            test_rows.append(len(parts[2]))
            for c, params in enumerate(candidates):
                fit_times[s, c], score_times[s, c], te, tr = _fit_and_score(
                    estimator, params, parts, scorers, error_score, fit_params, self.return_train_score)
                for k in scorers:
                    test[k][s, c] = te[k]
                    if train is not None:
                        train[k][s, c] = tr[k]
            del parts                                  # the split's rows go before the next split is built
        if s + 1 != n_splits:
            raise ValueError("cv.split and cv.get_n_splits returned inconsistent results. Expected {} splits, got {}"
                             .format(n_splits, s + 1))

        from ..engine import Comm

        weights = None
        if self.iid:                                   # the global test-fold sizes
            weights = np.sum(np.asarray(Comm().allgather_obj(test_rows), dtype=np.float64), axis=0)
        results = {"params": candidates}
        _store(results, "fit_time", fit_times)
        _store(results, "score_time", score_times)
        for k in scorers:
            name = k if multimetric else "score"
            _store(results, "test_%s" % name, test[k], weights=weights, splits=True, rank=True)
            if train is not None:
                _store(results, "train_%s" % name, train[k], splits=True)
        params = defaultdict(lambda: MaskedArray(np.empty(len(candidates)), mask=True, dtype=object))
        for i, p in enumerate(candidates):
            for name, value in p.items():
                params["param_%s" % name][i] = value
        results.update(params)
        self.cv_results_ = results

        if self.refit:
            key = self.refit if multimetric else "score"
            self.best_index_ = int(np.flatnonzero(results["rank_test_{}".format(key)] == 1)[0])
            best = clone(estimator).set_params(**candidates[self.best_index_])
            self.best_estimator_ = best.fit(X, y, **fit_params)
        return self


_PARAMETERS = """
    estimator : estimator object
        Fitted and scored whole for every candidate and split (a Pipeline or FeatureUnion too).  It needs a ``score``
        method unless ``scoring`` is given.
    scoring : str, callable, list / tuple of names, dict of names to scorers, or None
        A name of ``dask_ml_b200.metrics.SCORERS``, a scorer ``scorer(estimator, X, y) -> float``, several of them,
        or None for ``estimator.score``.
    iid : bool, default True
        Weight the mean and standard deviation of the test scores by the test-fold sizes (summed over ranks).
    refit : bool or str, default True
        Refit the best candidate on all of X and y as ``best_estimator_``; with several scorers, the name of the one
        that chooses it (or False).
    cv : int, splitter, iterable of (train, test) index arrays, or None (3)
        See ``check_cv``.  ``KFold`` and ``ShuffleSplit`` of this package keep the folds on the blocks' devices.
    error_score : 'raise' or a number
        The score of a candidate whose fit fails (with a ``FitFailedWarning``), or 'raise' to raise.
    return_train_score : bool, default True
    scheduler, n_jobs, cache_cv :
        Accepted for the reference's signature (``n_jobs`` is validated as there).  Candidates run one after another
        on the device stream, and one split's rows are resident at a time.

    Attributes
    ----------
    cv_results_ : dict of numpy (masked) arrays, the reference's keys (``params``, ``param_<name>``,
        ``split<i>_test_<score>``, ``mean_`` / ``std_`` / ``rank_test_<score>``, the train keys, the fit and score
        times)
    best_estimator_, best_params_, best_score_, best_index_, scorer_, n_splits_, multimetric_
"""


class GridSearchCV(DaskBaseSearchCV):
    __doc__ = """Exhaustive search over a parameter grid (API of dask_ml.model_selection.GridSearchCV).

    Parameters
    ----------
    param_grid : dict or list of dicts
        Parameter names mapped to lists of values; every combination is a candidate (scikit-learn's ParameterGrid).
""" + _PARAMETERS

    def __init__(self, estimator, param_grid, scoring=None, iid=True, refit=True, cv=None, error_score="raise",
                 return_train_score=True, scheduler=None, n_jobs=-1, cache_cv=True):
        super(GridSearchCV, self).__init__(estimator=estimator, scoring=scoring, iid=iid, refit=refit, cv=cv,
                                           error_score=error_score, return_train_score=return_train_score,
                                           scheduler=scheduler, n_jobs=n_jobs, cache_cv=cache_cv)
        _check_param_grid(param_grid)
        self.param_grid = param_grid

    def _get_param_iterator(self):
        return model_selection.ParameterGrid(self.param_grid)


class RandomizedSearchCV(DaskBaseSearchCV):
    __doc__ = """Randomized search over parameter distributions (API of dask_ml.model_selection.RandomizedSearchCV).

    Parameters
    ----------
    param_distributions : dict
        Parameter names mapped to distributions (with an ``rvs`` method) or lists to sample from (scikit-learn's
        ParameterSampler).
    n_iter : int, default 10
        The number of candidates sampled.
    random_state : int, RandomState instance or None
""" + _PARAMETERS

    def __init__(self, estimator, param_distributions, n_iter=10, random_state=None, scoring=None, iid=True,
                 refit=True, cv=None, error_score="raise", return_train_score=True, scheduler=None, n_jobs=-1,
                 cache_cv=True):
        super(RandomizedSearchCV, self).__init__(estimator=estimator, scoring=scoring, iid=iid, refit=refit, cv=cv,
                                                 error_score=error_score, return_train_score=return_train_score,
                                                 scheduler=scheduler, n_jobs=n_jobs, cache_cv=cache_cv)
        self.param_distributions = param_distributions
        self.n_iter = n_iter
        self.random_state = random_state

    def _get_param_iterator(self):
        return model_selection.ParameterSampler(self.param_distributions, self.n_iter, random_state=self.random_state)
