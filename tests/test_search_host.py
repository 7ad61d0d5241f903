"""KFold, check_cv / compute_n_splits, the scorers and the searches on host blocks: KFold against scikit-learn and the
reference's chunk structure, and GridSearchCV driving scikit-learn estimators against scikit-learn's GridSearchCV on the
same rows."""
import numpy as np
import pytest
import sklearn.model_selection as skms
from scipy.stats import loguniform
from sklearn.exceptions import FitFailedWarning, NotFittedError
from sklearn.linear_model import LogisticRegression, Ridge
from sklearn.model_selection._split import _CVIterableWrapper

from dask_ml_b200 import ChunkedArray
from dask_ml_b200.metrics import SCORERS, accuracy_score, check_scoring, get_scorer, r2_score
from dask_ml_b200.model_selection import (
    GridSearchCV,
    KFold,
    RandomizedSearchCV,
    ShuffleSplit,
    check_cv,
    compute_n_splits,
)
from dask_ml_b200.model_selection._split import _take, permutation_indices

# The reference's tests/model_selection/test_split.py::test_kfold: 110 rows in blocks (50, 50, 10), five folds.
REF_KFOLD_CHUNKS = [
    ((28, 50, 10), (22,)),
    ((22, 6, 50, 10), (22,)),
    ((44, 34, 10), (6, 16)),
    ((50, 16, 12, 10), (22,)),
    ((50, 38), (12, 10)),
]


def _chunked(a, chunks):
    return ChunkedArray.from_array(a, (tuple(chunks),))


def _expected_chunks(chunks, k):
    """The reference's pieces restated: per block, train before the window, test, train after it."""
    n = sum(chunks)
    sizes = [n // k + (1 if f < n % k else 0) for f in range(k)]
    out, t0 = [], 0
    for s in sizes:
        t1, train, test, start = t0 + s, [], [], 0
        for c in chunks:
            stop = start + c
            a, b = max(t0, start), min(t1, stop)
            if min(a, stop) > start:
                train.append(min(a, stop) - start)
            if a < b:
                test.append(b - a)
            if max(b, start) < stop:
                train.append(stop - max(b, start))
            start = stop
        out.append((tuple(train), tuple(test)))
        t0 = t1
    return out


@pytest.mark.parametrize("shuffle", [False, True])
def test_kfold_chunks_equal_the_reference(shuffle):
    X = _chunked(np.arange(220.0).reshape(110, 2), (50, 50, 10))
    folds = list(KFold(n_splits=5, shuffle=shuffle, random_state=0).split(X))
    assert [(tr.chunks[0], te.chunks[0]) for tr, te in folds] == REF_KFOLD_CHUNKS
    assert KFold(5).get_n_splits() == 5
    for tr, te in folds:
        assert tr.dtype == np.int64 and te.dtype == np.int64
        np.testing.assert_array_equal(np.sort(np.concatenate([tr.compute(), te.compute()])), np.arange(110))


@pytest.mark.parametrize("chunks,k", [((50, 50, 10), 5), ((7, 30, 1, 13, 49), 4), ((100,), 3), ((5, 3, 4), 12),
                                      ((1, 1, 1), 3), ((33, 0, 21), 7)])
def test_kfold_unshuffled_equals_scikit_learn(chunks, k):
    n = sum(chunks)
    X = _chunked(np.zeros((n, 3)), chunks)
    ours = list(KFold(k, random_state=0).split(X))               # random_state is ignored without shuffle
    theirs = list(skms.KFold(k).split(np.zeros((n, 3))))
    assert len(ours) == len(theirs) == k
    for (tr, te), (str_, ste) in zip(ours, theirs):
        np.testing.assert_array_equal(tr.compute(), str_)
        np.testing.assert_array_equal(te.compute(), ste)
    assert [(tr.chunks[0], te.chunks[0]) for tr, te in ours] == _expected_chunks(chunks, k)


@pytest.mark.parametrize("chunks,k", [((50, 50, 10), 5), ((7, 30, 1, 13, 49), 4), ((64,), 3), ((5, 3, 4), 12)])
def test_kfold_shuffled_pieces_are_the_block_permutation(chunks, k):
    n = sum(chunks)
    X = _chunked(np.zeros(n), chunks)
    seeds = np.random.RandomState(7).randint(0, 2 ** 32 - 1, size=len(chunks), dtype="u8")   # ShuffleSplit's draw
    offsets = np.hstack([0, np.cumsum(chunks)])
    tests = []
    folds = list(KFold(k, shuffle=True, random_state=7).split(X))
    starts = np.cumsum([0] + [n // k + (1 if f < n % k else 0) for f in range(k)])
    for f, (tr, te) in enumerate(folds):
        a, b = tr.compute(), te.compute()
        assert not np.intersect1d(a, b).size
        np.testing.assert_array_equal(np.sort(np.concatenate([a, b])), np.arange(n))
        tests.append(b)
        # every piece of the test window is offset + pi_seed(p) over its positions
        t0, t1, got = starts[f], starts[f + 1], []
        for i, c in enumerate(chunks):
            lo, hi = max(t0, offsets[i]), min(t1, offsets[i + 1])
            if lo < hi:
                got.append(permutation_indices(seeds[i], c, np.arange(lo, hi) - offsets[i]) + offsets[i])
        np.testing.assert_array_equal(b, np.concatenate(got))
    np.testing.assert_array_equal(np.sort(np.concatenate(tests)), np.arange(n))
    again = list(KFold(k, shuffle=True, random_state=7).split(X))
    for (tr, te), (tr2, te2) in zip(folds, again):
        np.testing.assert_array_equal(tr.compute(), tr2.compute())
        np.testing.assert_array_equal(te.compute(), te2.compute())


def test_kfold_validation():
    X = _chunked(np.zeros(4), (2, 2))
    with pytest.raises(ValueError, match="greater than the number of samples"):
        next(KFold(5).split(X))
    for bad in (1, 0, 2.0, "3"):
        with pytest.raises(ValueError):
            KFold(bad)
    assert len(list(KFold(4).split(X))) == 4                  # n_splits == n: one row per test part


def test_take_cuts_index_blocks_at_block_boundaries():
    X = _chunked(np.arange(40.0).reshape(20, 2), (6, 4, 10))
    idx = ChunkedArray([np.array([0, 3, 5, 6, 9, 10, 19]), np.array([12, 11])])
    out = _take(X, idx)
    assert out.chunks[0] == (3, 2, 2, 2)
    np.testing.assert_array_equal(out.compute(), X.compute()[[0, 3, 5, 6, 9, 10, 19, 12, 11]])
    shuffled = _take(X, ChunkedArray([np.array([10, 0, 12, 1])]))  # grouped by source block, stable within
    np.testing.assert_array_equal(shuffled.compute(), X.compute()[[0, 1, 10, 12]])
    with pytest.raises(IndexError):
        _take(X, ChunkedArray([np.array([20])]))


# ---- check_cv / compute_n_splits (the reference's test_check_cv) ---------------------------------------------------
def test_check_cv():
    cv = check_cv(3, classifier=False)
    assert isinstance(cv, KFold) and cv.n_splits == 3
    cv = check_cv(5, classifier=False)
    assert isinstance(cv, KFold) and cv.n_splits == 5
    assert isinstance(check_cv(None), KFold) and check_cv(None).n_splits == 3

    dy = _chunked(np.array([1, 0, 1, 0, 1]), (2, 2, 1))
    assert isinstance(check_cv(y=dy, classifier=False), KFold)

    for y in (np.array([0, 1, 0, 1, 0, 0, 1, 1, 1]), np.array([0, 1, 0, 1, 2, 1, 2, 0, 2])):
        cv = check_cv(5, y, classifier=True)
        assert isinstance(cv, skms.StratifiedKFold) and cv.n_splits == 5
        cv = check_cv(5, _chunked(y, (2, 2, 2, 2, 1)), classifier=True)
        assert isinstance(cv, skms.StratifiedKFold) and cv.n_splits == 5

    y = np.array([[1, 2], [0, 3], [0, 0], [3, 1], [2, 0]])
    assert isinstance(check_cv(y=y, classifier=True), KFold)
    dy = _chunked(y, (2, 2, 1))
    assert isinstance(check_cv(y=dy, classifier=True), KFold)

    cv = [np.array([True, False, True]), np.array([False, True, False])]
    assert isinstance(check_cv(cv, y=dy, classifier=True), _CVIterableWrapper)

    cv = skms.ShuffleSplit()
    assert check_cv(cv, dy, classifier=True) is cv
    assert check_cv(cv, dy, classifier=False) is cv
    ours = ShuffleSplit()
    assert check_cv(ours, dy, classifier=True) is ours


def test_compute_n_splits():
    X = np.zeros((12, 2))
    dX = _chunked(X, (5, 7))
    assert compute_n_splits(KFold(4), dX) == 4
    assert compute_n_splits(skms.StratifiedKFold(3), dX) == 3
    assert compute_n_splits(skms.ShuffleSplit(6), dX) == 6
    assert compute_n_splits(skms.LeaveOneOut(), dX) == 12
    assert compute_n_splits(skms.PredefinedSplit([0, 0, 1, 1, 2, 2, -1, -1, 0, 1, 2, 0]), dX) == 3
    groups = np.array([0, 0, 1, 1, 2, 2, 3, 3, 0, 1, 2, 3])
    assert compute_n_splits(skms.LeaveOneGroupOut(), dX, groups=_chunked(groups, (5, 7))) == 4
    assert compute_n_splits(check_cv([(np.arange(3), np.arange(3, 6))]), dX) == 1
    assert compute_n_splits(skms.KFold(3), X) == 3


# ---- scorers -------------------------------------------------------------------------------------------------------
class _NoScore(object):
    def fit(self, X, y=None):
        return self


def test_scorers():
    assert set(SCORERS) == {"accuracy", "neg_mean_squared_error", "neg_mean_absolute_error", "r2", "neg_log_loss"}
    assert get_scorer("r2") is SCORERS["r2"]
    assert check_scoring(Ridge(), "accuracy") is SCORERS["accuracy"]
    with pytest.raises(ValueError, match="Valid options are"):
        get_scorer("no_such_score")
    with pytest.raises(ValueError, match="Valid options are"):
        check_scoring(Ridge(), "no_such_score")
    with pytest.raises(ValueError, match="metric function"):
        check_scoring(Ridge(), accuracy_score)
    with pytest.raises(TypeError, match="score"):
        check_scoring(_NoScore())

    def mine(est, X, y):
        return 1.0

    assert check_scoring(Ridge(), mine) is mine
    rng = np.random.RandomState(0)
    X = rng.randn(80, 3)
    y = X @ [1.0, -1.0, 2.0] + 0.1 * rng.randn(80)
    est = Ridge().fit(X, y)
    dX, dy = _chunked(X, (30, 50)), _chunked(y, (30, 50))
    np.testing.assert_allclose(SCORERS["r2"](est, dX, dy), r2_score(y, est.predict(X)), rtol=1e-12)
    np.testing.assert_allclose(SCORERS["neg_mean_squared_error"](est, dX, dy),
                               -np.mean((y - est.predict(X)) ** 2), rtol=1e-12)
    np.testing.assert_allclose(SCORERS["neg_mean_absolute_error"](est, dX, dy),
                               -np.mean(np.abs(y - est.predict(X))), rtol=1e-12)
    np.testing.assert_allclose(check_scoring(est)(est, dX, dy), est.score(X, y), rtol=1e-12)
    yc = (y > 0).astype(np.int64)
    clf = LogisticRegression().fit(X, yc)
    np.testing.assert_allclose(SCORERS["accuracy"](clf, dX, _chunked(yc, (30, 50))), clf.score(X, yc), rtol=1e-12)
    from sklearn.metrics import log_loss as sk_log_loss

    np.testing.assert_allclose(SCORERS["neg_log_loss"](clf, dX, _chunked(yc, (30, 50))),
                               -sk_log_loss(yc, clf.predict_proba(X)), rtol=1e-12)


# ---- searches against scikit-learn ---------------------------------------------------------------------------------
def _regression(n=251, d=6, seed=0):
    rng = np.random.RandomState(seed)
    X = rng.randn(n, d)
    return X, X @ rng.randn(d) + 0.5 * rng.randn(n)


CASES = [
    ("ridge", Ridge(), {"alpha": [0.01, 0.3, 3.0, 100.0]}),
    ("logistic", LogisticRegression(), {"C": [0.001, 0.03, 1.0, 30.0]}),
]


@pytest.mark.parametrize("name,est,grid", CASES, ids=[c[0] for c in CASES])
def test_grid_search_equals_scikit_learn(name, est, grid):
    X, y = _regression()
    if name == "logistic":
        y = (y > 0.3).astype(np.int64)
    chunks = (60, 100, 91)
    dX, dy = _chunked(X, chunks), _chunked(y, chunks)
    theirs = skms.GridSearchCV(est, grid, cv=skms.KFold(5), return_train_score=True).fit(X, y)
    ours = GridSearchCV(est, grid, cv=KFold(5), iid=False).fit(dX, dy)
    r, s = ours.cv_results_, theirs.cv_results_
    for i in range(5):
        np.testing.assert_array_equal(r["split%d_test_score" % i], s["split%d_test_score" % i])
        np.testing.assert_array_equal(r["split%d_train_score" % i], s["split%d_train_score" % i])
    np.testing.assert_allclose(r["mean_test_score"], s["mean_test_score"], rtol=1e-12)
    np.testing.assert_allclose(r["std_test_score"], s["std_test_score"], rtol=1e-10, atol=1e-15)
    np.testing.assert_array_equal(r["rank_test_score"], s["rank_test_score"])
    assert ours.best_params_ == theirs.best_params_ and ours.best_index_ == theirs.best_index_
    assert ours.n_splits_ == 5 and not ours.multimetric_
    np.testing.assert_array_equal(ours.best_estimator_.coef_, theirs.best_estimator_.coef_)
    np.testing.assert_array_equal(ours.predict(X), theirs.predict(X))
    assert ours.score(X, y) == theirs.score(X, y)
    assert [p for p in r["param_" + next(iter(grid))]] == list(grid[next(iter(grid))])

    iid = GridSearchCV(est, grid, cv=KFold(5)).fit(dX, dy).cv_results_
    split = np.stack([iid["split%d_test_score" % i] for i in range(5)], axis=1)
    w = np.array([51, 50, 50, 50, 50], dtype=np.float64)
    mean = (split * w).sum(1) / w.sum()
    np.testing.assert_allclose(iid["mean_test_score"], mean, rtol=1e-12)
    np.testing.assert_allclose(iid["std_test_score"], np.sqrt((((split - mean[:, None]) ** 2) * w).sum(1) / w.sum()),
                               rtol=1e-10)


def test_grid_search_host_splitters_and_numpy_input():
    X, y = _regression(120)
    yc = (y > 0).astype(np.int64)
    grid = {"C": [0.01, 1.0]}
    for cv in (skms.StratifiedKFold(4), skms.ShuffleSplit(3, random_state=0),
               list(skms.KFold(3, shuffle=True, random_state=1).split(X))):
        theirs = skms.GridSearchCV(LogisticRegression(), grid, cv=cv).fit(X, yc)
        for Xin, yin in ((X, yc), (_chunked(X, (50, 70)), _chunked(yc, (50, 70)))):
            ours = GridSearchCV(LogisticRegression(), grid, cv=cv, iid=False).fit(Xin, yin)
            np.testing.assert_allclose(ours.cv_results_["mean_test_score"], theirs.cv_results_["mean_test_score"],
                                       rtol=1e-12)
    # an integer cv and a classifier: scikit-learn's StratifiedKFold, as there
    ours = GridSearchCV(LogisticRegression(), grid, cv=3, iid=False).fit(X, yc)
    theirs = skms.GridSearchCV(LogisticRegression(), grid, cv=3).fit(X, yc)
    np.testing.assert_array_equal(ours.cv_results_["split0_test_score"], theirs.cv_results_["split0_test_score"])


def test_multimetric_and_refit_false():
    X, y = _regression()
    dX, dy = _chunked(X, (100, 151)), _chunked(y, (100, 151))
    grid = {"alpha": [0.1, 10.0, 1000.0]}
    gs = GridSearchCV(Ridge(), grid, scoring=["r2", "neg_mean_squared_error"], refit="r2", cv=KFold(4)).fit(dX, dy)
    r = gs.cv_results_
    assert gs.multimetric_ and set(gs.scorer_) == {"r2", "neg_mean_squared_error"}
    for key in ("r2", "neg_mean_squared_error"):
        for part in ("split0_test_", "mean_test_", "std_test_", "rank_test_", "split3_train_", "mean_train_"):
            assert part + key in r
    assert "mean_test_score" not in r
    assert gs.best_index_ == int(np.argmax(r["mean_test_r2"]))
    assert gs.best_score_ == r["mean_test_r2"][gs.best_index_]
    assert gs.best_params_ == r["params"][gs.best_index_]
    np.testing.assert_allclose(gs.score(dX, dy), r2_score(y, gs.predict(X)), rtol=1e-12)
    dict_gs = GridSearchCV(Ridge(), grid, scoring={"a": "r2", "b": SCORERS["r2"]}, refit="b", cv=KFold(4)).fit(dX, dy)
    np.testing.assert_array_equal(dict_gs.cv_results_["mean_test_a"], r["mean_test_r2"])

    for refit in (True, "nope"):
        with pytest.raises(ValueError, match="refit must be set to a scorer key"):
            GridSearchCV(Ridge(), grid, scoring=["r2"], refit=refit).fit(dX, dy)
    nor = GridSearchCV(Ridge(), grid, scoring=("r2", "neg_mean_squared_error"), refit=False, cv=KFold(4)).fit(dX, dy)
    np.testing.assert_array_equal(nor.cv_results_["mean_test_r2"], r["mean_test_r2"])
    for attr in ("best_params_", "best_score_", "best_index_", "best_estimator_"):
        with pytest.raises(AttributeError):
            getattr(nor, attr)
    with pytest.raises(NotFittedError):
        nor.predict(dX)


class _FailingRidge(Ridge):
    def fit(self, X, y=None):
        if self.alpha > 50:
            raise RuntimeError("this alpha fails")
        return super().fit(X, y)


def test_error_score():
    X, y = _regression(90)
    dX, dy = _chunked(X, (40, 50)), _chunked(y, (40, 50))
    grid = {"alpha": [1.0, 100.0]}
    with pytest.warns(FitFailedWarning):
        gs = GridSearchCV(_FailingRidge(), grid, cv=KFold(3), error_score=np.nan).fit(dX, dy)
    r = gs.cv_results_
    assert np.isnan(r["split0_test_score"][1]) and np.isnan(r["mean_test_score"][1])
    assert np.isfinite(r["mean_test_score"][0]) and gs.best_index_ == 0
    assert list(r["rank_test_score"]) == [1, 2]
    with pytest.raises(RuntimeError, match="this alpha fails"):
        GridSearchCV(_FailingRidge(), grid, cv=KFold(3)).fit(dX, dy)
    with pytest.raises(ValueError, match="error_score"):
        GridSearchCV(Ridge(), grid, error_score="ignore").fit(dX, dy)


def test_randomized_search_samples_like_parameter_sampler():
    X, y = _regression(100)
    dist = {"alpha": loguniform(1e-3, 1e3), "fit_intercept": [True, False]}
    rs = RandomizedSearchCV(Ridge(), dist, n_iter=7, random_state=3, cv=KFold(3)).fit(_chunked(X, (50, 50)), y)
    assert rs.cv_results_["params"] == list(skms.ParameterSampler(dist, 7, random_state=3))
    assert len(rs.cv_results_["mean_test_score"]) == 7


def test_constructor_validation():
    with pytest.raises(ValueError, match="one-dimensional"):
        GridSearchCV(Ridge(), {"alpha": np.ones((2, 2))})
    with pytest.raises(ValueError, match="sequence"):
        GridSearchCV(Ridge(), {"alpha": 1.0})
    with pytest.raises(ValueError, match="non-empty"):
        GridSearchCV(Ridge(), {"alpha": []})
    X, y = _regression(30)
    with pytest.raises(TypeError, match="n_jobs"):
        GridSearchCV(Ridge(), {"alpha": [1.0]}, n_jobs=1.5).fit(X, y)
    gs = GridSearchCV(Ridge(), {"alpha": [1.0]}, n_jobs=-2, scheduler="sync", cache_cv=False, cv=KFold(3)).fit(X, y)
    assert gs.get_params()["n_jobs"] == -2 and gs.n_splits_ == 3


def test_pipeline_is_one_estimator():
    from sklearn.pipeline import make_pipeline
    from sklearn.preprocessing import StandardScaler

    X, y = _regression(150)
    yc = (y > 0).astype(np.int64)
    pipe = make_pipeline(StandardScaler(), LogisticRegression())
    grid = {"logisticregression__C": [0.01, 1.0]}
    ours = GridSearchCV(pipe, grid, cv=KFold(3), iid=False).fit(_chunked(X, (70, 80)), _chunked(yc, (70, 80)))
    theirs = skms.GridSearchCV(pipe, grid, cv=skms.KFold(3)).fit(X, yc)
    np.testing.assert_array_equal(ours.cv_results_["split1_test_score"], theirs.cv_results_["split1_test_score"])
    np.testing.assert_array_equal(ours.predict_proba(X), theirs.predict_proba(X))
    assert hasattr(ours, "decision_function") and not hasattr(ours, "transform")
