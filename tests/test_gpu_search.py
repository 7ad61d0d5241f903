"""KFold and the searches on device blocks: shuffled pieces against the numpy restatement bit for bit, materialised
folds against numpy indexing, unshuffled folds as launch-free views, per-split scores bit-identical to a hand-written
loop over the same folds, agreement with scikit-learn's GridSearchCV driving the same estimator on numpy, and a search
that never copies a block to the host."""
import numpy as np
import pytest
import sklearn.model_selection as skms
import torch
from scipy.stats import loguniform

from dask_ml_b200 import ChunkedArray, chunked
from dask_ml_b200.datasets import make_classification, make_regression
from dask_ml_b200.linear_model import LinearRegression, LogisticRegression
from dask_ml_b200.metrics import SCORERS
from dask_ml_b200.model_selection import GridSearchCV, KFold, RandomizedSearchCV
from dask_ml_b200.model_selection._search import _splits
from dask_ml_b200.model_selection._split import _take, permutation_indices
from dask_ml_b200.naive_bayes import GaussianNB

pytestmark = pytest.mark.gpu

CHUNKS = (30_000, 30_000, 17_001)


@pytest.fixture(scope="module")
def be():
    from dask_ml_b200.engine import CudaBackend

    return CudaBackend()


def _device(a, chunks=CHUNKS, dtype=None):
    t = torch.as_tensor(a).cuda()
    return ChunkedArray.from_array(t if dtype is None else t.to(dtype), (tuple(chunks),))


def _classification(dtype):
    X, y = make_classification(sum(CHUNKS), 16, chunks=CHUNKS[0], device="cuda", dtype=dtype, random_state=0)
    return ChunkedArray.from_array(torch.cat(X.blocks), (CHUNKS,)), ChunkedArray.from_array(torch.cat(y.blocks),
                                                                                            (CHUNKS,))


def _windows(n, k):
    sizes = [n // k + (1 if f < n % k else 0) for f in range(k)]
    starts = np.cumsum([0] + sizes)
    return list(zip(starts[:-1], starts[1:]))


def _hand_folds(a, k):
    """Fold f of a row-chunked array, restated: per block, the rows before the window, in it, after it, as views."""
    offsets = np.cumsum((0,) + a.chunks[0])
    out = []
    for t0, t1 in _windows(len(a), k):
        train, test = [], []
        for b, lo, hi in zip(a.blocks, offsets[:-1], offsets[1:]):
            s, e = min(max(t0, lo), hi) - lo, max(min(t1, hi), lo) - lo
            train += [b[:s]] if s > 0 else []
            test += [b[s:e]] if e > s else []
            train += [b[max(e, s):]] if max(e, s) < hi - lo else []
        out.append((ChunkedArray(train), ChunkedArray(test)))
    return out


def _hand_scores(est, candidates, X, y, k, scorer):
    """(n_splits, n_candidates) test scores of a hand-written loop over the same fold views."""
    out = np.zeros((k, len(candidates)))
    for s, ((X_tr, X_te), (y_tr, y_te)) in enumerate(zip(_hand_folds(X, k), _hand_folds(y, k))):
        for c, p in enumerate(candidates):
            fitted = type(est)(**{**est.get_params(), **p}).fit(X_tr, y_tr)
            out[s, c] = scorer(fitted, X_te, y_te)
    return out


def _split_scores(search, k):
    return np.stack([search.cv_results_["split%d_test_score" % i] for i in range(k)])


# ---- KFold on device blocks ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64, torch.bfloat16, torch.int64],
                         ids=lambda t: str(t).split(".")[-1])
def test_device_kfold_equals_host_restatement_and_numpy_indexing(be, dtype):
    rng = np.random.RandomState(0)
    n = sum(CHUNKS)
    Xh = (rng.standard_normal((n, 13)) * 100).astype(np.float64)
    yh = rng.randint(0, 5, size=n)
    X, y = _device(Xh, dtype=dtype), _device(yh)
    Xn = X.compute() if dtype != torch.bfloat16 else torch.cat(X.blocks).float().cpu().numpy()
    host = list(KFold(4, shuffle=True, random_state=9).split(ChunkedArray.from_array(np.zeros(n), (CHUNKS,))))
    for (tr, te), (htr, hte) in zip(KFold(4, shuffle=True, random_state=9).split(X), host):
        for idx, hidx in ((tr, htr), (te, hte)):
            assert all(b.is_cuda and b.dtype == torch.int64 for b in idx.blocks)
            assert idx.chunks == hidx.chunks
            np.testing.assert_array_equal(idx.compute(), hidx.compute())
            rows = idx.compute()
            got = _take(X, idx)
            assert all(b.is_cuda and b.dtype == dtype for b in got.blocks)
            want = Xn[rows]
            got = got.compute() if dtype != torch.bfloat16 else torch.cat(got.blocks).float().cpu().numpy()
            np.testing.assert_array_equal(got, want)
            np.testing.assert_array_equal(_take(y, idx).compute(), yh[rows])
    # the first test piece is offset + pi_seed(p) over its positions
    seed = np.random.RandomState(9).randint(0, 2 ** 32 - 1, size=len(CHUNKS), dtype="u8")[0]
    te = next(KFold(4, shuffle=True, random_state=9).split(X))[1]
    np.testing.assert_array_equal(te.blocks[0].cpu().numpy(), permutation_indices(seed, CHUNKS[0], np.arange(19_251)))


def test_unshuffled_folds_are_views_and_launch_nothing(be):
    X, y = _classification("float32")
    ptrs = [(b.data_ptr(), b.data_ptr() + b.numel() * b.element_size()) for b in X.blocks]
    before = be.launch_count()
    folds = list(_splits(KFold(5), X, y, None))
    assert be.launch_count() == before
    for parts, (tr, te) in zip(folds, _hand_folds(X, 5)):
        X_tr, y_tr, X_te, y_te = parts
        for b in X_tr.blocks + X_te.blocks:
            assert b.is_cuda and any(lo <= b.data_ptr() < hi for lo, hi in ptrs)
        assert torch.equal(torch.cat(X_tr.blocks), torch.cat(tr.blocks))
        assert torch.equal(torch.cat(X_te.blocks), torch.cat(te.blocks))
        assert X_tr.chunks[0] == y_tr.chunks[0] and X_te.chunks[0] == y_te.chunks[0]


# ---- searches ------------------------------------------------------------------------------------------------------
CS = [0.001, 0.1, 10.0]


@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_grid_search_equals_the_hand_loop_and_scikit_learn(dtype):
    X, y = _classification(dtype)
    est = LogisticRegression(solver="lbfgs")
    gs = GridSearchCV(est, {"C": CS}, cv=5).fit(X, y)
    candidates = [{"C": c} for c in CS]
    hand = _hand_scores(est, candidates, X, y, 5, lambda e, a, b: e.score(a, b))
    np.testing.assert_array_equal(_split_scores(gs, 5), hand)
    assert gs.best_params_ == candidates[gs.best_index_]
    assert all(b.is_cuda for b in gs.predict(X).blocks)

    theirs = skms.GridSearchCV(est, {"C": CS}, cv=skms.KFold(5)).fit(X.compute(), y.compute())
    np.testing.assert_allclose(_split_scores(gs, 5), np.stack([theirs.cv_results_["split%d_test_score" % i]
                                                               for i in range(5)]), atol=2e-3)
    refit = LogisticRegression(solver="lbfgs", **gs.best_params_).fit(X.compute(), y.compute())
    np.testing.assert_allclose(gs.best_estimator_.coef_, refit.coef_, rtol=1e-2, atol=1e-3)


@pytest.mark.parametrize("scoring", ["r2", "neg_mean_squared_error"])
def test_linear_regression_search(scoring):
    X, y = make_regression(sum(CHUNKS), 12, noise=5.0, chunks=CHUNKS[0], device="cuda", dtype="float64",
                           random_state=1)
    X, y = [ChunkedArray.from_array(torch.cat(a.blocks), (CHUNKS,)) for a in (X, y)]
    grid = {"fit_intercept": [True, False]}
    gs = GridSearchCV(LinearRegression(), grid, scoring=scoring, cv=4).fit(X, y)
    hand = _hand_scores(LinearRegression(), [{"fit_intercept": True}, {"fit_intercept": False}], X, y, 4,
                        SCORERS[scoring])
    np.testing.assert_array_equal(_split_scores(gs, 4), hand)
    if scoring == "r2":
        assert 0.5 < gs.best_score_ <= 1.0


@pytest.mark.parametrize("scoring", ["accuracy", "neg_log_loss"])
def test_gaussian_nb_search(scoring):
    X, y = _classification("float32")
    grid = {"classes": [None, [0, 1]]}
    gs = GridSearchCV(GaussianNB(), grid, scoring=scoring, cv=3).fit(X, y)
    hand = _hand_scores(GaussianNB(), [{"classes": None}, {"classes": [0, 1]}], X, y, 3, SCORERS[scoring])
    np.testing.assert_array_equal(_split_scores(gs, 3), hand)
    assert all(b.is_cuda for b in gs.predict_proba(X).blocks)


def test_pipeline_search():
    from sklearn.pipeline import make_pipeline

    from dask_ml_b200.preprocessing import StandardScaler

    X, y = _classification("float32")
    pipe = make_pipeline(StandardScaler(), LogisticRegression(solver="lbfgs"))
    gs = GridSearchCV(pipe, {"logisticregression__C": [0.01, 1.0]}, cv=3).fit(X, y)
    hand = np.zeros((3, 2))
    for s, ((X_tr, X_te), (y_tr, y_te)) in enumerate(zip(_hand_folds(X, 3), _hand_folds(y, 3))):
        for c, C in enumerate([0.01, 1.0]):
            p = make_pipeline(StandardScaler(), LogisticRegression(solver="lbfgs", C=C)).fit(X_tr, y_tr)
            hand[s, c] = p.score(X_te, y_te)
    np.testing.assert_array_equal(_split_scores(gs, 3), hand)
    assert all(b.is_cuda for b in gs.predict(X).blocks)


def test_randomized_search_and_shuffled_kfold():
    X, y = _classification("float32")
    dist = {"C": loguniform(1e-3, 1e2)}
    rs = RandomizedSearchCV(LogisticRegression(solver="lbfgs"), dist, n_iter=3, random_state=0,
                            cv=KFold(3, shuffle=True, random_state=2)).fit(X, y)
    candidates = list(skms.ParameterSampler(dist, 3, random_state=0))
    assert rs.cv_results_["params"] == candidates
    # the hand loop gathers the same pieces with torch indexing
    hand = np.zeros((3, 3))
    offsets = np.cumsum((0,) + CHUNKS)
    for s, (tr, te) in enumerate(KFold(3, shuffle=True, random_state=2).split(X)):
        def rows(a, idx):
            out = []
            for ix in idx.blocks:
                k = int(np.searchsorted(offsets, int(ix[0]), side="right")) - 1
                out.append(a.blocks[k][ix - int(offsets[k])])
            return ChunkedArray(out)

        for c, p in enumerate(candidates):
            fitted = LogisticRegression(solver="lbfgs", **p).fit(rows(X, tr), rows(y, tr))
            hand[s, c] = fitted.score(rows(X, te), rows(y, te))
    np.testing.assert_array_equal(_split_scores(rs, 3), hand)


def test_search_stays_on_the_device(monkeypatch):
    X, y = _classification("float32")
    seen = []

    class Watched(LogisticRegression):
        def fit(self, X, y=None):
            seen.extend([X, y])
            return super().fit(X, y)

        def predict(self, X):
            out = super().predict(X)
            seen.append(out)
            return out

    def refuse(*args, **kwargs):
        raise AssertionError("a block was copied to the host")

    with monkeypatch.context() as m:
        m.setattr(ChunkedArray, "compute", refuse)
        m.setattr(chunked, "block_to_numpy", refuse)
        gs = GridSearchCV(Watched(solver="lbfgs"), {"C": [0.1, 1.0]}, scoring="accuracy", cv=4).fit(X, y)
        outs = [gs.predict(X), gs.predict_proba(X)]
    assert len(seen) > 2 * 4 * 2
    for a in seen + outs:
        assert all(b.is_cuda for b in a.blocks)
    assert np.isfinite(gs.best_score_)
