"""The linear models without a GPU: the estimators' host logic (solvers, the reference's quirks, y handling, pickling,
2 ranks over gloo) on a CPU backend whose two passes are float64 numpy, against live scikit-learn fits of the same
objective on [X, 1] with fit_intercept=False (so the intercept is penalised, as in the reference)."""
import os
import pickle
import socket
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp
from sklearn import linear_model as sk

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle_backend import OracleBackend  # noqa: E402


def glm_terms(family, eta, y):
    """(mu, loss, r, w) per row, the definition of DESIGN.md A22."""
    if family == 0:
        mu = np.where(eta >= 0, 1.0 / (1.0 + np.exp(-np.abs(eta))), np.exp(-np.abs(eta)) / (1.0 + np.exp(-np.abs(eta))))
        return mu, np.maximum(eta, 0) + np.log1p(np.exp(-np.abs(eta))) - y * eta, mu - y, mu * (1 - mu)
    if family == 1:
        return eta, (y - eta) ** 2, 2.0 * (eta - y), np.full_like(eta, 2.0)
    with np.errstate(over="ignore"):
        mu = np.exp(eta)
    return mu, mu - y * eta, mu - y, mu


class GLMOracleBackend(OracleBackend):
    """The CPU checker backend plus the two passes of the linear models, in float64 numpy."""

    def glm_pass_chunk(self, x, y, beta, family, mode, grad=None, hrow=None, w=None, out=None, first=False):
        self.launches += 1
        xs = x.to(torch.float64).numpy()
        b = beta.numpy()
        eta = xs @ b[:-1] + b[-1]
        mu, loss, r, ww = glm_terms(family, eta, y.numpy() if y is not None else np.zeros_like(eta))
        if mode >= 2:
            out.copy_(torch.from_numpy(mu if mode == 2 else (mu > 0.5).astype(np.uint8)))
            return
        g = np.concatenate([r @ xs, [r.sum(), loss.sum()]])
        grad.copy_(torch.from_numpy(g)) if first else grad.add_(torch.from_numpy(g))
        if mode == 1:
            w.copy_(torch.from_numpy(ww))
            h = np.concatenate([ww @ xs, [ww.sum()]])
            hrow.copy_(torch.from_numpy(h)) if first else hrow.add_(torch.from_numpy(h))

    def gram_weighted_chunk(self, x, w, gram, first=False):
        self.launches += 1
        xs = x.to(torch.float64).numpy()
        G = torch.from_numpy((xs * w.numpy()[:, None]).T @ xs)
        gram.copy_(G) if first else gram.add_(G)


@pytest.fixture
def cpu_backend(monkeypatch):
    from dask_ml_b200.cluster import k_means as km

    monkeypatch.setattr(km, "_BACKEND_FACTORY", GLMOracleBackend)


def _np(a):
    return a.compute() if hasattr(a, "compute") else np.asarray(a)


def make(family, n=600, d=5, seed=0):
    rng = np.random.RandomState(seed)
    X = rng.standard_normal((n, d))
    beta = rng.uniform(-0.6, 0.6, d)
    eta = X @ beta + 0.3
    if family == "logistic":
        y = (rng.uniform(size=n) < 1 / (1 + np.exp(-eta))).astype(np.float64)
    elif family == "normal":
        y = eta + 0.5 * rng.standard_normal(n)
    else:
        y = rng.poisson(np.exp(eta)).astype(np.float64)
    return X, y


def _ones(X):
    return np.hstack([X, np.ones((len(X), 1))])


def sk_ref(family, penalty, C, X, y):
    """scikit-learn's optimum of the same objective, beta = [coef, intercept] of a fit on [X, 1]."""
    Xo, n = _ones(X), len(X)
    if family == "logistic":
        if penalty is None:
            m = sk.LogisticRegression(penalty=None, fit_intercept=False, tol=1e-12, max_iter=10000)
        elif penalty == "l2":
            m = sk.LogisticRegression(C=C, fit_intercept=False, tol=1e-12, max_iter=10000)
        else:
            m = sk.LogisticRegression(penalty="l1", C=C, solver="liblinear", fit_intercept=False, tol=1e-12,
                                      max_iter=100000)
        return m.fit(Xo, y).coef_.ravel()
    if family == "normal":
        if penalty is None:
            return sk.LinearRegression(fit_intercept=False).fit(Xo, y).coef_
        if penalty == "l2":
            return sk.Ridge(alpha=1 / (2 * C), fit_intercept=False, solver="cholesky").fit(Xo, y).coef_
        return sk.Lasso(alpha=1 / (2 * n * C), fit_intercept=False, tol=1e-14, max_iter=100000).fit(Xo, y).coef_
    assert penalty != "l1"
    alpha = 0.0 if penalty is None else 1 / (n * C)
    return sk.PoissonRegressor(alpha=alpha, fit_intercept=False, solver="newton-cholesky", tol=1e-14,
                               max_iter=1000).fit(Xo, y).coef_


EST = {"logistic": "LogisticRegression", "normal": "LinearRegression", "poisson": "PoissonRegression"}
CASES = [(f, p, s) for f in EST for (p, s) in
         [("l2", "admm"), ("l2", "lbfgs"), ("l1", "proximal_grad"), (None, "newton"), (None, "gradient_descent")]
         if not (f == "poisson" and p == "l1")]


def _est(family, **kw):
    from dask_ml_b200 import linear_model

    return getattr(linear_model, EST[family])(**kw)


def _rel(got, want):
    return np.abs(got - want).max() / np.abs(want).max()


def fit_case(family, penalty, solver, X, y, C=0.7):
    tight = {"newton": 1e-12, "admm": 1e-12, "lbfgs": 1e-12, "proximal_grad": 1e-13, "gradient_descent": 1e-15}
    kw = {"factr": 10.0} if solver == "lbfgs" else None
    return _est(family, penalty=penalty or "l2", solver=solver, C=C, tol=tight[solver], max_iter=20000,
                solver_kwargs=kw).fit(X, y)


@pytest.mark.parametrize("family,penalty,solver", CASES)
def test_optimum_matches_sklearn(cpu_backend, family, penalty, solver):
    X, y = make(family)
    est = fit_case(family, penalty, solver, X, y)
    beta = np.append(est.coef_, est.intercept_)
    assert _rel(beta, sk_ref(family, penalty, 0.7, X, y)) < 1e-6


def counts(mean, n=600, d=5, seed=0):
    """Poisson counts of the given mean: the intercept's optimum is near log(mean), far from the start at 0."""
    rng = np.random.RandomState(seed)
    X = rng.standard_normal((n, d))
    return X, rng.poisson(np.exp(X @ rng.uniform(-0.3, 0.3, d) + np.log(mean))).astype(np.float64)


def check_large_counts(mean, solver, to_input=lambda a: a):
    """The default PoissonRegression (tol 1e-4, max_iter 100) on counts of a large mean: a full Newton step from 0
    overshoots the intercept to about mean - 1 (exp(eta) overflows from mean ~ 710), so the step must be damped."""
    from dask_ml_b200.linear_model import PoissonRegression

    X, y = counts(mean)
    est = PoissonRegression(solver=solver).fit(to_input(X), y)
    beta = np.append(est.coef_, est.intercept_)
    assert _rel(beta, sk_ref("poisson", "l2" if solver == "admm" else None, 1.0, X, y)) < 1e-6
    np.testing.assert_allclose(_np(est.predict(to_input(X))), np.exp(X @ est.coef_ + est.intercept_), rtol=1e-11)


@pytest.mark.parametrize("mean", [200, 2000])
@pytest.mark.parametrize("solver", ["admm", "newton"])
def test_poisson_large_counts(cpu_backend, mean, solver):
    check_large_counts(mean, solver)


@pytest.mark.parametrize("family", ["logistic", "normal", "poisson"])
def test_l1_kkt(cpu_backend, family):
    """At the l1 optimum |dL/dbeta_j| <= lambda where beta_j = 0 and dL/dbeta_j = -lambda sign(beta_j) elsewhere."""
    X, y = make(family, d=8)
    C = 0.02 if family != "normal" else 0.002
    est = _est(family, penalty="l1", solver="proximal_grad", C=C, tol=1e-14, max_iter=50000).fit(X, y)
    beta = np.append(est.coef_, est.intercept_)
    lam = 1 / C
    eta = _ones(X) @ beta
    _, _, r, _ = glm_terms({"logistic": 0, "normal": 1, "poisson": 2}[family], eta, y)
    g = _ones(X).T @ r
    zero = beta == 0
    assert zero.any() and (~zero).any()
    assert (np.abs(g[zero]) <= lam * (1 + 1e-9)).all()
    np.testing.assert_allclose(g[~zero], -lam * np.sign(beta[~zero]), rtol=1e-6, atol=1e-6 * lam)


def test_reference_defaults_and_ignored_params():
    from dask_ml_b200.linear_model import LinearRegression

    p = LinearRegression().get_params()
    assert {k: p[k] for k in ("penalty", "tol", "C", "fit_intercept", "solver", "max_iter", "solver_kwargs")} == {
        "penalty": "l2", "tol": 1e-4, "C": 1.0, "fit_intercept": True, "solver": "admm", "max_iter": 100,
        "solver_kwargs": None}
    for k in ("dual", "intercept_scaling", "class_weight", "random_state", "multiclass", "verbose", "warm_start",
              "n_jobs"):
        assert k in p


def test_attributes_and_quirks(cpu_backend):
    X, y = make("logistic")
    est = _est("logistic").fit(X, y)
    assert est.coef_.shape == (5,) and est.coef_.dtype == np.float64 and type(est.intercept_) is float
    p = _np(est.predict(X))
    assert p.dtype == np.bool_                                        # predict_proba(X) > 0.5, a bool array
    proba = _np(est.predict_proba(X))
    assert proba.shape == (600,) and proba.dtype == np.float64
    np.testing.assert_array_equal(p, proba > 0.5)
    assert est.score(X, y) == pytest.approx(np.mean(y == p), abs=0)  # accuracy

    no = _est("logistic", fit_intercept=False).fit(X, y)
    assert not hasattr(no, "intercept_") and no.coef_.shape == (5,)
    np.testing.assert_allclose(_np(no.predict_proba(X)), 1 / (1 + np.exp(-(X @ no.coef_))), rtol=1e-12)

    Xn, yn = make("normal")
    lr = _est("normal").fit(Xn, yn)
    pred = _np(lr.predict(Xn))
    np.testing.assert_allclose(pred, Xn @ lr.coef_ + lr.intercept_, rtol=1e-12)
    assert lr.score(Xn, yn) == pytest.approx(np.mean((yn - pred) ** 2), rel=1e-12)   # the MSE, not R^2

    Xp, yp = make("poisson")
    pr = _est("poisson").fit(Xp, yp)
    mu = _np(pr.predict(Xp))
    np.testing.assert_allclose(mu, np.exp(Xp @ pr.coef_ + pr.intercept_), rtol=1e-12)
    assert (yp == 0).any()
    with np.errstate(divide="ignore", invalid="ignore"):
        t = np.where(yp > 0, yp * np.log(yp / mu), 0.0)
    assert pr.get_deviance(Xp, yp) == pytest.approx(2 * np.sum(t - (yp - mu)), rel=1e-12)


def test_solver_and_penalty_errors(cpu_backend):
    X, y = make("normal")
    with pytest.raises(ValueError, match="^'solver' must be "):
        _est("normal", solver="sag").fit(X, y)
    with pytest.raises(ValueError, match="'penalty' must be"):
        _est("normal", penalty="elastic_net").fit(X, y)
    _est("normal", penalty="elastic_net", solver="newton").fit(X, y)   # newton drops the regulariser
    with pytest.raises(ValueError, match="inconsistent numbers of samples"):
        _est("normal").fit(X, y[:-1])
    with pytest.raises(ValueError, match="needs the labels"):
        _est("normal").fit(X)
    from sklearn.exceptions import NotFittedError

    with pytest.raises(NotFittedError):
        _est("normal").predict(X)


def test_lamduh_from_solver_kwargs(cpu_backend):
    X, y = make("normal")
    a = _est("normal", C=0.25, tol=1e-12).fit(X, y)
    b = _est("normal", C=1.0, tol=1e-12, solver_kwargs={"lamduh": 4.0}).fit(X, y)
    np.testing.assert_allclose(a.coef_, b.coef_, rtol=1e-12)


def test_nonfinite_input(cpu_backend):
    from dask_ml_b200 import ChunkedArray

    X, y = make("logistic")
    Xb = X.copy()
    Xb[407, 2] = np.nan
    with pytest.raises(ValueError, match="NaN, infinity"):
        _est("logistic").fit(ChunkedArray.from_array(torch.as_tensor(Xb), 200), y)
    yb = y.copy()
    yb[3] = np.inf
    with pytest.raises(ValueError, match="NaN, infinity"):
        _est("logistic", solver="lbfgs").fit(X, yb)


def test_separable_logistic_stays_finite(cpu_backend):
    X, _ = make("logistic")
    y = (X[:, 0] > 0).astype(np.float64)
    for solver in ("newton", "gradient_descent"):
        est = _est("logistic", solver=solver, max_iter=30).fit(X, y)
        assert np.isfinite(est.coef_).all() and np.isfinite(est.intercept_)
        assert np.abs(est.coef_[0]) > 10 * np.abs(est.coef_[1:]).max()
    assert est.score(X, y) > 0.99


def test_y_forms_and_chunking(cpu_backend):
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.engine import host_resident
    from dask_ml_b200.cluster import k_means as km

    X, y = make("poisson")
    base = _est("poisson", tol=1e-12).fit(ChunkedArray.from_array(X, 250), y)
    forms = [torch.as_tensor(y), ChunkedArray.from_array(y, 170), ChunkedArray.from_array(torch.as_tensor(y), 77),
             y.astype(np.int64)]
    for yy in forms:
        est = _est("poisson", tol=1e-12).fit(ChunkedArray.from_array(X, 250), yy)
        np.testing.assert_allclose(est.coef_, base.coef_, rtol=1e-12)
    hr = host_resident(ChunkedArray.from_array(X, 250), backend=km._get_backend(), block_rows=64)
    est = _est("poisson", tol=1e-12).fit(hr, ChunkedArray.from_array(y, 33))
    np.testing.assert_allclose(est.coef_, base.coef_, rtol=1e-12)
    np.testing.assert_allclose(np.concatenate([_np(b) for b in est.predict(hr).blocks]), _np(base.predict(X)),
                               rtol=1e-12)


def test_pickle_round_trip(cpu_backend):
    from sklearn.base import clone

    X, y = make("logistic")
    est = _est("logistic", C=2.0).fit(X, y)
    back = pickle.loads(pickle.dumps(est))
    np.testing.assert_array_equal(back.coef_, est.coef_)
    assert back.intercept_ == est.intercept_
    np.testing.assert_array_equal(_np(back.predict_proba(X)), _np(est.predict_proba(X)))
    assert clone(est).get_params()["C"] == 2.0


def test_launches_per_iteration(cpu_backend):
    from dask_ml_b200.cluster import k_means as km
    from dask_ml_b200.engine import DeviceData

    X, y = make("logistic")
    be = km._get_backend()
    data = DeviceData([be.to_device(b, torch.float64) for b in (X[:200], X[200:450], X[450:])], be)
    _est("logistic", solver="newton", tol=0.0, max_iter=4).fit(data, y)
    # the Newton pass at beta = 0, then one per iteration (no step is halved here): two launches per chunk each
    assert be.launch_count() == (4 + 1) * 3 * 2
    before = be.launch_count()
    _est("logistic", solver="lbfgs", max_iter=3).fit(data, y)
    assert (be.launch_count() - before) % 3 == 0                      # one launch per chunk per evaluation
    est = _est("logistic", solver="newton", max_iter=2).fit(data, y)
    before = be.launch_count()
    est.predict(data)
    assert be.launch_count() - before == 3


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


SHARDS = [(0, 170), (170, 170), (170, 600)]                           # rank 1 holds no rows


def _worker(rank, world, port, out_dir):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    import torch.distributed as dist

    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from dask_ml_b200 import ChunkedArray
        from dask_ml_b200.cluster import k_means as km
        from dask_ml_b200.engine import DeviceData
        from test_glm_host import GLMOracleBackend, _est, make

        km._BACKEND_FACTORY = GLMOracleBackend
        lo, hi = SHARDS[rank]
        res = {}
        for family, solver in (("logistic", "admm"), ("poisson", "lbfgs"), ("normal", "proximal_grad")):
            X, y = make(family)
            be = km._get_backend()
            Xs = ChunkedArray.from_array(X[lo:hi], 100) if hi > lo else DeviceData([be.to_device(X[:0], torch.float64)], be)
            est = _est(family, solver=solver, penalty="l1" if solver == "proximal_grad" else "l2", tol=1e-12,
                       max_iter=5000).fit(Xs, y[lo:hi])
            res[family] = np.append(est.coef_, est.intercept_)
        np.savez(os.path.join(out_dir, "rank%d.npz" % rank), **res)
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(600)
def test_three_ranks_equal_one_rank(tmp_path, cpu_backend):
    mp.start_processes(_worker, args=(3, _free_port(), str(tmp_path)), nprocs=3, join=True, start_method="spawn")
    r = [np.load(tmp_path / ("rank%d.npz" % k)) for k in range(3)]
    for family, solver in (("logistic", "admm"), ("poisson", "lbfgs"), ("normal", "proximal_grad")):
        for k in (1, 2):
            np.testing.assert_array_equal(r[0][family], r[k][family])
        X, y = make(family)
        one = _est(family, solver=solver, penalty="l1" if solver == "proximal_grad" else "l2", tol=1e-12,
                   max_iter=5000).fit(X, y)
        np.testing.assert_allclose(r[0][family], np.append(one.coef_, one.intercept_), rtol=1e-7)
