"""PCA / TruncatedSVD without a GPU against the fixtures written by the reference's own pca.py / truncated_svd.py
(tests/golden/ref_decomposition.py), on the float64 numpy checker backend; plus the corner cases the fixtures do not
reach: n_components=0, ties of the sign rule, and finite values whose squares overflow float64."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import decomp_golden as dg  # noqa: E402
from test_decomposition_host import GramOracleBackend  # noqa: E402


@pytest.fixture
def cpu_backend(monkeypatch):
    from dask_ml_b200.cluster import k_means as km

    monkeypatch.setattr(km, "_BACKEND_FACTORY", GramOracleBackend)


@pytest.mark.parametrize("name", dg.CASES)
def test_reference_fixture_replays(cpu_backend, name):
    dg.replay(name)


@pytest.mark.parametrize("i", range(len(dg.ERRORS)))
def test_reference_errors(cpu_backend, i):
    dg.check_error(dg.ERRORS[i])


def test_zero_components(cpu_backend):
    from sklearn import decomposition as skd

    from dask_ml_b200.decomposition import PCA

    rng = np.random.RandomState(0)
    X = rng.standard_normal((300, 5))
    p = PCA(n_components=0, svd_solver="full")
    T = p.fit_transform(X)
    assert T.compute().shape == (300, 0)
    assert p.components_.shape == (0, 5) and p.explained_variance_.shape == (0,) and p.n_components_ == 0
    ref = skd.PCA(n_components=5, svd_solver="full").fit(X)
    np.testing.assert_allclose(p.noise_variance_, ref.explained_variance_.mean(), rtol=1e-12)
    assert p.transform(X[:10]).compute().shape == (10, 0)


def test_sign_rule_ties_take_the_lowest_row(cpu_backend):
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.decomposition import TruncatedSVD

    rng = np.random.RandomState(1)
    X = rng.uniform(-1, 1, size=(900, 4))
    X[[10, 400, 850]] = [5.0, -4.0, 3.0, 2.0]           # equal extremes, in different chunks
    X[[20, 600]] = [-5.0, 4.0, -3.0, -2.0]              # their negation: |t| ties between opposite signs
    t = TruncatedSVD(n_components=2).fit(ChunkedArray.from_array(X, 300))
    U = X @ t.components_.T
    for j in range(2):
        a = np.abs(U[:, j])
        first = int(np.nonzero(a == a.max())[0][0])
        assert U[first, j] > 0


def test_overflowing_values_are_not_reported_as_nan(cpu_backend):
    from dask_ml_b200.decomposition import PCA

    rng = np.random.RandomState(2)
    X = rng.standard_normal((100, 3))
    X[5, 1] = 1e160
    with pytest.raises(ValueError, match="too large for a float64 Gram matrix"):
        PCA(n_components=2).fit(X)
