"""The passes of the linear models on the H100: bkm_glm_pass_chunk in every mode and bkm_gram_weighted_chunk against
float64 numpy, bit-identical repeats, and the estimators against the scikit-learn optima of the CPU suite on resident
and host-resident input."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_glm_host import CASES, _est, _np, _rel, check_large_counts, fit_case, glm_terms, make, sk_ref  # noqa: E402

pytestmark = pytest.mark.gpu

DT = {"f32": torch.float32, "f64": torch.float64, "bf16": torch.bfloat16}


@pytest.fixture(scope="module")
def be():
    from dask_ml_b200.engine import CudaBackend

    return CudaBackend()


def _rows(be, n, d, dt, seed, pitch=None):
    rng = np.random.RandomState(seed)
    X = torch.as_tensor(rng.standard_normal((n, d)))
    if pitch is None:
        x = X.to(device=be.device, dtype=DT[dt]).contiguous()
    else:
        x = torch.zeros((n, pitch), dtype=DT[dt], device=be.device)[:, :d]
        x.copy_(X.to(DT[dt]))
    return x, x.to(torch.float64).cpu().numpy()


def _passes(be, x, y, beta, family):
    n, d = x.shape
    grad = torch.full((d + 2,), 7.0, dtype=torch.float64, device=be.device)
    hrow = torch.full((d + 1,), 7.0, dtype=torch.float64, device=be.device)
    w = torch.empty((n,), dtype=torch.float64, device=be.device)
    G = torch.full((d, d), 7.0, dtype=torch.float64, device=be.device)
    be.glm_pass_chunk(x, y, beta, family, 1, grad=grad, hrow=hrow, w=w, first=True)
    be.gram_weighted_chunk(x, w, G, first=True)
    g0 = torch.empty_like(grad)
    be.glm_pass_chunk(x, y, beta, family, 0, grad=g0, first=True)
    mu = torch.empty((n,), dtype=torch.float64, device=be.device)
    lab = torch.empty((n,), dtype=torch.uint8, device=be.device)
    be.glm_pass_chunk(x, None, beta, family, 2, out=mu)
    be.glm_pass_chunk(x, None, beta, family, 3, out=lab)
    torch.cuda.synchronize()
    return [t.cpu().numpy() for t in (grad, hrow, w, G, g0, mu, lab)]


def _check(be, x, xs, family, scale, seed=1):
    n, d = xs.shape
    rng = np.random.RandomState(seed)
    b = rng.standard_normal(d + 1) * scale / np.sqrt(d)
    y = {0: (rng.uniform(size=n) < 0.5) * 1.0, 1: rng.standard_normal(n), 2: rng.poisson(2.0, n) * 1.0}[family]
    yd = torch.as_tensor(y).to(be.device)
    bd = torch.as_tensor(b).to(be.device)
    got = _passes(be, x, yd, bd, family)
    eta = xs @ b[:-1] + b[-1]
    mu, loss, r, w = glm_terms(family, eta, y)
    want = [np.concatenate([r @ xs, [r.sum(), loss.sum()]]), np.concatenate([w @ xs, [w.sum()]]), w,
            (xs * w[:, None]).T @ xs]
    xm = np.abs(xs).max() if n else 0.0
    scale_of = [np.abs(r).sum() * xm + np.abs(loss).sum(), np.abs(w).sum() * max(1.0, xm),
                np.abs(w).max(initial=0.0), (np.abs(w) @ (xs * xs)).max(initial=0.0)]
    for name, gv, wv, sc in zip(("grad", "hrow", "w", "gram"), got[:4], want, scale_of):
        assert gv.shape == wv.shape, name
        if n:
            assert np.abs(gv - wv).max() <= 1e-12 * max(sc, 1.0), (name, np.abs(gv - wv).max(), sc)
        else:
            assert not gv.any(), name
    np.testing.assert_array_equal(got[4], got[0])                    # gradient mode = the gradient half of Newton
    if n:                                                              # eta's sum order differs from numpy's
        np.testing.assert_allclose(got[5], mu, rtol=1e-12, atol=1e-14 * (np.abs(xs).sum(1).max() + 1))
    np.testing.assert_array_equal(got[6].astype(bool), got[5] > 0.5)
    again = _passes(be, x, yd, bd, family)
    for a, b2 in zip(got, again):
        np.testing.assert_array_equal(a, b2)                           # bit-identical repeat


@pytest.mark.parametrize("dt", ["f32", "f64", "bf16"])
@pytest.mark.parametrize("d", [1, 13, 64, 65, 128, 300])
@pytest.mark.parametrize("family", [0, 1, 2])
def test_passes_against_numpy(be, dt, d, family):
    for n in (0, 1, 33, 4099):
        x, xs = _rows(be, n, d, dt, seed=d + n)
        _check(be, x, xs, family, scale=1.0)


@pytest.mark.parametrize("dt", ["f32", "bf16"])
def test_million_rows_and_unaligned_pitch(be, dt):
    x, xs = _rows(be, 1 << 20, 64, dt, seed=3)
    _check(be, x, xs, 0, scale=1.0)
    x, xs = _rows(be, 1000, 13, dt, seed=4, pitch=17)                 # rows not 16-byte aligned
    assert x.stride(0) == 17
    for family in (0, 1, 2):
        _check(be, x, xs, family, scale=1.0)


def test_large_eta(be):
    """|eta| up to 800: the logistic loss and mu stay finite; exp overflows to +inf for the Poisson family."""
    n, d = 257, 4
    rng = np.random.RandomState(5)
    xs = rng.uniform(-1, 1, (n, d))
    xs[:, 0] = np.linspace(-1, 1, n)
    x = torch.as_tensor(xs).to(be.device)
    _check(be, x, xs, 0, scale=1.0)
    b = np.array([800.0, 0, 0, 0, 0])
    bd = torch.as_tensor(b).to(be.device)
    y = torch.as_tensor((rng.uniform(size=n) < 0.5) * 1.0).to(be.device)
    grad, hrow, w, G, g0, mu, lab = _passes(be, x, y, bd, 0)
    eta = xs @ b[:-1]
    mw, lw, rw, ww = glm_terms(0, eta, y.cpu().numpy())
    assert np.isfinite(grad).all() and np.isfinite(G).all()
    np.testing.assert_allclose(grad[-1], lw.sum(), rtol=1e-13)
    np.testing.assert_allclose(mu, mw, rtol=1e-13, atol=1e-300)
    grad, hrow, w, G, g0, mu, lab = _passes(be, x, y, bd, 2)
    assert grad[-1] == np.inf and (mu[eta > 709.8] == np.inf).all() and np.isfinite(mu[eta < 709]).all()


@pytest.mark.parametrize("family,penalty,solver", CASES)
@pytest.mark.parametrize("resident", [True, False])
def test_estimators_match_sklearn(family, penalty, solver, resident):
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.engine import host_resident

    X, y = make(family)
    Xin = ChunkedArray.from_array(X, 250) if resident else host_resident(X, block_rows=128)
    est = fit_case(family, penalty, solver, Xin, ChunkedArray.from_array(y, 111))
    beta = np.append(est.coef_, est.intercept_)
    assert _rel(beta, sk_ref(family, penalty, 0.7, X, y)) < 1e-6
    p = est.predict(Xin)
    assert all(b.is_cuda for b in p.blocks)
    eta = X @ est.coef_ + est.intercept_
    if family == "logistic":
        np.testing.assert_allclose(_np(est.predict_proba(Xin)), 1 / (1 + np.exp(-eta)), rtol=1e-12)
        np.testing.assert_array_equal(_np(p), 1 / (1 + np.exp(-eta)) > 0.5)
    else:
        np.testing.assert_allclose(_np(p), eta if family == "normal" else np.exp(eta), rtol=1e-11, atol=1e-12)


@pytest.mark.parametrize("mean", [200, 2000])
@pytest.mark.parametrize("solver", ["admm", "newton"])
@pytest.mark.parametrize("resident", [True, False])
def test_poisson_large_counts(mean, solver, resident):
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.engine import host_resident

    check_large_counts(mean, solver, (lambda a: ChunkedArray.from_array(a, 250)) if resident
                       else (lambda a: host_resident(a, block_rows=128)))


def test_fp32_fit_and_launches(be):
    from dask_ml_b200 import _lib

    X, y = make("logistic", n=5000, d=20)
    lib = _lib.load()
    c0 = lib.bkm_launch_count()
    est = _est("logistic", solver="newton", tol=0.0, max_iter=3).fit(
        __import__("dask_ml_b200").ChunkedArray.from_array(X.astype(np.float32), 2000), y)
    assert lib.bkm_launch_count() - c0 == (3 + 1) * 3 * 2           # the pass at beta = 0, then one per iteration
    ref = _est("logistic", solver="newton", tol=0.0, max_iter=3).fit(X.astype(np.float32).astype(np.float64), y)
    np.testing.assert_allclose(est.coef_, ref.coef_, rtol=1e-10)
