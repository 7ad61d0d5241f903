"""make_classification / make_regression / make_counts on the device (bkm_make_glm_chunk) against the host stream,
chunking invariance, float32 output, the Poisson error flag, and fits that recover the generating models."""
import math

import numpy as np
import pytest
import torch

from dask_ml_b200 import datasets as D

pytestmark = pytest.mark.gpu


def _np(a):
    return np.asarray(a.compute())


def _params(fn, n, d, n_informative, scale, seed):
    rng = np.random.RandomState(seed)
    key = D._draw_key(rng)
    return key, D._informative(rng, d, n_informative, scale)


def _ulps(a, b, dt):
    return np.abs(a.astype(np.float64) - b.astype(np.float64)) / np.spacing(np.abs(b).astype(dt)).astype(np.float64)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_device_matches_host_stream_classification(dtype):
    n, d = 300_000, 13
    Xd, yd = D.make_classification(n, d, n_informative=6, scale=2.0, random_state=7, chunks=70_000, device="cuda",
                                   dtype=dtype)
    Xh, yh = D.make_classification(n, d, n_informative=6, scale=2.0, random_state=7, chunks=70_000, dtype=dtype)
    Xd, yd, Xh, yh = _np(Xd), _np(yd), _np(Xh), _np(yh)
    assert Xd.dtype == dtype and yd.dtype == np.int64
    u = _ulps(Xd, Xh, dtype)
    print("max ulps", u.max(), "share of elements off by one ulp or more", (u >= 1).mean())
    assert u.max() <= (4 if dtype == np.float64 else 1)
    key, info = _params("c", n, d, 6, 2.0, 7)
    z = D._linear(Xh, info, 0)
    w0, w1, _, _ = D._philox4(key, np.arange(n, dtype=np.uint64), 0, D._TAG_RESPONSE)
    margin = np.abs(D._u53(w0, w1) - 1.0 / (1.0 + np.exp(-z)))
    diff = yd != yh
    print("label differences", int(diff.sum()), "rows with margin < 1e-12", int((margin < 1e-12).sum()))
    assert np.all(margin[diff] < 1e-12)
    assert diff.sum() <= 5


def test_device_matches_host_stream_counts():
    n, d = 300_000, 9
    Xd, yd = D.make_counts(n, d, n_informative=4, scale=2.0, chunks=100_000, random_state=3, device="cuda")
    Xh, yh = D.make_counts(n, d, n_informative=4, scale=2.0, chunks=100_000, random_state=3)
    Xd, yd, Xh, yh = _np(Xd), _np(yd), _np(Xh), _np(yh)
    assert _ulps(Xd, Xh, np.float64).max() <= 4
    key, info = _params("p", n, d, 4, 2.0, 3)
    lam = np.exp(D._linear(Xh, info, 0))
    assert (lam >= 10).sum() > 1000 and (lam < 10).sum() > 1000          # both branches run
    _, mg = D._poisson(lam, key, np.arange(n, dtype=np.uint64), margin=True)
    diff = yd != yh
    print("count differences", int(diff.sum()), "rows with margin < 1e-12", int((mg < 1e-12).sum()))
    assert np.all(mg[diff] < 1e-12)
    assert diff.sum() <= 5


def test_device_matches_host_stream_regression():
    n, d = 200_000, 17
    kw = dict(n_informative=6, n_targets=2, bias=0.75, noise=1.5, chunks=50_000, random_state=5, coef=True)
    Xd, yd, cd = D.make_regression(n, d, device="cuda", **kw)
    Xh, yh, ch = D.make_regression(n, d, **kw)
    assert np.array_equal(cd, ch)
    Xd, yd, Xh, yh = _np(Xd), _np(yd), _np(Xh), _np(yh)
    assert _ulps(Xd, Xh, np.float64).max() <= 4
    assert yd.shape == (n, 2) and yd.dtype == np.float64
    scale = np.abs(Xh) @ np.abs(ch) + 0.75 + 1.5 * 8
    assert np.all(np.abs(yd - yh) <= 1e-14 * scale)


@pytest.mark.parametrize("fn", ["make_classification", "make_counts", "make_regression"])
def test_device_chunking_invariance(fn):
    kw = dict(n_features=11, n_informative=4, random_state=2, device="cuda")
    if fn == "make_regression":
        kw.update(noise=0.5)
        chunk_sets = [40_000, ((40_000, 40_000, 20_000), (11,)), ((40_000, 1, 59_999), (11,))]
    else:
        chunk_sets = [40_000, 33_333, 100_000]
    outs = [getattr(D, fn)(100_000, chunks=c, **kw) for c in chunk_sets]
    for X, y in outs[1:]:
        assert torch.equal(torch.cat(list(X.blocks)), torch.cat(list(outs[0][0].blocks)))
        assert torch.equal(torch.cat(list(y.blocks)), torch.cat(list(outs[0][1].blocks)))


def test_float32_z_from_stored_values():
    n, d = 100_000, 10
    X, y, coef = D.make_regression(n, d, n_informative=5, chunks=30_000, random_state=4, coef=True, device="cuda",
                                   dtype=np.float32)
    X, y = _np(X), _np(y)
    assert X.dtype == np.float32
    nz = np.flatnonzero(coef)
    want = np.zeros(n)
    for f in nz:
        want = want + X[:, f].astype(np.float64) * coef[f]
    assert np.array_equal(y, want)


def test_poisson_error_flag_raises_value_error():
    with pytest.raises(ValueError, match="^lam value too large$"):
        D.make_counts(50_000, 10, n_informative=10, scale=1e3, chunks=10_000, random_state=0, device="cuda")
    torch.cuda.synchronize()
    X, y = D.make_counts(1000, 10, chunks=500, random_state=0, device="cuda")      # the device is still usable
    assert _np(y).shape == (1000,)


def test_logistic_regression_recovers_effective_coefficients():
    from dask_ml_b200.linear_model import LogisticRegression

    n, d, k = 2_000_000, 20, 5
    X, y = D.make_classification(n, d, n_informative=k, random_state=11, chunks=1 << 19, device="cuda")
    _, info = _params("c", n, d, k, 1.0, 11)
    eff = np.zeros(d)
    for f, b in info:
        eff[int(f)] += b
    est = LogisticRegression(solver="newton", fit_intercept=False).fit(X, y)
    se = 1.0 / math.sqrt(n * 0.15)                # Fisher information of a unit-variance feature, p(1-p) >= ~0.15
    err = np.abs(np.asarray(est.coef_) - eff)
    print("max |coef - effective beta|", err.max(), "bound", 6 * se)
    assert err.max() < 6 * se


def test_poisson_regression_recovers_effective_coefficients():
    from dask_ml_b200.linear_model import PoissonRegression

    n, d, k = 2_000_000, 12, 4
    X, y = D.make_counts(n, d, n_informative=k, scale=0.5, random_state=12, chunks=1 << 19, device="cuda")
    _, info = _params("p", n, d, k, 0.5, 12)
    eff = np.zeros(d)
    for f, b in info:
        eff[int(f)] += b
    est = PoissonRegression(solver="newton", fit_intercept=False).fit(X, y)
    se = 1.0 / math.sqrt(n * 0.3)                 # E[mu] >= exp(-|z|) ~ 0.3 for these scales
    err = np.abs(np.asarray(est.coef_) - eff)
    print("max |coef - effective beta|", err.max(), "bound", 6 * se)
    assert err.max() < 6 * se


def test_linear_regression_recovers_coef_without_noise():
    from dask_ml_b200.linear_model import LinearRegression

    X, y, coef = D.make_regression(500_000, 30, n_informative=8, bias=3.5, noise=0.0, chunks=1 << 17,
                                   random_state=13, coef=True, device="cuda")
    est = LinearRegression(solver="newton", tol=1e-12).fit(X, y)
    rel = np.abs(np.asarray(est.coef_) - coef).max() / np.abs(coef).max()
    print("relative coef error", rel, "intercept", est.intercept_)
    assert rel < 1e-9
    assert abs(est.intercept_ - 3.5) < 1e-9 * max(1.0, np.abs(coef).max())
