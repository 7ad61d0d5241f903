"""make_classification / make_regression / make_counts on the host (device=None): the reference fixtures of
tests/golden/ref_datasets.py, the host-side draws and quirks, the stream against a scalar restatement, chunking
invariance and the distributions."""
import json
import math
import os

import numpy as np
import pytest
import sklearn.datasets
from scipy import stats

from dask_ml_b200 import datasets as D
from oracle.kmeans_oracle import philox_uniform

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
with open(os.path.join(GOLDEN, "REF_DATASETS_MANIFEST.json")) as f:
    MANIFEST = json.load(f)


def _tuples(v):
    return tuple(_tuples(x) for x in v) if isinstance(v, list) else v


def _kw(kw):
    return {k: _tuples(v) for k, v in kw.items()}


def _np(a):
    return np.asarray(a.compute())


# ---- reference fixtures ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(MANIFEST["coef"]))
def test_coef_bit_identical_to_reference(name):
    g = np.load(os.path.join(GOLDEN, "ref_datasets_%s.npz" % name))
    X, y, coef = D.make_regression(coef=True, **_kw(MANIFEST["coef"][name]["kwargs"]))
    assert np.asarray(coef).dtype == g["coef"].dtype and np.shape(coef) == g["coef"].shape
    assert np.array_equal(np.asarray(coef), g["coef"])
    assert list(X.shape) == list(g["X_shape"]) and list(y.shape) == list(g["y_shape"])


@pytest.mark.parametrize("name", sorted(MANIFEST["coef"]))
def test_key_is_the_references_seed_draw(name):
    """make_regression's key is the first two words of the reference's random_state_data(1, rng) after coef."""
    g = np.load(os.path.join(GOLDEN, "ref_datasets_%s.npz" % name))
    kw = _kw(MANIFEST["coef"][name]["kwargs"])
    rng = np.random.RandomState(kw["random_state"])
    sizes = D._row_chunks(kw.get("chunks"), kw["n_samples"], kw["n_features"])
    skw = {k: v for k, v in kw.items() if k not in ("chunks", "random_state", "n_samples")}
    sklearn.datasets.make_regression(n_samples=sizes[0], coef=True, random_state=rng, **skw)
    w = g["seed_words"].astype(np.uint64)
    assert D._draw_key(rng) == int(w[0] | (w[1] << np.uint64(32)))


@pytest.mark.parametrize("name", sorted(MANIFEST["shapes"]))
def test_shapes_and_dtypes_match_reference(name):
    case = MANIFEST["shapes"][name]
    out = getattr(D, case["function"])(**_kw(case["kwargs"]))
    X, y = out[0], out[1]
    assert list(X.shape) == case["X_shape"] and str(X.dtype) == case["X_dtype"]
    assert list(y.shape) == case["y_shape"] and str(y.dtype) == case["y_dtype"]
    assert _np(X).dtype == np.dtype(case["X_dtype"]) and _np(y).dtype == np.dtype(case["y_dtype"])


@pytest.mark.parametrize("name", sorted(MANIFEST["errors"]))
def test_errors_match_reference(name):
    case = MANIFEST["errors"][name]
    exc = {"ValueError": ValueError, "NotImplementedError": NotImplementedError}[case["type"]]
    with pytest.raises(exc) as e:
        getattr(D, case["function"])(**_kw(case["kwargs"]))
    assert type(e.value) is exc and str(e.value) == case["message"]


# ---- host-side draws and quirks ----------------------------------------------------------------------------------
def test_parameter_draw_order_and_ranges():
    rng = np.random.RandomState(5)
    key = D._draw_key(rng)
    idx = rng.choice(30, 12)
    beta = (rng.random_sample(30) - 1) * 2.5
    rng2 = np.random.RandomState(5)                        # key, then idx, then beta
    assert D._draw_key(rng2) == key
    info = D._informative(rng2, 30, 12, 2.5)
    assert np.array_equal(info[:, 0].astype(int), idx) and np.array_equal(info[:, 1], beta[idx])
    X, y = D.make_classification(64, 30, n_informative=12, scale=2.5, random_state=5, chunks=64)
    assert np.array_equal(_np(y), D._response_host(D._x_block(key, 0, 64, 30, np.float64), D._LOGISTIC, info, key, 0))
    assert len(np.unique(idx)) < len(idx)                     # with replacement: seed 5 repeats an index
    assert np.all(beta >= -2.5) and np.all(beta < 0)


def test_repeated_index_doubles_its_term():
    info = np.array([[3.0, -0.25], [3.0, -0.25], [1.0, -0.5]])
    Xb = D._x_block(77, 0, 50, 5, np.float64)
    z = D._linear(Xb, info, 0)
    assert np.allclose(z, 2 * (-0.25) * Xb[:, 3] - 0.5 * Xb[:, 1], rtol=0, atol=1e-15)


def test_classification_ignores_shape_parameters():
    X0, y0 = D.make_classification(400, 9, n_informative=3, random_state=3, chunks=100)
    X1, y1 = D.make_classification(400, 9, n_informative=3, n_redundant=5, n_repeated=2, n_clusters_per_class=4,
                                   weights=[0.9, 0.1], flip_y=0.5, class_sep=9.0, hypercube=False, shift=3.0,
                                   shuffle=False, random_state=3, chunks=100)
    assert np.array_equal(_np(X0), _np(X1)) and np.array_equal(_np(y0), _np(y1))


@pytest.mark.parametrize("flag", [True, False, 1, "yes"])
def test_coef_returned_only_for_true(flag):
    out = D.make_regression(50, 4, n_informative=2, coef=flag, random_state=0, chunks=25)
    assert len(out) == (3 if flag is True else 2)


def test_n_classes_message_and_dtype_check():
    with pytest.raises(NotImplementedError, match="n_classes != 2"):
        D.make_classification(10, 4, n_classes=1)
    with pytest.raises(ValueError, match="float32 or float64"):
        D.make_counts(10, 4, dtype=np.float16)


# ---- the stream against a scalar restatement ---------------------------------------------------------------------
def _philox_scalar(key, row, j, tag):
    c = [row & 0xFFFFFFFF, row >> 32, j, tag]
    k0, k1 = key & 0xFFFFFFFF, key >> 32
    for _ in range(10):
        p0, p1 = 0xD2511F53 * c[0], 0xCD9E8D57 * c[2]
        c = [(p1 >> 32) ^ c[1] ^ k0, p1 & 0xFFFFFFFF, (p0 >> 32) ^ c[3] ^ k1, p0 & 0xFFFFFFFF]
        k0, k1 = (k0 + 0x9E3779B9) & 0xFFFFFFFF, (k1 + 0xBB67AE85) & 0xFFFFFFFF
    return c


def test_philox_known_answers():
    key = 0x0123456789ABCDEF
    rows = np.array([0, 1, 2 ** 32 + 5, 2 ** 40 + 17], dtype=np.uint64)
    w0, _, _, _ = D._philox4(key, rows, 0, 0)
    assert np.array_equal(w0.astype(np.float64) / 4294967296.0, philox_uniform(key, rows))
    for r in rows.tolist():
        for j, tag in ((0, 0), (7, 0), (3, 1), (2, 2)):
            got = [int(v[0]) for v in D._philox4(key, np.array([r], dtype=np.uint64), j, tag)]
            assert got == _philox_scalar(key, r, j, tag)


def _u53_scalar(a, b):
    return ((a >> 5) * 67108864.0 + (b >> 6)) / 9007199254740992.0


def _normal_scalar(w0, w1):
    u1 = (w0 + 1.0) / 4294967296.0
    u2 = w1 / 4294967296.0
    rad = math.sqrt(-2.0 * math.log(u1))
    return rad * math.cos(2 * math.pi * u2), rad * math.sin(2 * math.pi * u2)


def test_stream_matches_scalar_restatement():
    key, row0, m, d = 987654321987, 1000, 40, 7
    Xb = D._x_block(key, row0, m, d, np.float64)
    for i in range(m):
        for p in range((d + 1) // 2):
            w = _philox_scalar(key, row0 + i, p, 0)
            n0, n1 = _normal_scalar(w[0], w[1])
            assert abs(Xb[i, 2 * p] - n0) <= 1e-13 * max(1.0, abs(n0))
            if 2 * p + 1 < d:
                assert abs(Xb[i, 2 * p + 1] - n1) <= 1e-13 * max(1.0, abs(n1))
    info = np.array([[2.0, -0.7], [5.0, -0.1], [2.0, -0.7]])
    y = D._response_host(Xb, D._LOGISTIC, info, key, row0)
    for i in range(m):
        z = 0.0
        for f, c in info:
            z = z + Xb[i, int(f)] * c
        w = _philox_scalar(key, row0 + i, 0, 1)
        assert y[i] == int(_u53_scalar(w[0], w[1]) < 1.0 / (1.0 + math.exp(-z)))
    yr = D._response_host(Xb, D._NORMAL, info, key, row0, 1, 0.5, 2.0)[:, 0]
    for i in range(m):
        z = 0.0
        for f, c in info:
            z = z + Xb[i, int(f)] * c
        w = _philox_scalar(key, row0 + i, 0, 2)
        assert abs(yr[i] - (z + 0.5 + 2.0 * _normal_scalar(w[0], w[1])[0])) <= 1e-12


def _poisson_scalar(lam, key, row):
    att = 0
    if lam < 10:
        enlam, X, prod = math.exp(-lam), 0, 1.0
        while True:
            w = _philox_scalar(key, row, att, 1)
            att += 1
            prod *= _u53_scalar(w[0], w[1])
            if prod > enlam:
                X += 1
            else:
                return X
    slam, loglam = math.sqrt(lam), math.log(lam)
    b = 0.931 + 2.53 * slam
    a = -0.059 + 0.02483 * b
    invalpha = 1.1239 + 1.1328 / (b - 3.4)
    vr = 0.9277 - 3.6224 / (b - 2)
    while True:
        w = _philox_scalar(key, row, att, 1)
        att += 1
        U = _u53_scalar(w[0], w[1]) - 0.5
        V = _u53_scalar(w[2], w[3])
        us = 0.5 - abs(U)
        k = math.floor((2 * a / us + b) * U + lam + 0.43)
        if us >= 0.07 and V <= vr:
            return k
        if k < 0 or (us < 0.013 and V > us):
            continue
        if math.log(V) + math.log(invalpha) - math.log(a / (us * us) + b) <= -lam + k * loglam - math.lgamma(k + 1):
            return k


def test_poisson_matches_scalar_restatement():
    key = 31337
    lam = np.array([0.0, 1e-3, 0.5, 3.0, 9.99, 10.0, 12.5, 40.0, 300.0, 1e4] * 20)
    rows = np.arange(lam.size, dtype=np.uint64) + np.uint64(2 ** 33)
    y, mg = D._poisson(lam, key, rows, margin=True)
    for i in range(lam.size):
        if mg[i] > 1e-9:
            assert y[i] == _poisson_scalar(lam[i], key, int(rows[i])), (i, lam[i])


def test_loggam_matches_lgamma():
    x = np.arange(1, 400, dtype=np.float64)
    assert np.allclose(D._loggam(x), [math.lgamma(v) for v in x], rtol=1e-13, atol=1e-13)


# ---- chunks invariance ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fn,kw", [
    ("make_classification", dict(n_features=11, n_informative=4)),
    ("make_regression", dict(n_features=6, n_informative=3, n_targets=2, noise=0.3, bias=1.5)),
    ("make_counts", dict(n_features=5, n_informative=3)),
])
def test_chunks_invariance(fn, kw):
    outs = []
    for chunks in (1000, 333, None):
        if fn == "make_counts" and chunks is None:
            chunks = 3000
        outs.append(getattr(D, fn)(3000, random_state=4, chunks=chunks, **kw))
    if fn == "make_regression":       # coef depends on the first block's size, as in the reference: compare same coef
        outs = [getattr(D, fn)(3000, random_state=4, chunks=c, **kw) for c in (1000, ((1000, 1000, 1000), (6,)))]
    for o in outs[1:]:
        assert np.array_equal(_np(o[0]), _np(outs[0][0])) and np.array_equal(_np(o[1]), _np(outs[0][1]))


def test_regression_chunks_change_only_coef():
    X0, y0, c0 = D.make_regression(2000, 8, n_informative=3, random_state=9, chunks=1000, coef=True)
    X1, y1, c1 = D.make_regression(2000, 8, n_informative=3, random_state=9, chunks=500, coef=True)
    assert np.array_equal(c0, c1) or not np.array_equal(_np(y0), _np(y1))


# ---- distributions --------------------------------------------------------------------------------------------------
N = 1_000_000


def test_x_moments():
    X, _ = D.make_counts(N, 4, n_informative=1, chunks=250_000, random_state=0)
    X = _np(X)
    se = 1.0 / math.sqrt(X.size)
    assert abs(X.mean()) < 5 * se
    assert abs(X.var() - 1) < 5 * math.sqrt(2) * se
    assert abs(stats.skew(X.ravel())) < 5 * math.sqrt(6) * se
    assert abs(stats.kurtosis(X.ravel())) < 5 * math.sqrt(24) * se
    assert abs(np.corrcoef(X[:, 0], X[:, 1])[0, 1]) < 5 / math.sqrt(N)


def test_logistic_response_in_bins_of_z():
    X, y = D.make_classification(N, 4, n_informative=3, scale=3.0, random_state=1, chunks=250_000)
    rng = np.random.RandomState(1)
    D._draw_key(rng)
    info = D._informative(rng, 4, 3, 3.0)
    X, y = _np(X), _np(y)
    z = D._linear(X, info, 0)
    p = 1 / (1 + np.exp(-z))
    edges = np.quantile(z, np.linspace(0, 1, 21))
    b = np.clip(np.searchsorted(edges, z, side="right") - 1, 0, 19)
    for k in range(20):
        s = b == k
        se = math.sqrt(max(p[s].mean() * (1 - p[s].mean()), 1e-6) / s.sum())
        assert abs(y[s].mean() - p[s].mean()) < 5 * se, k


def test_poisson_mean_variance_in_bins_and_chi_square():
    lam_grid = np.array([0.3, 2.0, 7.5, 9.9, 10.0, 14.0, 60.0])
    per = 150_000
    lam = np.repeat(lam_grid, per)
    rows = np.arange(lam.size, dtype=np.uint64)
    y = D._poisson(lam, 2024, rows)
    for i, l in enumerate(lam_grid):
        v = y[i * per:(i + 1) * per].astype(np.float64)
        assert abs(v.mean() - l) < 5 * math.sqrt(l / per), l
        assert abs(v.var() - l) < 5 * l * math.sqrt((2 + 1 / l) / per), l
    for i in (0, 1):
        v = y[i * per:(i + 1) * per]
        kmax = int(lam_grid[i] * 4 + 6)
        obs = np.bincount(np.minimum(v, kmax), minlength=kmax + 1)
        pmf = stats.poisson.pmf(np.arange(kmax), lam_grid[i])
        exp = np.append(pmf, 1 - pmf.sum()) * per
        keep = exp > 5
        chi = ((obs[keep] - exp[keep]) ** 2 / exp[keep]).sum() + 0.0
        assert stats.chi2.sf(chi, keep.sum() - 1) > 1e-4


def test_counts_use_exp_of_z():
    X, y = D.make_counts(200_000, 5, n_informative=2, scale=1.0, chunks=100_000, random_state=3)
    rng = np.random.RandomState(3)
    D._draw_key(rng)
    info = D._informative(rng, 5, 2, 1.0)
    lam = np.exp(D._linear(_np(X), info, 0))
    y = _np(y)
    assert y.dtype == np.int64 and y.min() >= 0
    assert abs(y.sum() - lam.sum()) < 5 * math.sqrt(lam.sum())


def test_regression_noise_free_and_noise_std():
    X, y, coef = D.make_regression(N, 5, n_informative=3, bias=1.25, noise=0.0, chunks=300_000, random_state=6,
                                   coef=True)
    X, y = _np(X), _np(y)
    r = y - X @ coef - 1.25
    assert np.abs(r).max() <= 64 * np.finfo(np.float64).eps * (np.abs(X) @ np.abs(coef) + 1.25).max()
    X, y, coef = D.make_regression(N, 5, n_informative=3, bias=0.0, noise=2.5, chunks=300_000, random_state=6,
                                   coef=True)
    r = _np(y) - _np(X) @ coef
    assert abs(r.std() - 2.5) < 5 * 2.5 / math.sqrt(2 * N)
    assert abs(r.mean()) < 5 * 2.5 / math.sqrt(N)


def test_regression_targets_shape_and_float32():
    X, y, coef = D.make_regression(1000, 6, n_informative=4, n_targets=3, chunks=400, random_state=2, coef=True,
                                   dtype=np.float32)
    X, y = _np(X), _np(y)
    assert X.dtype == np.float32 and y.shape == (1000, 3) and y.dtype == np.float64 and coef.shape == (6, 3)
    assert np.allclose(y, X.astype(np.float64) @ coef, rtol=0, atol=1e-10)


def test_overlarge_poisson_rate_raises_numpys_error():
    with pytest.raises(ValueError) as ref:
        np.random.RandomState(0).poisson(np.array([1.0, np.inf]))
    with pytest.raises(ValueError) as e:
        D.make_counts(2000, 10, n_informative=10, scale=1e3, chunks=500, random_state=0)
    assert str(e.value) == str(ref.value) == "lam value too large"
