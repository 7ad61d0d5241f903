"""Replay of the fixtures written by the reference's own pca.py / truncated_svd.py (tests/golden/ref_decomposition.py),
shared by the CPU replay (tests/test_decomposition_golden.py) and the device replay (tests/test_gpu_decomposition_ref.py).

Tolerances are norm-wise: the largest difference over the largest magnitude of the reference array.  Float64 fixtures
replay at 1e-10, signs included (a flipped component differs by 2).  For float32 fixtures the reference itself computes
in float32 (its mean, its centring and its SVD), so it carries float32 rounding, amplified by an offset of 1e4 (the
float32 mean of such data is off by about 1e4 * 2^-24 per column); they replay at 1e-3, signs included.
"""
import json
import os
import re

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def manifest():
    with open(os.path.join(GOLDEN, "REF_DECOMPOSITION_MANIFEST.json")) as f:
        return json.load(f)


CASES = sorted(manifest()["cases"])
ERRORS = manifest()["errors"]


def _np(a):
    return a.compute() if hasattr(a, "compute") else np.asarray(a)


def _close(name, got, want, tol):
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    assert got.shape == want.shape, (name, got.shape, want.shape)
    if want.size == 0:
        return
    err = np.abs(got - want).max() / max(np.abs(want).max(), 1e-300)
    assert err <= tol, "%s: norm-wise error %.3g > %.3g" % (name, err, tol)


def replay(name, to_input=None):
    """Fit / fit_transform / transform / inverse_transform / score_samples / score of this package's estimator on the
    fixture's X (row chunks as in the reference run), compared with what the reference computed."""
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.decomposition import PCA, TruncatedSVD

    meta = manifest()["cases"][name]
    f = np.load(os.path.join(GOLDEN, name + ".npz"))
    X = f["X"]
    tol = 1e-10 if X.dtype == np.float64 else 1e-3
    to_input = to_input or (lambda a, rows: ChunkedArray.from_array(a, rows))
    cls = PCA if meta["estimator"] == "pca" else TruncatedSVD
    est = cls(**meta["params"])
    T = _np(est.fit_transform(to_input(X, int(f["chunks"]))))
    est2 = cls(**meta["params"]).fit(to_input(X, int(f["chunks"])))
    assert est.components_.dtype == X.dtype and T.dtype == X.dtype
    _close("components_", est.components_, f["components"], tol)
    _close("fit components_", est2.components_, f["fit_components"], tol)
    _close("explained_variance_", est.explained_variance_, f["explained_variance"], tol)
    _close("explained_variance_ratio_", est.explained_variance_ratio_, f["explained_variance_ratio"], tol)
    _close("singular_values_", est.singular_values_, f["singular_values"], tol)
    _close("fit_transform", T, f["fit_transform"], tol)
    Xt = X[:300]
    _close("transform", _np(est2.transform(to_input(Xt, 150))), f["transform"], tol)
    _close("inverse_transform", _np(est2.inverse_transform(f["transform"])), f["inverse_transform"], tol)
    if meta["estimator"] == "pca":
        _close("mean_", est.mean_, f["mean"], tol)
        _close("noise_variance_", est.noise_variance_, f["noise_variance"], tol)
        assert est.n_components_ == int(f["n_components_"])
        _close("score_samples", _np(est2.score_samples(to_input(Xt, 150))), f["score_samples"], tol)
        _close("score", est2.score(to_input(Xt, 150)), f["score"], tol)
    return est


def check_error(rec):
    """The reference's exception type and message for the same estimator, parameters and shape."""
    import pytest

    from dask_ml_b200.decomposition import PCA, TruncatedSVD

    rng = np.random.RandomState(9)
    X = rng.standard_normal((rec["n"], rec["d"]))
    cls = PCA if rec["estimator"] == "pca" else TruncatedSVD
    exc = {"ValueError": ValueError, "NotImplementedError": NotImplementedError, "TypeError": TypeError}[rec["error"]]
    msg = rec["message"]
    m = re.match(r"(Invalid solver '.*'\. Must be one of )\{(.*)\}$", msg)
    with pytest.raises(exc) as info:
        cls(**rec["params"]).fit(X)
    got = str(info.value)
    if m:                                     # the solver set prints in hash order: compare its members
        g = re.match(r"(Invalid solver '.*'\. Must be one of )\{(.*)\}$", got)
        assert g and g.group(1) == m.group(1)
        assert sorted(g.group(2).split(", ")) == sorted(m.group(2).split(", "))
    else:
        assert got == msg
