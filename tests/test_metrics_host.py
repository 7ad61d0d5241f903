"""The scoring metrics on host blocks against scikit-learn on the same arrays, the rules kept from the reference
(dask_ml/metrics/classification.py, regression.py) and the one deviation of log_loss.  No GPU."""
import numpy as np
import pytest
import sklearn.metrics as skm
import torch

from dask_ml_b200 import ChunkedArray
from dask_ml_b200.metrics import accuracy_score, log_loss, mean_absolute_error, mean_squared_error, r2_score

RTOL = 1e-12


def _chunk(a, sizes):
    return ChunkedArray.from_array(a, (tuple(sizes),))


def _rng(seed=0):
    return np.random.RandomState(seed)


# ---- accuracy ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["int", "bool", "float"])
@pytest.mark.parametrize("weighted", [False, True])
def test_accuracy_matches_sklearn(kind, weighted):
    rng = _rng(1)
    n = 1000
    t = rng.randint(0, 3 if kind != "bool" else 2, size=n)
    p = np.where(rng.rand(n) < 0.7, t, rng.randint(0, 3 if kind != "bool" else 2, size=n))
    t, p = {"int": (t, p), "bool": (t.astype(bool), p.astype(bool)), "float": (t.astype(float), p.astype(np.float32))}[kind]
    w = rng.rand(n) if weighted else None
    sizes = [400, 350, 250]
    got = accuracy_score(_chunk(t, sizes), _chunk(p, sizes), sample_weight=None if w is None else _chunk(w, sizes))
    np.testing.assert_allclose(got, skm.accuracy_score(t, p, sample_weight=w), rtol=RTOL)
    cnt = accuracy_score(_chunk(t, sizes), _chunk(p, sizes), normalize=False,
                         sample_weight=None if w is None else _chunk(w, sizes))            # M4
    np.testing.assert_allclose(cnt, skm.accuracy_score(t, p, normalize=False, sample_weight=w), rtol=RTOL)
    if w is None:
        assert isinstance(cnt, int)


def test_accuracy_multilabel_rows_and_differently_chunked_inputs():
    rng = _rng(2)
    t = rng.randint(0, 2, size=(500, 3))
    p = np.where(rng.rand(500, 3) < 0.8, t, 1 - t)
    got = accuracy_score(_chunk(t, [200, 300]), _chunk(p, [100, 100, 300]))
    np.testing.assert_allclose(got, skm.accuracy_score(t, p), rtol=RTOL)
    assert accuracy_score(t, torch.as_tensor(p)) == got
    with pytest.raises(ValueError, match="inconsistent numbers of samples"):
        accuracy_score(t, p[:-1])


# ---- log loss ------------------------------------------------------------------------------------------------------------------
def _clip_log_loss(t, P, w=None, eps=1e-15, normalize=True):
    """clip, renormalise, log: the statement of log_loss with its ``eps``, which scikit-learn no longer takes."""
    P = np.clip(P.astype(np.float64), eps, 1 - eps)
    if P.ndim == 1:
        P = np.column_stack([1 - P, P])
    P = P / P.sum(1, keepdims=True)
    cls = np.searchsorted(np.unique(t), t)
    w = np.ones(len(t)) if w is None else w
    loss = -(w * np.log(P[np.arange(len(t)), cls])).sum()
    return loss / w.sum() if normalize else loss


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("shape", ["binary_1d", "binary_2d", "multiclass"])
def test_log_loss_matches_sklearn(shape, weighted):
    rng = _rng(3)
    n, K = 900, 2 if shape != "multiclass" else 4
    P = np.clip(rng.dirichlet(np.ones(K), size=n), 1e-12, None)
    P = P / P.sum(1, keepdims=True)
    labels = np.array([-3, 5]) if K == 2 else np.array([1.0, 2.0, 7.0, 9.0])
    t = labels[rng.randint(0, K, size=n)]
    t[:K] = labels
    w = rng.rand(n) + 0.1 if weighted else None
    pred = P[:, 1] if shape == "binary_1d" else P
    sizes = [100, 500, 300]
    got = log_loss(_chunk(t, sizes), _chunk(pred, sizes), sample_weight=None if w is None else _chunk(w, sizes))
    np.testing.assert_allclose(got, skm.log_loss(t, pred, sample_weight=w), rtol=RTOL)
    tot = log_loss(_chunk(t, sizes), _chunk(pred, sizes), normalize=False,
                   sample_weight=None if w is None else _chunk(w, sizes))
    np.testing.assert_allclose(tot, skm.log_loss(t, pred, normalize=False, sample_weight=w), rtol=RTOL)


def test_log_loss_clips_with_its_own_eps():
    t = np.array([0, 1, 1, 0, 1])
    p = np.array([0.0, 1.0, 0.0, 1.0, 0.3])
    np.testing.assert_allclose(log_loss(t, p), _clip_log_loss(t, p), rtol=RTOL)
    np.testing.assert_allclose(log_loss(t, p, eps=1e-3), _clip_log_loss(t, p, eps=1e-3), rtol=RTOL)
    P = np.array([[0.0, 1.0, 0.0], [0.2, 0.3, 0.5], [1.0, 0.0, 0.0]])
    np.testing.assert_allclose(log_loss(np.array([0, 2, 1]), P), _clip_log_loss(np.array([0, 2, 1]), P), rtol=RTOL)


def test_log_loss_is_the_global_mean_over_unequal_blocks():
    """The deviation from the reference: unequal blocks, one of which sees a single class, give scikit-learn's value on
    the whole array (the reference would average the block losses unweighted, and raise on the one-class block)."""
    rng = _rng(4)
    t = np.r_[np.zeros(50, int), rng.randint(0, 2, size=450)]
    p = np.clip(rng.rand(500), 1e-6, 1 - 1e-6)
    got = log_loss(_chunk(t, [50, 150, 300]), _chunk(p, [50, 150, 300]))
    np.testing.assert_allclose(got, skm.log_loss(t, p), rtol=RTOL)


def test_log_loss_labels_and_errors():
    p = np.array([0.2, 0.4, 0.9])
    with pytest.raises(ValueError, match="only one label"):
        log_loss(np.array([1, 1, 1]), p)
    np.testing.assert_allclose(log_loss(np.array([1, 1, 1]), p, labels=[0, 1]),
                               skm.log_loss(np.array([1, 1, 1]), p, labels=[0, 1]), rtol=RTOL)
    with pytest.raises(ValueError, match="different number of classes"):
        log_loss(np.array([0, 1, 2]), p)
    assert np.isnan(log_loss(np.array([0, 1, 7]), p, labels=[0, 1]))


# ---- regression ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("m", [None, 1, 3])
@pytest.mark.parametrize("dtype", ["float64", "float32"])
def test_regression_metrics_match_sklearn(m, dtype):
    rng = _rng(5)
    n = 1200
    shape = (n,) if m is None else (n, m)
    t = (rng.standard_normal(shape) * 3 + 10).astype(dtype)
    p = (t + rng.standard_normal(shape)).astype(dtype)
    sizes = [500, 500, 200]
    T, P = _chunk(t, sizes), _chunk(p, sizes)
    t64, p64 = t.astype(np.float64), p.astype(np.float64)
    np.testing.assert_allclose(mean_squared_error(T, P), skm.mean_squared_error(t64, p64), rtol=RTOL)
    np.testing.assert_allclose(mean_absolute_error(T, P), skm.mean_absolute_error(t64, p64), rtol=RTOL)
    np.testing.assert_allclose(r2_score(T, P), skm.r2_score(t64, p64), rtol=1e-11)
    raw = mean_squared_error(T, P, multioutput="raw_values")
    assert isinstance(raw, np.ndarray) and raw.shape == (1 if m is None else m,)
    np.testing.assert_allclose(raw, np.atleast_1d(skm.mean_squared_error(t64, p64, multioutput="raw_values")), rtol=RTOL)
    np.testing.assert_allclose(mean_absolute_error(T, P, multioutput="raw_values"),
                               np.atleast_1d(skm.mean_absolute_error(t64, p64, multioutput="raw_values")), rtol=RTOL)


def test_r2_of_offset_targets_keeps_its_digits():
    rng = _rng(6)
    t = 1e8 + rng.standard_normal(5000)
    p = t + 0.1 * rng.standard_normal(5000)
    np.testing.assert_allclose(r2_score(_chunk(t, [3000, 2000]), _chunk(p, [3000, 2000])), skm.r2_score(t, p),
                               rtol=1e-9)


def test_rules_kept_from_the_reference():
    t, p = np.arange(10.0), np.arange(10.0) + 1
    for fn in (mean_squared_error, mean_absolute_error, r2_score):                          # M1
        with pytest.raises(ValueError, match="'sample_weight' is not supported."):
            fn(t, p, sample_weight=np.ones(10))
    with pytest.raises(NotImplementedError, match="'multioutput' must be 'uniform_average'"):   # M2
        r2_score(t, p, multioutput="raw_values")
    for fn in (mean_squared_error, mean_absolute_error):
        with pytest.raises(ValueError, match="Weighted 'multioutput' not supported."):
            fn(t, p, multioutput=[0.5, 0.5])
    const = np.full((10, 2), 4.0)                                                          # M3
    assert r2_score(const, const) == 1.0
    assert r2_score(const, const + 1) == 0.0
    half = np.column_stack([np.full(10, 4.0), np.arange(10.0)])
    assert r2_score(half, half) == 1.0
    assert r2_score(half, half + np.array([1.0, 0.0])) == 0.5
    assert np.isnan(mean_squared_error(np.array([1.0, np.nan]), np.array([1.0, 2.0])))
