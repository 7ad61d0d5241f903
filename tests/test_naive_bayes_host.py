"""GaussianNB without a GPU: the estimator's host logic (y handling, the float64 algebra, the reference's quirks,
pickling, 2 ranks over gloo) on a CPU backend whose passes are float64 numpy, against the fixtures written by the
reference's own naive_bayes.py (tests/golden/ref_naive_bayes.py) and live scikit-learn."""
import json
import os
import pickle
import socket
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp
from sklearn.naive_bayes import GaussianNB as SkGaussianNB

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle_backend import OracleBackend  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
with open(os.path.join(GOLDEN, "REF_NAIVE_BAYES_MANIFEST.json")) as _f:
    CASES = sorted(json.load(_f)["cases"])


class NBOracleBackend(OracleBackend):
    """The CPU checker backend plus GaussianNB's passes, in float64 numpy."""

    def class_moments_chunk(self, x, cls, K, sums, counts=None, theta=None, first=False):
        self.launches += 1
        xs = x.to(torch.float64).numpy()
        c = cls.numpy()
        S = np.zeros((K, xs.shape[1]))
        cnt = np.zeros(K)
        for k in range(K):
            rows = xs[c == k]
            if theta is None:
                S[k] = rows.sum(0)
                cnt[k] = len(rows)
            else:
                S[k] = ((rows - theta.numpy()[k]) ** 2).sum(0)
        if first:
            sums.copy_(torch.from_numpy(S))
            if theta is None:
                counts.copy_(torch.from_numpy(cnt))
        else:
            sums += torch.from_numpy(S)
            if theta is None:
                counts += torch.from_numpy(cnt)

    def nb_jll_chunk(self, x, theta, inv_sigma, logc, labels=None, out=None, exp_out=False, n_deferred=None):
        self.launches += 1
        xs = x.to(torch.float64).numpy()
        t, w, c = theta.numpy(), inv_sigma.numpy(), logc.numpy()
        jll = c[None, :] - 0.5 * (((xs[:, None, :] - t[None]) ** 2) * w[None]).sum(2)
        if labels is not None:
            labels.copy_(torch.from_numpy(np.argmax(jll, axis=1).astype(np.int32)))
        if out is not None:
            with np.errstate(invalid="ignore", over="ignore"):
                vmax = jll.max(1)
                lp = jll - (np.log(np.exp(jll - vmax[:, None]).sum(1)) + vmax)[:, None]
            out.copy_(torch.from_numpy(np.exp(lp) if exp_out else lp))


@pytest.fixture
def cpu_backend(monkeypatch):
    from dask_ml_b200.cluster import k_means as km

    monkeypatch.setattr(km, "_BACKEND_FACTORY", NBOracleBackend)


def _np(a):
    return a.compute() if hasattr(a, "compute") else np.asarray(a)


def _data(n=900, d=5, K=3, seed=0, offset=0.0, dtype=np.float64):
    rng = np.random.RandomState(seed)
    means = rng.uniform(-3, 3, size=(K, d)) + offset
    y = rng.randint(0, K, size=n)
    X = means[y] + rng.uniform(0.5, 2.0, size=(K, d))[y] * rng.standard_normal((n, d))
    return X.astype(dtype), y


def _close(name, got, want, rtol):
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    assert got.shape == want.shape, (name, got.shape, want.shape)
    np.testing.assert_array_equal(np.isnan(got), np.isnan(want), err_msg=name)
    ok = ~np.isnan(want)
    if ok.any():
        err = np.abs(got[ok] - want[ok]).max() / max(np.abs(want[ok]).max(), 1e-300)
        assert err <= rtol, "%s: relative error %.3g > %.3g" % (name, err, rtol)


def replay(name, to_input=None, rtol_attr=None, rtol_lp=1e-10):
    """Fit of this package's GaussianNB on the fixture's X and y (row chunks as in the reference run) and its three
    predict methods on X's first rows, compared with what the reference computed."""
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.naive_bayes import GaussianNB

    f = np.load(os.path.join(GOLDEN, name + ".npz"))
    X, y, rows = f["X"], f["y"], int(f["chunks"])
    to_input = to_input or (lambda a, r: ChunkedArray.from_array(a, r))
    f32 = X.dtype == np.float32
    rtol_attr = rtol_attr if rtol_attr is not None else (1e-4 if f32 else 1e-12)
    classes = f["classes"] if "classes" in f.files else None
    est = GaussianNB(classes=classes).fit(to_input(X, rows), ChunkedArray.from_array(y, rows))
    np.testing.assert_array_equal(est.classes_, f["classes_"])
    assert est.theta_.dtype == f["theta"].dtype and est.sigma_.dtype == f["sigma"].dtype
    assert est.class_count_.dtype == np.float64 and est.class_prior_.dtype == np.float64
    _close("theta_", est.theta_, f["theta"], rtol_attr)
    _close("sigma_", est.sigma_, f["sigma"], rtol_attr)
    np.testing.assert_array_equal(est.class_count_, f["class_count"])
    _close("class_prior_", est.class_prior_, f["class_prior"], 1e-15)
    Xp, prow = X[: len(f["predict"])], int(f["predict_chunks"])       # the reference predicted on the first rows
    np.testing.assert_array_equal(_np(est.predict(to_input(Xp, prow))), f["predict"])
    lp_tol = 1e-4 if f32 else rtol_lp
    _close("predict_log_proba", _np(est.predict_log_proba(to_input(Xp, prow))), f["predict_log_proba"], lp_tol)
    _close("predict_proba", _np(est.predict_proba(to_input(Xp, prow))), f["predict_proba"], lp_tol)
    return est


@pytest.mark.parametrize("name", CASES)
def test_fixture_replay(cpu_backend, name):
    replay(name)


def test_manifest_quirks_are_pinned():
    """Every quirk the estimator keeps has a fixture that exhibits it."""
    with open(os.path.join(GOLDEN, "REF_NAIVE_BAYES_MANIFEST.json")) as f:
        m = json.load(f)["cases"]
    c = m["ref_nb_f64_classes"]
    assert c["class_prior_sum"] < 1.0 and c["class_count"][3] == 0.0 and c["nan_theta_classes"] == [3]
    assert c["predict_counts"] == {"9": c["predict_rows"]} and c["nan_log_proba_rows"] == c["predict_rows"]
    q = m["ref_nb_f64_nan_classes"]
    assert q["class_count"][1] == 1.0 and q["predict_counts"] == {"1": q["predict_rows"]}
    assert q["nan_log_proba_rows"] == q["predict_rows"]
    assert m["ref_nb_f32_k4"]["theta_dtype"] == "float32"


@pytest.mark.parametrize("offset", [0.0, 1e4])
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_matches_sklearn(cpu_backend, offset, dtype):
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.naive_bayes import GaussianNB

    X, y = _data(offset=offset, dtype=dtype)
    ref = SkGaussianNB(var_smoothing=0).fit(X.astype(np.float64), y)
    got = GaussianNB().fit(ChunkedArray.from_array(X, 250), y)
    tol = 1e-12 if dtype == np.float64 else 1e-6
    _close("theta_", got.theta_, ref.theta_, tol)
    _close("sigma_", got.sigma_, ref.var_, tol if not offset else tol * 10)
    np.testing.assert_array_equal(got.class_count_, ref.class_count_)
    np.testing.assert_allclose(got.class_prior_, ref.class_prior_, rtol=1e-15)
    np.testing.assert_array_equal(_np(got.predict(X)), ref.predict(X.astype(np.float64)))
    # float32 attributes (as the reference stores them) are what predict uses: theta ~ 1e4 carries ~5e-4 of rounding
    lp_tol = 1e-9 if dtype == np.float64 else (5e-3 if offset else 1e-4)
    _close("log_proba", _np(got.predict_log_proba(X)), ref.predict_log_proba(X.astype(np.float64)), lp_tol)
    _close("proba", _np(got.predict_proba(X)), ref.predict_proba(X.astype(np.float64)), lp_tol)


def test_priors_are_ignored(cpu_backend):
    from dask_ml_b200.naive_bayes import GaussianNB

    X, y = _data()
    a = GaussianNB().fit(X, y)
    b = GaussianNB(priors=[0.9, 0.05, 0.05]).fit(X, y)
    assert b.priors == [0.9, 0.05, 0.05]
    np.testing.assert_array_equal(a.class_prior_, b.class_prior_)
    np.testing.assert_array_equal(_np(a.predict_log_proba(X)), _np(b.predict_log_proba(X)))


def test_classes_subset_and_empty_class(cpu_backend):
    from dask_ml_b200.naive_bayes import GaussianNB

    X, y = _data(K=4)
    est = GaussianNB(classes=[2, 0, 7]).fit(X, y)
    np.testing.assert_array_equal(est.classes_, [2, 0, 7])
    n = len(y)
    np.testing.assert_array_equal(est.class_count_, [(y == 2).sum(), (y == 0).sum(), 0])
    np.testing.assert_allclose(est.class_prior_, est.class_count_ / n, rtol=1e-15)   # rows of 1 and 3 count in n
    np.testing.assert_allclose(est.theta_[0], X[y == 2].mean(0), rtol=1e-12)
    assert np.isnan(est.theta_[2]).all() and np.isnan(est.sigma_[2]).all()
    assert (_np(est.predict(X)) == 7).all()                         # the empty class is NaN on every row: it wins
    assert np.isnan(_np(est.predict_log_proba(X))).all()


def test_zero_variance_class_is_nan_everywhere(cpu_backend):
    from dask_ml_b200.naive_bayes import GaussianNB

    X, y = _data(K=3)
    y = y.copy()
    y[y == 2] = 1
    y[5] = 2                                                        # class 2: one row, zero variance
    est = GaussianNB().fit(X, y)
    assert (est.sigma_[2] == 0).all()
    assert (_np(est.predict(X)) == 2).all()
    assert np.isnan(_np(est.predict_proba(X))).all()


def test_y_forms_and_chunking(cpu_backend):
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.naive_bayes import GaussianNB

    X, y = _data()
    base = GaussianNB().fit(ChunkedArray.from_array(X, 300), y)
    for yy in (torch.as_tensor(y), ChunkedArray.from_array(y, 170), ChunkedArray.from_array(torch.as_tensor(y), 77),
               y.astype(np.float64)):
        est = GaussianNB().fit(ChunkedArray.from_array(X, 300), yy)
        np.testing.assert_allclose(est.theta_, base.theta_, rtol=1e-14)
        np.testing.assert_allclose(est.sigma_, base.sigma_, rtol=1e-14)
        np.testing.assert_array_equal(est.class_count_, base.class_count_)


def test_string_labels(cpu_backend):
    from dask_ml_b200.naive_bayes import GaussianNB

    X, y = _data()
    names = np.array(["cat", "ant", "bee"])[y]
    est = GaussianNB().fit(X, names)
    ref = SkGaussianNB(var_smoothing=0).fit(X, names)
    np.testing.assert_array_equal(est.classes_, ref.classes_)
    _close("theta_", est.theta_, ref.theta_, 1e-12)
    np.testing.assert_array_equal(_np(est.predict(X)), ref.predict(X))


def test_errors(cpu_backend):
    from dask_ml_b200.naive_bayes import GaussianNB

    X, y = _data()
    with pytest.raises(ValueError, match="inconsistent numbers of samples"):
        GaussianNB().fit(X, y[:-1])
    with pytest.raises(ValueError, match="needs the labels"):
        GaussianNB().fit(X)
    from sklearn.exceptions import NotFittedError

    with pytest.raises(NotFittedError):
        GaussianNB().predict(X)


def test_pickle_round_trip(cpu_backend):
    from sklearn.base import clone

    from dask_ml_b200.naive_bayes import GaussianNB

    X, y = _data()
    est = GaussianNB(classes=[0, 1, 2]).fit(X, y)
    back = pickle.loads(pickle.dumps(est))
    for a in ("classes_", "theta_", "sigma_", "class_count_", "class_prior_"):
        np.testing.assert_array_equal(getattr(back, a), getattr(est, a))
    np.testing.assert_array_equal(_np(back.predict_log_proba(X[:40])), _np(est.predict_log_proba(X[:40])))
    assert clone(est).get_params() == {"priors": None, "classes": [0, 1, 2]}


def test_launches_per_fit(cpu_backend):
    from dask_ml_b200.cluster import k_means as km
    from dask_ml_b200.engine import DeviceData
    from dask_ml_b200.naive_bayes import GaussianNB

    X, y = _data()
    be = km._get_backend()
    data = DeviceData([be.to_device(b, torch.float64) for b in (X[:200], X[200:450], X[450:])], be)
    est = GaussianNB().fit(data, y)
    assert be.launch_count() == 6                                    # two moments calls per chunk
    est.predict(data)
    assert be.launch_count() == 9                                    # one predict call per chunk


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


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
        from dask_ml_b200.naive_bayes import GaussianNB
        from test_naive_bayes_host import NBOracleBackend, _data

        km._BACKEND_FACTORY = NBOracleBackend
        X, y = _data(K=4, offset=50.0)
        lo, hi = (0, 170) if rank == 0 else (170, 900)
        yy = y[lo:hi]
        if rank == 0:
            yy = np.where(yy == 3, 0, yy)                            # label 3 only on rank 1: classes_ is the union
            X = X.copy()
            y = y.copy()
            y[lo:hi] = yy
        est = GaussianNB().fit(ChunkedArray.from_array(X[lo:hi], 100), yy)
        np.savez(os.path.join(out_dir, "rank%d.npz" % rank), C=est.classes_, T=est.theta_, S=est.sigma_,
                 N=est.class_count_, P=est.class_prior_, y=y[lo:hi])
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(600)
def test_two_ranks_equal_one_rank(tmp_path, cpu_backend):
    from dask_ml_b200.naive_bayes import GaussianNB

    mp.start_processes(_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True, start_method="spawn")
    r0, r1 = np.load(tmp_path / "rank0.npz"), np.load(tmp_path / "rank1.npz")
    for key in ("C", "T", "S", "N", "P"):
        np.testing.assert_array_equal(r0[key], r1[key])
    X, _ = _data(K=4, offset=50.0)
    y = np.concatenate([r0["y"], r1["y"]])
    one = GaussianNB().fit(X, y)
    np.testing.assert_array_equal(r0["C"], one.classes_)
    np.testing.assert_allclose(r0["T"], one.theta_, rtol=1e-13)
    np.testing.assert_allclose(r0["S"], one.sigma_, rtol=1e-11)
    np.testing.assert_array_equal(r0["N"], one.class_count_)
    np.testing.assert_array_equal(r0["P"], one.class_prior_)
