"""SimpleImputer on the device, against scikit-learn 1.9's SimpleImputer on the same (float32-widened for bf16) numpy
data: median and most_frequent statistics_ bit-equal, constant equal, the mean within a bound on its float64 summation
error, the transform and the inverse bit-equal to scikit-learn's run with the device's statistics_; for every dtype,
chunking, missing value and resident / host-resident input.  Also the contention and all-distinct extremes of the mode
pass, a forced column group boundary, the invalid-input errors, the input left unmodified, the output feeding
StandardScaler and KMeans, and two GPUs against one."""
import os
import socket
import sys
import warnings

import numpy as np
import pytest
import sklearn.impute
import torch
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from test_impute_host import CASES, STRATS, assert_stats, data, replay  # noqa: E402

DTYPES = {"f32": torch.float32, "f64": torch.float64, "bf16": torch.bfloat16}


def _inputs(n, dt, missing, seed=0):
    X = data(seed, n=n, missing=missing)
    X[:, 3] = np.arange(n)[::-1] * 0.25 - 7           # all distinct: the tie goes to the minimum
    if missing == 0:
        X[::7, 5] = -0.0
    t = torch.as_tensor(X).to(DTYPES[dt])
    return t, (t.float() if dt == "bf16" else t).numpy()


def _as_input(t, chunks, resident):
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.engine import host_resident

    rows = t.shape[0] if chunks == "whole" else chunks
    if resident:
        return ChunkedArray([t[i:i + rows].cuda() for i in range(0, t.shape[0], rows)])
    return host_resident(ChunkedArray([t[i:i + rows] for i in range(0, t.shape[0], rows)]), block_rows=rows)


def sk(Xh, **params):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return sklearn.impute.SimpleImputer(**params).fit(Xh)


def mean_bound_ok(got, Xh, missing):
    """|got - mu| <= 8 2^-52 (|mu| + sum |x - s| / m) per column, mu the exact mean (math.fsum) of the m non-missing
    values and s the statistics pass's shift."""
    import math

    from dask_ml_b200.decomposition.pca import SHIFT_ROWS

    v = Xh.astype(np.float64)
    miss = np.isnan(v) if np.isnan(missing) else v == missing
    head = v[:SHIFT_ROWS]
    ok = np.isfinite(head) & ~miss[:SHIFT_ROWS]
    s = np.where(ok, head, 0).sum(0) / np.maximum(ok.sum(0), 1)
    for j in range(v.shape[1]):
        col = v[~miss[:, j], j]
        if len(col) == 0:
            assert np.isnan(got[j])
            continue
        mu = math.fsum(col) / len(col)
        bound = 8 * 2.0 ** -52 * (abs(mu) + np.abs(col - s[j]).sum() / len(col))
        assert abs(got[j] - mu) <= bound, (j, got[j], mu, bound)


@pytest.mark.parametrize("dt", ["f32", "f64", "bf16"])
@pytest.mark.parametrize("chunks", ["whole", 777, 2048])
@pytest.mark.parametrize("missing", [np.nan, -1.0, 0])
@pytest.mark.parametrize("resident", [True, False])
def test_matches_scikit_learn(dt, chunks, missing, resident):
    from dask_ml_b200.impute import SimpleImputer

    t, Xh = _inputs(5000, dt, missing)
    keep = t.clone()
    src = _as_input(t, chunks, resident)
    before = [b.clone() for b in src.blocks] if resident else None
    for strategy in STRATS:
        params = dict(strategy=strategy, missing_values=missing, add_indicator=True)
        want = sk(Xh, **params)
        est = SimpleImputer(**params).fit(src)
        if strategy == "mean":
            assert est.statistics_.dtype == want.statistics_.dtype
            mean_bound_ok(est.statistics_, Xh, missing)
        else:
            assert_stats(est.statistics_, want.statistics_)
        np.testing.assert_array_equal(est.indicator_.features_, want.indicator_.features_)
        want.statistics_ = est.statistics_.copy()
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            out = est.transform(src)
            want_t = want.transform(Xh)
        assert all(b.is_cuda and b.dtype == (torch.float64 if dt == "f64" else torch.float32) for b in out.blocks)
        got = out.compute()
        np.testing.assert_array_equal(got, want_t.astype(Xh.dtype))
        np.testing.assert_array_equal(est.inverse_transform(out).compute(),
                                      want.inverse_transform(want_t).astype(Xh.dtype))
    torch.testing.assert_close(t, keep, rtol=0, atol=0, equal_nan=True)          # the input is not modified
    if resident:                                                                  # nor are the device blocks passed in
        for b, b0 in zip(src.blocks, before):
            assert b.is_cuda
            torch.testing.assert_close(b, b0, rtol=0, atol=0, equal_nan=True)


@pytest.mark.parametrize("dt", ["f32", "f64", "bf16"])
@pytest.mark.parametrize("missing", [np.nan, -1.0])
def test_signed_zeros_are_one_value(dt, missing):
    """-0.0 and +0.0 count as one value of the mode (+0.0): 3 + 3 zeros outnumber 4 ones."""
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.impute import SimpleImputer

    col = np.array([0.0, -0.0, 1.0, 0.0, -0.0, 1.0, 0.0, -0.0, 1.0, 1.0, missing, 2.0])
    X = np.stack([col, col[::-1]], axis=1)
    t = torch.as_tensor(X).to(DTYPES[dt])
    Xh = (t.float() if dt == "bf16" else t).numpy()
    est = SimpleImputer(strategy="most_frequent", missing_values=missing).fit(ChunkedArray([t[:5].cuda(), t[5:].cuda()]))
    assert_stats(est.statistics_, sk(Xh, strategy="most_frequent", missing_values=missing).statistics_)
    assert (est.statistics_ == 0).all() and not np.signbit(est.statistics_).any()


@pytest.mark.parametrize("name", CASES)
@pytest.mark.parametrize("resident", [True, False])
def test_fixture_replay(name, resident):
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.engine import host_resident

    if resident:
        replay(name)
    else:
        replay(name, to_input=lambda a, r: host_resident(ChunkedArray.from_array(a, r), block_rows=r))


@pytest.mark.parametrize("dt", ["f32", "f64", "bf16"])
def test_mode_extremes_and_groups(dt, monkeypatch):
    from dask_ml_b200 import impute

    n = 200000
    rng = np.random.RandomState(7)
    X = np.empty((n, 5))
    X[:, 0] = np.where(rng.uniform(size=n) < 0.97, 3.0, rng.randint(0, 16, n))     # one value: contention
    X[:, 1] = rng.permutation(n) - 1000.5                                           # all distinct
    X[:, 2] = rng.randint(0, 16, n)                                                 # 16 categories
    X[:, 3] = np.nan                                                                # all missing
    X[:, 4] = np.repeat([1.0, 2.0], n // 2)                                         # an exact tie
    X[rng.uniform(size=(n, 5)) < 0.1] = np.nan
    t = torch.as_tensor(X).to(DTYPES[dt])
    Xh = (t.float() if dt == "bf16" else t).numpy()
    want = sk(Xh, strategy="most_frequent").statistics_
    C = _as_input(t, 65536, True)
    assert_stats(impute.SimpleImputer(strategy="most_frequent").fit(C).statistics_, want)
    monkeypatch.setattr(impute, "MODE_BUDGET", 1)                   # one column per group
    assert_stats(impute.SimpleImputer(strategy="most_frequent").fit(C).statistics_, want)
    assert_stats(impute.SimpleImputer(strategy="median").fit(C).statistics_, sk(Xh, strategy="median").statistics_)


def test_invalid_input_errors():
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.impute import SimpleImputer

    t, Xh = _inputs(3000, "f32", -1.0)
    bad = Xh.copy()
    bad[100, 1] = np.inf
    for est in (SimpleImputer(), SimpleImputer(missing_values=-1)):
        with pytest.raises(ValueError) as info:
            est.fit(ChunkedArray.from_array(bad, 1000))
        assert "Input X contains infinity" in str(info.value)
    nan = Xh.copy()
    nan[5, 0] = np.nan
    with pytest.raises(ValueError, match="Input X contains NaN"):
        SimpleImputer(missing_values=-1).fit(ChunkedArray.from_array(nan, 1000))
    est = SimpleImputer(missing_values=-1, strategy="median").fit(ChunkedArray.from_array(Xh, 1000))
    with pytest.raises(ValueError, match="Input X contains NaN"):
        est.transform(ChunkedArray.from_array(nan, 1000))
    with pytest.raises(ValueError, match="Input X contains infinity"):
        est.transform(ChunkedArray.from_array(bad, 1000))


def test_output_feeds_scaler_and_kmeans():
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.cluster import KMeans
    from dask_ml_b200.impute import SimpleImputer
    from dask_ml_b200.preprocessing import StandardScaler

    rng = np.random.RandomState(3)
    cent = rng.uniform(-10, 10, size=(8, 30))
    X = (cent[rng.randint(0, 8, 60000)] + rng.standard_normal((60000, 30))).astype(np.float32)
    X[rng.uniform(size=X.shape) < 0.05] = np.nan
    X0 = X.copy()
    imp = SimpleImputer(strategy="median")
    Z = imp.fit_transform(ChunkedArray.from_array(X, 25000))
    Zh = sk(X, strategy="median").transform(X)
    np.testing.assert_array_equal(Z.compute(), Zh)
    S = StandardScaler().fit_transform(Z)
    Sh = StandardScaler().fit_transform(ChunkedArray.from_array(Zh, 25000))
    np.testing.assert_array_equal(S.compute(), Sh.compute())
    init = Sh.compute()[:8].copy()
    a = KMeans(n_clusters=8, init=init, max_iter=20, tol=0.0).fit(S)
    b = KMeans(n_clusters=8, init=init, max_iter=20, tol=0.0).fit(Sh)
    np.testing.assert_array_equal(a.cluster_centers_, b.cluster_centers_)
    np.testing.assert_array_equal(X, X0)


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _data():
    X = data(9, n=40000).astype(np.float32)
    X[:, 0] = np.round(X[:, 0] * 4) / 4
    return X


def _worker(rank, world, port, out_dir):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    import torch.distributed as dist

    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world)
    try:
        from dask_ml_b200 import ChunkedArray
        from dask_ml_b200.impute import SimpleImputer

        X = _data()
        lo, hi = (0, 9000) if rank == 0 else (9000, 40000)
        res = {s: np.asarray(SimpleImputer(strategy=s).fit(ChunkedArray.from_array(X[lo:hi], 6000)).statistics_,
                             dtype=np.float64) for s in STRATS}
        np.savez(os.path.join(out_dir, "rank%d.npz" % rank), **res)
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpus_equal_one(tmp_path):
    from dask_ml_b200.impute import SimpleImputer

    mp.start_processes(_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True, start_method="spawn")
    r0, r1 = np.load(tmp_path / "rank0.npz"), np.load(tmp_path / "rank1.npz")
    for s in STRATS:
        np.testing.assert_array_equal(r0[s], r1[s])
        want = np.asarray(SimpleImputer(strategy=s).fit(_data()).statistics_, dtype=np.float64)
        if s == "mean":
            np.testing.assert_allclose(r0[s], want, rtol=1e-12)
        else:
            np.testing.assert_array_equal(r0[s], want)
