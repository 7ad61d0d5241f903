"""QuantileTransformer on the device: the fixture replay (resident and host-resident input), quantiles_ bit-equal to
np.percentile for every dtype, chunking and number of quantiles, the transform pass bit-identical to the numpy
restatement for the uniform distribution and within NORMAL_TOL of scipy for the normal one, both staging paths of the
transform, the input untouched, the output feeding KMeans, and two GPUs against one."""
import os
import socket
import sys
import warnings

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from test_quantile_host import CASES, replay, transform_restated  # noqa: E402

DTYPES = {"f32": torch.float32, "f64": torch.float64, "bf16": torch.bfloat16}
# The normal distribution's ppf / cdf are CUDA's normcdfinv / normcdf, scipy's ndtri / ndtr on the host.  An output
# may differ from scipy's by NORMAL_TOL units of 2^-52 times (|y| + 1 + s), where s is the column's largest
# interpolation slope: the inverse interpolates the cdf value, so an error in it grows by the slope.
NORMAL_TOL = 64


def normal_error(got, want, quantiles, references):
    """The largest |got - want| over each column's scale 2^-52 (|want| + 1 + slope); NaN / inf patterns equal."""
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    np.testing.assert_array_equal(np.isnan(got), np.isnan(want))
    fin = np.isfinite(want)
    np.testing.assert_array_equal(got[~fin & ~np.isnan(want)], want[~fin & ~np.isnan(want)])
    with np.errstate(all="ignore"):
        slope = np.diff(quantiles, axis=0) / np.diff(references)[:, None] if len(references) > 1 else \
            np.zeros((1, quantiles.shape[1]))
    slope = np.nan_to_num(np.where(np.isfinite(slope), np.abs(slope), 0.0)).max(0)
    scale = 2.0 ** -52 * (np.abs(np.where(fin, want, 0.0)) + 1.0 + slope[None, :])
    err = np.where(fin, np.abs(np.where(fin, got - want, 0.0)) / scale, 0.0)
    return float(err.max()) if err.size else 0.0


def _compare_normal(key, got, want, est):
    e = normal_error(got, want, est.quantiles_, est.references_)
    assert e <= NORMAL_TOL, (key, e)


@pytest.mark.parametrize("name", CASES)
@pytest.mark.parametrize("resident", [True, False])
def test_fixture_replay(name, resident):
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.engine import host_resident

    if resident:
        replay(name, compare_normal=_compare_normal)
    else:
        replay(name, to_input=lambda a, r: host_resident(ChunkedArray.from_array(a, r), block_rows=333),
               compare_normal=_compare_normal)


def _column_data(n, d, seed, dt, infinite=True):
    rng = np.random.RandomState(seed)
    X = rng.standard_normal((n, d)) * rng.uniform(0.5, 3.0, d)
    X[:, 0] = rng.randint(-3, 4, n)                               # duplicates, and -0.0 next to +0.0
    X[rng.randint(0, n, n // 10), 0] = -0.0
    if d > 2 and infinite:
        X[rng.randint(0, n, 5), 2] = np.inf
        X[rng.randint(0, n, 5), 2] = -np.inf
    if d > 3:
        X[:, 3] = 7.25                                            # constant
    t = torch.as_tensor(X).to(DTYPES[dt])
    return t, (t.float() if dt == "bf16" else t).numpy()


@pytest.mark.parametrize("dt", ["f32", "f64", "bf16"])
@pytest.mark.parametrize("n_quantiles", [1, 10, 1000, 10000])
@pytest.mark.parametrize("chunks", ["whole", 777, 2048])
def test_quantiles_exact(dt, n_quantiles, chunks):
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.preprocessing import QuantileTransformer

    n = 12000
    t, Xh = _column_data(n, 5, 11, dt)
    rows = n if chunks == "whole" else chunks
    C = ChunkedArray([t[i:i + rows].cuda() for i in range(0, n, rows)])
    qt = QuantileTransformer(n_quantiles=n_quantiles, subsample=max(n_quantiles, 10000)).fit(C)
    want = np.percentile(Xh, qt.references_ * 100, axis=0)
    np.testing.assert_array_equal(qt.quantiles_, want)
    assert qt.quantiles_.dtype == np.float64


@pytest.mark.parametrize("dt", ["f32", "f64", "bf16"])
def test_quantiles_one_row_chunks(dt):
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.preprocessing import QuantileTransformer

    t, Xh = _column_data(600, 3, 12, dt)
    C = ChunkedArray([t[i:i + 1].cuda() for i in range(600)])
    qt = QuantileTransformer(n_quantiles=100).fit(C)
    np.testing.assert_array_equal(qt.quantiles_, np.percentile(Xh, qt.references_ * 100, axis=0))


def test_quantiles_nan_column_and_column_groups(monkeypatch):
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.preprocessing import QuantileTransformer
    from dask_ml_b200.preprocessing import data as pp

    t, Xh = _column_data(5000, 6, 13, "f32")
    Xh = Xh.copy()
    Xh[17, 4] = np.nan
    qt = QuantileTransformer(n_quantiles=500).fit(ChunkedArray.from_array(Xh, 1500))
    with np.errstate(invalid="ignore"):
        want = np.percentile(Xh, qt.references_ * 100, axis=0)
    np.testing.assert_array_equal(qt.quantiles_, want)
    assert np.isnan(qt.quantiles_[:, 4]).all()
    monkeypatch.setattr(pp, "HIST_BUDGET", 1000 * 256 * 8 * 2)            # two columns per group
    np.testing.assert_array_equal(QuantileTransformer(n_quantiles=500).fit(ChunkedArray.from_array(Xh, 1500))
                                  .quantiles_, want)


@pytest.mark.parametrize("dt", ["f32", "f64", "bf16"])
@pytest.mark.parametrize("n_quantiles", [1, 2, 57, 1000, 4000])     # 4000: quantiles searched in global memory
@pytest.mark.parametrize("distribution", ["uniform", "normal"])
def test_transform_matches_restatement(dt, n_quantiles, distribution):
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.preprocessing import QuantileTransformer

    n, d = 9000, 5
    # no infinite values: between two infinities np.percentile gives NaN quantiles, on which numpy's interp depends on
    # the previous element's search (DESIGN.md, "The passes of QuantileTransformer")
    t, Xh = _column_data(n, d, 14, dt, infinite=False)
    fit_n = max(n_quantiles, 10)
    qt = QuantileTransformer(n_quantiles=n_quantiles, output_distribution=distribution)
    qt.fit(ChunkedArray.from_array(Xh[:fit_n] if n_quantiles < 1000 else Xh, 4000))
    rng = np.random.RandomState(15)
    Y = Xh * 1.5 + rng.uniform(-1, 1, (1, d))
    Y[::97, 1] = np.nan
    Yt = torch.as_tensor(Y).to(DTYPES[dt])
    Yh = (Yt.float() if dt == "bf16" else Yt).numpy()
    C = ChunkedArray([Yt[i:i + 3000].cuda() for i in range(0, n, 3000)])
    keep = Yt.clone()
    fwd = qt.transform(C)
    assert all(b.dtype == torch.float64 and b.is_cuda for b in fwd.blocks)
    got = fwd.compute()
    want = transform_restated(Yh, qt.quantiles_, qt.references_, False, distribution)
    U = np.clip(np.random.RandomState(16).uniform(-0.1, 1.1, (n, d)), 0, 1) if distribution == "uniform" else \
        np.random.RandomState(16).standard_normal((n, d)) * 3
    U[::89, 2] = np.nan
    U[::101, 0] = 0.0
    inv = qt.inverse_transform(U).compute()
    want_inv = transform_restated(U, qt.quantiles_, qt.references_, True, distribution)
    if distribution == "uniform":
        np.testing.assert_array_equal(got, want)
        np.testing.assert_array_equal(inv, want_inv)
    else:
        assert normal_error(got, want, qt.quantiles_, qt.references_) <= NORMAL_TOL
        assert normal_error(inv, want_inv, qt.quantiles_, qt.references_) <= NORMAL_TOL
    torch.testing.assert_close(torch.cat([b.cpu() for b in C.blocks]), keep, rtol=0, atol=0, equal_nan=True)


def test_output_feeds_kmeans():
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.cluster import KMeans
    from dask_ml_b200.preprocessing import QuantileTransformer

    rng = np.random.RandomState(3)
    cent = rng.uniform(-10, 10, size=(8, 30))
    X = (cent[rng.randint(0, 8, 60000)] + rng.standard_normal((60000, 30)) * 2 + 50).astype(np.float32)
    X0 = X.copy()
    with warnings.catch_warnings():
        warnings.simplefilter("error", RuntimeWarning)
        qt = QuantileTransformer(n_quantiles=200)
        Z = qt.fit_transform(ChunkedArray.from_array(X, 25000))
        assert all(b.is_cuda and b.dtype == torch.float64 for b in Z.blocks)
        Zh = transform_restated(X, qt.quantiles_, qt.references_, False, "uniform")
        np.testing.assert_array_equal(Z.compute(), Zh)
        init = Zh[:8].copy()
        a = KMeans(n_clusters=8, init=init, max_iter=20, tol=0.0).fit(Z)
        b = KMeans(n_clusters=8, init=init, max_iter=20, tol=0.0).fit(ChunkedArray.from_array(Zh, 25000))
    np.testing.assert_array_equal(a.cluster_centers_, b.cluster_centers_)
    np.testing.assert_array_equal(a.labels_.compute(), b.labels_.compute())
    np.testing.assert_array_equal(X, X0)                             # the input is not modified


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _data():
    rng = np.random.RandomState(4)
    return (1e3 + rng.standard_normal((50000, 7)) * rng.uniform(0.5, 3, 7)).astype(np.float32)


def _worker(rank, world, port, out_dir):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    import torch.distributed as dist

    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world)
    try:
        from dask_ml_b200 import ChunkedArray
        from dask_ml_b200.preprocessing import QuantileTransformer

        X = _data()
        lo, hi = (0, 9000) if rank == 0 else (9000, 50000)
        qt = QuantileTransformer().fit(ChunkedArray.from_array(X[lo:hi], 6000))
        np.savez(os.path.join(out_dir, "rank%d.npz" % rank), quantiles=qt.quantiles_)
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpus_equal_one(tmp_path):
    from dask_ml_b200.preprocessing import QuantileTransformer

    mp.start_processes(_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True, start_method="spawn")
    r0, r1 = np.load(tmp_path / "rank0.npz"), np.load(tmp_path / "rank1.npz")
    np.testing.assert_array_equal(r0["quantiles"], r1["quantiles"])
    np.testing.assert_array_equal(r0["quantiles"], QuantileTransformer().fit(_data()).quantiles_)
