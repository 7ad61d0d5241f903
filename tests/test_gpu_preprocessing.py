"""The scalers on the H100: fixture replay (resident and host-resident), the affine pass bit for bit against numpy's
two-step expression, the statistics pass against float64 numpy (non-finite rules, fixed summation order), exact
percentiles for every chunking, StandardScaler feeding KMeans in place, and two ranks against one."""
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
from test_preprocessing_host import CASES, replay  # noqa: E402

DTYPES = {"f32": torch.float32, "f64": torch.float64, "bf16": torch.bfloat16}


def _backend():
    from dask_ml_b200.engine import CudaBackend

    return CudaBackend()


def _rows(n, d, dt, seed, pitch=None, offset=0.0):
    rng = np.random.RandomState(seed)
    X = rng.standard_normal((n, d)) * rng.uniform(0.5, 2, d) + offset
    t = torch.as_tensor(X).to(DTYPES[dt])
    if pitch is not None:
        buf = torch.zeros((n, pitch), dtype=t.dtype)
        buf[:, :d] = t
        t = buf[:, :d]
    return t.cuda(), (t.float() if dt == "bf16" else t).numpy()


@pytest.mark.parametrize("name", CASES)
@pytest.mark.parametrize("resident", [True, False])
def test_fixture_replay(name, resident):
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.engine import host_resident

    if resident:
        replay(name)
    else:
        replay(name, to_input=lambda a, r: host_resident(ChunkedArray.from_array(a, r), block_rows=333))


@pytest.mark.parametrize("dt", ["f32", "f64", "bf16"])
@pytest.mark.parametrize("d", [1, 3, 41, 64, 100, 257])
def test_affine_bit_identical(dt, d):
    be = _backend()
    rng = np.random.RandomState(d)
    for n in (0, 1, 1023, 1025, 4097):
        for pitch in (None, d + 3):
            x, h = _rows(n, d, dt, n + d, pitch=pitch)
            for adt in (np.float32, np.float64):
                odt = np.result_type(h.dtype, adt)
                a = (rng.standard_normal(d) * 3).astype(adt)
                b = rng.uniform(0.1, 4, d).astype(adt)
                b[0] = 0.0                                            # a zero scale gives inf / NaN, as in numpy
                hx = h.astype(odt)
                for op1, op2 in ((1, 1), (2, 2), (0, 1), (1, 0), (0, 2), (0, 0)):
                    out = be.rows_buffer(n, d, torch.float64 if odt == np.float64 else torch.float32)
                    be.affine_chunk(x, torch.as_tensor(a.astype(np.float64)).cuda(),
                                    torch.as_tensor(b.astype(np.float64)).cuda(), op1, op2, out)
                    want = hx
                    with np.errstate(all="ignore"):
                        if op1:
                            want = want - a.astype(odt) if op1 == 1 else want * a.astype(odt)
                        if op2:
                            want = want / b.astype(odt) if op2 == 1 else want + b.astype(odt)
                    got = out.cpu().numpy()
                    assert got.dtype == want.dtype
                    np.testing.assert_array_equal(got.view(np.uint8), np.ascontiguousarray(want).view(np.uint8),
                                                  err_msg="n=%d pitch=%s ops=%d,%d" % (n, pitch, op1, op2))


def _stats(be, xs, shift):
    d = xs[0].shape[1]
    acc = torch.full((5, d), np.nan, dtype=torch.float64, device="cuda")
    mm = torch.full((2, d), np.nan, dtype=torch.float64, device="cuda")
    s = torch.as_tensor(shift).cuda()
    for i, x in enumerate(xs):
        be.colstats_chunk(x, s, acc, mm, first=i == 0)
    torch.cuda.synchronize()
    return acc.cpu().numpy(), mm.cpu().numpy()


@pytest.mark.parametrize("dt", ["f32", "f64", "bf16"])
@pytest.mark.parametrize("d", [1, 13, 64, 128, 300])
def test_colstats_match_float64(dt, d):
    be = _backend()
    xs, hs = [], []
    for i, n in enumerate([0, 1, 257, 40000]):
        x, h = _rows(n, d, dt, i + d, pitch=d + 5 if i == 2 else None, offset=1e3)
        xs.append(x), hs.append(h.astype(np.float64))
    H = np.concatenate(hs)
    shift = H[:100].mean(0)
    acc, mm = _stats(be, xs, shift)
    t = H - shift
    np.testing.assert_allclose(acc[0], t.sum(0), rtol=1e-12, atol=1e-9 * np.abs(t).sum(0).max())
    # a raw sum of 40K squares: the kernel's row-order sum and numpy's pairwise sum differ by up to ~n eps
    np.testing.assert_allclose(acc[1], (t * t).sum(0), rtol=1e-11)
    assert (acc[2:] == 0).all()
    np.testing.assert_array_equal(mm[0], H.min(0))
    np.testing.assert_array_equal(mm[1], H.max(0))
    acc2, mm2 = _stats(be, xs, shift)                                # fixed order: the same bits
    np.testing.assert_array_equal(acc2.view(np.uint64), acc.view(np.uint64))
    np.testing.assert_array_equal(mm2, mm)


def test_variance_on_offset_data_and_nonfinite_rules():
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.preprocessing.data import column_stats
    from dask_ml_b200.decomposition.pca import _device_data

    rng = np.random.RandomState(5)
    X = 1e6 + rng.standard_normal((300000, 6))
    mean, var, lo, hi = column_stats(_device_data(ChunkedArray.from_array(X, 70000)))
    np.testing.assert_allclose(mean, X.mean(0), rtol=1e-12)
    np.testing.assert_allclose(var, X.var(0), rtol=1e-9)
    X[17, 0] = np.nan
    X[5, 1], X[99, 1] = np.inf, -np.inf
    X[8, 2] = np.inf
    X[200000, 3] = -np.inf
    mean, var, lo, hi = column_stats(_device_data(ChunkedArray.from_array(X, 70000)))
    with np.errstate(all="ignore"):
        wm, wv, wl, wh = X.mean(0), X.var(0), X.min(0), X.max(0)
    for got, want in ((mean, wm), (var, wv), (lo, wl), (hi, wh)):
        np.testing.assert_array_equal(np.isnan(got), np.isnan(want))
        np.testing.assert_array_equal(got[~np.isfinite(want)], want[~np.isfinite(want)])
    np.testing.assert_allclose(mean[4:], wm[4:], rtol=1e-12)
    np.testing.assert_array_equal(lo, wl)


def _percentile_cases():
    rng = np.random.RandomState(11)
    cols = rng.standard_normal((5000, 4))
    cols[:, 1] = rng.randint(-3, 4, 5000)                           # many duplicates
    cols[::7, 2] = 0.0
    cols[::11, 2] = -0.0
    cols[:3, 3] = [np.inf, -np.inf, np.inf]
    return cols


@pytest.mark.parametrize("dt", ["f32", "f64", "bf16"])
@pytest.mark.parametrize("chunks", [5000, 1, 777, 2048])
def test_percentiles_exact(dt, chunks):
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.decomposition.pca import _device_data
    from dask_ml_b200.preprocessing.data import percentiles

    X = _percentile_cases()[: (5000 if chunks != 1 else 60)]
    t = torch.as_tensor(X).to(DTYPES[dt])
    h = (t.float() if dt == "bf16" else t).numpy()
    for q in ([25, 50.0, 75], [0, 50.0, 100], [10, 50.0, 90], [50, 50.0, 50], [0.1, 50.0, 99.9]):
        for n in (len(h), 1, 2):
            got = percentiles(_device_data(ChunkedArray.from_array(t[:n].cuda(), chunks)), q)
            with np.errstate(invalid="ignore"):
                want = np.stack([np.percentile(h[:n, j], q) for j in range(h.shape[1])])
            assert got.dtype == want.dtype == np.float64
            np.testing.assert_array_equal(got, want, err_msg="q=%s n=%d" % (q, n))   # == : zeros may differ in sign


def test_percentiles_nan_column():
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.preprocessing.data import percentiles
    from dask_ml_b200.decomposition.pca import _device_data

    X = np.random.RandomState(2).standard_normal((999, 3)).astype(np.float32)
    X[10, 1] = np.nan
    got = percentiles(_device_data(ChunkedArray.from_array(X, 400)), [25, 50.0, 75])   # ndarrays are checked finite
    with np.errstate(invalid="ignore"):
        want = np.stack([np.percentile(X[:, j], [25, 50.0, 75]) for j in range(3)])
    np.testing.assert_array_equal(got, want)


def test_standard_scaler_feeds_kmeans():
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.cluster import KMeans
    from dask_ml_b200.preprocessing import StandardScaler

    rng = np.random.RandomState(3)
    cent = rng.uniform(-10, 10, size=(8, 30))
    X = (cent[rng.randint(0, 8, 60000)] + rng.standard_normal((60000, 30)) * 2 + 50).astype(np.float32)
    X0 = X.copy()
    with warnings.catch_warnings():
        warnings.simplefilter("error", RuntimeWarning)
        sc = StandardScaler()
        Z = sc.fit_transform(ChunkedArray.from_array(X, 25000))
        assert all(b.is_cuda and b.stride(0) == 32 for b in Z.blocks)       # the pitch to_device gives d = 30
        Zh = (X - sc.mean_) / sc.scale_
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
        from dask_ml_b200.preprocessing import MinMaxScaler, RobustScaler, StandardScaler

        X = _data()
        lo, hi = (0, 9000) if rank == 0 else (9000, 50000)
        C = ChunkedArray.from_array(X[lo:hi], 6000)
        s, m, r = StandardScaler().fit(C), MinMaxScaler().fit(C), RobustScaler().fit(C)
        np.savez(os.path.join(out_dir, "rank%d.npz" % rank), mean=s.mean_, var=s.var_, lo=m.data_min_,
                 hi=m.data_max_, center=r.center_, scale=r.scale_)
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpus_equal_one(tmp_path):
    from dask_ml_b200.preprocessing import MinMaxScaler, RobustScaler, StandardScaler

    mp.start_processes(_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True, start_method="spawn")
    r0, r1 = np.load(tmp_path / "rank0.npz"), np.load(tmp_path / "rank1.npz")
    for key in r0.files:
        np.testing.assert_array_equal(r0[key], r1[key])
    X = _data()
    s, m, r = StandardScaler().fit(X), MinMaxScaler().fit(X), RobustScaler().fit(X)
    np.testing.assert_allclose(r0["mean"], s.mean_, rtol=1e-6)
    np.testing.assert_allclose(r0["var"], s.var_, rtol=1e-6)
    np.testing.assert_array_equal(r0["lo"], m.data_min_)
    np.testing.assert_array_equal(r0["hi"], m.data_max_)
    np.testing.assert_array_equal(r0["center"], r.center_)
    np.testing.assert_array_equal(r0["scale"], r.scale_)
