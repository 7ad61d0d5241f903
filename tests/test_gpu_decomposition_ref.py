"""PCA / TruncatedSVD on the H100 against the fixtures written by the reference's own pca.py / truncated_svd.py, and
the corner cases of the projection's arg-max epilogue: equal |t| in the same thread, across the row groups of a warp,
across warps, across CTAs and across chunks must all resolve to the lowest global row."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import decomp_golden as dg  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", dg.CASES)
def test_reference_fixture_replays_on_the_device(name):
    dg.replay(name)


@pytest.mark.parametrize("name", ["ref_decomp_pca_f64_offset_k3", "ref_decomp_tsvd_f32_k3"])
def test_reference_fixture_replays_host_resident(name):
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.engine import host_resident

    dg.replay(name, to_input=lambda a, rows: host_resident(ChunkedArray.from_array(a, rows), block_rows=rows))


@pytest.mark.parametrize("dt", [torch.float32, torch.float64, torch.bfloat16])
@pytest.mark.parametrize("k", [3, 20, 40, 70])
def test_argmax_ties_take_the_lowest_global_row(dt, k):
    from dask_ml_b200.engine import CudaBackend

    be = CudaBackend()
    n, d = 200_000, 24
    rng = np.random.RandomState(3)
    X = rng.uniform(-1e-3, 1e-3, size=(n, d))
    ext = rng.choice([-8.0, 8.0], size=d)
    # row r of a 64-row tile: warp r // 16 % 4 (shared-memory fold), row group r % 8 (shuffles), half r // 8 % 2 (the
    # same thread's two rows); tile 5 is one CTA, tile 1500 another, row 150000 lies in the second chunk
    dup = [64 * 5 + 43, 64 * 5 + 11, 64 * 5 + 3, 64 * 5 + 27, 64 * 1500 + 1, 150_000]
    neg = [64 * 5 + 50, 64 * 7 + 2, 160_000]                   # the negated extreme: equal |t|, opposite sign
    X[dup] = ext
    X[neg] = -ext
    Xt = torch.as_tensor(X).to(dt)
    h = Xt.to(torch.float64).numpy()
    W = rng.standard_normal((k, d))
    x = Xt.cuda()
    Wd = torch.as_tensor(W).cuda()
    rec = be.colmax_new(k)
    split = 100_000
    be.project_chunk(x[:split], None, Wd, colmax=rec, row_offset=0)
    be.project_chunk(x[split:], None, Wd, colmax=rec, row_offset=split)
    r = rec.cpu()
    rows = r[:, 1:2].contiguous().view(torch.int64).numpy()[:, 0]
    t = h @ W.T
    a = np.abs(t)
    want = np.argmax(a, axis=0)                                # first row among equal maxima
    assert set(want.tolist()) <= set(dup + neg)               # the extremes win every column
    np.testing.assert_array_equal(rows, want)
    np.testing.assert_array_equal(np.sign(r[:, 2].numpy()), np.sign(t[want, np.arange(k)]))
    np.testing.assert_array_equal(r[:, 0].numpy(), a[want, np.arange(k)])


def test_zero_components_and_overflow():
    from dask_ml_b200.decomposition import PCA

    rng = np.random.RandomState(0)
    X = rng.standard_normal((3000, 7))
    p = PCA(n_components=0, svd_solver="full")
    assert p.fit_transform(X).compute().shape == (3000, 0)
    assert p.components_.shape == (0, 7) and p.transform(X).compute().shape == (3000, 0)
    X[17, 3] = 1e160
    with pytest.raises(ValueError, match="too large for a float64 Gram matrix"):
        PCA(n_components=2).fit(X)
    X[17, 3] = np.nan
    with pytest.raises(ValueError, match="Input contains NaN"):
        PCA(n_components=2).fit(torch.as_tensor(X).cuda())


def test_transform_runs_no_argmax_epilogue():
    """transform projects only: one launch per chunk and no host read of arg-max records (the records are not even
    allocated)."""
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.decomposition import PCA
    from dask_ml_b200.decomposition import pca as pca_mod

    rng = np.random.RandomState(1)
    X = rng.standard_normal((20000, 16))
    p = PCA(n_components=4).fit(X)
    data = pca_mod._device_data(ChunkedArray.from_array(X, 5000))
    calls = []
    orig = data.backend.colmax_new
    data.backend.colmax_new = lambda k: calls.append(k) or orig(k)
    lib = data.backend.lib
    c0 = int(lib.bkm_launch_count())
    T = p.transform(data).compute()
    assert int(lib.bkm_launch_count()) - c0 == 4 and calls == []
    np.testing.assert_allclose(T, (X - p.mean_) @ p.components_.T, atol=1e-9)
