"""The split kernels on the device: bkm_split_indices_chunk against the numpy restatement of the permutation bit for
bit, bkm_gather_rows_chunk against torch indexing bit for bit, and train_test_split on device blocks against the host
path on the same data."""
import numpy as np
import pytest
import torch

from dask_ml_b200 import ChunkedArray
from dask_ml_b200.model_selection import train_test_split
from dask_ml_b200.model_selection._split import _blockwise_slice, permutation_indices

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def be():
    from dask_ml_b200.engine import CudaBackend

    return CudaBackend()


@pytest.mark.parametrize("c", [1, 2, 3, 4, 5, 16, 17, 1000, 4 ** 8, 4 ** 8 + 1, 10 ** 6 + 3, 3 * 10 ** 6])
def test_device_indices_equal_the_numpy_restatement(be, c):
    for seed in (0, 1, 2 ** 32 - 2, 2 ** 63 + 12345):
        got = be.split_indices_chunk(seed, c, 0, c, 0).cpu().numpy()
        np.testing.assert_array_equal(got, permutation_indices(seed, c, np.arange(c)))
    start, count = c // 3, c - c // 3 - c // 5
    got = be.split_indices_chunk(9, c, start, count, 10 ** 12).cpu().numpy()
    np.testing.assert_array_equal(got, permutation_indices(9, c, np.arange(start, start + count)) + 10 ** 12)
    assert be.split_indices_chunk(9, c, 0, 0, 0).shape == (0,)


def _block(n, d, dtype, device):
    g = torch.Generator().manual_seed(n + (d or 0))
    shape = (n,) if d is None else (n, d)
    if dtype == torch.bool:
        t = torch.rand(shape, generator=g) < 0.5
    elif dtype in (torch.int32, torch.int64):
        t = torch.randint(-2 ** 30, 2 ** 30, shape, generator=g).to(dtype)
    else:
        t = (torch.randn(shape, generator=g) * 100).to(dtype)
    return t.to(device)


DTYPES = [torch.bfloat16, torch.float16, torch.float32, torch.float64, torch.int32, torch.int64, torch.bool]


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda t: str(t).split(".")[-1])
@pytest.mark.parametrize("d", [None, 1, 3, 13, 64, 100, 128])
def test_gather_equals_indexing(be, dtype, d):
    n = 5003
    src = _block(n, d, dtype, be.device)
    idx = torch.as_tensor(np.random.RandomState(0).permutation(n)[:3001]).to(be.device)
    out = be.gather_rows_chunk(src, idx + 77, 77)
    assert out.dtype == dtype and out.is_cuda and out.is_contiguous()
    assert torch.equal(out, src[idx])
    assert be.gather_rows_chunk(src, idx[:0]).shape[0] == 0


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32, torch.float64, torch.bool],
                         ids=lambda t: str(t).split(".")[-1])
def test_gather_of_padded_pitches_and_unaligned_views(be, dtype):
    n = 2049
    idx = torch.as_tensor(np.random.RandomState(1).randint(0, n, size=4000)).to(be.device)     # repeats allowed
    wide = _block(n, 72, dtype, be.device)
    for view in (wide[:, :64], wide[:, :61], wide[:, 1:66], wide[:, 3:8], wide[:, 5], wide[1:, 2:67], wide.t()[:70]):
        rows = idx % view.shape[0]
        assert torch.equal(be.gather_rows_chunk(view, rows), view[rows])
    flat = _block(n * 3 + 1, None, dtype, be.device)
    assert torch.equal(be.gather_rows_chunk(flat[1:][:n], idx), flat[1:][:n][idx])              # misaligned base
    assert torch.equal(be.gather_rows_chunk(flat[::3][:n], idx), flat[::3][:n][idx])           # strided 1-D


def test_gather_launches_once_and_rows_buffer_blocks_split(be):
    x = be.rows_buffer(1000, 13, torch.float32)                    # the padded pitch to_device gives fp32 rows
    x.copy_(torch.randn(1000, 13))
    idx = be.split_indices_chunk(3, 1000, 0, 1000, 0)
    before = be.launch_count()
    out = be.gather_rows_chunk(x, idx)
    assert be.launch_count() == before + 1
    assert torch.equal(out, x[idx])


def test_train_test_split_on_device_equals_the_host_path(be):
    from dask_ml_b200.datasets import make_classification

    X, y = make_classification(50_000, 20, chunks=12_000, device="cuda", dtype="float32", random_state=0)
    w = ChunkedArray([torch.rand(b.shape[0], dtype=torch.float64, device=b.device) for b in y.blocks])
    dev = train_test_split(X, y, w, test_size=0.2, random_state=0)
    host_in = [ChunkedArray([b.cpu().numpy() for b in a.blocks]) for a in (X, y, w)]
    host = train_test_split(*host_in, test_size=0.2, random_state=0)
    assert len(dev) == 6
    for a, b in zip(dev, host):
        assert all(blk.is_cuda for blk in a.blocks)
        assert a.chunks == b.chunks and a.dtype == b.dtype
        np.testing.assert_array_equal(a.compute(), b.compute())
    # a host array next to device arrays is split on the host with the same indices
    mixed = train_test_split(X, host_in[1], test_size=0.2, random_state=0)
    assert isinstance(mixed[2].blocks[0], np.ndarray)
    np.testing.assert_array_equal(mixed[3].compute(), host[3].compute())


def test_blockwise_slice_rejects_foreign_indices_on_the_device(be):
    X = ChunkedArray([torch.arange(20.0, device=be.device).reshape(10, 2), torch.arange(20.0, 40.0, device=be.device).reshape(10, 2)])
    with pytest.raises(IndexError):
        _blockwise_slice(X, ChunkedArray([np.array([0, 10]), np.array([11])]))
    ok = _blockwise_slice(X, ChunkedArray([np.array([9, 0]), np.array([11])]))
    np.testing.assert_array_equal(ok.compute()[:, 0], [18.0, 0.0, 22.0])


def test_supervised_chain_stays_on_the_device():
    from dask_ml_b200.datasets import make_classification
    from dask_ml_b200.linear_model import LogisticRegression
    from dask_ml_b200.metrics import accuracy_score, log_loss

    X, y = make_classification(200_000, 64, chunks=1 << 16, device="cuda", dtype="float32", random_state=0)
    parts = train_test_split(X, y, test_size=0.2, random_state=0)
    X_train, X_test, y_train, y_test = parts
    assert all(b.is_cuda for a in parts for b in a.blocks)
    assert X_train.shape[0] + X_test.shape[0] == 200_000 and len(y_test) == X_test.shape[0]
    clf = LogisticRegression().fit(X_train, y_train)
    pred, proba = clf.predict(X_test), clf.predict_proba(X_test)
    assert all(b.is_cuda for a in (pred, proba) for b in a.blocks)
    acc, ll = accuracy_score(y_test, pred), log_loss(y_test, proba)
    assert 0.5 < acc <= 1.0 and np.isfinite(ll)
    h = [ChunkedArray([b.cpu().numpy() for b in a.blocks]) for a in (y_test, pred, proba)]
    np.testing.assert_allclose(acc, accuracy_score(h[0], h[1]), rtol=1e-12)
    np.testing.assert_allclose(ll, log_loss(h[0], h[2]), rtol=1e-12)
    np.testing.assert_allclose(acc, clf.score(X_test, y_test), rtol=1e-12)
