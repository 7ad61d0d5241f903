"""GPU tests of the public distance operators (dask_ml/metrics/pairwise.py) — ports of the reference's
tests/metrics/test_metrics.py:46-84 plus the tensor-path transform kernel at larger shapes."""
import numpy as np
import pytest
import sklearn.metrics

pytestmark = pytest.mark.gpu


def _chunked(a, rows):
    from dask_ml_b200 import ChunkedArray

    return ChunkedArray.from_array(a, rows)


def test_euclidean_distances():
    """tests/metrics/test_metrics.py:46-61 (X, Y uniform 100 x 4, chunks of 50; with and without given norms)."""
    import dask_ml_b200.metrics as m

    rng = np.random.RandomState(0)
    X, Y = rng.uniform(size=(100, 4)), rng.uniform(size=(100, 4))
    b = sklearn.metrics.euclidean_distances(X, Y)
    a = m.euclidean_distances(_chunked(X, 50), Y).compute()
    np.testing.assert_allclose(a, b, atol=1e-12)
    xns = (X ** 2).sum(axis=1)[:, np.newaxis]
    a = m.euclidean_distances(_chunked(X, 50), Y, X_norm_squared=xns).compute()
    np.testing.assert_allclose(a, sklearn.metrics.euclidean_distances(X, Y, X_norm_squared=xns), atol=1e-12)
    yns = (Y ** 2).sum(axis=1)[np.newaxis, :]
    a = m.euclidean_distances(_chunked(X, 50), Y, Y_norm_squared=yns).compute()
    np.testing.assert_allclose(a, sklearn.metrics.euclidean_distances(X, Y, Y_norm_squared=yns), atol=1e-12)
    with pytest.raises(ValueError):
        m.euclidean_distances(_chunked(X, 50), Y, X_norm_squared=np.ones((3, 1)))


def test_euclidean_distances_same():
    """tests/metrics/test_metrics.py:64-71: X against itself, explicitly and with Y=None."""
    import dask_ml_b200.metrics as m

    X = np.random.RandomState(1).uniform(size=(100, 4))
    b = sklearn.metrics.euclidean_distances(X, X)
    np.testing.assert_allclose(m.euclidean_distances(_chunked(X, 50), X).compute(), b, atol=1e-4)
    np.testing.assert_allclose(m.euclidean_distances(_chunked(X, 50)).compute(), b, atol=1e-4)
    Xf = X.astype(np.float32)
    a = m.euclidean_distances(_chunked(Xf, 50)).compute()
    assert a.dtype == np.float32
    # float32 GEMM-form distances cancel at ||x||^2 + ||y||^2: the diagonal is sqrt(rounding error), not 0 (the
    # reference's float32 formula, pairwise.py:93-97, behaves the same way)
    np.testing.assert_allclose(a, b, atol=5e-3)


def test_rbf_kernel_and_pairwise_kernels():
    """tests/metrics/test_metrics.py:74-84 for the kernel on the distance path."""
    import dask_ml_b200.metrics as m

    rng = np.random.RandomState(2)
    X, Y = rng.uniform(size=(100, 4)), rng.uniform(size=(30, 4))
    np.testing.assert_allclose(m.rbf_kernel(_chunked(X, 50), Y).compute(), sklearn.metrics.pairwise.rbf_kernel(X, Y), atol=1e-12)
    np.testing.assert_allclose(m.pairwise_kernels(_chunked(X, 50), Y, metric="rbf", gamma=0.7).compute(),
                               sklearn.metrics.pairwise.rbf_kernel(X, Y, gamma=0.7), atol=1e-12)
    np.testing.assert_allclose(m.rbf_kernel(_chunked(X.astype(np.float32), 50)).compute(),
                               sklearn.metrics.pairwise.rbf_kernel(X, X), atol=2e-6)
    with pytest.raises(ValueError):
        m.pairwise_kernels(_chunked(X, 50), Y, metric="nope")


@pytest.mark.parametrize("n,d,k", [(20000, 64, 256), (5001, 41, 100), (3000, 64, 300), (777, 13, 20), (100, 8, 600)])
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_transform_tensor_path(n, d, k, mode):
    """fp32 blocks of distances / squared distances / rbf values from the tensor-core transform epilogue (column blocks of
    256 for wider Y) against float64 on the device; error relative to ||x||^2 + ||y||^2 like the reference's own
    float32 formula (pairwise.py:93-97 cancels at that scale)."""
    import torch
    import dask_ml_b200.metrics as m
    from dask_ml_b200.metrics.pairwise import _as_device, _distance_blocks

    g = torch.Generator(device="cuda").manual_seed(n + k)
    X = torch.randn((n, d), device="cuda", generator=g) * 3.0 + 1.0
    Y = (torch.randn((k, d), device="cuda", generator=g) * 3.0 + 1.0).double()
    Xd = _as_device(X)
    gamma = 0.01
    out = _distance_blocks(Xd, Y.cpu().numpy(), mode, gamma)[0]
    assert out.shape == (n, k) and out.dtype == torch.float32
    X64 = X.double()
    d2 = torch.clamp((X64 * X64).sum(1, keepdim=True) + (Y * Y).sum(1)[None, :] - 2.0 * X64 @ Y.T, min=0.0)
    scale = (X64 * X64).sum(1, keepdim=True) + (Y * Y).sum(1)[None, :]
    got = out.double()
    if mode == 0:
        err = ((got * got - d2).abs() / scale).max()
    elif mode == 1:
        err = ((got - d2).abs() / scale).max()
    else:
        err = (got - torch.exp(-gamma * d2)).abs().max() / (gamma * float(scale.max()))
    assert float(err) < 2e-6, float(err)


def test_kmeans_transform_matches_sklearn():
    from dask_ml_b200.cluster import KMeans
    from sklearn.cluster import KMeans as SK

    X = np.random.RandomState(3).standard_normal((5000, 16)).astype(np.float32)
    init = X[:8].copy()
    a = KMeans(n_clusters=8, init=init, max_iter=5).fit(X)
    b = SK(n_clusters=8, init=init, n_init=1, max_iter=5, algorithm="lloyd").fit(X)
    np.testing.assert_allclose(a.transform(X).compute(), b.transform(X), rtol=2e-3, atol=2e-3)
