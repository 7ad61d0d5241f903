"""Host-side logic without a GPU: the C-ABI library loads and exports every declared symbol; the
estimator's validation / error contract; the Lloyd control flow (reference quirks Q1-Q6) and the
k-means|| bookkeeping driven through a TEST-ONLY checker backend built on the CPU oracle."""
import ctypes
import os
import re

import numpy as np
import pytest
import sklearn.datasets
from sklearn.cluster import KMeans as SKKMeans, kmeans_plusplus

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture
def cpu_engine(monkeypatch, oracle):
    from dask_ml_b200.cluster import k_means as km
    from oracle_backend import OracleBackend

    monkeypatch.setattr(km, "_BACKEND_FACTORY", OracleBackend)
    return km


# ------------------------------------------------------------------------------------------ C ABI
def test_library_exports_every_declared_symbol():
    """include/bkm_b200.h vs the built .so vs the ctypes table: all three must agree (no compute calls)."""
    from dask_ml_b200 import _lib

    hdr = open(os.path.join(ROOT, "include", "bkm_b200.h")).read()
    declared = set(re.findall(r"\b(bkm_[a-z0-9_]+)\s*\(", hdr))
    assert declared == set(_lib.SIGNATURES), declared ^ set(_lib.SIGNATURES)
    lib = _lib.load()
    for name in declared:
        assert hasattr(lib, name), name
    assert lib.bkm_version() == 200
    assert lib.bkm_error_string(-3) == b"shape not supported by any kernel"
    out = ctypes.c_size_t(0)
    assert lib.bkm_centers_pack_bytes(256, 64, 0, ctypes.byref(out)) == 0 and out.value > 256 * 64 * 4
    assert lib.bkm_workspace_bytes(1000, 64, 256, 0, ctypes.byref(out)) == 0 and out.value > 0
    assert lib.bkm_workspace_bytes(1000, 64, 256, 7, ctypes.byref(out)) == -2          # BKM_EDTYPE
    assert lib.bkm_kernel_family(64, 256, 0, 0) == 1      # tensor-core path
    assert lib.bkm_kernel_family(41, 100, 0, 0) == 1      # tensor-core path too (given a 16-byte row pitch; else the launch falls back)
    assert lib.bkm_kernel_family(100, 100, 0, 0) == 0     # CUDA-core path: d > 64
    assert lib.bkm_kernel_family(13, 20, 0, 0) == 2       # streaming CUDA-core kernel: tiny k*d is HBM-bound
    assert lib.bkm_kernel_family(13, 20, 0, 1) == 0       # FORCE_SIMT -> the generic CUDA-core kernel
    assert lib.bkm_kernel_family(13, 20, 0, 2) == 1       # ... unless forced
    assert lib.bkm_kernel_family(64, 300, 0, 0) == 0      # CUDA-core path: k > 256
    assert lib.bkm_kernel_family(64, 256, 1, 0) == 0      # float64 -> CUDA cores
    assert lib.bkm_kernel_family(64, 1024, 0, 2) == -3    # FORCE_TC on an unsupported shape


def test_no_gpu_means_loud_failure():
    import torch

    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from dask_ml_b200.cluster import KMeans

    with pytest.raises(RuntimeError, match="no CPU fallback"):
        KMeans(3).fit(np.random.rand(50, 2))


def test_product_never_imports_oracle():
    """The oracle is test infrastructure: nothing under dask_ml_b200/ may reference it."""
    for dirpath, _, files in os.walk(os.path.join(ROOT, "dask_ml_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f)).read()
                assert "kmeans_oracle" not in src and "oracle_c" not in src and "from oracle" not in src, f


# ------------------------------------------------------------------------------------------ ChunkedArray
def test_chunked_array_protocol():
    from dask_ml_b200 import ChunkedArray

    X = np.arange(70.0).reshape(35, 2)
    c = ChunkedArray.from_array(X, 10)
    assert c.chunks == ((10, 10, 10, 5), (2,)) and c.shape == (35, 2) and c.dtype == np.float64
    assert c.numblocks == (4, 1) and len(c) == 35
    np.testing.assert_array_equal(c.compute(), X)
    np.testing.assert_array_equal(np.asarray(c), X)
    np.testing.assert_array_equal(c.rows([34, 0, 12]), X[[34, 0, 12]])
    assert c.astype("f4").dtype == np.float32
    with pytest.raises(ValueError):
        ChunkedArray([np.zeros((3, 2)), np.zeros((3, 3))])


# ------------------------------------------------------------------------------------------ estimator
def test_fit_given_init(cpu_engine):
    """reference tests/test_kmeans.py:87-98 through the estimator + host loop."""
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.cluster import KMeans

    X_, _ = sklearn.datasets.make_blobs(n_samples=1000, n_features=4, random_state=1)
    init, _ = kmeans_plusplus(X_, 3, random_state=np.random.RandomState(0))
    dkkm = KMeans(3, init=init, random_state=0).fit(ChunkedArray.from_array(X_, 500))
    skkm = SKKMeans(3, init=init, random_state=0, n_init=1).fit(X_)
    np.testing.assert_allclose(dkkm.inertia_, skkm.inertia_)
    np.testing.assert_array_equal(dkkm.labels_.compute(), skkm.labels_)
    assert dkkm.labels_.dtype == np.int32 and isinstance(dkkm.inertia_, np.float64)
    assert dkkm.cluster_centers_.dtype == X_.dtype and dkkm.n_iter_ == 2


def test_host_loop_equals_oracle_on_all_branches(cpu_engine, oracle):
    """Same control flow as k_means.py:499-569 on: converged (<=1e-7), tol break with re-label, max_iter."""
    from dask_ml_b200.cluster import KMeans

    centers = np.array([[-7, -7], [0, 0], [7, 7]])
    Xs, _ = oracle.make_blobs(cluster_std=0.1, centers=centers, chunks=50, random_state=0)
    X = np.concatenate(Xs)
    init = centers.astype(np.float64)
    for tol, max_iter in ((1e-4, 300), (0.5, 300), (0.0, 3), (0.0, 1), (1e-12, 300)):
        km = KMeans(3, init=init, tol=tol, max_iter=max_iter).fit(X)
        lab, inertia, C, n_iter = oracle.kmeans_single_lloyd(Xs, 3, init=init, tol=tol, max_iter=max_iter)
        assert km.n_iter_ == n_iter
        np.testing.assert_allclose(km.inertia_, inertia, rtol=1e-12)
        np.testing.assert_allclose(km.cluster_centers_, C, rtol=1e-13, atol=1e-15)
        np.testing.assert_array_equal(km.labels_.compute(), np.concatenate(lab))


def test_predict_transform_and_dtypes(cpu_engine):
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.cluster import KMeans

    X = np.random.RandomState(0).uniform(size=(100, 2))
    X2 = X.astype("f4")
    for xx, yy in [(X, X), (X2, X2), (X, X2), (X2, X)]:
        a = KMeans(random_state=0).fit(ChunkedArray.from_array(xx, 50))
        b = SKKMeans(n_init=1, random_state=0).fit(xx)
        assert a.cluster_centers_.dtype == b.cluster_centers_.dtype
        assert a.labels_.dtype == b.labels_.dtype
        assert a.transform(xx).dtype == b.transform(xx).dtype
        assert a.transform(yy).dtype == b.transform(yy).dtype
        p = a.predict(xx)
        assert p.dtype == np.int32 and p.shape == (100,)
        with pytest.raises(ValueError, match="features"):
            a.predict(np.zeros((5, 3)))
        d = ((xx[:, None, :].astype(float) - a.cluster_centers_[None].astype(float)) ** 2).sum(-1)
        np.testing.assert_array_equal(p.compute(), d.argmin(1))


def test_error_contract(cpu_engine):
    """reference tests/test_kmeans.py:45-51,131-147,162-166 + NaN/inf (k_means.py:179-185)."""
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.cluster import KMeans, k_means as km_mod

    km = KMeans()
    with pytest.raises(ValueError):
        km.fit(np.array([]).reshape(0, 1))
    with pytest.raises(ValueError):
        km.fit(np.array([]).reshape(1, 0))
    X = np.random.RandomState(0).uniform(size=(100, 3))
    Xc = ChunkedArray.from_array(X, 25)
    with pytest.raises(ValueError):
        km_mod.k_init(Xc, 3, X[:2])
    with pytest.raises(ValueError):
        km_mod.k_init(Xc, 2, X[:2, :-1])
    with pytest.raises(ValueError):
        km_mod.k_init(Xc, 2, "invalid")
    with pytest.raises(TypeError):
        km_mod.k_init(Xc, 2, 2)
    X[7, 1] = np.nan
    with pytest.raises(ValueError, match="NaN"):
        km.fit(ChunkedArray.from_array(X, 25))

    class FakeDaskDataFrame(object):
        pass
    FakeDaskDataFrame.__module__ = "dask.dataframe.core"
    with pytest.raises(TypeError):
        km.fit(FakeDaskDataFrame())


def test_inputs_and_too_small(cpu_engine):
    """reference tests/test_kmeans.py:39-42,149-160."""
    import pandas as pd

    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.cluster import KMeans

    rng = np.random.RandomState(0)
    KMeans(random_state=0).fit(ChunkedArray.from_array(rng.uniform(size=(20, 2)), 10))
    for X in (rng.uniform(size=(100, 4)), ChunkedArray.from_array(rng.uniform(size=(100, 4)), (10, 4)),
              pd.DataFrame(rng.uniform(size=(100, 4))), rng.randint(0, 9, size=(100, 4)).astype(np.int32)):
        km = KMeans(n_clusters=3, random_state=0).fit(X)
        assert km.transform(X).shape == (100, 3)


def test_sklearn_params_protocol():
    from sklearn.base import clone

    from dask_ml_b200.cluster import KMeans

    km = KMeans(n_clusters=5, init="random", tol=1e-3, n_jobs=4, algorithm="elkan")
    p = km.get_params()
    assert p["n_clusters"] == 5 and p["oversampling_factor"] == 2 and p["precompute_distances"] == "auto"
    assert clone(km).get_params() == p
    km.set_params(max_iter=7)
    assert km.max_iter == 7


def test_kmeans_parallel_init_is_chunking_invariant(cpu_engine, oracle):
    """The Philox draw is keyed by the global row index, so k-means|| picks the same candidates whatever
    the chunking; and it matches the oracle's init_scalable driven by the same stream."""
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.cluster import k_means as km_mod

    rng = np.random.RandomState(3)
    cent = rng.uniform(-20, 20, size=(6, 5))
    X = cent[rng.randint(0, 6, size=3000)] + 0.3 * rng.standard_normal((3000, 5))
    a = km_mod.k_init(ChunkedArray.from_array(X, 3000), 6, "k-means||", random_state=5, oversampling_factor=8)
    b = km_mod.k_init(ChunkedArray.from_array(X, 700), 6, "k-means||", random_state=5, oversampling_factor=8)
    np.testing.assert_allclose(a, b, rtol=1e-12)
    assert a.shape == (6, 5)


# ------------------------------------------------------------------------------------------ datasets.make_blobs
def test_make_blobs_host_path_is_the_reference_contract(oracle):
    """datasets.py:154-202: prototype centres from one scikit-learn call with the user seed, block i from
    sklearn.make_blobs(random_state=i).  The product's host path must equal the oracle's restatement bit for bit."""
    import sklearn.datasets
    from dask_ml_b200.datasets import make_blobs

    X, y = make_blobs(n_samples=1000, n_features=16, centers=8, random_state=0, chunks=125)
    Xo, yo = oracle.make_blobs(n_samples=1000, n_features=16, centers=8, random_state=0, chunks=125)
    assert X.chunks == ((125,) * 8, (16,)) and y.chunks == ((125,) * 8,)
    assert X.dtype == np.float64 and y.dtype == np.int64
    for a, b in zip(X.blocks, Xo):
        np.testing.assert_array_equal(a, b)
    for a, b in zip(y.blocks, yo):
        np.testing.assert_array_equal(a, b)
    # block 3 is sklearn's block with random_state=3 around the same prototype centres
    Xp, yp = sklearn.datasets.make_blobs(n_samples=125, n_features=16, centers=8, random_state=0)
    proto = np.stack([Xp[yp == i].mean(0) for i in range(8)])
    X3, _ = sklearn.datasets.make_blobs(n_samples=125, n_features=16, centers=proto, random_state=3)
    np.testing.assert_array_equal(X.blocks[3], X3)
    # explicit centres, ragged last block, blockshape form
    C = np.array([[0.0, 0.0], [5.0, 5.0]])
    X2, y2 = make_blobs(n_samples=250, n_features=2, centers=C, cluster_std=0.1, chunks=(100, 2), random_state=1)
    assert X2.chunks[0] == (100, 100, 50)
    assert np.abs(X2.compute()[y2.compute() == 1].mean(0) - 5.0).max() < 0.1
    with pytest.raises(ValueError):
        make_blobs(n_samples=100, n_features=4, chunks=(50, 2))


def test_host_resident_streaming_gives_the_same_fit(cpu_engine, oracle):
    """Out-of-core path: rows that stay in host memory and are streamed block by block on every sweep must give exactly
    the fit of the resident path (same kernels in the same order; here through the CPU checker backend)."""
    from oracle_backend import OracleBackend
    from dask_ml_b200.cluster import KMeans
    from dask_ml_b200.engine import host_resident

    rng = np.random.RandomState(5)
    X = (rng.uniform(-5, 5, size=(4, 6))[rng.randint(0, 4, size=3000)] + rng.standard_normal((3000, 6))).astype(np.float32)
    init = X[:4].copy()
    a = KMeans(4, init=init, max_iter=10).fit(X)
    Xh = host_resident(X, backend=OracleBackend(), block_rows=700)       # 5 streamed blocks
    assert Xh.chunk_rows == [700, 700, 700, 700, 200] and Xh.n_local == 3000
    b = KMeans(4, init=init, max_iter=10).fit(Xh)
    assert a.n_iter_ == b.n_iter_
    np.testing.assert_array_equal(a.labels_.compute(), b.labels_.compute())
    np.testing.assert_allclose(a.cluster_centers_, b.cluster_centers_, rtol=1e-12)
    np.testing.assert_array_equal(b.predict(Xh).compute(), a.predict(X).compute())
    c = KMeans(4, init="k-means||", random_state=0, oversampling_factor=6, max_iter=5).fit(Xh)
    d = KMeans(4, init="k-means||", random_state=0, oversampling_factor=6, max_iter=5).fit(X)
    np.testing.assert_allclose(c.cluster_centers_, d.cluster_centers_, rtol=1e-9)


def test_metrics_operators_host_logic(monkeypatch):
    """dask_ml/metrics/pairwise.py:55-139, 172-195 on the checker backend: blocks of 256 columns, Y=None, caller-supplied
    norms, dtype promotion, rbf gamma default, the error contract (the GPU suite repeats the numerics on the device)."""
    import sklearn.metrics.pairwise as skp
    from oracle_backend import OracleBackend
    from dask_ml_b200 import ChunkedArray, metrics
    from dask_ml_b200.cluster import k_means as km

    monkeypatch.setattr(km, "_BACKEND_FACTORY", OracleBackend)
    rng = np.random.RandomState(3)
    X = rng.standard_normal((700, 9)).astype(np.float32)
    Y = rng.standard_normal((300, 9)).astype(np.float32)          # > 256 rows: two column blocks
    Xc = ChunkedArray.from_array(X, 256)
    D = metrics.euclidean_distances(Xc, Y).compute()
    assert D.dtype == np.float32 and D.shape == (700, 300)
    np.testing.assert_allclose(D, skp.euclidean_distances(X, Y), rtol=1e-4, atol=1e-4)
    D2 = metrics.euclidean_distances(Xc, Y, squared=True).compute()
    np.testing.assert_allclose(D2, skp.euclidean_distances(X, Y, squared=True), rtol=1e-4, atol=1e-3)
    # Y = None: X against itself; float64 Y promotes the result
    S = metrics.euclidean_distances(X[:100]).compute()
    np.testing.assert_allclose(S, skp.euclidean_distances(X[:100]), rtol=1e-3, atol=5e-3)
    assert metrics.euclidean_distances(X[:50], Y.astype(np.float64)).compute().dtype == np.float64
    # caller-supplied norms are USED (pairwise.py:72-91): wrong norms give the reference's (wrong) numbers
    yy = (Y.astype(np.float64) ** 2).sum(1) + 1.0
    got = metrics.euclidean_distances(X[:64], Y, Y_norm_squared=yy, squared=True).compute()
    want = skp.euclidean_distances(X[:64].astype(np.float64), Y.astype(np.float64), squared=True) + 1.0
    np.testing.assert_allclose(got, want, rtol=1e-4, atol=1e-3)
    with pytest.raises(ValueError):
        metrics.euclidean_distances(X[:10], Y, Y_norm_squared=np.ones(7))
    with pytest.raises(ValueError):
        metrics.euclidean_distances(X[:10], Y[:, :5])
    # rbf_kernel / pairwise_kernels
    K = metrics.rbf_kernel(Xc, Y).compute()
    np.testing.assert_allclose(K, skp.rbf_kernel(X, Y), rtol=1e-4, atol=1e-6)
    K2 = metrics.pairwise_kernels(X[:40], Y[:30], metric="rbf", gamma=0.3).compute()
    np.testing.assert_allclose(K2, skp.rbf_kernel(X[:40], Y[:30], gamma=0.3), rtol=1e-4, atol=1e-6)
    with pytest.raises(NotImplementedError):
        metrics.pairwise_kernels(X[:4], Y[:4], metric="polynomial")
    with pytest.raises(ValueError):
        metrics.pairwise_kernels(X[:4], Y[:4], metric="nope")
    with pytest.raises(TypeError):
        metrics.pairwise_distances(X[:4], type("A", (), {"__module__": "dask.array.core"})())
    with pytest.raises(NotImplementedError):
        metrics.pairwise_distances(X[:4], Y[:4], metric="cosine")


def test_p2p_mailbox_sizing_and_argument_checks():
    """Host-side contract of the peer-memory collective (include/bkm_b200.h): mailbox size = 1 KB header + 2 parities x
    world slots of max_elems float64; argument errors are return codes (no device needed)."""
    import ctypes
    from dask_ml_b200 import _lib

    lib = _lib.load()
    nb = ctypes.c_size_t(0)
    assert lib.bkm_p2p_mailbox_bytes(8, 1 << 16, ctypes.byref(nb)) == 0
    assert nb.value == 1024 + 2 * 8 * (1 << 16) * 8
    assert lib.bkm_p2p_mailbox_bytes(1, 1, ctypes.byref(nb)) == 0 and nb.value == 1024 + 16
    for world, m in ((0, 16), (65, 16), (2, 0)):
        assert lib.bkm_p2p_mailbox_bytes(world, m, ctypes.byref(nb)) < 0
    # n > max_elems, bad rank, null pointers: rejected before anything touches a device
    dummy = ctypes.c_void_p(16)
    assert lib.bkm_allreduce_p2p(dummy, 10, dummy, 0, 2, 5, 1, None) < 0
    assert lib.bkm_allreduce_p2p(dummy, 4, dummy, 2, 2, 5, 1, None) < 0
    assert lib.bkm_allreduce_p2p(None, 4, dummy, 0, 2, 5, 1, None) < 0
    assert lib.bkm_allreduce_p2p(dummy, 0, dummy, 0, 2, 5, 1, None) == 0          # empty payload: nothing to do
