"""PCA and TruncatedSVD without a GPU: the estimators' host logic (validation, the float64 algebra on the Gram matrix,
the sign convention, pickling, 2 ranks over gloo) on a CPU backend whose two passes are float64 numpy, against live
scikit-learn."""
import os
import pickle
import socket
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp
from sklearn import decomposition as skd

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle_backend import OracleBackend  # noqa: E402


class GramOracleBackend(OracleBackend):
    """The CPU checker backend plus the two passes of PCA / TruncatedSVD, in float64 numpy."""

    def gram_chunk(self, x, shift, colsum, gram, first=False):
        self.launches += 1
        xc = x.numpy().astype(np.float64) - shift.numpy()
        m, G = torch.from_numpy(xc.sum(0)), torch.from_numpy(xc.T @ xc)
        if first:
            colsum.copy_(m)
            gram.copy_(G)
        else:
            colsum += m
            gram += G

    def project_chunk(self, x, shift, W, out=None, colmax=None, row_offset=0):
        self.launches += 1
        xc = x.numpy().astype(np.float64)
        if shift is not None:
            xc = xc - shift.numpy()
        t = xc @ W.numpy().T
        if out is not None:
            out.copy_(torch.from_numpy(t).to(out.dtype))
        if colmax is not None and t.shape[0]:
            i = np.argmax(np.abs(t), axis=0)                  # first row on ties
            a = np.abs(t[i, np.arange(t.shape[1])])
            rows = colmax[:, 1:2].view(torch.int64)
            for j in range(t.shape[1]):
                if a[j] > colmax[j, 0].item():
                    colmax[j, 0] = float(a[j])
                    rows[j, 0] = int(row_offset + i[j])
                    colmax[j, 2] = float(t[i[j], j])

    def colmax_new(self, k):
        rec = torch.zeros((k, 4), dtype=torch.float64)
        rec[:, 0] = -1.0
        rec[:, 1:2].view(torch.int64).fill_(-1)
        return rec


@pytest.fixture
def cpu_backend(monkeypatch):
    from dask_ml_b200.cluster import k_means as km

    monkeypatch.setattr(km, "_BACKEND_FACTORY", GramOracleBackend)


def _data(n=600, d=12, seed=0, offset=0.0, dtype=np.float64):
    rng = np.random.RandomState(seed)
    A = rng.standard_normal((d, d)) * np.linspace(3, 0.2, d)[:, None]
    return (rng.standard_normal((n, d)) @ A + offset).astype(dtype)


def _chunked(X, rows):
    from dask_ml_b200 import ChunkedArray

    return ChunkedArray.from_array(X, rows)


def _np(a):
    return a.compute() if hasattr(a, "compute") else np.asarray(a)


@pytest.mark.parametrize("whiten", [False, True])
@pytest.mark.parametrize("n_components", [None, 5])
@pytest.mark.parametrize("offset", [0.0, 1e4])
def test_pca_matches_sklearn(cpu_backend, whiten, n_components, offset):
    from dask_ml_b200.decomposition import PCA

    X = _data(offset=offset)
    ref = skd.PCA(n_components=n_components, whiten=whiten, svd_solver="full").fit(X)
    got = PCA(n_components=n_components, whiten=whiten, svd_solver="full").fit(_chunked(X, 250))
    tol = 1e-9 if offset else 1e-11
    # scikit-learn >= 1.5 flips signs by V, the reference by U (test_pca_sign_convention_is_svd_flip): compare up to sign
    sgn = np.sign((got.components_ * ref.components_).sum(1))
    np.testing.assert_allclose(got.components_ * sgn[:, None], ref.components_, rtol=0, atol=tol * 1e3 if offset else tol)
    np.testing.assert_allclose(got.explained_variance_, ref.explained_variance_, rtol=tol)
    np.testing.assert_allclose(got.explained_variance_ratio_, ref.explained_variance_ratio_, rtol=tol)
    np.testing.assert_allclose(got.singular_values_, ref.singular_values_, rtol=tol)
    np.testing.assert_allclose(got.mean_, ref.mean_, rtol=1e-13)
    np.testing.assert_allclose(got.noise_variance_, ref.noise_variance_, rtol=1e-8, atol=1e-12)
    assert got.n_components_ == ref.n_components_ and got.n_samples_ == X.shape[0] and got.n_features_ == X.shape[1]
    Xt = X[:100]
    np.testing.assert_allclose(_np(got.transform(Xt)) * sgn, ref.transform(Xt), rtol=0, atol=1e-6)
    np.testing.assert_allclose(_np(got.fit_transform(_chunked(X, 250))) * sgn, ref.transform(X), rtol=0, atol=1e-6)
    T = ref.transform(Xt)
    np.testing.assert_allclose(_np(got.inverse_transform(T * sgn)), ref.inverse_transform(T), rtol=1e-8, atol=1e-6)
    np.testing.assert_allclose(got.get_covariance(), ref.get_covariance(), rtol=1e-7, atol=1e-9)
    if n_components is not None:
        np.testing.assert_allclose(_np(got.score_samples(Xt)), ref.score_samples(Xt), rtol=1e-8)
        np.testing.assert_allclose(got.score(Xt), ref.score(Xt), rtol=1e-8)


def test_pca_float32_attributes(cpu_backend):
    from dask_ml_b200.decomposition import PCA

    X = _data(dtype=np.float32)
    got = PCA(n_components=4).fit(X)
    ref = skd.PCA(n_components=4, svd_solver="full").fit(X.astype(np.float64))
    assert got.components_.dtype == np.float32 and got.explained_variance_.dtype == np.float32
    sgn = np.sign((got.components_ * ref.components_).sum(1))
    np.testing.assert_allclose(got.components_ * sgn[:, None], ref.components_, atol=1e-5)
    np.testing.assert_allclose(got.explained_variance_, ref.explained_variance_, rtol=1e-6)
    assert _np(got.transform(X)).dtype == np.float32


def test_pca_randomized_is_the_exact_top_k(cpu_backend):
    from dask_ml_b200.decomposition import PCA

    X = _data(n=800, d=20)
    got = PCA(n_components=3, svd_solver="randomized", random_state=0).fit(X)
    ref = skd.PCA(n_components=3, svd_solver="full").fit(X)
    sgn = np.sign((got.components_ * ref.components_).sum(1))
    np.testing.assert_allclose(got.components_ * sgn[:, None], ref.components_, atol=1e-10)
    np.testing.assert_allclose(got.singular_values_, ref.singular_values_, rtol=1e-11)
    total = X.var(ddof=1, axis=0).sum()
    np.testing.assert_allclose(got.explained_variance_ratio_, ref.explained_variance_ / total, rtol=1e-11)
    np.testing.assert_allclose(got.noise_variance_, (total - ref.explained_variance_.sum()) / 17, rtol=1e-10)


@pytest.mark.parametrize("algorithm", ["tsqr", "randomized"])
def test_truncated_svd_matches_sklearn(cpu_backend, algorithm):
    from dask_ml_b200.decomposition import TruncatedSVD

    X = _data(offset=3.0)
    ref = skd.TruncatedSVD(n_components=4, algorithm="arpack").fit(X)
    got = TruncatedSVD(n_components=4, algorithm=algorithm)
    T = _np(got.fit_transform(_chunked(X, 200)))
    # scikit-learn's arpack path flips signs by V (u_based_decision=False); compare up to sign, then the sign rule
    sgn = np.sign((got.components_ * ref.components_).sum(1))
    np.testing.assert_allclose(got.components_ * sgn[:, None], ref.components_, atol=1e-10)
    np.testing.assert_allclose(got.singular_values_, ref.singular_values_, rtol=1e-11)
    np.testing.assert_allclose(got.explained_variance_, ref.explained_variance_, rtol=1e-9)
    np.testing.assert_allclose(got.explained_variance_ratio_, ref.explained_variance_ratio_, rtol=1e-9)
    U = X @ got.components_.T
    i = np.argmax(np.abs(U), axis=0)
    assert (U[i, np.arange(4)] > 0).all()                      # svd_flip: the largest |U_ij| of every column is > 0
    np.testing.assert_allclose(T, U, atol=1e-9)
    np.testing.assert_allclose(_np(got.transform(X[:50])), U[:50], atol=1e-9)
    np.testing.assert_allclose(_np(got.inverse_transform(U[:50])), U[:50] @ got.components_, atol=1e-9)


def test_pca_sign_convention_is_svd_flip(cpu_backend):
    from sklearn.utils.extmath import svd_flip

    from dask_ml_b200.decomposition import PCA

    X = _data(n=300, d=6, seed=3)
    Xc = X - X.mean(0)
    U, S, V = np.linalg.svd(Xc, full_matrices=False)
    U, V = svd_flip(U, V)
    got = PCA(n_components=6, svd_solver="full").fit(_chunked(X, 70))
    np.testing.assert_allclose(got.components_, V, atol=1e-11)


def test_errors(cpu_backend):
    from dask_ml_b200.decomposition import PCA, TruncatedSVD

    X = _data(n=50, d=6)
    with pytest.raises(ValueError, match="Invalid solver 'arpack'"):
        PCA(svd_solver="arpack").fit(X)
    with pytest.raises(NotImplementedError, match="Fractional 'n_components'"):
        PCA(n_components=0.5).fit(X)
    with pytest.raises(ValueError, match=r"n_components=7 must be between 0 and min\(n_samples, n_features\)=6 with "
                                         r"svd_solver='full'"):
        PCA(n_components=7).fit(X)
    with pytest.raises(ValueError, match="n_components must be < n_features; got 6 >= 6"):
        TruncatedSVD(n_components=6).fit(X)
    with pytest.raises(ValueError):
        TruncatedSVD(algorithm="bogus").fit(X)
    Xn = X.copy()
    Xn[7, 2] = np.nan
    with pytest.raises(ValueError, match="Input contains"):
        PCA(n_components=2).fit(Xn)
    Xi = X.copy()
    Xi[40, 0] = np.inf
    with pytest.raises(ValueError, match="Input contains"):
        TruncatedSVD(n_components=2).fit(Xi)


def test_pickle_round_trip(cpu_backend):
    from dask_ml_b200.decomposition import PCA, TruncatedSVD

    X = _data()
    for est in (PCA(n_components=3, whiten=True).fit(X), TruncatedSVD(n_components=3).fit(X)):
        back = pickle.loads(pickle.dumps(est))
        np.testing.assert_array_equal(back.components_, est.components_)
        np.testing.assert_array_equal(_np(back.transform(X[:20])), _np(est.transform(X[:20])))


def test_launches_per_fit(cpu_backend):
    from dask_ml_b200.cluster import k_means as km
    from dask_ml_b200.decomposition import PCA

    X = _data()
    be = km._get_backend()
    from dask_ml_b200.engine import DeviceData

    data = DeviceData([be.to_device(b, torch.float64) for b in (X[:200], X[200:450], X[450:])], be)
    PCA(n_components=3).fit(data)
    assert be.launch_count() == 6                                  # one gram + one project call per chunk


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
        from dask_ml_b200.decomposition import PCA
        from test_decomposition_host import GramOracleBackend, _data

        km._BACKEND_FACTORY = GramOracleBackend
        X = _data(offset=50.0)
        lo, hi = (0, 170) if rank == 0 else (170, 600)
        p = PCA(n_components=4).fit(ChunkedArray.from_array(X[lo:hi], 100))
        np.savez(os.path.join(out_dir, "rank%d.npz" % rank), C=p.components_, E=p.explained_variance_, M=p.mean_,
                 N=p.noise_variance_)
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(600)
def test_two_ranks_give_identical_attributes(tmp_path, cpu_backend):
    mp.start_processes(_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True, start_method="spawn")
    r0, r1 = np.load(tmp_path / "rank0.npz"), np.load(tmp_path / "rank1.npz")
    for key in ("C", "E", "M", "N"):
        np.testing.assert_array_equal(r0[key], r1[key])
    ref = skd.PCA(n_components=4, svd_solver="full").fit(_data(offset=50.0))
    sgn = np.sign((r0["C"] * ref.components_).sum(1))
    np.testing.assert_allclose(r0["C"] * sgn[:, None], ref.components_, atol=1e-9)
    np.testing.assert_allclose(r0["E"], ref.explained_variance_, rtol=1e-10)
