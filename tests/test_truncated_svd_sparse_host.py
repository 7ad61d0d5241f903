"""TruncatedSVD on sparse X without a GPU: both regimes of the sparse fit, their host algebra, the intake and errors, and
2 ranks over gloo, on a CPU backend whose passes are float64 numpy / scipy restatements (the Gram, column and
projection passes of the existing checkers, plus the two panel products)."""
import os
import socket
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch
import torch.multiprocessing as mp
from sklearn import decomposition as skd
from sklearn.utils.validation import check_random_state

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from test_decomposition_host import GramOracleBackend  # noqa: E402
from test_glm_sparse_host import SparseOracleBackend, _csr, chunked, torch_csr  # noqa: E402


def fold_colmax(colmax, t, row_offset):
    """The arg-max epilogue on a host block t: larger |t| wins, the lower global row on ties."""
    if not t.shape[0]:
        return
    i = np.argmax(np.abs(t), axis=0)                      # first row on ties
    a = np.abs(t[i, np.arange(t.shape[1])])
    rows = colmax[:, 1:2].view(torch.int64)
    for j in range(t.shape[1]):
        if a[j] > colmax[j, 0].item():
            colmax[j, 0] = float(a[j])
            rows[j, 0] = int(row_offset + i[j])
            colmax[j, 2] = float(t[i[j], j])


class SvdOracleBackend(SparseOracleBackend, GramOracleBackend):
    """The sparse and Gram checkers plus float64 scipy restatements of the two panel products."""

    def csr_panel_chunk(self, blk, d, W, out=None, colmax=None, row_offset=0):
        self.launches += 1
        t = _csr(blk, d) @ W.numpy()
        if out is not None:
            out.copy_(torch.from_numpy(t).to(out.dtype))
        if colmax is not None:
            fold_colmax(colmax, t, row_offset)

    def csc_panel_chunk(self, csc, d, P, out, first=False):
        self.launches += 1
        colptr, rows, vals, _plan = csc
        C = sp.csc_matrix((vals.numpy().astype(np.float64), rows.numpy(), colptr.numpy()), shape=(int(P.shape[0]), d))
        Z = torch.from_numpy(np.asarray(C.T @ P.numpy()))
        out.copy_(Z) if first else out.add_(Z)


@pytest.fixture
def cpu_backend(monkeypatch):
    from dask_ml_b200.cluster import k_means as km

    monkeypatch.setattr(km, "_BACKEND_FACTORY", SvdOracleBackend)


@pytest.fixture
def low_bound(monkeypatch):
    from dask_ml_b200.decomposition import truncated_svd

    monkeypatch.setattr(truncated_svd, "SPARSE_EXACT_MAX_P", 8)


def make_sparse(n=500, p=40, density=0.15, seed=0, offset=0.0):
    rng = np.random.RandomState(seed)
    X = sp.random(n, p, density=density, format="csr", random_state=rng, data_rvs=rng.standard_normal)
    X = X @ sp.diags(np.linspace(4.0, 0.5, p))
    X.data += offset
    X[7] = 0                                              # an empty row
    X.eliminate_zeros()
    X.sort_indices()
    return X.tocsr()


def _np(a):
    return a.compute() if hasattr(a, "compute") else np.asarray(a)


def _svd(**kw):
    from dask_ml_b200.decomposition import TruncatedSVD

    return TruncatedSVD(**kw)


def restated(X, k, n_iter, seed):
    """The power iterator in numpy, with Omega from datasets._x_block: (components, singular values, U S, explained
    variance, total variance), svd_flip's signs by U."""
    from dask_ml_b200.datasets import _draw_key, _x_block

    n, p = X.shape
    l = min(max(20, k + 10), min(n, p))
    Om = _x_block(_draw_key(check_random_state(seed)), 0, p, l, np.float64)
    Q = np.linalg.qr(X @ Om)[0]
    for _ in range(n_iter):
        Q = np.linalg.qr(X @ (X.T @ Q))[0]
    Q2, R = np.linalg.qr(np.asarray(X.T @ Q))
    Ur, Sr, Vrt = np.linalg.svd(R)
    S, Ub = Sr[:k], Vrt.T[:, :k]
    V = (Q2 @ Ur[:, :k]).T
    US = Q @ (Ub * S)
    i = np.argmax(np.abs(US), axis=0)
    sg = np.where(US[i, np.arange(k)] < 0, -1.0, 1.0)
    return V * sg[:, None], S, US * sg, US.var(0), X.toarray().var(0).sum()


def _close(a, b, tol):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    assert np.linalg.norm(a - b) <= tol * max(np.linalg.norm(b), 1e-300), np.linalg.norm(a - b) / np.linalg.norm(b)


@pytest.mark.parametrize("algorithm", ["tsqr", "randomized"])
def test_exact_regime_equals_the_dense_fit(cpu_backend, algorithm):
    X = make_sparse(offset=0.3)
    s = _svd(n_components=5, algorithm=algorithm)
    T = _np(s.fit_transform(chunked(X, 170)))
    dn = _svd(n_components=5, algorithm=algorithm)
    Td = _np(dn.fit_transform(X.toarray()))
    for a in ("components_", "singular_values_", "explained_variance_", "explained_variance_ratio_"):
        _close(getattr(s, a), getattr(dn, a), 1e-10)
    _close(T, Td, 1e-10)
    _close(_np(s.transform(X)), _np(dn.transform(X.toarray())), 1e-10)
    _close(_np(s.transform(chunked(X, 90))), T, 1e-10)
    ref = skd.TruncatedSVD(n_components=5, algorithm="arpack").fit(X)
    np.testing.assert_allclose(s.singular_values_, ref.singular_values_, rtol=1e-10)
    assert s.components_.dtype == np.float64 and T.dtype == np.float64


@pytest.mark.parametrize("n_iter", [0, 2])
def test_randomized_regime_equals_the_restated_iterator(cpu_backend, low_bound, n_iter):
    X = make_sparse()
    s = _svd(n_components=4, algorithm="randomized", n_iter=n_iter, random_state=3)
    T = _np(s.fit_transform(chunked(X, 170)))
    V, S, US, ev, full = restated(X, 4, n_iter, 3)
    _close(s.components_, V, 1e-10)
    _close(s.singular_values_, S, 1e-10)
    _close(T, US, 1e-10)
    _close(s.explained_variance_, ev, 1e-10)
    _close(s.explained_variance_ratio_, ev / full, 1e-10)
    _close(_np(s.transform(X)), X @ s.components_.T, 1e-10)


def test_convergence_on_a_spectral_gap(cpu_backend, low_bound):
    rng = np.random.RandomState(5)
    n, p = 400, 120
    d = np.r_[[100.0, 80.0, 60.0, 45.0], np.linspace(1.0, 0.1, p - 4)]
    D = sp.csr_matrix((d, (rng.permutation(n)[:p], rng.permutation(p))), shape=(n, p))
    X = (D + sp.random(n, p, density=0.01, random_state=rng) * 0.01).tocsr()
    s = _svd(n_components=4, algorithm="randomized", n_iter=5, random_state=0).fit(X)
    exact = np.linalg.svd(X.toarray(), compute_uv=False)[:4]
    np.testing.assert_allclose(s.singular_values_, exact, rtol=1e-8)


def test_blocks_do_not_change_the_fit(cpu_backend, low_bound):
    X = make_sparse(seed=2)
    fits = [_svd(n_components=3, algorithm="randomized", random_state=1).fit(Xin)
            for Xin in (X, chunked(X, 500), chunked(X, 137))]
    for f in fits[1:]:
        _close(f.components_, fits[0].components_, 1e-10)
        _close(f.singular_values_, fits[0].singular_values_, 1e-10)
        _close(f.explained_variance_, fits[0].explained_variance_, 1e-10)


def test_seeds(cpu_backend, low_bound):
    X = make_sparse(seed=4)
    a = _svd(n_components=3, algorithm="randomized", n_iter=0, random_state=7).fit(X)
    b = _svd(n_components=3, algorithm="randomized", n_iter=0, random_state=7).fit(X)
    c = _svd(n_components=3, algorithm="randomized", n_iter=0, random_state=8).fit(X)
    np.testing.assert_array_equal(a.components_, b.components_)
    np.testing.assert_array_equal(a.singular_values_, b.singular_values_)
    assert not np.array_equal(a.singular_values_, c.singular_values_)


def test_rank_deficient(cpu_backend, low_bound):
    rng = np.random.RandomState(6)
    A = sp.random(300, 3, density=0.5, random_state=rng)
    B = sp.random(3, 60, density=0.5, random_state=rng)
    X = (A @ B).tocsr()                                   # rank 3 < l = 20
    X.sort_indices()
    s = _svd(n_components=5, algorithm="randomized", random_state=0).fit(X)
    np.testing.assert_allclose(s.components_ @ s.components_.T, np.eye(5), atol=1e-10)
    exact = np.linalg.svd(X.toarray(), compute_uv=False)
    np.testing.assert_allclose(s.singular_values_[:3], exact[:3], rtol=1e-10)
    assert (s.singular_values_[3:] < 1e-10 * exact[0]).all()


def test_errors(cpu_backend, monkeypatch):
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.decomposition import truncated_svd

    X = make_sparse(n=200, p=10)
    with pytest.raises(ValueError, match="n_components must be < n_features; got 10 >= 10"):
        _svd(n_components=10).fit(X)
    with pytest.raises(ValueError):
        _svd(algorithm="bogus").fit(X)
    nan = X.copy()
    nan.data[5] = np.nan
    with pytest.raises(ValueError, match="NaN, infinity"):
        _svd().fit(nan)
    bad = X[100:].copy()
    r = int(np.nonzero(np.diff(bad.indptr) >= 2)[0][0])
    k = bad.indptr[r]
    bad.indices[k], bad.indices[k + 1] = bad.indices[k + 1], bad.indices[k]
    with pytest.raises(ValueError, match="canonical CSR: the column indices of block 1"):
        _svd().fit(ChunkedArray([torch_csr(X[:100]), torch_csr(bad)]))
    with pytest.raises(TypeError, match="mixes dense and sparse"):
        _svd().fit(ChunkedArray([torch_csr(X[:100]), torch.as_tensor(X[100:].toarray())]))

    inf = X.copy()
    inf.data[3] = np.inf
    monkeypatch.setattr(truncated_svd, "SPARSE_EXACT_MAX_P", 4)
    with pytest.raises(ValueError, match="NaN, infinity"):
        _svd(algorithm="randomized").fit(inf)
    with pytest.raises(ValueError, match="bounded at 4 features.*'randomized'"):
        _svd(algorithm="tsqr").fit(X)

@pytest.mark.parametrize("vdtype", [torch.float32, torch.int32, torch.bool])
def test_intake_forms_and_dtypes(cpu_backend, vdtype):
    from dask_ml_b200 import ChunkedArray

    X = make_sparse(n=300, p=12, seed=8)
    if vdtype != torch.float32:
        X.data[:] = 1.0 if vdtype == torch.bool else np.round(np.abs(X.data)) + 1
    want = _svd(n_components=3).fit(X.toarray().astype(np.float32 if vdtype == torch.float32 else np.float64))
    vals = torch.from_numpy(X.data).to(vdtype)
    forms = [torch_csr(X, values=vals), chunked(sp.csr_matrix((vals.numpy(), X.indices, X.indptr), shape=X.shape), 70),
             ChunkedArray([torch_csr(X[i:i + 100], torch.int32, torch.from_numpy(X[i:i + 100].data).to(vdtype))
                           for i in range(0, 300, 100)])]
    if vdtype == torch.float32:
        forms += [X.astype(np.float32).tocsc(), X.astype(np.float32).tocoo()]
    dt = np.float32 if vdtype == torch.float32 else np.float64
    for Xin in forms:
        s = _svd(n_components=3)
        T = _np(s.fit_transform(Xin))
        assert s.components_.dtype == dt and s.singular_values_.dtype == dt and T.dtype == dt
        tol = 1e-5 if dt == np.float32 else 1e-10
        _close(s.components_, want.components_, tol)
        _close(s.singular_values_, want.singular_values_, tol)
        _close(T, _np(s.transform(Xin)), tol)


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
        from dask_ml_b200.cluster import k_means as km
        from dask_ml_b200.decomposition import truncated_svd
        from test_truncated_svd_sparse_host import SvdOracleBackend, _np, _svd, chunked, make_sparse

        km._BACKEND_FACTORY = SvdOracleBackend
        X = make_sparse(seed=9)
        lo, hi = (0, 180) if rank == 0 else (180, 500)
        res = {}
        for name, bound in (("exact", 4096), ("randomized", 8)):
            truncated_svd.SPARSE_EXACT_MAX_P = bound
            s = _svd(n_components=4, algorithm="randomized", random_state=2)
            T = _np(s.fit_transform(chunked(X[lo:hi], 70)))
            res[name + "_C"], res[name + "_S"], res[name + "_E"] = (s.components_, s.singular_values_,
                                                                    s.explained_variance_)
            res[name + "_T"] = T
        np.savez(os.path.join(out_dir, "rank%d.npz" % rank), **res)
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(600)
def test_two_ranks_equal_one_rank(tmp_path, cpu_backend, monkeypatch):
    from dask_ml_b200.decomposition import truncated_svd

    mp.start_processes(_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True, start_method="spawn")
    r = [np.load(tmp_path / ("rank%d.npz" % k)) for k in range(2)]
    X = make_sparse(seed=9)
    for name, bound in (("exact", 4096), ("randomized", 8)):
        for a in "CSE":
            np.testing.assert_array_equal(r[0][name + "_" + a], r[1][name + "_" + a])
        monkeypatch.setattr(truncated_svd, "SPARSE_EXACT_MAX_P", bound)
        one = _svd(n_components=4, algorithm="randomized", random_state=2)
        T = _np(one.fit_transform(X))
        _close(r[0][name + "_C"], one.components_, 1e-10)
        _close(r[0][name + "_S"], one.singular_values_, 1e-10)
        _close(r[0][name + "_E"], one.explained_variance_, 1e-10)
        _close(np.concatenate([r[0][name + "_T"], r[1][name + "_T"]]), T, 1e-10)
