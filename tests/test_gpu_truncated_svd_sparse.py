"""TruncatedSVD on sparse X on the H100: the two panel products against float64 scipy for float32 and float64 values
(l from 1 to 266, the edge shapes of the linear models' sparse passes), the arg-max epilogue and its ties, bit-identical
repeats, the device fit against the CPU checker and the dense fit, and the pipelines that feed it."""
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_gpu_glm_sparse import device_blk, rand_csr  # noqa: E402
from test_glm_sparse_host import torch_csr  # noqa: E402
from test_truncated_svd_sparse_host import SvdOracleBackend, make_sparse  # noqa: E402

pytestmark = pytest.mark.gpu

LS = [1, 20, 32, 33, 110, 266]


@pytest.fixture(scope="module")
def be():
    from dask_ml_b200.engine import CudaBackend

    return CudaBackend()


def _np(a):
    return a.compute() if hasattr(a, "compute") else np.asarray(a)


def run_panels(be, blk, csc, p, W, P, row_offset):
    n, l = blk[3], int(W.shape[1])
    dev = be.device
    o64 = torch.full((n, l + 3), 7.0, dtype=torch.float64, device=dev)[:, :l]      # a row pitch above l
    o32 = torch.full((n, l), 7.0, dtype=torch.float32, device=dev)
    rec = be.colmax_new(l)
    be.csr_panel_chunk(blk, p, W, out=o64, colmax=rec, row_offset=row_offset)
    be.csr_panel_chunk(blk, p, W, out=o32)
    rec2 = be.colmax_new(l)
    be.csr_panel_chunk(blk, p, W, colmax=rec2, row_offset=row_offset)             # the epilogue alone
    Z = torch.full((p, l), 7.0, dtype=torch.float64, device=dev)
    be.csc_panel_chunk(csc, p, P, Z, first=True)
    Z2 = Z.clone()
    be.csc_panel_chunk(csc, p, P, Z2)                                               # accumulated
    torch.cuda.synchronize()
    return [t.cpu().numpy() for t in (o64, o32, rec, rec2, Z, Z2)]


def check(be, m, l, seed=1, row_offset=11):
    n, p = m.shape
    rng = np.random.RandomState(seed)
    W, P = rng.standard_normal((p, l)), rng.standard_normal((n, l))
    blk = device_blk(be, m)
    csc = be.csr_transpose_chunk(blk, p)
    Wd, Pd = torch.as_tensor(W).to(be.device), torch.as_tensor(P).to(be.device)
    got = run_panels(be, blk, csc, p, Wd, Pd, row_offset)
    o64, o32, rec, rec2, Z, Z2 = got
    X = m.astype(np.float64)
    A = abs(X)
    assert (np.abs(o64 - X @ W) <= 1e-13 * (A @ np.abs(W)) + 1e-300).all()
    np.testing.assert_array_equal(o32, o64.astype(np.float32))
    XtP = np.asarray(X.T @ P)
    bound = 1e-13 * np.asarray(A.T @ np.abs(P)) + 1e-300
    assert (np.abs(Z - XtP) <= bound).all()
    assert (np.abs(Z2 - 2 * XtP) <= 2 * bound).all()
    if n:
        i = np.argmax(np.abs(o64), axis=0)                                          # lowest row on ties
        a = np.abs(o64[i, np.arange(l)])
        np.testing.assert_array_equal(rec[:, 0], a)
        np.testing.assert_array_equal(rec[:, 1:2].view(np.int64)[:, 0], i + row_offset)
        np.testing.assert_array_equal(rec[:, 2], o64[i, np.arange(l)])
        np.testing.assert_array_equal(rec, rec2)
    again = run_panels(be, blk, csc, p, Wd, Pd, row_offset)
    for a1, a2 in zip(got, again):
        np.testing.assert_array_equal(a1, a2)                                       # bit-identical repeat


@pytest.mark.parametrize("dt", ["f32", "f64"])
@pytest.mark.parametrize("l", LS)
@pytest.mark.parametrize("n,p,density", [(1, 5, 0.6), (3000, 700, 0.05), (2000, 50, 0.6)])
def test_panels_against_scipy(be, dt, l, n, p, density):
    check(be, rand_csr(n, p, density, dt, seed=n + p + l), l)


@pytest.mark.parametrize("dt", ["f32", "f64"])
@pytest.mark.parametrize("l", [1, 33, 266])
def test_edge_shapes(be, dt, l):
    check(be, sp.csr_matrix((5, 9), dtype=np.float32 if dt == "f32" else np.float64), l)      # nnz = 0
    m = rand_csr(1000, 30, 0.2, dt, seed=2)
    m[100:400] = 0                                                                           # empty rows
    m.eliminate_zeros()
    check(be, m, l)
    if l < 266:                                                                              # W of 2^20 x 266 is 2 GB
        check(be, rand_csr(20000, 1 << 20, 3e-5, dt, seed=3), l)                            # p = 2^20
    check(be, rand_csr(60000, 16, 0.02, dt, seed=4, heavy=[0, 9]), l)                        # a column in every row


def test_colmax_ties_take_the_lowest_row(be):
    m = rand_csr(300, 20, 0.3, "f64", seed=5)
    check(be, sp.vstack([m, m, m]).tocsr(), 7, row_offset=1000)                 # every maximum appears three times


def _fit(X, **kw):
    from dask_ml_b200.decomposition import TruncatedSVD

    s = TruncatedSVD(**kw)
    T = _np(s.fit_transform(X))
    return s, T


def _close(a, b, tol):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    assert np.linalg.norm(a - b) <= tol * max(np.linalg.norm(b), 1e-300), np.linalg.norm(a - b) / np.linalg.norm(b)


@pytest.mark.parametrize("bound", [4096, 64])
def test_device_fit_matches_checker(monkeypatch, bound):
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.cluster import k_means as km
    from dask_ml_b200.decomposition import truncated_svd

    monkeypatch.setattr(truncated_svd, "SPARSE_EXACT_MAX_P", bound)                # exact, then randomized
    X = make_sparse(n=6000, p=300, density=0.05, seed=11)
    sizes = [0, 1, 1000, 37, 2962, 2000]
    off = np.cumsum([0] + sizes)
    blocks = ChunkedArray([torch_csr(X[off[i]:off[i + 1]]).cuda() for i in range(len(sizes))])
    kw = dict(n_components=8, algorithm="randomized", n_iter=4, random_state=5)
    s, T = _fit(blocks, **kw)
    monkeypatch.setattr(km, "_BACKEND_FACTORY", SvdOracleBackend)
    c, Tc = _fit(X, **kw)
    for a in ("components_", "singular_values_", "explained_variance_", "explained_variance_ratio_"):
        _close(getattr(s, a), getattr(c, a), 1e-9)
    _close(T, Tc, 1e-9)
    assert [int(b.shape[0]) for b in s.transform(blocks).blocks] == sizes


def test_exact_regime_matches_dense_device_fit():
    X = make_sparse(n=20000, p=200, density=0.05, seed=12, offset=0.5)
    s, T = _fit(X, n_components=6)
    d, Td = _fit(X.toarray(), n_components=6)
    for a in ("components_", "singular_values_", "explained_variance_", "explained_variance_ratio_"):
        _close(getattr(s, a), getattr(d, a), 1e-9)
    _close(T, Td, 1e-9)


def test_hashed_text_to_kmeans():
    from dask_ml_b200.cluster import KMeans
    from dask_ml_b200.feature_extraction import HashingVectorizer
    from test_text_host import chunked, word_docs

    docs = word_docs(3000, seed=13, vocab=400)
    X = HashingVectorizer().transform(chunked(docs, 700))                          # 2^20 features: randomized
    svd, T = _fit(X, n_components=100, algorithm="randomized", random_state=0)
    assert T.shape == (3000, 100) and svd.components_.shape == (100, 1 << 20)
    np.testing.assert_allclose(svd.components_ @ svd.components_.T, np.eye(100), atol=1e-10)
    assert (np.diff(svd.singular_values_) <= 0).all() and svd.singular_values_[-1] > 0
    Xh = X.compute()
    _close(_np(svd.transform(X)), Xh @ svd.components_.T, 1e-10)   # X V^T; fit_transform returns U S = Q Q^T X V^T
    top = np.sort(np.linalg.svd(Xh[:, np.unique(Xh.indices)].toarray(), compute_uv=False))[::-1][:5]
    np.testing.assert_allclose(svd.singular_values_[:5], top, rtol=1e-2)      # gaps of ~5 %: n_iter=5 is close
    km = KMeans(n_clusters=5, random_state=0).fit(svd.transform(X))
    assert _np(km.labels_).shape == (3000,)


def test_one_hot_to_truncated_svd():
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.preprocessing import OneHotEncoder

    rng = np.random.RandomState(14)
    Xc = torch.as_tensor(rng.randint(0, 12, (100000, 4))).cuda()
    Xcc = ChunkedArray([Xc[i:i + 30000] for i in range(0, 100000, 30000)])
    Xs = OneHotEncoder(sparse=True).fit_transform(Xcc)
    Xd = OneHotEncoder(sparse=False).fit_transform(Xcc)
    s, T = _fit(Xs, n_components=5)
    d, Td = _fit(Xd, n_components=5)
    _close(s.singular_values_, d.singular_values_, 1e-9)                         # the spectrum has repeated values
    assert T.shape == Td.shape == (100000, 5)
