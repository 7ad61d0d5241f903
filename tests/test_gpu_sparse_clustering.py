"""PartialMiniBatchKMeans, SpectralClustering and rbf_kernel on sparse CSR blocks on the H100: the sparse Nystrom passes
and the sparse mini-batch step against scipy / numpy float64, bit-identical repeats and edge shapes, the estimators
against the CPU checker, and the HashingVectorizer and OneHotEncoder pipelines against scikit-learn and the dense fit."""
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

pytestmark = [pytest.mark.gpu,
              pytest.mark.filterwarnings("ignore:'PartialMiniBatchKMeans' is deprecated:FutureWarning")]


def _be():
    from dask_ml_b200.engine import CudaBackend

    return CudaBackend()


def _np(a):
    return a.compute() if hasattr(a, "compute") else np.asarray(a)


def _rand_csr(n, p, nnz_per_row, seed, dtype=np.float64):
    from test_gpu_kmeans_sparse import _rand_csr as rc

    return rc(n, p, nnz_per_row, seed, dtype)


def _blk(X, be):
    from dask_ml_b200._sparse import _csr_block

    return _csr_block(X, be.device)


def _d2(X, C):
    X = X.astype(np.float64)
    xn = np.asarray(X.multiply(X).sum(1)).ravel()
    return np.maximum(xn[:, None] - 2.0 * np.asarray(X @ C.T) + (C * C).sum(1)[None, :], 0.0)


def _pack(be, C):
    return be.sparse_pack_centers(torch.as_tensor(np.ascontiguousarray(C)).to(be.device))


@pytest.mark.parametrize("l", [1, 31, 32, 33, 128, 129, 300])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_colsum_and_embed_against_scipy(l, dtype):
    be = _be()
    p = 90
    X = _rand_csr(700, p, 6, l, dtype)
    rng = np.random.RandomState(l)
    C = 0.3 * rng.standard_normal((l, p))
    gamma = 0.2
    pack = _pack(be, C)
    blk = _blk(X, be)
    d2 = _d2(X, C)
    # colsum: FIRST overwrites, then accumulates
    c = torch.full((l,), 7.0, dtype=torch.float64, device=be.device)
    be.csr_kernel_colsum(blk, p, pack, l, gamma, c, first=True)
    ref = np.exp(-gamma * d2).sum(0)
    np.testing.assert_allclose(c.cpu().numpy(), ref, rtol=1e-12)
    c1 = c.clone()
    be.csr_kernel_colsum(blk, p, pack, l, gamma, c, first=False)
    np.testing.assert_allclose(c.cpu().numpy(), 2 * ref, rtol=1e-12)
    be.csr_kernel_colsum(blk, p, pack, l, gamma, c, first=True)
    assert torch.equal(c, c1)                                     # repeats give the same bits
    # embed, k up to 65, float32 and float64 output with a padded pitch
    for k in sorted({1, min(l, 8), min(l, 65)}):
        W = rng.standard_normal((l, k))
        Wd = torch.as_tensor(W).to(be.device)
        m = d2.min(1, keepdims=True)
        e = np.exp(-gamma * (d2 - m)) @ W
        want = e / np.sqrt((e * e).sum(1, keepdims=True))
        for odt, tol in ((torch.float64, 1e-10), (torch.float32, 1e-5)):
            out = torch.zeros((X.shape[0], k + 3), dtype=odt, device=be.device)[:, :k]
            be.csr_nystrom_embed(blk, p, pack, l, gamma, Wd, out)
            np.testing.assert_allclose(out.cpu().numpy(), want, rtol=tol, atol=tol)
            again = torch.zeros_like(out)
            be.csr_nystrom_embed(blk, p, pack, l, gamma, Wd, again)
            assert torch.equal(out, again)


def test_empty_block_and_nan_rule():
    be = _be()
    p, l = 20, 40
    rng = np.random.RandomState(0)
    C = rng.standard_normal((l, p))
    pack = _pack(be, C)
    c = torch.full((l,), 3.0, dtype=torch.float64, device=be.device)
    empty = _blk(sp.csr_matrix((0, p)), be)
    be.csr_kernel_colsum(empty, p, pack, l, 0.5, c, first=True)
    assert (c == 0).all()
    # rows at squared distance m from the nearest keep row: gamma m just inside / beyond 745.13
    cn = (C * C).sum(1)
    near = np.zeros((2, p))                     # two empty rows: d2_j = ||c_j||^2, m = min_j ||c_j||^2
    X = sp.csr_matrix(near)
    m = cn.min()
    W = torch.as_tensor(rng.standard_normal((l, 4))).to(be.device)
    for g, nan in ((745.12 / m, False), (745.14 / m, True)):
        out = torch.empty((2, 4), dtype=torch.float64, device=be.device)
        be.csr_nystrom_embed(_blk(X, be), p, pack, l, g, W, out)
        assert torch.isnan(out).all().item() == nan and (torch.isfinite(out).all().item() != nan)


def test_minibatch_step_against_numpy():
    be = _be()
    p, k = 300, 37
    rng = np.random.RandomState(3)
    C = rng.standard_normal((k, p))
    w = rng.randint(0, 50, k).astype(np.float64)
    red = np.concatenate([rng.standard_normal(p * k), rng.randint(0, 5, k).astype(np.float64), [1.0]])
    red_d = torch.as_tensor(red).to(be.device)
    pin = _pack(be, C)
    w_in = torch.as_tensor(w).to(be.device)
    pout = torch.empty_like(pin)
    w_out = torch.empty_like(w_in)
    be.sparse_minibatch_step(red_d, pin, w_in, pout, w_out, k, p)
    S, n = red[: p * k].reshape(p, k), red[p * k: p * k + k]
    CT = C.T
    with np.errstate(divide="ignore", invalid="ignore"):
        upd = (CT * w[None, :] + S) * (1.0 / (w + n))[None, :]
    CT2 = np.where((n > 0)[None, :], upd, CT)
    got = pout.cpu().numpy()
    np.testing.assert_array_equal(got[: p * k], CT2.ravel())
    np.testing.assert_allclose(got[p * k:], (CT2 * CT2).sum(0), rtol=1e-14)      # another order of 300 terms
    np.testing.assert_array_equal(w_out.cpu().numpy(), w + n)


def _checker():
    from test_sparse_clustering_host import SparseClusteringChecker

    return SparseClusteringChecker


def _on_checker(fn):
    from dask_ml_b200.cluster import k_means as km

    saved = km._BACKEND_FACTORY
    km._BACKEND_FACTORY = _checker()
    try:
        return fn()
    finally:
        km._BACKEND_FACTORY = saved


def test_estimators_against_the_checker():
    from dask_ml_b200.cluster import PartialMiniBatchKMeans, SpectralClustering
    from dask_ml_b200.metrics import rbf_kernel
    from test_glm_sparse_host import chunked
    from test_kmeans_sparse_host import blobs
    from test_spectral_host import Recorder
    import spectral_oracle as so

    X = blobs(n=1500, p=60, k=4, seed=1)

    def mb():
        np.random.seed(2)
        return PartialMiniBatchKMeans(n_clusters=4, random_state=0, reassignment_ratio=0.3).fit(chunked(X, 300))

    a, b = mb(), _on_checker(mb)
    np.testing.assert_allclose(a.cluster_centers_, b.cluster_centers_, rtol=1e-12, atol=1e-12)
    np.testing.assert_array_equal(a._counts, b._counts)
    np.testing.assert_array_equal(_np(a.labels_), _np(b.labels_))
    np.testing.assert_allclose(a.inertia_, b.inertia_, rtol=1e-12)
    assert a.labels_.blocks[0].is_cuda

    def sc():
        rec = Recorder()
        s = SpectralClustering(n_clusters=4, n_components=50, gamma=0.05, random_state=3, assign_labels=rec)
        s.fit(chunked(X, 400))
        return s, rec.X_

    (sa, ua), (sb, ub) = sc(), _on_checker(sc)
    np.testing.assert_allclose(sa.eigenvalues_, sb.eigenvalues_, rtol=1e-12)
    assert so.procrustes_err(ua, ub) < 1e-10
    Y = np.random.RandomState(0).standard_normal((7, X.shape[1]))
    K = rbf_kernel(chunked(X, 500), Y, gamma=0.05)
    assert K.blocks[0].is_cuda
    from sklearn.metrics.pairwise import rbf_kernel as sk_rbf

    np.testing.assert_allclose(_np(K), sk_rbf(X, Y, gamma=0.05), rtol=1e-12, atol=1e-15)


def test_hashing_vectorizer_into_minibatch_kmeans():
    from sklearn.cluster import MiniBatchKMeans
    from sklearn.feature_extraction.text import HashingVectorizer as SkHV

    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.cluster import PartialMiniBatchKMeans
    from dask_ml_b200.feature_extraction.text import HashingVectorizer
    from test_text_host import chunked as docs_chunked

    rng = np.random.RandomState(0)
    topics = [["gpu", "kernel", "warp", "memory", "cuda"], ["cat", "dog", "bird", "fish", "horse"],
              ["red", "green", "blue", "yellow", "black"]]
    docs = [" ".join(rng.choice(topics[i % 3], 6)) for i in range(1200)]
    Xd = HashingVectorizer(n_features=1 << 12).transform(docs_chunked(docs, 300))   # 4 blocks of 300 rows
    Xs = SkHV(n_features=1 << 12).transform(docs)
    a = PartialMiniBatchKMeans(n_clusters=3, random_state=0, batch_size=300)
    s = MiniBatchKMeans(n_clusters=3, random_state=0, batch_size=300, n_init=1)
    assert [int(b.shape[0]) for b in Xd.blocks] == [300] * 4
    for i in range(4):
        a.partial_fit(ChunkedArray([Xd.blocks[i]]))
        s.partial_fit(Xs[i * 300:(i + 1) * 300])
        np.testing.assert_allclose(a.cluster_centers_, s.cluster_centers_, rtol=1e-12, atol=1e-12)
        np.testing.assert_array_equal(a._counts, s._counts)
        np.testing.assert_array_equal(_np(a.labels_), s.labels_)


def test_onehot_into_spectral_clustering():
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.cluster import SpectralClustering
    from dask_ml_b200.preprocessing import OneHotEncoder

    rng = np.random.RandomState(1)
    grp = rng.randint(0, 3, 2000)
    Z = np.stack([grp * 3 + rng.randint(0, 2, 2000), grp * 2 + rng.randint(0, 2, 2000), grp], 1)
    Zc = ChunkedArray([torch.from_numpy(Z[i:i + 500]).cuda() for i in range(0, 2000, 500)])
    Xd = OneHotEncoder(sparse=True).fit(Zc).transform(Zc)
    dense = np.concatenate([b.to_dense().cpu().numpy() for b in Xd.blocks]).astype(np.float64)
    kw = dict(n_clusters=3, n_components=60, gamma=0.5, random_state=0)
    a = SpectralClustering(**kw).fit(Xd)
    b = SpectralClustering(**kw).fit(dense)
    np.testing.assert_allclose(a.eigenvalues_, b.eigenvalues_, rtol=1e-10)
    la, lb = _np(a.labels_), _np(b.labels_)
    # the same partition (label ids may be permuted by the dense fp32/fp64 engine's KMeans)
    pairs = set(zip(la.tolist(), lb.tolist()))
    assert len(pairs) == 3
