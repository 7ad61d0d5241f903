"""KMeans on sparse CSR blocks on the H100: the sparse KMeans passes against scipy float64, bit-identical repeats, edge
shapes, the no-op after the loop is done, and the device fit against the CPU checker, the dense device fit and
scikit-learn (HashingVectorizer and OneHotEncoder pipelines)."""
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

pytestmark = pytest.mark.gpu


def _be():
    from dask_ml_b200.engine import CudaBackend

    return CudaBackend()


def _np(a):
    return a.compute() if hasattr(a, "compute") else np.asarray(a)


def _rand_csr(n, p, nnz_per_row, seed, dtype=np.float64, long_col=None):
    rng = np.random.RandomState(seed)
    nnz = rng.poisson(nnz_per_row, n)
    nnz[:: 7] = 0                                      # rows with no entries
    nnz = np.minimum(nnz, p)
    rows = np.repeat(np.arange(n), nnz)
    cols = np.concatenate([rng.choice(p, m, replace=False) if m else np.zeros(0, int) for m in nnz]) if n else \
        np.zeros(0, int)
    X = sp.csr_matrix((rng.standard_normal(len(rows)), (rows, cols)), shape=(n, p))
    if long_col is not None:
        X = X.tolil()
        X[np.arange(0, n, 2), long_col] = 1.5
        X = X.tocsr()
    X.sum_duplicates()
    X.sort_indices()
    return X.astype(dtype)


def _blk(X, be):
    from dask_ml_b200._sparse import _csr_block

    return _csr_block(X, be.device)


def _check_assign(X, C, k, be):
    from dask_ml_b200._sparse import _SparseData

    p = X.shape[1]
    blk = _blk(X, be)
    pack = be.sparse_pack_centers(torch.as_tensor(C).to(be.device))
    n = X.shape[0]
    lab = be.empty((n,), torch.int32)
    mn = be.empty((n,), torch.float64)
    s = be.zeros((1,), torch.float64)
    cnt = be.zeros((k,), torch.float64)
    be.csr_assign_chunk(blk, p, pack, k, labels=lab, min_dist=mn, dist_sum=s, counts=cnt, first=True)
    X64 = X.astype(np.float64)
    xn = np.asarray(X64.multiply(X64).sum(1)).ravel()
    cn = (C * C).sum(1)
    d2 = np.maximum(xn[:, None] - 2.0 * np.asarray(X64 @ C.T) + cn[None, :], 0.0)
    scale = xn[:, None] + cn.max()
    got = mn.cpu().numpy()
    assert np.all(np.abs(got - d2.min(1)) <= 1e-13 * np.maximum(scale[:, 0], 1e-300))
    L = lab.cpu().numpy()
    if n and k > 1:
        srt = np.sort(d2, axis=1)
        clear = (srt[:, 1] - srt[:, 0]) > 1e-12 * scale[:, 0]
        np.testing.assert_array_equal(L[clear], d2.argmin(1)[clear])
    np.testing.assert_array_equal(cnt.cpu().numpy(), np.bincount(L, minlength=k).astype(np.float64))
    np.testing.assert_allclose(s.item(), got.sum(), rtol=1e-12, atol=1e-300)
    # transform mode
    if n:
        out = be.empty((n, k), torch.float64)
        be.csr_assign_chunk(blk, p, pack, k, out=out, mode=2)
        assert np.all(np.abs(out.cpu().numpy() - d2) <= 1e-13 * np.maximum(scale, 1e-300))
    # the label sums against scipy
    sd = _SparseData([blk], p, be)
    csc = sd.transposes()[0]
    sumsT = be.empty((p, k), torch.float64)
    be.csc_label_sums_chunk(csc, p, lab, k, sumsT, first=True)
    onehot = sp.csr_matrix((np.ones(n), L.astype(np.int64), np.arange(n + 1)), shape=(n, k))
    ref = np.asarray((X64.T @ onehot).todense())
    bound = np.asarray(abs(X64).sum(0)).ravel()[:, None]
    assert np.all(np.abs(sumsT.cpu().numpy() - ref) <= 1e-12 * np.maximum(bound, 1e-300))
    return lab, mn, s, cnt, sumsT, blk, csc, pack


@pytest.mark.parametrize("k", [1, 31, 33, 257, 1000])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_passes_against_scipy(k, dtype):
    be = _be()
    X = _rand_csr(3000, 300, 12, k, dtype, long_col=17 if k == 33 else None)
    C = np.random.RandomState(k).standard_normal((k, 300))
    r1 = _check_assign(X, C, k, be)
    r2 = _check_assign(X, C, k, be)
    for a, b in zip(r1[:5], r2[:5]):
        assert torch.equal(a, b)                        # bit-identical repeats


def test_long_column_segment_fold():
    be = _be()
    X = _rand_csr(9000, 64, 3, 1, long_col=5)            # column 5 holds 4500 entries: three segments
    assert np.diff(X.tocsc().indptr)[5] > 2048
    C = np.random.RandomState(0).standard_normal((40, 64))
    _check_assign(X, C, 40, be)


def test_wide_p_and_p_one():
    be = _be()
    X = _rand_csr(500, 1 << 20, 30, 3)
    C = np.zeros((7, 1 << 20))
    rng = np.random.RandomState(1)
    C[:, rng.choice(1 << 20, 5000, replace=False)] = rng.standard_normal((7, 5000))
    C[:, X.indices[:200]] = rng.standard_normal((7, 200))
    _check_assign(X, C, 7, be)
    X1 = _rand_csr(400, 1, 1, 4)
    _check_assign(X1, np.array([[0.3], [-1.0]]), 2, be)


def test_empty_block_writes_zeros_on_first():
    be = _be()
    X = sp.csr_matrix((0, 20))
    blk = _blk(X, be)
    pack = be.sparse_pack_centers(torch.ones((3, 20), dtype=torch.float64, device=be.device))
    s = torch.full((1,), 5.0, dtype=torch.float64, device=be.device)
    cnt = torch.full((3,), 5.0, dtype=torch.float64, device=be.device)
    be.csr_assign_chunk(blk, 20, pack, 3, dist_sum=s, counts=cnt, first=True)
    assert s.item() == 0.0 and cnt.sum().item() == 0.0


def test_noop_after_done():
    be = _be()
    X = _rand_csr(1000, 50, 8, 2)
    C = np.random.RandomState(2).standard_normal((5, 50))
    from dask_ml_b200._sparse import _SparseData

    blk = _blk(X, be)
    csc = _SparseData([blk], 50, be).transposes()[0]
    pack = be.sparse_pack_centers(torch.as_tensor(C).to(be.device))
    state, _ = be.loop_state_new(1e300, 10)          # every shift is below tol: the first step stops the loop
    red = be.zeros((50 * 5 + 5 + 1,), torch.float64)
    lab = be.empty((1000,), torch.int32)
    be.csr_assign_chunk(blk, 50, pack, 5, labels=lab, counts=red[250:255], first=True, loop_state=state)
    be.csc_label_sums_chunk(csc, 50, lab, 5, red[:250].view(50, 5), first=True, loop_state=state)
    out = torch.full_like(pack, -7.0)
    be.sparse_finalize_step(red, pack, out, state, 5, 50)
    done, n_iter, _ = be.loop_state_read(state)
    assert (done, n_iter) == (1, 1)
    lab.fill_(-3)
    red.fill_(-3.0)
    out.fill_(-3.0)
    be.csr_assign_chunk(blk, 50, pack, 5, labels=lab, counts=red[250:255], first=True, loop_state=state)
    be.csc_label_sums_chunk(csc, 50, lab, 5, red[:250].view(50, 5), first=True, loop_state=state)
    be.sparse_finalize_step(red, pack, out, state, 5, 50)
    assert (lab == -3).all() and (red == -3.0).all() and (out == -3.0).all()
    assert be.loop_state_read(state)[:2] == (1, 1)


def _blobs(n, p, k, seed):
    rng = np.random.RandomState(seed)
    lab = rng.randint(0, k, n)
    cols = np.array_split(np.arange(p), k)
    X = sp.lil_matrix((n, p))
    for i in range(n):
        c = cols[lab[i]]
        use = c[rng.rand(len(c)) < 0.6]
        X[i, use] = 3.0 + 0.2 * rng.standard_normal(len(use))
        X[i, rng.randint(0, p)] = 0.1
    return X.tocsr()


def test_device_fit_against_checker_and_dense():
    from dask_ml_b200.cluster import KMeans, k_means as km
    from test_glm_sparse_host import chunked
    from test_kmeans_sparse_host import KMeansSparseOracleBackend

    X = _blobs(3000, 80, 6, 0)
    C0 = X[[0, 1, 2, 3, 4, 5]].toarray()
    dev = KMeans(n_clusters=6, init=C0, tol=1e-10, max_iter=60).fit(chunked(X, 700))
    assert dev.labels_.blocks[0].is_cuda
    saved = km._BACKEND_FACTORY
    km._BACKEND_FACTORY = KMeansSparseOracleBackend
    try:
        cpu = KMeans(n_clusters=6, init=C0, tol=1e-10, max_iter=60).fit(chunked(X, 700))
    finally:
        km._BACKEND_FACTORY = saved
    np.testing.assert_array_equal(_np(dev.labels_), _np(cpu.labels_))
    np.testing.assert_allclose(dev.cluster_centers_, cpu.cluster_centers_, rtol=0, atol=1e-12)
    dense = KMeans(n_clusters=6, init=C0, tol=1e-10, max_iter=60).fit(X.toarray())
    np.testing.assert_array_equal(_np(dev.labels_), _np(dense.labels_))
    np.testing.assert_allclose(dev.cluster_centers_, dense.cluster_centers_, rtol=0, atol=1e-12)
    assert dev.n_iter_ == dense.n_iter_
    T = dev.transform(chunked(X, 700))
    assert T.blocks[0].is_cuda
    np.testing.assert_allclose(_np(T), _np(dense.transform(X.toarray())), rtol=1e-10, atol=1e-10)
    np.testing.assert_array_equal(_np(dev.predict(X)), _np(dense.labels_))
    kp = KMeans(n_clusters=6, random_state=0).fit(chunked(X, 700))          # k-means||
    kd = KMeans(n_clusters=6, random_state=0).fit(X.toarray())
    np.testing.assert_allclose(kp.cluster_centers_, kd.cluster_centers_, rtol=0, atol=1e-10)


def test_hashing_vectorizer_pipeline():
    from sklearn.cluster import KMeans as SkKMeans
    from sklearn.feature_extraction.text import HashingVectorizer as SkHV

    from dask_ml_b200.cluster import KMeans
    from dask_ml_b200.feature_extraction.text import HashingVectorizer
    from test_text_host import chunked as docs_chunked

    rng = np.random.RandomState(0)
    topics = [["gpu", "kernel", "warp", "memory", "cuda"], ["cat", "dog", "bird", "fish", "horse"],
              ["red", "green", "blue", "yellow", "black"]]
    docs = [" ".join(rng.choice(topics[i % 3], 6)) for i in range(600)]
    hv = HashingVectorizer(n_features=1 << 12)
    Xd = hv.transform(docs_chunked(docs, 4))
    Xs = SkHV(n_features=1 << 12).transform(docs)
    C0 = Xs[[0, 1, 2]].toarray()
    a = KMeans(n_clusters=3, init=C0, tol=0.0, max_iter=50).fit(Xd)
    s = SkKMeans(n_clusters=3, init=C0, n_init=1, algorithm="lloyd", tol=0.0, max_iter=50).fit(Xs)
    np.testing.assert_array_equal(_np(a.labels_), s.labels_)
    np.testing.assert_allclose(a.cluster_centers_, s.cluster_centers_, rtol=0, atol=1e-10)


def test_onehot_pipeline():
    from sklearn.cluster import KMeans as SkKMeans
    from sklearn.preprocessing import OneHotEncoder as SkOHE

    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.cluster import KMeans
    from dask_ml_b200.preprocessing import OneHotEncoder

    rng = np.random.RandomState(1)
    grp = rng.randint(0, 4, 2000)
    Z = np.stack([grp * 3 + rng.randint(0, 2, 2000), grp * 2 + rng.randint(0, 2, 2000), rng.randint(0, 3, 2000)], 1)
    Zc = ChunkedArray([torch.from_numpy(Z[i:i + 500]).cuda() for i in range(0, 2000, 500)])
    Xd = OneHotEncoder(sparse=True).fit(Zc).transform(Zc)
    Xs = SkOHE().fit_transform(Z)
    C0 = Xs[[0, 1, 2, 3]].toarray()
    a = KMeans(n_clusters=4, init=C0, tol=0.0, max_iter=50).fit(Xd)
    s = SkKMeans(n_clusters=4, init=C0, n_init=1, algorithm="lloyd", tol=0.0, max_iter=50).fit(Xs)
    np.testing.assert_array_equal(_np(a.labels_), s.labels_)
    np.testing.assert_allclose(a.cluster_centers_, s.cluster_centers_, rtol=0, atol=1e-10)
