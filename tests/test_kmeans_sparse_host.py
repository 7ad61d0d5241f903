"""KMeans on sparse X without a GPU: the sparse Lloyd loop, the three inits, predict / transform and the intake, on a
CPU backend whose sparse passes are float64 scipy restatements of bkm_csr_assign_chunk, bkm_csc_label_sums_chunk and the
sparse pack, checked against the dense checker fit of X.toarray() and scikit-learn; and 2 ranks over gloo."""
import os
import socket
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch
import torch.multiprocessing as mp
from sklearn.cluster import KMeans as SkKMeans

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from test_glm_sparse_host import _csr, chunked, torch_csr  # noqa: E402
from test_glm_sparse_host import SparseOracleBackend as _Sparse  # noqa: E402
from oracle_backend import OracleBackend  # noqa: E402


class KMeansSparseOracleBackend(OracleBackend):
    """The KMeans checker plus the block transpose and float64 scipy restatements of the sparse KMeans passes."""

    csr_transpose_chunk = _Sparse.csr_transpose_chunk

    def sparse_pack_centers(self, C64, out=None):
        C = C64.to(torch.float64)
        pack = torch.cat([C.t().reshape(-1), (C * C).sum(1)])
        if out is not None:
            out.copy_(pack)
            return out
        return pack

    @staticmethod
    def _unpack(pack, k, d):
        return pack[: d * k].view(d, k).numpy(), pack[d * k:].numpy()

    def csr_assign_chunk(self, blk, d, pack, k, labels=None, min_dist=None, squared=True, dist_sum=None, counts=None,
                         out=None, mode=0, first=False, loop_state=None):
        self.launches += 1
        X = _csr(blk, d)
        CT, cn = self._unpack(pack, k, d)
        xn = np.asarray(X.multiply(X).sum(1)).ravel()
        d2 = np.maximum(xn[:, None] - 2.0 * np.asarray(X @ CT) + cn[None, :], 0.0)
        if mode:
            out.copy_(torch.from_numpy(d2 if mode == 2 else np.sqrt(d2)).to(out.dtype))
            return
        lab = np.argmin(d2, axis=1) if k else np.zeros(0, np.int64)
        mn = d2[np.arange(len(lab)), lab]
        mn = mn if squared else np.sqrt(mn)
        if labels is not None:
            labels.copy_(torch.from_numpy(lab.astype(np.int32)))
        if min_dist is not None:
            min_dist.copy_(torch.from_numpy(mn))
        if dist_sum is not None:
            v = float(mn.sum())
            dist_sum.fill_(v) if first else dist_sum.add_(v)
        if counts is not None:
            c = torch.from_numpy(np.bincount(lab, minlength=k).astype(np.float64))
            counts.copy_(c) if first else counts.add_(c)

    def csc_label_sums_chunk(self, csc, d, labels, k, sumsT, first=False, loop_state=None):
        self.launches += 1
        colptr, rows, vals, _plan = csc
        n = int(labels.numel())
        C = sp.csc_matrix((vals.numpy().astype(np.float64), rows.numpy(), colptr.numpy()), shape=(n, d))
        onehot = sp.csr_matrix((np.ones(n), labels.numpy().astype(np.int64), np.arange(n + 1)), shape=(n, k))
        S = torch.from_numpy(np.asarray((C.T @ onehot).todense()))
        sumsT.copy_(S) if first else sumsT.add_(S)

    def sparse_finalize(self, red, pack_in, pack_out, shift, k, d):
        sumsT = red[: d * k].view(d, k)
        cnt = torch.clamp(red[d * k: d * k + k], min=1.0)
        CT = sumsT / cnt[None, :]
        pack_out.copy_(torch.cat([CT.reshape(-1), (CT * CT).sum(0)]))
        shift.copy_(((pack_in[: d * k].view(d, k) - CT) ** 2).sum().reshape(1))


@pytest.fixture
def cpu_backend(monkeypatch):
    from dask_ml_b200.cluster import k_means as km

    monkeypatch.setattr(km, "_BACKEND_FACTORY", KMeansSparseOracleBackend)


def blobs(n=400, p=30, k=4, seed=0, density=0.3, spread=0.15):
    """Sparse rows around k sparse centres (each centre on its own columns), one empty row."""
    rng = np.random.RandomState(seed)
    lab = rng.randint(0, k, n)
    cols = np.array_split(np.arange(p), k)
    rows, cs, vs = [], [], []
    for i in range(n):
        if i == 5:
            continue
        c = cols[lab[i]]
        sel = c[rng.rand(len(c)) < max(density, 0.5)]
        noise = rng.choice(p, max(1, int(density * p / 4)), replace=False)
        use = np.union1d(sel, noise)
        v = np.where(np.isin(use, c), 3.0 + spread * rng.standard_normal(len(use)), spread * rng.standard_normal(len(use)))
        rows += [i] * len(use)
        cs += list(use)
        vs += list(v)
    X = sp.csr_matrix((vs, (rows, cs)), shape=(n, p))
    X.sort_indices()
    return X


def _np(a):
    return a.compute() if hasattr(a, "compute") else np.asarray(a)


def _km(**kw):
    from dask_ml_b200.cluster import KMeans

    return KMeans(**kw)


def _dense_fit(X, **kw):
    return _km(**kw).fit(X.toarray())


@pytest.mark.parametrize("init", ["array", "random"])
def test_fit_equals_the_dense_fit(cpu_backend, init):
    X = blobs()
    C0 = X[[0, 1, 2, 3]].toarray() if init == "array" else "random"
    kw = dict(n_clusters=4, init=C0, random_state=3, tol=1e-8, max_iter=50)
    a = _km(**kw).fit(chunked(X, 130))
    b = _dense_fit(X, **kw)
    np.testing.assert_array_equal(_np(a.labels_), _np(b.labels_))
    np.testing.assert_allclose(a.cluster_centers_, b.cluster_centers_, rtol=0, atol=1e-12)
    assert a.n_iter_ == b.n_iter_
    assert a.cluster_centers_.dtype == np.float64 and isinstance(a.inertia_, np.float64)
    np.testing.assert_allclose(a.inertia_, b.inertia_, rtol=1e-12)
    assert a.n_features_in_ == X.shape[1]


def test_kmeans_parallel_equals_the_dense_fit(cpu_backend):
    from dask_ml_b200.cluster import k_means as km

    X = blobs(n=500, seed=1)
    seen = []
    orig = km._reduce_candidates

    def spy(cand, *a, **kw):
        seen.append(cand.toarray() if sp.issparse(cand) else np.asarray(cand))
        return orig(cand, *a, **kw)

    km._reduce_candidates = spy
    try:
        a = _km(n_clusters=4, random_state=5, tol=1e-8).fit(chunked(X, 170))
        b = _dense_fit(X, n_clusters=4, random_state=5, tol=1e-8)
    finally:
        km._reduce_candidates = orig
    assert len(seen) == 2
    np.testing.assert_array_equal(seen[0], seen[1])
    np.testing.assert_allclose(a.cluster_centers_, b.cluster_centers_, rtol=0, atol=1e-10)
    np.testing.assert_array_equal(_np(a.labels_), _np(b.labels_))


def test_kmeans_plusplus(cpu_backend):
    X = blobs(seed=2)
    a = _km(n_clusters=4, init="k-means++", random_state=0).fit(X)
    b = _dense_fit(X, n_clusters=4, init="k-means++", random_state=0)
    np.testing.assert_allclose(a.cluster_centers_, b.cluster_centers_, rtol=0, atol=1e-10)


def test_matches_sklearn(cpu_backend):
    X = blobs(n=600, seed=4)
    C0 = X[[0, 1, 2, 3]].toarray()
    a = _km(n_clusters=4, init=C0, tol=0.0, max_iter=100).fit(X)
    s = SkKMeans(n_clusters=4, init=C0, n_init=1, algorithm="lloyd", tol=0.0, max_iter=100).fit(X)
    np.testing.assert_array_equal(_np(a.labels_), s.labels_)
    np.testing.assert_allclose(a.cluster_centers_, s.cluster_centers_, rtol=0, atol=1e-10)


def test_predict_transform_fit_transform(cpu_backend):
    X = blobs(seed=6)
    C0 = X[[0, 1, 2, 3]].toarray()
    a = _km(n_clusters=4, init=C0).fit(chunked(X, 100))
    b = _dense_fit(X, n_clusters=4, init=C0)
    np.testing.assert_array_equal(_np(a.predict(chunked(X, 77))), _np(b.predict(X.toarray())))
    np.testing.assert_allclose(_np(a.transform(X)), _np(b.transform(X.toarray())), rtol=1e-12, atol=1e-12)
    T = _km(n_clusters=4, init=C0).fit_transform(X)
    assert _np(T).shape == (X.shape[0], 4)


def test_metrics_on_sparse_x(cpu_backend):
    from dask_ml_b200.metrics import euclidean_distances, pairwise_distances_argmin_min

    X = blobs(n=120, seed=7)
    Y = np.random.RandomState(0).standard_normal((5, X.shape[1]))
    D = X.toarray()
    ref = np.sqrt(np.maximum((D ** 2).sum(1)[:, None] - 2 * D @ Y.T + (Y ** 2).sum(1)[None], 0))
    np.testing.assert_allclose(_np(euclidean_distances(X, Y)), ref, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(_np(euclidean_distances(X, Y, squared=True)), ref ** 2, rtol=1e-12, atol=1e-12)
    lab, mn = pairwise_distances_argmin_min(chunked(X, 50), Y)
    np.testing.assert_array_equal(_np(lab), ref.argmin(1))
    np.testing.assert_allclose(_np(mn), ref.min(1), rtol=1e-12)
    with pytest.raises(NotImplementedError):
        euclidean_distances(X, Y, Y_norm_squared=(Y ** 2).sum(1))
    with pytest.raises(NotImplementedError):
        euclidean_distances(X, Y, X_norm_squared=(D ** 2).sum(1)[:, None])


def test_ragged_and_empty_blocks_and_empty_cluster(cpu_backend):
    from dask_ml_b200 import ChunkedArray

    X = blobs(n=300, seed=8)
    blocks = [torch_csr(X[0:0]), torch_csr(X[0:17]), torch_csr(X[17:200]), torch_csr(X[200:200]), torch_csr(X[200:])]
    # the fifth centre is far from every row: its cluster stays empty and its centre becomes 0
    C0 = np.vstack([X[[0, 1, 2, 3]].toarray(), np.full((1, X.shape[1]), 100.0)])
    a = _km(n_clusters=5, init=C0, max_iter=1, tol=0.0).fit(ChunkedArray(blocks))
    b = _dense_fit(X, n_clusters=5, init=C0, max_iter=1, tol=0.0)
    np.testing.assert_array_equal(_np(a.labels_), _np(b.labels_))
    np.testing.assert_allclose(a.cluster_centers_, b.cluster_centers_, rtol=0, atol=1e-12)
    np.testing.assert_array_equal(a.cluster_centers_[4], 0.0)
    assert [int(l.shape[0]) for l in a.labels_.blocks] == [0, 17, 183, 0, 100]
    # an empty row's distance to centre j is ||c_j||
    d = _np(a.transform(X[5:6]))[0]
    np.testing.assert_allclose(d, np.linalg.norm(a.cluster_centers_, axis=1), rtol=1e-12)


@pytest.mark.parametrize("vdtype", [np.float32, np.float64, np.int64, np.bool_])
def test_intake_forms_and_value_dtypes(cpu_backend, vdtype):
    X = blobs(seed=9)
    X = sp.csr_matrix((np.round(X.data).astype(vdtype) if vdtype != np.bool_ else X.data > 1.0, X.indices, X.indptr),
                      shape=X.shape)
    X.eliminate_zeros()
    D = X.toarray().astype(np.float64)
    C0 = D[[0, 1, 2, 3]]
    forms = [X, X.tocoo(), torch_csr(X), chunked(X, 150), chunked(X, 150).__class__([b.to("cpu") for b in chunked(X, 150).blocks])]
    dt = np.float32 if vdtype == np.float32 else np.float64
    ref = _km(n_clusters=4, init=C0.astype(dt)).fit(D.astype(dt))
    for f in forms:
        a = _km(n_clusters=4, init=C0.astype(dt)).fit(f)
        assert a.cluster_centers_.dtype == dt
        np.testing.assert_array_equal(_np(a.labels_), _np(ref.labels_))
        np.testing.assert_allclose(a.cluster_centers_, ref.cluster_centers_, rtol=1e-6 if dt == np.float32 else 1e-12,
                                   atol=1e-6 if dt == np.float32 else 1e-12)


def test_intake_errors(cpu_backend):
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.cluster.k_means import _NONFINITE_MSG, k_init

    X = blobs(seed=10)
    C0 = X[[0, 1, 2, 3]].toarray()
    with pytest.raises(TypeError, match="mixes dense and sparse"):
        _km(n_clusters=4, init=C0).fit(ChunkedArray([torch_csr(X[:100]), torch.from_numpy(X[100:].toarray())]))
    bad = X.copy()
    bad.data[3] = np.nan
    with pytest.raises(ValueError, match="NaN"):
        _km(n_clusters=4, init=C0).fit(bad)
    assert "NaN" in _NONFINITE_MSG
    a = _km(n_clusters=4, init=C0).fit(X)
    with pytest.raises(ValueError, match="features"):
        a.predict(X[:, :10])
    with pytest.raises(ValueError, match="features"):
        a.transform(X[:, :10])
    noncanon = torch.sparse_csr_tensor(torch.tensor([0, 2]), torch.tensor([3, 1]), torch.tensor([1.0, 2.0]),
                                       size=(1, X.shape[1]), dtype=torch.float64)
    with pytest.raises(ValueError, match="canonical"):
        _km(n_clusters=1, init=np.zeros((1, X.shape[1]))).fit(ChunkedArray([noncanon]))
    with pytest.raises(NotImplementedError):
        k_init(X, 4, init="k-means||", random_state=0, weighted=True)


def test_k_means_and_k_init_take_sparse(cpu_backend):
    from dask_ml_b200.cluster.k_means import k_init, k_means

    X = blobs(seed=11)
    C = k_init(X, 4, init="random", random_state=1)
    np.testing.assert_array_equal(C, k_init(X.toarray(), 4, init="random", random_state=1))
    labels, centers, inertia = k_means(X, 4, init=C)
    l2, c2, i2 = k_means(X.toarray(), 4, init=C)
    np.testing.assert_array_equal(_np(labels), _np(l2))
    np.testing.assert_allclose(centers, c2, rtol=0, atol=1e-12)


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


SHARDS = [(0, 170), (170, 400)]


def _worker(rank, world, port, out_dir):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    import torch.distributed as dist

    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from dask_ml_b200.cluster import KMeans, k_means as km
        from test_kmeans_sparse_host import KMeansSparseOracleBackend, blobs, chunked

        km._BACKEND_FACTORY = KMeansSparseOracleBackend
        lo, hi = SHARDS[rank]
        X = blobs()
        res = {}
        for init in ("array", "k-means||"):
            C0 = X[[0, 1, 2, 3]].toarray() if init == "array" else init
            est = KMeans(n_clusters=4, init=C0, random_state=2, tol=1e-8).fit(chunked(X[lo:hi], 60))
            res[init] = est.cluster_centers_
            res[init + "_labels"] = est.labels_.compute()
            res[init + "_inertia"] = np.array([est.inertia_])
        np.savez(os.path.join(out_dir, "rank%d.npz" % rank), **res)
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(600)
def test_two_ranks_equal_one_rank(tmp_path, cpu_backend):
    mp.start_processes(_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True, start_method="spawn")
    r = [np.load(tmp_path / ("rank%d.npz" % k)) for k in range(2)]
    X = blobs()
    for init in ("array", "k-means||"):
        np.testing.assert_array_equal(r[0][init], r[1][init])
        C0 = X[[0, 1, 2, 3]].toarray() if init == "array" else init
        one = _km(n_clusters=4, init=C0, random_state=2, tol=1e-8).fit(chunked(X, 60))
        np.testing.assert_allclose(r[0][init], one.cluster_centers_, rtol=0, atol=1e-12)
        labels = np.concatenate([r[0][init + "_labels"], r[1][init + "_labels"]])
        np.testing.assert_array_equal(labels, _np(one.labels_))
        np.testing.assert_allclose(r[0][init + "_inertia"][0], one.inertia_, rtol=1e-12)
