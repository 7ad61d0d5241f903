"""PartialMiniBatchKMeans, SpectralClustering, rbf_kernel and pairwise_kernels on sparse X without a GPU: a CPU checker
backend whose sparse passes (the KMeans ones of test_kmeans_sparse_host plus bkm_sparse_minibatch_step,
bkm_csr_kernel_colsum_chunk and bkm_csr_nystrom_embed_chunk) are float64 scipy restatements, checked against
scikit-learn and against the dense fits of the densified X; and 2 ranks over gloo."""
import os
import pickle
import socket
import sys
import warnings

import numpy as np
import pytest
import scipy.sparse as sp
import torch
import torch.multiprocessing as mp
from sklearn.cluster import MiniBatchKMeans
from sklearn.metrics.pairwise import rbf_kernel as sk_rbf_kernel

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import spectral_oracle as so  # noqa: E402
from test_glm_sparse_host import _csr, chunked, torch_csr  # noqa: E402
from test_kmeans_sparse_host import KMeansSparseOracleBackend, blobs  # noqa: E402
from test_minibatch_host import MiniBatchChecker  # noqa: E402
from test_spectral_host import NystromOracleBackend, Recorder  # noqa: E402

pytestmark = pytest.mark.filterwarnings("ignore:'PartialMiniBatchKMeans' is deprecated:FutureWarning")


class SparseClusteringChecker(KMeansSparseOracleBackend, MiniBatchChecker, NystromOracleBackend):
    """The dense checkers of the mini-batch step and the Nystrom passes, the sparse KMeans checker, and float64 scipy
    restatements of the three sparse passes of this file."""

    def _d2(self, blk, d, pack, k):
        X = _csr(blk, d)
        CT, cn = self._unpack(pack, k, d)
        xn = np.asarray(X.multiply(X).sum(1)).ravel()
        return np.maximum(xn[:, None] - 2.0 * np.asarray(X @ CT) + cn[None, :], 0.0)

    def csr_kernel_colsum(self, blk, d, pack, l, gamma, colsum, first=False):
        self.launches += 1
        c = torch.from_numpy(np.exp(-gamma * self._d2(blk, d, pack, l)).sum(0))
        colsum.copy_(c) if first else colsum.add_(c)

    def csr_nystrom_embed(self, blk, d, pack, l, gamma, W, out):
        self.launches += 1
        d2 = self._d2(blk, d, pack, l)
        m = d2.min(1, keepdims=True)
        e = np.exp(-gamma * (d2 - m)) @ W.numpy()
        with np.errstate(invalid="ignore"):
            e = e / np.sqrt((e * e).sum(1, keepdims=True))
        e[(gamma * m[:, 0]) > 745.13] = np.nan
        out.copy_(torch.from_numpy(e).to(out.dtype))

    def sparse_minibatch_step(self, red, pack_in, w_in, pack_out, w_out, k, d):
        self.launches += 1
        r = red.numpy()
        S, n = r[: d * k].reshape(d, k), r[d * k: d * k + k]
        CT, w = pack_in[: d * k].view(d, k).numpy(), w_in.numpy()
        with np.errstate(divide="ignore", invalid="ignore"):
            upd = (CT * w[None, :] + S) * (1.0 / (w + n))[None, :]
        CT2 = np.where((n > 0)[None, :], upd, CT)
        pack_out.copy_(torch.from_numpy(np.concatenate([CT2.ravel(), (CT2 * CT2).sum(0)])))
        w_out.copy_(torch.from_numpy(w + n))


@pytest.fixture(autouse=True)
def checker(monkeypatch):
    from dask_ml_b200.cluster import k_means as km

    monkeypatch.setattr(km, "_BACKEND_FACTORY", SparseClusteringChecker)


def _mbk(**kw):
    from dask_ml_b200.cluster import PartialMiniBatchKMeans

    return PartialMiniBatchKMeans(**kw)


def _np(a):
    return a.compute() if hasattr(a, "compute") else np.asarray(a)


def _same_state(a, b, rtol=1e-12):
    np.testing.assert_allclose(a.cluster_centers_, b.cluster_centers_, rtol=rtol, atol=rtol)
    np.testing.assert_array_equal(a._counts, b._counts)
    assert a.n_steps_ == b.n_steps_
    assert a._n_since_last_reassign == b._n_since_last_reassign
    if hasattr(b, "labels_"):
        np.testing.assert_array_equal(_np(a.labels_), _np(b.labels_))
        np.testing.assert_allclose(a.inertia_, b.inertia_, rtol=rtol)


def _batches(n_batches, n=300, p=30, k=4, seed=0):
    return [blobs(n=n, p=p, k=k, seed=seed + i) for i in range(n_batches)]


# ---------------------------------------------------------------------------------------------- PartialMiniBatchKMeans
@pytest.mark.parametrize("init", ["k-means++", "random", "array"])
def test_partial_fit_matches_sklearn(init):
    batches = _batches(4)
    C0 = batches[0][[0, 1, 2, 3]].toarray() if init == "array" else init
    kw = dict(n_clusters=4, init=C0, batch_size=300, n_init=1)
    a, b = _mbk(random_state=7, **kw), MiniBatchKMeans(random_state=7, **kw)
    for X in batches:
        a.partial_fit(X)
        b.partial_fit(X)
        _same_state(a, b)
    np.testing.assert_array_equal(a._random_state.get_state()[1], b._random_state.get_state()[1])


def test_partial_fit_with_reassignment_matches_sklearn():
    batches = _batches(8, n=60, k=3, seed=20)
    kw = dict(n_clusters=12, batch_size=60, reassignment_ratio=0.5, n_init=1)
    a, b = _mbk(random_state=3, **kw), MiniBatchKMeans(random_state=3, **kw)
    draws = []
    for X in batches:
        a.partial_fit(X)
        b.partial_fit(X)
        _same_state(a, b)
        draws.append(a._n_since_last_reassign)
    assert 0 in draws[1:]                          # a reassignment happened after the first step


def test_fit_is_partial_fit_in_shuffled_order():
    X = blobs(n=1200, seed=3)
    np.random.seed(5)
    a = _mbk(n_clusters=4, random_state=0).fit(chunked(X, 300))
    np.random.seed(5)
    order = list(range(4))
    np.random.shuffle(order)
    b = MiniBatchKMeans(n_clusters=4, random_state=0, n_init=1)
    for i in order:
        b.partial_fit(X[i * 300:(i + 1) * 300])
    _same_state(a, b)


def test_sparse_fit_equals_the_dense_fit():
    X = blobs(n=900, seed=4)
    np.random.seed(1)
    a = _mbk(n_clusters=4, random_state=2).fit(chunked(X, 300))
    np.random.seed(1)
    from dask_ml_b200 import ChunkedArray

    b = _mbk(n_clusters=4, random_state=2).fit(ChunkedArray.from_array(X.toarray(), 300))
    _same_state(a, b)
    np.testing.assert_array_equal(_np(a.predict(X)), _np(b.predict(X.toarray())))
    np.testing.assert_allclose(_np(a.transform(X)), _np(b.transform(X.toarray())), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(a.score(X), b.score(X.toarray()), rtol=1e-12)


def test_predict_transform_score_against_sklearn():
    X = blobs(n=600, seed=6)
    a = _mbk(n_clusters=4, random_state=0).partial_fit(X)
    b = MiniBatchKMeans(n_clusters=4, random_state=0, n_init=1).partial_fit(X)
    np.testing.assert_array_equal(_np(a.predict(X)), b.predict(X))
    np.testing.assert_allclose(_np(a.transform(X)), b.transform(X), rtol=1e-10)
    np.testing.assert_allclose(a.score(X), b.score(X), rtol=1e-10)


def test_dense_and_sparse_batches_continue_the_same_state():
    batches = _batches(4, seed=30)
    a = _mbk(n_clusters=4, random_state=1)
    b = _mbk(n_clusters=4, random_state=1)
    for i, X in enumerate(batches):
        a.partial_fit(X if i % 2 == 0 else X.toarray())
        b.partial_fit(X.toarray())
        _same_state(a, b)


def test_pickle_round_trip():
    batches = _batches(3, seed=40)
    a = _mbk(n_clusters=4, random_state=0).partial_fit(batches[0])
    b = pickle.loads(pickle.dumps(a))
    assert "_mb" not in vars(b)
    for X in batches[1:]:
        a.partial_fit(X)
        b.partial_fit(X)
    assert torch.equal(a._mb.C, b._mb.C) and torch.equal(a._mb.W, b._mb.W)
    np.testing.assert_array_equal(a.cluster_centers_, b.cluster_centers_)


def test_empty_blocks_and_empty_rows():
    from dask_ml_b200 import ChunkedArray

    X = blobs(n=300, seed=50)                      # row 5 is empty
    blocks = ChunkedArray([torch_csr(X[0:0]), torch_csr(X[0:120]), torch_csr(X[120:120]), torch_csr(X[120:])])
    kw = dict(n_clusters=4, random_state=0, init=X[[0, 1, 2, 3]].toarray())
    a = _mbk(**kw).partial_fit(blocks)
    b = MiniBatchKMeans(n_init=1, **kw).partial_fit(X)
    _same_state(a, b)
    assert [int(l.shape[0]) for l in a.labels_.blocks] == [0, 120, 0, 180]


def test_non_canonical_block_and_feature_mismatch():
    from dask_ml_b200 import ChunkedArray

    X = blobs(n=200, seed=60)
    a = _mbk(n_clusters=4, random_state=0).partial_fit(X)
    C, W = a._mb.C.clone(), a._mb.W.clone()
    noncanon = torch.sparse_csr_tensor(torch.tensor([0, 2, 3, 4]), torch.tensor([3, 1, 0, 2]), torch.tensor([1.0, 2.0, 1.0, 1.0]),
                                       size=(3, X.shape[1]), dtype=torch.float64)
    with pytest.raises(ValueError, match="canonical"):
        a.partial_fit(ChunkedArray([noncanon]))
    assert torch.equal(a._mb.C, C) and torch.equal(a._mb.W, W)    # the step was undone
    with pytest.raises(ValueError, match="features"):
        a.partial_fit(X[:, :10])


# ---------------------------------------------------------------------------------------------- SpectralClustering
def _spectral(**kw):
    from dask_ml_b200.cluster import SpectralClustering

    return SpectralClustering(**kw)


def test_spectral_equals_the_dense_fit():
    X = blobs(n=500, p=24, k=3, seed=70)
    kw = dict(n_clusters=3, n_components=40, gamma=0.05, random_state=4)
    r1, r2 = Recorder(), Recorder()
    a = _spectral(assign_labels=r1, **kw).fit(chunked(X, 130))
    b = _spectral(assign_labels=r2, **kw).fit(X.toarray())
    np.testing.assert_allclose(a.eigenvalues_, b.eigenvalues_, rtol=1e-12)
    assert so.procrustes_err(r1.X_, r2.X_) < 1e-10
    assert r1.X_.dtype == np.float64
    # the default label assignment on well separated data
    la = _np(_spectral(**kw).fit(X).labels_)
    lb = _np(_spectral(**kw).fit(X.toarray()).labels_)
    np.testing.assert_array_equal(la, lb)


def test_spectral_float32_values_give_a_float32_embedding():
    X = blobs(n=300, p=24, k=3, seed=71).astype(np.float32)
    rec = Recorder()
    _spectral(n_clusters=3, n_components=30, gamma=0.05, random_state=0, assign_labels=rec).fit(X)
    assert rec.X_.dtype == np.float32


def test_spectral_callable_affinity_equals_rbf():
    X = blobs(n=400, p=24, k=3, seed=72)
    seen = []

    def kern(A, B=None, gamma=None, degree=None, coef0=None):
        seen.append(sp.issparse(A) and (B is None or sp.issparse(B)))
        return sk_rbf_kernel(A, B, gamma=gamma)

    r1, r2 = Recorder(), Recorder()
    kw = dict(n_clusters=3, n_components=25, gamma=0.05, random_state=2)
    a = _spectral(assign_labels=r1, **kw).fit(chunked(X, 150))
    b = _spectral(assign_labels=r2, affinity=kern, **kw).fit(chunked(X, 150))
    assert seen and all(seen)
    assert so.procrustes_err(r2.X_, r1.X_) < 1e-10
    np.testing.assert_allclose(b.eigenvalues_, a.eigenvalues_, rtol=1e-12)


def test_spectral_sparse_tag():
    assert _spectral().__sklearn_tags__().input_tags.sparse


# ---------------------------------------------------------------------------------------------- rbf_kernel
def test_rbf_kernel_and_pairwise_kernels():
    from dask_ml_b200.metrics import pairwise_kernels, rbf_kernel

    X = blobs(n=150, seed=80)
    Y = np.random.RandomState(0).standard_normal((6, X.shape[1]))
    for g in (None, 0.02):
        ref = sk_rbf_kernel(X, Y, gamma=g)
        got = _np(rbf_kernel(chunked(X, 70), Y, gamma=g))
        assert got.dtype == np.float64
        np.testing.assert_allclose(got, ref, rtol=1e-12, atol=1e-15)
        np.testing.assert_allclose(_np(pairwise_kernels(X, Y, metric="rbf", gamma=g)), ref, rtol=1e-12, atol=1e-15)
    got32 = _np(rbf_kernel(X.astype(np.float32), Y.astype(np.float32), gamma=0.02))
    assert got32.dtype == np.float32
    np.testing.assert_allclose(got32, sk_rbf_kernel(X, Y, gamma=0.02), rtol=1e-5, atol=1e-7)
    with pytest.raises(NotImplementedError, match="dense Y"):
        rbf_kernel(X)


# ---------------------------------------------------------------------------------------------- two ranks
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, out_dir):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    warnings.simplefilter("ignore")
    import torch.distributed as dist

    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from dask_ml_b200.cluster import SpectralClustering, k_means as km
        from test_sparse_clustering_host import SparseClusteringChecker, Recorder, blobs, chunked

        km._BACKEND_FACTORY = SparseClusteringChecker
        X = blobs(n=600, p=24, k=3, seed=90)
        lo, hi = (0, 250) if rank == 0 else (250, 600)
        rec = Recorder()
        sc = SpectralClustering(n_clusters=3, n_components=30, gamma=0.05, random_state=6, assign_labels=rec)
        sc.fit(chunked(X[lo:hi], 100))
        np.savez(os.path.join(out_dir, "rank%d.npz" % rank), U=rec.X_, S=sc.eigenvalues_)
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(600)
def test_two_ranks_give_the_single_process_embedding(tmp_path):
    mp.start_processes(_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True, start_method="spawn")
    r0, r1 = np.load(tmp_path / "rank0.npz"), np.load(tmp_path / "rank1.npz")
    X = blobs(n=600, p=24, k=3, seed=90)
    rec = Recorder()
    one = _spectral(n_clusters=3, n_components=30, gamma=0.05, random_state=6, assign_labels=rec).fit(chunked(X, 100))
    for r in (r0, r1):
        assert np.abs(r["U"] - rec.X_).max() < 1e-12
        np.testing.assert_allclose(r["S"], one.eigenvalues_, rtol=1e-12)
