"""SpectralClustering without a GPU: the float64 restatement of the reference's Nystrom embedding (unfused and fused
forms) and the estimator, both against fixtures written by the reference's own spectral.py, and the estimator's host logic (validation, draws, host algebra, 2 ranks over gloo) on a CPU backend whose two
Nystrom passes are numpy."""
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp
from sklearn.base import BaseEstimator

import spectral_oracle as so

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle_backend import OracleBackend  # noqa: E402


class NystromOracleBackend(OracleBackend):
    """The CPU checker backend plus the two Nystrom passes, in float64 numpy."""

    def kernel_colsum(self, x, pack, l, gamma, colsum, first=False):
        c = torch.from_numpy(so.colsum(x.numpy(), pack.numpy(), gamma)) if x.shape[0] else torch.zeros(l, dtype=torch.float64)
        if first:
            colsum.copy_(c)
        else:
            colsum += c

    def nystrom_embed(self, x, pack, l, gamma, W, out):
        e = so.project(x.numpy(), pack.numpy(), W.numpy().astype(np.float64), gamma)
        out.copy_(torch.from_numpy(e).to(out.dtype))


class Recorder(BaseEstimator):
    """Label assignment that keeps what it was fitted on."""

    def __init__(self, n_clusters=2):
        self.n_clusters = n_clusters

    def fit(self, X, y=None):
        self.X_ = np.asarray(X)
        self.labels_ = np.zeros(len(self.X_), dtype=np.int32)
        return self


def _blobs(n, d, k, seed, dtype=np.float64):
    rng = np.random.RandomState(seed)
    cent = rng.uniform(-3, 3, size=(k, d))
    return (cent[rng.randint(0, k, size=n)] + 0.5 * rng.standard_normal((n, d))).astype(dtype)


@pytest.fixture
def cpu_backend(monkeypatch):
    from dask_ml_b200.cluster import k_means as km

    monkeypatch.setattr(km, "_BACKEND_FACTORY", NystromOracleBackend)


# ---------------------------------------------------------------------------------------------- reference fixtures
# written by the reference's own spectral.py (tests/golden/ref_spectral.py)
GOLDEN = os.path.join(ROOT, "tests", "golden")
FIXTURES = ["ref_spectral_f64_2000x5", "ref_spectral_f32_gamma_none", "ref_spectral_kmeans_branch",
            "ref_spectral_test_basic"]


def load_fixture(name):
    f = np.load(os.path.join(GOLDEN, name + ".npz"))
    g = float(f["gamma"])
    X = f["X"]
    return dict(X=X, chunks=int(f["chunks"]), keep=f["keep"], U2=f["U2"], S=f["S"], k=int(f["n_clusters"]),
                l=int(f["n_components"]), gamma=None if np.isnan(g) else g, seed=int(f["seed"]),
                km_seed=int(f["km_seed"]), gamma_eff=(1.0 / X.shape[1]) if np.isnan(g) else g)


class RecordingRandomState(np.random.RandomState):
    """Remembers what ``choice`` returned: the keep rows the estimator drew."""

    def choice(self, *a, **k):
        out = super().choice(*a, **k)
        self.chosen = np.sort(out)
        return out


@pytest.mark.parametrize("name", FIXTURES)
def test_restatements_reproduce_the_reference(name):
    fx = load_fixture(name)
    X64 = fx["X"].astype(np.float64)                     # the reference casts to float (spectral.py:177)
    U_u, S_u = so.embed_unfused(X64, fx["keep"], fx["k"], fx["gamma_eff"])
    U_f, S_f = so.embed_fused(X64, fx["keep"], fx["k"], fx["gamma_eff"])
    for U, S in ((U_u, S_u), (U_f, S_f)):
        assert np.abs(U - fx["U2"]).max() < 1e-12          # same SVD, same signs: no alignment needed
        np.testing.assert_allclose(S, fx["S"], rtol=1e-12)


@pytest.mark.parametrize("name", FIXTURES)
def test_estimator_reproduces_the_reference(cpu_backend, monkeypatch, name):
    """Embedding, eigenvalues, keep rows and (default branch) the KMeans seed of the reference's own fit."""
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.cluster import SpectralClustering, spectral

    fx = load_fixture(name)
    seen = {}

    class KM(spectral.KMeans):
        def fit(self, X, y=None):
            seen["seed"] = self.random_state
            seen["U"] = np.concatenate([c.numpy() for c in X.chunks])
            return super().fit(X)

    monkeypatch.setattr(spectral, "KMeans", KM)
    rs = RecordingRandomState(fx["seed"])
    kw = dict(n_clusters=fx["k"], n_components=fx["l"], gamma=fx["gamma"], random_state=rs)
    if fx["km_seed"] < 0:
        rec = Recorder()
        sc = SpectralClustering(assign_labels=rec, **kw).fit(ChunkedArray.from_array(fx["X"], fx["chunks"]))
        U = rec.X_
    else:
        sc = SpectralClustering(**kw).fit(ChunkedArray.from_array(fx["X"], fx["chunks"]))
        U = seen["U"]
        assert seen["seed"] == fx["km_seed"]
    np.testing.assert_array_equal(rs.chosen, fx["keep"])
    assert U.dtype == fx["X"].dtype
    tol = 1e-10 if fx["X"].dtype == np.float64 else 1e-6     # float32 input: the embedding is float32
    assert so.procrustes_err(U, fx["U2"]) < tol
    np.testing.assert_allclose(sc.eigenvalues_, fx["S"], rtol=1e-10)


# ---------------------------------------------------------------------------------------------- the estimator
def test_error_contract(cpu_backend):
    from dask_ml_b200.cluster import SpectralClustering

    X = _blobs(200, 2, 3, 0)
    with pytest.raises(ValueError, match="Unknown 'assign_labels' 'foo'"):
        SpectralClustering(assign_labels="foo").fit(X)
    with pytest.raises(TypeError, match="Invalid type "):
        SpectralClustering(assign_labels=dict()).fit(X)
    with pytest.raises(ValueError, match="n_components"):
        SpectralClustering(n_components=200).fit(X)
    with pytest.raises(ValueError, match="Unknown affinity metric name 'foo'"):
        SpectralClustering(affinity="foo", n_components=25).fit(X)
    with pytest.raises(TypeError, match="Unexpected type for 'affinity'"):
        SpectralClustering(affinity=np.array([]), n_components=25).fit(X)
    for name in ("linear", "polynomial", "sigmoid"):
        with pytest.raises(NotImplementedError):
            SpectralClustering(affinity=name, n_components=25).fit(X)
    with pytest.raises(ValueError, match="n_clusters"):
        SpectralClustering(n_clusters=30, n_components=25, assign_labels=Recorder()).fit(X)
    # kmeans_params reach the label assignment through set_params
    rec = Recorder()
    SpectralClustering(n_components=25, assign_labels=rec, kmeans_params={"n_clusters": 5}, random_state=0).fit(X)
    assert rec.n_clusters == 5


def test_callable_affinity_equals_rbf(cpu_backend):
    from dask_ml_b200.cluster import SpectralClustering

    X = _blobs(300, 4, 3, 9)

    def kern(A, B=None, gamma=None, degree=None, coef0=None):
        return so.rbf(A, A if B is None else B, gamma)

    r1, r2 = Recorder(), Recorder()
    a = SpectralClustering(n_clusters=3, n_components=20, gamma=0.3, random_state=2, assign_labels=r1).fit(X)
    b = SpectralClustering(n_clusters=3, n_components=20, gamma=0.3, random_state=2, assign_labels=r2,
                           affinity=kern).fit(X)
    assert so.procrustes_err(r2.X_, r1.X_) < 1e-10
    np.testing.assert_allclose(b.eigenvalues_, a.eigenvalues_, rtol=1e-12)


# ---------------------------------------------------------------------------------------------- two ranks
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, out_dir):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    import torch.distributed as dist

    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from dask_ml_b200 import ChunkedArray
        from dask_ml_b200.cluster import SpectralClustering, k_means as km
        from test_spectral_host import NystromOracleBackend, Recorder, _blobs

        km._BACKEND_FACTORY = NystromOracleBackend
        X = _blobs(1500, 4, 3, 11)
        lo, hi = (0, 400) if rank == 0 else (400, 1500)            # uneven shards
        rec = Recorder()
        sc = SpectralClustering(n_clusters=3, n_components=30, gamma=0.4, random_state=6, assign_labels=rec)
        sc.fit(ChunkedArray.from_array(X[lo:hi], 300))
        np.savez(os.path.join(out_dir, "rank%d.npz" % rank), U=rec.X_, S=sc.eigenvalues_)
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(600)
def test_two_ranks_give_the_single_process_embedding(tmp_path, cpu_backend):
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.cluster import SpectralClustering

    mp.start_processes(_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True, start_method="spawn")
    r0, r1 = np.load(tmp_path / "rank0.npz"), np.load(tmp_path / "rank1.npz")
    X = _blobs(1500, 4, 3, 11)
    rec = Recorder()
    one = SpectralClustering(n_clusters=3, n_components=30, gamma=0.4, random_state=6, assign_labels=rec)
    one.fit(ChunkedArray.from_array(X, 500))
    for r in (r0, r1):
        assert np.abs(r["U"] - rec.X_).max() < 1e-12
        np.testing.assert_allclose(r["S"], one.eigenvalues_, rtol=1e-12)
    np.testing.assert_array_equal(r0["S"], r1["S"])
