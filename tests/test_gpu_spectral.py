"""SpectralClustering on the H100: the two Nystrom passes (bkm_kernel_colsum_chunk, bkm_nystrom_embed_chunk) on both
kernel paths against float64, their scale invariance, the estimator end to end against the float64 restatement of the
reference (tests/spectral_oracle.py), and ports of the reference's tests/test_spectral_clustering.py.

The reference's ``test_slice_mostly_sorted`` is not ported: it tests a dask-only helper that puts the rows back in input
order, and this design keeps the rows in input order throughout."""
import os
import subprocess
import sys
from functools import partial

import numpy as np
import pytest
import torch

import spectral_oracle as so
from dask_ml_b200 import _lib

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TAU_TC = lambda d: (8.0 * np.sqrt(3.0 * ((d + 7) // 8)) + 16.0) * 2.0 ** -24      # bkm_api.cu tau_for, family 1
TAU_SIMT = lambda d: 8.0 * (np.sqrt(d) + 2.0) * 2.0 ** -24                          # CUDA-core kernels


@pytest.fixture(scope="module")
def be():
    from dask_ml_b200.engine import CudaBackend

    return CudaBackend()


def _data(n, d, k_true, seed, scale=1.0):
    rng = np.random.RandomState(seed)
    cent = rng.uniform(-scale, scale, size=(k_true, d))
    return cent[rng.randint(0, k_true, size=n)] + 0.3 * scale * rng.standard_normal((n, d))


def _dev(be, X, dtype):
    return be.to_device(np.ascontiguousarray(X), dtype)


def _pack(be, C, dtype):
    return be.pack_centers(torch.as_tensor(np.ascontiguousarray(C, dtype=np.float64)).to(be.device), dtype)


def _d2(X, C):
    X = torch.as_tensor(np.asarray(X, dtype=np.float64), device="cuda")
    C = torch.as_tensor(np.asarray(C, dtype=np.float64), device="cuda")
    return torch.clamp((X * X).sum(1)[:, None] - 2.0 * X @ C.T + (C * C).sum(1)[None, :], min=0.0)


def _colsum(be, x, pack, l, gamma, flags=0, chunks=1):
    c = be.zeros((l,), torch.float64)
    old = be.flags
    be.flags = flags
    try:
        rows = int(x.shape[0])
        step = (rows + chunks - 1) // chunks
        for i, s0 in enumerate(range(0, rows, step)):
            be.kernel_colsum(x[s0:s0 + step], pack, l, gamma, c, first=i == 0)
    finally:
        be.flags = old
    torch.cuda.synchronize()
    return c.cpu().numpy()


def _embed(be, x, pack, l, gamma, W, flags=0):
    out = be.zeros((int(x.shape[0]), W.shape[1]), x.dtype)
    old = be.flags
    be.flags = flags
    try:
        be.nystrom_embed(x, pack, l, gamma, torch.as_tensor(W).to(device=be.device, dtype=x.dtype), out)
    finally:
        be.flags = old
    return out.cpu().numpy()


# ---------------------------------------------------------------------------------------------- column sums
COLSUM_CASES = [
    # (n, d, l, dtype, flags, expected family: 1 tensor / 0 CUDA cores)
    (100_003, 64, 256, torch.float32, 0, 1),
    (50_001, 41, 100, torch.float32, 0, 1),
    (20_000, 2, 25, torch.float32, 0, 1),
    (777, 13, 5, torch.float32, 0, 1),
    (30_000, 100, 50, torch.float32, 0, 0),       # d > 64
    (30_000, 16, 300, torch.float32, 0, 0),       # l > 256
    (5_000, 16, 100, torch.float64, 0, 0),
    (50_001, 41, 100, torch.float32, _lib.FLAG_FORCE_SIMT, 0),
]


@pytest.mark.parametrize("n,d,l,dtype,flags,fam", COLSUM_CASES)
def test_colsum_matches_float64(be, n, d, l, dtype, flags, fam):
    X = _data(n, d, 12, n + d)
    gamma = 1.0 / d
    keep = X[np.random.RandomState(1).choice(n, l, replace=False)]
    x = _dev(be, X, dtype)
    Xq = x.double().cpu().numpy()                               # the rows as stored
    pack = _pack(be, keep, dtype)
    got = _colsum(be, x, pack, l, gamma, flags)
    d2 = _d2(Xq, keep)
    v = torch.exp(-gamma * d2)
    want = v.sum(0).cpu().numpy()
    if dtype == torch.float64:
        np.testing.assert_allclose(got, want, rtol=1e-12)
    else:
        tau = TAU_TC(d) if fam == 1 else TAU_SIMT(d)
        xn = torch.as_tensor((Xq * Xq).sum(1), device="cuda")
        cmax = float((keep ** 2).sum(1).max())
        bound = (v * (gamma * tau * (xn[:, None] + cmax) + 4e-6)[:, :]).sum(0).cpu().numpy() + 1e-6 * want
        assert np.all(np.abs(got - want) <= bound), np.max(np.abs(got - want) / want)
        assert np.max(np.abs(got - want) / want) < 2e-5
    # bit-identical on a repeat call, and split into chunks: FIRST overwrites, later calls add
    np.testing.assert_array_equal(_colsum(be, x, pack, l, gamma, flags), got)
    multi = _colsum(be, x, pack, l, gamma, flags, chunks=3)
    np.testing.assert_allclose(multi, got, rtol=1e-12 if dtype == torch.float64 else 1e-6)


def test_force_tc_rejects_shapes_outside_the_tensor_path(be):
    x = _dev(be, _data(100, 100, 3, 0), torch.float32)
    pack = _pack(be, _data(10, 100, 3, 1), torch.float32)
    with pytest.raises(RuntimeError, match="not supported"):
        _colsum(be, x, pack, 10, 0.01, _lib.FLAG_FORCE_TC)


# ---------------------------------------------------------------------------------------------- embedding rows
def _embed_ref(Xq, keep, W, gamma):
    d2 = _d2(Xq, keep)
    m = d2.min(1, keepdim=True).values
    e = torch.exp(-gamma * (d2 - m)) @ torch.as_tensor(W, dtype=torch.float64, device="cuda")
    return (e / torch.sqrt((e * e).sum(1, keepdim=True))).cpu().numpy(), m[:, 0].cpu().numpy()


@pytest.mark.parametrize("n,d,l,k,dtype,flags", [
    (40_001, 64, 256, 64, torch.float32, 0),
    (20_000, 41, 100, 8, torch.float32, 0),
    (10_000, 7, 30, 3, torch.float32, 0),
    (3_000, 13, 5, 1, torch.float32, 0),
    (10_000, 41, 100, 65, torch.float32, 0),                    # k > 64: CUDA cores
    (10_000, 41, 100, 8, torch.float32, _lib.FLAG_FORCE_SIMT),
    (4_000, 16, 60, 8, torch.float64, 0),
])
def test_embed_matches_float64(be, n, d, l, k, dtype, flags):
    X = _data(n, d, 10, n + k)
    gamma = 1.0 / d
    keep = X[np.random.RandomState(2).choice(n, l, replace=False)]
    W = np.random.RandomState(3).standard_normal((l, k))
    x = _dev(be, X, dtype)
    Xq = x.double().cpu().numpy()
    pack = _pack(be, keep, dtype)
    Wq = W.astype(np.float32).astype(np.float64) if dtype == torch.float32 else W
    got = _embed(be, x, pack, l, gamma, W, flags)
    want, _ = _embed_ref(Xq, keep, Wq, gamma)
    err = np.abs(got.astype(np.float64) - want).max()
    assert err < (1e-12 if dtype == torch.float64 else 1e-4), err
    np.testing.assert_array_equal(_embed(be, x, pack, l, gamma, W, flags), got)


@pytest.mark.parametrize("flags", [0, _lib.FLAG_FORCE_SIMT])
def test_embed_far_rows_are_shifted_and_unreachable_rows_are_nan(be, flags):
    rng = np.random.RandomState(4)
    d, l, k, gamma = 8, 40, 4, 1.0
    keep = rng.standard_normal((l, d))
    near = keep[rng.randint(0, l, 500)] + 0.3 * rng.standard_normal((500, d))
    u = rng.standard_normal((1000, d))
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    far = keep[rng.randint(0, l, 1000)] + u * 20.0                    # gamma * min d^2 of a few hundred
    gone = keep[rng.randint(0, l, 100)] + u[:100] * 100.0             # gamma * min d^2 about 1e4
    X = np.concatenate([near, far, gone])
    W = rng.standard_normal((l, k))
    x = _dev(be, X, torch.float32)
    Xq = x.double().cpu().numpy()
    got = _embed(be, x, _pack(be, keep, torch.float32), l, gamma, W, flags).astype(np.float64)
    want, m = _embed_ref(Xq, keep, W.astype(np.float32).astype(np.float64), gamma)
    ok = gamma * m <= 745.13
    assert np.all(gamma * m[500:1500] > 110) and ok[:1500].all() and not ok[1500:].any()
    assert np.abs(got[:1500] - want[:1500]).max() < 1e-3
    assert np.isnan(got[1500:]).all()
    # the unshifted fp32 kernel values underflow on the far rows (the point of the shift)
    assert np.all(np.exp(-gamma * m[500:1500]).astype(np.float32) == 0)


# ---------------------------------------------------------------------------------------------- power-of-two scale
@pytest.mark.parametrize("flags", [0, _lib.FLAG_FORCE_SIMT])
def test_scaling_x_by_a_power_of_two_changes_nothing(be, flags):
    from _util import grid_blobs

    d, l, k = 16, 64, 6
    X = grid_blobs(20_000, d, 8, 5, 2.0 ** -12, 2.0 ** 4)
    keep = X[np.random.RandomState(6).choice(len(X), l, replace=False)]
    W = np.random.RandomState(7).standard_normal((l, k))
    gamma = 0.1
    res = []
    for p in (-40, 0, 40):
        s = 2.0 ** p
        x = _dev(be, X * s, torch.float32)
        pack = _pack(be, keep * s, torch.float32)
        g = gamma * 4.0 ** -p
        res.append((_colsum(be, x, pack, l, g, flags), _embed(be, x, pack, l, g, W, flags)))
    for c, e in res[1:]:
        np.testing.assert_array_equal(c, res[0][0])
        np.testing.assert_array_equal(e, res[0][1])


# ---------------------------------------------------------------------------------------------- the estimator
def _recorder():
    from sklearn.base import BaseEstimator

    class Rec(BaseEstimator):
        def __init__(self, n_clusters=2):
            self.n_clusters = n_clusters

        def fit(self, X, y=None):
            self.X_ = np.asarray(X)
            self.labels_ = np.zeros(len(self.X_), dtype=np.int32)
            return self

    return Rec()


@pytest.mark.parametrize("name", ["ref_spectral_f64_2000x5", "ref_spectral_f32_gamma_none", "ref_spectral_kmeans_branch",
                                  "ref_spectral_test_basic"])
def test_estimator_reproduces_the_reference(name, monkeypatch):
    """End to end against fixtures written by the reference's own spectral.py (tests/golden/ref_spectral.py)."""
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.cluster import SpectralClustering, spectral
    from test_spectral_host import RecordingRandomState, load_fixture

    fx = load_fixture(name)
    seen = {}

    class KM(spectral.KMeans):
        def fit(self, X, y=None):
            seen["seed"] = self.random_state
            seen["U"] = torch.cat([c.cpu() for c in X.chunks]).numpy()
            return super().fit(X)

    monkeypatch.setattr(spectral, "KMeans", KM)
    rs = RecordingRandomState(fx["seed"])
    kw = dict(n_clusters=fx["k"], n_components=fx["l"], gamma=fx["gamma"], random_state=rs)
    if fx["km_seed"] < 0:
        rec = _recorder()
        sc = SpectralClustering(assign_labels=rec, **kw).fit(ChunkedArray.from_array(fx["X"], fx["chunks"]))
        U = rec.X_
    else:
        sc = SpectralClustering(**kw).fit(ChunkedArray.from_array(fx["X"], fx["chunks"]))
        U = seen["U"]
        assert seen["seed"] == fx["km_seed"]
        assert len(sc.labels_.compute()) == len(fx["X"])
    np.testing.assert_array_equal(rs.chosen, fx["keep"])
    f64 = fx["X"].dtype == np.float64
    assert so.procrustes_err(U, fx["U2"]) < (1e-9 if f64 else 1e-4)
    np.testing.assert_allclose(sc.eigenvalues_, fx["S"], rtol=1e-9 if f64 else 1e-5)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_embedding_is_fitted_in_place_and_host_resident_input_agrees(dtype):
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.cluster import SpectralClustering, spectral
    from dask_ml_b200.engine import host_resident

    X = _data(30_000, 6, 5, 8, scale=3.0).astype(dtype)
    seen = {}

    class KM(spectral.KMeans):
        def fit(self, Xd, y=None):
            seen["chunks"] = list(Xd.chunks)
            return super().fit(Xd)

    old = spectral.KMeans
    spectral.KMeans = KM
    try:
        lib = _lib.load()
        before = int(lib.bkm_debug_fallback_count())
        a = SpectralClustering(n_clusters=5, n_components=50, gamma=0.5, random_state=3).fit(
            ChunkedArray.from_array(X, 10_000))
        assert int(lib.bkm_debug_fallback_count()) == before          # every KMeans chunk call on its own kernel family
        emb = seen["chunks"]
        b = SpectralClustering(n_clusters=5, n_components=50, gamma=0.5, random_state=3).fit(
            host_resident(ChunkedArray.from_array(X, 10_000), block_rows=10_000))
        emb_h = seen["chunks"]
    finally:
        spectral.KMeans = old
    want = torch.float32 if dtype == np.float32 else torch.float64
    for e in emb:
        assert e.dtype == want and e.is_cuda
        if want == torch.float32:
            assert e.stride(0) % 4 == 0                               # 16-byte rows: the tensor path reads it in place
    # the same row partition streamed from host memory: the same kernels in the same order, the same bits
    np.testing.assert_array_equal(torch.cat([e.cpu() for e in emb]).numpy(), torch.cat([e.cpu() for e in emb_h]).numpy())
    np.testing.assert_array_equal(a.eigenvalues_, b.eigenvalues_)
    assert len(a.labels_.compute()) == len(X)


def test_rings_are_separated():
    """Two concentric rings, 100k fp32 rows.  Parameters chosen on the float64 restatement: with n_clusters = 2 the
    Nystrom embedding cannot separate rings (the outer ring's first angular mode outranks the ring indicator whenever
    the kernel is narrow enough to decouple the rings), with 6 embedding columns it does; the 2-way split of that
    embedding is then a k-means problem with a poor local minimum, so the label step runs 10 k-means restarts."""
    import sklearn.cluster
    from sklearn.datasets import make_circles
    from sklearn.metrics import adjusted_rand_score

    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.cluster import KMeans, SpectralClustering

    X, y = make_circles(n_samples=100_000, factor=0.4, noise=0.04, random_state=0)
    X = X.astype(np.float32)
    km = sklearn.cluster.KMeans(2, n_init=10, random_state=0)
    sc = SpectralClustering(n_clusters=6, n_components=200, gamma=5.0, random_state=0, assign_labels=km,
                            kmeans_params={"n_clusters": 2}).fit(ChunkedArray.from_array(X, 40_000))
    got = np.asarray(sc.labels_)
    keep, _ = so.keep_rows(len(X), 200, 0, kmeans_branch=False)
    U_ref, _ = so.embed_fused(X.astype(np.float64), keep, 6, 5.0)
    want = sklearn.cluster.KMeans(2, n_init=10, random_state=0).fit_predict(U_ref)
    assert adjusted_rand_score(want, got) >= 0.999
    assert adjusted_rand_score(y, got) >= 0.999
    plain = KMeans(2, random_state=0).fit(ChunkedArray.from_array(X, 40_000))
    assert adjusted_rand_score(y, plain.labels_.compute()) < 0.5


def test_bfloat16_input_runs_in_float32():
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.cluster import SpectralClustering

    X = _data(20_000, 8, 4, 13, scale=3.0).astype(np.float32)
    Xb = torch.as_tensor(X).to(torch.bfloat16)
    Xq = Xb.float().numpy()                                           # the rows as bf16 stores them
    r1, r2 = _recorder(), _recorder()
    a = SpectralClustering(n_clusters=4, n_components=60, gamma=0.3, random_state=2, assign_labels=r1).fit(
        ChunkedArray([Xb[:12_000].cuda(), Xb[12_000:].cuda()]))
    b = SpectralClustering(n_clusters=4, n_components=60, gamma=0.3, random_state=2, assign_labels=r2).fit(
        ChunkedArray.from_array(Xq, 12_000))
    assert r1.X_.dtype == np.float32
    np.testing.assert_array_equal(r1.X_, r2.X_)
    np.testing.assert_array_equal(a.eigenvalues_, b.eigenvalues_)


def test_many_keep_rows_run_in_blocks(be):
    """l = 20000 float64 keep rows exceed one CTA's shared memory: the CUDA-core kernel walks them in blocks."""
    n, d, l, k, gamma = 3_000, 4, 20_000, 3, 0.5
    X = _data(n, d, 6, 21)
    keep = _data(l, d, 6, 22)
    W = np.random.RandomState(5).standard_normal((l, k))
    x = _dev(be, X, torch.float64)
    pack = _pack(be, keep, torch.float64)
    got = _colsum(be, x, pack, l, gamma)
    np.testing.assert_allclose(got, torch.exp(-gamma * _d2(X, keep)).sum(0).cpu().numpy(), rtol=1e-12)
    e = _embed(be, x, pack, l, gamma, W)
    want, _ = _embed_ref(X, keep, W, gamma)
    assert np.abs(e - want).max() < 1e-12


# ---------------------------------------------------------------------------------------------- reference test ports
def _ref_X():
    from dask_ml_b200.datasets import make_blobs

    return make_blobs(n_samples=200, chunks=100, random_state=0)


@pytest.mark.parametrize("as_ndarray", [False, True])
@pytest.mark.parametrize("persist_embedding", [True, False])
def test_basic(as_ndarray, persist_embedding):
    from dask_ml_b200.cluster import SpectralClustering

    X, _ = _ref_X()
    sc = SpectralClustering(n_components=25, random_state=0, persist_embedding=persist_embedding)
    X_ = X.compute() if as_ndarray else X
    sc.fit(X_)
    assert len(sc.labels_) == len(X_)


@pytest.mark.parametrize("assign_labels", ["estimator", "sklearn-kmeans"])
def test_sklearn_kmeans(assign_labels):
    import sklearn.cluster

    from dask_ml_b200.cluster import SpectralClustering

    X, _ = _ref_X()
    al = sklearn.cluster.KMeans(n_init=2) if assign_labels == "estimator" else assign_labels
    sc = SpectralClustering(n_components=25, random_state=0, assign_labels=al, kmeans_params={"n_clusters": 8})
    sc.fit(X)
    assert isinstance(sc.assign_labels_, sklearn.cluster.KMeans)


def test_callable_affinity():
    from dask_ml_b200 import metrics
    from dask_ml_b200.cluster import SpectralClustering

    X, _ = _ref_X()
    affinity = partial(metrics.pairwise.pairwise_kernels, metric="rbf", filter_params=True)
    sc = SpectralClustering(affinity=affinity)
    sc.fit(X)


def test_n_components_raises():
    from dask_ml_b200.cluster import SpectralClustering

    X, _ = _ref_X()
    sc = SpectralClustering(n_components=len(X))
    with pytest.raises(ValueError) as m:
        sc.fit(X)
    assert m.match("n_components")


def test_assign_labels_raises():
    from dask_ml_b200.cluster import SpectralClustering

    X, _ = _ref_X()
    with pytest.raises(ValueError) as m:
        SpectralClustering(assign_labels="foo").fit(X)
    assert m.match("Unknown 'assign_labels' 'foo'")
    with pytest.raises(TypeError) as m:
        SpectralClustering(assign_labels=dict()).fit(X)
    assert m.match("Invalid type ")


def test_affinity_raises():
    from dask_ml_b200.cluster import SpectralClustering

    X, _ = _ref_X()
    with pytest.raises(ValueError) as m:
        SpectralClustering(affinity="foo").fit(X)
    assert m.match("Unknown affinity metric name 'foo'")
    with pytest.raises(TypeError):
        SpectralClustering(affinity=np.array([])).fit(X)


def test_spectral_clustering():
    from dask_ml_b200.cluster import SpectralClustering
    from dask_ml_b200.datasets import make_blobs

    # the reference's Xl_blobs_easy fixture (tests/conftest.py:60-68)
    centers = np.array([[-7, -7], [0, 0], [7, 7]])
    X, y = make_blobs(cluster_std=0.1, centers=centers, chunks=50, random_state=0)
    X = X.compute()
    X = (X - X.mean(0)) / X.std(0)
    model = SpectralClustering(random_state=0, n_clusters=3, n_components=5, gamma=None).fit(X)
    labels = model.labels_.compute()
    y = y.compute()
    idx = [(y == i).argmax() for i in range(3)]
    grouped_idx = [np.where(y == y[idx[i]])[0] for i in range(3)]
    for indices in grouped_idx:
        assert len(set(labels[indices])) == 1


# ---------------------------------------------------------------------------------------------- several GPUs
def test_multi_gpu_embedding_equals_single_gpu(tmp_path):
    world = min(torch.cuda.device_count(), 8)
    if world < 2:
        pytest.skip("needs at least 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world),
           "--master-addr", "127.0.0.1", "--master-port", "29581",
           os.path.join(ROOT, "tests", "dist_spectral_worker.py"), str(tmp_path)]
    subprocess.run(cmd, check=True, timeout=600, cwd=ROOT)
    import dist_spectral_worker as w

    U, S = w.single_gpu()
    for r in range(world):
        g = np.load(tmp_path / ("rank%d.npz" % r))
        assert np.abs(g["U"] - U).max() < 1e-6
        np.testing.assert_array_equal(g["S"], np.load(tmp_path / "rank0.npz")["S"])
        np.testing.assert_allclose(g["S"], S, rtol=1e-6)
