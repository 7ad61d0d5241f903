"""PartialMiniBatchKMeans on CPU: the host control flow of scikit-learn's ``partial_fit`` and the reference's block-wise
``fit``, with the device kernels replaced by a float64 numpy checker backend.

Pins the estimator against live scikit-learn ``MiniBatchKMeans.partial_fit`` sequences (reassignment steps included),
replays the reference fixtures tests/golden/ref_minibatch_*.npz (tests/golden/ref_minibatch.py), covers the error
contract and ports the reference's tests/test_minibatch.py."""
import json
import os
import socket
import sys
import warnings

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp
from sklearn.base import clone
from sklearn.cluster import MiniBatchKMeans

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
GOLDEN = os.path.join(ROOT, "tests", "golden")

from oracle_backend import OracleBackend  # noqa: E402

from dask_ml_b200 import ChunkedArray  # noqa: E402
from dask_ml_b200.cluster import PartialMiniBatchKMeans, k_means as km  # noqa: E402

DEPRECATION = ("'PartialMiniBatchKMeans' is deprecated. Use 'dask_ml.wrappers.Incremental(MiniBatchKMeans(), "
               "**kwargs)' instead.")
FIXTURES = sorted(f[:-4] for f in os.listdir(GOLDEN) if f.startswith("ref_minibatch_") and f.endswith(".npz"))

pytestmark = pytest.mark.filterwarnings("ignore:'PartialMiniBatchKMeans' is deprecated:FutureWarning")


class MiniBatchChecker(OracleBackend):
    """The oracle backend plus the two calls of a mini-batch step: the fused E+M pass with FIRST_CHUNK and float64
    counts, and ``minibatch_step`` as the float64 numpy expression of scikit-learn's _minibatch_update_dense."""

    steps = 0

    # like the library, a chunk without rows is a no-op whatever the flags say
    def lloyd_chunk(self, x, pack, k, labels, min_d2, sums, counts, inertia, first=False, loop_state=None):
        if int(x.shape[0]) == 0:
            return
        if first:
            sums.zero_()
            counts.zero_()
            if inertia is not None:
                inertia.zero_()
        super().lloyd_chunk(x, pack, k, labels, min_d2, sums, counts, inertia)

    def assign_chunk(self, x, pack, k, labels, min_dist, squared, dist_sum):
        if int(x.shape[0]):
            super().assign_chunk(x, pack, k, labels, min_dist, squared, dist_sum)

    def minibatch_step(self, red, c_in, w_in, c_out, w_out, pack, dtype):
        MiniBatchChecker.steps += 1
        k, d = c_in.shape
        r = red.numpy()
        S, n = r[: k * d].reshape(k, d), r[k * d: k * d + k]
        c, w = c_in.numpy(), w_in.numpy()
        with np.errstate(divide="ignore", invalid="ignore"):
            upd = (c * w[:, None] + S) * (1.0 / (w + n))[:, None]
        c_out.copy_(torch.from_numpy(np.where((n > 0)[:, None], upd, c)))
        w_out.copy_(torch.from_numpy(w + n))
        pack.copy_(c_out)


@pytest.fixture(autouse=True)
def checker(monkeypatch):
    monkeypatch.setattr(km, "_BACKEND_FACTORY", MiniBatchChecker)


def _blobs(n, d, k, seed, weights=None, dtype=np.float64):
    rng = np.random.RandomState(seed)
    cent = rng.uniform(-10, 10, size=(k, d))
    return (cent[rng.choice(k, size=n, p=weights)] + rng.standard_normal((n, d))).astype(dtype)


class CountingRandomState(np.random.RandomState):
    """Counts the reassignment draws (``choice`` without replacement and without weights)."""

    reassign_draws = 0

    def choice(self, a, size=None, replace=True, p=None):
        if not replace and p is None:
            self.reassign_draws += 1
        return super().choice(a, size=size, replace=replace, p=p)


def _assert_same_state(a, b, rtol=1e-12):
    np.testing.assert_allclose(a.cluster_centers_, b.cluster_centers_, rtol=rtol, atol=rtol)
    np.testing.assert_array_equal(a._counts, b._counts)
    assert a._counts.dtype == b._counts.dtype
    assert a.n_steps_ == b.n_steps_
    assert a._n_since_last_reassign == b._n_since_last_reassign
    if hasattr(b, "labels_"):
        np.testing.assert_array_equal(a.labels_.compute(), b.labels_)
        np.testing.assert_allclose(a.inertia_, b.inertia_, rtol=rtol)


# ---------------------------------------------------------------------------------------------------------------
# live scikit-learn partial_fit sequences
# ---------------------------------------------------------------------------------------------------------------
SEQUENCES = {
    "kmeans++": (dict(n_clusters=5), [(700, 3)] * 4),
    "random": (dict(n_clusters=4, init="random"), [(500, 2)] * 3),
    "batch_sizes": (dict(n_clusters=6, batch_size=300), [(300, 4), (520, 4), (260, 4), (900, 4)]),
    "reassign": (dict(n_clusters=20, batch_size=60, reassignment_ratio=0.2), [(60, 3)] * 10),
    "no_labels": (dict(n_clusters=3, compute_labels=False), [(400, 5)] * 3),
}


@pytest.mark.parametrize("name", sorted(SEQUENCES))
def test_matches_sklearn_partial_fit(name):
    kw, shapes = SEQUENCES[name]
    weights = [0.45, 0.45, 0.1] if name == "reassign" else None
    blocks = [_blobs(n, d, 3 if weights else 5, 10 + i, weights) for i, (n, d) in enumerate(shapes)]
    a = PartialMiniBatchKMeans(random_state=CountingRandomState(7), **kw)
    b = MiniBatchKMeans(random_state=CountingRandomState(7), **kw)
    for blk in blocks:
        a.partial_fit(blk)
        b.partial_fit(blk)
        _assert_same_state(a, b)
    st_a, st_b = a._random_state.get_state(), b._random_state.get_state()
    np.testing.assert_array_equal(st_a[1], st_b[1])
    assert st_a[2:] == st_b[2:]
    assert a._random_state.reassign_draws == b._random_state.reassign_draws
    if name == "reassign":
        assert a._random_state.reassign_draws > 0
    if name == "no_labels":
        assert not hasattr(a, "labels_")


def test_array_init_and_int_seed():
    X = _blobs(900, 4, 4, 3)
    init = X[:4].copy()
    a = PartialMiniBatchKMeans(n_clusters=4, init=init, random_state=0)
    b = MiniBatchKMeans(n_clusters=4, init=init, random_state=0)
    for blk in (X[:300], X[300:600], X[600:]):
        a.partial_fit(blk)
        b.partial_fit(blk)
    _assert_same_state(a, b)
    np.testing.assert_array_equal(init, X[:4])         # the caller's init is not modified


@pytest.mark.parametrize("sizes", [(0, 250, 250), (250, 0, 250), (250, 250, 0)])
def test_batch_with_an_empty_block(sizes):
    """A later batch whose blocks include an empty one: the step's sums start from that batch's first rows, not from
    what the previous batch left in the accumulators."""
    X = _blobs(900, 3, 4, 8)
    a = PartialMiniBatchKMeans(n_clusters=4, random_state=0)
    b = MiniBatchKMeans(n_clusters=4, random_state=0)
    a.partial_fit(X[:400])
    b.partial_fit(X[:400])
    a.partial_fit(ChunkedArray.from_array(X[400:900], (sizes,)))
    b.partial_fit(X[400:900])
    _assert_same_state(a, b)


def test_fit_is_partial_fit_per_block_in_shuffled_order():
    X = _blobs(2000, 3, 4, 5)
    a = PartialMiniBatchKMeans(n_clusters=4, random_state=0)
    np.random.seed(11)
    a.fit(ChunkedArray.from_array(X, 500))
    np.random.seed(11)
    order = list(range(4))
    np.random.shuffle(order)
    b = MiniBatchKMeans(n_clusters=4, random_state=0)
    for i in order:
        b.partial_fit(X[i * 500:(i + 1) * 500])
    _assert_same_state(a, b)
    assert len(a.labels_.compute()) == 500
    # a second fit continues from the learned state
    a.fit(ChunkedArray.from_array(X, 500))
    assert a.n_steps_ == 8


def test_fit_labels_only_after_the_last_block(monkeypatch):
    X = _blobs(1200, 3, 3, 6)
    calls = []
    orig = MiniBatchChecker.assign_chunk
    monkeypatch.setattr(MiniBatchChecker, "assign_chunk", lambda self, *a: (calls.append(1), orig(self, *a))[1])
    MiniBatchChecker.steps = 0
    PartialMiniBatchKMeans(n_clusters=3, random_state=0).fit(ChunkedArray.from_array(X, 300))
    assert MiniBatchChecker.steps == 4
    assert len(calls) == 1


@pytest.mark.parametrize("name", FIXTURES)
def test_replays_reference_fixture(name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    params = json.loads(str(z["params"]))
    init = str(z["init"]) if z["init"].dtype.kind == "U" else z["init"]
    X = z["X"]
    np.random.seed(int(z["seed"]))
    est = PartialMiniBatchKMeans(init=init, **params)
    for _ in range(int(z["n_fits"])):
        est.fit(ChunkedArray.from_array(X, int(z["rows"])))
    rtol = 1e-12 if X.dtype == np.float64 else 1e-4
    np.testing.assert_allclose(est.cluster_centers_, z["centers"], rtol=rtol, atol=rtol * 10)
    assert est.cluster_centers_.dtype == X.dtype
    np.testing.assert_array_equal(est._counts, z["counts"])
    assert est.n_steps_ == int(z["n_steps"])
    if z["labels"].size:
        np.testing.assert_array_equal(est.labels_.compute(), z["labels"])
        np.testing.assert_allclose(est.inertia_, float(z["inertia"]), rtol=rtol)
    else:
        assert not hasattr(est, "labels_")


# ---------------------------------------------------------------------------------------------------------------
# API and error contract
# ---------------------------------------------------------------------------------------------------------------
def test_future_warning_text():
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        PartialMiniBatchKMeans(n_clusters=3)
    assert [str(x.message) for x in w if x.category is FutureWarning] == [DEPRECATION]


def test_params_repr_clone():
    a = PartialMiniBatchKMeans(n_clusters=3, batch_size=50, random_state=1)
    assert a.get_params() == MiniBatchKMeans(n_clusters=3, batch_size=50, random_state=1).get_params()
    b = clone(a)
    assert type(b) is PartialMiniBatchKMeans and b.get_params() == a.get_params()
    assert repr(a).startswith("PartialMiniBatchKMeans(")


def test_sklearn_validation_messages():
    X = _blobs(100, 2, 3, 1)
    with pytest.raises(ValueError, match=r"n_samples=3 should be >= n_clusters=8\."):
        PartialMiniBatchKMeans().partial_fit(X[:3])
    with pytest.raises(ValueError, match="The 'batch_size' parameter of PartialMiniBatchKMeans must be an int"):
        PartialMiniBatchKMeans(batch_size=0).partial_fit(X)
    with pytest.raises(ValueError, match="The 'init' parameter of PartialMiniBatchKMeans must be"):
        PartialMiniBatchKMeans(init="k-means||").fit(X)
    with pytest.raises(ValueError, match=r"The shape of the initial centers \(3, 3\) does not match the number of "
                                         r"features of the data 2\."):
        PartialMiniBatchKMeans(n_clusters=3, init=np.zeros((3, 3))).partial_fit(X)


def test_feature_mismatch_on_a_later_batch():
    a = PartialMiniBatchKMeans(n_clusters=2, random_state=0).partial_fit(_blobs(50, 2, 2, 1))
    with pytest.raises(ValueError, match="X has 3 features, but PartialMiniBatchKMeans is expecting 2 features as input"):
        a.partial_fit(_blobs(50, 3, 2, 1))
    with pytest.raises(ValueError, match="X has 3 features"):
        a.predict(_blobs(50, 3, 2, 1))


def test_nan_input():
    X = _blobs(100, 2, 3, 1)
    X[7, 1] = np.nan
    with pytest.raises(ValueError, match="Input contains NaN"):
        PartialMiniBatchKMeans(n_clusters=3).fit(X)


def test_compute_false_and_sample_weight():
    X = _blobs(100, 2, 3, 1)
    with pytest.raises(NotImplementedError):
        PartialMiniBatchKMeans(n_clusters=3).fit(X, compute=False)
    with pytest.raises(NotImplementedError):
        PartialMiniBatchKMeans(n_clusters=3).partial_fit(X, sample_weight=np.ones(100))


def test_predict_transform_score():
    X = _blobs(600, 3, 3, 2)
    a = PartialMiniBatchKMeans(n_clusters=3, random_state=0).fit(X)
    b = MiniBatchKMeans(n_clusters=3, random_state=0).partial_fit(X)
    np.testing.assert_array_equal(np.asarray(a.predict(X).compute()), b.predict(X))
    np.testing.assert_allclose(np.asarray(a.transform(X).compute()), b.transform(X), rtol=1e-10)
    np.testing.assert_allclose(a.score(X), b.score(X), rtol=1e-10)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_pickle_keeps_the_float64_state(dtype):
    import pickle

    X = _blobs(900, 3, 3, 4, dtype=dtype)
    a = PartialMiniBatchKMeans(n_clusters=3, random_state=0).partial_fit(X[:300])
    b = pickle.loads(pickle.dumps(a))
    assert "_mb" not in vars(b)
    for blk in (X[300:600], X[600:]):
        a.partial_fit(blk)
        b.partial_fit(blk)
    # the float64 centres and weight sums continue bit for bit, not from values rounded to X's dtype
    assert torch.equal(a._mb.C, b._mb.C) and torch.equal(a._mb.W, b._mb.W)
    np.testing.assert_array_equal(a.cluster_centers_, b.cluster_centers_)
    np.testing.assert_array_equal(a._counts, b._counts)


# ---------------------------------------------------------------------------------------------------------------
# torch.distributed: every rank raises before any collective
# ---------------------------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _dist_worker(rank, world, port, out_dir):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    import torch.distributed as dist

    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from dask_ml_b200.cluster import PartialMiniBatchKMeans as P

        X = np.random.RandomState(rank).standard_normal((100 + 50 * rank, 2))
        got = []
        for call in (lambda e: e.fit(X), lambda e: e.partial_fit(X)):
            try:
                with warnings.catch_warnings():
                    warnings.simplefilter("ignore", FutureWarning)
                    call(P(n_clusters=2))
                got.append("no error")
            except NotImplementedError as e:
                got.append("NotImplementedError: %s" % e)
        with open(os.path.join(out_dir, "rank%d.json" % rank), "w") as f:
            json.dump(got, f)
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(300)
def test_two_ranks_raise_without_hanging(tmp_path):
    mp.start_processes(_dist_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True, start_method="spawn")
    for r in range(2):
        got = json.load(open(tmp_path / ("rank%d.json" % r)))
        assert len(got) == 2 and all(g.startswith("NotImplementedError") for g in got), got


# ---------------------------------------------------------------------------------------------------------------
# the reference's tests/test_minibatch.py
# ---------------------------------------------------------------------------------------------------------------
def test_basic():
    from sklearn.datasets import make_blobs

    X, _ = make_blobs(n_samples=100, random_state=0)           # one block of 100 rows (single_chunk_blobs)
    a = PartialMiniBatchKMeans(n_clusters=3, random_state=0)
    b = MiniBatchKMeans(n_clusters=3, random_state=0)
    a.fit(ChunkedArray.from_array(X, 100))
    b.partial_fit(X)
    left = {x for x in vars(a) if x.endswith("_") and not x.startswith("_")}
    right = {x for x in vars(b) if x.endswith("_") and not x.startswith("_")}
    assert left == right
    for attr in left:
        l, r = getattr(a, attr), getattr(b, attr)
        l = l.compute() if isinstance(l, ChunkedArray) else l
        np.testing.assert_allclose(l, r, rtol=1e-12, atol=1e-12)
