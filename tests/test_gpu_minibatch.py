"""PartialMiniBatchKMeans on the H100: ``bkm_minibatch_step`` against its float64 expression and against
``bkm_pack_centers``, the reference fixtures, every kernel family against the checker backend of
tests/test_minibatch_host.py, host-resident input, and the calls a fit issues per block."""
import json
import os
import sys
import warnings

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
GOLDEN = os.path.join(ROOT, "tests", "golden")

from dask_ml_b200 import ChunkedArray  # noqa: E402
from dask_ml_b200.cluster import PartialMiniBatchKMeans, k_means as km  # noqa: E402
from dask_ml_b200.engine import CudaBackend, host_resident  # noqa: E402

pytestmark = [pytest.mark.gpu,
              pytest.mark.filterwarnings("ignore:'PartialMiniBatchKMeans' is deprecated:FutureWarning")]

FIXTURES = sorted(f[:-4] for f in os.listdir(GOLDEN) if f.startswith("ref_minibatch_") and f.endswith(".npz"))


@pytest.fixture(scope="module")
def be():
    return CudaBackend()


@pytest.fixture(autouse=True)
def no_fallback(be):
    """No chunk of a tensor-core / streaming shape ran on the generic kernel (the library's counter, which does not
    depend on what earlier tests of the session did, unlike the once-per-process warning)."""
    before = int(be.lib.bkm_debug_fallback_count())
    yield
    assert int(be.lib.bkm_debug_fallback_count()) == before


def _step_inputs(k, d, seed):
    rng = np.random.RandomState(seed)
    c = rng.standard_normal((k, d)) * 5
    w = rng.randint(0, 5000, size=k).astype(np.float64)
    n = rng.randint(0, 300, size=k).astype(np.float64)
    n[::7] = 0.0                                                # clusters the batch does not touch
    S = rng.standard_normal((k, d)) * 40 + n[:, None] * c
    red = np.concatenate([S.ravel(), n, [123.5]])
    with np.errstate(divide="ignore", invalid="ignore"):
        want = np.where((n > 0)[:, None], (c * w[:, None] + S) * (1.0 / (w + n))[:, None], c)
    return red, c, w, n, want


# k*d <= 64 K with the staged centres in shared memory / without them; a large shape (three kernels)
SHAPES = [(256, 64), (32, 5), (2048, 32), (1024, 128)]


@pytest.mark.parametrize("k,d", SHAPES)
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64, torch.bfloat16])
def test_step_is_the_float64_expression_and_packs_like_pack_centers(be, k, d, dtype):
    if dtype == torch.bfloat16 and (d % 8 or d > 128):
        pytest.skip("bf16 rows: d a multiple of 8, <= 128")
    red, c, w, n, want = _step_inputs(k, d, k + d)
    dev = be.device
    t = lambda a: torch.as_tensor(np.ascontiguousarray(a)).to(dev)
    red_d, c_in, w_in = t(red), t(c), t(w)
    c_out, w_out = be.empty((k, d), torch.float64), be.empty((k,), torch.float64)
    # both packs start from the same bytes, so that bytes neither writer touches compare equal too
    pack = be.pack_centers(c_in, dtype)
    pack.fill_(0xA5)
    be.minibatch_step(red_d, c_in, w_in, c_out, w_out, pack, dtype)
    got_c, got_w = c_out.cpu().numpy(), w_out.cpu().numpy()
    np.testing.assert_array_equal(got_c.view(np.uint64), want.view(np.uint64))
    np.testing.assert_array_equal(got_w, w + n)
    np.testing.assert_array_equal(c_in.cpu().numpy(), c)                       # inputs untouched
    ref = be.pack_centers(c_out.clone(), dtype, out=torch.full_like(pack, 0xA5))
    assert torch.equal(pack, ref)


def test_step_rejects_in_place_buffers(be):
    red, c, w, n, _ = _step_inputs(8, 4, 0)
    c_in = torch.as_tensor(c).to(be.device)
    w_in = torch.as_tensor(w).to(be.device)
    pack = be.pack_centers(c_in, torch.float32)
    with pytest.raises(RuntimeError, match="invalid argument"):
        be.minibatch_step(torch.as_tensor(red).to(be.device), c_in, w_in, c_in, w_in.clone(), pack, torch.float32)


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
    rtol = 1e-9 if X.dtype == np.float64 else 1e-4
    np.testing.assert_allclose(est.cluster_centers_, z["centers"], rtol=rtol, atol=rtol * 10)
    np.testing.assert_array_equal(est._counts, z["counts"])
    assert est.n_steps_ == int(z["n_steps"])
    assert est.labels_.blocks[0].is_cuda if z["labels"].size else not hasattr(est, "labels_")
    if z["labels"].size:
        np.testing.assert_array_equal(est.labels_.compute(), z["labels"])
        np.testing.assert_allclose(est.inertia_, float(z["inertia"]), rtol=rtol)


def _blobs(n, d, k, seed, dtype):
    rng = np.random.RandomState(seed)
    cent = rng.uniform(-20, 20, size=(k, d))
    return (cent[rng.randint(0, k, size=n)] + 0.5 * rng.standard_normal((n, d))).astype(dtype)


# (n, d, k, dtype, family): fp32 tensor cores; tiny k*d (streaming kernel); bf16 tensor cores; float64 / odd d
FAMILIES = {
    "fp32_tc": (24000, 32, 128, np.float32, 1),
    "tiny": (24000, 4, 8, np.float32, 2),
    "bf16": (24000, 128, 1024, "bf16", 3),
    "f64_odd_d": (12000, 7, 10, np.float64, 0),
}


@pytest.mark.parametrize("name", sorted(FAMILIES))
def test_each_kernel_family_matches_the_checker(be, monkeypatch, name):
    from test_minibatch_host import MiniBatchChecker

    n, d, k, dtype, family = FAMILIES[name]
    X = _blobs(n, d, k // 2 if name == "bf16" else k, 3, np.float32 if dtype == "bf16" else dtype)
    tdt = torch.bfloat16 if dtype == "bf16" else {np.float32: torch.float32, np.float64: torch.float64}[dtype]
    assert be.kernel_family(d, k, tdt) == family
    if dtype == "bf16":
        X = torch.from_numpy(X).to(torch.bfloat16)
        Xh = X.float().numpy()                                   # the same values for the checker
        blocks = ChunkedArray([X[i:i + 4000] for i in range(0, n, 4000)])
    else:
        Xh = X
        blocks = ChunkedArray.from_array(X, 4000)
    kw = dict(n_clusters=k, random_state=0, batch_size=4000, init=Xh[:k].copy())
    np.random.seed(5)
    a = PartialMiniBatchKMeans(**kw).fit(blocks)
    monkeypatch.setattr(km, "_BACKEND_FACTORY", MiniBatchChecker)
    np.random.seed(5)
    b = PartialMiniBatchKMeans(**kw).fit(ChunkedArray.from_array(Xh, 4000))
    np.testing.assert_array_equal(a._counts, b._counts)
    np.testing.assert_allclose(a.cluster_centers_, b.cluster_centers_, rtol=1e-6, atol=1e-5)
    np.testing.assert_array_equal(a.labels_.compute(), b.labels_.compute())
    np.testing.assert_allclose(a.inertia_, b.inertia_, rtol=1e-5)
    assert a.n_steps_ == b.n_steps_ == n // 4000


def test_host_resident_gives_the_same_bits():
    X = _blobs(30000, 16, 32, 4, np.float32)
    Xc = ChunkedArray.from_array(X, 5000)
    np.random.seed(9)
    a = PartialMiniBatchKMeans(n_clusters=32, random_state=1, reassignment_ratio=0.2).fit(Xc)
    np.random.seed(9)
    b = PartialMiniBatchKMeans(n_clusters=32, random_state=1, reassignment_ratio=0.2).fit(
        host_resident(Xc, block_rows=5000))
    np.testing.assert_array_equal(a.cluster_centers_, b.cluster_centers_)
    np.testing.assert_array_equal(a._counts, b._counts)
    np.testing.assert_array_equal(a.labels_.compute(), b.labels_.compute())
    assert a.inertia_ == b.inertia_
    np.testing.assert_array_equal(a.predict(X).compute(), b.predict(host_resident(X)).compute())


def test_later_batch_with_an_empty_first_block(be, monkeypatch):
    """The empty block launches nothing; the step's sums are those of the second batch only (the checker treats an
    empty chunk as the library does)."""
    from test_minibatch_host import MiniBatchChecker

    X = _blobs(6000, 32, 128, 8, np.float32)
    out = []
    for factory in (CudaBackend, MiniBatchChecker):
        monkeypatch.setattr(km, "_BACKEND_FACTORY", factory)
        est = PartialMiniBatchKMeans(n_clusters=128, random_state=0, init=X[:128].copy())
        est.partial_fit(X[:2000])
        est.partial_fit(ChunkedArray.from_array(X[2000:], ((0, 2000, 2000),)))
        out.append(est)
    a, b = out
    np.testing.assert_array_equal(a._counts, b._counts)
    np.testing.assert_allclose(a.cluster_centers_, b.cluster_centers_, rtol=1e-6, atol=1e-5)
    np.testing.assert_array_equal(a.labels_.compute(), b.labels_.compute())


class _Counting(CudaBackend):
    """Records, per backend call, how many kernels the library launched during it."""

    calls = None

    def _counted(self, name, fn, *a, **k):
        before = self.launch_count()
        out = fn(*a, **k)
        _Counting.calls.setdefault(name, []).append(self.launch_count() - before)
        return out

    def lloyd_chunk(self, *a, **k):
        return self._counted("lloyd_chunk", super().lloyd_chunk, *a, **k)

    def minibatch_step(self, *a, **k):
        return self._counted("minibatch_step", super().minibatch_step, *a, **k)

    def pack_centers(self, *a, **k):
        return self._counted("pack_centers", super().pack_centers, *a, **k)

    def assign_chunk(self, *a, **k):
        return self._counted("assign_chunk", super().assign_chunk, *a, **k)

    def check_finite(self, *a, **k):
        return self._counted("check_finite", super().check_finite, *a, **k)


def test_launches_per_block(be, monkeypatch):
    from test_minibatch_host import CountingRandomState

    k, d, rows = 40, 8, 1000
    X = _blobs(12 * rows, d, 4, 6, np.float32)               # 40 centres on 4 blobs: some get few rows, reassigned
    # launches of one fused E+M call and of one relabel call on a block of this shape
    x = be.to_device(X[:rows], torch.float32)
    red = be.zeros((k * d + k + 1,), torch.float64)
    pack = be.pack_centers(torch.as_tensor(X[:k].astype(np.float64)).to(be.device), torch.float32)
    n0 = be.launch_count()
    be.lloyd_chunk(x, pack, k, None, None, red[: k * d], red[k * d: k * d + k], red[-1:], first=True)
    em = be.launch_count() - n0
    n0 = be.launch_count()
    be.assign_chunk(x, pack, k, be.empty((rows,), torch.int32), None, True, be.zeros((1,), torch.float64))
    relabel = be.launch_count() - n0

    monkeypatch.setattr(km, "_BACKEND_FACTORY", _Counting)
    _Counting.calls = {}
    rs = CountingRandomState(0)
    n0 = be.launch_count()
    PartialMiniBatchKMeans(n_clusters=k, batch_size=rows, reassignment_ratio=0.2, random_state=rs).fit(
        ChunkedArray.from_array(X, rows))
    total = be.launch_count() - n0
    assert rs.reassign_draws > 0
    c = _Counting.calls
    assert c["lloyd_chunk"] == [em] * 12                           # per block: one fused E+M pass ...
    assert c["minibatch_step"] == [1] * 12                         # ... and one step kernel (small shape)
    assert c["pack_centers"] == [1] * (1 + rs.reassign_draws)      # the initial pack, then one per reassignment
    assert c["assign_chunk"] == [relabel]                          # one relabel, after the last block
    assert total == sum(sum(v) for v in c.values())                # no other library launch
