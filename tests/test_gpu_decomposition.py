"""PCA / TruncatedSVD on the H100: the Gram and projection kernels against float64 numpy, bit-reproducibility, the
launch count of a fit, and the estimators against scikit-learn."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DTYPES = {"f32": torch.float32, "f64": torch.float64, "bf16": torch.bfloat16}


def _backend():
    from dask_ml_b200.engine import CudaBackend

    return CudaBackend()


def _rows(n, d, dt, seed, pitch=None, offset=3.0):
    rng = np.random.RandomState(seed)
    X = rng.standard_normal((n, d)) * rng.uniform(0.5, 2, d) + offset
    t = torch.as_tensor(X).to(DTYPES[dt])
    if pitch is not None:
        buf = torch.zeros((n, pitch), dtype=t.dtype)
        buf[:, :d] = t
        t = buf[:, :d]
    x64 = t.to(torch.float64).numpy()          # what the kernel sees (bf16 / f32 rows widened exactly)
    return t.cuda(), x64


def _gram(be, chunks, shift):
    d = chunks[0].shape[1]
    G = torch.full((d, d), np.nan, dtype=torch.float64, device="cuda")
    m = torch.full((d,), np.nan, dtype=torch.float64, device="cuda")
    s = torch.as_tensor(shift).cuda()
    for i, x in enumerate(chunks):
        be.gram_chunk(x, s, m, G, first=i == 0)
    torch.cuda.synchronize()
    return G.cpu().numpy(), m.cpu().numpy()


def _rel(a, b):
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


@pytest.mark.parametrize("dt", ["f32", "f64", "bf16"])
@pytest.mark.parametrize("d", [1, 3, 13, 64, 100, 128, 256, 784])
def test_gram_matches_float64(dt, d):
    be = _backend()
    ns = [0, 1, 31, 33, 1000, 4096] if d <= 256 else [0, 1, 33, 2048]
    xs, hs = zip(*[_rows(n, d, dt, 10 + i) for i, n in enumerate(ns)])
    shift = np.linspace(2.5, 3.5, d)
    G, m = _gram(be, list(xs), shift)
    xc = np.concatenate(hs) - shift
    np.testing.assert_array_equal(G, G.T)
    assert _rel(G, xc.T @ xc) < 1e-12
    assert _rel(m, xc.sum(0)) < 1e-12
    G2, m2 = _gram(be, list(xs), shift)
    np.testing.assert_array_equal(G, G2)                 # fixed summation order: the same bits
    np.testing.assert_array_equal(m, m2)


@pytest.mark.parametrize("n", [0, 1, 2 ** 10, 2 ** 14, 2 ** 18, 2 ** 20 + 3])
def test_gram_power_of_two_scales(n):
    be = _backend()
    x, h = _rows(n, 64, "f32", 3)
    shift = np.full(64, 3.0)
    G, m = _gram(be, [x], shift)
    xc = h - shift
    assert _rel(G, xc.T @ xc) < 1e-12 if n else (np.all(G == 0) and np.all(m == 0))


@pytest.mark.parametrize("dt", ["f32", "f64", "bf16"])
def test_gram_unaligned_pitch(dt):
    be = _backend()
    x, h = _rows(777, 13, dt, 5, pitch=15)
    shift = np.zeros(13)
    G, m = _gram(be, [x], shift)
    assert _rel(G, h.T @ h) < 1e-12 and _rel(m, h.sum(0)) < 1e-12


@pytest.mark.parametrize("dt", ["f32", "f64", "bf16"])
@pytest.mark.parametrize("d,k", [(3, 2), (64, 16), (100, 40), (128, 64), (784, 70)])
def test_project_matches_float64(dt, d, k):
    be = _backend()
    x, h = _rows(5003, d, dt, 7)
    rng = np.random.RandomState(1)
    W = rng.standard_normal((k, d))
    shift = np.linspace(2.5, 3.5, d)
    odt = torch.float64 if dt == "f64" else torch.float32
    out = torch.empty((5003, k), dtype=torch.float64, device="cuda")
    rec = be.colmax_new(k)
    be.project_chunk(x[:2000], torch.as_tensor(shift).cuda(), torch.as_tensor(W).cuda(), out=out[:2000], colmax=rec,
                     row_offset=100)
    be.project_chunk(x[2000:], torch.as_tensor(shift).cuda(), torch.as_tensor(W).cuda(), out=out[2000:], colmax=rec,
                     row_offset=2100)
    t = (h - shift) @ W.T
    got = out.cpu().numpy()
    assert np.abs(got - t).max() <= 1e-12 * np.abs(t).max()
    r = rec.cpu()
    rows = r[:, 1:2].contiguous().view(torch.int64).numpy()[:, 0]
    i = np.argmax(np.abs(t), axis=0)
    np.testing.assert_array_equal(rows, i + 100)
    np.testing.assert_array_equal(np.sign(r[:, 2].numpy()), np.sign(t[i, np.arange(k)]))
    o32 = torch.empty((5003, k), dtype=odt, device="cuda")
    be.project_chunk(x, torch.as_tensor(shift).cuda(), torch.as_tensor(W).cuda(), out=o32)
    np.testing.assert_array_equal(o32.cpu().numpy(), got.astype(o32.cpu().numpy().dtype))


def test_pca_fit_launches_and_matches_sklearn():
    from sklearn import decomposition as skd

    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.decomposition import PCA, TruncatedSVD

    rng = np.random.RandomState(0)
    X = rng.standard_normal((20000, 24)) @ rng.standard_normal((24, 24)) + 1e4
    be = _backend()
    lib = be.lib
    fb = int(lib.bkm_debug_fallback_count())
    Xc = ChunkedArray.from_array(X, 6000)                   # 4 chunks
    PCA(n_components=5).fit(Xc)                            # warm-up (uploads happen before the count starts)
    from dask_ml_b200.cluster import k_means as km

    data = km._to_device_data(Xc, check_finite=False)
    c0 = int(lib.bkm_launch_count())
    p = PCA(n_components=5).fit(data)
    assert int(lib.bkm_launch_count()) - c0 == 8            # 4 gram + 4 project launches
    assert int(lib.bkm_debug_fallback_count()) == fb
    ref = skd.PCA(n_components=5, svd_solver="full").fit(X)
    sgn = np.sign((p.components_ * ref.components_).sum(1))
    np.testing.assert_allclose(p.components_ * sgn[:, None], ref.components_, atol=1e-8)
    np.testing.assert_allclose(p.explained_variance_, ref.explained_variance_, rtol=1e-9)
    np.testing.assert_allclose(p.mean_, ref.mean_, rtol=1e-13)
    T = p.fit_transform(data)
    assert T.blocks[0].is_cuda
    np.testing.assert_allclose(T.compute() * sgn, ref.transform(X), atol=1e-7)
    Xf = X - X.mean(0)
    U = Xf @ p.components_.T
    i = np.argmax(np.abs(U), axis=0)
    assert (U[i, np.arange(5)] > 0).all()                   # the reference's svd_flip(U, V)
    t = TruncatedSVD(n_components=3).fit(Xc)
    rt = skd.TruncatedSVD(n_components=3, algorithm="arpack").fit(X)
    np.testing.assert_allclose(t.singular_values_, rt.singular_values_, rtol=1e-8)   # uncentred, offset 1e4: cond ~ 3e7


@pytest.mark.parametrize("dt", [np.float32, np.float64])
def test_host_resident_gives_the_same_bits(dt):
    from dask_ml_b200.decomposition import PCA
    from dask_ml_b200.engine import host_resident

    rng = np.random.RandomState(4)
    X = (rng.standard_normal((30000, 20)) * 3 + 7).astype(dt)
    a = PCA(n_components=4).fit(X)
    b = PCA(n_components=4).fit(host_resident(X, block_rows=30000))
    for key in ("components_", "explained_variance_", "mean_", "singular_values_"):
        np.testing.assert_array_equal(getattr(a, key), getattr(b, key))


def test_bf16_pca():
    from sklearn import decomposition as skd

    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.decomposition import PCA

    rng = np.random.RandomState(2)
    X = torch.as_tensor(rng.standard_normal((8192, 128)) * np.linspace(3, 0.1, 128)).to(torch.bfloat16).cuda()
    p = PCA(n_components=8).fit(ChunkedArray([X]))
    ref = skd.PCA(n_components=8, svd_solver="full").fit(X.double().cpu().numpy())
    assert p.components_.dtype == np.float32
    np.testing.assert_allclose(p.explained_variance_, ref.explained_variance_, rtol=1e-5)
