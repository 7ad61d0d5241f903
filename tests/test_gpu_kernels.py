"""GPU parity tests of the C-ABI chunk operators against the CPU oracle (run with -m gpu)."""
import numpy as np
import pytest

from _util import TC_ARGMIN, assert_labels_match, sm_count, tc_layout

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def be():
    from dask_ml_b200.engine import CudaBackend

    return CudaBackend()


def _blobs(n, d, k_true, seed, dtype, scale=10.0, std=1.0):
    rng = np.random.RandomState(seed)
    cent = rng.uniform(-scale, scale, size=(k_true, d))
    lab = rng.randint(0, k_true, size=n)
    X = cent[lab] + std * rng.standard_normal((n, d))
    return X.astype(dtype)


SHAPES = [
    # n, d, k, dtype
    (1000, 4, 10, "float32"),
    (777, 2, 3, "float32"),
    (5000, 13, 20, "float32"),
    (3001, 41, 100, "float32"),
    (4096, 64, 256, "float32"),
    (9000, 64, 256, "float32"),
    (2500, 16, 8, "float64"),
    (1200, 41, 100, "float64"),
    (300, 128, 300, "float32"),     # k*d too large for the smem-resident mode -> GLOBAL mode
    (100, 7, 1, "float32"),
    (5, 3, 2, "float32"),
    # wide rows (the reference works for any d, e.g. 784 pixels): the generic kernel shrinks its row tile
    (600, 256, 12, "float32"),
    (500, 784, 10, "float32"),
    (300, 1024, 5, "float32"),
    (400, 784, 10, "float64"),
    (200, 1024, 7, "float64"),
]


@pytest.mark.parametrize("n,d,k,dtype", SHAPES)
@pytest.mark.parametrize("flags", [1, 0])      # 1 = FORCE_SIMT, 0 = auto (tensor cores where supported)
def test_lloyd_chunk_matches_oracle(be, oracle, n, d, k, dtype, flags):
    import torch

    be.flags = flags
    X = _blobs(n, d, max(2, k // 2), 0, dtype)
    C = X[np.random.RandomState(1).choice(n, k, replace=n < k)].astype(np.float64)
    tdt = torch.float32 if dtype == "float32" else torch.float64
    x = be.to_device(X, tdt)
    pack = be.pack_centers(torch.as_tensor(C).to(be.device), tdt)
    labels = be.empty((n,), torch.int32)
    mind2 = be.empty((n,), tdt)
    sums = be.zeros((k * d,), torch.float64)
    counts = be.zeros((k,), torch.int64)
    inertia = be.zeros((1,), torch.float64)
    be.lloyd_chunk(x, pack, k, labels, mind2, sums, counts, inertia)
    torch.cuda.synchronize()

    (olab,), (omin,) = oracle.pairwise_distances_argmin_min([X], C,
                                                          metric_kwargs={"squared": True})
    got = labels.cpu().numpy()
    assert_labels_match(got, olab, X, C)
    # M-step against the oracle scatter-add evaluated on the GPU's own labels (exactly comparable)
    osums = oracle.centers_dense(X, got, k)
    np.testing.assert_allclose(sums.cpu().numpy().reshape(k, d), osums, rtol=2e-6, atol=1e-6 * np.abs(osums).max())
    np.testing.assert_array_equal(counts.cpu().numpy(), np.bincount(got, minlength=k))
    # min distance and inertia
    gmin = mind2.cpu().numpy().astype(np.float64)
    scale = (X.astype(np.float64) ** 2).sum(1) + (C ** 2).sum(1).max()
    tol = 2e-6 if dtype == "float32" else 1e-12
    assert np.max(np.abs(gmin - omin) / scale) < tol
    assert abs(inertia.item() - omin.sum()) <= 1e-5 * omin.sum() + tol * scale.sum()
    be.flags = 0


def test_assign_non_contiguous_rows(be, oracle):
    import torch

    rng = np.random.RandomState(3)
    big = rng.standard_normal((3000, 24)).astype(np.float32)
    xb = torch.from_numpy(big).to(be.device)
    x = xb[:, :13]                     # ldx = 24 > d = 13
    C = big[:20, :13].astype(np.float64)
    pack = be.pack_centers(torch.as_tensor(C).to(be.device), torch.float32)
    labels = be.empty((3000,), torch.int32)
    mn = be.empty((3000,), torch.float32)
    acc = be.zeros((1,), torch.float64)
    be.assign_chunk(x, pack, 20, labels, mn, False, acc)
    (olab,), (omin,) = oracle.pairwise_distances_argmin_min([big[:, :13]], C)
    assert_labels_match(labels.cpu().numpy(), olab, big[:, :13], C)
    np.testing.assert_allclose(mn.cpu().numpy(), omin, rtol=1e-4, atol=1e-4)
    assert abs(acc.item() - omin.sum()) < 1e-4 * omin.sum()


def test_ties_go_to_lowest_index(be):
    """Appendix B.1: duplicate centres -> the lower index wins."""
    import torch

    rng = np.random.RandomState(0)
    X = rng.standard_normal((2000, 8)).astype(np.float32)
    C = rng.standard_normal((6, 8))
    C[4] = C[1]
    C[5] = C[0]
    pack = be.pack_centers(torch.as_tensor(C).to(be.device), torch.float32)
    labels = be.empty((2000,), torch.int32)
    acc = be.zeros((1,), torch.float64)
    be.assign_chunk(be.to_device(X, torch.float32), pack, 6, labels, None, True, acc)
    got = labels.cpu().numpy()
    assert not np.isin(got, [4, 5]).any()


def test_finalize_and_empty_cluster(be):
    """Q1: empty cluster -> zero vector; shift = ||C - C'||_F^2."""
    import torch

    k, d = 5, 3
    sums = torch.arange(k * d, dtype=torch.float64, device=be.device)
    counts = torch.tensor([2, 0, 4, 1, 3], dtype=torch.int64, device=be.device)
    sums.view(k, d)[1] = 0
    Cold = torch.ones((k, d), dtype=torch.float64, device=be.device)
    Cnew = be.empty((k, d), torch.float64)
    shift = be.zeros((1,), torch.float64)
    be.finalize(sums, counts, Cold, Cnew, shift)
    want = sums.view(k, d).cpu().numpy() / np.maximum(counts.cpu().numpy(), 1)[:, None]
    np.testing.assert_allclose(Cnew.cpu().numpy(), want, rtol=1e-15)
    assert (Cnew.cpu().numpy()[1] == 0).all()
    np.testing.assert_allclose(shift.item(), ((1 - want) ** 2).sum(), rtol=1e-14)


def test_sample_matches_philox_restatement(be, oracle):
    import torch

    n = 20000
    rng = np.random.RandomState(5)
    d2 = rng.gamma(2.0, 1.0, size=n).astype(np.float32)
    seed, off = 0x1234567890ABCDEF, 777
    eop = 50.0 / d2.sum()
    picked = be.empty((4096,), torch.int64)
    cnt = be.zeros((1,), torch.int32)
    be.sample_chunk(torch.from_numpy(d2).to(be.device), eop, seed, off, picked, cnt)
    m = int(cnt.item())
    got = np.sort(picked[:m].cpu().numpy())
    u = oracle.philox_uniform(seed, np.arange(n, dtype=np.uint64) + np.uint64(off))
    want = np.nonzero(eop * d2.astype(np.float64) > u)[0] + off
    np.testing.assert_array_equal(got, want)


def test_transform_chunk(be, oracle):
    import torch

    for dtype, tdt, tol in (("float32", torch.float32, 2e-3), ("float64", torch.float64, 1e-9)):
        X = _blobs(1000, 13, 5, 0, dtype)
        C = X[:7].astype(np.float64)
        pack = be.pack_centers(torch.as_tensor(C).to(be.device), tdt)
        out = be.empty((1000, 7), tdt)
        be.transform_chunk(be.to_device(X, tdt), pack, 7, out)
        want = oracle.euclidean_distances([X], C.astype(dtype))[0]
        # compare squared distances: ||x||^2 - 2x.c + ||c||^2 cancels near zero in the dtype of X, both
        # in the reference formula (pairwise.py:93-97) and here
        scale = (X.astype(np.float64) ** 2).sum(1)[:, None] + (C ** 2).sum(1)[None, :]
        err = np.abs(out.cpu().numpy().astype(np.float64) ** 2 - want.astype(np.float64) ** 2) / scale
        assert err.max() < (1e-5 if dtype == "float32" else 1e-13)


def test_check_finite(be):
    import torch

    X = np.random.RandomState(0).standard_normal((5000, 7)).astype(np.float32)
    assert int(be.check_finite([be.to_device(X, torch.float32)]).item()) == 0
    X[4321, 3] = np.inf
    assert int(be.check_finite([be.to_device(X, torch.float32)]).item()) != 0
    X[4321, 3] = np.nan
    assert int(be.check_finite([be.to_device(X, torch.float64)]).item()) != 0


def _exact_labels_f64(x, C):
    """float64 arg-min on the device, in row blocks (sizes the CPU oracle would take minutes for)."""
    import torch

    C64 = C.double()
    cn = (C64 * C64).sum(1)
    out = torch.empty((x.shape[0],), dtype=torch.int64, device=x.device)
    second = torch.empty((x.shape[0],), dtype=torch.float64, device=x.device)
    for s in range(0, x.shape[0], 1 << 18):
        xb = x[s:s + (1 << 18)].double()
        d2 = (xb * xb).sum(1, keepdim=True) + cn[None, :] - 2.0 * xb @ C64.T
        if C64.shape[0] > 1:
            top = torch.topk(d2, 2, dim=1, largest=False)
            out[s:s + xb.shape[0]] = top.indices[:, 0]
            second[s:s + xb.shape[0]] = top.values[:, 1] - top.values[:, 0]
        else:
            out[s:s + xb.shape[0]] = 0
            second[s:s + xb.shape[0]] = 1.0
    return out, second


# Pipeline stress of the tensor-core kernel: row counts that leave every kind of tail (fewer tiles than SMs, a partial
# last tile, three passes of every CTA's X ring and one more tile on two CTAs, the second partial; G SMs, 64-row tiles,
# S ring slots), the Lloyd variants with and without distances, N = 16, 128 and 256 (N = 256: an odd ring of 5).
TAIL_ROWS = {"64G-1": lambda G, S: 64 * G - 1, "64G*3S+77": lambda G, S: 64 * G * 3 * S + 77}


@pytest.mark.parametrize("n", [1, 127, 128, 129, "64G-1", "64G*3S+77", 200_000, 1_000_003])
@pytest.mark.parametrize("d,k", [(64, 256), (64, 100), (32, 130), (8, 16)])
@pytest.mark.parametrize("want_dist", [False, True])
def test_pipeline_tails(be, n, d, k, want_dist):
    import torch

    if n in TAIL_ROWS:
        n = TAIL_ROWS[n](sm_count(be.lib, be.device.index or 0), tc_layout(be.lib, d, k, TC_ARGMIN, mstep=1)[2])
    be.flags = 2          # FORCE_TC: also the shapes the dispatcher would leave to the CUDA cores (k d < 512)
    g = torch.Generator(device=be.device).manual_seed(n + d + k)
    cent = torch.empty((max(2, k // 2), d), device=be.device).uniform_(-10, 10, generator=g)
    X = cent[torch.randint(0, cent.shape[0], (n,), device=be.device, generator=g)] + \
        torch.randn((n, d), device=be.device, generator=g)
    C = X[torch.randint(0, n, (k,), device=be.device, generator=g)].double() + \
        0.01 * torch.randn((k, d), device=be.device, generator=g, dtype=torch.float64)
    pack = be.pack_centers(C.contiguous(), torch.float32)
    labels = be.empty((n,), torch.int32)
    mind2 = be.empty((n,), torch.float32) if want_dist else None
    sums = be.zeros((k * d,), torch.float64)
    counts = be.zeros((k,), torch.int64)
    inertia = be.zeros((1,), torch.float64) if want_dist else None
    for _ in range(2):          # twice: the second launch reuses every barrier / list / ring of a warm SM
        sums.zero_(); counts.zero_()
        if inertia is not None:
            inertia.zero_()
        be.lloyd_chunk(X, pack, k, labels, mind2, sums, counts, inertia)
    torch.cuda.synchronize()
    assert be.lib.bkm_debug_abort_code() == 0
    want, margin = _exact_labels_f64(X, C)
    got = labels.long()
    bad = got != want
    # a label may differ from the float64 arg-min only where float64 itself is (nearly) tied
    if bool(bad.any()):
        xs = (X.double() ** 2).sum(1)[bad] + (C ** 2).sum(1).max()
        assert bool((margin[bad] <= 1e-9 * xs).all()), int(bad.sum())
    assert torch.equal(counts, torch.bincount(got, minlength=k))
    ref = torch.zeros((k, d), dtype=torch.float64, device=be.device).index_add_(0, got, X.double())
    assert float((sums.view(k, d) - ref).abs().max()) <= 2e-6 * float(ref.abs().max()) + 1e-9
    # the assignment-only kernels (labels only / labels + distances) must agree with the Lloyd pass
    lab2 = be.empty((n,), torch.int32)
    if want_dist:
        md = be.empty((n,), torch.float32)
        ds = be.zeros((1,), torch.float64)
        be.assign_chunk(X, pack, k, lab2, md, True, ds)
        torch.cuda.synchronize()
        exact = ((X.double() - C[lab2.long()]) ** 2).sum(1)
        scale = (X.double() ** 2).sum(1) + (C ** 2).sum(1).max()       # fp32 centres: error relative to the norms
        assert float(((md.double() - exact).abs() / scale).max()) < 2e-6
        assert abs(float(ds[0]) - float(exact.sum())) <= 1e-5 * float(exact.sum()) + 2e-6 * float(scale.sum())
    else:
        be.assign_chunk(X, pack, k, lab2, None, True, None)
        torch.cuda.synchronize()
    be.flags = 0
    assert be.lib.bkm_debug_abort_code() == 0
    assert torch.equal(lab2, labels)


def test_tcgen05_out_of_range_and_mixed_scales(be):
    """Rows far outside the centres' range (beyond fp16 after scaling), features of very different scale and
    non-finite entries must take the float64 path and still give the float64 labels."""
    import torch

    n, d, k = 50_000, 64, 256
    g = torch.Generator(device=be.device).manual_seed(7)
    fscale = torch.logspace(-6, 3, d, device=be.device)                 # features from 1e-6 to 1e3
    cent = torch.empty((k, d), device=be.device).uniform_(-1, 1, generator=g) * fscale
    X = cent[torch.randint(0, k, (n,), device=be.device, generator=g)] + \
        0.05 * fscale * torch.randn((n, d), device=be.device, generator=g)
    X[::97] *= 3000.0                                                    # far beyond 64x the largest centre entry
    X[5, 3] = 3.0e38
    C = X[torch.randperm(n, device=be.device, generator=g)[:k] | 1].double().contiguous()   # odd rows: none of the scaled ones
    pack = be.pack_centers(C, torch.float32)
    labels = be.empty((n,), torch.int32)
    sums = be.zeros((k * d,), torch.float64)
    counts = be.zeros((k,), torch.int64)
    be.lloyd_chunk(X, pack, k, labels, None, sums, counts, None)
    torch.cuda.synchronize()
    assert be.lib.bkm_debug_abort_code() == 0
    want, margin = _exact_labels_f64(X, C)
    got = labels.long()
    bad = got != want
    bad[5] = False                                                       # the overflowing row has no float64 answer either
    if bool(bad.any()):
        xs = (X.double() ** 2).sum(1)[bad] + (C ** 2).sum(1).max()
        assert bool((margin[bad] <= 1e-9 * xs).all()), int(bad.sum())
    assert int(counts.sum()) == n


@pytest.mark.parametrize("n", [1000, 300_001])
@pytest.mark.parametrize("d,k", [(1, 3), (3, 5), (13, 20), (41, 100), (63, 256)])
def test_tcgen05_odd_feature_counts(be, oracle, n, d, k):
    """d not a multiple of 4 runs on the tensor path once the rows are uploaded with a padded pitch
    (BASELINE configs C3: d=41, k=100 and C4: d=13, k=20)."""
    import torch

    X = _blobs(n, d, max(2, k // 2), 3, "float32")
    x = be.to_device(X, torch.float32)
    assert x.stride(0) % 4 == 0 and x.shape == (n, d)
    C = torch.as_tensor(X[np.random.RandomState(2).choice(n, k, replace=False)].astype(np.float64)).to(be.device)
    C += 0.01 * torch.randn(C.shape, dtype=torch.float64, device=be.device, generator=torch.Generator(device=be.device).manual_seed(1))
    be.flags = 2                      # FORCE_TC: fail instead of falling back to the CUDA-core kernel
    try:
        pack = be.pack_centers(C.contiguous(), torch.float32)
        labels = be.empty((n,), torch.int32)
        sums = be.zeros((k * d,), torch.float64)
        counts = be.zeros((k,), torch.int64)
        be.lloyd_chunk(x, pack, k, labels, None, sums, counts, None)
        md = be.empty((n,), torch.float32)
        ds = be.zeros((1,), torch.float64)
        lab2 = be.empty((n,), torch.int32)
        be.assign_chunk(x, pack, k, lab2, md, True, ds)
        torch.cuda.synchronize()
    finally:
        be.flags = 0
    assert be.lib.bkm_debug_abort_code() == 0
    want, margin = _exact_labels_f64(x, C)
    got = labels.long()
    bad = got != want
    if bool(bad.any()):
        xs = (x.double() ** 2).sum(1)[bad] + (C ** 2).sum(1).max()
        assert bool((margin[bad] <= 1e-9 * xs).all()), int(bad.sum())
    assert torch.equal(lab2, labels)
    assert torch.equal(counts, torch.bincount(got, minlength=k))
    ref = torch.zeros((k, d), dtype=torch.float64, device=be.device).index_add_(0, got, x.double())
    assert float((sums.view(k, d) - ref).abs().max()) <= 2e-6 * float(ref.abs().max()) + 1e-9
    exact = ((x.double() - C[got]) ** 2).sum(1)
    scale = (x.double() ** 2).sum(1) + (C ** 2).sum(1).max()
    assert float(((md.double() - exact).abs() / scale).max()) < 2e-6


# ------------------------------------------------------------------------------------------ streaming kernel (family 2)
@pytest.mark.parametrize("n", [1, 31, 32, 33, 255, 256, 257, 4097, 148 * 8 * 32 * 3 + 5, 1_000_003])
@pytest.mark.parametrize("d,k,pitch", [(13, 20, 13), (13, 20, 16), (13, 20, 14), (16, 31, 16), (1, 2, 1), (3, 5, 3),
                                       (7, 1, 7), (9, 31, 12), (5, 8, 24), (16, 28, 16), (14, 32, 14), (4, 30, 4),
                                       (5, 8, 40)])
def test_stream_kernel_tails(be, n, d, k, pitch):
    """Family 2 (bkm_stream.cu): every tail of the per-warp ring (fewer tiles than warps, a partial last tile, rows with
    and without a padded pitch), all entry points, against the float64 arg-min evaluated on the device.  Every call runs
    on a streaming kernel, none on the generic fallback."""
    import torch

    assert be.kernel_family(d, k, torch.float32) == 2
    fallbacks = int(be.lib.bkm_debug_fallback_count())
    g = torch.Generator(device=be.device).manual_seed(n * 31 + d * 7 + k)
    cent = torch.empty((max(2, k // 2), d), device=be.device).uniform_(-10, 10, generator=g)
    Xc = cent[torch.randint(0, cent.shape[0], (n,), device=be.device, generator=g)] + \
        torch.randn((n, d), device=be.device, generator=g)
    if pitch != d:
        buf = torch.full((n, pitch), 7.5e4, device=be.device)       # the padding must never leak into a result
        buf[:, :d] = Xc
        X = buf[:, :d]
    else:
        X = Xc.contiguous()
    C = Xc[torch.randint(0, n, (k,), device=be.device, generator=g)].double() + \
        0.01 * torch.randn((k, d), device=be.device, generator=g, dtype=torch.float64)
    pack = be.pack_centers(C.contiguous(), torch.float32)
    labels = be.empty((n,), torch.int32)
    mind2 = be.empty((n,), torch.float32)
    sums = be.zeros((k * d,), torch.float64)
    counts = be.zeros((k,), torch.int64)
    inertia = be.zeros((1,), torch.float64)
    be.lloyd_chunk(X, pack, k, labels, mind2, sums, counts, inertia)
    torch.cuda.synchronize()
    want, margin = _exact_labels_f64(Xc, C)
    got = labels.long()
    bad = got != want
    if bool(bad.any()):
        xs = (Xc.double() ** 2).sum(1)[bad] + (C ** 2).sum(1).max()
        assert bool((margin[bad] <= 1e-9 * xs).all()), int(bad.sum())
    assert torch.equal(counts, torch.bincount(got, minlength=k))
    ref = torch.zeros((k, d), dtype=torch.float64, device=be.device).index_add_(0, got, Xc.double())
    assert float((sums.view(k, d) - ref).abs().max()) <= 2e-6 * float(ref.abs().max()) + 1e-9
    exact = ((Xc.double() - C[got]) ** 2).sum(1)
    scale = (Xc.double() ** 2).sum(1) + (C ** 2).sum(1).max()
    assert float(((mind2.double() - exact).abs() / scale).max()) < 2e-6
    assert abs(float(inertia[0]) - float(exact.sum())) <= 1e-5 * float(exact.sum()) + 2e-6 * float(scale.sum())
    # assignment-only entry point (no M-step), non-squared distances
    lab2 = be.empty((n,), torch.int32)
    md = be.empty((n,), torch.float32)
    ds = be.zeros((1,), torch.float64)
    be.assign_chunk(X, pack, k, lab2, md, False, ds)
    torch.cuda.synchronize()
    assert torch.equal(lab2, labels)
    assert float(((md.double() ** 2 - exact).abs() / scale).max()) < 4e-6
    # Lloyd step without distances (what fit runs)
    sums2 = be.zeros((k * d,), torch.float64)
    counts2 = be.zeros((k,), torch.int64)
    lab3 = be.empty((n,), torch.int32)
    be.lloyd_chunk(X, pack, k, lab3, None, sums2, counts2, None)
    torch.cuda.synchronize()
    assert torch.equal(lab3, labels) and torch.equal(counts2, counts)
    assert torch.equal(sums2, sums)            # bit-reproducible: fixed CTA / warp order
    assert int(be.lib.bkm_debug_fallback_count()) == fallbacks


def test_stream_kernel_matches_generic_kernel(be):
    """Family 2 against the generic CUDA-core kernel (FORCE_SIMT) on badly scaled data with many near-ties."""
    import torch

    n, d, k = 200_000, 13, 20
    g = torch.Generator(device=be.device).manual_seed(11)
    scales = torch.logspace(0, 3, d, device=be.device)
    X = (torch.randn((n, d), device=be.device, generator=g) * scales).contiguous()
    C = X[:k].double().contiguous()
    pack = be.pack_centers(C, torch.float32)
    out = []
    for flags in (0, 1):
        be.flags = flags
        labels = be.empty((n,), torch.int32)
        sums = be.zeros((k * d,), torch.float64)
        counts = be.zeros((k,), torch.int64)
        be.lloyd_chunk(X, pack, k, labels, None, sums, counts, None)
        torch.cuda.synchronize()
        out.append((labels.clone(), sums.clone(), counts.clone()))
    be.flags = 0
    want, margin = _exact_labels_f64(X, C)
    for labels, sums, counts in out:
        bad = labels.long() != want
        if bool(bad.any()):
            xs = (X.double() ** 2).sum(1)[bad] + (C ** 2).sum(1).max()
            assert bool((margin[bad] <= 1e-9 * xs).all()), int(bad.sum())
    assert int((out[0][0] != out[1][0]).sum()) <= 2


# ------------------------------------------------------------------------------------------ BASELINE sizes
@pytest.mark.parametrize("name,n,d,k", [("C2", 10_000_000, 64, 256), ("C3", 4_898_431, 41, 100), ("C4", 15_000_000, 13, 20)])
def test_baseline_size_parity(be, name, n, d, k):
    """Labels, counts and sums at the FULL BASELINE.json sizes against the float64 arg-min evaluated on the device (every
    row), plus the size-independent invariants: counts sum to n, the sums add up to the column sums of X."""
    import torch
    from bench import synth_config_device, synth_blobs_device

    X = synth_blobs_device(n, d, k, 5, be.device, torch.float32) if name == "C2" else synth_config_device(name, n, 0, be.device)
    x = be.to_device(X, torch.float32) if (d % 4 and be.kernel_family(d, k, torch.float32) == 1) else X
    C = X[:k].double().contiguous()
    pack = be.pack_centers(C, torch.float32)
    labels = be.empty((n,), torch.int32)
    sums = be.zeros((k * d,), torch.float64)
    counts = be.zeros((k,), torch.int64)
    be.lloyd_chunk(x, pack, k, labels, None, sums, counts, None)
    torch.cuda.synchronize()
    assert be.lib.bkm_debug_abort_code() == 0
    got = labels.long()
    assert int(counts.sum()) == n and torch.equal(counts, torch.bincount(got, minlength=k))
    colsum = torch.zeros((d,), dtype=torch.float64, device=be.device)
    for s in range(0, n, 1 << 20):
        colsum += X[s:s + (1 << 20)].double().sum(0)
    assert float((sums.view(k, d).sum(0) - colsum).abs().max()) <= 1e-6 * float(colsum.abs().max()) + 1e-3
    want, margin = _exact_labels_f64(X, C)
    bad = got != want
    nbad = int(bad.sum())
    if nbad:
        xs = (X.double() ** 2).sum(1)[bad] + (C ** 2).sum(1).max()
        assert bool((margin[bad] <= 1e-9 * xs).all()), nbad
    assert nbad <= 1e-5 * n
    if be.kernel_family(d, k, torch.float32) == 1:
        # the rounding bound tau defers only a small fraction of rows to the float64 re-check
        assert be.deferred_rows(n, d, k, torch.float32) < 0.01 * n


@pytest.mark.parametrize("d,k,dtype_name,flags", [
    pytest.param(32, 64, "float32", 0, id="32-64-float32"),
    pytest.param(13, 20, "float32", 0, id="13-20-float32"),
    pytest.param(64, 256, "float32", 0, id="64-256-float32"),
    pytest.param(128, 600, "bfloat16", 0, id="128-600-bfloat16"),
    # the generic kernel: GLOBAL mode (k * d too large for shared memory: one slot for the whole chunk), SMEM mode
    pytest.param(128, 300, "float32", 0, id="128-300-float32-global"),
    pytest.param(64, 512, "float32", 0, id="64-512-float32-global"),
    pytest.param(64, 256, "float32", 1, id="64-256-float32-simt"),
    pytest.param(64, 256, "float64", 0, id="64-256-float64-global"),
])
def test_sums_with_a_dominant_cluster_and_offset_data(be, d, k, dtype_name, flags):
    """The fused kernels keep per-CTA (per-warp) partial sums in fp32 and widen them to float64 once per chunk call
    (the reference accumulates in float64, k_means.py:576); the generic kernel's GLOBAL mode adds the whole chunk into
    one float64 slot.  Worst case for that: one cluster owns 90 % of 2M rows and the data sit far from the origin.  The
    sums must still agree with the float64 sums of the SAME labels to ~1e-5 of the data's magnitude (the centres move by
    less than 1e-3 of the cluster's standard deviation)."""
    import torch

    be.flags = flags
    dtype = getattr(torch, dtype_name)
    n = 2_000_000
    g = torch.Generator(device=be.device).manual_seed(d * 1000 + k)
    cent = torch.empty((k, d), device=be.device).uniform_(-3, 3, generator=g) + 100.0
    which = torch.where(torch.rand(n, device=be.device, generator=g) < 0.9, torch.zeros(n, device=be.device, dtype=torch.long),
                        torch.randint(0, k, (n,), device=be.device, generator=g))
    X = (cent[which] + torch.randn((n, d), device=be.device, generator=g)).to(dtype)
    x = be.to_device(X, dtype)
    C = cent.double().contiguous()
    pack = be.pack_centers(C, dtype)
    labels = be.empty((n,), torch.int32)
    sums = be.zeros((k * d,), torch.float64); counts = be.zeros((k,), torch.int64)
    try:
        be.lloyd_chunk(x, pack, k, labels, None, sums, counts, None)
        torch.cuda.synchronize()
    finally:
        be.flags = 0
    lab = labels.long()
    want = torch.zeros((k, d), dtype=torch.float64, device=be.device).index_add_(0, lab, X.double())
    wcnt = torch.bincount(lab, minlength=k)
    assert torch.equal(counts, wcnt)
    got = sums.view(k, d)
    scale = (X.double().abs().max() * wcnt.clamp(min=1).double())[:, None]        # |x| * rows of the cluster
    rel = ((got - want).abs() / scale).max()
    assert float(rel) < 1e-5, float(rel)
    newC = got / wcnt.clamp(min=1).double()[:, None]
    assert float((newC - want / wcnt.clamp(min=1).double()[:, None]).abs().max()) < 1e-3
