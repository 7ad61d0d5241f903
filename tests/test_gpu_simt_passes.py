"""The CUDA-core Nystrom and transform passes (nystrom_kernel, transform_kernel in bkm_aux.cu) on the H100 at their
keep-row blocks, warp counts and row tiles (tests/simt_pass_cases.py), from the strongest check to the weakest:

* exact data: integer rows and keep rows make every norm and dot product exact, so the distances and squared distances
  are bit-exact against numpy, the column sums at gamma = 1000 are exact counts, and an embedding row equal to keep row
  j is exactly the signed one-hot row W_j.  Rows at squared distance 1 from the keep set are finite at gamma = 745.12
  and NaN at 745.14; rows with odd coordinates are NaN.  Rows come with a NaN-padded pitch, outputs go into buffers of
  a larger pitch whose padding must keep its poison;
* bit-identity across blockings: zero W columns and zero features move lb, nw and TR without changing a bit; COLSUM's
  sums do not change when only lb moves;
* float64 references on random data, with tolerances derived from the kernels' arithmetic;
* SpectralClustering with a blocked embedding against the float64 restatement, and rbf_kernel / euclidean_distances at a
  row tile below 64 against scikit-learn.

The launch count of each call is held against the restated geometry (one COLSUM launch per keep-row block, then the
fold), and every pass runs twice with the same bits."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import simt_pass_cases as sc  # noqa: E402

pytestmark = pytest.mark.gpu

TD = {"f32": torch.float32, "f64": torch.float64}
NP = {"f32": np.float32, "f64": np.float64}
EPS = {"f32": 2.0 ** -24, "f64": 2.0 ** -53}
POISON = 12345.0
PAD = 5
TAU_SIMT = lambda d: 8.0 * (np.sqrt(d) + 2.0) * 2.0 ** -24     # fp32 CUDA-core distance bound (test_gpu_spectral.py)


def tau(dt, d):
    """Relative bound of a computed squared distance, in units of ||x||^2 + ||c||^2: fp64 the worst case of the d-term
    dot product, the two norms and the two adds ((2 d + 4) u); fp32 the bound the other fp32 tests use."""
    return (d + 2) * 2.0 ** -52 if dt == "f64" else TAU_SIMT(d)


@pytest.fixture(scope="module")
def be():
    from dask_ml_b200.engine import CudaBackend

    return CudaBackend()


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _rows(h, dt):
    """Device rows of a pitch d + PAD whose padding is NaN: a read past column d - 1 turns the result into NaN."""
    n, d = h.shape
    buf = torch.full((n, d + PAD), float("nan"), dtype=TD[dt], device="cuda")
    buf[:, :d] = torch.from_numpy(np.ascontiguousarray(h)).cuda().to(TD[dt])
    return buf[:, :d]


def _pack(be, C, dt):
    return be.pack_centers(torch.from_numpy(np.ascontiguousarray(C, dtype=np.float64)).cuda(), TD[dt])


def _fallbacks(be):
    return int(be.lib.bkm_debug_fallback_count())


def _embed(be, x, pack, l, gamma, W, launches=1, fill=POISON):
    """(n, kw + 3) output buffer of one EMBED call into its first kw columns."""
    n, kw = x.shape[0], W.shape[1]
    buf = torch.full((n, kw + 3), fill, dtype=x.dtype, device="cuda")
    w = W.to(x.dtype) if torch.is_tensor(W) else torch.from_numpy(np.ascontiguousarray(W)).cuda().to(x.dtype)
    c0 = be.launch_count()
    be.nystrom_embed(x, pack, l, gamma, w, buf[:, :kw])
    torch.cuda.synchronize()
    if launches is not None:
        assert be.launch_count() - c0 == launches
    return buf.cpu().numpy()


def _colsum(be, x, pack, l, gamma, chunks=1, launches=None):
    """COLSUM over ``chunks`` row chunks: the first overwrites, the others add.  ``launches`` per chunk: its kernel
    launches plus the fold."""
    c = torch.full((l,), float("nan"), dtype=torch.float64, device="cuda")
    n = int(x.shape[0])
    step = -(-n // chunks)
    for i, s0 in enumerate(range(0, n, step)):
        c0 = be.launch_count()
        be.kernel_colsum(x[s0:s0 + step], pack, l, gamma, c, first=i == 0)
        if launches is not None:
            assert be.launch_count() - c0 == launches
    torch.cuda.synchronize()
    return c.cpu().numpy()


def _transform(be, x, pack, k, mode, gamma=0.0):
    """(n, k + 3) NaN-filled output buffer of one call into its first k columns."""
    buf = torch.full((x.shape[0], k + 3), float("nan"), dtype=x.dtype, device="cuda")
    c0 = be.launch_count()
    be.transform_chunk(x, pack, k, buf[:, :k], mode=mode, gamma=gamma)
    torch.cuda.synchronize()
    assert be.launch_count() - c0 == 1
    return buf.cpu().numpy()


def _same(a, b):
    assert np.asarray(a).tobytes() == np.asarray(b).tobytes()


def _d2_exact(X, C):
    """Squared distances of integer rows in float64 on the device: every term and partial sum is an integer below 2^53."""
    X = torch.from_numpy(np.ascontiguousarray(X)).cuda().double()
    C = torch.from_numpy(np.ascontiguousarray(C)).cuda().double()
    return ((X * X).sum(1)[:, None] - 2.0 * X @ C.T + (C * C).sum(1)[None, :]).cpu().numpy()


# ---------------------------------------------------------------------------------------------------------------------
# a) exact data
# ---------------------------------------------------------------------------------------------------------------------
EMBED = [(dt,) + s for dt in ("f32", "f64") for s in sc.embed_shapes(dt)]
COLSUM = [(dt,) + s for dt in ("f32", "f64") for s in sc.colsum_shapes(dt)]
TRANSFORM = [(dt,) + s for dt in ("f32", "f64") for s in sc.transform_shapes(dt)]


@pytest.mark.parametrize("dt,name,d,l,kw", EMBED, ids=["%s-%s" % (c[0], c[1]) for c in EMBED])
def test_embed_exact(be, sms, dt, name, d, l, kw):
    keep = sc.keep_rows(l, d, seed=l + d)
    col, sgn = sc.one_hot_parts(l, kw, seed=kw)
    colt, sgnt = torch.from_numpy(col).cuda(), torch.from_numpy(sgn).cuda()
    W = torch.zeros((l, kw), dtype=TD[dt], device="cuda")
    W[torch.arange(l, device="cuda"), colt] = sgnt.to(TD[dt])
    pack = _pack(be, keep, dt)
    nw = sc.nystrom_geom(1, 1, d, l, kw, dt, sms).nw
    for n in sc.row_counts(nw, sms, big=name not in sc.LB1024_SHORT):
        g = sc.nystrom_geom(1, n, d, l, kw, dt, sms)
        X, kind, j = sc.exact_rows(keep, n, seed=n)
        x = _rows(X, dt)
        lo = _embed(be, x, pack, l, sc.GAMMA_LO, W)
        _same(lo, _embed(be, x, pack, l, sc.GAMMA_LO, W))
        hi = _embed(be, x, pack, l, sc.GAMMA_HI, W)
        cp = np.nonzero(kind == sc.COPY)[0]
        want_cp = np.zeros((len(cp), kw))
        want_cp[np.arange(len(cp)), col[j[cp]]] = sgn[j[cp]]
        for out in (lo, hi):
            assert (out[:, kw:] == POISON).all(), "the output padding was written"
            assert np.array_equal(out[cp, :kw], want_cp), "n=%d: copies of keep rows (blocks of %d)" % (n, g.lb)
            assert np.isnan(out[kind == sc.ODD, :kw]).all()
        near = np.nonzero(kind == sc.NEAR)[0]
        assert np.isnan(hi[near, :kw]).all(), "gamma m = 745.14 must give NaN"
        if len(near):
            d2 = torch.from_numpy(_d2_exact(X[near], keep)).cuda()
            assert bool((d2.min(1).values == 1).all())
            # e = exp(-gamma (y - 1)) W in float64, one nonzero per row of W
            v = torch.exp(-sc.GAMMA_LO * (d2 - 1.0))
            e = torch.zeros((len(near), kw), dtype=torch.float64, device="cuda")
            e.index_add_(1, colt, v * sgnt[None, :])
            e = e.cpu().numpy()
            # two nearest keep rows of opposite sign in one column cancel: e = 0, and 0 / 0 is NaN on both sides
            live = (e != 0).any(1)
            assert live.mean() > 0.5
            want = e[live] / np.sqrt((e[live] ** 2).sum(1, keepdims=True))
            got = lo[near, :kw]
            assert np.isfinite(got[live]).all(), "gamma m = 745.12 must stay finite"
            assert np.abs(got[live] - want).max() <= 8 * EPS[dt]
            assert np.isnan(got[~live]).all()


@pytest.mark.parametrize("dt,name,d,l", COLSUM, ids=["%s-%s" % (c[0], c[1]) for c in COLSUM])
def test_colsum_exact_counts(be, sms, dt, name, d, l):
    keep = sc.keep_rows(l, d, seed=l + d)
    pack = _pack(be, keep, dt)
    nw = sc.nystrom_geom(0, 1, d, l, 0, dt, sms).nw
    for n in sc.row_counts(nw, sms, big=True):
        g = sc.nystrom_geom(0, n, d, l, 0, dt, sms)
        X, kind, j = sc.exact_rows(keep, n, seed=n + 1)
        want = np.bincount(j[kind == sc.COPY], minlength=l).astype(np.float64)
        x = _rows(X, dt)
        got = _colsum(be, x, pack, l, sc.GAMMA_COUNT, launches=g.launches + 1)
        assert np.array_equal(got, want), "n=%d: %d launches of %d keep rows" % (n, g.launches, g.lb)
        _same(got, _colsum(be, x, pack, l, sc.GAMMA_COUNT))
        if n >= 3:
            assert np.array_equal(_colsum(be, x, pack, l, sc.GAMMA_COUNT, chunks=3), want)


@pytest.mark.parametrize("dt,name,d,k", TRANSFORM, ids=["%s-%s" % (c[0], c[1]) for c in TRANSFORM])
def test_transform_exact(be, sms, dt, name, d, k):
    g = sc.transform_geom(1, d, k, dt, sms)
    n = sc.transform_rows(g.TR, sms)
    g = sc.transform_geom(n, d, k, dt, sms)
    assert g.last_rows == 1 and g.ntiles > g.grid
    rng = np.random.RandomState(d + k)
    X = rng.randint(-3, 4, (n, d)).astype(np.int8)
    C = rng.randint(-3, 4, (k, d)).astype(np.int8)
    x = _rows(X, dt)
    pack = _pack(be, C, dt)
    route, counted = sc.route("transform", dt, d, k, base_bytes=x.data_ptr() % 16, ldx=x.stride(0))
    assert route == "simt"
    d2 = _d2_exact(X, C).astype(NP[dt])
    f0 = _fallbacks(be)
    sq = _transform(be, x, pack, k, 1)
    assert _fallbacks(be) - f0 == int(counted)
    _same(sq, _transform(be, x, pack, k, 1))
    dist = _transform(be, x, pack, k, 0)
    gamma = 1.0 / d
    rb = _transform(be, x, pack, k, 2, gamma)
    for out in (sq, dist, rb):
        assert np.isnan(out[:, k:]).all()
    assert np.array_equal(sq[:, :k], d2)
    assert np.array_equal(dist[:, :k], np.sqrt(d2))
    ref = np.exp(-gamma * d2.astype(np.float64))
    tol = ref * (gamma * d2 * 2 * EPS[dt] + 4 * EPS[dt]) + np.finfo(NP[dt]).tiny
    assert (np.abs(rb[:, :k] - ref) <= tol).all()


# ---------------------------------------------------------------------------------------------------------------------
# b) the same bits under other blockings
# ---------------------------------------------------------------------------------------------------------------------
def _random_case(n, d, l, seed):
    """n random rows around 6 centres and l keep rows drawn apart from them, as stored in fp32 (so both precisions see
    the same values)."""
    rng = np.random.RandomState(seed)
    cent = rng.uniform(-1, 1, (6, d))

    def draw(m):
        return (cent[rng.randint(0, 6, m)] + 0.3 * rng.standard_normal((m, d))).astype(np.float32).astype(np.float64)

    return draw(n), draw(l)


def _zpad(A, d):
    return np.concatenate([A, np.zeros((A.shape[0], d - A.shape[1]))], 1)


# (dt, base d, l, k, padded kw, padded widths): the base fits one block at nw = 8; padding moves (nw, lb)
EMBED_PADS = [("f64", 6, 1500, 5, 2000, (2000, 5000)), ("f32", 6, 3000, 5, 4000, (4000, 10000))]


@pytest.mark.parametrize("dt,d,l,k,kwp,dps", EMBED_PADS, ids=[c[0] for c in EMBED_PADS])
def test_embed_blockings_give_the_same_bits(be, sms, dt, d, l, k, kwp, dps):
    n = 4 * sms * 8 + 9
    X, keep = _random_case(n, d, l, 31)
    W = np.random.RandomState(32).standard_normal((l, k))
    gamma = 0.5
    base = _embed(be, _rows(X, dt), _pack(be, keep, dt), l, gamma, W)[:, :k]
    assert np.isfinite(base).all()
    geoms = [sc.nystrom_geom(1, n, d, l, k, dt, sms)]
    # zero W columns: more outputs per warp, fewer kernel values per block
    Wp = np.concatenate([W, np.zeros((l, kwp - k))], 1)
    geoms.append(sc.nystrom_geom(1, n, d, l, kwp, dt, sms))
    _same(_embed(be, _rows(X, dt), _pack(be, keep, dt), l, gamma, Wp)[:, :k], base)
    # zero features: a wider row per warp
    for dp in dps:
        geoms.append(sc.nystrom_geom(1, n, dp, l, k, dt, sms))
        _same(_embed(be, _rows(_zpad(X, dp), dt), _pack(be, _zpad(keep, dp), dt), l, gamma, W)[:, :k], base)
    assert geoms[0].one and all(not g.one for g in geoms[1:])
    assert {g.nw for g in geoms} == {8, 4}


# (dt, base d, l, padded d): lb moves, nw and the grid do not
COLSUM_PADS = [("f64", 6, 1500, 1000), ("f32", 6, 2000, 1000)]


@pytest.mark.parametrize("dt,d,l,dp", COLSUM_PADS, ids=[c[0] for c in COLSUM_PADS])
def test_colsum_does_not_depend_on_the_keep_row_blocks(be, sms, dt, d, l, dp):
    n = 3 * 4 * sms * 8 + 5
    X, keep = _random_case(n, d, l, 41)
    g0, g1 = (sc.nystrom_geom(0, n, w, l, 0, dt, sms) for w in (d, dp))
    assert (g0.nw, g0.grid) == (g1.nw, g1.grid) and g0.launches == 1 and g1.launches > 1
    a = _colsum(be, _rows(X, dt), _pack(be, keep, dt), l, 0.5, launches=2)
    b = _colsum(be, _rows(_zpad(X, dp), dt), _pack(be, _zpad(keep, dp), dt), l, 0.5, launches=g1.launches + 1)
    _same(a, b)


@pytest.mark.parametrize("dt", ["f32", "f64"])
def test_transform_tiles_give_the_same_bits(be, sms, dt):
    n, d, k = 3001, 6, 9
    X, C = _random_case(n, d, k, 51)
    outs = {}
    for TR in (64, 32, 8, 1):
        dp = sc.first_d_of_tr(TR, dt) if TR < 64 else d
        assert sc.transform_geom(n, dp, k, dt, sms).TR == TR
        x, pack = _rows(_zpad(X, dp), dt), _pack(be, _zpad(C, dp), dt)
        outs[TR] = [_transform(be, x, pack, k, m, 0.25) for m in (0, 1, 2)]
    for TR in (32, 8, 1):
        for a, b in zip(outs[TR], outs[64]):
            _same(a, b)


# ---------------------------------------------------------------------------------------------------------------------
# c) float64 references on random data
# ---------------------------------------------------------------------------------------------------------------------
def _ref_parts(Xq, keep):
    X = torch.from_numpy(Xq).cuda()
    C = torch.from_numpy(np.ascontiguousarray(keep)).cuda()
    xn, cn = (X * X).sum(1), (C * C).sum(1)
    return torch.clamp(xn[:, None] - 2.0 * X @ C.T + cn[None, :], min=0.0), xn, cn


# (dt, n, d, l): COLSUM with several keep-row blocks
COLSUM_REF = [("f64", 3000, 600, 1700), ("f32", 2000, 600, 4000), ("f64", 1500, 3000, 300)]


@pytest.mark.parametrize("dt,n,d,l", COLSUM_REF, ids=["%s-d%d" % (c[0], c[2]) for c in COLSUM_REF])
def test_colsum_matches_float64(be, sms, dt, n, d, l):
    X, keep = _random_case(n, d, l, 61)
    gamma = 1.0 / d
    g = sc.nystrom_geom(0, n, d, l, 0, dt, sms)
    x, pack = _rows(X, dt), _pack(be, keep, dt)
    got = _colsum(be, x, pack, l, gamma, launches=g.launches + 1)
    _same(got, _colsum(be, x, pack, l, gamma))
    y, xn, cn = _ref_parts(X, keep)
    v = torch.exp(-gamma * y)
    want = v.sum(0)
    # per term: exponent off by gamma tau (||x||^2 + ||c||^2), exp and the float64 adds of n terms on both sides
    bound = 2 * gamma * tau(dt, d) * (v.T @ xn + cn * want) + (n + 8) * 2.0 ** -52 * want
    if dt == "f32":
        bound = bound + 4e-6 * want
    want, bound = want.cpu().numpy(), bound.cpu().numpy()
    assert (np.abs(got - want) <= bound).all(), np.max(np.abs(got - want) / bound)
    chain = _colsum(be, x, pack, l, gamma, chunks=3)
    assert (np.abs(chain - want) <= bound).all()


# (dt, n, d, l, k): EMBED run blocked
EMBED_REF = [("f64", 2000, 600, 2700, 10), ("f32", 2000, 600, 6000, 70), ("f64", 1000, 3000, 1500, 3)]


@pytest.mark.parametrize("dt,n,d,l,k", EMBED_REF, ids=["%s-d%d" % (c[0], c[2]) for c in EMBED_REF])
def test_embed_matches_float64(be, sms, dt, n, d, l, k):
    X, keep = _random_case(n, d, l, 71)
    W = np.random.RandomState(72).standard_normal((l, k))
    Wq = W.astype(NP[dt]).astype(np.float64)
    gamma = 1.0 / d
    g = sc.nystrom_geom(1, n, d, l, k, dt, sms)
    assert not g.one
    x, pack = _rows(X, dt), _pack(be, keep, dt)
    got = _embed(be, x, pack, l, gamma, W)[:, :k].astype(np.float64)
    _same(got, _embed(be, x, pack, l, gamma, W)[:, :k].astype(np.float64))
    y, xn, cn = _ref_parts(X, keep)
    m = y.min(1, keepdim=True).values
    v = torch.exp(-gamma * (y - m))
    Wd = torch.from_numpy(Wq).cuda()
    e = v @ Wd
    ne = torch.sqrt((e * e).sum(1, keepdim=True))
    want = (e / ne).cpu().numpy()
    # each kernel value off by its exponent's bound (twice: y and m) plus rounding, the fma chain over l keep rows and the
    # norm over k outputs; relative to ||e||, the sum of |v W| sets the scale
    delta = 2 * gamma * tau(dt, d) * (xn + cn.max()) * 2 + (l + k + 8) * 2 * EPS[dt]
    scale = torch.sqrt(((v @ Wd.abs()) ** 2).sum(1)) / ne[:, 0]
    bound = (2 * delta * scale + 8 * EPS[dt]).cpu().numpy()
    err = np.abs(got - want).max(1)
    assert (err <= bound).all(), np.max(err / bound)


# (dt, n, d, k): every row tile below 64
TRANSFORM_REF = [("f64", 3000, 900, 300), ("f32", 3000, 1700, 100), ("f64", 700, 12800, 9)]


@pytest.mark.parametrize("dt,n,d,k", TRANSFORM_REF, ids=["%s-d%d" % (c[0], c[2]) for c in TRANSFORM_REF])
def test_transform_matches_float64(be, sms, dt, n, d, k):
    X, C = _random_case(n, d, k, 81)
    assert sc.transform_geom(n, d, k, dt, sms).TR < 64
    x, pack = _rows(X, dt), _pack(be, C, dt)
    y, xn, cn = _ref_parts(X, C)
    ebound = (2 * tau(dt, d) * (xn[:, None] + cn[None, :]) + 4 * EPS[dt] * y).cpu().numpy()
    y = y.cpu().numpy()
    sq = _transform(be, x, pack, k, 1)[:, :k].astype(np.float64)
    _same(sq, _transform(be, x, pack, k, 1)[:, :k].astype(np.float64))
    assert (np.abs(sq - y) <= ebound).all()
    dist = _transform(be, x, pack, k, 0)[:, :k].astype(np.float64)
    assert (np.abs(dist ** 2 - y) <= ebound + 4 * EPS[dt] * y).all()
    gamma = 1.0 / d
    rb = _transform(be, x, pack, k, 2, gamma)[:, :k].astype(np.float64)
    ref = np.exp(-gamma * y)
    assert (np.abs(rb - ref) <= ref * (gamma * ebound + 4 * EPS[dt] * (1 + gamma * y))).all()


# ---------------------------------------------------------------------------------------------------------------------
# routing: the tensor-path shapes on rows that are not 16-byte aligned fall back, counted, to the same CUDA-core kernel
# ---------------------------------------------------------------------------------------------------------------------
def test_unaligned_tensor_shapes_fall_back_to_the_cuda_core_pass(be):
    from dask_ml_b200 import _lib

    n, d, l = 3000, 5, 7
    X, keep = _random_case(n, d, l, 91)
    x = _rows(X, "f32")                                     # pitch d + 5 = 10 floats: not a multiple of 4
    pack = _pack(be, keep, "f32")
    W = np.random.RandomState(92).standard_normal((l, 64))
    assert sc.route("colsum", "f32", d, l, ldx=x.stride(0)) == ("simt", True)
    assert sc.route("embed", "f32", d, l, kw=64, ldx=x.stride(0)) == ("simt", True)
    assert sc.route("embed", "f32", d, l, kw=65, ldx=x.stride(0)) == ("simt", False)
    assert sc.route("transform", "f32", d, l, ldx=x.stride(0), force_simt=True) == ("simt", False)

    def both(run):
        f0 = _fallbacks(be)
        a = run()
        counted = _fallbacks(be) - f0
        old = be.flags
        be.flags = _lib.FLAG_FORCE_SIMT
        try:
            f0 = _fallbacks(be)
            b = run()
            assert _fallbacks(be) == f0
        finally:
            be.flags = old
        _same(a, b)
        return counted

    assert both(lambda: _colsum(be, x, pack, l, 0.5)) == 1
    assert both(lambda: _embed(be, x, pack, l, 0.5, W)) == 1
    assert both(lambda: _embed(be, x, pack, l, 0.5, np.ones((l, 65)))) == 0
    assert both(lambda: _transform(be, x, pack, l, 1)) == 1


# ---------------------------------------------------------------------------------------------------------------------
# d) the estimators
# ---------------------------------------------------------------------------------------------------------------------
def test_spectral_clustering_with_a_blocked_embedding():
    """float64 rows with d4 + l + k = 600 + 2700 + 3 > 3200: the embedding pass runs two blocks of keep rows."""
    from sklearn.base import BaseEstimator

    import spectral_oracle as so
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.cluster import SpectralClustering

    class Rec(BaseEstimator):
        def __init__(self, n_clusters=2):
            self.n_clusters = n_clusters

        def fit(self, X, y=None):
            self.X_ = np.asarray(X)
            self.labels_ = np.zeros(len(self.X_), dtype=np.int32)
            return self

    n, d, l, k = 3000, 600, 2700, 3
    assert not sc.nystrom_geom(1, n, d, l, k, "f64", 132).one
    X, _ = _random_case(n, d, 1, 101)
    gamma = 1.0 / d
    rec = Rec()
    m = SpectralClustering(n_clusters=k, n_components=l, gamma=gamma, random_state=0, assign_labels=rec).fit(
        ChunkedArray.from_array(X, 1000))
    keep, _ = so.keep_rows(n, l, 0, kmeans_branch=False)
    U, S = so.embed_fused(X, keep, k, gamma)
    assert so.procrustes_err(rec.X_, U) < 1e-9
    np.testing.assert_allclose(m.eigenvalues_, S, rtol=1e-9)


def test_pairwise_metrics_at_a_narrow_row_tile():
    """d = 450 float64 rows: row tile 32, and 300 columns in two column blocks (the second with a row pitch above k)."""
    import sklearn.metrics.pairwise as skp

    from dask_ml_b200.metrics import pairwise

    X, Y = _random_case(700, 450, 300, 111)
    assert sc.transform_geom(700, 450, 256, "f64", 132).TR == 32
    got = np.asarray(pairwise.euclidean_distances(X, Y))
    np.testing.assert_allclose(got, skp.euclidean_distances(X, Y), rtol=1e-11)
    got = np.asarray(pairwise.rbf_kernel(X, Y, gamma=0.01))
    np.testing.assert_allclose(got, skp.rbf_kernel(X, Y, gamma=0.01), rtol=1e-11)
