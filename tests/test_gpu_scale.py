"""Every kernel family at every power-of-two scale of the data (run with -m gpu).

The reference's E-step is float64 (scikit-learn's pairwise_distances_argmin_min on float64 centres), so its results are
equivariant under X -> 2^p X: same labels and n_iter, centres times 2^p, squared distances and inertia times 4^p
(tests/test_scale_oracle.py pins this on the CPU).  The engine's contract, "labels agree with float64 except on genuine
float64 near-ties", must therefore hold at every p that keeps the data inside the float's range, not only for data of
order 1.  The data sits on a grid (2^-12 below 2^5 for float32, 2^-4 below 2^4 for bfloat16) and the centres are rows of
it, so 2^p X and 2^p C are exact and every float64 reference at p follows from the one at p = 0 by exact scaling.

What is demanded at each p, through lloyd_chunk (with and without distances) and assign_chunk (squared and not):
  * labels equal to the float64 arg-min (up to genuine near-ties) and to the labels at p = 0; counts as at p = 0;
  * sums equal to 2^p sums(0): bit for bit on families 1 and 3 (fixed summation order, and scaling by 2^p commutes with
    rounding), to 1e-6 of the absolute row sum on families 0 and 2 (order depends on occupancy);
  * deferred rows: family 1 defers the same rows at every p (it works on s X with a power-of-two s chosen from the
    centres); families 1 and 3 defer < 1 % of the rows whose ||x||^2 + max ||c||^2 lies in [2^-100, 2^100];
  * inertia (float64) within 1e-6 of the float64 sum of the winning distances;
  * per-row distances (fp32 outputs) within 2e-6 (||x||^2 + max ||c||^2) wherever the float64 value is an fp32 normal;
    0 only where it is below fp32's range, inf only where it is above.
"""
import functools

import numpy as np
import pytest

from _util import assert_labels_match, blob_seeds, distinct_rows, grid_blobs

pytestmark = pytest.mark.gpu

P = [-112, -100, -90, -76, -64, -40, 0, 40, 64, 76, 90, 96]
P64 = P + [-400, 400]
F32_MAX = float(np.finfo(np.float32).max)
F32_TINY = float(np.finfo(np.float32).tiny)          # 2^-126
WINDOW = (2.0 ** -100, 2.0 ** 100)                   # ||x||^2 + max ||c||^2 served by the fast arithmetic

FORCE_SIMT, FORCE_TC = 1, 2
# name: (kernel family, n, d, k, dtype, backend flags)
CASES = {
    "f1_64x256": (1, 12000, 64, 256, "float32", FORCE_TC),
    "f1_41x100": (1, 12000, 41, 100, "float32", FORCE_TC),
    "f2_13x20": (2, 20000, 13, 20, "float32", 0),
    "f2_16x31": (2, 20000, 16, 31, "float32", 0),
    "f0_24x40": (0, 8000, 24, 40, "float32", FORCE_SIMT),
    "f0_128x300": (0, 3000, 128, 300, "float32", 0),      # k*d too large for shared memory: GLOBAL mode
    "f0_f64_16x8": (0, 8000, 16, 8, "float64", 0),
    "f3_128x1024": (3, 8192, 128, 1024, "bfloat16", 0),    # four centre slices
    "f3_64x300": (3, 12000, 64, 300, "bfloat16", 0),
}
CHUNK_PARAMS = [(name, p) for name in CASES for p in (P64 if CASES[name][4] == "float64" else P)]


def _grid(dtype):
    return (2.0 ** -4, 2.0 ** 4) if dtype == "bfloat16" else (2.0 ** -12, 2.0 ** 5)


def _tdt(dtype):
    import torch

    return {"float32": torch.float32, "float64": torch.float64, "bfloat16": torch.bfloat16}[dtype]


def _exact_d2(X, C):
    """Squared distances in float64.  Exact on the grid: products and their sums fit float64's mantissa."""
    return np.maximum((X * X).sum(1)[:, None] - 2.0 * (X @ C.T) + (C * C).sum(1)[None, :], 0.0)


@functools.lru_cache(maxsize=None)
def _backend(flags):
    from dask_ml_b200.engine import CudaBackend

    return CudaBackend(flags=flags)


@functools.lru_cache(maxsize=None)
def _base(name):
    """(X, C, float64 labels, float64 winning squared distances, ||x||^2 + max ||c||^2), all at p = 0."""
    fam, n, d, k, dt, _ = CASES[name]
    seed = n + d + k
    X = grid_blobs(n, d, max(2, k // 2), seed, *_grid(dt))
    C = distinct_rows(X, k, seed + 1)
    d2 = _exact_d2(X, C)
    lab = d2.argmin(1)
    scale = (X * X).sum(1) + (C * C).sum(1).max()
    return X, C, lab, d2[np.arange(n), lab], scale


@functools.lru_cache(maxsize=None)
def _run(name, p):
    """Outputs of the four chunk calls on 2^p X, 2^p C (numpy)."""
    import torch

    fam, n, d, k, dt, flags = CASES[name]
    be = _backend(flags)
    tdt, odt = _tdt(dt), (torch.float32 if dt == "bfloat16" else _tdt(dt))
    assert be.kernel_family(d, k, tdt) == fam
    X, C = _base(name)[:2]
    x = be.to_device(torch.from_numpy(np.ldexp(X, p)).to(tdt), tdt)
    pack = be.pack_centers(torch.from_numpy(np.ldexp(C, p)).to(be.device), tdt)
    r = {}
    for tag, want_dist in (("d", True), ("m", False)):
        lab = be.empty((n,), torch.int32)
        mind2 = be.empty((n,), odt) if want_dist else None
        inertia = be.zeros((1,), torch.float64) if want_dist else None
        sums, counts = be.zeros((k * d,), torch.float64), be.zeros((k,), torch.int64)
        be.lloyd_chunk(x, pack, k, lab, mind2, sums, counts, inertia)
        r["defer_" + tag] = be.deferred_rows(n, d, k, tdt)
        r["lab_" + tag] = lab.cpu().numpy()
        r["sums_" + tag] = sums.cpu().numpy().reshape(k, d)
        r["counts_" + tag] = counts.cpu().numpy()
        if want_dist:
            r["min_d"] = mind2.cpu().double().numpy()
            r["inertia_d"] = inertia.item()
    for tag, squared in (("sq", True), ("rt", False)):
        lab, mn, acc = be.empty((n,), torch.int32), be.empty((n,), odt), be.zeros((1,), torch.float64)
        be.assign_chunk(x, pack, k, lab, mn, squared, acc)
        r["defer_" + tag] = be.deferred_rows(n, d, k, tdt)
        r["lab_" + tag] = lab.cpu().numpy()
        r["min_" + tag] = mn.cpu().double().numpy()
        r["inertia_" + tag] = acc.item()
    return r


def _check_min(got, v, sc, root, fp32, what):
    """Per-row distances ``got`` against the float64 values ``v`` (``root``: distances, else squared distances)."""
    assert not np.isnan(got).any(), what
    err = np.abs(got * got - v * v) if root else np.abs(got - v)
    if not fp32:
        assert (err <= 1e-12 * sc).all(), (what, float((err / sc).max()))
        return
    normal = (v >= F32_TINY) & (v <= F32_MAX)
    rel = err[normal] / sc[normal]
    assert (rel <= 2e-6).all(), (what, "error / (||x||^2 + max ||c||^2) = %g" % rel.max())
    assert not ((got == 0) & (v >= F32_TINY)).any(), (what, "0 for an fp32-normal distance")
    assert not (np.isinf(got) & (v <= F32_MAX)).any(), (what, "inf for a distance inside fp32's range")
    below, above = v < F32_TINY, v > F32_MAX
    assert (np.abs(got[below] - v[below]) <= F32_TINY).all(), what
    assert (got[above] >= F32_MAX).all(), what


@pytest.mark.parametrize("name,p", CHUNK_PARAMS)
def test_chunk_outputs_are_power_of_two_equivariant(name, p):
    fam, n, d, k, dt, _ = CASES[name]
    X, C, lab_ref, dmin0, scale0 = _base(name)
    r, r0 = _run(name, p), _run(name, 0)

    for tag in ("d", "m", "sq", "rt"):
        assert_labels_match(r["lab_" + tag], lab_ref, X, C)      # the near-tie rule is scale-free: judged at p = 0
        np.testing.assert_array_equal(r["lab_" + tag], r0["lab_" + tag], err_msg="labels (%s) differ from p = 0" % tag)

    for tag in ("d", "m"):
        np.testing.assert_array_equal(r["counts_" + tag], r0["counts_" + tag])
        np.testing.assert_array_equal(r["counts_" + tag], np.bincount(r["lab_" + tag], minlength=k))
        want = np.ldexp(r0["sums_" + tag], p)
        if fam in (1, 3):
            np.testing.assert_array_equal(r["sums_" + tag], want, err_msg="sums (%s) != 2^p sums(0)" % tag)
        else:
            absum = np.zeros((k, d))
            np.add.at(absum, r["lab_" + tag], np.abs(np.ldexp(X, p)))
            err = np.abs(r["sums_" + tag] - want)
            assert (err <= 1e-6 * absum).all(), float((err / np.maximum(absum, 1e-300)).max())

    if fam in (1, 3):
        sc = np.ldexp(scale0, 2 * p)
        outside = int(((sc < WINDOW[0]) | (sc > WINDOW[1])).sum())
        for tag in ("d", "m", "sq", "rt"):
            if fam == 1:
                assert r["defer_" + tag] == r0["defer_" + tag], (tag, r["defer_" + tag], r0["defer_" + tag])
            assert r["defer_" + tag] <= outside + 0.01 * (n - outside), (tag, r["defer_" + tag], outside)

    fp32 = dt != "float64"
    v2, sc = np.ldexp(dmin0, 2 * p), np.ldexp(scale0, 2 * p)
    v1 = np.ldexp(np.sqrt(dmin0), p)
    for tag, v, root in (("d", v2, False), ("sq", v2, False), ("rt", v1, True)):
        want = v.sum()
        assert abs(r["inertia_" + tag] - want) <= 1e-6 * want, (tag, r["inertia_" + tag], want)
        _check_min(r["min_" + tag], v, sc, root, fp32, tag)


# ------------------------------------------------------------------------------------------ transform
XF_SHAPES = [(64, 256), (41, 100), (64, 300)]          # the family-1 shapes, and k > 256 (two column blocks)


@functools.lru_cache(maxsize=None)
def _xf_base(d, k):
    X = grid_blobs(3000, d, 16, d + k, 2.0 ** -12, 2.0 ** 5)
    Y = distinct_rows(X, k, d + k + 1)
    return X, Y, _exact_d2(X, Y), (X * X).sum(1)[:, None] + (Y * Y).sum(1)[None, :]


@functools.lru_cache(maxsize=None)
def _xf_run(d, k, mode, p):
    """_distance_blocks on 2^p X, 2^p Y; rbf with gamma 0.01 * 4^-p (so that gamma d^2 does not depend on p)."""
    import torch
    from dask_ml_b200.metrics.pairwise import _as_device, _distance_blocks

    X, Y = _xf_base(d, k)[:2]
    Xd = _as_device(torch.from_numpy(np.ldexp(X, p).astype(np.float32)).cuda())
    out = _distance_blocks(Xd, np.ldexp(Y, p), mode, 0.01 * 4.0 ** -p)[0]
    assert out.dtype == torch.float32
    return out.cpu().double().numpy()


@pytest.mark.parametrize("p", P)
@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("d,k", XF_SHAPES)
def test_transform_is_power_of_two_equivariant(d, k, mode, p):
    X, Y, d2_0, scale0 = _xf_base(d, k)
    got, got0 = _xf_run(d, k, mode, p), _xf_run(d, k, mode, 0)
    assert not np.isnan(got).any()
    sc = np.ldexp(scale0, 2 * p)
    if mode == 0:
        v = np.ldexp(np.sqrt(d2_0), p)
        err = (np.abs(got * got - v * v) / sc).max()
        assert err < 2e-6, err
        # sqrt is taken on the scaled value s^2 d^2, then divided by s: exact multiples of the p = 0 result
        want = np.ldexp(got0, p)
        ok = (want == 0) | ((want >= F32_TINY) & (want <= F32_MAX))
        np.testing.assert_array_equal(got[ok], want[ok])
    elif mode == 1:
        # the GEMM form is accurate to 2e-6 (||x||^2 + ||y||^2) (+ fp32's smallest normal): where that interval
        # reaches beyond fp32's range (e.g. the zero distance of a row to itself at p = 76), inf is inside it
        v = np.ldexp(d2_0, 2 * p)
        lo, hi = v - 2e-6 * sc - F32_TINY, v + 2e-6 * sc + F32_TINY
        ok = (np.isfinite(got) & (got >= lo) & (got <= hi)) | (np.isinf(got) & (hi > 0.5 * F32_MAX))
        assert ok.all(), "%d of %d outside the bound" % ((~ok).sum(), ok.size)
    else:
        err = np.abs(got - np.exp(-0.01 * d2_0)).max() / (0.01 * scale0.max())
        assert err < 2e-6, err
        np.testing.assert_array_equal(got, got0)


def test_euclidean_distances_tiny_data_matches_sklearn():
    """The public operator on float32 data of order 2^-75 (the tensor path scales it by 2^84 and back)."""
    import sklearn.metrics
    import dask_ml_b200.metrics as m
    from dask_ml_b200 import ChunkedArray

    X, Y = _xf_base(41, 100)[:2]
    Xs, Ys = np.ldexp(X, -80).astype(np.float32), np.ldexp(Y, -80).astype(np.float32)
    got = m.euclidean_distances(ChunkedArray.from_array(Xs, 1000), Ys).compute()
    assert got.dtype == np.float32
    want = sklearn.metrics.euclidean_distances(Xs.astype(np.float64), Ys.astype(np.float64))
    sc = (Xs.astype(np.float64) ** 2).sum(1)[:, None] + (Ys.astype(np.float64) ** 2).sum(1)[None, :]
    err = (np.abs(got.astype(np.float64) ** 2 - want ** 2) / sc).max()
    assert err < 2e-6, err


# ------------------------------------------------------------------------------------------ fit
P_FIT = [-100, -64, 0, 64, 96]
# name: (kernel family, n, d, k, dtype): a family-1, a family-2 and a family-3 shape
FITS = {"f1_41x100": (1, 20000, 41, 100, "float32"), "f2_13x20": (2, 20000, 13, 20, "float32"),
        "f3_64x100": (3, 20000, 64, 100, "bfloat16")}


@functools.lru_cache(maxsize=None)
def _fit_base(name):
    fam, n, d, k, dt = FITS[name]
    X, blob = grid_blobs(n, d, k, 3 * k + d, *_grid(dt), std=0.02, return_blob=True)
    return X, blob_seeds(X, blob, k)


def _as_input(X, dt):
    import torch

    return torch.from_numpy(X).to(torch.bfloat16) if dt == "bfloat16" else X.astype(np.float32)


@functools.lru_cache(maxsize=None)
def _fit(name, p):
    from dask_ml_b200.cluster import KMeans

    fam, n, d, k, dt = FITS[name]
    X, C = _fit_base(name)
    km = KMeans(n_clusters=k, init=np.ldexp(C, p), tol=1e-4 * 4.0 ** p, max_iter=30).fit(_as_input(np.ldexp(X, p), dt))
    return km.labels_.compute(), km.cluster_centers_, float(km.inertia_), km.n_iter_


@pytest.mark.parametrize("p", P_FIT)
@pytest.mark.parametrize("name", list(FITS))
def test_fit_is_power_of_two_equivariant(name, p):
    """KMeans(init=2^p C, tol=1e-4 4^p) on 2^p X: the fit at p = 0 scaled exactly.  The base fits end on a zero shift,
    so every p takes the squared-inertia branch of the reference (Q4's 1e-7 threshold is absolute).

    Families 1 and 3 form the winning distances the same way at every p (family 1 on s X, family 3 in float64), so
    their inertia scales to 1e-12.  Family 2 forms them in fp32 inside the magnitude window and in float64 outside it:
    there the bound is the 1e-6 of the fp32 distances."""
    fam = FITS[name][0]
    X = _fit_base(name)[0]
    lab0, cen0, in0, it0 = _fit(name, 0)
    assert it0 < 30
    lab, cen, inertia, n_iter = _fit(name, p)
    assert n_iter == it0
    np.testing.assert_array_equal(lab, lab0)
    np.testing.assert_array_equal(cen, np.ldexp(cen0, p))
    rtol = 1e-12 if fam in (1, 3) else 1e-6
    assert abs(inertia - 4.0 ** p * in0) <= rtol * 4.0 ** p * in0, (inertia, 4.0 ** p * in0)
    want = ((X - cen0.astype(np.float64)[lab0]) ** 2).sum() * 4.0 ** p        # float64, from the fit's own result
    assert abs(inertia - want) <= 1e-6 * want, (inertia, want)


def test_fit_kmeans_parallel_is_scale_free():
    """k-means|| compares l d^2 / phi with the Philox draw: the ratio, and so the sampled candidates, do not depend on
    a power-of-two scale of the data.  The number of rounds does: the reference runs min(init_max_iter,
    round(log(cost))) of them, so the lowest exponent is the one that keeps round(log(cost)) >= init_max_iter (cost
    ~1e8 at p = 0 here; at p = -40 the reference itself would run no round at all)."""
    from dask_ml_b200.cluster import KMeans

    X = _fit_base("f2_13x20")[0].astype(np.float32)
    res = []
    for p in (-8, 0, 40):
        km = KMeans(n_clusters=20, init="k-means||", random_state=0, init_max_iter=3, tol=1e-4 * 4.0 ** p,
                    max_iter=300).fit(np.ldexp(X, p))
        res.append((km.labels_.compute(), km.n_iter_))
    # a loop cut off by max_iter would end on a non-zero shift, and Q4's absolute threshold would then re-label at some
    # p and not at others
    assert res[1][1] < 300
    for lab, it in res[1:]:
        assert it == res[0][1], [r[1] for r in res]
        assert (lab == res[0][0]).all(), [int((r[0] != res[0][0]).sum()) for r in res]
