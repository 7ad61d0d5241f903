"""GaussianNB on the H100: fixture replay (resident and host-resident), the moments pass against float64 numpy, fixed
summation order, the fp32 predict path against the float64 arg-max with its error bound, ties and NaN classes, chunk
edge cases, and make_blobs data."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from test_naive_bayes_host import CASES, replay  # noqa: E402

DTYPES = {"f32": torch.float32, "f64": torch.float64, "bf16": torch.bfloat16}


def _backend(flags=0):
    from dask_ml_b200.engine import CudaBackend

    return CudaBackend(flags=flags)


def _rows(n, d, dt, seed, pitch=None, offset=0.0):
    rng = np.random.RandomState(seed)
    X = rng.standard_normal((n, d)) * rng.uniform(0.5, 2, d) + offset
    t = torch.as_tensor(X).to(DTYPES[dt])
    if pitch is not None:
        buf = torch.zeros((n, pitch), dtype=t.dtype)
        buf[:, :d] = t
        t = buf[:, :d]
    return t.cuda(), t.to(torch.float64).numpy()


def _rel(a, b):
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


@pytest.mark.parametrize("name", CASES)
@pytest.mark.parametrize("resident", [True, False])
def test_fixture_replay(name, resident):
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.engine import host_resident

    if resident:
        replay(name)
    else:
        replay(name, to_input=lambda a, r: host_resident(ChunkedArray.from_array(a, r), block_rows=333))


def _moments(be, xs, cs, K, theta=None):
    d = xs[0].shape[1]
    S = torch.full((K, d), np.nan, dtype=torch.float64, device="cuda")
    C = torch.full((K,), np.nan, dtype=torch.float64, device="cuda")
    th = None if theta is None else torch.as_tensor(theta).cuda()
    for i, (x, c) in enumerate(zip(xs, cs)):
        be.class_moments_chunk(x, c, K, S, None if th is not None else C, theta=th, first=i == 0)
    torch.cuda.synchronize()
    return S.cpu().numpy(), C.cpu().numpy()


@pytest.mark.parametrize("dt", ["f32", "f64", "bf16"])
@pytest.mark.parametrize("d", [1, 13, 64, 128, 300])
@pytest.mark.parametrize("K", [2, 10, 256, 600])
def test_moments_match_float64(dt, d, K):
    be = _backend()
    rng = np.random.RandomState(d * 1000 + K)
    ns = [0, 1, 257, 3000]
    xs, hs, cs, ys = [], [], [], []
    for i, n in enumerate(ns):
        x, h = _rows(n, d, dt, i, pitch=d + 3 if i == 2 else None, offset=100.0)
        y = rng.randint(-1, K + 1, size=n)                        # -1 and K are skipped
        xs.append(x), hs.append(h), ys.append(y)
        cs.append(torch.as_tensor(y.astype(np.int32)).cuda())
    H, Y = np.concatenate(hs), np.concatenate(ys)
    S, C = _moments(be, xs, cs, K)
    S_ref = np.stack([H[Y == k].sum(0) for k in range(K)])
    C_ref = np.array([(Y == k).sum() for k in range(K)], dtype=np.float64)
    np.testing.assert_array_equal(C, C_ref)
    assert _rel(S, S_ref) < 1e-12
    theta = np.where(C_ref[:, None] > 0, S_ref / np.maximum(C_ref, 1)[:, None], 0.0)
    Q, _ = _moments(be, xs, cs, K, theta)
    Q_ref = np.stack([((H[Y == k] - theta[k]) ** 2).sum(0) for k in range(K)])
    assert _rel(Q, Q_ref) < 1e-12
    S2, C2 = _moments(be, xs, cs, K)
    Q2, _ = _moments(be, xs, cs, K, theta)
    np.testing.assert_array_equal(S, S2)                          # fixed summation order: the same bits
    np.testing.assert_array_equal(C, C2)
    np.testing.assert_array_equal(Q, Q2)


def _model(K, d, seed, offset=0.0):
    rng = np.random.RandomState(seed)
    theta = rng.uniform(-2, 2, (K, d)) + offset
    sigma = rng.uniform(0.5, 3.0, (K, d))
    prior = rng.dirichlet(np.ones(K))
    logc = np.log(prior) - 0.5 * np.log(2 * np.pi * sigma).sum(1)
    return theta, 1.0 / sigma, logc


def _jll64(H, theta, w, logc):
    return logc[None] - 0.5 * (((H[:, None, :] - theta[None]) ** 2) * w[None]).sum(2)


def _predict(be, x, theta, w, logc, count=False, out=False, exp_out=False):
    dev = [torch.as_tensor(a).cuda() for a in (theta, w, logc)]
    n = x.shape[0]
    lab = torch.full((n,), -7, dtype=torch.int32, device="cuda")
    nd = torch.zeros(1, dtype=torch.int32, device="cuda")
    o = torch.full((n, theta.shape[0]), np.nan, dtype=torch.float64, device="cuda") if out else None
    be.nb_jll_chunk(x, *dev, labels=lab, out=o, exp_out=exp_out, n_deferred=nd)
    torch.cuda.synchronize()
    return lab.cpu().numpy(), int(nd.item()), (o.cpu().numpy() if out else None)


def _tau_bound(H, theta, w, jll):
    """E_c = tau (s_c + sqrt(s_c sum_j w theta^2)) + 2^-50 |jll_c|, tau = (d + 8) 2^-25 (DESIGN.md A21)."""
    d = H.shape[1]
    s = (((H[:, None, :] - theta[None]) ** 2) * w[None]).sum(2)
    big = (w * theta ** 2).sum(1)
    return (d + 8) * 2.0 ** -25 * (s + np.sqrt(s * big[None])) + 2.0 ** -50 * np.abs(jll)


@pytest.mark.parametrize("dt", ["f32", "bf16", "f64"])
@pytest.mark.parametrize("d,K", [(1, 3), (13, 10), (64, 10), (64, 256), (100, 40), (300, 7)])
@pytest.mark.parametrize("offset", [0.0, 1e3])
def test_labels_and_log_proba(dt, d, K, offset):
    from dask_ml_b200 import _lib

    n = 4000 if K * d <= 4000 else 1500
    theta, w, logc = _model(K, d, d + K, offset)
    rng = np.random.RandomState(7)
    # rows near class means so that the classes compete
    y = rng.randint(0, K, n)
    H0 = theta[y] + rng.standard_normal((n, d)) * 1.5
    x = torch.as_tensor(H0).to(DTYPES[dt]).cuda()
    H = x.to(torch.float64).cpu().numpy()
    jll = _jll64(H, theta, w, logc)
    srt = np.sort(jll, 1)
    margin = srt[:, -1] - srt[:, -2] if K > 1 else np.full(n, np.inf)
    want = np.argmax(jll, 1)
    lab, nd, lp = _predict(_backend(), x, theta, w, logc, out=True)
    ok = margin > 1e-9 * np.abs(srt[:, -1])                       # float64 near-ties may differ from numpy's order
    np.testing.assert_array_equal(lab[ok], want[ok])
    # labels equal the float64 path on the same rows widened to float64
    lab64, nd64, _ = _predict(_backend(), torch.as_tensor(H).cuda(), theta, w, logc)
    assert nd64 == 0
    np.testing.assert_array_equal(lab, lab64)
    if dt != "f64":
        if offset == 0.0:                                          # offset data: the bound's theta term dominates
            assert nd < 0.01 * n, nd
        lab_nr, _, _ = _predict(_backend(_lib.FLAG_NO_RECHECK), x, theta, w, logc)
        bad = np.nonzero(lab_nr != lab64)[0]
        if len(bad):
            E = _tau_bound(H, theta, w, jll)
            r = np.arange(n)
            m = jll[r, lab64][bad] - jll[r, lab_nr][bad]
            bound = (E[r, lab64] + E[r, lab_nr])[bad]
            assert (m <= bound / 4).all(), (m / bound).max()        # at least 4x headroom below the bound
    vmax = jll.max(1, keepdims=True)
    ref = jll - (np.log(np.exp(jll - vmax).sum(1, keepdims=True)) + vmax)
    if dt == "f64":
        tol = 1e-10 * np.maximum(1.0, np.abs(ref).max(1, keepdims=True))
    else:                                                          # each jll is within its E, so lse within max E
        tol = 2.0 * _tau_bound(H, theta, w, jll).max(1, keepdims=True) + 1e-12
    assert (np.abs(lp - ref) <= tol).all()
    _, _, p = _predict(_backend(), x, theta, w, logc, out=True, exp_out=True)
    assert (np.abs(p - np.exp(ref)) <= 1.01 * tol * np.maximum(p, np.exp(ref)) + 1e-300).all()
    lab2, _, lp2 = _predict(_backend(), x, theta, w, logc, out=True)
    np.testing.assert_array_equal(lab, lab2)
    np.testing.assert_array_equal(lp, lp2)                         # bit-identical on two runs


@pytest.mark.parametrize("dt", ["f32", "f64"])
def test_ties_and_nan_classes(dt):
    d, K = 5, 6
    theta, w, logc = _model(K, d, 3)
    theta[4], w[4], logc[4] = theta[1], w[1], logc[1]             # class 4 duplicates class 1: exact ties -> 1
    rng = np.random.RandomState(0)
    x = torch.as_tensor(theta[1] + 0.1 * rng.standard_normal((500, d))).to(DTYPES[dt]).cuda()
    lab, _, lp = _predict(_backend(), x, theta, w, logc, out=True)
    H = x.to(torch.float64).cpu().numpy()
    np.testing.assert_array_equal(lab, np.argmax(_jll64(H, theta, w, logc), 1))
    assert (lab != 4).all()
    np.testing.assert_array_equal(lp[:, 1], lp[:, 4])
    nanc = logc.copy()
    nanc[[2, 5]] = np.nan                                         # NaN classes: the first one wins on every row
    t2, w2 = theta.copy(), w.copy()
    t2[[2, 5]] = 0.0
    w2[[2, 5]] = 0.0
    lab, _, lp = _predict(_backend(), x, t2, w2, nanc, out=True)
    assert (lab == 2).all() and np.isnan(lp).all()
    xn = x.clone()
    xn[7, 3] = float("nan")                                       # a NaN feature: every class NaN -> class 0
    lab, _, lp = _predict(_backend(), xn, theta, w, logc, out=True)
    assert lab[7] == 0 and np.isnan(lp[7]).all() and np.isfinite(np.delete(lp, 7, 0)).all()


@pytest.mark.parametrize("dt", ["f32", "bf16", "f64"])
def test_chunk_cases(dt):
    """Empty chunks and rows with an unaligned pitch or base give what contiguous rows give."""
    d, K = 13, 9
    theta, w, logc = _model(K, d, 11)
    x, _ = _rows(1000, d, dt, 5)
    lab, _, lp = _predict(_backend(), x, theta, w, logc, out=True)
    xp, _ = _rows(1000, d, dt, 5, pitch=d + 1)
    lab_p, _, lp_p = _predict(_backend(), xp, theta, w, logc, out=True)
    np.testing.assert_array_equal(lab, lab_p)
    np.testing.assert_array_equal(lp, lp_p)
    big = torch.zeros((1001 * d + 1,), dtype=x.dtype, device="cuda")
    xo = big[1:1 + 1000 * d].view(1000, d)                          # base one element off alignment
    xo.copy_(x)
    lab_o, _, lp_o = _predict(_backend(), xo, theta, w, logc, out=True)
    np.testing.assert_array_equal(lab, lab_o)
    np.testing.assert_array_equal(lp, lp_o)
    lab_e, nd, _ = _predict(_backend(), x[:0], theta, w, logc, out=True)
    assert lab_e.shape == (0,) and nd == 0
    be = _backend()
    cls = torch.as_tensor(np.arange(1000) % K, dtype=torch.int32).cuda()
    S, C = _moments(be, [x[:0], xo, x[:0], xp], [cls[:0], cls, cls[:0], cls], K)
    S1, C1 = _moments(be, [x, x], [cls, cls], K)
    np.testing.assert_array_equal(C, C1)
    assert _rel(S, S1) < 1e-13


def test_make_blobs_device():
    from sklearn.naive_bayes import GaussianNB as SkGaussianNB

    from dask_ml_b200.datasets import make_blobs
    from dask_ml_b200.naive_bayes import GaussianNB

    X, y = make_blobs(n_samples=200_000, n_features=16, centers=12, chunks=50_000, random_state=0, device="cuda",
                      dtype=np.float32)
    assert X.blocks[0].is_cuda and y.blocks[0].is_cuda
    est = GaussianNB().fit(X, y)
    Xh, yh = X.compute(), y.compute()
    ref = SkGaussianNB(var_smoothing=0).fit(Xh.astype(np.float64), yh)
    np.testing.assert_array_equal(est.classes_, ref.classes_)
    np.testing.assert_allclose(est.theta_, ref.theta_, rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(est.sigma_, ref.var_, rtol=1e-5)
    pred = est.predict(X)
    assert pred.blocks[0].is_cuda
    agree = (pred.compute() == ref.predict(Xh.astype(np.float64))).mean()
    assert agree > 0.9999, agree
    lp = est.predict_log_proba(X)
    assert lp.blocks[0].dtype == torch.float64 and lp.shape == (200_000, 12)
