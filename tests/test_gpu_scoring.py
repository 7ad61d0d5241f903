"""bkm_metric_chunk on the device: every mode against the numpy statement of the same sums (metrics/_scoring.host_sums,
which tests/test_metrics_host.py holds against scikit-learn), every operand type, bit-identical repeats, offset targets,
NaN propagation; and the public metrics on device blocks against their host path."""
import numpy as np
import pytest
import torch

from dask_ml_b200 import ChunkedArray
from dask_ml_b200.metrics import _scoring as sc
from dask_ml_b200.metrics import accuracy_score, log_loss, mean_absolute_error, mean_squared_error, r2_score

pytestmark = pytest.mark.gpu
RTOL = 1e-12


@pytest.fixture(scope="module")
def be():
    from dask_ml_b200.engine import CudaBackend

    return CudaBackend()


def _dev(be, a):
    return a.to(be.device) if isinstance(a, torch.Tensor) else torch.as_tensor(a).to(be.device)


def _run(be, mode, a, b, w=None, shift=None, eps=0.0, m=1):
    acc = torch.full((4, m) if mode == sc.ERR else (2,), 123.0, dtype=torch.float64, device=be.device)
    be.metric_chunk(_dev(be, a), _dev(be, b), mode, acc, w=None if w is None else _dev(be, w),
                    shift=None if shift is None else _dev(be, shift), eps=eps, first=True)
    return acc.cpu().numpy()


@pytest.mark.parametrize("n", [1, 255, 70_001])
@pytest.mark.parametrize("m", [1, 3, 7, 300])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64, torch.bfloat16, torch.float16])
def test_err_mode(be, n, m, dtype):
    g = torch.Generator().manual_seed(n + m)
    a = (torch.randn(n, m, generator=g) * 3 + 5).to(dtype)
    b = (a.double() + torch.randn(n, m, generator=g).double()).to(torch.float64 if m % 2 else dtype)
    shift = a[0].double()
    got = _run(be, sc.ERR, a, b, shift=shift, m=m)
    want = sc.host_sums(sc.ERR, a.double().numpy(), b.double().numpy(), shift=shift.numpy())
    np.testing.assert_allclose(got, want, rtol=RTOL, atol=1e-9)
    again = _run(be, sc.ERR, a, b, shift=shift, m=m)
    assert got.tobytes() == again.tobytes()


@pytest.mark.parametrize("pair", [(torch.int64, torch.int64), (torch.int32, torch.int64), (torch.bool, torch.int64),
                                  (torch.bool, torch.bool), (torch.float32, torch.int64), (torch.float64, torch.bfloat16)],
                         ids=lambda p: "-".join(str(t).split(".")[-1] for t in p))
@pytest.mark.parametrize("m", [1, 4])
def test_eq_mode(be, pair, m):
    n = 40_003
    g = torch.Generator().manual_seed(m)
    hi = 2 if torch.bool in pair else 4
    a = torch.randint(0, hi, (n, m), generator=g)
    b = torch.where(torch.rand(n, m, generator=g) < 0.9, a, torch.randint(0, hi, (n, m), generator=g))
    a, b = a.to(pair[0]), b.to(pair[1])
    if m == 1:
        a, b = a.reshape(-1), b.reshape(-1)
    w = torch.rand(n, generator=g, dtype=torch.float64)
    for wt in (None, w):
        got = _run(be, sc.EQ, a, b, w=wt)
        want = sc.host_sums(sc.EQ, a.double().numpy() if a.dtype == torch.bfloat16 else a.numpy(),
                            b.double().numpy() if b.dtype == torch.bfloat16 else b.numpy(),
                            None if wt is None else wt.numpy())
        np.testing.assert_allclose(got, want, rtol=RTOL)
        assert got.tobytes() == _run(be, sc.EQ, a, b, w=wt).tobytes()


def test_eq_mode_compares_large_integers_exactly(be):
    a = torch.tensor([2 ** 62, 2 ** 62 + 1, 7], dtype=torch.int64)
    b = torch.tensor([2 ** 62 + 1, 2 ** 62 + 1, 7], dtype=torch.int64)
    np.testing.assert_array_equal(_run(be, sc.EQ, a, b), [2.0, 3.0])


@pytest.mark.parametrize("K", [1, 2, 5, 40])
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_logloss_mode(be, K, dtype):
    n = 30_011
    rng = np.random.RandomState(K)
    if K == 1:
        P = rng.rand(n)
        P[:4] = [0.0, 1.0, 1.0, 0.0]
        cls = rng.randint(0, 2, size=n).astype(np.int32)
    else:
        P = rng.dirichlet(np.ones(K), size=n)
        P[0] = np.eye(K)[0]
        cls = rng.randint(0, K, size=n).astype(np.int32)
        cls[0] = K - 1                                         # a clipped zero
    P = torch.as_tensor(P).to(dtype)
    w = rng.rand(n)
    for wt in (None, w):
        got = _run(be, sc.LOGLOSS, cls, P, w=wt, eps=1e-15)
        want = sc.host_sums(sc.LOGLOSS, cls, P.double().numpy(), wt, eps=1e-15)
        np.testing.assert_allclose(got, want, rtol=RTOL)
        assert got.tobytes() == _run(be, sc.LOGLOSS, cls, P, w=wt, eps=1e-15).tobytes()
    cls[5] = K + 3                                             # not a class of the row: NaN, as the host statement
    assert np.isnan(_run(be, sc.LOGLOSS, cls, P, eps=1e-15)[0])


def test_chunks_accumulate_and_first_overwrites(be):
    a, b = torch.arange(1000.0, dtype=torch.float64), torch.arange(1000.0, dtype=torch.float64) + 2
    acc = torch.full((4, 1), 5.0, dtype=torch.float64, device=be.device)
    be.metric_chunk(_dev(be, a[:600]), _dev(be, b[:600]), sc.ERR, acc, first=True)
    be.metric_chunk(_dev(be, a[600:]), _dev(be, b[600:]), sc.ERR, acc)
    np.testing.assert_allclose(acc.cpu().numpy()[:2, 0], [4000.0, 2000.0], rtol=RTOL)


def test_nan_propagates_as_in_numpy(be):
    a = torch.tensor([1.0, float("nan"), 3.0], dtype=torch.float64)
    b = torch.tensor([1.0, 2.0, 4.0], dtype=torch.float64)
    got = _run(be, sc.ERR, a, b, shift=torch.zeros(1, dtype=torch.float64))
    assert np.isnan(got).all()
    np.testing.assert_array_equal(_run(be, sc.EQ, a, b), sc.host_sums(sc.EQ, a.numpy(), b.numpy()))
    assert np.isnan(_run(be, sc.LOGLOSS, np.array([0, 1, 1], np.int32), torch.tensor([0.5, float("nan"), 0.2],
                                                                                      dtype=torch.float64), eps=1e-15)[0])


def _both(fn, arrays, be, sizes, **kw):
    dev = [ChunkedArray([_dev(be, b) for b in ChunkedArray.from_array(a, (tuple(sizes),)).blocks]) for a in arrays]
    host = [ChunkedArray.from_array(a, (tuple(sizes),)) for a in arrays]
    return fn(*dev, **kw), fn(*host, **kw)


def test_public_metrics_on_device_blocks_equal_the_host_path(be):
    rng = np.random.RandomState(0)
    n, sizes = 100_000, [40_000, 40_000, 20_000]
    t = 1e8 + rng.standard_normal((n, 2))                       # offset targets: r2's shift
    p = t + 0.3 * rng.standard_normal((n, 2))
    for fn in (mean_squared_error, mean_absolute_error, r2_score):
        d, h = _both(fn, [t, p], be, sizes)
        np.testing.assert_allclose(d, h, rtol=1e-10)
    import sklearn.metrics as skm

    d, _ = _both(r2_score, [t, p], be, sizes)
    np.testing.assert_allclose(d, skm.r2_score(t, p), rtol=1e-9)
    d, h = _both(mean_squared_error, [t.astype(np.float32), p], be, sizes, multioutput="raw_values")
    np.testing.assert_allclose(d, h, rtol=RTOL)
    y = rng.randint(0, 3, size=n)
    yp = np.where(rng.rand(n) < 0.8, y, 0)
    w = rng.rand(n)
    d, h = _both(lambda a, b, c, **k: accuracy_score(a, b, sample_weight=c, **k), [y, yp, w], be, sizes)
    np.testing.assert_allclose(d, h, rtol=RTOL)
    P = rng.dirichlet(np.ones(3), size=n)
    d, h = _both(lambda a, b, c: log_loss(a, b, sample_weight=c), [y, P, w], be, sizes)
    np.testing.assert_allclose(d, h, rtol=RTOL)
    np.testing.assert_allclose(d, skm.log_loss(y, P, sample_weight=w), rtol=1e-10)
    # differently chunked operands, and a host operand next to a device one
    yd = ChunkedArray([_dev(be, y[:30_000]), _dev(be, y[30_000:])])
    np.testing.assert_allclose(accuracy_score(yd, ChunkedArray.from_array(yp, 50_000)), accuracy_score(y, yp), rtol=RTOL)
