"""StandardScaler, MinMaxScaler and RobustScaler without a GPU: the estimators' host logic (attributes and their
dtypes, numpy's rules for NaN and inf, the percentile interpolation, errors, pickling, 2 ranks over gloo) on a CPU
backend whose passes are numpy, against the fixtures written by the reference's own data.py
(tests/golden/ref_preprocessing.py); and the argument checks of the new entry points, which need no device."""
import ctypes
import json
import os
import pickle
import socket
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle_backend import OracleBackend  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
with open(os.path.join(GOLDEN, "REF_PREPROCESSING_MANIFEST.json")) as _f:
    MANIFEST = json.load(_f)
CASES = sorted(MANIFEST["cases"])
_BITS = {torch.bfloat16: 16, torch.float32: 32, torch.float64: 64}


def _keys(x):
    """The order-preserving radix keys of a CPU tensor, as uint64 numpy."""
    bits = _BITS[x.dtype]
    if x.dtype == torch.bfloat16:
        u = x.contiguous().view(torch.int16).numpy().view(np.uint16).astype(np.uint64)
    elif x.dtype == torch.float32:
        u = x.contiguous().numpy().view(np.uint32).astype(np.uint64)
    else:
        u = x.contiguous().numpy().view(np.uint64)
    sign = np.uint64(1 << (bits - 1))
    mask = np.uint64((1 << bits) - 1) if bits < 64 else np.uint64(0xFFFFFFFFFFFFFFFF)
    return np.where(u & sign, ~u & mask, u | sign)


class PPOracleBackend(OracleBackend):
    """The CPU checker backend plus the scalers' passes, in numpy (the same algorithms, not the same code)."""

    def rows_buffer(self, n, d, dtype):
        return torch.empty((n, d), dtype=dtype)

    def colstats_chunk(self, x, shift, acc, minmax, first=False):
        self.launches += 1
        v = x.to(torch.float64).numpy()
        s = shift.numpy() if shift is not None else 0.0
        fin = np.isfinite(v)
        t = np.where(fin, v - s, 0.0)
        new = np.stack([t.sum(0), (t * t).sum(0), np.isnan(v).sum(0), (v == np.inf).sum(0), (v == -np.inf).sum(0)])
        with np.errstate(invalid="ignore"):
            lo = np.fmin.reduce(np.where(np.isnan(v), np.inf, v), axis=0, initial=np.inf)
            hi = np.fmax.reduce(np.where(np.isnan(v), -np.inf, v), axis=0, initial=-np.inf)
        if first:
            acc.copy_(torch.from_numpy(new))
            minmax.copy_(torch.from_numpy(np.stack([lo, hi])))
        else:
            acc += torch.from_numpy(new)
            minmax[0] = torch.fmin(minmax[0], torch.from_numpy(lo))
            minmax[1] = torch.fmax(minmax[1], torch.from_numpy(hi))

    def radix_state_new(self, d, T):
        return torch.zeros(d * T * 32, dtype=torch.uint8)

    def radix_hist_chunk(self, x, state, T, rnd, hist, first=False):
        from dask_ml_b200.preprocessing.data import SELECT_RECORD

        self.launches += 1
        d = int(x.shape[1])
        rec = state.numpy().view(SELECT_RECORD).reshape(d, T)
        sh = _BITS[x.dtype] - 8 * (rnd + 1)
        keys = _keys(x)
        nan = torch.isnan(x.float()).numpy()
        H = np.zeros((d, T, 256))
        for j in range(d):
            k = keys[~nan[:, j], j]
            digit = ((k >> np.uint64(sh)) & np.uint64(255)).astype(np.int64)
            if rnd == 0:
                H[j, 0] = np.bincount(digit, minlength=256)
                continue
            high = k >> np.uint64(sh + 8)
            for t in range(T):
                if rec["slot"][j, t] == t:
                    H[j, t] = np.bincount(digit[high == rec["key"][j, t]], minlength=256)
        if first:
            hist.copy_(torch.from_numpy(H))
        else:
            hist += torch.from_numpy(H)

    def radix_select_step(self, hist, state, d, T, rnd, dtype, q):
        from dask_ml_b200.preprocessing.data import SELECT_RECORD

        self.launches += 1
        rec = state.numpy().view(SELECT_RECORD).reshape(d, T)
        H = hist.numpy()
        for j in range(d):
            if rnd == 0:
                nv = H[j, 0].sum()
                for t in range(T):
                    vi = (nv - 1.0) * q[t // 2]
                    idx = np.floor(vi) + (t & 1)
                    idx = nv - 1 if vi >= nv - 1 else (0.0 if vi < 0 else idx)
                    rec[j, t] = (0, idx if nv > 0 else 0.0, nv, 0, 0)
            for t in range(T):
                cum = np.concatenate([[0.0], np.cumsum(H[j, rec["slot"][j, t]])])
                b = int(np.searchsorted(cum, rec["rank"][j, t], side="right")) - 1
                if rec["nvalid"][j, t] > 0:
                    rec["rank"][j, t] -= cum[b]
                    rec["key"][j, t] = (int(rec["key"][j, t]) << 8) | b
            for t in range(T):
                rec["slot"][j, t] = next(u for u in range(t + 1) if rec["key"][j, u] == rec["key"][j, t])

    def affine_chunk(self, x, a, b, op1, op2, out):
        self.launches += 1
        dt = np.float64 if out.dtype == torch.float64 else np.float32
        v = x.float().numpy().astype(dt) if x.dtype == torch.bfloat16 else x.numpy().astype(dt)
        if op1:
            av = a.numpy().astype(dt)
            v = v - av if op1 == 1 else v * av
        if op2:
            bv = b.numpy().astype(dt)
            v = v / bv if op2 == 1 else v + bv
        out.copy_(torch.from_numpy(np.ascontiguousarray(v)))


@pytest.fixture
def cpu_backend(monkeypatch):
    from dask_ml_b200.cluster import k_means as km

    monkeypatch.setattr(km, "_BACKEND_FACTORY", PPOracleBackend)


def _np(a):
    return a.compute() if hasattr(a, "compute") else np.asarray(a)


def _close(name, got, want, rtol):
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape and got.dtype == want.dtype, (name, got.shape, want.shape, got.dtype, want.dtype)
    np.testing.assert_array_equal(np.isnan(got), np.isnan(want), err_msg=name)
    if rtol == 0:
        np.testing.assert_array_equal(got, want, err_msg=name)
        return
    ok = np.isfinite(want)
    np.testing.assert_array_equal(got[~ok & ~np.isnan(want)], want[~ok & ~np.isnan(want)], err_msg=name)
    if ok.any():
        g, w = got[ok].astype(np.float64), want[ok].astype(np.float64)
        err = np.abs(g - w).max() / max(np.abs(w).max(), 1e-300)
        assert err <= rtol, "%s: relative error %.3g > %.3g" % (name, err, rtol)


def _estimator(case):
    from dask_ml_b200 import preprocessing

    return getattr(preprocessing, case["cls"])(**case.get("params", {}))


def replay(name, to_input=None):
    """Fit, transform and inverse_transform of this package's scaler on the fixture's X (row chunks as in the
    reference run), compared with what the reference computed.  MinMaxScaler and RobustScaler attributes and outputs
    are bit-equal (exact min / max and exact percentiles); StandardScaler's float64 statistics differ from numpy's
    pairwise sums in the last bits (float32: numpy sums in float32)."""
    from dask_ml_b200 import ChunkedArray

    case = MANIFEST["cases"][name]
    f = np.load(os.path.join(GOLDEN, name + ".npz"))
    X, rows = f["X"], int(f["chunks"])
    to_input = to_input or (lambda a, r: ChunkedArray.from_array(a, r))
    est = _estimator(case).fit(to_input(X, rows))
    f32 = X.dtype == np.float32
    exact = case["cls"] != "StandardScaler"
    for a, dt in case["attr_dtypes"].items():
        got, want = getattr(est, a), f["attr_" + a]
        if a == "n_samples_seen_":
            assert np.isnan(got) and np.isnan(want)
            continue
        tol = 0 if exact else (2e-6 if f32 else (1e-9 if a in ("var_", "scale_") else 1e-14))
        _close(a, np.asarray(got), want, tol)
        assert str(np.asarray(got).dtype) == dt
    t = _np(est.transform(to_input(X, rows)))
    tol = 0 if exact else (1e-4 if f32 else 1e-8)
    _close("transform", t, f["transform"], tol)
    inv = _np(est.inverse_transform(to_input(f["transform"], rows)))
    _close("inverse_transform", inv, f["inverse_transform"], 0 if exact else (1e-5 if f32 else 1e-12))
    np.testing.assert_array_equal(np.load(os.path.join(GOLDEN, name + ".npz"))["X"], X)   # input untouched
    return est


@pytest.mark.parametrize("name", CASES)
def test_fixture_replay(cpu_backend, name):
    replay(name)


def test_manifest_pins_dtypes_and_cases():
    c = MANIFEST["cases"]
    assert c["ref_pp_std_f32"]["attr_dtypes"]["mean_"] == "float32"
    assert c["ref_pp_rob_f32_10_90"]["attr_dtypes"]["center_"] == "float64"
    assert c["ref_pp_rob_f32_10_90"]["transform_dtype"] == "float64"
    assert c["ref_pp_mm_f32_range"]["attr_dtypes"]["scale_"] == "float32"
    f = np.load(os.path.join(GOLDEN, "ref_pp_std_nan.npz"))
    assert np.isnan(f["attr_mean_"][2]) and np.isfinite(np.delete(f["attr_mean_"], 2)).all()
    assert np.load(os.path.join(GOLDEN, "ref_pp_std_const.npz"))["attr_scale_"][1] == 1.0


@pytest.mark.parametrize("cls", sorted(MANIFEST["errors"]))
def test_reference_errors(cpu_backend, cls):
    from dask_ml_b200 import preprocessing

    e = MANIFEST["errors"][cls]
    params = {k: tuple(v) for k, v in e["params"].items()}
    with pytest.raises(ValueError) as info:
        getattr(preprocessing, cls)(**params).fit(np.ones((10, 2)))
    assert e["type"] == "ValueError" and str(info.value) == e["message"]


def test_errors_and_quirks(cpu_backend):
    from sklearn.exceptions import NotFittedError

    from dask_ml_b200.preprocessing import MinMaxScaler, RobustScaler, StandardScaler

    X = np.random.RandomState(0).standard_normal((50, 3))
    for cls in (StandardScaler, MinMaxScaler):
        with pytest.raises(NotImplementedError):
            cls().partial_fit(X)
        with pytest.raises(NotFittedError):
            cls().transform(X)
    with pytest.raises(ValueError, match="Invalid quantile range"):
        RobustScaler(quantile_range=(-1, 50)).fit(X)
    with pytest.raises(ValueError, match="Invalid quantile range"):
        RobustScaler(quantile_range=(10, 101)).fit(X)
    r = RobustScaler(with_centering=False, with_scaling=False, unit_variance=True).fit(X)
    assert r.center_.shape == (3,) and r.scale_.shape == (3,)            # always both (a reference quirk)
    np.testing.assert_array_equal(_np(r.transform(X)), X)
    s = StandardScaler(with_mean=False).fit(X)
    assert not hasattr(s, "mean_") and np.isnan(s.n_samples_seen_)
    m = MinMaxScaler(clip=True).fit(X)
    np.testing.assert_array_equal(_np(m.transform(X * 3)), X * 3 * m.scale_ + m.min_)   # clip is ignored
    with pytest.raises(TypeError, match="dask.dataframe"):
        StandardScaler().fit(type("DataFrame", (), {"__module__": "dask.dataframe.core"})())


def test_nonfinite_rules(cpu_backend):
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.preprocessing import MinMaxScaler, RobustScaler, StandardScaler

    X = np.random.RandomState(1).standard_normal((40, 5))
    X[3, 0] = np.nan
    X[5, 1], X[7, 1] = np.inf, -np.inf
    X[9, 2] = np.inf
    X[11, 3] = -np.inf
    C = ChunkedArray.from_array(X, 13)
    s = StandardScaler().fit(C)
    with np.errstate(all="ignore"):
        want_m, want_v = X.mean(0), X.var(0)
    np.testing.assert_array_equal(np.isnan(s.mean_), np.isnan(want_m))
    np.testing.assert_array_equal(s.mean_[1:4], want_m[1:4])
    np.testing.assert_allclose(s.mean_[4], want_m[4], rtol=1e-14)
    np.testing.assert_array_equal(np.isnan(s.var_), np.isnan(want_v))
    m = MinMaxScaler().fit(C)
    with np.errstate(all="ignore"):
        np.testing.assert_array_equal(m.data_min_, X.min(0))
        np.testing.assert_array_equal(m.data_max_, X.max(0))
        r = RobustScaler().fit(C)
        want = np.stack([np.percentile(X[:, j], [25, 50.0, 75]) for j in range(5)])
    np.testing.assert_array_equal(r.center_, want[:, 1])


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_percentile_helper_bit_equal(dtype):
    """percentile_from_order_stats on the order statistics numpy picks equals np.percentile bit for bit."""
    from dask_ml_b200.preprocessing.data import percentile_from_order_stats

    rng = np.random.RandomState(7)
    qs = [0, 0.1, 1, 10, 12.5, 25, 33.3, 49.99, 50.0, 66.7, 75, 90, 99.9, 100]
    for n in (1, 2, 3, 4, 7, 10, 99, 100, 101, 1000, 4097):
        cols = [rng.standard_normal(n), rng.randint(-3, 3, n).astype(float), np.full(n, -0.0),
                rng.standard_normal(n) * 1e30]
        if n > 2:
            c = rng.standard_normal(n)
            c[0], c[1] = np.inf, -np.inf
            cols.append(c)
        for c in cols:
            c = c.astype(dtype)
            s = np.sort(c)
            qf = np.asarray(qs, dtype=np.float64) / 100.0
            vi = (n - 1) * qf
            lo = np.clip(np.floor(vi), 0, n - 1).astype(int)
            lo = np.where(vi >= n - 1, n - 1, lo)
            hi = np.where(vi >= n - 1, n - 1, np.minimum(lo + 1, n - 1))
            got = percentile_from_order_stats(s[lo][None], s[hi][None], n, qs, dtype)[0]
            with np.errstate(invalid="ignore"):
                want = np.percentile(c, qs)
            assert got.dtype == want.dtype
            np.testing.assert_array_equal(got, want, err_msg="n=%d dtype=%s" % (n, np.dtype(dtype)))


def test_keys_round_trip():
    from dask_ml_b200.preprocessing.data import keys_to_values

    v = np.array([-np.inf, -3.5, -1e-38, -0.0, 0.0, 1e-45, 2.0, np.inf], dtype=np.float32)
    for dt, src in ((torch.float32, torch.from_numpy(v)), (torch.float64, torch.from_numpy(v.astype(np.float64))),
                    (torch.bfloat16, torch.from_numpy(v).to(torch.bfloat16))):
        k = _keys(src[:, None])[:, 0]
        assert (np.diff(k.astype(np.float64)) >= 0).all()
        back = keys_to_values(k, dt)
        want = src.float().numpy() if dt == torch.bfloat16 else src.numpy()
        np.testing.assert_array_equal(back.view(np.uint8), want.view(np.uint8))


def test_pickle_round_trip(cpu_backend):
    from dask_ml_b200.preprocessing import MinMaxScaler, RobustScaler, StandardScaler

    X = np.random.RandomState(2).standard_normal((60, 4))
    for est in (StandardScaler(), MinMaxScaler(feature_range=(-2, 2)), RobustScaler(quantile_range=(5, 95))):
        est.fit(X)
        back = pickle.loads(pickle.dumps(est))
        assert back.get_params() == est.get_params()
        np.testing.assert_array_equal(_np(back.transform(X)), _np(est.transform(X)))


def test_launches(cpu_backend):
    from dask_ml_b200.cluster import k_means as km
    from dask_ml_b200.engine import DeviceData
    from dask_ml_b200.preprocessing import RobustScaler, StandardScaler

    X = np.random.RandomState(3).standard_normal((300, 4))
    be = km._get_backend()
    data = DeviceData([be.to_device(b, torch.float64) for b in (X[:100], X[100:])], be)
    StandardScaler().fit(data)
    assert be.launch_count() == 2                                    # one statistics call per chunk
    RobustScaler().fit(data)
    assert be.launch_count() == 2 + 8 * 3                            # 8 rounds: a histogram per chunk + a select
    StandardScaler().fit_transform(data)
    assert be.launch_count() == 26 + 4


def test_abi_argument_errors():
    """The new entry points reject bad arguments before they touch a device."""
    from dask_ml_b200 import _lib

    lib = _lib.load()
    p = ctypes.c_void_p(16)
    nb = ctypes.c_size_t(0)
    assert lib.bkm_colstats_workspace_bytes(-1, 4, ctypes.byref(nb)) == -1
    assert lib.bkm_colstats_workspace_bytes(10, 0, ctypes.byref(nb)) == -1
    assert lib.bkm_colstats_chunk(p, 10, 4, 3, 0, None, p, p, p, 1 << 20, 0, None) == -1        # ldx < d
    assert lib.bkm_colstats_chunk(p, 10, 4, 4, 7, None, p, p, p, 1 << 20, 0, None) == -2        # dtype
    assert lib.bkm_colstats_chunk(p, 10, 4, 4, 0, None, None, p, p, 1 << 20, 0, None) == -1     # no acc
    assert lib.bkm_radix_state_bytes(4, 7, ctypes.byref(nb)) == -1                               # T > 6
    assert lib.bkm_radix_state_bytes(4, 6, ctypes.byref(nb)) == 0 and nb.value == 4 * 6 * 32
    assert lib.bkm_radix_hist_chunk(p, 10, 4, 4, 0, p, 6, 4, p, 0, None) == -1                  # fp32: 4 rounds
    assert lib.bkm_radix_hist_chunk(p, 10, 4, 4, 3, p, 6, 0, p, 0, None) == -2
    q = (ctypes.c_double * 3)(0.25, 0.5, 0.75)
    assert lib.bkm_radix_select_step(p, p, 4, 5, 0, 0, ctypes.cast(q, ctypes.c_void_p), None) == -1   # odd T
    assert lib.bkm_radix_select_step(p, p, 4, 6, 2, 2, ctypes.cast(q, ctypes.c_void_p), None) == -1   # bf16: 2
    assert lib.bkm_affine_chunk(p, 10, 4, 4, 1, p, p, 1, 1, p, 4, 0, None) == -2                # f64 -> f32
    assert lib.bkm_affine_chunk(p, 10, 4, 4, 0, None, p, 1, 1, p, 4, 0, None) == -1             # op1 without a
    assert lib.bkm_affine_chunk(p, 10, 4, 4, 0, p, p, 3, 1, p, 4, 0, None) == -1                # op1 out of range
    assert lib.bkm_affine_chunk(p, 10, 4, 4, 0, p, p, 1, 1, p, 3, 0, None) == -1                # ld_out < d
    assert lib.bkm_affine_chunk(p, 0, 4, 4, 0, p, p, 1, 1, None, 4, 0, None) == 0               # n = 0: nothing


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _data():
    rng = np.random.RandomState(4)
    X = 1e4 + rng.standard_normal((700, 5)) * rng.uniform(0.5, 3, 5)
    X[:, 3] = rng.randint(0, 4, 700)
    return X


def _worker(rank, world, port, out_dir):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    import torch.distributed as dist

    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from dask_ml_b200 import ChunkedArray
        from dask_ml_b200.cluster import k_means as km
        from dask_ml_b200.preprocessing import MinMaxScaler, RobustScaler, StandardScaler
        from test_preprocessing_host import PPOracleBackend, _data

        km._BACKEND_FACTORY = PPOracleBackend
        X = _data()
        lo, hi = (0, 130) if rank == 0 else (130, 700)
        C = ChunkedArray.from_array(X[lo:hi], 100)
        s, m, r = StandardScaler().fit(C), MinMaxScaler().fit(C), RobustScaler(quantile_range=(10, 90)).fit(C)
        np.savez(os.path.join(out_dir, "rank%d.npz" % rank), mean=s.mean_, var=s.var_, lo=m.data_min_,
                 hi=m.data_max_, center=r.center_, scale=r.scale_)
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(600)
def test_two_ranks_equal_one_rank(tmp_path, cpu_backend):
    from dask_ml_b200.preprocessing import MinMaxScaler, RobustScaler, StandardScaler

    mp.start_processes(_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True, start_method="spawn")
    r0, r1 = np.load(tmp_path / "rank0.npz"), np.load(tmp_path / "rank1.npz")
    for key in r0.files:
        np.testing.assert_array_equal(r0[key], r1[key])
    X = _data()
    s, m, r = StandardScaler().fit(X), MinMaxScaler().fit(X), RobustScaler(quantile_range=(10, 90)).fit(X)
    np.testing.assert_allclose(r0["mean"], s.mean_, rtol=1e-15)
    np.testing.assert_allclose(r0["var"], s.var_, rtol=1e-11)
    np.testing.assert_array_equal(r0["lo"], m.data_min_)
    np.testing.assert_array_equal(r0["hi"], m.data_max_)
    np.testing.assert_array_equal(r0["center"], r.center_)
    np.testing.assert_array_equal(r0["scale"], r.scale_)
