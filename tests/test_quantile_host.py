"""QuantileTransformer without a GPU: the estimator's host logic (attributes, warnings, errors, pickling, 2 ranks over
gloo) on a CPU backend whose passes are numpy, against the fixtures written by the reference's own data.py
(tests/golden/ref_quantile.py); a numpy restatement of the transform pass checked against np.interp and scipy; and
the argument checks of the new entry points, which need no device."""
import ctypes
import json
import os
import pickle
import re
import socket
import sys
import warnings

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp
from scipy import stats

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from test_preprocessing_host import PPOracleBackend, _BITS, _keys  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
with open(os.path.join(GOLDEN, "REF_QUANTILE_MANIFEST.json")) as _f:
    MANIFEST = json.load(_f)
CASES = sorted(MANIFEST["cases"])
BOUNDS = 1e-7


# ------------------------------------------------ numpy restatement of the transform pass ------------------------------
def interp(x, xp, fp):
    """numpy's interp restated branch by branch with numpy operations (each rounded once): the kernel's arithmetic."""
    x, xp, fp = np.asarray(x, dtype=np.float64), np.asarray(xp, dtype=np.float64), np.asarray(fp, dtype=np.float64)
    n = len(xp)
    if n == 1:
        return np.full(x.shape, fp[0])
    j = np.clip(np.searchsorted(xp, x, side="right") - 1, 0, n - 1)    # the last knot <= x (0 for NaN knots)
    j1 = np.minimum(j + 1, n - 1)
    with np.errstate(all="ignore"):
        slope = (fp[j1] - fp[j]) / (xp[j1] - xp[j])
        r = slope * (x - xp[j]) + fp[j]
        retry = slope * (x - xp[j1]) + fp[j1]
        bad = np.isnan(r)
        r = np.where(bad, retry, r)
        r = np.where(bad & np.isnan(retry) & (fp[j] == fp[j1]), fp[j], r)
    r = np.where((j == n - 1) | (xp[j] == x), fp[j], r)
    r = np.where(x < xp[0], fp[0], r)
    r = np.where(x > xp[-1], fp[-1], r)
    return np.where(np.isnan(x), x, r)


def transform_column(x, q, ref, inverse, distribution):
    """The reference's _transform_col on one column ``x`` (numpy of X's host dtype), restated: float64 output."""
    dist = stats.norm if distribution == "normal" else stats.uniform
    with np.errstate(all="ignore"):
        if not inverse:
            below, above = x - BOUNDS < q[0], x + BOUNDS > q[-1]               # in x's dtype (R3)
            xd = x.astype(np.float64)
            y = 0.5 * (interp(xd, q, ref) - interp(-xd, -q[::-1], -ref[::-1]))
            y[above] = 1
            y[below] = 0
            eps = BOUNDS - np.spacing(1)
            return np.clip(dist.ppf(y), dist.ppf(eps), dist.ppf(1 - eps))
        c = np.asarray(dist.cdf(x.astype(np.float64)), dtype=np.float64)
        below, above = c - BOUNDS < 0, c + BOUNDS > 1
        y = interp(c, ref, q)
        y[above] = q[-1]
        y[below] = q[0]
        return y


def transform_restated(X, quantiles, references, inverse, distribution):
    return np.stack([transform_column(X[:, j], quantiles[:, j], references, inverse, distribution)
                     for j in range(X.shape[1])], axis=1) if X.shape[0] else np.zeros(X.shape)


# ------------------------------------------------ numpy oracle of the passes ------------------------------------------
def _state_views(state, d, nq):
    from dask_ml_b200.preprocessing.data import QUANTILE_HEAD, SELECT_RECORD

    raw = state.numpy().reshape(d, 16 + 80 * nq)
    return (raw[:, :16].view(QUANTILE_HEAD)[:, 0], raw[:, 16: 16 + 64 * nq].view(SELECT_RECORD),
            raw[:, 16 + 64 * nq:].view("<u8"))


class QTOracleBackend(PPOracleBackend):
    """The CPU checker backend plus QuantileTransformer's passes, in numpy (the same algorithms, not the same code)."""

    def quantile_state_new(self, d, nq):
        return torch.zeros(d * (16 + 80 * nq), dtype=torch.uint8)

    def quantile_hist_chunk(self, x, state, nq, rnd, hist, first=False):
        self.launches += 1
        d = int(x.shape[1])
        head, rec, live = _state_views(state, d, nq)
        cap = min(2 * nq, 256 ** rnd)
        sh = _BITS[x.dtype] - 8 * (rnd + 1)
        keys = _keys(x.contiguous())
        nan = torch.isnan(x.float()).numpy()
        H = np.zeros((d, cap, 256))
        for j in range(d):
            k = keys[~nan[:, j], j]
            digit = ((k >> np.uint64(sh)) & np.uint64(255)).astype(np.int64)
            if rnd == 0:
                H[j, 0] = np.bincount(digit, minlength=256)
                continue
            L = int(head["L"][j])
            if L == 0:
                continue
            lv = live[j, :L]
            high = k >> np.uint64(sh + 8)
            pos = np.searchsorted(lv, high)
            ok = (pos < L) & (lv[np.minimum(pos, L - 1)] == high)
            np.add.at(H[j], (pos[ok], digit[ok]), 1.0)
        h = hist.view(d, cap, 256)
        if first:
            h.copy_(torch.from_numpy(H))
        else:
            h += torch.from_numpy(H)

    def quantile_select_step(self, hist, state, d, nq, rnd, dtype, qf):
        self.launches += 1
        head, rec, live = _state_views(state, d, nq)
        cap = min(2 * nq, 256 ** rnd)
        H = hist.numpy().reshape(d, cap, 256)
        qf = qf.numpy()
        for j in range(d):
            if rnd == 0:
                nv = H[j, 0].sum()
                vi = (nv - 1.0) * qf
                ranks = np.concatenate([np.floor(vi), np.floor(vi) + 1.0])
                ranks = np.where(np.concatenate([vi, vi]) >= nv - 1.0, nv - 1.0, ranks)
                ranks = np.unique(np.maximum(ranks, 0.0)) if nv > 0 else np.zeros(1)
                R = len(ranks)
                rec[j, :R] = [(0, r, nv, 0, 0) for r in ranks]
                head[j] = (nv, R, 1 if nv > 0 else 0)
            L, R = int(head["L"][j]), int(head["R"][j])
            if L == 0:
                continue
            C = np.cumsum(H[j, :L], axis=1)[rec["slot"][j, :R]]
            rank = rec["rank"][j, :R]
            b = (C <= rank[:, None]).sum(1)
            rec["rank"][j, :R] = rank - np.where(b > 0, C[np.arange(R), np.maximum(b - 1, 0)], 0.0)
            keys = (rec["key"][j, :R] << np.uint64(8)) | b.astype(np.uint64)
            rec["key"][j, :R] = keys
            start = np.concatenate([[True], keys[1:] != keys[:-1]])
            rec["slot"][j, :R] = np.cumsum(start) - 1
            live[j, : int(start.sum())] = keys[start]
            head["L"][j] = int(start.sum())

    def quantile_transform_chunk(self, x, qT, ref, inverse, distribution, clip_lo, clip_hi, out):
        self.launches += 1
        xv = x.float().numpy() if x.dtype == torch.bfloat16 else x.numpy()
        dist = "normal" if distribution == 1 else "uniform"
        out.copy_(torch.from_numpy(transform_restated(xv, qT.numpy().T, ref.numpy(), inverse, dist)))


@pytest.fixture
def cpu_backend(monkeypatch):
    from dask_ml_b200.cluster import k_means as km

    monkeypatch.setattr(km, "_BACKEND_FACTORY", QTOracleBackend)


def _np(a):
    return a.compute() if hasattr(a, "compute") else np.asarray(a)


def assert_same(name, got, want):
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape and got.dtype == want.dtype, (name, got.shape, want.shape, got.dtype, want.dtype)
    np.testing.assert_array_equal(got, want, err_msg=name)


def replay(name, to_input=None, compare_normal=None):
    """Fit, transform and inverse of this package's QuantileTransformer on the fixture's X (row chunks as in the
    reference run), compared with what the reference computed: n_quantiles_, references_, quantiles_ and uniform
    outputs bit-equal; normal outputs bit-equal, or as ``compare_normal(key, got, want, est)`` decides."""
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.preprocessing import QuantileTransformer

    case = MANIFEST["cases"][name]
    f = np.load(os.path.join(GOLDEN, name + ".npz"))
    X, Y, rows = f["X"], f["Y"], int(f["chunks"])
    to_input = to_input or (lambda a, r: ChunkedArray.from_array(a, r))
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        est = QuantileTransformer(**case.get("params", {})).fit(to_input(X, rows))
    assert [str(w.message) for w in caught if "n_quantiles" in str(w.message)] == case["warnings"]
    assert est.n_quantiles_ == int(f["n_quantiles_"])
    assert_same("references_", est.references_, f["references_"])
    assert_same("quantiles_", est.quantiles_, f["quantiles_"])
    normal = case.get("params", {}).get("output_distribution") == "normal"
    for key, src, inverse in (("transform_X", X, False), ("transform_Y", Y, False),
                              ("inverse_X", f["transform_X"], True), ("inverse_Y", f["transform_Y"], True)):
        out = est.inverse_transform(to_input(src, rows)) if inverse else est.transform(to_input(src, rows))
        got = _np(out)
        assert got.dtype == np.float64, key
        if normal and compare_normal is not None:
            compare_normal(key, got, f[key], est)
        else:
            assert_same(key, got, f[key])
    np.testing.assert_array_equal(np.load(os.path.join(GOLDEN, name + ".npz"))["X"], X)   # input untouched
    return est


@pytest.mark.parametrize("name", CASES)
def test_fixture_replay(cpu_backend, name):
    replay(name)


def test_manifest_pins_the_reference_quirks():
    c = MANIFEST["cases"]
    assert c["ref_qt_n_below_nq"]["n_quantiles_"] == 300 and c["ref_qt_n1"]["n_quantiles_"] == 1
    assert all(v["quantiles_dtype"] == "float64" and v["transform_dtype"] == "float64" for v in c.values())
    f = np.load(os.path.join(GOLDEN, "ref_qt_nan.npz"))
    assert np.isnan(f["quantiles_"][:, 1]).all() and np.isnan(f["transform_X"][:, 1]).all()       # R6
    assert np.isfinite(f["quantiles_"][:, [0, 2]]).all()
    f = np.load(os.path.join(GOLDEN, "ref_qt_f64_default.npz"))
    t = f["transform_Y"]
    assert t.min() == 9.999999977795539e-08 and t.max() == 0.9999999000000003         # the uniform clip (R2)
    # R3: the bounds test in float32 changes the outputs of the integer column against float64 input
    f = np.load(os.path.join(GOLDEN, "ref_qt_f32_integers.npz"))
    as64 = transform_restated(f["X"].astype(np.float64), f["quantiles_"], f["references_"], False, "uniform")
    assert (as64[:, 1] != f["transform_X"][:, 1]).any()
    np.testing.assert_array_equal(as64[:, [0, 2]], f["transform_X"][:, [0, 2]])


@pytest.mark.parametrize("key", sorted(MANIFEST["errors"]))
def test_reference_errors(cpu_backend, key):
    from dask_ml_b200.preprocessing import QuantileTransformer

    e = MANIFEST["errors"][key]
    with pytest.raises(ValueError) as info:
        QuantileTransformer(**e["params"]).fit(np.ones((10, 2)))
    assert type(info.value).__name__ == e["type"] and _sets_sorted(str(info.value)) == _sets_sorted(e["message"])


def _sets_sorted(msg):
    """A message with the items of each printed set sorted: a set's print order depends on the hash seed."""
    return re.sub(r"\{([^{}]*)\}", lambda m: "{%s}" % ", ".join(sorted(m.group(1).split(", "))), msg)


def test_restated_transform_matches_the_fixtures():
    for name in CASES:
        f = np.load(os.path.join(GOLDEN, name + ".npz"))
        dist = MANIFEST["cases"][name].get("params", {}).get("output_distribution", "uniform")
        for key, src, inverse in (("transform_X", f["X"], False), ("transform_Y", f["Y"], False),
                                  ("inverse_X", f["transform_X"], True), ("inverse_Y", f["transform_Y"], True)):
            got = transform_restated(src, f["quantiles_"], f["references_"], inverse, dist)
            np.testing.assert_array_equal(got, f[key], err_msg="%s %s" % (name, key))


KNOTS = [
    [0.0, 1.0, 1.0, 1.0, 2.0],                              # duplicates: the two directions land mid-run
    [-0.0, 0.0, 0.0, 1.0],                                  # signed zeros
    [-np.inf, -1.0, 0.0, 3.0, np.inf],                      # infinite knots: slope 0 on their intervals
    [-np.inf, -np.inf, 2.0, np.inf, np.inf],
    [np.nan] * 6,                                           # a NaN column's quantiles
    [3.0],                                                  # a single knot
    [1.0, 2.0],
    [0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0],                    # a constant column
    list(np.sort(np.random.RandomState(0).standard_normal(40))),
]


@pytest.mark.parametrize("k", range(len(KNOTS)))
def test_interp_restatement_matches_numpy(k):
    xp = np.asarray(KNOTS[k], dtype=np.float64)
    fp = np.linspace(0, 1, len(xp))
    x = np.concatenate([xp, np.nextafter(xp, np.inf), np.nextafter(xp, -np.inf), [-np.inf, np.inf, np.nan, -0.0, 0.0],
                        np.random.RandomState(k).uniform(-4, 4, 200)])
    for a, b, c in ((x, xp, fp), (-x, -xp[::-1], -fp[::-1]), (x, fp, xp), (x, xp, np.where(np.arange(len(xp)) % 2,
                                                                                          np.inf, fp))):
        with np.errstate(all="ignore"):
            want = np.interp(a, b, c)
        np.testing.assert_array_equal(interp(a, b, c), want)


def test_errors_and_input_kinds(cpu_backend):
    import scipy.sparse as sp
    from sklearn.exceptions import NotFittedError

    from dask_ml_b200.preprocessing import QuantileTransformer

    X = np.random.RandomState(0).standard_normal((50, 3))
    with pytest.raises(NotImplementedError):
        QuantileTransformer(n_quantiles=10).fit(sp.csr_matrix(X))
    with pytest.raises(NotFittedError):
        QuantileTransformer().transform(X)
    qt = QuantileTransformer(n_quantiles=20).fit(X)
    assert qt.n_features_in_ == 3
    with pytest.raises(ValueError, match="features"):
        qt.transform(X[:, :2])
    with pytest.raises(TypeError, match="dask.dataframe"):
        QuantileTransformer().fit(type("DataFrame", (), {"__module__": "dask.dataframe.core"})())
    keep = X.copy()
    out = qt.fit_transform(X)
    np.testing.assert_array_equal(X, keep)
    np.testing.assert_array_equal(_np(out), _np(qt.transform(X)))
    f32 = X.astype(np.float32)
    np.testing.assert_array_equal(qt.fit(f32).quantiles_, np.percentile(f32, qt.references_ * 100, axis=0))
    bad = X.copy()
    bad[3, 0], bad[4, 1], bad[5, 1] = np.nan, np.inf, -np.inf            # numpy input may hold NaN and inf
    out = _np(qt.fit(X).transform(bad))
    assert np.isnan(out[3, 0]) and out[4, 1] == np.nanmax(out) and out[5, 1] == np.nanmin(out)
    with np.errstate(invalid="ignore"):
        want = np.percentile(bad, qt.fit(bad).references_ * 100, axis=0)
    np.testing.assert_array_equal(qt.quantiles_, want)


def test_pickle_round_trip(cpu_backend):
    from dask_ml_b200.preprocessing import QuantileTransformer

    X = np.random.RandomState(2).standard_normal((60, 4))
    est = QuantileTransformer(n_quantiles=30, output_distribution="normal").fit(X)
    back = pickle.loads(pickle.dumps(est))
    assert back.get_params() == est.get_params()
    np.testing.assert_array_equal(back.quantiles_, est.quantiles_)
    np.testing.assert_array_equal(_np(back.transform(X)), _np(est.transform(X)))


def test_launches_and_column_groups(cpu_backend, monkeypatch):
    from dask_ml_b200.cluster import k_means as km
    from dask_ml_b200.engine import DeviceData
    from dask_ml_b200.preprocessing import QuantileTransformer
    from dask_ml_b200.preprocessing import data as pp

    X = np.random.RandomState(3).standard_normal((300, 5))
    be = km._get_backend()
    data = DeviceData([be.to_device(b, torch.float64) for b in (X[:100], X[100:])], be)
    qt = QuantileTransformer(n_quantiles=100).fit(data)
    assert be.launch_count() == 8 * 3                                  # 8 rounds: a histogram per chunk + a select
    want = np.percentile(X, qt.references_ * 100, axis=0)
    np.testing.assert_array_equal(qt.quantiles_, want)
    monkeypatch.setattr(pp, "HIST_BUDGET", 200 * 256 * 8 * 2)           # two columns per group: three groups
    np.testing.assert_array_equal(QuantileTransformer(n_quantiles=100).fit(data).quantiles_, want)
    assert be.launch_count() == 24 + 3 * 24


def test_abi_argument_errors():
    """The new entry points reject bad arguments before they touch a device."""
    from dask_ml_b200 import _lib

    lib = _lib.load()
    p = ctypes.c_void_p(16)
    nb = ctypes.c_size_t(0)
    assert lib.bkm_quantile_state_bytes(4, 0, ctypes.byref(nb)) == -1
    assert lib.bkm_quantile_state_bytes(0, 10, ctypes.byref(nb)) == -1
    assert lib.bkm_quantile_state_bytes(4, 1000, ctypes.byref(nb)) == 0 and nb.value == 4 * (16 + 80 * 1000)
    assert lib.bkm_quantile_hist_chunk(p, 10, 4, 3, 0, p, 10, 0, p, 0, None) == -1              # ldx < d
    assert lib.bkm_quantile_hist_chunk(p, 10, 4, 4, 0, p, 10, 4, p, 0, None) == -1              # fp32: 4 rounds
    assert lib.bkm_quantile_hist_chunk(p, 10, 4, 4, 2, p, 10, 2, p, 0, None) == -1              # bf16: 2 rounds
    assert lib.bkm_quantile_hist_chunk(p, 10, 4, 4, 5, p, 10, 0, p, 0, None) == -2              # dtype
    assert lib.bkm_quantile_hist_chunk(p, 10, 4, 4, 0, None, 10, 0, p, 0, None) == -1           # no state
    assert lib.bkm_quantile_select_step(p, p, 4, 0, 0, 0, p, None) == -1                        # n_q
    assert lib.bkm_quantile_select_step(p, p, 4, 10, 0, 0, None, None) == -1                    # no qf
    assert lib.bkm_quantile_select_step(p, p, 4, 10, 8, 1, p, None) == -1                       # fp64: 8 rounds
    assert lib.bkm_quantile_select_step(p, p, 4, 10, 0, 9, p, None) == -2
    args = [p, 10, 4, 4, 0, p, p, 10, 0, 0, 0.0, 1.0, p, 4, None]
    for i, bad in ((3, 3), (13, 3), (7, 0), (8, 2), (9, 2), (5, None), (6, None)):
        a = list(args)
        a[i] = bad
        assert lib.bkm_quantile_transform_chunk(*a) == -1, i
    a = list(args)
    a[4] = 7
    assert lib.bkm_quantile_transform_chunk(*a) == -2
    a = list(args)
    a[1], a[0], a[12] = 0, None, None
    assert lib.bkm_quantile_transform_chunk(*a) == 0                                            # n = 0: nothing


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _data():
    rng = np.random.RandomState(4)
    X = 1e4 + rng.standard_normal((700, 4)) * rng.uniform(0.5, 3, 4)
    X[:, 2] = rng.randint(0, 6, 700)
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
        from dask_ml_b200.preprocessing import QuantileTransformer
        from test_quantile_host import QTOracleBackend, _data

        km._BACKEND_FACTORY = QTOracleBackend
        X = _data()
        lo, hi = (0, 130) if rank == 0 else (130, 700)
        qt = QuantileTransformer(n_quantiles=150).fit(ChunkedArray.from_array(X[lo:hi], 100))
        np.savez(os.path.join(out_dir, "rank%d.npz" % rank), quantiles=qt.quantiles_, n=qt.n_quantiles_,
                 t=qt.transform(ChunkedArray.from_array(X[lo:hi], 100)).compute())
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(600)
def test_two_ranks_equal_one_rank(tmp_path, cpu_backend):
    from dask_ml_b200.preprocessing import QuantileTransformer

    mp.start_processes(_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True, start_method="spawn")
    r0, r1 = np.load(tmp_path / "rank0.npz"), np.load(tmp_path / "rank1.npz")
    np.testing.assert_array_equal(r0["quantiles"], r1["quantiles"])
    X = _data()
    qt = QuantileTransformer(n_quantiles=150).fit(X)
    np.testing.assert_array_equal(r0["quantiles"], qt.quantiles_)
    np.testing.assert_array_equal(np.concatenate([r0["t"], r1["t"]]), _np(qt.transform(X)))
