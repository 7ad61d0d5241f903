"""SimpleImputer without a GPU: the estimator's host logic (statistics_, dtypes, indicator_, warnings, errors,
pickling, two ranks over gloo) on a CPU backend whose new passes are numpy restatements, against the fixtures written
by the reference's own impute.py (tests/golden/ref_impute.py) and against scikit-learn 1.9's SimpleImputer on the same
numpy data; and the argument checks of the new entry points, which need no device."""
import ctypes
import json
import os
import pickle
import socket
import sys
import warnings

import numpy as np
import pytest
import sklearn.impute
import torch
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from test_preprocessing_host import _keys  # noqa: E402
from test_quantile_host import QTOracleBackend  # noqa: E402

EMPTY = -1                      # the all-ones key, as int64
GOLDEN = os.path.join(ROOT, "tests", "golden")
with open(os.path.join(GOLDEN, "REF_IMPUTE_MANIFEST.json")) as _f:
    MANIFEST = json.load(_f)
CASES = sorted(MANIFEST["cases"])


def _mask(v, miss_is_nan, miss):
    return np.isnan(v) if miss_is_nan else (v == miss)


def _mode_keys(x):
    """The radix keys of a CPU tensor with -0.0 folded to +0.0."""
    x = torch.where(x == 0, torch.zeros_like(x), x)
    return _keys(x.contiguous())


class ImputeOracleBackend(QTOracleBackend):
    """The CPU checker backend plus SimpleImputer's passes, in numpy (the same algorithms, not the same code).  Its
    hash tables keep each column's entries sorted in the first slots of the column's range: the kernels' layout is
    different, which the results must not depend on."""

    def impute_stats_chunk(self, x, miss_is_nan, miss, shift, acc, first=False):
        self.launches += 1
        v = x.to(torch.float64).numpy()
        m = _mask(v, miss_is_nan, miss)
        ok = ~m & np.isfinite(v)
        s = shift.numpy() if shift is not None else 0.0
        new = np.stack([m.sum(0), np.isnan(v).sum(0), np.isinf(v).sum(0), np.where(ok, v - s, 0.0).sum(0)])
        if first:
            acc.copy_(torch.from_numpy(new.astype(np.float64)))
        else:
            acc += torch.from_numpy(new.astype(np.float64))

    def quantile_hist_masked_chunk(self, x, miss, state, nq, rnd, hist, first=False):
        v = x.to(torch.float64)
        self.quantile_hist_chunk(torch.where(v == miss, torch.full_like(x, float("nan")), x), state, nq, rnd, hist,
                                 first)

    @staticmethod
    def _entries(keys, counts, off, j):
        k = keys.numpy()[off[j]: off[j + 1]]
        c = counts.numpy()[off[j]: off[j + 1]]
        used = k != EMPTY
        return k[used].view(np.uint64), c[used]

    @staticmethod
    def _store(keys, counts, off, j, k, c):
        cap = int(off[j + 1] - off[j])
        assert len(k) * 2 <= cap, (len(k), cap)              # the table never fills
        kk = np.full(cap, EMPTY, dtype=np.int64)
        cc = np.zeros(cap, dtype=np.int64)
        kk[: len(k)] = k.view(np.int64)
        cc[: len(k)] = c
        keys[off[j]: off[j + 1]] = torch.from_numpy(kk)
        counts[off[j]: off[j + 1]] = torch.from_numpy(cc)

    def _add(self, keys, counts, off, j, k_new, c_new):
        k, c = self._entries(keys, counts, off, j)
        allk = np.concatenate([k, k_new])
        allc = np.concatenate([c, c_new])
        u, inv = np.unique(allk, return_inverse=True)
        self._store(keys, counts, off, j, u, np.bincount(inv, weights=allc, minlength=len(u)).astype(np.int64))

    def mode_count_chunk(self, x, miss_is_nan, miss, keys, counts, off, total, first=False):
        self.launches += 1
        off = off.numpy()
        if first:
            keys.fill_(EMPTY)
            counts.zero_()
        v = x.to(torch.float64).numpy()
        K = _mode_keys(x)
        for j in range(x.shape[1]):
            if off[j + 1] == off[j]:
                continue
            ok = ~_mask(v[:, j], miss_is_nan, miss) & ~np.isnan(v[:, j])
            u, c = np.unique(K[ok, j], return_counts=True)
            self._add(keys, counts, off, j, u, c.astype(np.int64))

    def mode_best(self, keys, counts, off, g, total):
        self.launches += 1
        off = off.numpy()
        bk, bc, nd = np.zeros(g, dtype=np.uint64), np.zeros(g), np.zeros(g)
        for j in range(g):
            k, c = self._entries(keys, counts, off, j)
            nd[j] = len(k)
            if len(k):
                top = c == c.max()
                bk[j], bc[j] = k[top].min(), c.max()
            else:
                bk[j] = np.uint64(0xFFFFFFFFFFFFFFFF)
        return torch.from_numpy(bk.view(np.int64)), torch.from_numpy(bc), torch.from_numpy(nd)

    def mode_compact(self, keys, counts, off, g, entries):
        self.launches += 1
        off = off.numpy()
        rows = []
        for j in range(g):
            k, c = self._entries(keys, counts, off, j)
            for kk, cc in zip(k, c):
                rows.append([j, float(int(kk) >> 32), float(int(kk) & 0xFFFFFFFF), float(cc)])
        rows = rows[::-1]                                      # an order of its own
        entries[: len(rows)] = torch.tensor(rows, dtype=torch.float64).reshape(-1, 4)

    def mode_merge(self, entries, keys, counts, off, g, total):
        self.launches += 1
        off = off.numpy()
        keys.fill_(EMPTY)
        counts.zero_()
        e = entries.numpy()
        e = e[e[:, 3] > 0]
        for j in range(g):
            r = e[e[:, 0] == j]
            if len(r) and off[j + 1] > off[j]:
                k = (r[:, 1].astype(np.uint64) << np.uint64(32)) | r[:, 2].astype(np.uint64)
                self._add(keys, counts, off, j, k, r[:, 3].astype(np.int64))

    def impute_chunk(self, x, miss_is_nan, miss, stats, cols, n_keep, n_ind, n_check, inverse, out, invalid=None):
        self.launches += 1
        dt = np.float64 if out.dtype == torch.float64 else np.float32
        v = x.float().numpy() if x.dtype == torch.bfloat16 else x.numpy()
        cols = cols.numpy()
        if inverse:
            src, isrc = cols[:n_keep], cols[n_keep:]
            res = np.zeros((v.shape[0], n_keep), dtype=dt)
            for o in range(n_keep):
                if src[o] >= 0:
                    res[:, o] = v[:, src[o]]
                if isrc[o] >= 0:
                    res[v[:, isrc[o]] != 0, o] = dt(miss)
            out.copy_(torch.from_numpy(res))
            return
        m = _mask(v, miss_is_nan, miss)
        keep, ind, chk = cols[:n_keep], cols[n_keep:n_keep + n_ind], cols[n_keep + n_ind:]
        filled = np.where(m[:, keep], stats.numpy()[keep].astype(dt), v[:, keep].astype(dt))
        out.copy_(torch.from_numpy(np.hstack([filled, m[:, ind].astype(dt)])))
        if invalid is not None:
            seen = v[:, np.concatenate([keep, chk]).astype(np.int64)]
            invalid += torch.tensor([np.isnan(seen).sum(), np.isinf(seen).sum()], dtype=torch.float64)


@pytest.fixture
def cpu_backend(monkeypatch):
    from dask_ml_b200.cluster import k_means as km

    monkeypatch.setattr(km, "_BACKEND_FACTORY", ImputeOracleBackend)


def _np(a):
    return a.compute() if hasattr(a, "compute") else np.asarray(a)


def data(seed, n=300, dtype=np.float64, missing=np.nan):
    """Columns: continuous, categorical with a tie, all-missing, no-missing, skewed (one repeated value)."""
    rng = np.random.RandomState(seed)
    X = np.empty((n, 6))
    X[:, 0] = rng.standard_normal(n) * 3 + 10
    X[:, 1] = rng.randint(0, 4, n)
    X[:n // 2, 1] = np.repeat([5, 6], n // 4)                 # 5 and 6 tie
    X[:, 2] = missing
    X[:, 3] = rng.uniform(-1, 1, n)
    X[:, 4] = np.where(rng.uniform(size=n) < 0.9, 2.5, rng.standard_normal(n))
    X[:, 5] = rng.randint(-3, 3, n).astype(np.float64)
    hole = rng.uniform(size=(n, 6)) < 0.15
    hole[:, 3] = False
    X[hole] = missing
    return X.astype(dtype)


def sk_fit(X, **params):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return sklearn.impute.SimpleImputer(**params).fit(X)


def assert_stats(got, want):
    got, want = np.asarray(got), np.asarray(want)
    assert got.dtype == want.dtype and got.shape == want.shape, (got.dtype, want.dtype)
    if want.dtype == object:
        assert [repr(v) for v in got] == [repr(v) for v in want]
    else:
        np.testing.assert_array_equal(got, want)


STRATS = ["mean", "median", "most_frequent", "constant"]


def replay(name, to_input=None):
    """Fit, transform (and inverse) of this package's SimpleImputer on the fixture's X, in the reference run's row
    chunks, against what the reference computed: statistics_ bit-equal (the mean to rounding: its float64 sum is
    not numpy's sequential one), the transform and inverse bit-equal with the reference's statistics_, the
    indicator features and the warnings equal."""
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.impute import SimpleImputer

    case = MANIFEST["cases"][name]
    f = np.load(os.path.join(GOLDEN, name + ".npz"))
    X, rows, params = f["X"], int(f["chunks"]), case.get("params", {})
    to_input = to_input or (lambda a, r: ChunkedArray.from_array(a, r))
    est = SimpleImputer(**params).fit(to_input(X, rows))
    got = np.asarray(est.statistics_, dtype=np.float64)
    if params.get("strategy", "mean") == "mean":
        tol = 1e-6 if X.dtype == np.float32 else 1e-13
        np.testing.assert_allclose(got, f["statistics_"], rtol=tol, err_msg=name)
        est.statistics_ = f["statistics_"].copy()
    else:
        np.testing.assert_array_equal(got, f["statistics_"], err_msg=name)
    if case["path"] == "numpy":                  # the array path keeps X's dtype for constant, scikit-learn object
        assert str(np.asarray(est.statistics_).dtype) == case["statistics_dtype"], name
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        out = est.transform(to_input(X, rows))
    assert [str(w.message) for w in caught if "Skipping" in str(w.message)] == case["warnings"]
    t = _np(out)
    assert str(t.dtype) == case["transform_dtype"], name
    np.testing.assert_array_equal(t, f["transform"], err_msg=name)
    if "inverse" in f.files:
        np.testing.assert_array_equal(est.indicator_.features_, f["features_"])
        np.testing.assert_array_equal(_np(est.inverse_transform(to_input(t, rows))).astype(np.float64), f["inverse"])
    np.testing.assert_array_equal(np.load(os.path.join(GOLDEN, name + ".npz"))["X"], X)     # input untouched


@pytest.mark.parametrize("name", CASES)
def test_fixture_replay(cpu_backend, name):
    replay(name)


@pytest.mark.parametrize("key", sorted(MANIFEST["errors"]))
def test_reference_errors(cpu_backend, key):
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.impute import SimpleImputer

    e = MANIFEST["errors"][key]
    X = np.random.RandomState(0).uniform(size=(10, 4))
    X[X < 0.5] = np.nan
    est = SimpleImputer(**e["params"])
    if "expected_difference" in e:               # the reference's array path rejects it; here every strategy runs
        est.fit(ChunkedArray.from_array(X, 5))
        assert_stats(est.statistics_, sk_fit(X, **e["params"]).statistics_)
        return
    with pytest.raises(ValueError) as info:
        est.fit(ChunkedArray.from_array(X, 5))
    if key == "missing_values_foo":              # the reference's text names its old class; the test pins the phrase
        assert "non-NA values" in str(info.value) and "non-NA values" in e["message"]
    else:
        assert str(info.value) == e["message"]


@pytest.mark.parametrize("strategy", STRATS)
@pytest.mark.parametrize("missing", [np.nan, -1.0, 0])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("keep_empty", [False, True])
def test_matches_scikit_learn(cpu_backend, strategy, missing, dtype, keep_empty):
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.impute import SimpleImputer

    X = data(1, dtype=dtype, missing=missing)
    if missing == 0:
        X[::7, 5] = -0.0
    params = dict(strategy=strategy, missing_values=missing, keep_empty_features=keep_empty, add_indicator=True)
    want = sk_fit(X, **params)
    with warnings.catch_warnings(record=True) as w_sk:
        warnings.simplefilter("always")
        want_t = want.transform(X)
    est = SimpleImputer(**params).fit(ChunkedArray.from_array(X, 70))
    if strategy == "mean":
        np.testing.assert_allclose(est.statistics_, want.statistics_, rtol=1e-6 if dtype == np.float32 else 1e-13)
        assert est.statistics_.dtype == want.statistics_.dtype
        est.statistics_ = want.statistics_.copy()             # the transform is then compared bit for bit
    else:
        assert_stats(est.statistics_, want.statistics_)
    np.testing.assert_array_equal(est.indicator_.features_, want.indicator_.features_)
    assert list(est.get_feature_names_out()) == list(want.get_feature_names_out())
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        out = est.transform(ChunkedArray.from_array(X, 70))
    assert [str(m.message) for m in w] == [str(m.message) for m in w_sk]
    got = _np(out)
    assert got.dtype == X.dtype
    np.testing.assert_array_equal(got, want_t.astype(X.dtype))
    inv = _np(est.inverse_transform(out))
    if not keep_empty:          # scikit-learn's inverse skips kept all-missing columns and runs out of columns then
        np.testing.assert_array_equal(inv, want.inverse_transform(want_t).astype(X.dtype))


def test_median_overflow_and_ties(cpu_backend):
    from dask_ml_b200.impute import SimpleImputer

    X = np.array([[3e38, 1.0], [3e38, 2.0], [3e38, np.nan], [np.nan, 2.0], [np.nan, 1.0]], dtype=np.float32)
    for strategy in ("median", "most_frequent"):
        est = SimpleImputer(strategy=strategy).fit(X)
        assert_stats(est.statistics_, sk_fit(X, strategy=strategy).statistics_)
    assert np.isinf(SimpleImputer(strategy="median").fit(X).statistics_[0])
    assert SimpleImputer(strategy="most_frequent").fit(X).statistics_[1] == 1.0          # tie: the smaller


def test_errors(cpu_backend):
    from dask_ml_b200.impute import SimpleImputer

    X = data(2)
    with pytest.raises(ValueError, match="Can only use these strategies"):
        SimpleImputer(strategy="other").fit(X)
    with pytest.raises(ValueError, match="non-NA values"):
        SimpleImputer(missing_values="foo").fit(X)
    with pytest.raises(NotImplementedError):
        SimpleImputer(strategy=np.nanmean).fit(X)
    bad = X.copy()
    bad[3, 0] = np.inf
    for est in (SimpleImputer(), SimpleImputer(missing_values=-1)):
        with pytest.raises(ValueError) as info:
            est.fit(bad)
        with pytest.raises(ValueError) as sk:
            sklearn.impute.SimpleImputer(missing_values=est.missing_values).fit(bad)
        assert str(info.value) == str(sk.value)
    fitted = SimpleImputer(missing_values=-1).fit(np.nan_to_num(X, nan=-1))
    with pytest.raises(ValueError) as info:
        fitted.transform(X)                                    # NaN is invalid with a numeric missing value
    assert "Input X contains NaN" in str(info.value)
    with pytest.raises(ValueError) as info:
        fitted.transform(np.where(np.isnan(X), np.inf, X))
    assert "infinity" in str(info.value)
    with pytest.raises(ValueError, match="features"):
        fitted.transform(X[:, :3])
    with pytest.raises(ValueError, match="add_indicator"):
        fitted.inverse_transform(X)
    with pytest.raises(ValueError, match="cannot be cast"):
        SimpleImputer(strategy="constant", fill_value="x").fit(X)


def test_input_kinds_unmodified_and_pickle(cpu_backend):
    import torch

    from dask_ml_b200.impute import SimpleImputer

    X = data(3)
    keep = X.copy()
    want = _np(SimpleImputer(strategy="median").fit_transform(X))
    np.testing.assert_array_equal(X, keep)
    np.testing.assert_array_equal(_np(SimpleImputer(strategy="median").fit_transform(torch.from_numpy(X))), want)
    est = SimpleImputer(strategy="most_frequent", add_indicator=True).fit(X)
    back = pickle.loads(pickle.dumps(est))
    np.testing.assert_array_equal(_np(back.transform(X)), _np(est.transform(X)))
    i32 = np.nan_to_num(X, nan=-1).astype(np.int32)
    est = SimpleImputer(strategy="most_frequent", missing_values=-1).fit(i32)
    assert_stats(est.statistics_, sk_fit(i32, strategy="most_frequent", missing_values=-1).statistics_)
    assert _np(est.transform(i32)).dtype == np.float32                        # int32 is computed as float32


@pytest.mark.parametrize("missing", [np.nan, -1.0])
def test_signed_zeros_are_one_value(cpu_backend, missing):
    """-0.0 and +0.0 count as one value of the mode (+0.0): 3 + 3 zeros outnumber 4 ones."""
    from dask_ml_b200.impute import SimpleImputer

    col = np.array([0.0, -0.0, 1.0, 0.0, -0.0, 1.0, 0.0, -0.0, 1.0, 1.0, missing, 2.0])
    X = np.stack([col, col[::-1]], axis=1)
    est = SimpleImputer(strategy="most_frequent", missing_values=missing).fit(X)
    assert_stats(est.statistics_, sk_fit(X, strategy="most_frequent", missing_values=missing).statistics_)
    assert (est.statistics_ == 0).all() and not np.signbit(est.statistics_).any()


def test_column_groups(cpu_backend, monkeypatch):
    from dask_ml_b200 import impute

    X = data(4)
    want = sk_fit(X, strategy="most_frequent").statistics_
    monkeypatch.setattr(impute, "MODE_BUDGET", 1)                 # one column per group
    assert_stats(impute.SimpleImputer(strategy="most_frequent").fit(X).statistics_, want)


def test_abi_argument_errors():
    """The new entry points reject bad arguments before they touch a device."""
    from dask_ml_b200 import _lib

    lib = _lib.load()
    p = ctypes.c_void_p(16)
    nan = float("nan")
    assert lib.bkm_impute_stats_chunk(p, 10, 4, 3, 0, 1, 0.0, p, p, p, 1 << 20, 0, None) == -1      # ldx < d
    assert lib.bkm_impute_stats_chunk(p, 10, 4, 4, 0, 0, nan, p, p, p, 1 << 20, 0, None) == -1      # NaN value
    assert lib.bkm_impute_stats_chunk(p, 10, 4, 4, 0, 2, 0.0, p, p, p, 1 << 20, 0, None) == -1      # flag
    assert lib.bkm_impute_stats_chunk(p, 10, 4, 4, 7, 1, 0.0, p, p, p, 1 << 20, 0, None) == -2      # dtype
    assert lib.bkm_quantile_hist_masked_chunk(p, 10, 4, 4, 0, nan, p, 1, 0, p, 0, None) == -1       # NaN: unmasked
    assert lib.bkm_mode_count_chunk(p, 10, 4, 4, 0, 1, 0.0, p, p, None, 8, 0, None) == -1           # no offsets
    assert lib.bkm_mode_count_chunk(p, 10, 4, 4, 0, 1, 0.0, None, p, p, 8, 0, None) == -1           # no table
    assert lib.bkm_mode_count_chunk(p, 10, 4, 4, 3, 1, 0.0, p, p, p, 8, 0, None) == -2
    assert lib.bkm_mode_count_chunk(p, 0, 4, 4, 0, 1, 0.0, p, p, p, 0, 0, None) == 0                # nothing
    nb = ctypes.c_size_t(0)
    assert lib.bkm_mode_best_workspace_bytes(0, 8, ctypes.byref(nb)) == -1
    assert lib.bkm_mode_best_workspace_bytes(2, 1 << 26, ctypes.byref(nb)) == 0 and nb.value == 2 * 128 * 24
    assert lib.bkm_mode_best(p, p, p, 0, 8, p, p, p, p, 1 << 20, None) == -1
    assert lib.bkm_mode_best(p, p, p, 2, 1 << 26, p, p, p, p, 100, None) == -4                      # workspace
    assert lib.bkm_mode_compact(p, p, p, 4, None, p, None) == -1
    assert lib.bkm_mode_merge(None, 5, p, p, p, 4, 8, None) == -1
    assert lib.bkm_mode_merge(None, 0, None, None, p, 4, 0, None) == 0
    args = [p, 10, 4, 4, 0, 1, 0.0, p, p, 3, 1, 1, 0, p, 4, 0, None, None]
    for i, bad in ((3, 3), (8, None), (9, -1), (12, 2), (14, 3), (7, None)):
        a = list(args)
        a[i] = bad
        assert lib.bkm_impute_chunk(*a) == -1, i
    a = list(args)
    a[15] = 1                                                      # fp32 rows, fp64 output
    assert lib.bkm_impute_chunk(*a) == -2
    a = list(args)
    a[12], a[10], a[11] = 1, 3, 1                                  # inverse: n_ind == n_keep, no checks
    assert lib.bkm_impute_chunk(*a) == -1
    a = list(args)
    a[1], a[0], a[13] = 0, None, None
    assert lib.bkm_impute_chunk(*a) == 0                           # n = 0: nothing


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _rank_data():
    X = data(5, n=500)
    X[:250, 0] = np.round(X[:250, 0])          # rank 0 and rank 1 share some values, and each has its own
    X[200:, 0] = np.round(X[200:, 0] * 2) / 2
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
        from dask_ml_b200.impute import SimpleImputer
        from test_impute_host import ImputeOracleBackend, _rank_data

        km._BACKEND_FACTORY = ImputeOracleBackend
        X = _rank_data()
        lo, hi = (0, 230) if rank == 0 else (230, 500)
        res = {}
        for s in STRATS:
            est = SimpleImputer(strategy=s).fit(ChunkedArray.from_array(X[lo:hi], 100))
            res[s] = np.asarray(est.statistics_, dtype=np.float64)
        np.savez(os.path.join(out_dir, "rank%d.npz" % rank), **res)
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(600)
def test_two_ranks_equal_one_rank(tmp_path, cpu_backend):
    mp.start_processes(_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True, start_method="spawn")
    r0, r1 = np.load(tmp_path / "rank0.npz"), np.load(tmp_path / "rank1.npz")
    X = _rank_data()
    for s in STRATS:
        np.testing.assert_array_equal(r0[s], r1[s])
        want = np.asarray(sk_fit(X, strategy=s).statistics_, dtype=np.float64)
        if s == "mean":
            np.testing.assert_allclose(r0[s], want, rtol=1e-13)
        else:
            np.testing.assert_array_equal(r0[s], want)
