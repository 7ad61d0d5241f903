"""LabelEncoder and OneHotEncoder without a GPU: the estimators' host logic (categories_, classes_, dtypes, errors,
pickling, table growth, column groups, two ranks over gloo) on a CPU backend whose new passes are numpy restatements,
against scikit-learn 1.9 on the same numpy data; and the argument checks of the new entry points, which need no
device."""
import ctypes
import json
import os
import pickle
import socket
import sys

import numpy as np
import pytest
import scipy.sparse
import sklearn.preprocessing
import torch
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from test_impute_host import EMPTY, ImputeOracleBackend  # noqa: E402
from test_preprocessing_host import _keys  # noqa: E402

KEEP = 8
_NAN_KEY = {torch.bfloat16: 0xFFC0, torch.float32: 0xFFC00000, torch.float64: 0xFFF8000000000000}


def enc_keys(x):
    """The encoders' keys of a CPU tensor (numpy uint64, same shape): radix keys with -0.0 -> +0.0 and one NaN key for
    floats, the sign bit flipped for int32 / int64, the value for uint8 / bool."""
    if x.dtype in _NAN_KEY:
        nan = torch.isnan(x).numpy()
        z = torch.where(x == 0, torch.zeros_like(x), x)
        k = _keys(z.contiguous())
        k[nan] = np.uint64(_NAN_KEY[x.dtype])
        return k
    v = x.numpy()
    if x.dtype == torch.int32:
        return v.view(np.uint32).astype(np.uint64) ^ np.uint64(1 << 31)
    if x.dtype == torch.int64:
        return v.view(np.uint64) ^ np.uint64(1 << 63)
    return v.astype(np.uint64)


class EncodeOracleBackend(ImputeOracleBackend):
    """The CPU checker backend plus the encoders' passes, in numpy (the same algorithms, not the same code).  Its
    tables keep each column's keys sorted in the first slots of the column's range and flag a column whose keys
    exceed half its capacity, as the kernel does."""

    def distinct_chunk(self, x, keys, counts, off, total, state, first=False):
        self.launches += 1
        off = off.numpy()
        if first:
            keys.fill_(EMPTY)
            counts.zero_()
            state.zero_()
        K = enc_keys(x) if x.shape[0] else np.zeros((0, x.shape[1]), dtype=np.uint64)
        for j in range(x.shape[1]):
            cap = int(off[j + 1] - off[j])
            u = np.unique(K[:, j])
            if (u == np.uint64(0xFFFFFFFFFFFFFFFF)).any():
                state[1, j] |= 2
                u = u[u != np.uint64(0xFFFFFFFFFFFFFFFF)]
            old = keys.numpy()[off[j]: off[j + 1]]
            allk = np.union1d(old[old != EMPTY].view(np.uint64), u)
            if 2 * len(allk) > cap:
                state[1, j] |= 1
                allk = allk[: cap // 2]
            kk = np.full(cap, EMPTY, dtype=np.int64)
            kk[: len(allk)] = allk.view(np.int64)
            keys[off[j]: off[j + 1]] = torch.from_numpy(kk)
            counts[off[j]: off[j + 1]] = torch.from_numpy((kk != EMPTY).astype(np.int64))
            state[0, j] = len(allk)

    def encode_chunk(self, x, cat_keys, cat_off, n_cats, layout, out, unknown, indices=None):
        self.launches += 1
        n, d = x.shape
        off = cat_off.numpy()
        ck = cat_keys.numpy().view(np.uint64)
        K = enc_keys(x) if n else np.zeros((0, d), dtype=np.uint64)
        pos = np.full((n, d), -1, dtype=np.int64)
        for j in range(d):
            lst = ck[off[j]: off[j + 1]]
            p = np.searchsorted(lst, K[:, j])
            hit = (p < len(lst)) & (lst[np.minimum(p, max(len(lst) - 1, 0))] == K[:, j]) if len(lst) else np.zeros(n, bool)
            pos[hit, j] = off[j] + p[hit]
            bad = K[~hit, j]
            unknown[0] += len(bad)
            seen = int(unknown[1 + j])
            unknown[1 + j] += len(bad)
            take = bad[: max(0, KEEP - seen)]
            if len(take):
                unknown[1 + d + j * KEEP + seen: 1 + d + j * KEEP + seen + len(take)] = torch.from_numpy(
                    take.view(np.int64).copy())
        if layout == 0:
            out.copy_(torch.from_numpy(np.where(pos >= 0, pos - off[:-1][None, :], -1)))
        elif layout == 1:
            dense = np.zeros((n, int(n_cats)), dtype=np.int64)
            r, c = np.nonzero(pos >= 0)
            dense[r, pos[r, c]] = 1
            out.copy_(torch.from_numpy(dense).to(out.dtype))
        else:
            indices.copy_(torch.from_numpy(pos.reshape(-1)))
            out.fill_(1)

    def decode_chunk(self, codes, cat_vals, cat_off, out, unknown):
        self.launches += 1
        n, d = codes.shape
        off = cat_off.numpy()
        c = codes.to(torch.int64).numpy()
        vals = cat_vals.numpy()
        res = np.zeros((n, d), dtype=vals.dtype)
        for j in range(d):
            k = off[j + 1] - off[j]
            ok = (c[:, j] >= 0) & (c[:, j] < k)
            res[ok, j] = vals[off[j] + c[ok, j]]
            bad = c[~ok, j]
            unknown[0] += len(bad)
            seen = int(unknown[1 + j])
            unknown[1 + j] += len(bad)
            take = bad[: max(0, KEEP - seen)]
            if len(take):
                unknown[1 + d + j * KEEP + seen: 1 + d + j * KEEP + seen + len(take)] = torch.from_numpy(take)
        out.copy_(torch.from_numpy(res))


@pytest.fixture
def cpu_backend(monkeypatch):
    from dask_ml_b200.cluster import k_means as km

    monkeypatch.setattr(km, "_BACKEND_FACTORY", EncodeOracleBackend)


def _np(a):
    return a.compute() if hasattr(a, "compute") else np.asarray(a)


def int_data(seed, n=400, d=3, dtype=np.int64):
    rng = np.random.RandomState(seed)
    X = np.stack([rng.randint(0, 4, n), rng.randint(-50, 50, n), rng.choice([7, -3, 1000], n)], axis=1)[:, :d]
    return X.astype(dtype)


def float_data(seed, n=400, dtype=np.float64):
    rng = np.random.RandomState(seed)
    X = np.stack([rng.randint(0, 5, n) * 0.5, np.round(rng.standard_normal(n), 1), rng.choice([0.0, -0.0, 2.5], n)],
                 axis=1).astype(dtype)
    X[rng.uniform(size=n) < 0.1, 1] = np.nan
    return X


def assert_same_categories(got, want):
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert g.dtype == w.dtype, (g.dtype, w.dtype)
        assert len(g) == len(w)
        nan_g, nan_w = (np.isnan(g), np.isnan(w)) if g.dtype.kind == "f" else (np.zeros(len(g), bool),) * 2
        np.testing.assert_array_equal(nan_g, nan_w)
        assert (g[~nan_g] == w[~nan_w]).all()


def check_onehot(X, chunks, dtype=np.float64, **params):
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.preprocessing import OneHotEncoder

    sk = sklearn.preprocessing.OneHotEncoder(sparse_output=True, dtype=dtype).fit(X)
    want = sk.transform(X)
    for sparse in (True, False):
        enc = OneHotEncoder(sparse=sparse, dtype=dtype, **params).fit(ChunkedArray.from_array(X, chunks))
        assert_same_categories(enc.categories_, sk.categories_)
        assert enc.dtypes_ == [None] * X.shape[1]
        # a zero category is +0.0 here, where np.unique may keep -0.0 (a documented deviation)
        assert list(enc.get_feature_names_out()) == [f.replace("_-0.0", "_0.0") for f in sk.get_feature_names_out()]
        got = enc.transform(ChunkedArray.from_array(X, chunks)).compute()
        if sparse:
            assert scipy.sparse.issparse(got)
            np.testing.assert_array_equal(got.indptr, want.indptr)
            np.testing.assert_array_equal(got.indices, want.indices)
            np.testing.assert_array_equal(got.data, want.data)
            assert got.dtype == want.dtype
        else:
            assert got.dtype == np.dtype(dtype)
            np.testing.assert_array_equal(got, want.toarray())


def check_label(y, chunks):
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.preprocessing import LabelEncoder

    sk = sklearn.preprocessing.LabelEncoder().fit(y)
    le = LabelEncoder().fit(ChunkedArray.from_array(y, chunks))
    assert_same_categories([le.classes_], [np.unique(y)])
    codes = le.transform(ChunkedArray.from_array(y, chunks))
    assert codes.chunks == ChunkedArray.from_array(y, chunks).chunks
    want = sk.transform(y) if not (y.dtype.kind == "f" and np.isnan(y).any()) else np.searchsorted(np.unique(y), y)
    np.testing.assert_array_equal(codes.compute(), want)
    assert codes.compute().dtype == np.int64
    np.testing.assert_array_equal(_np(LabelEncoder().fit_transform(ChunkedArray.from_array(y, chunks))), want)
    back = le.inverse_transform(codes).compute()
    assert back.dtype == le.classes_.dtype
    np.testing.assert_array_equal(back, le.classes_[want])


DTYPES = [np.float64, np.float32, np.int64, np.int32, np.uint8, np.bool_, np.int8, np.int16, np.float16, np.uint16,
          np.uint32]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("chunks", [400, 130, 37])
def test_matches_scikit_learn(cpu_backend, dtype, chunks):
    X = (float_data(1) if np.dtype(dtype).kind == "f" else np.abs(int_data(1)) % 200).astype(dtype)
    check_onehot(X, chunks)
    check_label(X[:, 1].copy(), chunks)


@pytest.mark.parametrize("dtype", [np.float32, np.int32, np.uint8, np.bool_])
def test_output_dtypes(cpu_backend, dtype):
    check_onehot(int_data(2, d=2).astype(np.int32), 100, dtype=dtype)


def test_signed_zeros_are_one_category(cpu_backend):
    from dask_ml_b200.preprocessing import LabelEncoder, OneHotEncoder

    X = np.array([[0.0], [-0.0], [1.0], [-0.0]])
    enc = OneHotEncoder(sparse=False).fit(X)
    assert len(enc.categories_[0]) == 2 and enc.categories_[0][0] == 0 and not np.signbit(enc.categories_[0][0])
    np.testing.assert_array_equal(enc.transform(X).compute(), [[1, 0], [1, 0], [0, 1], [1, 0]])
    np.testing.assert_array_equal(LabelEncoder().fit_transform(X[:, 0]).compute(), [0, 0, 1, 0])


def test_wide_integers_stay_exact(cpu_backend):
    from dask_ml_b200.preprocessing import LabelEncoder, OneHotEncoder

    big = np.array([2 ** 53, 2 ** 53 + 1, 2 ** 53, np.iinfo(np.int64).max, np.iinfo(np.int64).min, 0], dtype=np.int64)
    le = LabelEncoder().fit(big)
    np.testing.assert_array_equal(le.classes_, np.unique(big))
    assert le.classes_.dtype == np.int64
    np.testing.assert_array_equal(le.transform(big).compute(), sklearn.preprocessing.LabelEncoder().fit_transform(big))
    np.testing.assert_array_equal(le.inverse_transform(le.transform(big)).compute(), big)
    check_onehot(np.stack([big, big[::-1]], axis=1), 4)
    enc = OneHotEncoder().fit(big[:, None])
    assert enc.categories_[0][-1] == np.iinfo(np.int64).max


def test_one_category_and_empty_blocks(cpu_backend):
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.preprocessing import LabelEncoder, OneHotEncoder

    X = np.full((50, 2), 3, dtype=np.int32)
    blocks = [X[:0], X[:20], X[20:20], X[20:]]
    enc = OneHotEncoder(sparse=False).fit(ChunkedArray(blocks))
    assert [list(c) for c in enc.categories_] == [[3], [3]]
    out = enc.transform(ChunkedArray(blocks))
    assert out.chunks[0] == (0, 20, 0, 30)
    np.testing.assert_array_equal(out.compute(), np.ones((50, 2)))
    le = LabelEncoder().fit(ChunkedArray([b[:, 0] for b in blocks]))
    np.testing.assert_array_equal(le.classes_, [3])


def test_table_growth_steps(cpu_backend, monkeypatch):
    from dask_ml_b200 import _keytables
    from dask_ml_b200.preprocessing import _encode

    X = np.stack([np.arange(3000) % 1500, np.arange(3000) % 3], axis=1).astype(np.int64)
    calls = []
    grow = _keytables.alloc

    def tables(be, caps):
        calls.append(list(caps))
        return grow(be, caps)

    monkeypatch.setattr(_encode, "INITIAL_SLOTS", 4)
    monkeypatch.setattr(_keytables, "alloc", tables)
    check_onehot(X, 700)
    # x8 per step: the 3-value column grows once (4 -> 32), the 1500-value one up to its cap (2 x 3000 rows -> 8192)
    assert calls[:5] == [[4, 4], [32, 32], [256, 32], [2048, 32], [8192, 32]]


def test_column_groups(cpu_backend, monkeypatch):
    from dask_ml_b200.preprocessing import _encode

    monkeypatch.setattr(_encode, "ENCODE_BUDGET", 1)                 # one column per group
    check_onehot(float_data(3), 150)


def test_errors_and_pickle(cpu_backend):
    from dask_ml_b200.preprocessing import LabelEncoder, OneHotEncoder

    X = int_data(4)
    with pytest.raises(NotImplementedError, match="handle_unkown='ignore'"):
        OneHotEncoder(handle_unknown="ignore").fit(X)
    with pytest.raises(ValueError, match="handle_unknown must be 'error'"):
        OneHotEncoder(handle_unknown="other").fit(X)
    with pytest.raises(ValueError, match="Unsorted categories are not yet supported"):
        OneHotEncoder(categories=[[3, 1, 2], [0], [0]]).fit(X)
    with pytest.raises(ValueError, match="Shape mismatch"):
        OneHotEncoder(categories=[[0, 1, 2, 3]]).fit(X)
    cats = [np.arange(4), np.arange(-50, 50), np.array([-3, 7, 1000])]
    with pytest.raises(ValueError) as info:
        OneHotEncoder(categories=[cats[0], cats[1][5:], cats[2]]).fit(X)
    with pytest.raises(ValueError) as sk:
        sklearn.preprocessing.OneHotEncoder(categories=[cats[0], cats[1][5:], cats[2]]).fit(X)
    assert str(info.value) == str(sk.value)
    enc = OneHotEncoder(categories=[np.arange(6)] + cats[1:]).fit(X)
    assert len(enc.get_feature_names_out()) == 6 + 100 + 3
    fitted = OneHotEncoder().fit(X)
    bad = X.copy()
    bad[7, 2] = 5
    with pytest.raises(ValueError, match=r"Found unknown categories \[np.int64\(5\)\] in column 2 during transform"):
        fitted.transform(bad)
    le = LabelEncoder().fit(X[:, 1])
    with pytest.raises(ValueError, match=r"previously unseen values \[77, 99\]"):
        le.transform(np.array([1, 99, 77, 99]))
    with pytest.raises(ValueError, match="previously unseen labels"):
        le.inverse_transform(np.array([0, 100]))
    back = pickle.loads(pickle.dumps(fitted))
    np.testing.assert_array_equal(back.transform(X).compute().toarray(), fitted.transform(X).compute().toarray())
    back = pickle.loads(pickle.dumps(le))
    np.testing.assert_array_equal(back.transform(X[:, 1]).compute(), le.transform(X[:, 1]).compute())
    with pytest.raises(NotImplementedError):
        fitted.inverse_transform(fitted.transform(X))


def test_non_numeric_goes_to_scikit_learn(cpu_backend):
    import pandas as pd

    from dask_ml_b200.preprocessing import LabelEncoder, OneHotEncoder

    s = np.array(["b", "a", "c", "a"])
    le = LabelEncoder().fit(s)
    np.testing.assert_array_equal(le.classes_, ["a", "b", "c"])
    np.testing.assert_array_equal(le.transform(s), [1, 0, 2, 0])
    enc = OneHotEncoder(sparse=False).fit(s[:, None])
    np.testing.assert_array_equal(enc.transform(s[:, None]), np.eye(3)[[1, 0, 2, 0]])
    cat = pd.Series(pd.Categorical(["x", "y", "x"], categories=["y", "x"]))
    le = LabelEncoder().fit(cat)
    np.testing.assert_array_equal(le.classes_, ["y", "x"])
    np.testing.assert_array_equal(le.transform(cat), [1, 0, 1])
    assert list(le.inverse_transform(np.array([0, 1]))) == ["y", "x"]
    num = pd.Series([3, 1, 3])
    np.testing.assert_array_equal(LabelEncoder().fit_transform(num).compute(), [1, 0, 1])


def test_input_kinds_unmodified(cpu_backend):
    from dask_ml_b200.preprocessing import LabelEncoder, OneHotEncoder

    X = float_data(5)
    keep = X.copy()
    t = torch.from_numpy(X.copy())
    a = OneHotEncoder(sparse=False).fit_transform(X).compute()
    b = OneHotEncoder(sparse=False).fit_transform(t).compute()
    np.testing.assert_array_equal(a, b)
    np.testing.assert_array_equal(X, keep)
    np.testing.assert_array_equal(t.numpy(), keep)
    np.testing.assert_array_equal(LabelEncoder().fit_transform(t[:, 0]).compute(),
                                  LabelEncoder().fit_transform(X[:, 0]).compute())


def test_abi_argument_errors():
    """The new entry points reject bad arguments before they touch a device."""
    from dask_ml_b200 import _lib

    lib = _lib.load()
    p = ctypes.c_void_p(16)
    assert lib.bkm_distinct_chunk(p, 10, 4, 3, 0, p, p, p, 8, p, 0, None) == -1          # ldx < g
    assert lib.bkm_distinct_chunk(p, 10, 4, 4, 0, p, p, None, 8, p, 0, None) == -1       # no offsets
    assert lib.bkm_distinct_chunk(p, 10, 4, 4, 0, p, p, p, 8, None, 0, None) == -1       # no state
    assert lib.bkm_distinct_chunk(p, 10, 4, 4, 3, p, p, p, 8, p, 0, None) == -2          # float16: widened first
    assert lib.bkm_distinct_chunk(p, 0, 4, 4, 5, p, p, p, 0, p, 0, None) == 0            # nothing
    args = [p, 10, 2, 2, 5, p, p, 6, 0, p, 2, 1, None, p, None]
    for i, bad in ((3, 1), (6, None), (8, 3), (10, 1), (13, None)):
        a = list(args)
        a[i] = bad
        assert lib.bkm_encode_chunk(*a) == -1, i
    a = list(args)
    a[8], a[10] = 1, 5                                                                   # dense: ld_out == n_cats
    assert lib.bkm_encode_chunk(*a) == -1
    a[10], a[9] = 6, ctypes.c_void_p(24)                                                 # dense: 16-byte aligned
    assert lib.bkm_encode_chunk(*a) == -5
    a = list(args)
    a[8], a[12] = 2, None                                                                # CSR needs indices
    assert lib.bkm_encode_chunk(*a) == -1
    a = list(args)
    a[4] = 3
    assert lib.bkm_encode_chunk(*a) == -2
    a = list(args)
    a[8], a[10], a[11] = 1, 6, 3                                                         # float16 one-hot
    assert lib.bkm_encode_chunk(*a) == -2
    dargs = [p, 10, 1, 1, 5, p, p, 8, p, 1, p, None]
    for i, bad in ((3, 0), (7, 3), (6, None), (10, None)):
        a = list(dargs)
        a[i] = bad
        assert lib.bkm_decode_chunk(*a) == -1, i
    a = list(dargs)
    a[4] = 0
    assert lib.bkm_decode_chunk(*a) == -2                                                # float codes
    a = list(dargs)
    a[1], a[0] = 0, None
    assert lib.bkm_decode_chunk(*a) == 0


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _rank_data():
    X = int_data(6, n=500)
    X[:250, 1] += 200                       # rank 0 has values rank 1 lacks, and the other way round
    X[0, 2] = np.iinfo(np.int64).max        # the empty-marker key, on one rank only
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
        from dask_ml_b200.preprocessing import LabelEncoder, OneHotEncoder
        from test_encoders_host import EncodeOracleBackend, _rank_data

        km._BACKEND_FACTORY = EncodeOracleBackend
        X = _rank_data()
        lo, hi = (0, 230) if rank == 0 else (230, 500)
        enc = OneHotEncoder(sparse=False).fit(ChunkedArray.from_array(X[lo:hi], 100))
        res = {"c%d" % j: c for j, c in enumerate(enc.categories_)}
        res["classes"] = LabelEncoder().fit(X[lo:hi, 1]).classes_
        res["onehot"] = enc.transform(X[lo:hi]).compute()
        bad = X[lo:hi].copy()
        if rank == 1:
            bad[3, 0] = 99                  # unknown on one rank: every rank raises
        try:
            enc.transform(bad)
            res["raised"] = 0
        except ValueError:
            res["raised"] = 1
        np.savez(os.path.join(out_dir, "rank%d.npz" % rank), **res)
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(600)
def test_two_ranks_equal_one_rank(tmp_path, cpu_backend):
    mp.start_processes(_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True, start_method="spawn")
    r0, r1 = np.load(tmp_path / "rank0.npz"), np.load(tmp_path / "rank1.npz")
    X = _rank_data()
    sk = sklearn.preprocessing.OneHotEncoder(sparse_output=False).fit(X)
    for j in range(3):
        np.testing.assert_array_equal(r0["c%d" % j], r1["c%d" % j])
        np.testing.assert_array_equal(r0["c%d" % j], sk.categories_[j])
    np.testing.assert_array_equal(r0["classes"], np.unique(X[:, 1]))
    np.testing.assert_array_equal(np.concatenate([r0["onehot"], r1["onehot"]]), sk.transform(X))
    assert int(r0["raised"]) == 1 and int(r1["raised"]) == 1


# ------------------------------------------------ reference fixtures ------------------------------------------------
GOLDEN = os.path.join(ROOT, "tests", "golden")
with open(os.path.join(GOLDEN, "REF_ENCODERS_MANIFEST.json")) as _f:
    MANIFEST = json.load(_f)
LABEL_CASES = sorted(k for k in MANIFEST["label"] if k.startswith("ref_enc_"))
ONEHOT_CASES = sorted(k for k in MANIFEST["onehot"] if k != "ref_enc_ohe_nan")


def _host_input(a, rows):
    from dask_ml_b200 import ChunkedArray

    return ChunkedArray.from_array(a, rows)


def replay_label(name, to_input=_host_input):
    """LabelEncoder on the fixture's y in the reference run's chunks: classes_, fit_transform, transform and inverse
    equal to the reference's; where the reference's transform rejects NaN (an expected difference) the codes are
    its fit_transform codes."""
    from dask_ml_b200.preprocessing import LabelEncoder

    case = MANIFEST["label"][name]
    f = np.load(os.path.join(GOLDEN, name + ".npz"))
    y, rows = f["y"], int(f["chunks"])
    le = LabelEncoder().fit(to_input(y, rows))
    assert_same_categories([le.classes_], [f["classes_"]])
    assert str(le.classes_.dtype) == case["classes_dtype"]
    np.testing.assert_array_equal(_np(LabelEncoder().fit_transform(to_input(y, rows))), f["fit_transform"])
    codes = le.transform(to_input(y, rows))
    if "transform_error" in case:
        assert "expected_difference" in case
        np.testing.assert_array_equal(_np(codes), f["fit_transform"])
    else:
        np.testing.assert_array_equal(_np(codes), f["transform"])
    back = _np(le.inverse_transform(codes))
    np.testing.assert_array_equal(back, f["inverse"])
    assert back.dtype == f["inverse"].dtype


def replay_onehot(name, to_input=_host_input):
    """OneHotEncoder on the fixture's X in the reference run's chunks: categories_, dtypes_ and the one-hot values
    equal to the reference's (in ``dtype``: the reference's float64 ones are an expected difference)."""
    from dask_ml_b200.preprocessing import OneHotEncoder

    case = MANIFEST["onehot"][name]
    f = np.load(os.path.join(GOLDEN, name + ".npz"))
    X, rows = f["X"], int(f["chunks"])
    params = dict(case["params"])
    if "categories" in params:
        params["categories"] = [np.asarray(c) for c in params["categories"]]
    enc = OneHotEncoder(**params).fit(to_input(X, rows))
    assert_same_categories(enc.categories_, [f["cat%d" % j] for j in range(X.shape[1])])
    assert enc.dtypes_ == case["dtypes_"]
    got = _np(enc.transform(to_input(X, rows)))
    want_dtype = np.dtype(params.get("dtype", "float64"))
    assert got.dtype == want_dtype
    assert (want_dtype == np.dtype(case["transform_dtype"])) != ("expected_difference" in case)
    if "t_indptr" in f.files:
        np.testing.assert_array_equal(got.indptr, f["t_indptr"])
        np.testing.assert_array_equal(got.indices, f["t_indices"])
        np.testing.assert_array_equal(got.data, f["t_data"])
    else:
        np.testing.assert_array_equal(got, f["t"])


def replay_nan_column(to_input=_host_input):
    """The NaN column: fit's categories are the reference's (NaN last); its transform rejects NaN (an expected
    difference), here NaN encodes as its category."""
    from dask_ml_b200.preprocessing import OneHotEncoder

    case = MANIFEST["onehot"]["ref_enc_ohe_nan"]
    assert case["transform_error"]["type"] == "ValueError" and "expected_difference" in case
    f = np.load(os.path.join(GOLDEN, "ref_enc_ohe_nan.npz"))
    X, rows = f["X"], int(f["chunks"])
    enc = OneHotEncoder(sparse=False).fit(to_input(X, rows))
    assert_same_categories(enc.categories_, [f["cat0"], f["cat1"]])
    got = _np(enc.transform(to_input(X, rows)))
    want = sklearn.preprocessing.OneHotEncoder(sparse_output=False, categories=enc.categories_).fit(X).transform(X)
    np.testing.assert_array_equal(got, want)


def replay_errors(to_input=_host_input):
    from dask_ml_b200.preprocessing import LabelEncoder, OneHotEncoder

    errs = MANIFEST["errors"]
    X = np.load(os.path.join(GOLDEN, "ref_enc_ohe_sparse_f32.npz"))["X"]
    for key in ("handle_unknown_ignore", "handle_unknown_other", "unsorted_categories", "shape_mismatch"):
        e = errs[key]
        with pytest.raises({"NotImplementedError": NotImplementedError, "ValueError": ValueError}[e["type"]]) as info:
            OneHotEncoder(**e["params"]).fit(to_input(X, 70))
        assert str(info.value) == e["message"], key
    e = errs["unknown_at_fit_numpy"]
    assert "expected_difference" in e
    with pytest.raises(ValueError) as info:
        OneHotEncoder(categories=[np.asarray(c) for c in e["params"]["categories"]]).fit(to_input(X, 70))
    assert str(info.value) == e["sklearn_message"]
    e = errs["unknown_at_transform"]
    r, c, v = e["bad"]
    bad = X.copy()
    bad[r, c] = v
    with pytest.raises(ValueError) as info:
        OneHotEncoder().fit(to_input(X, 70)).transform(to_input(bad, 70))
    assert "unseen values [np.int64(%d)]" % v in e["message"]
    assert str(info.value) == "Found unknown categories [np.int64(%d)] in column %d during transform" % (v, c)
    e = errs["le_unseen_array"]
    y = np.load(os.path.join(GOLDEN, e["fit"] + ".npz"))["y"]
    le = LabelEncoder().fit(to_input(y, 120))
    with pytest.raises(ValueError) as info:
        le.transform(to_input(np.array(e["y"]), 2))
    assert "previously unseen values" in e["message"] and "previously unseen values" in str(info.value)
    unseen = sorted(set(e["y"]) - set(y.tolist()))
    assert str(info.value).endswith(str(unseen))


@pytest.mark.parametrize("name", LABEL_CASES)
def test_fixture_label(cpu_backend, name):
    replay_label(name)


@pytest.mark.parametrize("name", ONEHOT_CASES)
def test_fixture_onehot(cpu_backend, name):
    replay_onehot(name)


def test_fixture_nan_column_and_errors(cpu_backend):
    replay_nan_column()
    replay_errors()


def test_fixture_numpy_branch_and_categorical(cpu_backend):
    """The reference's numpy branch (scikit-learn's fit, then a silent np.searchsorted for unseen labels: here an
    error, the expected difference) and its categorical branch."""
    import pandas as pd

    from dask_ml_b200.preprocessing import LabelEncoder

    c = MANIFEST["label"]["numpy_branch"]
    le = LabelEncoder().fit(np.array(c["y"]))
    np.testing.assert_array_equal(le.classes_, c["classes_"])
    np.testing.assert_array_equal(_np(le.transform(np.array(c["y"]))), c["transform"])
    assert "expected_difference" in c
    with pytest.raises(ValueError, match="previously unseen values"):
        le.transform(np.array(c["unseen_y"]))
    c = MANIFEST["label"]["categorical"]
    s = pd.Series(pd.Categorical(c["values"], categories=c["categories"]))
    np.testing.assert_array_equal(np.asarray(LabelEncoder().fit_transform(s)), c["fit_transform"])
    le = LabelEncoder().fit(s)
    assert list(le.classes_) == c["classes_"]
    np.testing.assert_array_equal(np.asarray(le.transform(s)), c["transform"])
    assert list(le.inverse_transform(np.array([2, 0, 1])).astype(str)) == c["inverse"]
