"""LabelEncoder and OneHotEncoder on the device, against scikit-learn 1.9 on the same numpy data (float32-widened for
bf16): categories, codes, dense one-hot and CSR bit-equal for every input dtype and three chunkings, a column of 10^5
categories (global-memory search and table growth), INT64_MAX / INT64_MIN and 2^53 + 1, the device input blocks left
unmodified, the unknown-value error after a multi-chunk transform, and the outputs fed to LogisticRegression and
GaussianNB; and the replay of the reference fixtures (tests/golden/ref_encoders.py) with device input."""
import os
import sys

import numpy as np
import pytest
import sklearn.preprocessing
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from test_encoders_host import (LABEL_CASES, ONEHOT_CASES, assert_same_categories, replay_errors,  # noqa: E402
                                replay_label, replay_nan_column, replay_onehot)

DTYPES = {"f32": torch.float32, "f64": torch.float64, "bf16": torch.bfloat16, "i32": torch.int32,
          "i64": torch.int64, "u8": torch.uint8, "bool": torch.bool}


def _data(dt, n=60000, seed=0, wide=False):
    """(device tensor, numpy of the same values) with columns of 4, ~200 and (``wide``) 10^5 categories, NaN and
    signed zeros for floats."""
    rng = np.random.RandomState(seed)
    cols = [rng.randint(0, 4, n), rng.randint(-100, 100, n)]
    if wide:
        cols.append(rng.permutation(np.arange(n) % 100000 if n >= 100000 else np.arange(n)) - 50000)
    X = np.stack(cols, axis=1).astype(np.float64)
    if dt in ("f32", "f64", "bf16"):
        X[:, 1] *= 0.5
        X[rng.uniform(size=n) < 0.05, 1] = np.nan
        X[::7, 0] = -0.0
    elif dt == "u8":
        X = np.abs(X) % 256
    elif dt == "bool":
        X = X % 2
    t = torch.as_tensor(X).to(DTYPES[dt]).cuda()
    h = (t.float() if dt == "bf16" else t).cpu().numpy()
    return t, h


def _device_input(a, rows):
    """The fixture's array as a ChunkedArray of CUDA blocks in the reference run's chunks."""
    t = torch.as_tensor(np.ascontiguousarray(a)).cuda()
    return _chunked(t, rows)


@pytest.mark.parametrize("name", LABEL_CASES)
def test_fixture_label(name):
    replay_label(name, _device_input)


@pytest.mark.parametrize("name", ONEHOT_CASES)
def test_fixture_onehot(name):
    replay_onehot(name, _device_input)


def test_fixture_nan_column_and_errors():
    replay_nan_column(_device_input)
    replay_errors(_device_input)


def _chunked(t, rows):
    from dask_ml_b200 import ChunkedArray

    return ChunkedArray([t[i:i + rows] for i in range(0, t.shape[0], rows)])


@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("rows", [60000, 17000, 4099])
def test_bit_equal_to_scikit_learn(dt, rows):
    from dask_ml_b200.preprocessing import LabelEncoder, OneHotEncoder

    t, h = _data(dt, wide=rows == 17000 and dt in ("f32", "f64", "i32", "i64"), n=120000 if rows == 17000 else 60000)
    keep = t.clone()
    sk = sklearn.preprocessing.OneHotEncoder(sparse_output=True, dtype=np.float32).fit(h)
    want = sk.transform(h)
    enc = OneHotEncoder(sparse=True, dtype=np.float32).fit(_chunked(t, rows))
    assert_same_categories(enc.categories_, sk.categories_)
    got = enc.transform(_chunked(t, rows))
    assert all(b.is_cuda and b.layout == torch.sparse_csr for b in got.blocks)
    got = got.compute()
    np.testing.assert_array_equal(got.indptr, want.indptr)
    np.testing.assert_array_equal(got.indices, want.indices)
    np.testing.assert_array_equal(got.data, want.data)
    if want.shape[1] * h.shape[0] <= 2e8:
        dense = OneHotEncoder(sparse=False, dtype=np.uint8).fit(_chunked(t, rows)).transform(_chunked(t, rows))
        assert dense.blocks[0].is_cuda and dense.blocks[0].dtype == torch.uint8
        np.testing.assert_array_equal(dense.compute(), want.toarray().astype(np.uint8))
    y = h[:, -1]
    le = LabelEncoder().fit(_chunked(t[:, -1], rows))
    assert_same_categories([le.classes_], [np.unique(y)])
    codes = le.transform(_chunked(t[:, -1], rows))
    assert codes.blocks[0].is_cuda and codes.chunks == _chunked(t[:, -1], rows).chunks
    want_codes = np.searchsorted(np.unique(y), y) if y.dtype.kind == "f" else sklearn.preprocessing.LabelEncoder() \
        .fit_transform(y)
    if y.dtype.kind == "f":
        want_codes[np.isnan(y)] = len(le.classes_) - 1
    np.testing.assert_array_equal(codes.compute(), want_codes)
    back = le.inverse_transform(codes)
    assert back.blocks[0].is_cuda
    np.testing.assert_array_equal(back.compute(), le.classes_[want_codes])
    assert torch.equal(torch.isnan(t.float()), torch.isnan(keep.float())) and torch.equal(
        torch.nan_to_num(t.float()), torch.nan_to_num(keep.float()))          # the device input is unchanged


def test_wide_integers_and_marker():
    from dask_ml_b200.preprocessing import LabelEncoder, OneHotEncoder

    big = np.array([2 ** 53, 2 ** 53 + 1, np.iinfo(np.int64).max, np.iinfo(np.int64).min, 0, 2 ** 53] * 1000,
                   dtype=np.int64)
    t = torch.as_tensor(big).cuda()
    le = LabelEncoder().fit(_chunked(t, 1000))
    np.testing.assert_array_equal(le.classes_, np.unique(big))
    np.testing.assert_array_equal(le.transform(t).compute(), sklearn.preprocessing.LabelEncoder().fit_transform(big))
    np.testing.assert_array_equal(le.inverse_transform(le.transform(t)).compute(), big)
    enc = OneHotEncoder(sparse=False).fit(_chunked(torch.stack([t, t.flip(0)], 1), 999))
    sk = sklearn.preprocessing.OneHotEncoder(sparse_output=False).fit(np.stack([big, big[::-1]], 1))
    assert_same_categories(enc.categories_, sk.categories_)


def test_growth_many_distinct():
    """5 * 10^5 distinct int64 values in one column: the table grows from its first 4096 slots."""
    from dask_ml_b200.preprocessing import LabelEncoder

    rng = np.random.RandomState(3)
    y = rng.permutation(500000).astype(np.int64) * 7919 - 10 ** 12
    le = LabelEncoder()
    codes = le.fit_transform(_chunked(torch.as_tensor(y).cuda(), 1 << 17)).compute()
    np.testing.assert_array_equal(le.classes_, np.unique(y))
    np.testing.assert_array_equal(codes, np.searchsorted(le.classes_, y))


def _table_entries(be, keys, counts, off, g, rows):
    """{(column, key): count} of the occupied slots of the tables (at most ``rows`` of them)."""
    e = be.zeros((rows, 4), torch.float64)
    be.mode_compact(keys, counts, off, g, e)
    e = e.cpu().numpy()
    return {(int(c), (int(hi) << 32) | int(lo)): int(n) for c, hi, lo, n in e[e[:, 3] > 0]}


@pytest.mark.parametrize("dt", ["f32", "f64", "bf16"])
def test_count_and_distinct_passes_share_keys(dt):
    """SimpleImputer's count pass (NaN missing) and the encoders' distinct pass put the same keys in the tables for
    the same columns of signed zeros, infinities, subnormals, NaN and repeats; the counts are torch.unique's, with
    -0.0 counted as +0.0."""
    from dask_ml_b200 import _keytables
    from dask_ml_b200.cluster import k_means as km
    from dask_ml_b200.preprocessing._encode import host_keys

    tdt = DTYPES[dt]
    tiny = float(torch.finfo(tdt).smallest_normal)
    pool = np.array([0.0, -0.0, 1.0, -1.0, 1.5, -2.25, np.inf, -np.inf, np.nan, tiny / 2, -tiny / 2, tiny / 4, tiny])
    rng = np.random.RandomState(7)
    n, g = 5000, 3
    idx = np.minimum(rng.geometric(0.25, (n, g)) - 1, len(pool) - 1)
    idx[: len(pool)] = np.arange(len(pool))[:, None]
    X = torch.as_tensor(pool[rng.permutation(idx)]).to(tdt).cuda()
    be = km._get_backend()
    keys, counts, off, total = _keytables.alloc(be, [_keytables.capacity(n, tdt)] * g)
    be.mode_count_chunk(X, True, float("nan"), keys, counts, off, total, first=True)
    counted = _table_entries(be, keys, counts, off, g, n * g)
    state = be.zeros((2, g), torch.int64)
    be.distinct_chunk(X, keys, counts, off, total, state, first=True)
    assert not (state[1].cpu().numpy() & 1).any()
    distinct = _table_entries(be, keys, counts, off, g, n * g)
    want = {}
    for j in range(g):
        col = X[:, j].double()
        u, c = torch.unique(col[~torch.isnan(col)], return_counts=True)
        for k, m in zip(host_keys(u.cpu().numpy(), tdt), c.cpu().numpy()):
            want[(j, int(k))] = want.get((j, int(k)), 0) + int(m)
    assert counted == want
    nan_key = int(host_keys(np.array([np.nan]), tdt)[0])
    assert {k for k in distinct if k[1] != nan_key} == set(want)
    assert {k for k in distinct if k[1] == nan_key} == {(j, nan_key) for j in range(g)}
    assert set(distinct.values()) == {1}


def test_unknown_after_multi_chunk_transform():
    from dask_ml_b200.preprocessing import LabelEncoder, OneHotEncoder

    t, h = _data("i64")
    enc = OneHotEncoder().fit(_chunked(t, 7000))
    bad = t.clone()
    bad[59000, 1] = 12345
    bad[3, 1] = -777
    with pytest.raises(ValueError, match=r"Found unknown categories \[np.int64\(-777\), np.int64\(12345\)\] in column 1"):
        enc.transform(_chunked(bad, 7000))
    le = LabelEncoder().fit(_chunked(t[:, 0], 7000))
    with pytest.raises(ValueError, match=r"previously unseen values \[9\]"):
        le.transform(_chunked(torch.where(t[:, 0] == 3, 9, t[:, 0]), 7000))


def test_outputs_feed_estimators():
    from dask_ml_b200.linear_model import LogisticRegression
    from dask_ml_b200.naive_bayes import GaussianNB
    from dask_ml_b200.preprocessing import LabelEncoder, OneHotEncoder

    rng = np.random.RandomState(5)
    n = 20000
    Xc = torch.as_tensor(rng.randint(0, 6, (n, 3))).cuda()
    y = (Xc[:, 0] >= 3).to(torch.int64)
    Xd = OneHotEncoder(sparse=False).fit_transform(_chunked(Xc, 5000))
    clf = LogisticRegression().fit(Xd, _chunked(y, 5000))
    assert (np.asarray(clf.predict(Xd).compute()).ravel() == y.cpu().numpy()).mean() > 0.99
    labels = torch.as_tensor(np.array([10, 20, 30])[rng.randint(0, 3, n)]).cuda()
    X = torch.as_tensor(rng.standard_normal((n, 4))).cuda() + (labels[:, None] / 10.0)
    nb = GaussianNB().fit(_chunked(X, 5000), LabelEncoder().fit_transform(_chunked(labels, 5000)))
    np.testing.assert_array_equal(nb.classes_, [0, 1, 2])
