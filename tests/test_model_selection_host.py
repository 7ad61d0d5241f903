"""ShuffleSplit / train_test_split on host blocks: the reference's seeds, sizes, chunks and errors (fixtures written by
tests/golden/ref_model_selection.py from the unmodified reference), and the properties of the split permutation that
replace numpy's shuffle (DESIGN.md A26).  No GPU."""
import json
import logging
import os

import numpy as np
import pytest
import torch
from scipy import stats

from dask_ml_b200 import ChunkedArray
from dask_ml_b200.model_selection import ShuffleSplit, train_test_split
from dask_ml_b200.model_selection import _split as sp
from dask_ml_b200.model_selection._split import permutation_indices

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
with open(os.path.join(GOLDEN, "REF_MODEL_SELECTION_MANIFEST.json")) as f:
    MANIFEST = json.load(f)


def _rs(spec):
    return np.random.RandomState(spec["RandomState"]) if isinstance(spec, dict) else spec


def _xy(chunks, d):
    n = sum(chunks)
    X = np.arange(n * d, dtype=np.float64).reshape(n, d)
    y = np.arange(n, dtype=np.int64)
    return ChunkedArray.from_array(X, (tuple(chunks),)), ChunkedArray.from_array(y, (tuple(chunks),))


# ---- S1 - S3: the reference's seeds, sizes and chunks -----------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(MANIFEST["cases"]))
def test_reference_seeds_sizes_and_chunks(name, monkeypatch):
    case, ref = MANIFEST["cases"][name], np.load(os.path.join(GOLDEN, name + ".npz"))
    X, y = _xy(case["chunks"], case["d"])
    seen = []
    real = sp.permutation_indices
    monkeypatch.setattr(sp, "permutation_indices",
                        lambda seed, c, pos: seen.append((int(seed), int(c), len(pos))) or real(seed, c, pos))
    kw = {k: case[k] for k in ("test_size", "train_size") if k in case}
    out = train_test_split(X, y, random_state=_rs(case["random_state"]), **kw)
    assert len(out) == case["n_outputs"]
    np.testing.assert_array_equal([s for s, _, _ in seen], ref["seeds"].astype(np.int64))
    np.testing.assert_array_equal([c for _, c, _ in seen], ref["block_rows"])
    np.testing.assert_array_equal([m for _, _, m in seen], ref["n_train"] + ref["n_test"])
    Xtr, Xte, ytr, yte = out
    assert Xtr.chunks[0] == tuple(ref["train_chunks"]) and Xte.chunks[0] == tuple(ref["test_chunks"])
    assert ytr.chunks[0] == tuple(ref["y_train_chunks"]) and yte.chunks[0] == tuple(ref["y_test_chunks"])
    assert list(Xtr.shape) == case["x_train_shape"] and list(yte.shape) == case["y_test_shape"]
    # S2 / S3: rows stay in their block, train and test are disjoint, X and y stay aligned
    bounds = np.cumsum([0] + case["chunks"])
    for i in range(len(case["chunks"])):
        tr, te = ytr.blocks[i], yte.blocks[i]
        both = np.concatenate([tr, te])
        assert len(np.unique(both)) == len(both)
        assert both.min() >= bounds[i] and both.max() < bounds[i + 1]
        np.testing.assert_array_equal(Xtr.blocks[i][:, 0], tr * case["d"])
        np.testing.assert_array_equal(Xte.blocks[i][:, 0], te * case["d"])
        perm = permutation_indices(ref["seeds"][i], case["chunks"][i], np.arange(len(both))) + bounds[i]
        np.testing.assert_array_equal(te, perm[:len(te)])
        np.testing.assert_array_equal(tr, perm[len(te):])


def test_shufflesplit_draws_seeds_again_at_every_split():
    sc, ref = MANIFEST["shufflesplit"], np.load(os.path.join(GOLDEN, "ref_split_shufflesplit.npz"))
    X, _ = _xy(sc["chunks"], 2)
    ss = ShuffleSplit(n_splits=sc["n_splits"], test_size=sc["test_size"], random_state=sc["random_state"])
    assert ss.get_n_splits() == sc["n_splits_reported"]
    splits = list(ss.split(X))
    assert len(splits) == sc["n_splits"]
    bounds = np.cumsum([0] + sc["chunks"])
    for s, (tr, te) in enumerate(splits):
        assert [list(tr.chunks[0]), list(te.chunks[0])] == ref["idx_chunks"][s].tolist()
        assert tr.dtype == np.int64 and te.dtype == np.int64
        for i, c in enumerate(sc["chunks"]):
            perm = permutation_indices(ref["seeds"][s, i], c, np.arange(c)) + bounds[i]
            np.testing.assert_array_equal(te.blocks[i], perm[:ref["n_test"][s, i]])
            np.testing.assert_array_equal(tr.blocks[i], perm[ref["n_test"][s, i]:][:ref["n_train"][s, i]])
    # an integer random_state yields identical splits, as in the reference
    np.testing.assert_array_equal(splits[0][0].compute(), splits[1][0].compute())
    assert (ref["seeds"][0] == ref["seeds"][1]).all()


# ---- S4: errors ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(MANIFEST["errors"]))
def test_reference_errors(name):
    spec = MANIFEST["errors"][name]
    chunks = spec.get("chunks", [10, 10])
    X, _ = _xy(chunks, 2)
    exc = {"ValueError": ValueError, "TypeError": TypeError, "NotImplementedError": NotImplementedError}[spec["type"]]
    with pytest.raises(exc) as info:
        if spec["fn"] == "ShuffleSplit":
            ShuffleSplit(**spec["kw"])
        elif spec["fn"] == "split":
            ss = ShuffleSplit(n_splits=1)
            for k, v in spec["kw"].items():
                setattr(ss, k, v)
            next(ss.split(X))
        else:
            train_test_split(X, **spec["kw"])
    assert str(info.value) == spec["message"]


def test_default_test_size_and_mismatched_chunks():
    X, y = _xy([50, 50], 3)
    out = train_test_split(X, y, random_state=0)
    assert out[1].chunks[0] == (5, 5) and out[0].chunks[0] == (45, 45)
    y2 = ChunkedArray.from_array(np.arange(100), 40)
    with pytest.raises(ValueError, match="Mismatched chunks"):
        train_test_split(X, y2, random_state=0)


# ---- S5: plain arrays go to scikit-learn -----------------------------------------------------------------------------------
def test_plain_numpy_falls_back_to_sklearn(caplog):
    import sklearn.model_selection as ms

    X, y = np.arange(40.0).reshape(20, 2), np.arange(20)
    with caplog.at_level(logging.WARNING, logger="dask_ml_b200.model_selection._split"):
        got = train_test_split(X, y, test_size=0.25, random_state=3)
    assert "Falling back to scikit-learn" in caplog.text
    want = ms.train_test_split(X, y, test_size=0.25, random_state=3)
    for g, w in zip(got, want):
        np.testing.assert_array_equal(g, w)


# ---- the permutation ---------------------------------------------------------------------------------------------------------
def test_permutation_is_a_bijection_for_every_small_block_size():
    for c in range(1, 2051):
        out = permutation_indices(c * 7919 + 1, c, np.arange(c))
        assert np.array_equal(np.sort(out), np.arange(c)), c


@pytest.mark.parametrize("c", [2 ** 20 - 1, 2 ** 20 + 1, 10 ** 6 + 3, 4 ** 10, 4 ** 10 + 1])
def test_permutation_is_a_bijection_for_large_blocks(c):
    out = permutation_indices(123456789, c, np.arange(c))
    assert out.dtype == np.int64
    assert np.array_equal(np.sort(out), np.arange(c))
    assert (out != np.arange(c)).mean() > 0.99


def test_permutation_windows_and_range_checks():
    full = permutation_indices(5, 1000, np.arange(1000))
    np.testing.assert_array_equal(permutation_indices(5, 1000, np.arange(300, 420)), full[300:420])
    with pytest.raises(ValueError):
        permutation_indices(5, 10, [10])
    with pytest.raises(ValueError):
        permutation_indices(5, 0, [])


# The tests that fix the round count (BKM_SPLIT_ROUNDS = SPLIT_ROUNDS): over a fixed list of 20 000 seeds, drawn the way
# ShuffleSplit draws them, the image of a position must be uniform over the block and the images of two positions
# uniform over the ordered pairs.  Every chi-square test is held at the 1e-4 level: 19 tests, so a correct permutation
# fails this file with probability below 2e-3, and the seed list is fixed, so it fails always or never.
SEEDS = np.random.RandomState(12345).randint(0, 2 ** 32 - 1, size=20000, dtype="u8")
ALPHA = 1e-4


@pytest.mark.parametrize("c", [3, 5, 64, 1000])
def test_position_uniformity(c):
    for i in sorted({0, 1, c // 2, c - 1}):
        counts = np.bincount(permutation_indices(SEEDS, c, i), minlength=c)
        assert stats.chisquare(counts).pvalue > ALPHA, (c, i)


def test_pair_independence():
    a, b = permutation_indices(SEEDS, 8, 0), permutation_indices(SEEDS, 8, 1)
    counts = np.zeros((8, 8))
    np.add.at(counts, (a, b), 1)
    assert np.trace(counts) == 0
    assert stats.chisquare(counts[~np.eye(8, dtype=bool)]).pvalue > ALPHA


def test_fewer_rounds_fail_the_uniformity_tests():
    a, b = permutation_indices(SEEDS, 8, 0, rounds=6), permutation_indices(SEEDS, 8, 1, rounds=6)
    pair = np.zeros((8, 8))
    np.add.at(pair, (a, b), 1)
    assert stats.chisquare(pair[~np.eye(8, dtype=bool)]).pvalue < ALPHA


def test_sequential_seeds_are_as_good_as_random_ones():
    seq = np.arange(20000, dtype=np.uint64)
    for c in (5, 64, 1000):
        assert stats.chisquare(np.bincount(permutation_indices(seq, c, 0), minlength=c)).pvalue > ALPHA


# ---- end to end on host blocks ---------------------------------------------------------------------------------------------------
def test_same_random_state_same_split_and_different_differs():
    X, y = _xy([300, 300, 77], 3)
    a = train_test_split(X, y, test_size=0.3, random_state=4)
    b = train_test_split(X, y, test_size=0.3, random_state=4)
    c = train_test_split(X, y, test_size=0.3, random_state=5)
    for u, v in zip(a, b):
        np.testing.assert_array_equal(u.compute(), v.compute())
    assert not np.array_equal(a[3].compute(), c[3].compute())


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32, torch.int32, torch.bool])
def test_torch_host_blocks_of_every_dtype_keep_their_dtype(dtype):
    g = torch.Generator().manual_seed(0)
    t = (torch.randn(90, 5, generator=g) * 4).to(dtype)
    X = ChunkedArray([t[:50], t[50:]])
    y = ChunkedArray([np.arange(50), np.arange(50, 90)])
    Xtr, Xte, ytr, yte = train_test_split(X, y, test_size=0.2, random_state=1)
    assert all(b.dtype == dtype for b in Xtr.blocks + Xte.blocks)
    for xb, yb in zip(Xtr.blocks + Xte.blocks, ytr.blocks + yte.blocks):
        assert torch.equal(xb, t[torch.as_tensor(yb)])


def test_one_torch_tensor_is_one_block_and_1d_arrays_split():
    t = torch.arange(60, dtype=torch.float64)
    w = np.linspace(0, 1, 60)
    ttr, tte, wtr, wte = train_test_split(t, w, test_size=0.25, random_state=2)
    assert tte.shape == (15,) and ttr.shape == (45,)
    np.testing.assert_array_equal(wte.compute(), w[tte.compute().astype(int)])
    np.testing.assert_array_equal(np.sort(np.concatenate([ttr.compute(), tte.compute()])), np.arange(60.0))


def test_blockwise_slice_checks_foreign_indices():
    X, _ = _xy([10, 10], 2)
    good = ChunkedArray([np.array([3, 1]), np.array([12])])
    np.testing.assert_array_equal(sp._blockwise_slice(X, good).compute()[:, 0], [6.0, 2.0, 24.0])
    with pytest.raises(IndexError):
        sp._blockwise_slice(X, ChunkedArray([np.array([3, 10]), np.array([12])]))
