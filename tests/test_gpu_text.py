"""HashingVectorizer on the device against scikit-learn 1.9, bit for bit: the reference's JUNK_FOOD_DOCS test, a matrix
of n_features, ngram_range, norm, binary, alternate_sign, lowercase and dtype, edge documents (empty, whitespace, one
letter, a token over 1 KB, one 10 MB document, a block of 10^6 short documents), mixed non-ASCII and bytes blocks,
ragged blocks, the token whose hash is -2^31, and the replay of the reference fixtures (tests/golden/ref_text.py)."""
import json
import os
import sys

import numpy as np
import pytest
import sklearn.feature_extraction.text
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from test_text_host import (JUNK_FOOD_DOCS, MIN_HASH_TOKEN, assert_same_csr, chunked, random_docs,  # noqa: E402
                            word_docs)

from dask_ml_b200 import ChunkedArray, _lib  # noqa: E402
from dask_ml_b200.feature_extraction import HashingVectorizer  # noqa: E402

SK = sklearn.feature_extraction.text.HashingVectorizer
GOLDEN = os.path.join(ROOT, "tests", "golden")


def _check(docs, chunks, **params):
    want = SK(**params).transform(docs)
    before = _lib.load().bkm_launch_count()
    got = HashingVectorizer(**params).transform(chunked(docs, chunks))
    assert all(b.is_cuda and b.layout == torch.sparse_csr for b in got.blocks)
    assert _lib.load().bkm_launch_count() > before
    assert_same_csr(got.compute(), want)
    return got


def test_junk_food_docs():
    _check(list(JUNK_FOOD_DOCS), 3)
    got = HashingVectorizer().fit_transform(chunked(list(JUNK_FOOD_DOCS), 3))
    np.testing.assert_array_equal(got.compute().toarray(), SK().fit_transform(JUNK_FOOD_DOCS).toarray())


CORPUS = word_docs(2000, 7) + random_docs(500, 8) + [MIN_HASH_TOKEN, MIN_HASH_TOKEN.upper() + " x " + MIN_HASH_TOKEN]
VARIANTS = [dict(), dict(norm="l1", dtype=np.float32), dict(norm=None, binary=True, lowercase=False),
            dict(alternate_sign=False, norm="l2", dtype=np.float32), dict(norm=None, alternate_sign=False)]


@pytest.mark.parametrize("ngram", [(1, 1), (1, 3), (2, 2)])
@pytest.mark.parametrize("n_features", [16, 1 << 20, 2 ** 31 - 1])
def test_matrix(n_features, ngram):
    for v in VARIANTS:
        _check(CORPUS, 700, n_features=n_features, ngram_range=ngram, **v)


def test_edge_documents():
    docs = ["", "   \n\t ", "a", "ab", "a b c", "__", "x" * 1500 + " y" * 3, "Z" * 4097, "9" * 2 + "," + "_" * 3]
    for params in (dict(), dict(ngram_range=(1, 3), norm=None), dict(ngram_range=(2, 2), binary=True)):
        _check(docs, 4, **params)
        _check(docs, len(docs), **params)


def test_ten_megabyte_document():
    rng = np.random.RandomState(3)
    words = np.array(["alpha", "Beta", "gamma_1", "de", "epsilonzeta", "x9"])
    doc = " ".join(rng.choice(words, 1_700_000))
    assert len(doc) > 10_000_000
    for params in (dict(), dict(ngram_range=(1, 2), norm="l1", dtype=np.float32), dict(n_features=16, norm=None)):
        _check([doc, "short one"], 2, **params)


def test_million_short_documents():
    rng = np.random.RandomState(4)
    vocab = np.array(["ab", "cd", "Ef", "gh1", "the", "of", "x", "and", "to", "in"])
    docs = [" ".join(rng.choice(vocab, k)) for k in rng.randint(0, 6, 1_000_000)]
    _check(docs, 1_000_000)
    _check(docs, 400_000, ngram_range=(1, 2), norm=None)


def test_mixed_non_ascii_and_bytes():
    docs = []
    for i, d in enumerate(word_docs(3000, 11)):
        docs.append(d.encode() if i % 3 == 0 else (d + " café" if i % 7 == 0 else d))
    docs += ["naïve".encode("utf-8"), "ünïcode only", b"", "plain"]
    for params in (dict(), dict(ngram_range=(1, 2), norm="l1", dtype=np.float32), dict(binary=True, norm=None)):
        _check(docs, 1000, **params)


def test_ragged_blocks():
    docs = word_docs(5000, 12)
    sizes = [1, 2000, 3, 1500, 1496]
    X = ChunkedArray.from_array(np.array(docs, dtype=object), (tuple(sizes),))
    got = HashingVectorizer(ngram_range=(1, 2)).transform(X)
    assert [b.shape[0] for b in got.blocks] == sizes
    assert_same_csr(got.compute(), SK(ngram_range=(1, 2)).transform(docs))


def test_reference_fixtures():
    """The unmodified reference's transform of chunked documents (tests/golden/ref_text.py), replayed on the device."""
    with open(os.path.join(GOLDEN, "REF_TEXT_MANIFEST.json")) as f:
        man = json.load(f)
    for case in man["cases"]:
        z = np.load(os.path.join(GOLDEN, case["file"]), allow_pickle=False)
        docs = [str(d) for d in z["docs"]]
        X = ChunkedArray.from_array(np.array(docs, dtype=object), (tuple(int(c) for c in z["chunks"]),))
        params = dict(case["params"])
        if "ngram_range" in params:
            params["ngram_range"] = tuple(params["ngram_range"])
        got = HashingVectorizer(**params).transform(X).compute()
        np.testing.assert_array_equal(got.indptr, z["indptr"])
        np.testing.assert_array_equal(got.indices, z["indices"])
        np.testing.assert_array_equal(got.data, z["data"])
