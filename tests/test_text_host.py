"""HashingVectorizer without a GPU: the estimator's host logic (routing of documents, the fallback configurations,
errors, parameters, pickling) on a CPU backend whose new passes are a Python restatement, against scikit-learn 1.9;
the restated tokeniser and MurmurHash3 against scikit-learn's on random ASCII corpora and on a token whose hash is
-2^31; and the argument checks of the new entry points, which need no device."""
import ctypes
import os
import pickle
import string
import sys

import numpy as np
import pytest
import scipy.sparse
import sklearn.feature_extraction.text
import torch
from sklearn.utils import murmurhash3_32

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle_backend import OracleBackend  # noqa: E402

from dask_ml_b200 import ChunkedArray  # noqa: E402
from dask_ml_b200.feature_extraction import HashingVectorizer  # noqa: E402

M32 = 0xFFFFFFFF
WORD = np.zeros(256, dtype=bool)
WORD[np.frombuffer((string.ascii_letters + string.digits + "_").encode(), dtype=np.uint8)] = True
JUNK_FOOD_DOCS = (
    "the pizza pizza beer copyright",
    "the pizza burger beer copyright",
    "the the pizza beer beer copyright",
    "the burger beer beer copyright",
    "the coke burger coke copyright",
    "the coke burger burger",
)


# ------------------------------------------------ restatement ------------------------------------------------
def _rotl(x, r):
    return ((x << r) | (x >> (32 - r))) & M32


def _scramble(k):
    return (_rotl((k * 0xCC9E2D51) & M32, 15) * 0x1B873593) & M32


def _fmix(h):
    h ^= h >> 16
    h = (h * 0x85EBCA6B) & M32
    h ^= h >> 13
    h = (h * 0xC2B2AE35) & M32
    return h ^ (h >> 16)


def murmur3(data):
    """MurmurHash3 x86_32, seed 0, as a signed int."""
    h, nb = 0, len(data) // 4
    for i in range(nb):
        h = (_rotl(h ^ _scramble(int.from_bytes(data[4 * i: 4 * i + 4], "little")), 13) * 5 + 0xE6546B64) & M32
    if len(data) & 3:
        h ^= _scramble(int.from_bytes(data[4 * nb:], "little"))
    h = _fmix(h ^ (len(data) & M32))
    return h - (1 << 32) if h >> 31 else h


def hash_key(h, nf, alternate_sign):
    col = (2147483647 - (nf - 1)) % nf if h == -(1 << 31) else abs(h) % nf
    return 2 * col + (1 if alternate_sign and h < 0 else 0)


def tokens(b, lowercase):
    """The tokens (bytes) of one ASCII document: maximal word runs of length >= 2."""
    w = WORD[np.frombuffer(b, dtype=np.uint8)] if b else np.zeros(0, dtype=bool)
    edges = np.flatnonzero(np.diff(np.concatenate([[0], w.astype(np.int8), [0]])))
    out = [b[s:e] for s, e in zip(edges[0::2], edges[1::2]) if e - s >= 2]
    return [t.lower() for t in out] if lowercase else out


def ngrams(toks, min_n, max_n):
    return [b" ".join(toks[i: i + n]) for n in range(min_n, max_n + 1) for i in range(len(toks) - n + 1)]


class TextOracleBackend(OracleBackend):
    """The CPU checker backend plus HashingVectorizer's passes in Python (the same algorithm, not the same code)."""

    def text_tokens_chunk(self, buf, doc_off, min_n, max_n, tok_start, tok_off, pair_off, totals):
        self.launches += 1
        b, off = buf.numpy(), doc_off.numpy()
        assert tok_start.numel() >= b.size // 3 + 1
        w = WORD[b]
        nxt = np.concatenate([w[1:], [False]])
        prev = np.concatenate([[False], w[:-1]])
        st = np.flatnonzero(w & nxt & ~prev)
        assert all(not WORD[b[o - 1]] for o in off[1:])        # every document ends in a separator
        tok_start[: st.size] = torch.from_numpy(st)
        to = np.searchsorted(st, off)
        tok_off.copy_(torch.from_numpy(to))
        T = np.diff(to)
        counts = sum(np.maximum(0, T - n + 1) for n in range(min_n, max_n + 1))
        pair_off.copy_(torch.from_numpy(np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)))
        totals[0], totals[1] = st.size, int(pair_off[-1])

    def _rows(self, keys, pair_off, binary, norm, dtype):
        """Per document: (columns, values in dtype, divisor)."""
        npdt = np.float32 if dtype == torch.float32 else np.float64
        k = keys.numpy().view(np.uint32)
        po = pair_off.numpy()
        out = []
        for d in range(po.size - 1):
            kd = k[po[d]: po[d + 1]].astype(np.int64)
            cols = np.unique(kd >> 1)
            pos = np.array([np.sum(kd == 2 * c) for c in cols], dtype=np.int64)
            neg = np.array([np.sum(kd == 2 * c + 1) for c in cols], dtype=np.int64)
            v = (np.ones_like(cols) if binary else pos - neg).astype(npdt)
            s = 0.0
            for x in v:
                s += abs(float(x)) if norm == "l1" else (float(npdt(x * x)) if norm == "l2" else 0.0)
            s = float(np.sqrt(s)) if norm == "l2" else s
            out.append((cols, v, s))
        return out

    def text_hash_chunk(self, buf, tok_start, tok_off, pair_off, n_tokens, n_pairs, min_n, max_n, lowercase,
                        n_features, alternate_sign, binary, norm, dtype, keys, indptr, scale, totals):
        self.launches += 1
        b = buf.numpy().tobytes()
        st, to, po = tok_start.numpy(), tok_off.numpy(), pair_off.numpy()
        kk = keys.numpy().view(np.uint32)
        for d in range(to.size - 1):
            toks = []
            for s in st[to[d]: to[d + 1]]:
                e = s
                while e < len(b) and WORD[b[e]]:
                    e += 1
                toks.append(b[s:e].lower() if lowercase else b[s:e])
            ks = sorted(hash_key(murmur3(g), n_features, alternate_sign) for g in ngrams(toks, min_n, max_n))
            assert len(ks) == po[d + 1] - po[d]
            kk[po[d]: po[d + 1]] = np.asarray(ks, dtype=np.uint32)
        rows = self._rows(keys, pair_off, binary, norm, dtype)
        nnz = np.array([r[0].size for r in rows], dtype=np.int64)
        indptr.copy_(torch.from_numpy(np.concatenate([[0], np.cumsum(nnz)]).astype(np.int64)))
        scale[: len(rows)] = torch.tensor([r[2] for r in rows], dtype=torch.float64)
        totals[2] = int(indptr[-1])

    def text_write_chunk(self, keys, pair_off, indptr, scale, binary, indices, data):
        self.launches += 1
        npdt = np.float32 if data.dtype == torch.float32 else np.float64
        ip = indptr.numpy()
        for d, (cols, v, _) in enumerate(self._rows(keys, pair_off, binary, None, data.dtype)):
            s = float(scale[d])
            if s != 0.0:
                v = (v.astype(np.float64) / s).astype(npdt)
            indices[ip[d]: ip[d + 1]] = torch.from_numpy(cols)
            data[ip[d]: ip[d + 1]] = torch.from_numpy(v)


@pytest.fixture
def cpu_backend(monkeypatch):
    from dask_ml_b200.cluster import k_means as km

    monkeypatch.setattr(km, "_BACKEND_FACTORY", TextOracleBackend)


# ------------------------------------------------ corpora ------------------------------------------------
def random_docs(n, seed, alphabet=string.printable, max_len=60):
    rng = np.random.RandomState(seed)
    chars = np.array(list(alphabet))
    return ["".join(rng.choice(chars, rng.randint(0, max_len))) for _ in range(n)]


def word_docs(n, seed, vocab=200, max_words=30):
    """Documents of words of every length mod 4, mixed case, with assorted separators."""
    rng = np.random.RandomState(seed)
    letters = np.array(list(string.ascii_letters + string.digits + "_"))
    words = ["".join(rng.choice(letters, L)) for L in rng.randint(1, 14, vocab)]
    seps = [" ", "  ", ", ", ".\n", "\t", "-", "'", "!?"]
    return ["".join(words[rng.randint(vocab)] + seps[rng.randint(len(seps))] for _ in range(rng.randint(0, max_words)))
            for _ in range(n)]


def _find_min_hash_token():
    """An 8-byte lowercase word token whose MurmurHash3 is -2^31: fix the first 4-byte block and invert the last
    block's mixing and the finaliser."""
    inv = lambda a: pow(a, -1, 1 << 32)                     # noqa: E731
    rotr = lambda x, r: _rotl(x, 32 - r)                    # noqa: E731

    def unfmix(h):
        h ^= h >> 16
        h = (h * inv(0xC2B2AE35)) & M32
        h ^= (h >> 13) ^ (h >> 26)
        h = (h * inv(0x85EBCA6B)) & M32
        return h ^ (h >> 16)

    h2 = unfmix(0x80000000) ^ 8
    alphabet = (string.ascii_lowercase + string.digits + "_").encode()
    ok = set(alphabet)
    for a in alphabet:
        for b in alphabet:
            for c in alphabet:
                for d in alphabet:
                    first = bytes([a, b, c, d])
                    h1 = (_rotl(_scramble(int.from_bytes(first, "little")), 13) * 5 + 0xE6546B64) & M32
                    s = rotr(((h2 - 0xE6546B64) * inv(5)) & M32, 13) ^ h1
                    k = (rotr((s * inv(0x1B873593)) & M32, 15) * inv(0xCC9E2D51)) & M32
                    last = k.to_bytes(4, "little")
                    if all(x in ok for x in last):
                        return (first + last).decode()
    raise AssertionError("no token found")


MIN_HASH_TOKEN = _find_min_hash_token()


def assert_same_csr(got, want):
    got, want = scipy.sparse.csr_matrix(got), scipy.sparse.csr_matrix(want)
    assert got.shape == want.shape
    np.testing.assert_array_equal(got.indptr, want.indptr)
    np.testing.assert_array_equal(got.indices, want.indices)
    assert got.data.dtype == want.data.dtype
    np.testing.assert_array_equal(got.data.view(np.uint8), want.data.view(np.uint8))


def chunked(docs, chunks):
    return ChunkedArray.from_array(np.array(docs, dtype=object), chunks)


# ------------------------------------------------ tests ------------------------------------------------
def test_murmur_restatement():
    rng = np.random.RandomState(0)
    for L in range(0, 40):
        for _ in range(5):
            b = bytes(rng.randint(0, 128, L).astype(np.uint8))
            assert murmur3(b) == murmurhash3_32(b, seed=0), b


def test_min_hash_token():
    t = MIN_HASH_TOKEN
    assert len(t) == 8 and t == t.lower() and all(WORD[ord(c)] for c in t)
    assert murmur3(t.encode()) == -(1 << 31) == murmurhash3_32(t, seed=0)
    for nf in (16, 1 << 20, 2 ** 31 - 1, 7):
        X = sklearn.feature_extraction.text.HashingVectorizer(n_features=nf, norm=None).transform([t])
        assert X.indices.tolist() == [hash_key(-(1 << 31), nf, True) >> 1]
        assert X.data.tolist() == [-1.0]


@pytest.mark.parametrize("seed", range(3))
def test_tokeniser_restatement(seed):
    """Tokens, lowercasing and n-grams against scikit-learn's analyzer: random printable text, words of every length mod
    4, and all 128 ASCII code points."""
    docs = random_docs(300, seed) + word_docs(300, seed) + ["".join(map(chr, range(128))), "a", " ", ""]
    for lowercase in (True, False):
        for ngram in ((1, 1), (1, 3), (2, 2)):
            an = sklearn.feature_extraction.text.HashingVectorizer(lowercase=lowercase, ngram_range=ngram)
            an = an.build_analyzer()
            for d in docs:
                want = [t.encode() for t in an(d)]
                assert ngrams(tokens(d.encode(), lowercase), *ngram) == want, d


PARAMS = [dict(), dict(ngram_range=(1, 3)), dict(ngram_range=(2, 2), norm="l1"), dict(n_features=16, norm=None),
          dict(n_features=16, alternate_sign=False, binary=True), dict(norm="l1", dtype=np.float32),
          dict(n_features=2 ** 31 - 1, lowercase=False, dtype=np.float32), dict(n_features=2, norm=None),
          dict(strip_accents="unicode", ngram_range=(1, 2), binary=True, norm="l2")]


@pytest.mark.parametrize("params", PARAMS, ids=[str(p) for p in PARAMS])
def test_device_path_matches_sklearn(cpu_backend, params):
    docs = list(JUNK_FOOD_DOCS) + word_docs(120, 1) + random_docs(60, 2) + ["", "   ", "x", MIN_HASH_TOKEN * 3,
                                                                          MIN_HASH_TOKEN + " " + MIN_HASH_TOKEN]
    want = sklearn.feature_extraction.text.HashingVectorizer(**params).transform(docs)
    got = HashingVectorizer(**params).transform(chunked(docs, 50))
    assert isinstance(got, ChunkedArray) and len(got.blocks) == 4
    b = got.blocks[0]
    assert b.layout == torch.sparse_csr and b.shape == (50, want.shape[1])
    assert b.crow_indices().dtype == torch.int64 and b.col_indices().dtype == torch.int64
    assert_same_csr(got.compute(), want)


def test_explicit_zeros_kept(cpu_backend):
    docs = list(JUNK_FOOD_DOCS)
    for params in (dict(norm=None), dict(norm="l2"), dict(binary=True, norm=None)):
        want = sklearn.feature_extraction.text.HashingVectorizer(n_features=2, **params).transform(docs)
        assert want.indptr[-1] == 9
        got = HashingVectorizer(n_features=2, **params).transform(chunked(docs, 4)).compute()
        assert_same_csr(got, want)
    assert want.data[-1] == 1.0 and got.data[-1] == 1.0                 # binary sets the stored zero to 1


def test_routing(cpu_backend):
    """Non-ASCII text and non-ASCII bytes go to scikit-learn, ASCII bytes to the device; rows stay in order."""
    docs = ["café au lait", b"plain bytes doc", "ascii text here", "naïve words", "éè".encode(),
            b"more bytes", "end doc", "café au lait"]
    for chunks in (3, 8):
        for params in (dict(), dict(ngram_range=(1, 2), norm="l1", dtype=np.float32)):
            want = sklearn.feature_extraction.text.HashingVectorizer(**params).transform(docs)
            got = HashingVectorizer(**params).transform(chunked(docs, chunks))
            assert_same_csr(got.compute(), want)


def test_all_host_documents(cpu_backend):
    docs = ["über alles", "ça va"]
    want = sklearn.feature_extraction.text.HashingVectorizer().transform(docs)
    assert_same_csr(HashingVectorizer().transform(chunked(docs, 2)).compute(), want)


def test_nan_raises_sklearn_error(cpu_backend):
    docs = ["fine doc", np.nan, "other doc"]
    with pytest.raises(ValueError, match="np.nan is an invalid document"):
        sklearn.feature_extraction.text.HashingVectorizer().transform(docs)
    with pytest.raises(ValueError, match="np.nan is an invalid document"):
        HashingVectorizer().transform(chunked(docs, 2))


def test_empty_block_raises(cpu_backend):
    """A block of no documents raises what scikit-learn raises for an empty sequence."""
    with pytest.raises(Exception) as want:
        sklearn.feature_extraction.text.HashingVectorizer().transform([])
    X = ChunkedArray([np.array(["some text"], dtype=object), np.array([], dtype=object)])
    with pytest.raises(want.type):
        HashingVectorizer().transform(X)


FALLBACK = [dict(analyzer="char", ngram_range=(2, 3)), dict(analyzer="char_wb"), dict(stop_words="english"),
            dict(token_pattern=r"(?u)\b\w+\b"), dict(tokenizer=str.split, token_pattern=None),
            dict(preprocessor=str.upper), dict(norm="max"), dict(dtype=np.int64, norm=None), dict(ngram_range=(0, 2)),
            dict(encoding="utf-16")]


@pytest.mark.parametrize("params", FALLBACK, ids=[str(p) for p in FALLBACK])
def test_fallback_configurations(cpu_backend, params):
    from dask_ml_b200.feature_extraction import text

    est = HashingVectorizer(**params)
    assert text.device_config(est) is None
    docs = list(JUNK_FOOD_DOCS) + ["Mixed CASE words, and the stop words"]
    want = sklearn.feature_extraction.text.HashingVectorizer(**params).transform(docs)
    got = est.transform(chunked(docs, 4))
    assert all(b.layout == torch.sparse_csr for b in got.blocks)
    assert_same_csr(got.compute(), want)


def test_device_config_accepts():
    from dask_ml_b200.feature_extraction import text

    for params in PARAMS + [dict(encoding="latin-1"), dict(encoding="ascii"), dict(strip_accents="ascii")]:
        assert text.device_config(HashingVectorizer(**params)) is not None, params


def test_bad_ngram_range_raises_sklearn_error(cpu_backend):
    with pytest.raises(ValueError, match="Invalid value for ngram_range"):
        HashingVectorizer(ngram_range=(3, 1)).transform(chunked(list(JUNK_FOOD_DOCS), 3))


def test_two_d_and_dataframe_raise():
    import pandas as pd

    msg = "1-dimensional array"
    with pytest.raises(ValueError, match=msg):
        HashingVectorizer().transform(ChunkedArray([np.array([["a b"], ["c d"]], dtype=object)]))
    with pytest.raises(ValueError, match=msg):
        HashingVectorizer().transform(pd.DataFrame({"text": list(JUNK_FOOD_DOCS)}))


def test_non_chunked_input_is_sklearn():
    import pandas as pd

    for X in (list(JUNK_FOOD_DOCS), np.array(JUNK_FOOD_DOCS, dtype=object), pd.Series(JUNK_FOOD_DOCS)):
        want = sklearn.feature_extraction.text.HashingVectorizer().fit_transform(X)
        got = HashingVectorizer().fit_transform(X)
        assert type(got) is type(want)
        assert_same_csr(got, want)


def test_params_and_pickle(cpu_backend):
    a = sklearn.feature_extraction.text.HashingVectorizer(n_features=64, ngram_range=(1, 2), binary=True)
    b = HashingVectorizer(n_features=64, ngram_range=(1, 2), binary=True)
    assert a.get_params() == b.get_params()
    c = pickle.loads(pickle.dumps(b))
    assert type(c) is HashingVectorizer and c.get_params() == b.get_params()
    assert_same_csr(c.fit_transform(chunked(list(JUNK_FOOD_DOCS), 2)).compute(), a.fit_transform(JUNK_FOOD_DOCS))


def test_pack_and_batches():
    from dask_ml_b200.feature_extraction import text

    buf, off = text.pack(["ab", "", "cde"])
    assert buf.tobytes() == b"ab\n\ncde\n" and off.tolist() == [0, 3, 4, 8]
    off = np.arange(0, 10 ** 10, 10 ** 9, dtype=np.int64)
    bt = text.batches(off, 3)
    assert bt[0][0] == 0 and bt[-1][1] == off.size - 1
    assert all(off[e] - off[s] <= 3 * ((2 ** 31 - 1) // 3 - 1) or e == s + 1 for s, e in bt)


def test_abi_argument_errors():
    """The new entry points reject bad arguments before they touch a device."""
    from dask_ml_b200 import _lib

    lib = _lib.load()
    p = ctypes.c_void_p(16)
    nb = ctypes.c_size_t(0)
    assert lib.bkm_text_workspace_bytes(-1, 4, 0, ctypes.byref(nb)) == -1
    assert lib.bkm_text_workspace_bytes(100, 4, 0, None) == -1
    assert lib.bkm_text_workspace_bytes(100, 4, 2 ** 31, ctypes.byref(nb)) == -3
    # buf, n_bytes, doc_off, n_docs, min_n, max_n, tok_start, tok_cap, tok_off, pair_off, totals, ws, ws_bytes, stream
    args = [p, 90, p, 4, 1, 2, p, 31, p, p, p, p, 1 << 30, None]
    for i, bad in ((1, -1), (3, -1), (4, 0), (5, 0), (7, 30), (2, None), (10, None), (11, None), (6, None)):
        a = list(args)
        a[i] = bad
        assert lib.bkm_text_tokens_chunk(*a) == -1, i
    hargs = [p, 90, p, p, p, 4, 10, 20, 1, 2, 1, 1024, 1, 0, 2, 0, p, p, p, p, p, 1 << 30, None]
    for i, bad in ((11, 0), (11, 2 ** 31), (14, 3), (8, 0), (16, None), (17, None), (20, None)):
        a = list(hargs)
        a[i] = bad
        assert lib.bkm_text_hash_chunk(*a) == -1, i
    a = list(hargs)
    a[15] = 2
    assert lib.bkm_text_hash_chunk(*a) == -2
    a = list(hargs)
    a[7] = 2 ** 31
    assert lib.bkm_text_hash_chunk(*a) == -3
    wargs = [p, p, p, p, 4, 0, p, p, 0, None]
    assert lib.bkm_text_write_chunk(*(wargs[:8] + [2] + wargs[9:])) == -2
    a = list(wargs)
    a[3] = None
    assert lib.bkm_text_write_chunk(*a) == -1
    a = list(wargs)
    a[4] = 0
    assert lib.bkm_text_write_chunk(*a) == 0


def test_reference_fixtures(cpu_backend):
    """The unmodified reference's transform of chunked documents (tests/golden/ref_text.py), replayed."""
    import json

    golden = os.path.join(ROOT, "tests", "golden")
    with open(os.path.join(golden, "REF_TEXT_MANIFEST.json")) as f:
        man = json.load(f)
    for case in man["cases"]:
        z = np.load(os.path.join(golden, case["file"]), allow_pickle=False)
        X = ChunkedArray.from_array(np.array([str(d) for d in z["docs"]], dtype=object),
                                    (tuple(int(c) for c in z["chunks"]),))
        params = dict(case["params"])
        if "ngram_range" in params:
            params["ngram_range"] = tuple(params["ngram_range"])
        got = HashingVectorizer(**params).transform(X)
        assert len(got.blocks) == case["blocks"]
        got = got.compute()
        np.testing.assert_array_equal(got.indptr, z["indptr"])
        np.testing.assert_array_equal(got.indices, z["indices"])
        np.testing.assert_array_equal(got.data, z["data"])
    with pytest.raises(ValueError) as e:
        HashingVectorizer().transform(ChunkedArray([np.array([["a b"], ["c d"]], dtype=object)]))
    assert str(e.value) == man["error_2d"]
