"""HashingVectorizer with the dask_ml.feature_extraction.text API, executed by the H100 engine.

Mirrors dask_ml/feature_extraction/text.py (reference @ 0310a90): scikit-learn's constructor, parameters and checks;
only ``transform`` is overridden.  Input that is not chunked goes to scikit-learn unchanged.  A 1-D ChunkedArray or
dask array of documents gives a ChunkedArray of device ``torch.sparse_csr_tensor`` blocks, (rows, n_features), whose
``.compute()`` equals scikit-learn's CSR for the concatenated documents bit for bit (DESIGN.md A31).

A block runs on the device (csrc/bkm_text.cu) when the configuration is one the passes restate exactly (``device_config``):
the word analyzer with the default token pattern and no tokenizer, preprocessor or stop words, ``input='content'``, a
float32 / float64 ``dtype`` and an encoding that maps ASCII bytes to themselves.  In such a block the ASCII ``str`` and
``bytes`` documents are tokenised, hashed and summed on the device; every other document (non-ASCII text, NaN, None,
numbers) goes through scikit-learn, which raises its own errors for them, and its rows are spliced in document order.
Other configurations run scikit-learn per block and upload its result as the same kind of block.
"""
import codecs
import numbers

import numpy as np
import sklearn.feature_extraction.text
import torch

from ..chunked import ChunkedArray, as_chunked, is_dask_array, is_dask_dataframe
from ..cluster import k_means as _km

TOKEN_PATTERN = r"(?u)\b\w\w+\b"
_ASCII_CODECS = ("utf-8", "ascii", "iso8859-1")
_DTYPES = {np.dtype("float32"): torch.float32, np.dtype("float64"): torch.float64}
_INT32_MAX = 2 ** 31 - 1
_MSG = "'X' should be a 1-dimensional array with length 'num_samples'."


def device_config(est):
    """The parameters of the device passes for ``est``'s configuration, or None when blocks run on scikit-learn."""
    if (est.analyzer != "word" or est.tokenizer is not None or est.preprocessor is not None
            or est.stop_words is not None or est.input != "content" or est.token_pattern != TOKEN_PATTERN):
        return None
    if est.strip_accents not in (None, "ascii", "unicode"):      # both leave ASCII text unchanged
        return None
    try:
        dtype = _DTYPES.get(np.dtype(est.dtype))
        ascii_codec = codecs.lookup(est.encoding).name in _ASCII_CODECS
    except (TypeError, LookupError):
        return None
    nf = est.n_features
    if dtype is None or not ascii_codec or est.norm not in (None, "l1", "l2"):
        return None
    if not isinstance(nf, numbers.Integral) or isinstance(nf, bool) or not 1 <= nf <= _INT32_MAX:
        return None
    try:
        min_n, max_n = est.ngram_range
    except (TypeError, ValueError):
        return None
    if not all(isinstance(v, numbers.Integral) for v in (min_n, max_n)) or not 1 <= min_n <= max_n:
        return None
    return dict(min_n=int(min_n), max_n=int(max_n), lowercase=bool(est.lowercase), n_features=int(nf),
                alternate_sign=bool(est.alternate_sign), binary=bool(est.binary), norm=est.norm, dtype=dtype)


def route(docs):
    """(device documents as one str each, their positions (None: all, in order), the positions of the other
    documents, and the device documents joined by '\\n' when they are all the documents)."""
    try:
        joined = "\n".join(docs)
        if joined.isascii():
            return docs, None, [], joined
    except TypeError:
        pass
    dev, pos, host = [], [], []
    for i, d in enumerate(docs):
        if isinstance(d, str) and d.isascii():
            dev.append(d)
            pos.append(i)
        elif isinstance(d, bytes) and d.isascii():
            dev.append(d.decode("ascii"))
            pos.append(i)
        else:
            host.append(i)
    return dev, pos, host, None


def pack(docs, joined=None):
    """The documents as one uint8 buffer, each followed by '\\n', and their int64 offsets (n + 1,)."""
    joined = "\n".join(docs) if joined is None else joined
    buf = np.frombuffer(bytearray(joined + "\n", "ascii"), dtype=np.uint8)
    off = np.zeros(len(docs) + 1, dtype=np.int64)
    np.cumsum(np.fromiter(map(len, docs), dtype=np.int64, count=len(docs)) + 1, out=off[1:])
    return buf, off


def batches(off, k):
    """[start, end) document ranges whose n-grams (at most k per token, a token per 3 bytes) fit the int32 counts of
    the sort."""
    limit = 3 * (_INT32_MAX // k - 1)
    n, out, s = len(off) - 1, [], 0
    while s < n:
        e = int(np.searchsorted(off, off[s] + limit, side="right")) - 1
        e = min(n, max(e, s + 1))
        out.append((s, e))
        s = e
    return out


def device_rows(be, buf, off, cfg):
    """The CSR (indptr, indices, data) of the documents packed in ``buf`` / ``off`` (device tensors)."""
    n, nb = int(off.numel()) - 1, int(buf.numel())
    tok_start = be.empty((nb // 3 + 1,), torch.int64)
    tok_off = be.empty((n + 1,), torch.int64)
    pair_off = be.empty((n + 1,), torch.int64)
    totals = be.zeros((3,), torch.int64)
    be.text_tokens_chunk(buf, off, cfg["min_n"], cfg["max_n"], tok_start, tok_off, pair_off, totals)
    n_tokens, n_pairs = (int(v) for v in totals[:2].tolist())
    keys = be.empty((max(n_pairs, 1),), torch.int32)
    indptr = be.empty((n + 1,), torch.int64)
    scale = be.empty((max(n, 1),), torch.float64)
    be.text_hash_chunk(buf, tok_start, tok_off, pair_off, n_tokens, n_pairs, cfg["min_n"], cfg["max_n"],
                       cfg["lowercase"], cfg["n_features"], cfg["alternate_sign"], cfg["binary"], cfg["norm"],
                       cfg["dtype"], keys, indptr, scale, totals)
    nnz = int(totals[2].item())
    indices = be.empty((nnz,), torch.int64)
    data = be.empty((nnz,), cfg["dtype"])
    be.text_write_chunk(keys, pair_off, indptr, scale, cfg["binary"], indices, data)
    return indptr, indices, data


def upload(X, device):
    """A scipy CSR matrix -> (indptr, indices, data) int64 / int64 / its dtype on ``device``."""
    return (torch.from_numpy(X.indptr.astype(np.int64)).to(device),
            torch.from_numpy(X.indices.astype(np.int64)).to(device),
            torch.from_numpy(np.ascontiguousarray(X.data)).to(device))


def splice(n, parts, device, dtype):
    """One CSR of n rows from ``parts``, each (rows, indptr, indices, data): rows int64 positions of its rows in
    the output (None: all of them, in order)."""
    if len(parts) == 1 and parts[0][0] is None:
        return parts[0][1:]
    lens = torch.zeros(n, dtype=torch.int64, device=device)
    for rows, ip, _, _ in parts:
        lens[rows] = ip[1:] - ip[:-1]
    crow = torch.zeros(n + 1, dtype=torch.int64, device=device)
    torch.cumsum(lens, 0, out=crow[1:])
    nnz = int(crow[-1].item())
    col = torch.empty(nnz, dtype=torch.int64, device=device)
    val = torch.empty(nnz, dtype=dtype, device=device)
    for rows, ip, c, v in parts:
        shift = crow[rows] - ip[:-1]
        dest = torch.arange(c.numel(), device=device) + torch.repeat_interleave(shift, ip[1:] - ip[:-1])
        col[dest] = c
        val[dest] = v.to(dtype)
    return crow, col, val


class HashingVectorizer(sklearn.feature_extraction.text.HashingVectorizer):
    """Convert a collection of text documents to a matrix of token occurrences, on the device for chunked input.

    scikit-learn's HashingVectorizer (same parameters).  ``transform`` of a 1-D ChunkedArray or dask array of documents
    returns a ChunkedArray with one device ``torch.sparse_csr_tensor`` block (rows, n_features) per input block; other
    input gets scikit-learn's ``transform``.
    """

    def transform(self, X):
        """Transform a sequence of documents to a document-term matrix.

        Parameters
        ----------
        X : ChunkedArray or dask array of raw text documents (1-D), or any input scikit-learn takes

        Returns
        -------
        X : ChunkedArray of device CSR blocks (rows, n_features) for chunked input, else scikit-learn's sparse matrix
        """
        if is_dask_dataframe(X) or type(X).__name__ == "DataFrame":
            raise ValueError(_MSG)
        if not (isinstance(X, ChunkedArray) or is_dask_array(X)):
            return super().transform(X)
        X = as_chunked(X)
        if X.ndim != 1:
            raise ValueError(_MSG)
        cfg = device_config(self)
        if cfg is not None:
            # the checks scikit-learn's transform runs before it tokenises
            self._validate_ngram_range()
            self.build_analyzer()
        be = _km._get_backend()
        return ChunkedArray([self._block(b, cfg, be) for b in X.blocks])

    def _block(self, block, cfg, be):
        docs = block.tolist() if hasattr(block, "tolist") else list(block)
        host_transform = super().transform
        n = len(docs)
        if cfg is None or n == 0:
            X = host_transform(docs)
            crow, col, val = upload(X, be.device)
        else:
            dev, pos, host, joined = route(docs)
            parts = []
            if dev:
                buf, off = pack(dev, joined)
                buf_d = torch.from_numpy(buf).to(be.device)
                off_d = torch.from_numpy(off).to(be.device)
                k = cfg["max_n"] - cfg["min_n"] + 1
                for s, e in batches(off, k):
                    ip, c, v = device_rows(be, buf_d[off[s]: off[e]], off_d[s: e + 1] - int(off[s]), cfg)
                    rows = None if pos is None and (s, e) == (0, n) else torch.as_tensor(
                        (np.arange(s, e) if pos is None else np.asarray(pos[s:e])), dtype=torch.int64).to(be.device)
                    parts.append((rows, ip, c, v))
            if host:
                parts.append((torch.as_tensor(host, dtype=torch.int64).to(be.device),)
                             + upload(host_transform([docs[i] for i in host]), be.device))
            crow, col, val = splice(n, parts, be.device, cfg["dtype"])
        return torch.sparse_csr_tensor(crow, col, val, size=(n, self.n_features), check_invariants=False)
