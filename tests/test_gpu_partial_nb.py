"""The four passes of PartialMultinomialNB / PartialBernoulliNB on the H100 against float64 numpy, and the estimators
end to end against scikit-learn.

Counts of integer data are exact; with arbitrary weights they agree to 1e-13 relative (the order of the sums differs
from BLAS).  The predict passes are held to the error bound of a float64 dot product: per row
E_i = (d + 8) 2^-53 max_c sum_j |f(x_ij) W_cj| + 2^-52 max_c |b_c|, which bounds both the kernel's and numpy's
rounding.  Labels must equal np.argmax of numpy's jll on every row whose top-two margin exceeds 2 E_i (the test
also asserts how many rows that excludes), and the normalised outputs agree to 1e-12 + 4 E_i absolute."""
import itertools
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch
from scipy.special import logsumexp
from sklearn import naive_bayes as sknb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from dask_ml_b200 import ChunkedArray  # noqa: E402
from dask_ml_b200.engine import CudaBackend, host_resident  # noqa: E402
from dask_ml_b200.naive_bayes import PartialBernoulliNB, PartialMultinomialNB  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.filterwarnings("ignore:'Partial.*' is deprecated:FutureWarning")]

DT = {"fp32": torch.float32, "fp64": torch.float64, "bf16": torch.bfloat16}


@pytest.fixture(scope="module")
def be():
    return CudaBackend()


def _rows(be, X, dtype, pitch):
    """X (numpy float64, exactly representable in dtype) on the device in dtype, with a row pitch of d + pitch."""
    n, d = X.shape
    buf = torch.zeros((n, d + pitch), dtype=DT[dtype], device=be.device)
    buf[:, :d] = torch.from_numpy(X).to(be.device, DT[dtype])
    return buf[:, :d]


def _counts_data(n, d, K, seed, lam=0.5, density=0.2):
    rng = np.random.RandomState(seed)
    X = rng.poisson(lam, size=(n, d)).astype(np.float64) * (rng.uniform(size=(n, d)) < density)
    return X, rng.randint(-1, K, size=n).astype(np.int32)           # -1: a label outside the classes


def _ref_counts(X, cls, K, w):
    Y = np.zeros((len(cls), K))
    ok = cls >= 0
    Y[np.nonzero(ok)[0], cls[ok]] = 1.0
    Y *= w[:, None]
    return Y.T @ X, Y.sum(axis=0)


SHAPES = [(d, K) for d, K in itertools.product([1, 31, 32, 33, 1000], [1, 2, 20, 64, 65, 200])] + \
    [(20000, K) for K in (1, 20, 65)]


@pytest.mark.parametrize("dtype", ["fp32", "fp64", "bf16"])
def test_dense_counts(be, dtype):
    for d, K in SHAPES:
        n = 3000 if d <= 1000 else 300
        X, cls = _counts_data(n, d, K, d + K)
        x = _rows(be, X, dtype, 3)
        c = torch.from_numpy(cls).to(be.device)
        for binarize in (None, 0.5):
            Xf = X if binarize is None else (X > binarize).astype(np.float64)
            fc, cc = be.empty((K, d), torch.float64), be.empty((K,), torch.float64)
            be.class_counts_chunk(x, c, K, fc, cc, binarize=binarize, first=True)
            rf, rc = _ref_counts(Xf, cls, K, np.ones(n))
            np.testing.assert_array_equal(fc.cpu().numpy(), rf, err_msg="%s d=%d K=%d" % (dtype, d, K))
            np.testing.assert_array_equal(cc.cpu().numpy(), rc)
        w = np.random.RandomState(d).uniform(0.1, 3.0, n)
        wt = torch.from_numpy(w).to(be.device)
        fc1, cc1 = be.zeros((K, d), torch.float64), be.zeros((K,), torch.float64)
        be.class_counts_chunk(x, c, K, fc1, cc1, w=wt)
        be.class_counts_chunk(x, c, K, fc1, cc1, w=wt)             # accumulates
        rf, rc = _ref_counts(X, cls, K, w)
        np.testing.assert_allclose(fc1.cpu().numpy(), 2 * rf, rtol=1e-13, atol=0)
        np.testing.assert_allclose(cc1.cpu().numpy(), 2 * rc, rtol=1e-13, atol=0)
        fc2, cc2 = be.empty((K, d), torch.float64), be.empty((K,), torch.float64)
        be.class_counts_chunk(x, c, K, fc2, cc2, w=wt, first=True)
        fc3, cc3 = be.empty((K, d), torch.float64), be.empty((K,), torch.float64)
        be.class_counts_chunk(x, c, K, fc3, cc3, w=wt, first=True)
        assert torch.equal(fc2, fc3) and torch.equal(cc2, cc3)


def _csr_block(be, A):
    A = sp.csr_matrix(A)
    return (torch.from_numpy(A.indptr.astype(np.int64)).to(be.device),
            torch.from_numpy(A.indices.astype(np.int64)).to(be.device),
            torch.from_numpy(A.data.astype(np.float64)).to(be.device), A.shape[0])


def _sparse_data(n, d, nnz_row, K, seed):
    rng = np.random.RandomState(seed)
    rows = []
    for i in range(n):
        k = 0 if i % 7 == 3 else rng.randint(0, 2 * nnz_row + 1)          # every 7th row empty
        cols = np.unique(rng.randint(0, d, size=k))
        rows.append((cols, rng.randint(1, 4, size=len(cols)).astype(np.float64)))
    indptr = np.cumsum([0] + [len(c) for c, _ in rows])
    A = sp.csr_matrix((np.concatenate([v for _, v in rows] + [np.zeros(0)]),
                       np.concatenate([c for c, _ in rows] + [np.zeros(0, dtype=np.int64)]), indptr), shape=(n, d))
    return A, rng.randint(-1, K, size=n).astype(np.int32)


SPARSE_SHAPES = [(50, 1), (1000, 20), (1000, 65), (1000, 200), (1 << 20, 20), (33, 2)]


def test_csr_counts(be):
    for d, K in SPARSE_SHAPES:
        A, cls = _sparse_data(2000, d, 20, K, d + K)
        for part in (A, sp.csr_matrix((500, d))):                            # and an all-empty block
            n = part.shape[0]
            c = torch.from_numpy(cls[:n]).to(be.device)
            blk = _csr_block(be, part)
            csc = be.csr_transpose_chunk(blk, d)
            for binarize in (None, 1.5):
                B = part.copy()
                if binarize is not None:
                    B.data = (B.data > binarize).astype(np.float64)
                w = np.random.RandomState(K).choice([0.5, 1.0, 2.0], size=n)
                fcT = be.empty((d, K), torch.float64)
                be.csc_class_counts_chunk(csc, d, c, K, fcT, w=torch.from_numpy(w).to(be.device), binarize=binarize,
                                          first=True)
                rf, _ = _ref_counts(B.toarray() if d <= 1000 else B, cls[:n], K, w)
                got = fcT.cpu().numpy().T
                np.testing.assert_array_equal(got, np.asarray(rf), err_msg="d=%d K=%d" % (d, K))
                again = be.empty((d, K), torch.float64)
                be.csc_class_counts_chunk(csc, d, c, K, again, w=torch.from_numpy(w).to(be.device),
                                          binarize=binarize, first=True)
                assert torch.equal(fcT, again)


def _margin_checks(jll, E, lab, what):
    s = np.sort(np.where(np.isnan(jll), np.inf, jll), axis=1)
    margin = s[:, -1] - s[:, -2] if jll.shape[1] > 1 else np.full(len(jll), np.inf)
    want = np.argmax(jll, axis=1)
    sure = margin > 2 * E
    assert (~sure).sum() <= max(2, len(jll) // 1000), (what, int((~sure).sum()))
    np.testing.assert_array_equal(lab[sure], want[sure], err_msg=what)


def _check_outputs(be, run, Xf, W, b, what):
    """run(labels, out, out_mode) launches the pass; the results against numpy's float64 product."""
    n = Xf.shape[0]
    K = W.shape[0]
    jll = np.asarray(Xf @ W.T) + b
    absdot = np.asarray(abs(Xf) @ np.abs(W).T)
    E = (Xf.shape[1] + 8) * 2.0 ** -53 * absdot.max(axis=1) + 2.0 ** -52 * np.abs(b).max()
    lab = be.empty((n,), torch.int32)
    outs = {m: be.empty((n, K), torch.float64) for m in (0, 1, 2)}
    run(lab, None, 0)
    _margin_checks(jll, E, lab.cpu().numpy(), what)
    lse = logsumexp(jll, axis=1)[:, None]
    for m, ref in ((0, jll), (1, jll - lse), (2, np.exp(jll - lse))):
        run(None, outs[m], m)
        got = outs[m].cpu().numpy()
        tol = 1e-12 + 4 * E[:, None] * (1 if m < 2 else np.maximum(ref, 1e-300))
        assert (np.abs(got - ref) <= tol).all(), (what, m, float(np.abs(got - ref).max()))
    lab2 = be.empty((n,), torch.int32)
    out2 = be.empty((n, K), torch.float64)
    run(lab2, out2, 1)                                       # both epilogues in one call, twice: the same bits
    assert torch.equal(out2, outs[1])
    run(lab2, out2, 1)
    assert torch.equal(out2, outs[1])
    np.testing.assert_array_equal(lab2.cpu().numpy(), lab.cpu().numpy())


def _model(K, d, seed):
    rng = np.random.RandomState(seed)
    flp = np.log(rng.dirichlet(np.ones(d), size=K)) if d > 1 else np.zeros((K, 1))
    return flp, np.log(rng.dirichlet(np.ones(K)))


@pytest.mark.parametrize("dtype", ["fp32", "fp64", "bf16"])
def test_dense_jll(be, dtype):
    for d, K in SHAPES:
        n = 2000 if d <= 1000 else 200
        X, _ = _counts_data(n, d, K, 7 * d + K)
        x = _rows(be, X, dtype, 5)
        W, b = _model(K, d, d + K)
        Wd, bd = torch.from_numpy(W).to(be.device), torch.from_numpy(b).to(be.device)
        for binarize in (None, 0.5):
            Xf = X if binarize is None else (X > binarize).astype(np.float64)

            def run(lab, out, m):
                be.nb_linear_jll_chunk(x, Wd, bd, labels=lab, out=out, out_mode=m, binarize=binarize)
            _check_outputs(be, run, Xf, W, b, "%s d=%d K=%d" % (dtype, d, K))


def test_csr_jll(be):
    for d, K in SPARSE_SHAPES:
        A, _ = _sparse_data(1500, d, 20, K, 3 * d + K)
        W, b = _model(K, d, K)
        WT = torch.from_numpy(np.ascontiguousarray(W.T)).to(be.device)
        bd = torch.from_numpy(b).to(be.device)
        blk = _csr_block(be, A)
        for binarize in (None, 1.5):
            B = A.copy()
            if binarize is not None:
                B.data = (B.data > binarize).astype(np.float64)
                B.eliminate_zeros()

            def run(lab, out, m):
                be.nb_csr_jll_chunk(blk, d, WT, bd, labels=lab, out=out, out_mode=m, binarize=binarize)
            _check_outputs(be, run, B, W, b, "csr d=%d K=%d" % (d, K))


def test_nan_rows(be):
    """0 (-inf) = NaN on the dense pass (as numpy's product); a CSR row reads only its stored entries."""
    X = np.array([[0.0, 2.0, 1.0], [1.0, 0.0, 3.0], [0.0, 0.0, 0.0], [2.0, 1.0, 1.0]])
    W = np.log(np.array([[0.2, 0.5, 0.3], [0.0, 0.6, 0.4], [0.3, 0.3, 0.4]]))          # -inf in class 1, feature 0
    b = np.log(np.array([0.3, 0.3, 0.4]))
    Wd, bd = torch.from_numpy(W).to(be.device), torch.from_numpy(b).to(be.device)
    with np.errstate(all="ignore"):
        ref = X @ W.T + b
    for dtype in DT:
        x = _rows(be, X, dtype, 1)
        lab = be.empty((4,), torch.int32)
        out = be.empty((4, 3), torch.float64)
        be.nb_linear_jll_chunk(x, Wd, bd, labels=lab, out=out, out_mode=0)
        np.testing.assert_array_equal(out.cpu().numpy(), ref)
        np.testing.assert_array_equal(lab.cpu().numpy(), np.argmax(ref, axis=1))            # the first NaN wins
        be.nb_linear_jll_chunk(x, Wd, bd, out=out, out_mode=1)
        got = out.cpu().numpy()
        assert np.isnan(got[[0, 2]]).all() and np.isfinite(got[[1, 3]][:, [0, 2]]).all()
        assert (got[[1, 3], 1] == -np.inf).all()
    blk = _csr_block(be, X)
    lab = be.empty((4,), torch.int32)
    out = be.empty((4, 3), torch.float64)
    be.nb_csr_jll_chunk(blk, 3, torch.from_numpy(np.ascontiguousarray(W.T)).to(be.device), bd, labels=lab, out=out)
    with np.errstate(all="ignore"):
        want = np.asarray(sp.csr_matrix(X) @ W.T) + b
    np.testing.assert_allclose(out.cpu().numpy(), want, rtol=1e-15)
    np.testing.assert_array_equal(lab.cpu().numpy(), np.argmax(want, axis=1))


def _np(a):
    return np.concatenate([b.cpu().numpy() for b in a.blocks]) if isinstance(a, ChunkedArray) else np.asarray(a)


def test_hashing_vectorizer_pipeline():
    from sklearn.feature_extraction.text import HashingVectorizer as SkHV

    from dask_ml_b200.feature_extraction.text import HashingVectorizer

    rng = np.random.RandomState(0)
    words = ["alpha", "beta", "gamma", "delta", "eps", "zeta", "eta", "theta", "iota", "kappa"]
    docs = np.array([" ".join(rng.choice(words, 15)) for _ in range(900)], dtype=object)
    y = np.array([("alpha" in d) + ("beta" in d) + ("iota" in d) for d in docs])
    Xh = HashingVectorizer(alternate_sign=False, norm=None).transform(ChunkedArray([docs[:400], docs[400:]]))
    np.random.seed(5)
    est = PartialMultinomialNB(classes=[0, 1, 2, 3]).fit(Xh, ChunkedArray([y[:400], y[400:]]))
    np.random.seed(5)
    order = [0, 1]
    np.random.shuffle(order)
    Xs = SkHV(alternate_sign=False, norm=None).transform(docs)
    ref = sknb.MultinomialNB()
    for i in order:
        a, z = (0, 400) if i == 0 else (400, 900)
        ref.partial_fit(Xs[a:z], y[a:z], classes=[0, 1, 2, 3])
    for k in ("feature_count_", "class_count_", "feature_log_prob_", "class_log_prior_"):
        np.testing.assert_array_equal(getattr(est, k), getattr(ref, k))
    pred = est.predict(Xh)
    assert pred.blocks[0].is_cuda
    np.testing.assert_array_equal(_np(pred), ref.predict(Xs))
    assert est.predict_proba(Xh).blocks[0].is_cuda
    np.testing.assert_allclose(_np(est.predict_log_proba(Xh)), ref.predict_log_proba(Xs), rtol=0, atol=1e-10)
    assert est.score(Xh, y) == ref.score(Xs, y)


@pytest.mark.parametrize("form", ["device", "host_resident", "numpy"])
def test_make_counts_blocks(form):
    from dask_ml_b200.datasets import make_counts

    X, y = make_counts(n_samples=6000, n_features=40, chunks=1500, random_state=3,
                       device=None if form != "device" else "cuda")
    Xh = np.concatenate([np.asarray(b.cpu() if isinstance(b, torch.Tensor) else b) for b in X.blocks])
    yh = np.concatenate([np.asarray(b.cpu() if isinstance(b, torch.Tensor) else b) for b in y.blocks])
    Xin = {"device": X, "host_resident": host_resident(Xh, block_rows=1500), "numpy": Xh}[form]
    classes = np.unique(yh)
    np.random.seed(9)
    est = PartialBernoulliNB(classes=classes, binarize=0.0).fit(Xin, y if form == "device" else yh)
    np.random.seed(9)
    nblk = 4 if form != "numpy" else 1
    order = list(range(nblk))
    np.random.shuffle(order)
    ref = sknb.BernoulliNB(binarize=0.0)
    rows = len(yh) // nblk
    for i in order:
        ref.partial_fit(Xh[i * rows:(i + 1) * rows], yh[i * rows:(i + 1) * rows], classes=classes)
    for k in ("feature_count_", "class_count_", "feature_log_prob_", "class_log_prior_"):
        np.testing.assert_array_equal(getattr(est, k), getattr(ref, k))
    pred = est.predict(Xin)
    np.testing.assert_array_equal(_np(pred), ref.predict(Xh))
    np.testing.assert_allclose(_np(est.predict_proba(Xin)), ref.predict_proba(Xh), rtol=0, atol=1e-12)
