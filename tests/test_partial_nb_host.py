"""PartialMultinomialNB and PartialBernoulliNB on CPU: the host control flow of ``_BaseDiscreteNB.partial_fit`` and the
reference's block-wise ``fit``, on a checker backend whose count and log-likelihood passes are float64 numpy / scipy
restatements.

Counts of integer data with dyadic weights are exact in any order, so ``feature_count_``, ``class_count_``,
``feature_log_prob_`` and ``class_log_prior_`` are pinned bit for bit against live scikit-learn ``partial_fit``
sequences; the reference's own fits (tests/golden/ref_partial_nb.py) are replayed from the fixtures."""
import json
import os
import pickle
import sys
import warnings

import numpy as np
import pytest
import scipy.sparse as sp
import torch
from scipy.special import logsumexp
from sklearn import naive_bayes as sknb
from sklearn.utils import check_random_state

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
GOLDEN = os.path.join(ROOT, "tests", "golden")

from test_glm_sparse_host import SparseOracleBackend  # noqa: E402

from dask_ml_b200 import ChunkedArray  # noqa: E402
from dask_ml_b200.cluster import k_means as km  # noqa: E402
from dask_ml_b200.naive_bayes import PartialBernoulliNB, PartialMultinomialNB  # noqa: E402

pytestmark = pytest.mark.filterwarnings("ignore:'Partial.*' is deprecated:FutureWarning")


def _onehot(cls, K, w):
    c = cls.numpy()
    Y = np.zeros((len(c), K))
    ok = (c >= 0) & (c < K)
    Y[np.nonzero(ok)[0], c[ok]] = 1.0
    return Y * (w.numpy()[:, None] if w is not None else 1.0)


def _bin_csr(A, t):
    if t is None:
        return A
    A = A.copy()
    A.data = (A.data > t).astype(np.float64)
    A.eliminate_zeros()
    return A


def _jll_out(jll, labels, out, out_mode):
    if labels is not None:
        labels.copy_(torch.from_numpy(np.argmax(jll, axis=1).astype(np.int32)))
    if out is not None:
        with np.errstate(invalid="ignore"):
            o = jll if out_mode == 0 else jll - logsumexp(jll, axis=1)[:, None]
        out.copy_(torch.from_numpy(np.exp(o) if out_mode == 2 else o))


class NBChecker(SparseOracleBackend):
    """The CPU checker backend plus float64 restatements of the four passes of the discrete naive Bayes models."""

    def class_counts_chunk(self, x, cls, K, fc, cc, w=None, binarize=None, first=False):
        X = x.to(torch.float64).numpy()
        if binarize is not None:
            X = (X > binarize).astype(np.float64)
        Y = _onehot(cls, K, w)
        for acc, v in ((fc, Y.T @ X), (cc, Y.sum(axis=0))):
            acc.copy_(torch.from_numpy(v)) if first else acc.add_(torch.from_numpy(v))

    def csc_class_counts_chunk(self, csc, d, labels, K, fcT, w=None, binarize=None, first=False):
        colptr, rows, vals, _plan = csc
        C = sp.csc_matrix((vals.numpy().astype(np.float64), rows.numpy(), colptr.numpy()), shape=(len(labels), d))
        v = torch.from_numpy(np.asarray((_bin_csr(C.tocsr(), binarize).T @ _onehot(labels, K, w))))
        fcT.copy_(v) if first else fcT.add_(v)

    def nb_linear_jll_chunk(self, x, W, b, labels=None, out=None, out_mode=0, binarize=None):
        X = x.to(torch.float64).numpy()
        if binarize is not None:
            X = (X > binarize).astype(np.float64)
        with np.errstate(invalid="ignore"):
            _jll_out(X @ W.numpy().T + b.numpy(), labels, out, out_mode)

    def nb_csr_jll_chunk(self, blk, d, WT, b, labels=None, out=None, out_mode=0, binarize=None):
        crow, col, val, n = blk
        A = _bin_csr(sp.csr_matrix((val.to(torch.float64).numpy(), col.numpy(), crow.numpy()), shape=(n, d)),
                     binarize)
        _jll_out(np.asarray(A @ WT.numpy()) + b.numpy(), labels, out, out_mode)


@pytest.fixture(autouse=True)
def checker(monkeypatch):
    monkeypatch.setattr(km, "_BACKEND_FACTORY", NBChecker)


def _counts(n, d, K, seed, density=0.3):
    rng = np.random.RandomState(seed)
    X = rng.poisson(2.0, size=(n, d)).astype(np.float64) * (rng.uniform(size=(n, d)) < density)
    return X, rng.randint(0, K, size=n)


def _np(a):
    if isinstance(a, ChunkedArray):
        return np.concatenate([b.cpu().numpy() if isinstance(b, torch.Tensor) else np.asarray(b) for b in a.blocks])
    return a.cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)


def _assert_same(ours, ref):
    for name in ("feature_count_", "class_count_", "feature_log_prob_", "class_log_prior_"):
        np.testing.assert_array_equal(getattr(ours, name), getattr(ref, name), err_msg=name)
    np.testing.assert_array_equal(ours.classes_, ref.classes_)


def _assert_predict(ours, ref, X):
    Xr = X.toarray() if sp.issparse(X) else X
    np.testing.assert_array_equal(_np(ours.predict(X)), ref.predict(X))
    with np.errstate(all="ignore"):
        for m in ("predict_joint_log_proba", "predict_log_proba", "predict_proba"):
            np.testing.assert_allclose(_np(getattr(ours, m)(X)), getattr(ref, m)(X), rtol=1e-12, atol=1e-12,
                                       err_msg=m)
    assert ours.score(X, ref.predict(Xr)) == 1.0


CASES = {
    "mnb": (PartialMultinomialNB, dict()),
    "mnb_alpha_array": (PartialMultinomialNB, dict(alpha=np.linspace(0.5, 2.0, 9))),
    "mnb_no_prior": (PartialMultinomialNB, dict(fit_prior=False, alpha=0.25)),
    "mnb_class_prior": (PartialMultinomialNB, "prior"),
    "bnb": (PartialBernoulliNB, dict()),
    "bnb_none": (PartialBernoulliNB, dict(binarize=None)),
    "bnb_half": (PartialBernoulliNB, dict(binarize=0.5, alpha=2.0)),
    "bnb_class_prior": (PartialBernoulliNB, "prior"),
}


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("sparse", [False, True])
@pytest.mark.parametrize("K", [1, 2, 4])
@pytest.mark.parametrize("name", sorted(CASES))
def test_partial_fit_matches_sklearn(name, K, sparse, weighted):
    cls, kw = CASES[name]
    if kw == "prior":
        kw = dict(class_prior=np.arange(1, K + 1) / (K * (K + 1) / 2.0))
    classes = np.arange(K) * 3
    ours = cls(classes=classes, **kw)
    ref = getattr(sknb, cls.__name__[len("Partial"):])(**kw)
    for i in range(3):
        X, y = _counts(60 + 17 * i, 9, K, i)
        y = y * 3
        if sparse:
            X = sp.csr_matrix(X)
        swkw = {}
        if weighted:
            swkw["sample_weight"] = np.random.RandomState(i).choice([0.5, 1.0, 2.0], size=len(y))
        ours.partial_fit(X, y, classes=classes, **swkw)
        ref.partial_fit(X, y, classes=classes, **swkw)
        _assert_same(ours, ref)
    _assert_predict(ours, ref, X)


def test_fit_steps_blocks_in_shuffled_order():
    X, y = _counts(600, 7, 3, 5)
    chunks = [(0, 150), (150, 350), (350, 600)]
    Xc = ChunkedArray([X[a:b] for a, b in chunks])
    yc = ChunkedArray([y[a:b] for a, b in chunks])
    np.random.seed(11)
    ours = PartialMultinomialNB(classes=[0, 1, 2], alpha=0.5).fit(Xc, yc)
    np.random.seed(11)
    order = list(range(3))
    check_random_state(None).shuffle(order)
    ref = sknb.MultinomialNB(alpha=0.5)
    for i in order:
        a, b = chunks[i]
        ref.partial_fit(X[a:b], y[a:b], classes=[0, 1, 2])
    _assert_same(ours, ref)
    with pytest.raises(NotImplementedError):
        ours.fit(Xc, yc, compute=False)


def test_float32_threshold_and_torch_input():
    X = (np.random.RandomState(0).uniform(size=(200, 5)) * 0.3).astype(np.float32)
    X[:, 0] = np.float32(0.1)                            # on the threshold as float32 compares it
    y = np.arange(200) % 2
    ours = PartialBernoulliNB(classes=[0, 1], binarize=0.1).partial_fit(torch.from_numpy(X), torch.from_numpy(y),
                                                                    classes=[0, 1])
    ref = sknb.BernoulliNB(binarize=0.1).partial_fit(X, y, classes=[0, 1])
    _assert_same(ours, ref)
    _assert_predict(ours, ref, X)


def test_string_labels_unknown_labels_and_binary_column():
    X, _ = _counts(90, 4, 3, 1)
    y = np.array(["a", "b", "zz"])[np.arange(90) % 3]
    for classes in (["a", "b", "c"], ["a", "b"]):
        ours = PartialMultinomialNB(classes=classes).partial_fit(X, y, classes=classes)
        ref = sknb.MultinomialNB().partial_fit(X, y, classes=classes)
        _assert_same(ours, ref)
        assert isinstance(ours.predict(X), np.ndarray)
        np.testing.assert_array_equal(ours.predict(X), ref.predict(X))
    # two classes and two distinct labels: label_binarize's binary column counts "zz" for the first class
    y2 = np.where(np.arange(90) % 2 == 0, "b", "zz")
    ours = PartialMultinomialNB(classes=["a", "b"]).partial_fit(X, y2, classes=["a", "b"])
    ref = sknb.MultinomialNB().partial_fit(X, y2, classes=["a", "b"])
    _assert_same(ours, ref)


def test_classes_must_match_between_calls():
    X, y = _counts(40, 3, 2, 0)
    est = PartialMultinomialNB(classes=[0, 1])
    with pytest.raises(ValueError, match="classes must be passed on the first call"):
        est.partial_fit(X, y)
    est.partial_fit(X, y, classes=[0, 1])
    with pytest.raises(ValueError, match="is not the same as on last call"):
        est.partial_fit(X, y, classes=[0, 1, 2])


def test_error_messages():
    X, y = _counts(40, 3, 2, 0)
    with pytest.raises(ValueError, match=r"Negative values in data passed to MultinomialNB \(input X\)"):
        PartialMultinomialNB(classes=[0, 1]).partial_fit(-X - 1, y, classes=[0, 1])
    with pytest.raises(ValueError, match=r"Negative values in data passed to MultinomialNB \(input X\)"):
        PartialMultinomialNB(classes=[0, 1]).partial_fit(sp.csr_matrix(-X), y, classes=[0, 1])
    PartialBernoulliNB(classes=[0, 1]).partial_fit(-X, y, classes=[0, 1])         # BernoulliNB takes them
    with pytest.raises(ValueError, match="The 'binarize' parameter of PartialBernoulliNB must be None or a float"):
        PartialBernoulliNB(classes=[0, 1], binarize=-1.0).partial_fit(sp.csr_matrix(X), y, classes=[0, 1])
    bnb = PartialBernoulliNB(classes=[0, 1]).partial_fit(X, y, classes=[0, 1])
    bnb.binarize = -1.0                                  # predict validates no parameter, as in scikit-learn
    with pytest.raises(ValueError, match="Cannot binarize a sparse matrix with threshold < 0"):
        bnb.predict(sp.csr_matrix(X))
    Xn = X.copy()
    Xn[3, 1] = np.nan
    with pytest.raises(ValueError, match="Input X contains NaN"):
        PartialMultinomialNB(classes=[0, 1]).partial_fit(Xn, y, classes=[0, 1])
    Xn[3, 1] = np.inf
    with pytest.raises(ValueError, match="Input X contains infinity"):
        PartialMultinomialNB(classes=[0, 1]).partial_fit(Xn, y, classes=[0, 1])
    with pytest.raises(ValueError, match="Input y contains NaN"):
        PartialMultinomialNB(classes=[0.0, 1.0]).partial_fit(X, np.where(y == 0, np.nan, 1.0), classes=[0.0, 1.0])
    est = PartialMultinomialNB(classes=[0, 1]).partial_fit(X, y, classes=[0, 1])
    with pytest.raises(ValueError, match="X has 4 features, but PartialMultinomialNB is expecting 3 features"):
        est.partial_fit(np.ones((5, 4)), np.zeros(5, dtype=int))
    with pytest.raises(ValueError, match="X has 4 features"):
        est.predict(np.ones((5, 4)))
    with pytest.raises(ValueError, match="Sample weights must be 1D array or scalar"):
        est.partial_fit(X, y, sample_weight=np.ones((len(y), 2)))
    with pytest.raises(ValueError, match="When alpha is an array, it should contains `n_features`"):
        PartialMultinomialNB(classes=[0, 1], alpha=np.ones(5)).partial_fit(X, y, classes=[0, 1])
    with pytest.raises(ValueError, match="Number of priors must match number of classes"):
        PartialMultinomialNB(classes=[0, 1], class_prior=[1.0]).partial_fit(X, y, classes=[0, 1])


def test_force_alpha_zero_keeps_nan_rows():
    X, y = _counts(50, 6, 2, 3, density=0.5)
    X[:, 0] = 0.0
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        ours = PartialMultinomialNB(classes=[0, 1], alpha=0.0, force_alpha=True).partial_fit(X, y, classes=[0, 1])
        ref = sknb.MultinomialNB(alpha=0.0, force_alpha=True).partial_fit(X, y, classes=[0, 1])
        _assert_same(ours, ref)
        np.testing.assert_array_equal(_np(ours.predict(X)), ref.predict(X))
        np.testing.assert_array_equal(_np(ours.predict_joint_log_proba(X)), ref.predict_joint_log_proba(X))
        A = sp.csr_matrix(X)
        np.testing.assert_array_equal(_np(ours.predict_joint_log_proba(A)), ref.predict_joint_log_proba(A))
    assert np.isnan(_np(ours.predict_joint_log_proba(X))).all()
    assert np.isfinite(_np(ours.predict_joint_log_proba(sp.csr_matrix(X)))[X[:, 0] >= 0]).any()


def test_pickle_warning_and_params():
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        est = PartialBernoulliNB(classes=[0, 1], alpha=0.5)
    msgs = [str(w.message) for w in rec if issubclass(w.category, FutureWarning)]
    assert msgs == ["'PartialBernoulliNB' is deprecated. Use 'dask_ml.wrappers.Incremental(BernoulliNB(), **kwargs)' "
                    "instead."]
    params = est.get_params()
    assert params["classes"] == [0, 1] and params["alpha"] == 0.5 and "binarize" in params
    with pytest.raises(TypeError, match="requires the keyword arguments"):
        PartialMultinomialNB()
    X, y = _counts(80, 5, 2, 2)
    est.partial_fit(X, y, classes=[0, 1])
    est2 = pickle.loads(pickle.dumps(est))
    X2, y2 = _counts(70, 5, 2, 3)
    est.partial_fit(X2, y2)
    est2.partial_fit(X2, y2)
    _assert_same(est2, est)
    np.testing.assert_array_equal(_np(est2.predict(X2)), _np(est.predict(X2)))


def _torch_csr(B):
    return torch.sparse_csr_tensor(torch.from_numpy(B.indptr.astype(np.int64)),
                                   torch.from_numpy(B.indices.astype(np.int64)), torch.from_numpy(B.data), size=B.shape)


def test_reference_fixtures():
    with open(os.path.join(GOLDEN, "REF_PARTIAL_NB_MANIFEST.json")) as f:
        manifest = json.load(f)
    for name, case in manifest["cases"].items():
        z = np.load(os.path.join(GOLDEN, name + ".npz"), allow_pickle=False)
        X, y, rows = z["X"], z["y"], int(z["rows"])
        if case["sparse"]:
            X = sp.csr_matrix(X)
        cls = {"PartialMultinomialNB": PartialMultinomialNB, "PartialBernoulliNB": PartialBernoulliNB}[case["cls"]]
        with warnings.catch_warnings(record=True) as rec:
            warnings.simplefilter("always")
            est = cls(**case["params"])
        assert [str(w.message) for w in rec if issubclass(w.category, FutureWarning)] == case["deprecation"]
        bounds = list(range(0, X.shape[0], rows)) + [X.shape[0]]
        Xc = ChunkedArray([_torch_csr(X[a:b]) if case["sparse"] else X[a:b] for a, b in zip(bounds[:-1], bounds[1:])])
        yc = ChunkedArray([y[a:b] for a, b in zip(bounds[:-1], bounds[1:])])
        np.random.seed(int(z["seed"]))
        est.fit(Xc, yc)
        for k in ("feature_count", "class_count", "feature_log_prob", "class_log_prior"):
            np.testing.assert_array_equal(getattr(est, k + "_"), z[k], err_msg=name + " " + k)
        np.testing.assert_array_equal(_np(est.predict(X)), z["predict"])
        np.testing.assert_allclose(_np(est.predict_log_proba(X)), z["predict_log_proba"], rtol=1e-12, atol=1e-12)
