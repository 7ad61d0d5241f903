"""The SGD family on CPU: the host control flow of scikit-learn's ``partial_fit`` and the reference's block-wise ``fit``,
with the device epoch replaced by a checker backend that runs the installed ``_plain_sgd64`` on the rows in the order
the host computed (``shuffle=False``).

Pins the numpy draw sequence, the row orders of ``bkm_sgd_order``, ``t_``, the intercept bookkeeping and the switch to
averaged coefficients against live scikit-learn ``partial_fit`` sequences, bit for bit."""
import ctypes
import os
import pickle
import sys
import warnings

import numpy as np
import pytest
import scipy.sparse as sp
import torch
from sklearn import linear_model as sklm
from sklearn._loss._loss import CyHalfBinomialLoss, CyHalfSquaredError, CyHuberLoss
from sklearn.linear_model._sgd_fast import (EpsilonInsensitive, Hinge, ModifiedHuber, SquaredEpsilonInsensitive,
                                            SquaredHinge, _plain_sgd64)
from sklearn.utils._seq_dataset import ArrayDataset64, CSRDataset64

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle_backend import OracleBackend  # noqa: E402

from dask_ml_b200 import ChunkedArray  # noqa: E402
from dask_ml_b200 import _lib  # noqa: E402
from dask_ml_b200.cluster import k_means as km  # noqa: E402
from dask_ml_b200.linear_model import (PartialPassiveAggressiveClassifier, PartialPassiveAggressiveRegressor,  # noqa: E402
                                       PartialPerceptron, PartialSGDClassifier, PartialSGDRegressor)
from dask_ml_b200.linear_model._sgd import _sklearn_base  # noqa: E402

pytestmark = [pytest.mark.filterwarnings("ignore:'Partial.*' is deprecated:FutureWarning"),
              pytest.mark.filterwarnings("ignore::FutureWarning")]


def _loss_object(code, eps):
    return [lambda: Hinge(eps), CyHalfBinomialLoss, ModifiedHuber, lambda: SquaredHinge(eps), CyHalfSquaredError,
            lambda: CyHuberLoss(eps), lambda: EpsilonInsensitive(eps), lambda: SquaredEpsilonInsensitive(eps)][code]()


class SgdChecker(OracleBackend):
    """The oracle backend plus the SGD epoch: scikit-learn's ``_plain_sgd64`` per problem on the rows in the given
    order, without shuffling."""

    calls = 0
    power_t = 0.25      # the host passes 'invscaling' as a table of rates; every case here uses SGDRegressor's default

    def _epoch(self, rows, order, y, sw, cw, prm, w, aw, st):
        SgdChecker.calls += 1
        P, n = order.shape
        swn = np.ones(n) if sw is None else sw.numpy()
        for p in range(P):
            o = order[p].numpy().astype(np.int64)
            ds = rows(o, np.ascontiguousarray(y[p].numpy()[o]), np.ascontiguousarray(swn[o]))
            wp = w[p].numpy().copy()
            awp = aw[p].numpy().copy() if prm.average > 0 else None
            try:
                res = _plain_sgd64(wp, float(st[p, 0]), awp, float(st[p, 1]), _loss_object(prm.loss, prm.epsilon),
                                   prm.penalty, prm.alpha, prm.l1_ratio, ds, np.zeros(n, dtype=np.uint8), False,
                                   None, 5, 1, -np.inf, prm.fit_intercept, 0, False, 1, float(cw[p, 0]),
                                   float(cw[p, 1]), prm.learning_rate, prm.eta0, self.power_t, 0, prm.t0,
                                   prm.intercept_decay, int(prm.average))
            except ValueError:
                st[p, 2] = 1.0
                continue
            w[p] = torch.from_numpy(res[0])
            if awp is not None:
                aw[p] = torch.from_numpy(res[2])
            st[p, 0], st[p, 1] = res[1], res[3]

    def sgd_block(self, x, order, y, sw, eta, cw, params, w, aw, q, st):
        X = x.to(torch.float64).numpy()
        self._epoch(lambda o, yy, ss: ArrayDataset64(np.ascontiguousarray(X[o]), yy, ss, 1),
                    order, y, sw, cw, params, w, aw, st)

    def sgd_csr_block(self, blk, d, order, y, sw, eta, cw, params, w, aw, q, st):
        crow, col, val, n = blk
        A = sp.csr_matrix((val.to(torch.float64).numpy(), col.numpy(), crow.numpy()), shape=(n, d))

        def rows(o, yy, ss):
            B = A[o]
            return CSRDataset64(B.data, B.indptr, B.indices.astype(np.int32), yy, ss, 1)

        self._epoch(rows, order, y, sw, cw, params, w, aw, st)

    def project_chunk(self, x, shift, W, out=None, colmax=None, row_offset=0):
        out.copy_(torch.from_numpy(x.to(torch.float64).numpy() @ W.numpy().T))

    def csr_panel_chunk(self, blk, d, W, out=None, colmax=None, row_offset=0):
        crow, col, val, n = blk
        A = sp.csr_matrix((val.to(torch.float64).numpy(), col.numpy(), crow.numpy()), shape=(n, d))
        out.copy_(torch.from_numpy(A @ W.numpy()))


@pytest.fixture(autouse=True)
def checker(monkeypatch):
    monkeypatch.setattr(km, "_BACKEND_FACTORY", SgdChecker)


def _data(n, d, k, seed, regression=False):
    rng = np.random.RandomState(seed)
    X = rng.standard_normal((n, d))
    if regression:
        return X, X @ rng.standard_normal(d) + 0.1 * rng.standard_normal(n)
    return X, rng.randint(0, k, size=n)


def _assert_same(a, b):
    np.testing.assert_array_equal(np.atleast_2d(a.coef_), np.atleast_2d(b.coef_))
    np.testing.assert_array_equal(np.atleast_1d(a.intercept_), np.atleast_1d(b.intercept_))
    assert a.t_ == b.t_
    assert a.n_iter_ == b.n_iter_


# ---------------------------------------------------------------------------------------------------------------
def test_order_matches_sklearn_shuffle():
    lib = _lib.load()
    for n in (1, 2, 3, 10, 1000, 10 ** 5):
        for seed in (1, 7, 12345, 2 ** 31 - 2):
            o = np.empty(n, dtype=np.int32)
            assert lib.bkm_sgd_order(n, seed, o.ctypes.data_as(ctypes.c_void_p)) == 0
            ds = ArrayDataset64(np.zeros((n, 1)), np.zeros(n), np.ones(n), 1)
            ds._shuffle_py(seed)
            want = [ds._next_py()[-1] for _ in range(n)]
            np.testing.assert_array_equal(o, want)


CLF_CASES = {
    "binary_hinge": (PartialSGDClassifier, dict(), 2, False),
    "multiclass_3": (PartialSGDClassifier, dict(loss="modified_huber", penalty="elasticnet"), 3, False),
    "multiclass_20": (PartialSGDClassifier, dict(loss="squared_hinge", learning_rate="constant", eta0=0.01), 20,
                      False),
    "average": (PartialSGDClassifier, dict(average=True, penalty="l1"), 3, False),
    "average_binary_10": (PartialSGDClassifier, dict(average=10), 2, False),
    "class_weight": (PartialSGDClassifier, dict(class_weight={0: 2.0, 1: 0.5}), 2, False),
    "sample_weight": (PartialSGDClassifier, dict(loss="perceptron"), 3, True),
    "log_loss": (PartialSGDClassifier, dict(loss="log_loss"), 2, False),
    "no_shuffle": (PartialSGDClassifier, dict(shuffle=False, fit_intercept=False), 3, False),
    "perceptron": (PartialPerceptron, dict(penalty="l2", alpha=1e-3), 3, False),
    "pa1": (PartialPassiveAggressiveClassifier, dict(C=0.5), 3, False),
    "pa2": (PartialPassiveAggressiveClassifier, dict(loss="squared_hinge"), 2, False),
}


@pytest.mark.parametrize("sparse", [False, True])
@pytest.mark.parametrize("name", sorted(CLF_CASES))
def test_classifier_matches_sklearn(name, sparse):
    cls, kw, k, weighted = CLF_CASES[name]
    classes = np.arange(k)
    ours = cls(classes=classes, random_state=3, **kw)
    ref = _sklearn_base(cls)(random_state=3, **kw)
    for i in range(3):
        X, y = _data(200 + 13 * i, 7, k, i)
        Xi = sp.csr_matrix(X * (np.abs(X) > 0.5)) if sparse else X
        swkw = {"sample_weight": np.random.RandomState(i).uniform(0.5, 2, len(y))} if weighted else {}
        ours.partial_fit(Xi, y, classes=classes, **swkw)
        ref.partial_fit(Xi, y, classes=classes, **swkw)
        _assert_same(ours, ref)


REG_CASES = {
    "squared_error": (PartialSGDRegressor, dict()),
    "huber": (PartialSGDRegressor, dict(loss="huber", penalty="l1", learning_rate="constant", eta0=0.001)),
    "eps": (PartialSGDRegressor, dict(loss="epsilon_insensitive", average=True)),
    "sq_eps": (PartialSGDRegressor, dict(loss="squared_epsilon_insensitive", penalty="elasticnet", average=50)),
    "pa1": (PartialPassiveAggressiveRegressor, dict()),
    "pa2": (PartialPassiveAggressiveRegressor, dict(loss="squared_epsilon_insensitive", C=0.1)),
}


@pytest.mark.parametrize("sparse", [False, True])
@pytest.mark.parametrize("name", sorted(REG_CASES))
def test_regressor_matches_sklearn(name, sparse):
    cls, kw = REG_CASES[name]
    ours = cls(random_state=5, **kw)
    ref = _sklearn_base(cls)(random_state=5, **kw)
    for i in range(3):
        X, y = _data(150 + 7 * i, 6, 0, 10 + i, regression=True)
        Xi = sp.csr_matrix(X * (np.abs(X) > 0.5)) if sparse else X
        ours.partial_fit(Xi, y)
        ref.partial_fit(Xi, y)
        _assert_same(ours, ref)


def test_fit_steps_blocks_in_shuffled_order():
    X, y = _data(600, 5, 3, 0)
    chunks = [(0, 150), (150, 350), (350, 600)]
    Xc = ChunkedArray([X[a:b] for a, b in chunks])
    yc = ChunkedArray([y[a:b] for a, b in chunks])
    np.random.seed(11)
    ours = PartialSGDClassifier(classes=[0, 1, 2], random_state=0).fit(Xc, yc)
    np.random.seed(11)
    order = list(range(3))
    from sklearn.utils import check_random_state
    check_random_state(None).shuffle(order)
    ref = sklm.SGDClassifier(random_state=0)
    for i in order:
        a, b = chunks[i]
        ref.partial_fit(X[a:b], y[a:b], classes=[0, 1, 2])
    _assert_same(ours, ref)


def test_partial_fit_of_several_chunks_is_one_batch():
    X, y = _data(300, 4, 2, 1)
    ours = PartialSGDClassifier(classes=[0, 1], random_state=2)
    ours.partial_fit(ChunkedArray([X[:100], X[100:]]), y, classes=[0, 1])
    ref = sklm.SGDClassifier(random_state=2).partial_fit(X, y, classes=[0, 1])
    _assert_same(ours, ref)


def test_pickle_keeps_float64_state():
    X, y = _data(200, 4, 3, 2)
    a = PartialSGDClassifier(classes=[0, 1, 2], random_state=1, average=True).partial_fit(X, y, classes=[0, 1, 2])
    b = pickle.loads(pickle.dumps(a))
    a.partial_fit(X, y)
    b.partial_fit(X, y)
    _assert_same(a, b)


def test_predict_and_scores():
    X, y = _data(300, 5, 3, 4)
    ours = PartialSGDClassifier(classes=[0, 1, 2], loss="log_loss", random_state=1).partial_fit(X, y, [0, 1, 2])
    ref = sklm.SGDClassifier(loss="log_loss", random_state=1).partial_fit(X, y, classes=[0, 1, 2])
    np.testing.assert_allclose(ours.decision_function(X).compute(), ref.decision_function(X), rtol=1e-12)
    np.testing.assert_array_equal(ours.predict(X).compute(), ref.predict(X))
    np.testing.assert_allclose(ours.predict_proba(X).compute(), ref.predict_proba(X), rtol=1e-12)
    assert ours.score(X, y) == ref.score(X, y)
    Xr, yr = _data(200, 4, 0, 5, regression=True)
    r = PartialSGDRegressor(random_state=0).partial_fit(Xr, yr)
    rr = sklm.SGDRegressor(random_state=0).partial_fit(Xr, yr)
    np.testing.assert_allclose(r.predict(Xr).compute(), rr.predict(Xr), rtol=1e-12)
    np.testing.assert_allclose(r.score(Xr, yr), rr.score(Xr, yr), rtol=1e-12)


def test_errors_match_sklearn():
    X, y = _data(50, 3, 2, 0)
    with pytest.warns(FutureWarning, match="'PartialSGDClassifier' is deprecated. Use "
                                           r"'dask_ml.wrappers.Incremental\(SGDClassifier\(\), \*\*kwargs\)' instead."):
        PartialSGDClassifier(classes=[0, 1])
    with pytest.raises(TypeError, match="requires the keyword arguments"):
        PartialSGDClassifier()
    for kw in (dict(class_weight="balanced"), dict(early_stopping=True)):
        with pytest.raises(ValueError) as ours:
            PartialSGDClassifier(classes=[0, 1], **kw).partial_fit(X, y, classes=[0, 1])
        with pytest.raises(ValueError) as ref:
            sklm.SGDClassifier(**kw).partial_fit(X, y, classes=[0, 1])
        assert str(ours.value) == str(ref.value)
    est = PartialSGDClassifier(classes=[0, 1]).partial_fit(X, y, classes=[0, 1])
    with pytest.raises(ValueError, match="X has 4 features, but PartialSGDClassifier is expecting 3"):
        est.partial_fit(np.ones((5, 4)), np.ones(5))
    with pytest.raises(ValueError) as ours:
        PartialSGDRegressor(learning_rate="constant", eta0=1e200).partial_fit(X * 1e200, y * 1e200)
    with pytest.raises(ValueError) as ref:
        sklm.SGDRegressor(learning_rate="constant", eta0=1e200).partial_fit(X * 1e200, y * 1e200)
    assert str(ours.value) == str(ref.value)
    params = PartialSGDClassifier(classes=[0, 1]).get_params()
    assert params["classes"] == [0, 1] and "alpha" in params


def test_abi_argument_errors():
    """The new entry points reject bad arguments before they touch a device."""
    lib = _lib.load()
    p = ctypes.c_void_p(16)
    o = np.empty(4, dtype=np.int32)
    assert lib.bkm_sgd_order(-1, 1, o.ctypes.data_as(ctypes.c_void_p)) == -1
    assert lib.bkm_sgd_order(4, 1, None) == -1
    assert lib.bkm_sgd_order(2 ** 31, 1, o.ctypes.data_as(ctypes.c_void_p)) == -1
    assert lib.bkm_sgd_order(0, 1, None) == 0
    prm = _lib.SgdParams(loss=0, penalty=2, learning_rate=2, fit_intercept=1, alpha=1e-4, t0=1.0)
    # X, n, d, ldx, dtype, order, y, sw, eta, cw, P, params, w, aw, q, st, stream
    args = [p, 10, 4, 4, 1, p, p, None, None, p, 1, ctypes.byref(prm), p, None, None, p, None]
    for i, bad in ((1, -1), (2, 0), (3, 3), (10, 0), (0, None), (5, None), (6, None), (9, None), (12, None),
                   (15, None), (11, None)):
        a = list(args)
        a[i] = bad
        assert lib.bkm_sgd_block(*a) == -1, i
    a = list(args)
    a[4] = 2
    assert lib.bkm_sgd_block(*a) == -2
    for field, bad in (("loss", 8), ("penalty", 4), ("learning_rate", 0), ("learning_rate", 7)):
        q = _lib.SgdParams(loss=0, penalty=2, learning_rate=2, fit_intercept=1, alpha=1e-4, t0=1.0)
        setattr(q, field, bad)
        a = list(args)
        a[11] = ctypes.byref(q)
        assert lib.bkm_sgd_block(*a) == -1, field
    for field, bad in (("penalty", 1), ("learning_rate", 3), ("average", 1.0)):   # q, eta, aw missing
        q = _lib.SgdParams(loss=0, penalty=2, learning_rate=2, fit_intercept=1, alpha=1e-4, t0=1.0)
        setattr(q, field, bad)
        a = list(args)
        a[11] = ctypes.byref(q)
        assert lib.bkm_sgd_block(*a) == -1, field
    a = list(args)
    a[1] = 0
    assert lib.bkm_sgd_block(*a) == 0
    # crow, col, val, dtype, n, d, nnz, order, y, sw, eta, cw, P, params, w, aw, q, st, stream
    cargs = [p, p, p, 1, 10, 4, 20, p, p, None, None, p, 1, ctypes.byref(prm), p, None, None, p, None]
    for i, bad in ((4, -1), (5, 0), (6, -1), (0, None), (1, None), (2, None), (12, 0)):
        a = list(cargs)
        a[i] = bad
        assert lib.bkm_sgd_csr_block(*a) == -1, i
    a = list(cargs)
    a[3] = 5
    assert lib.bkm_sgd_csr_block(*a) == -2


# ---------------------------------------------------------------------------------------------------------------
# the unmodified reference's block-wise fit (tests/golden/ref_sgd.py), replayed
# ---------------------------------------------------------------------------------------------------------------
GOLDEN = os.path.join(ROOT, "tests", "golden")
SGD_FIXTURES = sorted(f[:-4] for f in os.listdir(GOLDEN) if f.startswith("ref_sgd_") and f.endswith(".npz"))


def replay_reference_fixture(name, to_block, exact_average=True):
    """Fit the fixture's estimator block-wise with the recorded global seed and compare with the reference's result.
    Shared with tests/test_gpu_sgd.py."""
    import json

    from dask_ml_b200 import linear_model

    with open(os.path.join(GOLDEN, "REF_SGD_MANIFEST.json")) as f:
        case = json.load(f)["cases"][name]
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        est = getattr(linear_model, case["cls"])(**case["params"])
    assert [str(w.message) for w in rec if issubclass(w.category, FutureWarning)] == case["deprecation"]
    X, y, rows = z["X"], z["y"], int(z["rows"])
    blocks = range(0, len(X), rows)
    Xc = ChunkedArray([to_block(X[i:i + rows]) for i in blocks])
    yc = ChunkedArray([y[i:i + rows] for i in blocks])
    np.random.seed(case["seed"])
    order = list(range(len(blocks)))
    np.random.shuffle(order)
    assert order == case["order"]
    np.random.seed(case["seed"])
    est.fit(Xc, yc)
    assert est.t_ == case["t"]
    if exact_average or not case["params"].get("average"):
        np.testing.assert_array_equal(est.coef_, z["coef"])
        np.testing.assert_array_equal(np.atleast_1d(est.intercept_), z["intercept"])
    else:
        np.testing.assert_allclose(est.coef_, z["coef"], rtol=1e-13, atol=1e-15)
        np.testing.assert_allclose(np.atleast_1d(est.intercept_), z["intercept"], rtol=1e-13, atol=1e-15)
    return est


@pytest.mark.parametrize("name", SGD_FIXTURES)
def test_reference_fixtures(name):
    replay_reference_fixture(name, lambda b: b)


def test_input_errors_match_sklearn():
    X, y = _data(40, 3, 2, 0)
    Xr, yr = _data(40, 3, 0, 1, regression=True)
    bad_X = [np.where(X > 1, np.nan, X), np.where(X > 1, np.inf, X)]
    for Xb in bad_X:
        for cls, ref, yy, kw in ((PartialSGDClassifier, sklm.SGDClassifier, y, {"classes": [0, 1]}),
                                 (PartialSGDRegressor, sklm.SGDRegressor, yr, {})):
            est = cls(classes=[0, 1]) if kw else cls()
            with pytest.raises(ValueError) as ours:
                est.partial_fit(Xb, yy, **kw)
            with pytest.raises(ValueError) as want:
                ref().partial_fit(Xb, yy, **kw)
            assert str(ours.value) == str(want.value).replace(ref.__name__, cls.__name__)
    for yb in (np.where(yr > 0, np.nan, yr), np.where(yr > 0, np.inf, yr), np.ones((40, 2))):
        with pytest.raises(ValueError) as ours:
            PartialSGDRegressor().partial_fit(Xr, yb)
        with pytest.raises(ValueError) as want:
            sklm.SGDRegressor().partial_fit(Xr, yb)
        assert str(ours.value) == str(want.value)


def test_non_canonical_torch_csr_is_refused():
    crow = torch.tensor([0, 2, 3], dtype=torch.int64)
    for col in ([1, 1, 0], [2, 1, 0]):              # a duplicate column, a row out of order
        A = torch.sparse_csr_tensor(crow, torch.tensor(col, dtype=torch.int64), torch.ones(3, dtype=torch.float64),
                                    size=(2, 4))
        with pytest.raises(ValueError, match="canonical CSR"):
            PartialSGDClassifier(classes=[0, 1]).partial_fit(ChunkedArray([A]), np.array([0, 1]), classes=[0, 1])


def test_predict_proba_only_for_probabilistic_losses():
    X, y = _data(60, 3, 2, 0)
    hinge = PartialSGDClassifier(classes=[0, 1]).partial_fit(X, y, classes=[0, 1])
    assert not hasattr(hinge, "predict_proba") and not hasattr(hinge, "predict_log_proba")
    assert not hasattr(PartialPassiveAggressiveClassifier(classes=[0, 1]), "predict_proba")
    est = PartialSGDClassifier(classes=[0, 1], loss="modified_huber", random_state=0).partial_fit(X, y, [0, 1])
    ref = sklm.SGDClassifier(loss="modified_huber", random_state=0).partial_fit(X, y, [0, 1])
    with np.errstate(divide="ignore"):
        np.testing.assert_allclose(est.predict_log_proba(X).compute(), ref.predict_log_proba(X), rtol=1e-12)
