"""The block-wise SGD family (PartialSGDClassifier, PartialSGDRegressor, PartialPerceptron and the PassiveAggressive
pair), executed by the H100 engine.

Mirrors dask_ml/linear_model/{stochastic_gradient,perceptron,passive_aggressive}.py on top of dask_ml/_partial.py
(reference @ 0310a90): a scikit-learn estimator whose ``fit`` calls ``partial_fit`` once per row block, in the order
``check_random_state(None).shuffle`` gives.

``partial_fit`` is scikit-learn's own (its validation, ``_check_partial_fit_first_call``, the 'balanced' and
early-stopping refusals, the passive-aggressive learning-rate choice); this module replaces the ``_partial_fit`` it
calls.  The replacement follows ``BaseSGDClassifier._partial_fit`` / ``BaseSGDRegressor._partial_fit`` of scikit-learn
1.9 step for step: the numpy draws of ``fit_binary``, ``_fit_multiclass`` and ``_fit_regressor`` and the row orders
they seed (``bkm_sgd_order``, scikit-learn's Fisher-Yates shuffle) are made on the host; the epoch of ``_plain_sgd``
over the rows of every binary problem runs in one launch of ``bkm_sgd_block`` / ``bkm_sgd_csr_block``; ``t_``,
``n_iter_``, the intercept bookkeeping (with scikit-learn's aliasing of ``intercept_``, ``_standard_intercept`` and
``_average_intercept``) and the switch between standard and averaged coefficients run on the host.  The host reads
the intercepts and the non-finite flags of a block in one copy, plus one read of the input checks per call; the coefficients stay on the device
in float64 and are copied to ``coef_`` after ``partial_fit`` and at the end of ``fit``.
"""
import math

import numpy as np
import torch
from sklearn.utils import check_random_state, compute_class_weight
from sklearn.utils.multiclass import _check_partial_fit_first_call
from sklearn.utils._available_if import available_if
from sklearn.utils.validation import _check_sample_weight, check_is_fitted

from .. import _lib
from .._partial import _PartialMixin, _accuracy, _block_data, _copy_partial_doc, _sklearn_base  # noqa: F401
from .._sparse import _SparseData
from ..chunked import ChunkedArray, _is_torch, _y_flat
from ..engine import single_process as _single_process

MAX_INT = np.iinfo(np.int32).max
SPARSE_INTERCEPT_DECAY = 0.01
_LOSS = {"hinge": 0, "log_loss": 1, "modified_huber": 2, "squared_hinge": 3, "perceptron": 0,
         "squared_error": 4, "huber": 5, "epsilon_insensitive": 6, "squared_epsilon_insensitive": 7}
_THRESHOLD = {"hinge": 1.0, "perceptron": 0.0, "squared_hinge": 1.0}
_LEARNING_RATE = {"constant": 1, "optimal": 2, "invscaling": 3, "adaptive": 4, "pa1": 5, "pa2": 6}
_PENALTY = {None: 0, "l1": 1, "l2": 2, "elasticnet": 3}
_OVERFLOW = ("Floating-point under-/overflow occurred at epoch #1. Scaling input data with StandardScaler or "
             "MinMaxScaler might help.")


def _dloss(loss, eps, y, p):
    """``cy_gradient(y, p)`` on the host (the ``optimal_init`` of ``_plain_sgd``), in the kernel's order."""
    if loss in ("hinge", "perceptron"):
        return -y if p * y <= eps else 0.0
    if loss == "log_loss":
        if p > -37:
            e = math.exp(-p)
            return ((1 - y) - y * e) / (1 + e)
        return math.exp(p) - y
    if loss == "modified_huber":
        z = p * y
        return 0.0 if z >= 1.0 else (2.0 * (1.0 - z) * -y if z >= -1.0 else -4.0 * y)
    if loss == "squared_hinge":
        z = eps - p * y
        return -2 * y * z if z > 0 else 0.0
    if loss == "squared_error":
        return p - y
    if loss == "huber":
        r = p - y
        return r if abs(r) <= eps else (eps if r >= 0 else -eps)
    if loss == "epsilon_insensitive":
        return -1.0 if y - p > eps else (1.0 if p - y > eps else 0.0)
    z = y - p
    return -2 * (z - eps) if z > eps else (2 * (-z - eps) if z < -eps else 0.0)


class _SGDState(object):
    """The float64 coefficients of the P binary problems on the device: W (standard) and AW (average, with
    ``average``)."""

    def __init__(self, be, P, d, average):
        self.W = be.zeros((P, d), torch.float64)
        self.AW = be.zeros((P, d), torch.float64) if average else None
        self.coef_is_average = False


class _PartialSGDMixin(_PartialMixin):
    """What the five estimators share: the device ``_partial_fit`` and its state."""

    _state_attr = "_sgd"
    _partial_doc = """
    This class wraps scikit-learn's {classname}.  ``fit`` passes the row blocks of X, in a random order, to
    ``partial_fit``; each ``partial_fit`` runs one epoch of scikit-learn's ``_plain_sgd`` over the block on the GPU
    (every binary problem of a one-vs-all fit in the same launch).  X may be any input the linear models take:
    device ChunkedArrays, ``host_resident`` streams, numpy, and CSR blocks from torch, scipy or HashingVectorizer.

    Differences from scikit-learn: the state is float64 on the device whatever the dtype of X (scikit-learn keeps
    float32 weights for float32 X); the gradient of ``log_loss`` calls CUDA's ``exp``, which is not glibc's, so
    log_loss coefficients agree to a tolerance rather than bit for bit (every other loss matches scikit-learn's float64
    path exactly); the averaged coefficients of ``average`` may differ in the last bits on hosts whose BLAS ``daxpy``
    does not fuse; ``decision_function``, ``predict``, ``predict_proba`` and ``score`` are computed in float64 on the
    device; scipy input is canonicalised (rows visited in sorted column order) and torch CSR blocks whose rows repeat a
    column or are not sorted are refused.
"""

    def __getstate__(self):
        state = dict(self.__dict__)
        st = state.pop("_sgd", None)
        if st is not None:
            state["_sgd_host"] = (st.W.cpu().numpy(), None if st.AW is None else st.AW.cpu().numpy(),
                                  st.coef_is_average)
        return state

    def _state(self, be, P, d):
        st = getattr(self, "_sgd", None)
        if st is None and "_sgd_host" in self.__dict__:
            W, AW, is_avg = self.__dict__.pop("_sgd_host")
            st = _SGDState(be, P, d, AW is not None)
            st.W.copy_(torch.from_numpy(W))
            if AW is not None:
                st.AW.copy_(torch.from_numpy(AW))
            st.coef_is_average = is_avg
            self._sgd = st
        return st

    def _params(self, b, alpha, loss, learning_rate):
        """The ``bkm_sgd_params`` of this call and the invscaling eta table (or None)."""
        prm = _lib.SgdParams()
        prm.loss = _LOSS[loss]
        prm.epsilon = self.epsilon if loss in ("huber", "epsilon_insensitive", "squared_epsilon_insensitive") \
            else _THRESHOLD.get(loss, 0.0)
        prm.penalty = _PENALTY[self.penalty]
        prm.learning_rate = _LEARNING_RATE[learning_rate]
        prm.fit_intercept = int(self.fit_intercept)
        prm.alpha = float(alpha)
        prm.l1_ratio = float(self._get_l1_ratio())
        prm.eta0 = float(self.eta0)
        prm.t0 = float(self.t_)
        prm.intercept_decay = SPARSE_INTERCEPT_DECAY if b.sparse else 1.0
        prm.average = float(self.average)
        if learning_rate == "optimal":
            typw = np.sqrt(1.0 / np.sqrt(alpha))
            g = _dloss(loss, prm.epsilon, 1.0, -typw)
            initial_eta0 = typw / (g if g > 1.0 else 1.0)
            prm.optimal_init = 1.0 / (initial_eta0 * alpha)
        eta = None
        if learning_rate == "invscaling":
            t0, pt, e0 = float(self.t_), float(self.power_t), float(self.eta0)
            eta = np.array([e0 / math.pow(t0 + i, pt) for i in range(b.n)], dtype=np.float64)
        return prm, eta

    def _orders(self, n, seeds):
        """int32 (P, n): the row order of each problem (scikit-learn's shuffle, or the stored order)."""
        out = np.empty((len(seeds), n), dtype=np.int32)
        for p, seed in enumerate(seeds):
            if self.shuffle:
                _lib.call("bkm_sgd_order", n, int(seed), out[p].ctypes.data)
            else:
                out[p] = np.arange(n, dtype=np.int32)
        return out

    def _run(self, b, st, Y, sw, seeds, cw, intercepts, avg_intercepts, prm, eta):
        """One launch for the P problems; returns (intercepts, average intercepts) after the epoch."""
        be = b.backend
        P = st.W.shape[0]
        order = torch.from_numpy(self._orders(b.n, seeds)).to(be.device)
        s = np.zeros((P, 4))
        s[:, 0], s[:, 1] = intercepts, avg_intercepts
        stt = torch.from_numpy(s).to(be.device)
        cwt = torch.from_numpy(np.asarray(cw, dtype=np.float64).reshape(P, 2)).to(be.device)
        swt = None if sw is None else torch.from_numpy(np.ascontiguousarray(sw, dtype=np.float64)).to(be.device)
        etat = None if eta is None else torch.from_numpy(eta).to(be.device)
        q = be.empty(tuple(st.W.shape), torch.float64) if prm.penalty in (1, 3) else None
        aw = st.AW if prm.average > 0 else None
        if b.sparse:
            be.sgd_csr_block(b.block, b.d, order, Y, swt, etat, cwt, prm, st.W, aw, q, stt)
        else:
            be.sgd_block(b.block, order, Y, swt, etat, cwt, prm, st.W, aw, q, stt)
        h = stt.cpu().numpy()                       # the one host read of the block
        if (h[:, 2] != 0).any():
            raise ValueError(_OVERFLOW)
        return h[:, 0].copy(), h[:, 1].copy()

    def _publish(self, np_dtype):
        st = self._sgd
        C = (st.AW if st.coef_is_average else st.W).cpu().numpy()
        self.coef_ = C.astype(np_dtype)
        self.intercept_ = np.asarray(self._intercept, dtype=np_dtype)

    def _sample_weight(self, sample_weight, n):
        if sample_weight is None:
            return None
        return _check_sample_weight(sample_weight, np.empty((n, 0)), dtype=np.float64,
                                    allow_all_zero_weights=self.early_stopping)

    def _finish(self, b):
        if not getattr(self, "_defer_publish", False):
            self._publish(b.np_dtype)
        else:
            self.intercept_ = np.asarray(self._intercept, dtype=b.np_dtype)

    # -- scoring on the device -------------------------------------------------------------------------------------
    def _scores(self, X):
        """(device float64 (n, P) decision values, n): X coef^T + intercept, through the projection passes."""
        check_is_fitted(self, "intercept_")
        Xd = _block_data(X)
        if Xd.d != self.n_features_in_:
            raise ValueError("X has {} features, but {} is expecting {} features as input.".format(
                Xd.d, type(self).__name__, self.n_features_in_))
        be = Xd.backend
        st = self._sgd_or_upload(be)
        C = (st.AW if st.coef_is_average else st.W).contiguous()
        b = torch.as_tensor(np.asarray(self._intercept, dtype=np.float64)).to(be.device)
        outs = []
        if isinstance(Xd, _SparseData):
            CT = C.t().contiguous()
            for blk in Xd.blocks:
                o = be.empty((int(blk[3]), C.shape[0]), torch.float64)
                if int(blk[3]):
                    be.csr_panel_chunk(blk, Xd.d, CT, out=o)
                outs.append(o + b)
        else:
            for x in Xd.chunks:
                o = be.empty((int(x.shape[0]), C.shape[0]), torch.float64)
                if int(x.shape[0]):
                    be.project_chunk(x, None, C, out=o)
                outs.append(o + b)
        return Xd, outs

    def _sgd_or_upload(self, be):
        st = getattr(self, "_sgd", None)
        if st is not None:
            return st
        st = self._state(be, *np.atleast_2d(self.coef_).shape)
        if st is None:                                   # coefficients set by hand
            C = np.atleast_2d(np.asarray(self.coef_, dtype=np.float64))
            st = _SGDState(be, C.shape[0], C.shape[1], False)
            st.W.copy_(torch.from_numpy(C))
            self._sgd = st
        return st


class _PartialSGDClassifierMixin(_PartialSGDMixin):
    _init_kwargs = ["classes"]
    _fit_kwargs = ["classes"]

    def _partial_fit(self, X, y, alpha, loss, learning_rate, max_iter, classes, sample_weight, coef_init,
                     intercept_init):
        """``BaseSGDClassifier._partial_fit`` with one epoch (``max_iter`` = 1) of every binary problem on the
        device."""
        _single_process(type(self).__name__)
        first_call = not hasattr(self, "classes_")
        b = self._batch(X, y)
        self._check_features(b, first_call)
        _check_partial_fit_first_call(self, classes)
        n_classes = self.classes_.shape[0]
        yf = b.y
        y_labels = torch.unique(yf).cpu().numpy() if _is_torch(yf) else yf
        self._expanded_class_weight = compute_class_weight(self.class_weight, classes=self.classes_, y=y_labels)
        sw = self._sample_weight(sample_weight, b.n)
        be = b.backend
        P = 1 if n_classes == 2 else n_classes
        st = self._state(be, P, b.d)
        if st is None:                                  # _allocate_parameter_mem
            st = self._sgd = _SGDState(be, P, b.d, self.average > 0)
            self._intercept = np.zeros(P)
            if self.average > 0:
                self._standard_intercept = self._intercept
                self._average_intercept = np.zeros(P)
        if n_classes < 2:
            raise ValueError("The number of classes has to be greater than one; got %d class" % n_classes)
        if not hasattr(self, "t_"):
            self.t_ = 1.0
        neg = 0.0 if loss == "log_loss" else -1.0
        pos_classes = self.classes_[1:] if P == 1 else self.classes_
        Y = self._labels(b, yf, pos_classes, neg)
        prm, eta = self._params(b, alpha, loss, learning_rate)
        avg = self.average > 0
        std_int = self._standard_intercept if avg else self._intercept
        if P == 1:                                      # _fit_binary
            rs = check_random_state(self.random_state)
            rs.randint(1, MAX_INT)
            seeds = [rs.randint(MAX_INT)]
            cw = [self._expanded_class_weight[1], self._expanded_class_weight[0]]
        else:                                           # _fit_multiclass
            class_seeds = check_random_state(self.random_state).randint(MAX_INT, size=len(self.classes_))
            seeds = []
            for s in class_seeds:
                rs = check_random_state(s)
                rs.randint(1, MAX_INT)
                seeds.append(rs.randint(MAX_INT))
            cw = [[self._expanded_class_weight[i], 1.0] for i in range(P)]
        a_in = self._average_intercept if avg else np.zeros(P)
        ints, avg_ints = self._run(b, st, Y, sw, seeds, cw, std_int.copy(), a_in.copy(), prm, eta)
        if avg:
            self._average_intercept[:] = avg_ints
        self.t_ += b.n
        self.n_iter_ = 1
        if P == 1:
            if avg:
                if self.average <= self.t_ - 1:
                    st.coef_is_average = True
                    self._intercept = self._average_intercept
                else:
                    st.coef_is_average = False
                    self._standard_intercept = np.atleast_1d(ints[0]).astype(np.float64)
                    self._intercept = self._standard_intercept
            else:
                self._intercept = np.atleast_1d(ints[0]).astype(np.float64)
        else:
            self._intercept[:] = ints                   # into whichever array intercept_ is, as scikit-learn does
            if avg:
                if self.average <= self.t_ - 1.0:
                    st.coef_is_average = True
                    self._intercept = self._average_intercept
                else:
                    st.coef_is_average = False
                    self._standard_intercept = self._intercept
        self._finish(b)
        return self

    def _labels(self, b, yf, pos_classes, neg):
        """float64 (P, n) on the device: 1 where y is the problem's positive class, ``neg`` elsewhere."""
        be = b.backend
        if _is_torch(yf) and np.asarray(self.classes_).dtype.kind in "biuf" and yf.dtype != torch.bool:
            yd = yf.to(device=be.device, dtype=torch.float64)
            cls = torch.as_tensor(np.asarray(pos_classes, dtype=np.float64)).to(be.device)
            one = torch.ones((), dtype=torch.float64, device=be.device)
            return torch.where(yd[None, :] == cls[:, None], one, one * neg).contiguous()
        yh = yf.cpu().numpy() if _is_torch(yf) else np.asarray(yf)
        Y = np.where(yh[None, :] == np.asarray(pos_classes)[:, None], 1.0, neg)
        return torch.from_numpy(np.ascontiguousarray(Y, dtype=np.float64)).to(be.device)

    def decision_function(self, X):
        """X coef^T + intercept on the device: a float64 ChunkedArray, (n,) for two classes, (n, K) otherwise."""
        _, outs = self._scores(X)
        if len(self.classes_) == 2:
            outs = [o[:, 0] for o in outs]
        return ChunkedArray(outs)

    def _labels_of(self, outs):
        if len(self.classes_) == 2:
            return [(o[:, 0] > 0).to(torch.int64) for o in outs]
        return [o.argmax(dim=1) for o in outs]

    def predict(self, X):
        """The class of largest decision value (scikit-learn's rule), on the device for numeric classes."""
        _, outs = self._scores(X)
        idx = self._labels_of(outs)
        cls = np.asarray(self.classes_)
        if cls.dtype.kind in "biuf":
            ct = torch.as_tensor(cls).to(outs[0].device if outs else "cpu")
            return ChunkedArray([ct[i] for i in idx])
        return np.concatenate([cls[i.cpu().numpy()] for i in idx])

    def _check_proba(self):
        # scikit-learn's SGDClassifier._check_proba: the method exists for log_loss and modified_huber only
        if self.loss not in ("log_loss", "modified_huber"):
            raise AttributeError("probability estimates are not available for loss=%r" % self.loss)
        return True

    @available_if(_check_proba)
    def predict_proba(self, X):
        """scikit-learn's probability estimates (log_loss, modified_huber), in float64 on the device."""
        check_is_fitted(self, "intercept_")
        _, outs = self._scores(X)
        res = []
        for o in outs:
            if self.loss == "log_loss":
                p = torch.sigmoid(o)
                if len(self.classes_) == 2:
                    p = torch.cat([1 - p, p], dim=1)
                else:
                    s = p.sum(dim=1, keepdim=True)
                    p = torch.where(s == 0, torch.full_like(p, 1.0 / p.shape[1]), p / torch.where(s == 0, 1.0, s))
            else:
                if len(self.classes_) == 2:
                    p1 = (o[:, 0].clamp(-1, 1) + 1) / 2
                    p = torch.stack([1 - p1, p1], dim=1)
                else:
                    p = (o.clamp(-1, 1) + 1) / 2
                    s = p.sum(dim=1, keepdim=True)
                    k = p.shape[1]
                    p = torch.where(s == 0, torch.full_like(p, 1.0 / k), p / torch.where(s == 0, 1.0, s))
            res.append(p)
        return ChunkedArray(res)

    @available_if(_check_proba)
    def predict_log_proba(self, X):
        """The log of ``predict_proba``, in float64 on the device."""
        return ChunkedArray([torch.log(p) for p in self.predict_proba(X).blocks])

    def score(self, X, y, sample_weight=None):
        """Mean accuracy of ``predict(X)``, computed in float64."""
        return _accuracy(self, X, y, sample_weight)


class _PartialSGDRegressorMixin(_PartialSGDMixin):

    def _partial_fit(self, X, y, alpha, loss, learning_rate, max_iter, sample_weight, coef_init, intercept_init):
        """``BaseSGDRegressor._partial_fit`` / ``_fit_regressor`` with the epoch on the device."""
        _single_process(type(self).__name__)
        st0 = getattr(self, "_sgd", None)
        first_call = st0 is None and "_sgd_host" not in self.__dict__
        b = self._batch(X, y)
        self._check_features(b, first_call)
        sw = self._sample_weight(sample_weight, b.n)
        be = b.backend
        st = self._state(be, 1, b.d)
        if st is None:
            st = self._sgd = _SGDState(be, 1, b.d, self.average > 0)
            self._intercept = np.zeros(1)
            if self.average > 0:
                self._standard_intercept = self._intercept
                self._average_intercept = np.zeros(1)
        if not hasattr(self, "t_"):
            self.t_ = 1.0
        yf = b.y
        if _is_torch(yf):
            Y = yf.to(device=be.device, dtype=torch.float64).reshape(1, -1).contiguous()
        else:
            Y = torch.from_numpy(np.ascontiguousarray(np.asarray(yf, dtype=np.float64)).reshape(1, -1)).to(be.device)
        prm, eta = self._params(b, alpha, loss, learning_rate)
        rs = check_random_state(self.random_state)
        seed = rs.randint(0, MAX_INT)
        rs.randint(1, MAX_INT)
        avg = self.average > 0
        i_in = self._standard_intercept if avg else self._intercept
        a_in = self._average_intercept if avg else np.zeros(1)
        ints, avg_ints = self._run(b, st, Y, sw, [seed], [1.0, 1.0], i_in.copy(), a_in.copy(), prm, eta)
        self.n_iter_ = 1
        self.t_ += b.n
        if avg:
            self._average_intercept = np.atleast_1d(avg_ints[0]).astype(np.float64)
            self._standard_intercept = np.atleast_1d(ints[0]).astype(np.float64)
            if self.average <= self.t_ - 1.0:
                st.coef_is_average = True
                self._intercept = np.atleast_1d(avg_ints[0]).astype(np.float64)
            else:
                st.coef_is_average = False
                self._intercept = np.atleast_1d(ints[0]).astype(np.float64)
        else:
            self._intercept = np.atleast_1d(ints[0]).astype(np.float64)
        self._finish(b)
        return self

    def _publish(self, np_dtype):
        super(_PartialSGDRegressorMixin, self)._publish(np_dtype)
        self.coef_ = self.coef_.ravel()

    def predict(self, X):
        """X coef + intercept on the device: a float64 ChunkedArray."""
        _, outs = self._scores(X)
        return ChunkedArray([o[:, 0] for o in outs])

    def score(self, X, y, sample_weight=None):
        """R^2 of ``predict(X)``, computed in float64."""
        if sample_weight is not None:
            raise NotImplementedError("sample_weight is not supported by score")
        p = torch.cat(list(self.predict(X).blocks))
        yf = _y_flat(y, type(self).__name__ + ".score")
        yt = yf.to(p.device, torch.float64) if _is_torch(yf) else torch.as_tensor(
            np.asarray(yf, dtype=np.float64)).to(p.device)
        ss_res = ((yt - p) ** 2).sum()
        ss_tot = ((yt - yt.mean()) ** 2).sum()
        return float(1.0 - ss_res / ss_tot) if float(ss_tot) != 0 else (1.0 if float(ss_res) == 0 else 0.0)
