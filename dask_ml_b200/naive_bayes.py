"""GaussianNB with the dask_ml.naive_bayes.GaussianNB API, executed by the H100 engine.

Mirrors dask_ml/naive_bayes.py:10-122 (reference @ 0310a90).  The reference builds one boolean mask per class
(``X[y == c]``, a mean and a variance each) and, for ``predict``, K stacked elementwise passes over X.  Here a fit reads
X twice and a predict call once, whatever K is:

    pass 1 (bkm_class_moments_chunk, float64):  S_c = sum_{y_i = c} x_i,  n_c = #{y_i = c}     one all-reduce of
                                                                                                [K*d sums | K counts | n]
    host:                                       theta_c = S_c / n_c
    pass 2 (bkm_class_moments_chunk, float64):  Q_c = sum_{y_i = c} (x_i - theta_c)^2            one all-reduce of [K*d]
    host:                                       sigma_c = Q_c / n_c,  class_prior_ = n_c / n
    predict (bkm_nb_jll_chunk):                 jll_ic = log prior_c - 1/2 sum_j log(2 pi sigma_cj)
                                                         - 1/2 sum_j (x_ij - theta_cj)^2 / sigma_cj
                                                labels = argmax_c jll_ic, or jll - logsumexp(jll) per row

The centred second pass keeps the variance of data far from the origin (a one-pass sum of squares would lose it).
Attributes are computed in float64 and cast to the dtype of X (float32 for bf16 rows), as the reference's
``theta_`` / ``sigma_`` have X's dtype; ``class_count_`` and ``class_prior_`` are float64.  Predictions use the
attributes as stored.

The reference's quirks are kept (DESIGN.md A21): ``priors`` is ignored; with ``classes=`` rows whose label is not in
``classes`` enter no sum but still count in n; an empty class has NaN ``theta_`` / ``sigma_``; there is no variance
smoothing, so a class with a zero variance (every single-row class) has a NaN log-likelihood on every row, which
``predict`` picks as ``np.argmax`` does (the first NaN) and which makes the row's log-probabilities NaN throughout.

PartialMultinomialNB and PartialBernoulliNB mirror naive_bayes.py:125-134 on dask_ml/_partial.py: scikit-learn's
MultinomialNB / BernoulliNB whose ``fit`` calls ``partial_fit`` once per row block (``_partial.py``).  ``partial_fit``
follows ``_BaseDiscreteNB.partial_fit`` of scikit-learn 1.9 step by step with the counts on the device:

    count (bkm_class_counts_chunk, float64; CSR: bkm_csr_transpose_chunk + bkm_csc_class_counts_chunk):
          feature_count_ (+)= sum_{y_i = c} w_i f(x_i),  class_count_ (+)= sum_{y_i = c} w_i     f = x, or x > binarize
    host: scikit-learn's own _check_alpha, _update_feature_log_prob and _update_class_log_prior on the published counts
    predict (bkm_nb_linear_jll_chunk on the fp64 tensor cores; CSR: bkm_nb_csr_jll_chunk):
          jll = f(x) W^T + b,  MultinomialNB: W = feature_log_prob_, b = class_log_prior_;
          BernoulliNB: neg = log(1 - exp(feature_log_prob_)), W = feature_log_prob_ - neg, b = class_log_prior_ + sum neg
          labels = argmax_c jll, or jll - logsumexp(jll) (and its exp) per row

Counts of integer data (and of dyadic weights) are exact, so the log-probabilities are scikit-learn's bit for bit.
"""
import types

import numpy as np
import torch
from sklearn import naive_bayes as _naive_bayes
from sklearn.base import BaseEstimator, _fit_context
from sklearn.exceptions import NotFittedError
from sklearn.utils.multiclass import _check_partial_fit_first_call
from sklearn.utils.validation import _check_sample_weight, check_is_fitted

from . import _lib
from ._partial import _PartialMixin, _accuracy, _block_data, _copy_partial_doc
from ._sparse import _SparseData, check_label_sum_classes
from .chunked import ChunkedArray, _is_torch, _y_flat, block_to_numpy
from .decomposition.pca import _device_data
from .engine import single_process as _single_process


def _device_classes(classes):
    """classes as a device-comparable torch tensor (CPU), or None when they are not numeric."""
    classes = np.asarray(classes)
    if classes.dtype.kind not in "biuf":
        return None
    try:
        return torch.as_tensor(classes)
    except TypeError:                                   # numpy dtypes torch has no counterpart for
        return None


def _local_unique(yf):
    if _is_torch(yf):
        return torch.unique(yf).cpu().numpy()
    return np.unique(yf)


def class_indices(yf, classes, X):
    """int32 class index of every local row (-1 for a label not in ``classes``), split to the row boundaries of X's
    chunks (``DeviceData.chunk_offsets``) and resident on the device.  Numeric labels are mapped with a device
    ``searchsorted``; other labels (strings, objects) on the host."""
    be = X.backend
    classes = np.asarray(classes)
    K = len(classes)
    order = np.argsort(classes, kind="stable")
    srt = classes[order]
    cdev = _device_classes(srt)
    if cdev is not None and not (isinstance(yf, np.ndarray) and yf.dtype.kind not in "biuf"):
        t = yf if _is_torch(yf) else torch.as_tensor(np.ascontiguousarray(yf))
        t = t.to(be.device)
        wide = torch.float64 if (cdev.is_floating_point() or t.is_floating_point()) else torch.int64
        if cdev.dtype == torch.bool and t.dtype == torch.bool:
            wide = torch.int64
        t = t.to(wide)
        s = cdev.to(device=be.device, dtype=wide)
        pos = torch.searchsorted(s, t).clamp_(max=K - 1)
        hit = s[pos] == t
        cls = torch.where(hit, torch.as_tensor(order, device=be.device)[pos], torch.full_like(pos, -1)).to(torch.int32)
    else:
        h = np.asarray(block_to_numpy(yf) if _is_torch(yf) else yf)
        pos = np.clip(np.searchsorted(srt, h), 0, K - 1)
        hit = srt[pos] == h
        cls = torch.as_tensor(np.where(hit, order[pos], -1).astype(np.int32)).to(be.device)
    off = X.chunk_offsets
    return [cls[int(off[i]):int(off[i + 1])].contiguous() for i in range(len(off) - 1)]


def _predict_params(theta, sigma, prior):
    """(theta, 1 / sigma, logc) in float64 for the predict pass.  A class whose log-likelihood the reference's formula
    makes NaN on every row (NaN or zero variance, empty class) gets logc = NaN and zero theta / w, so the kernel never
    sees a zero variance."""
    theta = np.asarray(theta, dtype=np.float64)
    sigma = np.asarray(sigma, dtype=np.float64)
    prior = np.asarray(prior, dtype=np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        w = 1.0 / sigma
        logc = np.log(prior) - 0.5 * np.sum(np.log(2.0 * np.pi * sigma), axis=1)
    bad = ~(np.isfinite(theta).all(1) & np.isfinite(w).all(1) & (sigma > 0).all(1) & np.isfinite(logc))
    theta = np.where(bad[:, None], 0.0, theta)
    w = np.where(bad[:, None], 0.0, w)
    logc = np.where(bad, np.nan, logc)
    return np.ascontiguousarray(theta), np.ascontiguousarray(w), np.ascontiguousarray(logc)


class GaussianNB(BaseEstimator):
    """Gaussian naive Bayes (API of dask_ml.naive_bayes.GaussianNB, naive_bayes.py:10-122).

    Parameters
    ----------
    priors : ignored (as in the reference: the priors are always the class frequencies)
    classes : array-like or None
        The labels to model, in this order.  None: the sorted labels of y.  Rows whose label is not in ``classes``
        enter no per-class sum but still count in the number of rows that divides the class counts.

    Attributes
    ----------
    classes_ : numpy array
    theta_, sigma_ : numpy (n_classes, n_features), dtype of X (float32 for bf16 rows)
    class_count_, class_prior_ : numpy (n_classes,) float64
    """

    def __init__(self, priors=None, classes=None):
        self.priors = priors
        self.classes = classes
        self.classes_ = classes
        self.class_prior_ = None
        self.class_count_ = None
        self.theta_ = None
        self.sigma_ = None

    def fit(self, X, y=None):
        X = _device_data(X)
        be, comm, d = X.backend, X.comm, X.d
        yf = _y_flat(y)
        if int(yf.shape[0]) != X.n_local:
            raise ValueError("Found input variables with inconsistent numbers of samples: [%d, %d]"
                             % (X.n_local, int(yf.shape[0])))
        if self.classes is None:
            parts = comm.allgather_obj(_local_unique(yf))
            nonempty = [p for p in parts if len(p)]
            classes = np.unique(np.concatenate(nonempty)) if nonempty else parts[0]
        else:
            classes = np.asarray(self.classes)
            if classes.ndim != 1:
                classes = classes.reshape(-1)
            if len(np.unique(classes)) != len(classes):
                raise ValueError("classes must not contain duplicates")
        K = len(classes)
        if K == 0:
            raise ValueError("GaussianNB.fit needs at least one class")
        cls = class_indices(yf, classes, X)

        # pass 1: per-class sums and counts, one all-reduce of [K*d sums | K counts | n]
        red = be.zeros((K * d + K + 1,), torch.float64)
        sums, counts = red[: K * d].view(K, d), red[K * d: K * d + K]
        for i, x in enumerate(X.chunks):
            be.class_moments_chunk(x, cls[i], K, sums, counts, first=i == 0)
        red[-1] = float(X.n_local)
        comm.allreduce_sum_(red)
        h = red.cpu().numpy()
        S, cnt, N = h[: K * d].reshape(K, d), h[K * d: K * d + K].copy(), h[-1]
        with np.errstate(divide="ignore", invalid="ignore"):
            theta = S / cnt[:, None]

        # pass 2: per-class centred squares, one all-reduce of [K*d]
        th_dev = torch.as_tensor(np.ascontiguousarray(np.where(np.isfinite(theta), theta, 0.0))).to(be.device)
        sq = be.zeros((K * d,), torch.float64)
        for i, x in enumerate(X.chunks):
            be.class_moments_chunk(x, cls[i], K, sq.view(K, d), theta=th_dev, first=i == 0)
        comm.allreduce_sum_(sq)
        with np.errstate(divide="ignore", invalid="ignore"):
            sigma = sq.cpu().numpy().reshape(K, d) / cnt[:, None]
            prior = cnt / N

        dt = X.np_dtype
        self.classes_ = classes
        self.theta_ = theta.astype(dt)
        self.sigma_ = sigma.astype(dt)
        self.class_count_ = cnt
        self.class_prior_ = prior
        return self

    # -- predict ---------------------------------------------------------------------------------------------------
    def _check_fitted(self):
        if self.theta_ is None or self.sigma_ is None or self.class_prior_ is None:
            raise NotFittedError("This GaussianNB instance is not fitted yet. Call 'fit' with appropriate arguments "
                                 "before using this estimator.")

    def _jll_pass(self, X, labels, log_proba, exp_out=False):
        self._check_fitted()
        X = _device_data(X)
        be = X.backend
        theta, w, logc = _predict_params(self.theta_, self.sigma_, self.class_prior_)
        K = theta.shape[0]
        dev = [torch.as_tensor(a).to(be.device) for a in (theta, w, logc)]
        labs, outs = [], []
        for x in X.chunks:
            n = int(x.shape[0])
            lab = be.empty((n,), torch.int32) if labels else None
            out = be.empty((n, K), torch.float64) if log_proba else None
            if n:
                be.nb_jll_chunk(x, dev[0], dev[1], dev[2], labels=lab, out=out, exp_out=exp_out)
            labs.append(lab)
            outs.append(out)
        return labs, outs

    def predict(self, X):
        """The class of largest joint log-likelihood per row (values of ``classes_``): a ChunkedArray, device-resident
        when ``classes_`` is numeric."""
        labs, _ = self._jll_pass(X, True, False)
        classes = np.asarray(self.classes_)
        cdev = _device_classes(classes)
        if cdev is not None:
            cdev = cdev.to(labs[0].device)
            return ChunkedArray([cdev[lab.long()] for lab in labs])
        return ChunkedArray([classes[lab.cpu().numpy()] for lab in labs])

    def predict_log_proba(self, X):
        """(n, n_classes) float64 log-probabilities, jll - logsumexp(jll) per row: a device-resident ChunkedArray."""
        _, outs = self._jll_pass(X, False, True)
        return ChunkedArray(outs)

    def predict_proba(self, X):
        """(n, n_classes) float64 probabilities, exp of ``predict_log_proba``: a device-resident ChunkedArray."""
        _, outs = self._jll_pass(X, False, True, exp_out=True)
        return ChunkedArray(outs)


# ---------------------------------------------------------------------------------------------------------------------
# PartialMultinomialNB / PartialBernoulliNB
# ---------------------------------------------------------------------------------------------------------------------
class _CountState(object):
    """The float64 counts on the device: FC (K, d) = feature_count_, CC (K,) = class_count_."""

    def __init__(self, be, K, d):
        self.FC = be.zeros((K, d), torch.float64)
        self.CC = be.zeros((K,), torch.float64)


class _PartialDiscreteNBMixin(_PartialMixin):
    """What the two estimators share: the device ``partial_fit`` (counts) and the device predict methods."""

    _init_kwargs = ["classes"]
    _fit_kwargs = ["classes"]
    _state_attr = "_nb"
    _partial_doc = """
    This class wraps scikit-learn's {classname}.  ``fit`` passes the row blocks of X, in a random order, to
    ``partial_fit``; each ``partial_fit`` adds the block's weighted per-class feature counts on the GPU, in float64,
    and then runs scikit-learn's own smoothing and prior updates on the host.  X may be any input the linear models
    take: device ChunkedArrays, ``host_resident`` streams, numpy, and CSR blocks from torch, scipy or
    HashingVectorizer.

    ``predict``, ``predict_proba``, ``predict_log_proba``, ``predict_joint_log_proba`` and ``score`` run on the GPU in
    float64 and return device ChunkedArrays (string classes come back from ``predict`` as a host array).  Counts of
    integer data with integer or dyadic weights are scikit-learn's bit for bit, hence so are ``feature_log_prob_`` and
    ``class_log_prior_``; the joint log-likelihoods differ from numpy's BLAS product by the order of the sums only.
    A CSR row reads its stored entries only, as scipy's product does.
"""

    def _binarize(self):
        """The threshold of f(x) = x > t, or None (f the identity)."""
        return None

    def __getstate__(self):
        state = dict(self.__dict__)
        state.pop("_nb_w", None)
        st = state.pop("_nb", None)
        if st is not None:
            state["_nb_host"] = (st.FC.cpu().numpy(), st.CC.cpu().numpy())
        return state

    def _state(self, be):
        st = getattr(self, "_nb", None)
        if st is None and "_nb_host" in self.__dict__:
            FC, CC = self.__dict__.pop("_nb_host")
            st = _CountState(be, *FC.shape)
            st.FC.copy_(torch.from_numpy(FC))
            st.CC.copy_(torch.from_numpy(CC))
            self._nb = st
        return st

    def _threshold(self, np_dtype, sparse):
        """The binarising threshold as numpy compares it with X of ``np_dtype`` (a Python number is rounded to X's
        dtype), with scikit-learn's refusal of a negative threshold for sparse X; None without binarising."""
        t = self._binarize()
        if t is None:
            return None
        if sparse and t < 0:
            raise ValueError("Cannot binarize a sparse matrix with threshold < 0")
        return float(np.asarray(t, dtype=np.result_type(np.dtype(np_dtype), t)))

    def _class_index(self, b):
        """int32 (n,) class index of every row on the device: -1 for a label not in ``classes_``, as label_binarize
        leaves it out; with one class every row counts (scikit-learn's ``np.ones_like(Y)``); with two classes and at
        most two distinct labels every row that is not the second class counts for the first (label_binarize's binary
        column)."""
        K = len(self.classes_)
        if K == 1:
            return torch.zeros(b.n, dtype=torch.int32, device=b.backend.device)
        cls = class_indices(b.y, self.classes_, types.SimpleNamespace(backend=b.backend, chunk_offsets=[0, b.n]))[0]
        if K == 2 and len(_local_unique(b.y)) <= 2:
            cls = (cls == 1).to(torch.int32)
        return cls

    @_fit_context(prefer_skip_nested_validation=True)
    def partial_fit(self, X, y, classes=None, sample_weight=None):
        """``_BaseDiscreteNB.partial_fit`` with the counts of the block added on the device.  ``fit`` defers the copy
        of the counts and the host updates to its end."""
        _single_process(type(self).__name__)
        first_call = not hasattr(self, "classes_")
        b = self._batch(X, y)
        thr = self._threshold(b.np_dtype, b.sparse)
        self._check_features(b, first_call)
        if b.sparse and (classes is not None or not first_call):
            check_label_sum_classes(len(np.unique(classes)) if classes is not None else len(self.classes_), "classes")
        be = b.backend
        if _check_partial_fit_first_call(self, classes):
            self._nb = _CountState(be, len(classes), b.d)
            self.__dict__.pop("_nb_host", None)
        st = self._state(be)
        K = len(self.classes_)
        cls = self._class_index(b)
        w = None
        if sample_weight is not None:
            sw = _check_sample_weight(sample_weight, np.empty((b.n, 0), dtype=b.np_dtype))
            w = torch.from_numpy(np.ascontiguousarray(sw, dtype=np.float64)).to(be.device)
        if self._check_negative and b.negative:
            raise ValueError("Negative values in data passed to MultinomialNB (input X)")
        if b.sparse:
            csc = be.csr_transpose_chunk(b.block, b.d)
            fcT = be.empty((b.d, K), torch.float64)
            be.csc_class_counts_chunk(csc, b.d, cls, K, fcT, w=w, binarize=thr, first=True)
            st.FC += fcT.t()
            col = (w if w is not None else torch.ones(b.n, dtype=torch.float64, device=be.device)).view(b.n, 1)
            cc = be.empty((K, 1), torch.float64)
            be.class_counts_chunk(col, cls, K, cc, be.empty((K,), torch.float64), first=True)
            st.CC += cc[:, 0]
        else:
            be.class_counts_chunk(b.block, cls, K, st.FC, st.CC, w=w, binarize=thr)
        if not getattr(self, "_defer_publish", False):
            self._publish(b.np_dtype)
        return self

    def _publish(self, np_dtype):
        """The counts to ``feature_count_`` / ``class_count_``, then scikit-learn's own host updates."""
        st = self._nb
        self.feature_count_ = st.FC.cpu().numpy()
        self.class_count_ = st.CC.cpu().numpy()
        alpha = self._check_alpha()
        self._update_feature_log_prob(alpha)
        self._update_class_log_prior(class_prior=self.class_prior)

    # -- predict on the device -----------------------------------------------------------------------------------------
    def _linear(self, flp, prior):
        """(W (K, d), b (K,)) float64 of jll = f(X) W^T + b, with scikit-learn's expressions."""
        return flp, prior

    def _device_weights(self, be):
        """(W, W^T, b) on the device, uploaded once per pair of attribute arrays (the attributes as stored)."""
        flp, prior = self.feature_log_prob_, self.class_log_prior_
        c = getattr(self, "_nb_w", None)
        if c is None or c[0] is not flp or c[1] is not prior:
            W, b = self._linear(np.asarray(flp, dtype=np.float64), np.asarray(prior, dtype=np.float64))
            Wd = torch.from_numpy(np.ascontiguousarray(W)).to(be.device)
            c = (flp, prior, Wd, Wd.t().contiguous(), torch.from_numpy(np.ascontiguousarray(b)).to(be.device))
            self._nb_w = c
        return c[2:]

    def _jll_pass(self, X, labels, out_mode=None):
        """Per block: int32 labels (with ``labels``) and / or the (n, K) float64 output of ``out_mode``."""
        check_is_fitted(self, "feature_log_prob_")
        Xd = _block_data(X)
        if Xd.d != self.n_features_in_:
            raise ValueError("X has {} features, but {} is expecting {} features as input.".format(
                Xd.d, type(self).__name__, self.n_features_in_))
        sparse = isinstance(Xd, _SparseData)
        thr = self._threshold(Xd.np_dtype, sparse)
        be = Xd.backend
        W, WT, bias = self._device_weights(be)
        K = int(W.shape[0])
        labs, outs = [], []
        for blk in (Xd.blocks if sparse else Xd.chunks):
            n = int(blk[3]) if sparse else int(blk.shape[0])
            lab = be.empty((n,), torch.int32) if labels else None
            out = be.empty((n, K), torch.float64) if out_mode is not None else None
            if n and sparse:
                be.nb_csr_jll_chunk(blk, Xd.d, WT, bias, labels=lab, out=out, out_mode=out_mode or 0, binarize=thr)
            elif n:
                be.nb_linear_jll_chunk(blk, W, bias, labels=lab, out=out, out_mode=out_mode or 0, binarize=thr)
            labs.append(lab)
            outs.append(out)
        return labs, outs

    def predict(self, X):
        """The class of largest joint log-likelihood per row: a device ChunkedArray of ``classes_`` values when they
        are numeric, else a host array."""
        labs, _ = self._jll_pass(X, True)
        classes = np.asarray(self.classes_)
        cdev = _device_classes(classes)
        if cdev is not None:
            cdev = cdev.to(labs[0].device if labs else "cpu")
            return ChunkedArray([cdev[lab.long()] for lab in labs])
        return np.concatenate([classes[lab.cpu().numpy()] for lab in labs])

    def predict_joint_log_proba(self, X):
        """(n, n_classes) float64 joint log-likelihoods: a device ChunkedArray."""
        return ChunkedArray(self._jll_pass(X, False, _lib.NB_JLL)[1])

    def predict_log_proba(self, X):
        """(n, n_classes) float64 log-probabilities, jll - logsumexp(jll) per row: a device ChunkedArray."""
        return ChunkedArray(self._jll_pass(X, False, _lib.NB_LOG_PROBA)[1])

    def predict_proba(self, X):
        """(n, n_classes) float64 probabilities, exp of ``predict_log_proba``: a device ChunkedArray."""
        return ChunkedArray(self._jll_pass(X, False, _lib.NB_PROBA)[1])

    def score(self, X, y, sample_weight=None):
        """Mean accuracy of ``predict(X)``, computed in float64 on the device."""
        return _accuracy(self, X, y, sample_weight)


@_copy_partial_doc
class PartialMultinomialNB(_PartialDiscreteNBMixin, _naive_bayes.MultinomialNB):
    _check_negative = True


@_copy_partial_doc
class PartialBernoulliNB(_PartialDiscreteNBMixin, _naive_bayes.BernoulliNB):

    def _binarize(self):
        return self.binarize

    def _linear(self, flp, prior):
        neg = np.log(1 - np.exp(flp))
        return flp - neg, prior + neg.sum(axis=1)
