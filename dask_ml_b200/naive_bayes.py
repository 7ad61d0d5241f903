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
"""
import numpy as np
import torch
from sklearn.base import BaseEstimator
from sklearn.exceptions import NotFittedError

from .chunked import ChunkedArray, _is_torch, as_chunked, block_to_numpy, is_dask_array
from .decomposition.pca import _device_data


def _y_flat(y, who="GaussianNB.fit"):
    """y (numpy, torch on any device, ChunkedArray or dask array, any chunking) -> one flat numpy array or tensor."""
    if y is None:
        raise ValueError("%s needs the labels y; got None" % who)
    if isinstance(y, ChunkedArray):
        blocks = y.blocks
    elif is_dask_array(y):
        blocks = as_chunked(y).blocks
    else:
        blocks = [y]
    if all(_is_torch(b) for b in blocks):
        flat = [b.detach().reshape(-1) for b in blocks]
        return flat[0] if len(flat) == 1 else torch.cat([f.to(flat[0].device) for f in flat])
    flat = [np.asarray(block_to_numpy(b) if _is_torch(b) else b).reshape(-1) for b in blocks]
    return flat[0] if len(flat) == 1 else np.concatenate(flat)


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
