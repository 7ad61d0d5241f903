"""SimpleImputer with the dask_ml.impute API, executed by the H100 engine.

Mirrors dask_ml/impute.py (reference @ 0310a90), which subclasses scikit-learn's SimpleImputer and hands numpy input to
it.  Here every input kind (ndarray, torch, ChunkedArray, dask-like arrays, ``host_resident``) goes through the engine's
one intake and gets what scikit-learn gives for numpy input, for all four strategies and any numeric or NaN
``missing_values``.  The passes (DESIGN.md, "The passes of SimpleImputer"):

    fit, every strategy (bkm_impute_stats_chunk, one read of X, float64): per column the missing, NaN and inf counts
                    and S = sum (x - s) over the non-missing finite x, s a shift shared by every rank     one all-reduce
    mean            s + S / m over the m non-missing values
    median          the order statistics a[m // 2] (odd m) or a[m / 2 - 1], a[m / 2] of the non-missing values by the
                    exact radix selection of QuantileTransformer (bkm_quantile_hist_chunk, or its masked variant for a
                    numeric missing value), then np.ma.median's (lo + hi) / 2 in X's dtype
    most_frequent   per column a hash table of value counts (bkm_mode_count_chunk) and the entry of largest count,
                    smallest value on ties (bkm_mode_best); with several ranks the tables are compacted, gathered by the
                    sum all-reduce and merged on every rank
    transform / inverse_transform (bkm_impute_chunk): the fill, the dropped columns and the indicator columns in one read
                    and one write

Documented deviations from scikit-learn (DESIGN.md): the mean is a float64 sum about a shift (scikit-learn sums float32
columns in float32); integer input is computed as float32 / float64, so outputs are float; a zero mode is +0.0; a
callable ``strategy`` raises NotImplementedError; outputs are device-resident ChunkedArrays in X's dtype (float32 for
bf16 rows), also for ``inverse_transform``.
"""
import numbers
import warnings

import numpy as np
import sklearn.impute
import torch
from sklearn.utils._mask import _get_mask
from sklearn.utils._missing import is_pandas_na, is_scalar_nan
from sklearn.utils.validation import check_is_fitted

from . import _keytables
from .chunked import ChunkedArray
from .decomposition.pca import SHIFT_ROWS, _device_data, _on_rank0
from .preprocessing.data import keys_to_values, order_statistics

STRATEGIES = ["mean", "median", "most_frequent", "constant"]
MODE_BUDGET = 1 << 30        # bytes of one column group's hash tables (plus, with several ranks, its gathered lists):
                             # wider data runs in column groups, each of which reads its columns of X once


def _missing_is_nan(missing_values):
    return is_scalar_nan(missing_values) or is_pandas_na(missing_values)


def _shift(X, miss_is_nan, miss):
    """Per column the mean of the non-missing finite values among the first <= SHIFT_ROWS rows of rank 0 (0 where there
    is none), broadcast: the shift of the statistics pass."""
    def fn():
        m = min(SHIFT_ROWS, X.n_local)
        if m == 0:
            return np.zeros(X.d)
        r = X.local_rows(np.arange(m)).astype(np.float64)
        ok = np.isfinite(r) if miss_is_nan else np.isfinite(r) & (r != miss)
        return np.where(ok, r, 0.0).sum(0) / np.maximum(ok.sum(0), 1)

    return _on_rank0(X.comm, fn)


def missing_stats(X, miss_is_nan, miss):
    """(missing, nan, inf, S, s, local_missing): per column the global missing / NaN / inf counts, the global sum of
    x - s over the non-missing finite x, the shift s and this rank's missing count, float64 numpy."""
    be, comm, d = X.backend, X.comm, X.d
    s = _shift(X, miss_is_nan, miss)
    s_dev = torch.as_tensor(np.ascontiguousarray(s, dtype=np.float64)).to(be.device)
    acc = be.zeros((4, d), torch.float64)
    for i, x in enumerate(X.chunks):
        be.impute_stats_chunk(x, miss_is_nan, miss, s_dev, acc, first=i == 0)
    local_missing = acc[0].cpu().numpy().copy()
    comm.allreduce_sum_(acc.view(-1))
    missing, nan, inf, S = acc.cpu().numpy()
    return missing, nan, inf, S, s, local_missing


def mode_statistics(X, miss_is_nan, miss, local_valid, global_valid):
    """The most frequent non-missing value of every column over every row of every rank (the smallest on ties, +0.0
    for a zero), NaN for a column without one: float64 numpy."""
    be, comm, d = X.backend, X.comm, X.d
    world = comm.world
    cost = [16 * _keytables.capacity(m, X.dtype) + (32 * int(m) if world > 1 else 0) for m in global_valid]
    groups, j0 = [], 0
    while j0 < d:                        # identical on every rank: the costs come from global counts
        j1, used = j0 + 1, cost[j0]
        while j1 < d and used + cost[j1] <= MODE_BUDGET:
            used += cost[j1]
            j1 += 1
        groups.append((j0, j1))
        j0 = j1
    best_key = np.zeros(d, dtype=np.uint64)
    best_cnt = np.zeros(d)

    for j0, j1 in groups:
        g = j1 - j0
        tables = _keytables.alloc(be, [_keytables.capacity(m, X.dtype) for m in local_valid[j0:j1]])
        keys, counts, off, total = tables
        for i, x in enumerate(X.chunks):
            be.mode_count_chunk(x[:, j0:j1], miss_is_nan, miss, keys, counts, off, total, first=i == 0)
        key, cnt, nd = be.mode_best(keys, counts, off, g, total)
        if world > 1:
            _, (key, cnt, nd), _ = _keytables.merge_ranks(be, comm, tables, g, X.dtype, nd)
        best_key[j0:j1] = key.cpu().numpy().view(np.uint64)
        best_cnt[j0:j1] = cnt.cpu().numpy()
    vals = np.asarray(keys_to_values(best_key, X.dtype), dtype=np.float64)
    vals[best_cnt == 0] = np.nan
    return vals


def median_statistics(X, miss_is_nan, miss):
    """np.ma.median of every column's non-missing values in X's host dtype: (lo + hi) / 2 with lo = hi = a[m // 2]
    for odd m and a[m / 2 - 1], a[m / 2] for even m; NaN for a column without values."""
    lo, hi, m = order_statistics(X, np.array([0.5]), missing=None if miss_is_nan else miss)
    dt = X.np_dtype
    lo, hi = lo[:, 0].astype(dt), hi[:, 0].astype(dt)
    high = np.where(m % 2 == 1, lo, hi)
    with np.errstate(over="ignore", invalid="ignore"):
        med = np.true_divide(lo + high, dt.type(2))
    med[m == 0] = np.nan
    return med


class SimpleImputer(sklearn.impute.SimpleImputer):
    """Univariate imputer for completing missing values with simple strategies, on the device.

    Every input kind gets what scikit-learn's SimpleImputer gives for numpy input: ``statistics_``, ``indicator_``,
    the warnings and the errors.  ``median`` and ``most_frequent`` statistics are bit-equal to scikit-learn's; the
    ``mean`` is a float64 sum about a shift, divided by the float64 count (scikit-learn sums float32 columns in float32,
    which can be far off on long columns), and is NaN only when that sum is not finite.  Integer input is computed as
    float32 (int32) or float64 (int64), so outputs are float.  A zero mode is +0.0.  ``strategy`` must be one of the
    four names: a callable raises NotImplementedError.  ``transform`` and ``inverse_transform`` return device-resident
    ChunkedArrays in X's dtype (float32 for bf16 rows) with X's chunking; the input is never modified and ``copy`` has
    no effect.  Unlike dask_ml's array path, which allows only ``mean`` and ``constant``, every strategy and any numeric
    ``missing_values`` work on every input kind.  The scikit-learn docstring follows.
    """

    __doc__ = __doc__ + "\n".join(sklearn.impute.SimpleImputer.__doc__.split("\n")[1:])

    def _check_params(self):
        if callable(self.strategy):
            raise NotImplementedError("a callable strategy cannot run on the device; use one of %s" % STRATEGIES)
        if self.strategy not in STRATEGIES:
            raise ValueError("Can only use these strategies: {0}  got strategy={1}".format(STRATEGIES, self.strategy))
        if not (_missing_is_nan(self.missing_values) or isinstance(self.missing_values, numbers.Real)):
            raise ValueError("dask_ml_b200.impute.SimpleImputer only supports NaN or numeric non-NA values for "
                             "'missing_values'; got %r." % (self.missing_values,))
        self._validate_params()

    def _check_sample(self, X, in_fit, bad=None):
        """scikit-learn's input checks on one row of X's dtype (feature count, dtype compatibility, fill_value); with
        ``bad`` (NaN or inf) in it, scikit-learn's own error for that value is raised."""
        sample = np.zeros((1, X.d), dtype=X.np_dtype)
        if bad is not None:
            sample[0, 0] = bad
        self._validate_input(sample, in_fit=in_fit)

    def _missing(self, dtype):
        """(is_nan, value) of ``missing_values`` for data of the numpy ``dtype``, as the kernels take it."""
        if _missing_is_nan(self.missing_values):
            return True, float("nan")
        with np.errstate(over="ignore"):
            return False, float(np.asarray(self.missing_values).astype(dtype))

    def _raise_invalid(self, X, in_fit, miss_is_nan, nan, inf):
        if not miss_is_nan and nan > 0:
            self._check_sample(X, in_fit, bad=np.nan)
        if inf > 0:
            self._check_sample(X, in_fit, bad=np.inf)

    def fit(self, X, y=None):
        self._check_params()
        X = _device_data(X, allow_nonfinite=True)
        self._check_sample(X, in_fit=True)
        miss_is_nan, miss = self._missing(X.np_dtype)
        missing, nan, inf, S, s, local_missing = missing_stats(X, miss_is_nan, miss)
        self._raise_invalid(X, True, miss_is_nan, nan.sum(), inf.sum())
        valid = X.n_global - missing
        empty = valid == 0
        self._fill_dtype = X.np_dtype
        if self.strategy == "mean":
            with np.errstate(divide="ignore", invalid="ignore"):
                stats = s + S / valid
            stats[~np.isfinite(S)] = np.nan
        elif self.strategy == "median":
            stats = median_statistics(X, miss_is_nan, miss)
        elif self.strategy == "most_frequent":
            stats = mode_statistics(X, miss_is_nan, miss, X.n_local - local_missing, valid)
        else:
            fill_value = 0 if self.fill_value is None else self.fill_value
            stats = np.full(X.d, fill_value, dtype=np.object_)
        if self.strategy == "constant":
            if not self.keep_empty_features:
                stats[empty] = np.nan
        else:
            stats[empty] = 0 if self.keep_empty_features else np.nan
        self.statistics_ = stats
        # a mask whose column-wise any() is the global "had a missing value" flag of every feature
        super()._fit_indicator(np.asarray(missing > 0)[None, :])
        return self

    def fit_transform(self, X, y=None, **fit_params):
        """fit, then transform, with X uploaded once: a device-resident ChunkedArray."""
        X = _device_data(X, allow_nonfinite=True)
        return self.fit(X, y).transform(X)

    def transform(self, X):
        """X with its missing values imputed (and the indicator columns appended with ``add_indicator``): a
        device-resident ChunkedArray in X's dtype (float32 for bf16 rows)."""
        check_is_fitted(self)
        X = _device_data(X, allow_nonfinite=True)
        self._check_sample(X, in_fit=False)
        be, d = X.backend, X.d
        stats = self.statistics_
        if self.keep_empty_features:
            keep = np.arange(d)
        else:
            invalid_mask = _get_mask(stats, np.nan)
            keep = np.flatnonzero(~invalid_mask)
            if invalid_mask.any():
                invalid_features = np.arange(d)[invalid_mask]
                if hasattr(self, "feature_names_in_"):
                    invalid_features = self.feature_names_in_[invalid_features]
                warnings.warn("Skipping features without any observed values:"
                              f" {invalid_features}. At least one non-missing value is needed"
                              f" for imputation with strategy='{self.strategy}'.")
        fill = np.zeros(d)
        with np.errstate(over="ignore", invalid="ignore"):
            fill[keep] = stats[keep].astype(self._fill_dtype).astype(X.np_dtype)
        ind = np.asarray(self.indicator_.features_) if self.add_indicator else np.zeros(0, dtype=np.int64)
        check = np.setdiff1d(np.arange(d), keep)
        cols = torch.as_tensor(np.concatenate([keep, ind, check]).astype(np.int32)).to(be.device)
        fill_dev = torch.as_tensor(fill).to(be.device)
        miss_is_nan, miss = self._missing(X.np_dtype)
        out_t = torch.float64 if X.dtype == torch.float64 else torch.float32
        invalid = be.zeros((2,), torch.float64)
        blocks = []
        for x in X.chunks:
            o = be.rows_buffer(int(x.shape[0]), len(keep) + len(ind), out_t)
            be.impute_chunk(x, miss_is_nan, miss, fill_dev, cols, len(keep), len(ind), len(check), False, o, invalid)
            blocks.append(o)
        X.comm.allreduce_sum_(invalid)
        nan, inf = invalid.cpu().numpy()
        self._raise_invalid(X, False, miss_is_nan, nan, inf)
        return ChunkedArray(blocks)

    def inverse_transform(self, X):
        """The imputed values put back to ``missing_values`` where the indicator is 1: a device-resident ChunkedArray
        in X's dtype (float32 for bf16 rows).  Only with ``add_indicator=True``."""
        check_is_fitted(self)
        if not self.add_indicator:
            raise ValueError("'inverse_transform' works only when 'SimpleImputer' is instantiated with "
                             f"'add_indicator=True'. Got 'add_indicator={self.add_indicator}' instead.")
        X = _device_data(X, allow_nonfinite=True)
        be = X.backend
        feats = np.asarray(self.indicator_.features_)
        d_orig = len(self.statistics_)
        kept = np.arange(d_orig) if self.keep_empty_features else np.flatnonzero(~_get_mask(self.statistics_, np.nan))
        if X.d != len(kept) + len(feats):
            raise ValueError("X has %d features, but the imputer's output has %d (%d imputed, %d indicator columns)"
                             % (X.d, len(kept) + len(feats), len(kept), len(feats)))
        src = np.full(d_orig, -1)
        src[kept] = np.arange(len(kept))
        isrc = np.full(d_orig, -1)
        isrc[feats] = len(kept) + np.arange(len(feats))
        cols = torch.as_tensor(np.concatenate([src, isrc]).astype(np.int32)).to(be.device)
        miss_is_nan, miss = self._missing(X.np_dtype)
        out_t = torch.float64 if X.dtype == torch.float64 else torch.float32
        blocks = []
        for x in X.chunks:
            o = be.rows_buffer(int(x.shape[0]), d_orig, out_t)
            be.impute_chunk(x, miss_is_nan, miss, None, cols, d_orig, d_orig, 0, True, o)
            blocks.append(o)
        return ChunkedArray(blocks)
