"""StandardScaler, MinMaxScaler, RobustScaler and QuantileTransformer with the dask_ml.preprocessing API, executed by
the H100 engine.

Mirrors dask_ml/preprocessing/data.py:24-312 (reference @ 0310a90); QuantileTransformer's passes are described in
DESIGN.md, "The passes of QuantileTransformer".  Each class subclasses scikit-learn's, as the
reference does, and accepts what PCA accepts.  The passes (DESIGN.md, "The passes of the scalers"):

    fit, Standard / MinMax (bkm_colstats_chunk, one read of X, float64), with a shift s shared by every rank:
        per column  S = sum (x - s),  Q = sum (x - s)^2 over the finite x,  min, max over the non-NaN x,
                    and the NaN / +inf / -inf counts                     one all-reduce of [S | Q | counts | n] and
                                                                          one gather of [min | max]
    host:           mean = s + S / n,  var = (Q - S^2 / n) / n  (ddof = 0), then numpy's rules for NaN and inf
    fit, Robust (bkm_radix_hist_chunk + bkm_radix_select_step): the exact order statistics at floor and floor + 1 of
                    numpy's virtual index for q_min, 50 and q_max, one read of X and one all-reduce per 8-bit round
    host:           numpy's 'linear' interpolation of those values, the installed numpy's own formula
    transform / inverse_transform (bkm_affine_chunk): op2(op1(x, a), b), each step rounded once in the output dtype

Attributes are computed in float64 and take the dtypes the reference gives: X's dtype (float32 for bf16 rows) for
StandardScaler and MinMaxScaler (whose attributes come from the reference's own expressions on the exact min / max),
float64 for RobustScaler (numpy's percentile of a list of quantiles).  Transform outputs are device-resident
ChunkedArrays with X's chunking, in numpy's promotion of X's dtype with the attributes' dtype; the input is never
modified (the reference modifies numpy input in place).
"""
import numpy as np
import torch
from sklearn.preprocessing import _data as skdata
from sklearn.utils.validation import check_is_fitted

from ..chunked import ChunkedArray
from ..decomposition.pca import SHIFT_ROWS, _device_data, _on_rank0

OP1_NONE, OP1_SUB, OP1_MUL = 0, 1, 2
OP2_NONE, OP2_DIV, OP2_ADD = 0, 1, 2

# one record of the radix selection's device state per (column, target): include/bkm_b200.h
SELECT_RECORD = np.dtype([("key", "<u8"), ("rank", "<f8"), ("nvalid", "<f8"), ("slot", "<i4"), ("pad", "<i4")])
RADIX_ROUNDS = {torch.float32: 4, torch.bfloat16: 2, torch.float64: 8}


# ------------------------------------------------ column statistics ------------------------------------------------
def _shift(X):
    """Per column the mean of the finite values among the first <= SHIFT_ROWS rows of rank 0 (0 where there is none),
    broadcast: the shift of the statistics pass, which keeps data far from the origin from losing its variance."""
    def fn():
        m = min(SHIFT_ROWS, X.n_local)
        if m == 0:
            return np.zeros(X.d)
        r = X.local_rows(np.arange(m)).astype(np.float64)
        fin = np.isfinite(r)
        return np.where(fin, r, 0.0).sum(0) / np.maximum(fin.sum(0), 1)

    return _on_rank0(X.comm, fn)


def column_stats(X):
    """(mean, var, min, max) per column over every row of every rank, float64 numpy, with numpy's rules: a NaN makes
    all four NaN; +inf and -inf together make the mean NaN; a single-signed inf makes the mean that inf; any inf makes
    the variance NaN."""
    be, comm, d = X.backend, X.comm, X.d
    s = _shift(X)
    s_dev = torch.as_tensor(np.ascontiguousarray(s, dtype=np.float64)).to(be.device)
    red = be.zeros((5 * d + 1,), torch.float64)
    acc = red[: 5 * d].view(5, d)
    mm = be.zeros((2, d), torch.float64)
    for i, x in enumerate(X.chunks):
        be.colstats_chunk(x, s_dev, acc, mm, first=i == 0)
    red[-1] = float(X.n_local)
    comm.allreduce_sum_(red)
    parts = comm.allgather_obj(mm.cpu().numpy())
    lo = np.fmin.reduce([p[0] for p in parts])
    hi = np.fmax.reduce([p[1] for p in parts])
    h = red.cpu().numpy()
    S, Q, nan, pinf, ninf = h[: 5 * d].reshape(5, d)
    n = h[-1]
    with np.errstate(divide="ignore", invalid="ignore"):
        mu = S / n
        mean = s + mu
        var = np.maximum((Q - S * mu) / n, 0.0)
    inf = (pinf > 0) | (ninf > 0)
    mean = np.where(pinf > 0, np.inf, mean)
    mean = np.where(ninf > 0, -np.inf, mean)
    mean = np.where((pinf > 0) & (ninf > 0), np.nan, mean)
    var = np.where(inf, np.nan, var)
    bad = (nan > 0) | (n == 0)
    mean, var = np.where(bad, np.nan, mean), np.where(bad, np.nan, var)
    lo, hi = np.where(bad, np.nan, lo), np.where(bad, np.nan, hi)
    return mean, var, lo, hi


# ------------------------------------------------ percentiles ------------------------------------------------
def keys_to_values(keys, dtype):
    """Order-preserving radix keys (uint64 holding 16, 32 or 64 bits) -> values: numpy of X's host dtype."""
    keys = np.asarray(keys, dtype=np.uint64)
    bits = {torch.bfloat16: 16, torch.float32: 32, torch.float64: 64}[dtype]
    sign = np.uint64(1 << (bits - 1))
    mask = np.uint64((1 << bits) - 1) if bits < 64 else np.uint64(0xFFFFFFFFFFFFFFFF)
    u = np.where(keys & sign, keys ^ sign, ~keys & mask)
    if bits == 64:
        return u.view(np.float64)
    if bits == 32:
        return u.astype(np.uint32).view(np.float32)
    return (u.astype(np.uint32) << np.uint32(16)).view(np.float32)


def percentile_from_order_stats(prev, nxt, n, q, dtype):
    """np.percentile(column, q) of a column of n values given, per column, the order statistics at the indices
    np.percentile takes: ``prev`` / ``nxt`` (d, len(q)) of the column dtype hold the values at floor(v) and
    floor(v) + 1 of the virtual index v = (n - 1) q / 100 (both the last value when v >= n - 1).  Applies the installed
    numpy's 'linear' method step by step (numpy/lib/_function_base_impl.py: _get_indexes, _get_gamma, _lerp), so the
    result has numpy's bits and dtype: shape (d, len(q))."""
    prev, nxt = np.asarray(prev, dtype=dtype), np.asarray(nxt, dtype=dtype)
    quantiles = np.true_divide(np.asanyarray(q, dtype=np.float64), np.dtype(dtype).type(100))
    vi = np.asanyarray((n - 1) * quantiles)
    pi = np.asanyarray(np.floor(vi))
    pi[vi >= n - 1] = -1
    pi[vi < 0] = 0
    pi[np.isnan(vi)] = -1
    pi = pi.astype(np.intp)
    gamma = np.asanyarray(np.asanyarray(vi - pi), dtype=vi.dtype)
    gamma = np.broadcast_to(gamma, prev.shape)
    with np.errstate(invalid="ignore", over="ignore"):
        diff_b_a = np.subtract(nxt, prev)
        out = np.asanyarray(np.add(prev, diff_b_a * gamma))
        np.subtract(nxt, diff_b_a * (1 - gamma), out=out, where=gamma >= 0.5, casting="unsafe",
                    dtype=type(out.dtype))
    return out


def percentiles(X, q):
    """np.percentile of every whole column at the percentiles ``q`` (a list, values in [0, 100]) over every row of
    every rank, exact for any chunking or rank split: (d, len(q)) float64 (numpy's dtype for a list of quantiles)."""
    be, comm, d = X.backend, X.comm, X.d
    T = 2 * len(q)
    qf = np.true_divide(np.asarray(q, dtype=np.float64), 100.0)
    state = be.radix_state_new(d, T)
    hist = be.zeros((d, T, 256), torch.float64)
    for rnd in range(RADIX_ROUNDS[X.dtype]):
        for i, x in enumerate(X.chunks):
            be.radix_hist_chunk(x, state, T, rnd, hist, first=i == 0)
        comm.allreduce_sum_(hist.view(-1))
        be.radix_select_step(hist, state, d, T, rnd, X.dtype, qf)
    rec = state.cpu().numpy().view(SELECT_RECORD).reshape(d, T)
    vals = keys_to_values(rec["key"], X.dtype)
    n = X.n_global
    if n == 0:
        return np.full((d, len(q)), np.nan)
    P = percentile_from_order_stats(vals[:, 0::2], vals[:, 1::2], n, q, X.np_dtype)
    P[rec["nvalid"][:, 0] < n] = np.nan                  # a NaN in the column: numpy gives NaN
    return np.asarray(P, dtype=np.float64)


# ------------------------------------------------ transform ------------------------------------------------
def affine(X, a, b, op1, op2):
    """op2(op1(x, a), b) per element of every chunk -> device-resident ChunkedArray in numpy's promotion of X's dtype
    with the dtypes of ``a`` / ``b`` (numpy arrays or None), rows with the pitch ``CudaBackend.to_device`` gives."""
    X = _device_data(X)
    be = X.backend
    out_np = np.result_type(X.np_dtype, *[v.dtype for v in (a, b) if v is not None])
    tdt = torch.float64 if out_np == np.dtype("float64") else torch.float32

    def dev(v):
        if v is None:
            return None
        return torch.as_tensor(np.ascontiguousarray(np.asarray(v, dtype=out_np), dtype=np.float64)).to(be.device)

    a_dev, b_dev = dev(a), dev(b)
    blocks = []
    for x in X.chunks:
        o = be.rows_buffer(int(x.shape[0]), X.d, tdt)
        be.affine_chunk(x, a_dev, b_dev, op1 if a is not None else OP1_NONE, op2 if b is not None else OP2_NONE, o)
        blocks.append(o)
    return ChunkedArray(blocks)


class _DeviceFitTransform(object):
    def fit_transform(self, X, y=None, **fit_params):
        """fit, then transform, with X uploaded once: a device-resident ChunkedArray."""
        X = _device_data(X)
        return self.fit(X, y).transform(X)


class StandardScaler(_DeviceFitTransform, skdata.StandardScaler):
    __doc__ = skdata.StandardScaler.__doc__

    def fit(self, X, y=None):
        self._reset()
        X = _device_data(X)
        mean, var, _, _ = column_stats(X)
        dt = X.np_dtype
        if self.with_mean:
            self.mean_ = mean.astype(dt)
        if self.with_std:
            self.var_ = var.astype(dt)
            scale = self.var_.copy()
            scale[scale == 0] = 1
            self.scale_ = np.sqrt(scale)
        self.n_samples_seen_ = np.nan
        return self

    def partial_fit(self, X, y=None):
        raise NotImplementedError()

    def transform(self, X, y=None, copy=None):
        """(X - mean_) / scale_ (each step only when its flag is set): a device-resident ChunkedArray."""
        check_is_fitted(self, "n_samples_seen_")
        return affine(X, self.mean_ if self.with_mean else None, self.scale_ if self.with_std else None,
                      OP1_SUB, OP2_DIV)

    def inverse_transform(self, X, copy=None):
        check_is_fitted(self, "n_samples_seen_")
        return affine(X, self.scale_ if self.with_std else None, self.mean_ if self.with_mean else None,
                      OP1_MUL, OP2_ADD)


def _handle_zeros(scale):
    """dask_ml.utils.handle_zeros_in_scale: exact zeros become 1."""
    scale = scale.copy()
    scale[scale == 0.0] = 1.0
    return scale


class MinMaxScaler(_DeviceFitTransform, skdata.MinMaxScaler):
    __doc__ = skdata.MinMaxScaler.__doc__

    def fit(self, X, y=None):
        self._reset()
        feature_range = self.feature_range
        if feature_range[0] >= feature_range[1]:
            raise ValueError("Minimum of desired feature range must be smaller than maximum.")
        X = _device_data(X)
        _, _, lo, hi = column_stats(X)
        dt = X.np_dtype
        data_min, data_max = lo.astype(dt), hi.astype(dt)       # exact: the min and max are values of X
        with np.errstate(invalid="ignore", over="ignore"):               # inf / NaN columns give NaN, as in numpy
            data_range = data_max - data_min
            scale = (feature_range[1] - feature_range[0]) / _handle_zeros(data_range)
            self.min_ = feature_range[0] - data_min * scale
        self.data_min_ = data_min
        self.data_max_ = data_max
        self.data_range_ = data_range
        self.scale_ = scale
        self.n_samples_seen_ = np.nan
        return self

    def partial_fit(self, X, y=None):
        raise NotImplementedError()

    def transform(self, X, y=None, copy=None):
        """X * scale_ + min_ (``clip`` is ignored, as in the reference): a device-resident ChunkedArray."""
        check_is_fitted(self, "scale_")
        return affine(X, self.scale_, self.min_, OP1_MUL, OP2_ADD)

    def inverse_transform(self, X, y=None, copy=None):
        check_is_fitted(self, "scale_")
        return affine(X, self.min_, self.scale_, OP1_SUB, OP2_DIV)


class RobustScaler(_DeviceFitTransform, skdata.RobustScaler):
    __doc__ = skdata.RobustScaler.__doc__

    def fit(self, X, y=None):
        q_min, q_max = self.quantile_range
        if not 0 <= q_min <= q_max <= 100:
            raise ValueError("Invalid quantile range: %s" % str(self.quantile_range))
        X = _device_data(X)
        P = percentiles(X, [q_min, 50.0, q_max])
        self.center_ = P[:, 1]
        self.scale_ = skdata._handle_zeros_in_scale(P[:, 2] - P[:, 0], copy=False)
        return self

    def transform(self, X):
        """(X - center_) / scale_ (each step only when its flag is set): a device-resident ChunkedArray."""
        if self.with_centering:
            check_is_fitted(self, "center_")
        if self.with_scaling:
            check_is_fitted(self, "scale_")
        return affine(X, self.center_ if self.with_centering else None, self.scale_ if self.with_scaling else None,
                      OP1_SUB, OP2_DIV)

    def inverse_transform(self, X):
        check_is_fitted(self, ["center_", "scale_"])
        return affine(X, self.scale_ if self.with_scaling else None, self.center_ if self.with_centering else None,
                      OP1_MUL, OP2_ADD)


# ------------------------------------------------ QuantileTransformer ------------------------------------------------
# one selection's per-column record (include/bkm_b200.h): header, then 2 n_q SELECT_RECORDs, then 2 n_q live prefixes
QUANTILE_HEAD = np.dtype([("nvalid", "<f8"), ("R", "<i4"), ("L", "<i4")])
HIST_BUDGET = 512 << 20          # bytes of one round's [columns][live slots][256] float64 histogram: larger d * n_q
                                 # runs in column groups, each of which reads X once per round
DISTRIBUTIONS = {"uniform": 0, "normal": 1}


def _order_stat_ranks(nvalid, qf):
    """The floor / floor + 1 ranks of numpy's 'linear' virtual index (nvalid - 1) qf, as the selection derives them on
    the device: (lo, hi), each (d, len(qf)) float64."""
    nv = np.asarray(nvalid, dtype=np.float64)[:, None]
    vi = (nv - 1.0) * qf[None, :]
    lo, hi = np.floor(vi), np.floor(vi) + 1.0
    top, neg = vi >= nv - 1.0, vi < 0.0
    lo, hi = np.where(top, nv - 1.0, lo), np.where(top, nv - 1.0, hi)
    lo, hi = np.where(neg, 0.0, lo), np.where(neg, 0.0, hi)
    empty = np.broadcast_to(nv <= 0.0, vi.shape)
    return np.where(empty, 0.0, lo), np.where(empty, 0.0, hi)


def order_statistics(X, qf, missing=None):
    """The order statistics of every whole column at the floor / floor + 1 ranks of numpy's 'linear' virtual index
    (m - 1) qf over its m valid values, exact for any chunking or rank split: (lo, hi) of X's host dtype and m, each
    (d, len(qf)) / (d,).  Valid means not NaN and, with a number ``missing``, not equal to it (the masked count)."""
    be, comm, d = X.backend, X.comm, X.d
    nq = len(qf)
    qf_dev = torch.as_tensor(np.ascontiguousarray(qf, dtype=np.float64)).to(be.device)
    rounds = RADIX_ROUNDS[X.dtype]
    stride = 16 + 80 * nq
    state = be.quantile_state_new(d, nq)
    widest = min(2 * nq, 256 ** (rounds - 1))
    group = max(1, min(d, HIST_BUDGET // (widest * 256 * 8)))
    hist = be.empty((group * widest * 256,), torch.float64)
    for j0 in range(0, d, group):
        j1 = min(d, j0 + group)
        st = state[j0 * stride: j1 * stride]
        for rnd in range(rounds):
            h = hist[: (j1 - j0) * min(2 * nq, 256 ** rnd) * 256]
            for i, x in enumerate(X.chunks):
                if missing is None:
                    be.quantile_hist_chunk(x[:, j0:j1], st, nq, rnd, h, first=i == 0)
                else:
                    be.quantile_hist_masked_chunk(x[:, j0:j1], missing, st, nq, rnd, h, first=i == 0)
            comm.allreduce_sum_(h)
            be.quantile_select_step(h, st, j1 - j0, nq, rnd, X.dtype, qf_dev)
    raw = state.cpu().numpy().reshape(d, stride)
    head = np.ascontiguousarray(raw[:, :16]).view(QUANTILE_HEAD)[:, 0]
    rec = np.ascontiguousarray(raw[:, 16: 16 + 64 * nq]).view(SELECT_RECORD)
    lo, hi = _order_stat_ranks(head["nvalid"], qf)
    keys = np.empty((2, d, nq), dtype=np.uint64)
    for j in range(d):
        distinct = np.unique(np.concatenate([lo[j], hi[j]]))
        assert len(distinct) == head["R"][j], (j, len(distinct), head["R"][j])
        keys[0, j] = rec["key"][j, np.searchsorted(distinct, lo[j])]
        keys[1, j] = rec["key"][j, np.searchsorted(distinct, hi[j])]
    vals = keys_to_values(keys, X.dtype)
    return vals[0], vals[1], np.asarray(head["nvalid"], dtype=np.float64)


def quantiles_exact(X, references):
    """np.percentile(column, references * 100) of every whole column over every row of every rank, exact for any
    chunking or rank split: (len(references), d) float64, NaN for a column that holds a NaN."""
    d = X.d
    nq = len(references)
    q = np.asarray(references, dtype=np.float64) * 100
    qf = np.true_divide(q, 100.0)
    lo, hi, nvalid = order_statistics(X, qf)
    n = X.n_global
    if n == 0:
        return np.full((nq, d), np.nan)
    P = percentile_from_order_stats(lo, hi, n, q, X.np_dtype)
    P[nvalid < n] = np.nan                              # a NaN in the column: numpy gives NaN
    return np.ascontiguousarray(np.asarray(P, dtype=np.float64).T)


def quantile_transform(X, quantiles, references, inverse, distribution):
    """The reference's _transform_col on every column (forward, or inverse) -> device-resident float64 ChunkedArray,
    rows with the pitch ``CudaBackend.to_device`` gives."""
    from scipy import stats

    be = X.backend
    qT = torch.as_tensor(np.ascontiguousarray(np.asarray(quantiles, dtype=np.float64).T)).to(be.device)
    ref = torch.as_tensor(np.ascontiguousarray(references, dtype=np.float64)).to(be.device)
    dist = stats.norm if distribution == "normal" else stats.uniform
    eps = skdata.BOUNDS_THRESHOLD - np.spacing(1)
    lo, hi = (0.0, 0.0) if inverse else (float(dist.ppf(eps)), float(dist.ppf(1 - eps)))
    blocks = []
    for x in X.chunks:
        o = be.rows_buffer(int(x.shape[0]), X.d, torch.float64)
        be.quantile_transform_chunk(x, qT, ref, inverse, DISTRIBUTIONS[distribution], lo, hi, o)
        blocks.append(o)
    return ChunkedArray(blocks)


class _Rows(object):
    """Device rows as scikit-learn's fit sees them: an object with a shape."""

    def __init__(self, data):
        self.data = data
        self.shape = (data.n_global, data.d)


class QuantileTransformer(skdata.QuantileTransformer):
    """Transforms features using quantile information.

    The quantiles are exact: ``quantiles_[:, j]`` equals ``np.percentile(X[:, j], references_ * 100)`` over every row
    (``subsample`` is ignored, as in dask_ml).  Outputs are device-resident float64 ChunkedArrays.  The scikit-learn
    docstring follows.
    """

    __doc__ = __doc__ + "\n".join(skdata.QuantileTransformer.__doc__.split("\n")[1:])

    def _check_inputs(self, X, in_fit, accept_sparse_negative=False, copy=False):
        """X -> device rows; scikit-learn's checks run on a 5-row sample of X's dtype, as in dask_ml."""
        from scipy import sparse

        if sparse.issparse(X):
            raise NotImplementedError("QuantileTransformer does not accept sparse input")
        X = _device_data(X, allow_nonfinite=True)           # NaN and inf have defined results (as in dask_ml)
        sample = np.random.RandomState(0).uniform(size=(5, X.d)).astype(X.np_dtype)
        super(QuantileTransformer, self)._check_inputs(sample, in_fit, accept_sparse_negative=accept_sparse_negative)
        return _Rows(X)

    def fit_transform(self, X, y=None, **fit_params):
        """fit, then transform, with X uploaded once: a device-resident float64 ChunkedArray."""
        X = _device_data(X, allow_nonfinite=True)
        return self.fit(X, y).transform(X)

    def _sparse_fit(self, X, random_state):
        raise NotImplementedError

    def _dense_fit(self, X, random_state):
        self.quantiles_ = quantiles_exact(X.data, self.references_)

    def _transform(self, X, inverse=False):
        return quantile_transform(X.data, self.quantiles_, self.references_, inverse, self.output_distribution)

    def inverse_transform(self, X):
        """Back-projection to the original space: a device-resident float64 ChunkedArray."""
        check_is_fitted(self)
        return self._transform(self._check_inputs(X, in_fit=False), inverse=True)
