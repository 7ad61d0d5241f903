"""PCA with the dask_ml.decomposition.PCA API, executed by the H100 engine.

Mirrors dask_ml/decomposition/pca.py (reference @ 0310a90).  The reference centres X and takes ``da.linalg.svd`` (tsqr)
of it; for tall-and-skinny X (n >> d) the same components come from the (d, d) covariance, which one read of X gives:

    pass 1 (bkm_gram_chunk, float64 on the fp64 tensor cores), with a shift s shared by every rank:
        m = sum_i (x_i - s),   G = sum_i (x_i - s)(x_i - s)^T          one all-reduce of [G | m | n]
    host (float64, rank 0, broadcast):
        mean_ = s + m / n,   C = G - m m^T / n,   eigh(C) -> lambda (descending, clamped at 0), V
        singular values S = sqrt(lambda), components_ = rows of V^T
    pass 2 (bkm_project_chunk): t = (x - mean_) . v_j, and per column the signed arg-max of |t|

The shift (the mean of the first <= 65536 rows of rank 0) keeps data far from the origin from losing its variance to
cancellation.  The reference's ``svd_flip(U, V)`` gives component j the sign of the entry of U[:, j] with the largest
magnitude (the first row on ties); sign(U_ij) = sign(t_ij), so pass 2 returns that entry without forming U.

Every ``svd_solver`` runs this exact eigendecomposition.  For 'randomized' the reference's formulas for the total
variance and ``noise_variance_`` are kept: with the exact top-k vectors they are the limit ``svd_compressed``
approximates.  Attributes are computed in float64 and cast to the dtype of X (float32 for bf16 rows).
"""
import numpy as np
import torch
from sklearn.decomposition._base import _BasePCA
from sklearn.utils.extmath import fast_logdet
from sklearn.utils.validation import check_is_fitted, check_random_state

from ..chunked import ChunkedArray, is_dask_dataframe
from ..engine import DeviceData
from ..utils import check_array
from ..cluster import k_means as _km
from ..cluster.k_means import _NONFINITE_MSG

SHIFT_ROWS = 65536      # rows of rank 0 whose mean is the shift of the Gram pass


def _device_data(X, allow_nonfinite=False):
    """Validated input -> DeviceData (what KMeans accepts: ndarray, DataFrame, torch, ChunkedArray, dask arrays,
    ``host_resident``).  Non-finite values are detected from the Gram pass itself (a NaN or inf row makes G
    non-finite), so the fit reads X twice, not three times; only when G is non-finite is X scanned, to tell NaN / inf
    from finite values whose squares overflow float64 (``gram_pass``).  ``allow_nonfinite`` accepts NaN and inf in
    numpy input too, for estimators that define a result for them."""
    try:
        import pandas as pd

        if isinstance(X, pd.DataFrame):
            X = X.values
    except ImportError:  # pragma: no cover
        pass
    if is_dask_dataframe(X):
        raise TypeError("Cannot fit on dask.dataframe due to unknown partition lengths.")
    if isinstance(X, DeviceData):
        return X
    finite = {"ensure_all_finite": False} if allow_nonfinite else {}
    X = check_array(X, accept_dask_dataframe=False, accept_unknown_chunks=False, accept_sparse=False, **finite)
    return _km._to_device_data(X, check_finite=False)


def _chunks(X):
    return X.chunks


def _on_rank0(comm, fn):
    """fn() on rank 0, its result broadcast to every rank; an exception is handed to every rank, so that none waits
    in the broadcast."""
    res = err = None
    if comm.rank == 0:
        try:
            res = fn()
        except Exception as e:
            err = e
    res, err = comm.bcast_obj((res, err))
    if err is not None:
        raise err
    return res


def gram_pass(X):
    """(G, m, n, s): the shifted Gram matrix and column sums over every row of every rank, in float64 numpy."""
    be, comm, d = X.backend, X.comm, X.d

    def shift():
        m = min(SHIFT_ROWS, X.n_local)
        if m == 0:
            return np.zeros(d)
        return X.local_rows(np.arange(m)).astype(np.float64).mean(0)

    s = _on_rank0(comm, shift)
    s_dev = torch.as_tensor(np.ascontiguousarray(s, dtype=np.float64)).to(be.device)
    red = be.zeros((d * d + d + 1,), torch.float64)
    G, m = red[: d * d].view(d, d), red[d * d: d * d + d]
    first = True
    for x in _chunks(X):
        be.gram_chunk(x, s_dev, m, G, first=first)
        first = False
    red[-1] = float(X.n_local)
    comm.allreduce_sum_(red)
    h = red.cpu().numpy()
    G, m, n = h[: d * d].reshape(d, d).copy(), h[d * d: d * d + d].copy(), int(round(h[-1]))
    if not (np.isfinite(G).all() and np.isfinite(m).all()):
        # NaN / inf in X, or finite values whose squares overflow float64: one scan of X tells them apart (only on
        # this error path, collectively on every rank, since every rank holds the same reduced G)
        flag = torch.zeros(1, dtype=torch.float64, device=be.device)
        for x in _chunks(X):
            flag += be.check_finite([x]).to(torch.float64)
        comm.allreduce_sum_(flag)
        if float(flag.item()) != 0.0:
            raise ValueError(_NONFINITE_MSG)
        raise ValueError("Input contains values too large for a float64 Gram matrix: the sum of squares of a "
                         "column overflows float64")
    return G, m, n, s


def eig_desc(C):
    """Eigenvalues (descending, clamped at 0) and eigenvectors as rows of the symmetric matrix C."""
    lam, V = np.linalg.eigh(C)
    lam, V = lam[::-1], V[:, ::-1].T
    return np.maximum(lam, 0.0), np.ascontiguousarray(V)


def project_pass(X, shift, W, out_dtype=None, signs=True):
    """t = (x - shift) W^T per chunk.  Returns (output chunks or None, signs or None): ``out_dtype`` None writes nothing;
    with ``signs``, signs[j] is the sign of the t_ij of largest magnitude (lowest global row on ties) over every rank
    (the kernel's arg-max epilogue, one gather across ranks); without, the epilogue is not run."""
    be, comm = X.backend, X.comm
    k = int(W.shape[0])
    outs = [] if out_dtype is not None else None
    if k == 0:                                    # no components: nothing to project (the reference allows 0)
        if outs is not None:
            outs = [be.empty((int(x.shape[0]), 0), out_dtype) for x in _chunks(X)]
        return outs, (np.ones(0) if signs else None)
    W_dev = torch.as_tensor(np.ascontiguousarray(W, dtype=np.float64)).to(be.device)
    s_dev = None if shift is None else torch.as_tensor(np.ascontiguousarray(shift, dtype=np.float64)).to(be.device)
    rec = be.colmax_new(k) if signs else None
    for x, off in zip(_chunks(X), X.chunk_offsets[:-1]):
        o = be.empty((int(x.shape[0]), k), out_dtype) if out_dtype is not None else None
        be.project_chunk(x, s_dev, W_dev, out=o, colmax=rec, row_offset=X.row_offset + int(off))
        if outs is not None:
            outs.append(o)
    if not signs:
        return outs, None
    return outs, colmax_signs(comm, rec)


def colmax_signs(comm, rec):
    """Per column, the sign (-1 or +1) of the value of largest magnitude in the arg-max records ``rec`` (``colmax_new``)
    of every rank, the lowest global row winning ties: one gather across ranks."""
    k = int(rec.shape[0])
    r = rec.cpu()
    local = (r[:, 0].numpy().copy(), r[:, 1].contiguous().view(torch.int64).numpy().copy(), r[:, 2].numpy().copy())
    parts = comm.allgather_obj(local)
    best_abs = np.full(k, -1.0)
    best_row = np.full(k, np.iinfo(np.int64).max)
    best_val = np.zeros(k)
    for a, row, v in parts:
        take = (a > best_abs) | ((a == best_abs) & (row < best_row) & (a >= 0))
        best_abs = np.where(take, a, best_abs)
        best_row = np.where(take, row, best_row)
        best_val = np.where(take, v, best_val)
    return np.where(best_val < 0, -1.0, 1.0)


def negate_columns(outs, signs):
    """Flip the columns of the output chunks whose sign is -1, in place."""
    neg = np.nonzero(signs < 0)[0]
    if len(neg) and outs:
        idx = torch.as_tensor(neg, device=outs[0].device)
        for o in outs:
            if o.shape[0]:
                o[:, idx] = -o[:, idx]
    return outs


def _torch_dtype(np_dtype):
    return torch.float64 if np.dtype(np_dtype) == np.dtype("float64") else torch.float32


def _per_chunk(X, fn, out_dtype):
    """fn(x as float64 (m, d) tensor) per chunk -> device-resident ChunkedArray of out_dtype (the host-side outputs
    that are not on the hot path)."""
    X = _device_data(X)
    blocks = []
    for x in _chunks(X):
        blocks.append(fn(x.to(torch.float64)).to(out_dtype))
    return ChunkedArray(blocks)


class PCA(_BasePCA):
    """Principal component analysis (API of dask_ml.decomposition.PCA, pca.py:10-170).

    Parameters
    ----------
    n_components : int or None
        Number of components to keep; None keeps ``min(n_samples, n_features)``.  Fractional values and 'mle' are
        not supported (as in the reference).
    copy, tol : ignored
    whiten : bool, default False
    svd_solver : {'auto', 'full', 'tsqr', 'randomized'}
        Every solver runs the exact eigendecomposition of the covariance; 'randomized' keeps the reference's total
        variance and noise variance formulas, and draws ``random_state.randint`` once as the reference does.
    iterated_power : int, ignored (the decomposition is exact)
    random_state : int, RandomState or None

    Attributes
    ----------
    components_, explained_variance_, explained_variance_ratio_, singular_values_, mean_, noise_variance_ :
        numpy, dtype of X (float32 for bf16 rows)
    n_components_, n_samples_, n_features_ : int
    """

    def __init__(self, n_components=None, copy=True, whiten=False, svd_solver="auto", tol=0.0, iterated_power=0,
                 random_state=None):
        self.n_components = n_components
        self.copy = copy
        self.whiten = whiten
        self.svd_solver = svd_solver
        self.tol = tol
        self.iterated_power = iterated_power
        self.random_state = random_state

    def fit(self, X, y=None):
        self._fit(X, transform=False)
        return self

    def fit_transform(self, X, y=None):
        return self._fit(X, transform=True)

    def _fit(self, X, transform):
        solvers = {"full", "auto", "tsqr", "randomized"}
        solver = self.svd_solver
        if solver not in solvers:
            raise ValueError("Invalid solver '{}'. Must be one of {}".format(solver, solvers))
        X = _device_data(X)
        shape = (X.n_global, X.d)
        if self.n_components is None:
            n_components = min(shape)
        elif 0 < self.n_components < 1:
            raise NotImplementedError("Fractional 'n_components' is not currently supported")
        else:
            n_components = self.n_components
        n_samples, n_features = shape
        if solver == "auto":
            if max(shape) <= 500:
                solver = "full"
            elif n_components >= 1 and n_components < 0.8 * min(shape):
                solver = "randomized"
            else:
                solver = "full"
        lower_limit = 1 if solver == "randomized" else 0
        if not (min(n_samples, n_features) >= n_components >= lower_limit):
            raise ValueError("n_components={} must be between {} and min(n_samples, n_features)={} with "
                             "svd_solver='{}'".format(n_components, lower_limit, min(n_samples, n_features), solver))
        if solver == "randomized":
            random_state = check_random_state(self.random_state)
            random_state.randint(np.iinfo("int32").max)       # the reference's seed draw for svd_compressed
        k = int(n_components)
        r = min(n_samples, n_features)

        G, m, n, s = gram_pass(X)

        def algebra():
            mean = s + m / n
            C = G - np.outer(m, m) / n
            lam, V = eig_desc(C)
            return mean, lam[:r], V[:r], float(np.trace(C))

        mean, lam, V, trace = _on_rank0(X.comm, algebra)
        S = np.sqrt(lam)
        explained_variance = lam / (n_samples - 1)
        if solver == "randomized":
            total_var = trace / (n_samples - 1)
        else:
            total_var = explained_variance.sum()
        if k < r:
            if solver == "randomized":
                noise_variance = (total_var - explained_variance[:k].sum()) / (r - k)
            else:
                noise_variance = explained_variance[k:].mean()
        else:
            noise_variance = 0.0
        ev = explained_variance[:k]
        W = V[:k]
        if transform and self.whiten:
            W = W / np.sqrt(ev)[:, None]
        dt = X.np_dtype
        outs, signs = project_pass(X, mean, W, _torch_dtype(dt) if transform else None)

        self.n_samples_, self.n_features_, self.n_components_ = int(n_samples), int(n_features), k
        self.mean_ = mean.astype(dt)
        self.components_ = (V[:k] * signs[:, None]).astype(dt)
        self.explained_variance_ = ev.astype(dt)
        self.explained_variance_ratio_ = (ev / total_var).astype(dt)
        self.singular_values_ = S[:k].astype(dt)
        self.noise_variance_ = dt.type(noise_variance)
        if transform:
            return ChunkedArray(negate_columns(outs, signs))
        return None

    def _projection(self):
        W = self.components_.astype(np.float64)
        if self.whiten:
            W = W / np.sqrt(self.explained_variance_.astype(np.float64))[:, None]
        return W

    def transform(self, X):
        """(n, n_components) projection of X on the components: a device-resident ChunkedArray."""
        check_is_fitted(self, ["mean_", "components_"], all_or_any=all)
        X = _device_data(X)
        outs, _ = project_pass(X, self.mean_.astype(np.float64), self._projection(), _torch_dtype(X.np_dtype),
                               signs=False)
        return ChunkedArray(outs)

    def inverse_transform(self, X):
        check_is_fitted(self, "mean_")
        B = self.components_.astype(np.float64)
        if self.whiten:
            B = np.sqrt(self.explained_variance_.astype(np.float64))[:, None] * B
        dt = _torch_dtype(self.components_.dtype)
        mean = self.mean_.astype(np.float64)

        def fn(x):
            return x @ torch.as_tensor(B, device=x.device) + torch.as_tensor(mean, device=x.device)

        return _per_chunk(X, fn, dt)

    def score_samples(self, X):
        check_is_fitted(self, "mean_")
        precision = np.asarray(self.get_precision(), dtype=np.float64)
        n_features = precision.shape[0]
        const = 0.5 * (n_features * np.log(2.0 * np.pi) - fast_logdet(precision))
        mean = self.mean_.astype(np.float64)

        def fn(x):
            xr = x - torch.as_tensor(mean, device=x.device)
            return -0.5 * (xr * (xr @ torch.as_tensor(precision, device=x.device))).sum(1) - const

        return _per_chunk(X, fn, _torch_dtype(self.components_.dtype))

    def score(self, X, y=None):
        ll = self.score_samples(X)
        tot = sum(float(b.to(torch.float64).sum()) for b in ll.blocks)
        cnt = sum(int(b.shape[0]) for b in ll.blocks)
        return tot / cnt
