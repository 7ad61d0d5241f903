"""TruncatedSVD with the dask_ml.decomposition.TruncatedSVD API, executed by the H100 engine.

Mirrors dask_ml/decomposition/truncated_svd.py (reference @ 0310a90) with the two passes of ``pca.py``.  X is not
centred: the singular values and vectors are those of the uncentred Gram matrix, rebuilt on the host from the shifted
one, X^T X = G + s m^T + m s^T + n s s^T.  ``explained_variance_`` (the column variance of X V^T) and the total
variance come from the centred covariance C = G - m m^T / n: var(X v_j) = v_j^T C v_j / n and sum var(X) = tr(C) / n,
with no extra pass.  Both ``algorithm`` values run the exact eigendecomposition.

Sparse X (a ChunkedArray of torch sparse CSR blocks, one torch CSR tensor, or any scipy.sparse matrix; the intake of the
linear models) is never densified.  Its regime follows from p = n_features:

    p <= SPARSE_EXACT_MAX_P, both algorithms (exact):
        G = X^T X (bkm_gram_weighted_csr_chunk with w = 1), m = X^T 1 (bkm_csc_matvec_chunk), one all-reduce of
        [G | m | n], the host algebra of the dense fit with shift 0, then X V^T with the arg-max epilogue
        (bkm_csr_panel_chunk) for svd_flip's signs.  Without a shift, columns far from zero lose variance to
        cancellation in C = G - m m^T / n, as in scikit-learn's implicit centring.
    p > SPARSE_EXACT_MAX_P, algorithm='randomized' (dask's svd_compressed power iterator); 'tsqr' raises:
        l = min(max(20, k + 10), min(n, p)); Omega (p, l) standard normal from the package's stream (datasets.py) under
        a key drawn from ``random_state`` on rank 0; Y = X Omega, Q = qr(Y); n_iter times Y = X (X^T Q), Q = qr(Y);
        B^T = X^T Q (all-reduced), QR of B^T and an SVD of its R give V and U_b S; U S = Q (U_b S) is the projection
        pass over the float64 Q blocks (bkm_project_chunk), whose epilogue gives svd_flip(u, v)'s signs.
        X Omega and X P are bkm_csr_panel_chunk, X^T Q is bkm_csc_panel_chunk over each block's transpose.  The n-long
        panels are factored by TSQR: a Householder QR per rank, one QR of the gathered l x l factors on rank 0.
"""
import numpy as np
import torch
from sklearn.base import BaseEstimator, TransformerMixin
from sklearn.utils.validation import check_random_state

from .. import datasets
from .._sparse import _sparse_data
from ..chunked import ChunkedArray
from ..cluster.k_means import _NONFINITE_MSG
from ..engine import DeviceData
from .pca import (_device_data, _on_rank0, _torch_dtype, colmax_signs, eig_desc, gram_pass, negate_columns,
                  project_pass)

SPARSE_EXACT_MAX_P = 4096      # the largest n_features whose sparse fit forms the exact (p, p) Gram matrix


def _svd_algebra(G, m, n, s, k):
    """(squared singular values, right singular vectors as rows, explained variance, total variance) of the top k from
    the Gram matrix G and column sums m of n rows shifted by s."""
    U = G + np.outer(s, m) + np.outer(m, s) + n * np.outer(s, s)
    lam, V = eig_desc(U)
    C = G - np.outer(m, m) / n
    ev = np.einsum("ij,jk,ik->i", V[:k], C, V[:k]) / n
    return lam[:k], V[:k], ev, float(np.trace(C)) / n


def _values_dtype(X):
    """numpy dtype of the results for sparse X: float64 when any block's values are float64, else float32."""
    return np.dtype("float64") if any(b[2].dtype == torch.float64 for b in X.blocks) else np.dtype("float32")


def _check_sums(X, h):
    """The first reduction of a sparse fit is finite for finite values: a non-finite one is told apart (NaN / inf in the
    values, or squares that overflow float64) by one scan of the values, on every rank."""
    if np.isfinite(h).all():
        return
    be = X.backend
    flag = torch.zeros(1, dtype=torch.float64, device=be.device)
    for b in X.blocks:
        flag += be.check_finite([b[2].view(-1, 1)]).to(torch.float64)
    X.comm.allreduce_sum_(flag)
    if float(flag.item()) != 0.0:
        raise ValueError(_NONFINITE_MSG)
    raise ValueError("Input contains values too large for a float64 Gram matrix: the sum of squares of a column "
                     "overflows float64")


def panel_pass(X, W, row_offset, out_dtype=None, signs=True):
    """X W per sparse block (``W`` float64 (p, l), numpy or a device tensor).  Returns (output blocks or None, signs or
    None) as ``pca.project_pass`` does: signs[j] is the sign of the (X W)_ij of largest magnitude (lowest global row on
    ties) over every rank."""
    be = X.backend
    l = int(W.shape[1])
    if l == 0:
        outs = [be.empty((int(b[3]), 0), out_dtype) for b in X.blocks] if out_dtype is not None else None
        return outs, (np.ones(0) if signs else None)
    if not torch.is_tensor(W):
        W = torch.as_tensor(np.ascontiguousarray(W, dtype=np.float64)).to(be.device)
    rec = be.colmax_new(l) if signs else None
    outs = [] if out_dtype is not None else None
    for b, off in zip(X.blocks, X.chunk_offsets[:-1]):
        o = be.empty((int(b[3]), l), out_dtype) if out_dtype is not None else None
        be.csr_panel_chunk(b, X.d, W, out=o, colmax=rec, row_offset=row_offset + int(off))
        if outs is not None:
            outs.append(o)
    return outs, (colmax_signs(X.comm, rec) if signs else None)


def tsqr(comm, Y):
    """Q with orthonormal columns and Q R = Y over the rows of every rank (Y float64 (n_local, l) on the device): a
    Householder QR per rank, then one QR of the gathered l x l factors on rank 0, broadcast.  No Cholesky, so Q stays
    orthonormal when Y has rank below l."""
    n, l = int(Y.shape[0]), int(Y.shape[1])
    if n:
        Q, R = torch.linalg.qr(Y)
    else:
        Q, R = Y.new_zeros((0, 0)), Y.new_zeros((0, l))
    Rl = np.zeros((l, l))
    Rl[: R.shape[0]] = R.cpu().numpy()
    parts = comm.allgather_obj(Rl)
    Q2 = _on_rank0(comm, lambda: np.linalg.qr(np.concatenate(parts))[0])
    mine = Q2[comm.rank * l: comm.rank * l + int(R.shape[0])]
    return Q @ torch.as_tensor(np.ascontiguousarray(mine), device=Y.device)


class TruncatedSVD(TransformerMixin, BaseEstimator):
    """Dimensionality reduction by truncated SVD (API of dask_ml.decomposition.TruncatedSVD).

    Parameters
    ----------
    n_components : int, default 2, must be < n_features
    algorithm : {'tsqr', 'randomized'}: both run the exact decomposition, except on sparse X with more than
        ``SPARSE_EXACT_MAX_P`` features, where 'randomized' runs the power iterator and 'tsqr' raises
    n_iter, random_state : the power iterations and the seed of sparse 'randomized' fits; ignored otherwise
    tol : ignored

    Attributes
    ----------
    components_, explained_variance_, explained_variance_ratio_, singular_values_ : numpy, dtype of X (of its values
        for sparse X, integer and bool values giving float64)
    """

    def __init__(self, n_components=2, algorithm="tsqr", n_iter=5, random_state=None, tol=0.0):
        self.algorithm = algorithm
        self.n_components = n_components
        self.n_iter = n_iter
        self.random_state = random_state
        self.tol = tol

    def fit(self, X, y=None):
        self._fit(X, transform=False)
        return self

    def fit_transform(self, X, y=None):
        return self._fit(X, transform=True)

    def _fit(self, X, transform):
        Xs = _sparse_data(X)
        if Xs is not None:
            return self._fit_sparse(Xs, transform)
        X = _device_data(X)
        if self.n_components >= X.d:
            raise ValueError("n_components must be < n_features; got {} >= {}".format(self.n_components, X.d))
        if self.algorithm not in {"tsqr", "randomized"}:
            raise ValueError()
        k = int(self.n_components)
        G, m, n, s = gram_pass(X)
        lam, V, ev, full_var = _on_rank0(X.comm, lambda: _svd_algebra(G, m, n, s, k))
        dt = X.np_dtype
        outs, signs = project_pass(X, None, V, _torch_dtype(dt) if transform else None)
        return self._finish(V, signs, ev, full_var, np.sqrt(lam), dt, outs if transform else None)

    def _finish(self, V, signs, ev, full_var, S, dt, outs):
        self.components_ = (V * signs[:, None]).astype(dt)
        self.explained_variance_ = ev.astype(dt)
        self.explained_variance_ratio_ = (ev / full_var).astype(dt)
        self.singular_values_ = S.astype(dt)
        if outs is not None:
            return ChunkedArray(negate_columns(outs, signs))
        return None

    def _fit_sparse(self, X, transform):
        p = X.d
        if self.n_components >= p:
            raise ValueError("n_components must be < n_features; got {} >= {}".format(self.n_components, p))
        if self.algorithm not in {"tsqr", "randomized"}:
            raise ValueError()
        if p > SPARSE_EXACT_MAX_P and self.algorithm == "tsqr":
            raise ValueError("algorithm='tsqr' runs the exact SVD, which is bounded at %d features for sparse input "
                             "(got %d); use algorithm='randomized'" % (SPARSE_EXACT_MAX_P, p))
        k = int(self.n_components)
        csc = X.transposes()
        row_offset, n = X.global_layout()
        dt = _values_dtype(X)
        odt = _torch_dtype(dt) if transform else None
        be, comm = X.backend, X.comm
        ones = torch.ones(max([1] + X.chunk_rows), dtype=torch.float64, device=be.device)
        if p <= SPARSE_EXACT_MAX_P:
            red = be.zeros((p * p + p + 1,), torch.float64)
            G, m = red[: p * p].view(p, p), red[p * p: p * p + p]
            for i, b in enumerate(X.blocks):
                be.gram_weighted_csr_chunk(b, csc[i], p, ones[: b[3]], G, X.n_slots[i], first=i == 0)
                be.csc_matvec_chunk(csc[i], p, ones[: b[3]], m, first=i == 0)
            red[-1] = float(X.n_local)
            comm.allreduce_sum_(red)
            h = red.cpu().numpy()
            _check_sums(X, h)
            G, m = h[: p * p].reshape(p, p).copy(), h[p * p: p * p + p].copy()
            lam, V, ev, full_var = _on_rank0(comm, lambda: _svd_algebra(G, m, n, np.zeros(p), k))
            outs, signs = panel_pass(X, V.T, row_offset, odt)
            return self._finish(V, signs, ev, full_var, np.sqrt(lam), dt, outs)

        # the first reduction: [column sums | sum of the squared values | n]
        red = be.zeros((p + 2,), torch.float64)
        for i, b in enumerate(X.blocks):
            be.csc_matvec_chunk(csc[i], p, ones[: b[3]], red, first=i == 0)
            red[p] += b[2].to(torch.float64).square().sum()
        red[p + 1] = float(X.n_local)
        comm.allreduce_sum_(red)
        h = red.cpu().numpy()
        _check_sums(X, h)
        m, sq = h[:p], float(h[p])
        full_var = sq / n - float(m @ m) / n ** 2            # sum_c var(X_c)

        l = min(max(20, k + 10), min(n, p))                  # dask's compression_level
        key = _on_rank0(comm, lambda: datasets._draw_key(check_random_state(self.random_state)))
        off = [int(o) for o in X.chunk_offsets]
        Y = be.empty((X.n_local, l), torch.float64)

        def x_times(W):                                      # Y = X W
            for i, b in enumerate(X.blocks):
                be.csr_panel_chunk(b, p, W, out=Y[off[i]: off[i + 1]])

        def xt_times(Q):                                     # X^T Q over every rank
            Z = be.zeros((p, l), torch.float64)
            for i in range(len(X.blocks)):
                be.csc_panel_chunk(csc[i], p, Q[off[i]: off[i + 1]], Z, first=i == 0)
            comm.allreduce_sum_(Z)
            return Z

        x_times(datasets._normal_panel(key, p, l, be.device))
        Q = tsqr(comm, Y)
        for _ in range(int(self.n_iter)):
            x_times(xt_times(Q))
            Q = tsqr(comm, Y)
        Bt = xt_times(Q)                                     # (p, l), the same on every rank
        Q2, R = torch.linalg.qr(Bt)
        Ur, Sr, Vrt = np.linalg.svd(R.cpu().numpy())         # B = Q^T X = (Vrt^T) diag(Sr) (Q2 Ur)^T
        S, Ub = Sr[:k], Vrt.T[:, :k]
        V = (Q2 @ torch.as_tensor(np.ascontiguousarray(Ur[:, :k]), device=Q2.device)).T.cpu().numpy()
        qsum = Q.sum(0)
        comm.allreduce_sum_(qsum)
        mean = S * (qsum.cpu().numpy() @ Ub) / n             # column means of U S, with |u_j| = 1
        ev = S ** 2 / n - mean ** 2
        Qd = DeviceData([Q[off[i]: off[i + 1]] for i in range(len(X.blocks))] or [Q], be, comm)
        outs, signs = project_pass(Qd, None, (Ub * S).T, odt)
        return self._finish(V, signs, ev, full_var, S, dt, outs)

    def transform(self, X, y=None):
        """X V^T: a device-resident ChunkedArray."""
        Xs = _sparse_data(X)
        if Xs is not None:
            if Xs.d != self.components_.shape[1]:
                raise ValueError("X has %d features, but TruncatedSVD is expecting %d features as input"
                                 % (Xs.d, self.components_.shape[1]))
            outs, _ = panel_pass(Xs, self.components_.astype(np.float64).T, 0, _torch_dtype(_values_dtype(Xs)),
                                 signs=False)
            return ChunkedArray(outs)
        X = _device_data(X)
        outs, _ = project_pass(X, None, self.components_.astype(np.float64), _torch_dtype(X.np_dtype), signs=False)
        return ChunkedArray(outs)

    def inverse_transform(self, X):
        from .pca import _per_chunk

        B = self.components_.astype(np.float64)
        return _per_chunk(X, lambda x: x @ torch.as_tensor(B, device=x.device), _torch_dtype(self.components_.dtype))
