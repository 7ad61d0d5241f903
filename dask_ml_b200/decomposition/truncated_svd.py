"""TruncatedSVD with the dask_ml.decomposition.TruncatedSVD API, executed by the H100 engine.

Mirrors dask_ml/decomposition/truncated_svd.py (reference @ 0310a90) with the two passes of ``pca.py``.  X is not
centred: the singular values and vectors are those of the uncentred Gram matrix, rebuilt on the host from the shifted
one, X^T X = G + s m^T + m s^T + n s s^T.  ``explained_variance_`` (the column variance of X V^T) and the total
variance come from the centred covariance C = G - m m^T / n: var(X v_j) = v_j^T C v_j / n and sum var(X) = tr(C) / n,
with no extra pass.  Both ``algorithm`` values run the exact eigendecomposition.
"""
import numpy as np
from sklearn.base import BaseEstimator, TransformerMixin

from ..chunked import ChunkedArray
from .pca import (_device_data, _on_rank0, _torch_dtype, eig_desc, gram_pass, negate_columns, project_pass)


class TruncatedSVD(TransformerMixin, BaseEstimator):
    """Dimensionality reduction by truncated SVD (API of dask_ml.decomposition.TruncatedSVD).

    Parameters
    ----------
    n_components : int, default 2, must be < n_features
    algorithm : {'tsqr', 'randomized'}: both run the exact decomposition
    n_iter, random_state, tol : ignored (the decomposition is exact)

    Attributes
    ----------
    components_, explained_variance_, explained_variance_ratio_, singular_values_ : numpy, dtype of X
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
        X = _device_data(X)
        if self.n_components >= X.d:
            raise ValueError("n_components must be < n_features; got {} >= {}".format(self.n_components, X.d))
        if self.algorithm not in {"tsqr", "randomized"}:
            raise ValueError()
        k = int(self.n_components)
        G, m, n, s = gram_pass(X)

        def algebra():
            U = G + np.outer(s, m) + np.outer(m, s) + n * np.outer(s, s)
            lam, V = eig_desc(U)
            C = G - np.outer(m, m) / n
            ev = np.einsum("ij,jk,ik->i", V[:k], C, V[:k]) / n
            return lam[:k], V[:k], ev, float(np.trace(C)) / n

        lam, V, ev, full_var = _on_rank0(X.comm, algebra)
        dt = X.np_dtype
        outs, signs = project_pass(X, None, V, _torch_dtype(dt) if transform else None)
        self.components_ = (V * signs[:, None]).astype(dt)
        self.explained_variance_ = ev.astype(dt)
        self.explained_variance_ratio_ = (ev / full_var).astype(dt)
        self.singular_values_ = np.sqrt(lam).astype(dt)
        if transform:
            return ChunkedArray(negate_columns(outs, signs))
        return None

    def transform(self, X, y=None):
        """X V^T: a device-resident ChunkedArray."""
        X = _device_data(X)
        outs, _ = project_pass(X, None, self.components_.astype(np.float64), _torch_dtype(X.np_dtype), signs=False)
        return ChunkedArray(outs)

    def inverse_transform(self, X):
        import torch

        from .pca import _per_chunk

        B = self.components_.astype(np.float64)
        return _per_chunk(X, lambda x: x @ torch.as_tensor(B, device=x.device), _torch_dtype(self.components_.dtype))
