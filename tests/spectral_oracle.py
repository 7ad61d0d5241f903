"""float64 restatement of the reference's Nystrom embedding (dask_ml/cluster/spectral.py:209-287), in two forms.

``embed_unfused`` follows the reference step by step: the (l, l) block A and the (l, n - l) block B, ``pinv(A)``,
d1 / d2, the SVD of A2, Eq. 16 and the row normalisation, then the rows put back in input order (what
``_slice_mostly_sorted`` does).  ``embed_fused`` is the form the engine computes: column sums over all rows, W (l, k)
and e_i / ||e_i|| with e_i = sum_j K(x_i, keep_j) W_j, optionally with the per-row shift of the kernels.
"""
import numpy as np
from scipy.linalg import pinv, svd


def rbf(X, Y, gamma):
    X = np.asarray(X, dtype=np.float64)
    Y = np.asarray(Y, dtype=np.float64)
    d2 = np.maximum((X * X).sum(1)[:, None] - 2.0 * X @ Y.T + (Y * Y).sum(1)[None, :], 0.0)
    return np.exp(-gamma * d2)


def keep_rows(n, l, seed, kmeans_branch=True):
    """The reference's draws (spectral.py:185-225): the KMeans seed (default branch only), then the sorted keep rows."""
    rng = np.random.RandomState(seed)
    km_seed = rng.randint(2 ** 32 - 1) if kmeans_branch else None
    keep = rng.choice(np.arange(n), l, replace=False)
    keep.sort()
    return keep, km_seed


def embed_unfused(X, keep, k, gamma):
    """(U2 (n, k) in input order, S[:k])."""
    X = np.asarray(X, dtype=np.float64)
    n, l = len(X), len(keep)
    inds = np.arange(n)
    rest = ~np.isin(inds, keep)
    A = rbf(X[keep], X[keep], gamma)
    B = rbf(X[keep], X[rest], gamma)
    a, b1, b2 = A.sum(0), B.sum(1), B.sum(0)
    inner = pinv(A).dot(b1)
    d1_si = 1 / np.sqrt(a + b1)
    d2_si = 1 / np.sqrt(b2 + B.T.dot(inner))
    A2 = d1_si.reshape(-1, 1) * A * d1_si.reshape(1, -1)
    B2 = d1_si.reshape(-1, 1) * B * d2_si.reshape(1, -1)
    U, S, _ = svd(A2)
    V2 = np.sqrt(float(l) / n) * np.vstack([A2, B2.T]).dot(U[:, :k]).dot(np.diag(1.0 / np.sqrt(S[:k])))
    U2 = (V2.T / np.sqrt((V2 ** 2).sum(1))).T
    out = np.empty_like(U2)
    out[np.concatenate([keep, inds[rest]])] = U2
    return out, S[:k]


def weights(X_keep, c, k, gamma):
    """(W (l, k), S[:k]) from the keep rows and the column sums over all rows."""
    A = rbf(X_keep, X_keep, gamma)
    d1_si = 1.0 / np.sqrt(c)
    A2 = d1_si.reshape(-1, 1) * A * d1_si.reshape(1, -1)
    U, S, _ = svd(A2)
    return d1_si.reshape(-1, 1) * U[:, :k] * (1.0 / np.sqrt(S[:k])).reshape(1, -1), S[:k]


def colsum(X, X_keep, gamma):
    return rbf(X, X_keep, gamma).sum(0)


def project(X, X_keep, W, gamma, shift=True):
    """e_i / ||e_i||; ``shift`` subtracts min_j d^2 inside the exponential (it cancels in the normalisation)."""
    X = np.asarray(X, dtype=np.float64)
    Xk = np.asarray(X_keep, dtype=np.float64)
    d2 = np.maximum((X * X).sum(1)[:, None] - 2.0 * X @ Xk.T + (Xk * Xk).sum(1)[None, :], 0.0)
    m = d2.min(1, keepdims=True) if shift else 0.0
    e = np.exp(-gamma * (d2 - m)) @ W
    return e / np.sqrt((e * e).sum(1, keepdims=True))


def embed_fused(X, keep, k, gamma, shift=True):
    X = np.asarray(X, dtype=np.float64)
    W, S = weights(X[keep], colsum(X, X[keep], gamma), k, gamma)
    return project(X, X[keep], W, gamma, shift), S


def procrustes_err(got, want):
    """max |got R - want| over the orthogonal k x k R that best aligns got to want (absorbs SVD sign choices)."""
    got = np.asarray(got, dtype=np.float64)
    want = np.asarray(want, dtype=np.float64)
    u, _, vt = np.linalg.svd(got.T @ want)
    return float(np.abs(got @ (u @ vt) - want).max())
