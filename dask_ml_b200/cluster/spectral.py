"""SpectralClustering with the dask_ml.cluster.SpectralClustering API, executed by the H100 engine.

Mirrors dask_ml/cluster/spectral.py (reference @ 0310a90): the Nystrom approximation of Fowlkes et al. (2004) with
``l = n_components`` sampled rows ("keep").  The reference forms the (l, l) kernel block A and the (l, n - l) block B,
then ``pinv(A)``, the SVD of the normalised A2 and ``V2 = [A2; B2^T] U[:, :k] diag(S^-1/2)`` (spectral.py:237-282).
Each row of V2 is normalised before KMeans, which cancels the row factor d2 and the sqrt(l / n) of Eq. 16, so the
embedding needs no (n, l) matrix at all:

    c_j  = sum over ALL rows i of K(x_i, keep_j)                  (= a + b1 of the reference)
    A2   = diag(c^-1/2) K(keep, keep) diag(c^-1/2);   U, S, _ = svd(A2)
    W    = diag(c^-1/2) U[:, :k] diag(S[:k]^-1/2)                 (l, k)
    U2_i = e_i / ||e_i||,   e_i = sum_j K(x_i, keep_j) W_j

The same formula holds for keep rows and the other rows, so rows stay in input order (the reference's
``_slice_mostly_sorted`` reordering has nothing to undo).  For ``affinity='rbf'`` the two sums over X are two
streaming passes of CUDA kernels (``bkm_kernel_colsum_chunk`` and ``bkm_nystrom_embed_chunk``; on sparse CSR blocks
``bkm_csr_kernel_colsum_chunk`` and ``bkm_csr_nystrom_embed_chunk``); the rest is (l, l) host algebra in float64 and
one ``KMeans.fit`` on the device-resident embedding.
"""
import logging

import numpy as np
import scipy.sparse
import torch
from sklearn.base import BaseEstimator, ClusterMixin
from sklearn.utils import check_random_state

from .._sparse import _SparseData, _sparse_data
from ..chunked import ChunkedArray, is_dask_dataframe
from ..engine import DeviceData
from ..utils import check_array
from . import k_means as _km
from .k_means import KMeans, _NONFINITE_MSG

logger = logging.getLogger(__name__)

# the reference's kernel names (dask_ml/metrics/pairwise.py:165-175); only 'rbf' has an engine epilogue
PAIRWISE_KERNEL_FUNCTIONS = ("rbf", "linear", "polynomial", "sigmoid")


class SpectralClustering(BaseEstimator, ClusterMixin):
    """Spectral clustering through the Nystrom approximation (API of dask_ml.cluster.SpectralClustering,
    spectral.py:22-173).

    Parameters
    ----------
    n_clusters : int, default 8
        Dimension of the projection subspace and number of clusters of the default label assignment.
    random_state : int, RandomState or None
        Draws the ``n_components`` keep rows and, for ``assign_labels='kmeans'``, the KMeans seed.  ``None`` draws one
        seed on rank 0 and shares it, so every rank samples the same keep rows.
    gamma : float or None, default 1.0
        rbf kernel coefficient; ``None`` means ``1 / n_features``.
    affinity : 'rbf' or callable
        'rbf' runs on the engine.  'linear', 'polynomial' and 'sigmoid' raise NotImplementedError (as
        ``metrics.pairwise_kernels`` does).  A callable ``f(X_keep, Y=None, **kernel_params)`` is evaluated per chunk
        and reduced in float64 torch.
    assign_labels : 'kmeans', 'sklearn-kmeans' or an estimator
        'kmeans' fits this package's ``KMeans`` on the device-resident embedding; the others receive the embedding as
        a host ndarray.
    degree, coef0, kernel_params :
        Passed to a callable affinity (``gamma``, ``degree`` and ``coef0`` are added to ``kernel_params``).
    n_components : int, default 100
        Number of rows of X sampled for the Nystrom approximation.
    kmeans_params : dict
        Applied to the label-assignment estimator with ``set_params``.
    eigen_solver, n_init, n_neighbors, eigen_tol, n_jobs, persist_embedding :
        Accepted and ignored, as in the reference; the embedding is always resident.

    Attributes
    ----------
    assign_labels_ : the fitted label-assignment estimator
    labels_ : its ``labels_`` (a device-resident ChunkedArray for ``'kmeans'``)
    eigenvalues_ : np.ndarray (n_clusters,) float64, the largest singular values of A2
    """

    def __init__(
        self,
        n_clusters=8,
        eigen_solver=None,
        random_state=None,
        n_init=10,
        gamma=1.0,
        affinity="rbf",
        n_neighbors=10,
        eigen_tol=0.0,
        assign_labels="kmeans",
        degree=3,
        coef0=1,
        kernel_params=None,
        n_jobs=1,
        n_components=100,
        persist_embedding=False,
        kmeans_params=None,
    ):
        self.n_clusters = n_clusters
        self.eigen_solver = eigen_solver
        self.random_state = random_state
        self.n_init = n_init
        self.gamma = gamma
        self.affinity = affinity
        self.n_neighbors = n_neighbors
        self.eigen_tol = eigen_tol
        self.assign_labels = assign_labels
        self.degree = degree
        self.coef0 = coef0
        self.kernel_params = kernel_params
        self.n_jobs = n_jobs
        self.n_components = n_components
        self.persist_embedding = persist_embedding
        self.kmeans_params = kmeans_params

    def _check_array(self, X):
        try:
            import pandas as pd

            if isinstance(X, pd.DataFrame):
                X = X.values
        except ImportError:  # pragma: no cover
            pass
        if is_dask_dataframe(X):
            raise TypeError("Cannot fit on dask.dataframe due to unknown partition lengths.")
        if isinstance(X, (DeviceData, _SparseData)):
            return X
        sp = _sparse_data(X)                    # sparse CSR blocks (engine extension: the reference rejects them)
        if sp is not None:
            sp.check_finite()
            return sp
        X = check_array(X, accept_dask_dataframe=False, accept_unknown_chunks=False, accept_sparse=False)
        return _km._to_device_data(X)

    def __sklearn_tags__(self):
        tags = super().__sklearn_tags__()
        tags.input_tags.sparse = True           # sparse CSR blocks run through the sparse Nystrom passes
        return tags

    def fit(self, X, y=None):
        X = self._check_array(X)
        comm = X.comm
        l = int(self.n_components)
        k = int(self.n_clusters)
        metric = self.affinity
        # the same keep rows on every rank: without a seed, rank 0 draws one (k_means._as_random_state)
        rng = _km._as_random_state(None, comm) if self.random_state is None else check_random_state(self.random_state)

        # label assignment (spectral.py:188-207)
        if isinstance(self.assign_labels, str):
            if self.assign_labels == "kmeans":
                km = KMeans(n_clusters=k, random_state=rng.randint(2 ** 32 - 1))
            elif self.assign_labels == "sklearn-kmeans":
                import sklearn.cluster

                km = sklearn.cluster.KMeans(n_clusters=k, random_state=rng)
            else:
                raise ValueError("Unknown 'assign_labels' {!r}".format(self.assign_labels))
        elif isinstance(self.assign_labels, BaseEstimator):
            km = self.assign_labels
        else:
            raise TypeError("Invalid type {} for 'assign_labels'".format(type(self.assign_labels)))
        if self.kmeans_params:
            km.set_params(**self.kmeans_params)

        n = X.n_global
        if n <= l:
            raise ValueError("'n_components' must be smaller than the number of samples."
                             " Got {} components and {} samples".format(l, n))

        params = dict(self.kernel_params or {})
        params["gamma"] = self.gamma
        params["degree"] = self.degree
        params["coef0"] = self.coef0

        keep = rng.choice(np.arange(n), l, replace=False)
        keep.sort()

        if isinstance(metric, str):
            if metric not in PAIRWISE_KERNEL_FUNCTIONS:
                raise ValueError("Unknown affinity metric name '{}'. Expected one of '{}'".format(
                    metric, list(PAIRWISE_KERNEL_FUNCTIONS)))
            if metric != "rbf":
                raise NotImplementedError("kernel %r is outside the GPU engine: only 'rbf' runs on it" % metric)
        elif not callable(metric):
            raise TypeError("Unexpected type for 'affinity' '{}'. Must be string kernel name, array, or callable"
                            .format(type(metric).__name__))

        if k > l:
            # checked on every rank before any collective (the weights below are computed on rank 0 only)
            raise ValueError("n_clusters=%d exceeds n_components=%d: the embedding has at most n_components columns"
                             % (k, l))
        X_keep = X.global_rows(keep)
        if callable(metric):
            passes = _CallablePasses(X, X_keep, metric, params)
        elif isinstance(X, _SparseData):
            passes = _SparseRbfPasses(X, X_keep, self.gamma)
        else:
            passes = _RbfPasses(X, X_keep, self.gamma)

        # pass 1: column sums over every row of every rank -> A2, its SVD and W (rank 0, broadcast)
        c = passes.colsum()
        A = passes.keep_block()
        W = S = err = None
        if comm.rank == 0:
            try:
                W, S = _nystrom_weights(A, c, k)
            except Exception as e:                     # handed to every rank, so that none waits in the broadcast
                err = e
        W, S, err = comm.bcast_obj((W, S, err))
        if err is not None:
            raise err
        if W is None:
            raise ValueError(_NONFINITE_MSG)
        # pass 2: the embedding rows, in input order
        emb = passes.embed(W)

        if isinstance(km, KMeans):
            data = DeviceData(emb, X.backend, comm)
            flag = X.backend.check_finite(emb).to(torch.float64)
            comm.allreduce_sum_(flag)
            if float(flag.item()) != 0.0:
                raise ValueError(_NONFINITE_MSG)          # the reference's KMeans rejects the NaN rows of U2
            km.fit(data)
        else:
            U2 = np.concatenate([e.cpu().numpy() for e in emb], axis=0) if emb else np.empty((0, k))
            if comm.world > 1:
                U2 = np.concatenate(comm.allgather_obj(U2), axis=0)
            km.fit(U2)

        self.assign_labels_ = km
        self.labels_ = km.labels_
        self.eigenvalues_ = S
        return self


def _nystrom_weights(A, c, k):
    """(W (l, k), S[:k]) from the keep block A and the column sums c, or (None, None) when S[:k] has a zero (the
    reference's embedding is then non-finite)."""
    from scipy.linalg import svd

    d1_si = 1.0 / np.sqrt(c)
    A2 = d1_si.reshape(-1, 1) * A * d1_si.reshape(1, -1)
    U, S, _ = svd(A2)
    S = S[:k]
    if not np.all(S > 0):
        return None, None
    W = d1_si.reshape(-1, 1) * U[:, :k] * (1.0 / np.sqrt(S)).reshape(1, -1)
    return np.ascontiguousarray(W), np.asarray(S, dtype=np.float64)


def _embedding_buffer(be, m, k, dtype):
    """(m, k) embedding block whose row pitch is padded like ``CudaBackend.to_device`` pads fp32 rows, so that the
    KMeans fit reads it in place on the tensor path."""
    pitch = (k + 3) // 4 * 4 if (dtype == torch.float32 and k % 4 and k <= 64) else k
    return be.zeros((m, pitch), dtype)[:, :k]


class _RbfPasses(object):
    """K(x, c) = exp(-gamma ||x - c||^2): the two passes run in the engine's kernels."""

    def __init__(self, X, X_keep, gamma):
        if X.dtype == torch.bfloat16:
            # no bf16 epilogue: the rows go through in float32, as metrics.pairwise does for bf16 input
            X = DeviceData([c.to(torch.float32) for c in X.chunks], X.backend, X.comm)
        self.X, self.be = X, X.backend
        self.l = int(X_keep.shape[0])
        self.gamma = 1.0 / X.d if gamma is None else float(gamma)
        self.keep64 = np.asarray(X_keep, dtype=np.float64)
        self.pack = self.be.pack_centers(torch.as_tensor(self.keep64).to(self.be.device), X.dtype)

    def colsum(self):
        be, X = self.be, self.X
        c = be.zeros((self.l,), torch.float64)
        first = True
        for x in X.chunks:
            be.kernel_colsum(x, self.pack, self.l, self.gamma, c, first=first)
            first = False
        X.comm.allreduce_sum_(c)
        return c.cpu().numpy()

    def keep_block(self):
        from sklearn.metrics.pairwise import rbf_kernel

        return rbf_kernel(self.keep64, gamma=self.gamma)

    def embed(self, W):
        be, X = self.be, self.X
        k = int(W.shape[1])
        Wd = torch.as_tensor(np.ascontiguousarray(W)).to(device=be.device, dtype=X.dtype)
        out = []
        for x in X.chunks:
            e = _embedding_buffer(be, int(x.shape[0]), k, X.dtype)
            if int(x.shape[0]):
                be.nystrom_embed(x, self.pack, self.l, self.gamma, Wd, e)
            out.append(e)
        return out


class _SparseRbfPasses(object):
    """``_RbfPasses`` on sparse CSR blocks: the keep rows (a host CSR) densified on the device into a sparse pack, which
    takes 8 (p + 1) l bytes (839 MB at p = 2^20 features and l = 100); every distance and kernel value is float64.  The
    embedding has the dtype of the values (float32 or float64)."""

    def __init__(self, X, X_keep, gamma):
        self.X, self.be = X, X.backend
        self.l = int(X_keep.shape[0])
        self.gamma = 1.0 / X.d if gamma is None else float(gamma)
        self.keep = X_keep
        self.pack = self.be.sparse_pack_centers(_km._dense_centres(X_keep, X.d, self.be))

    def colsum(self):
        be, X = self.be, self.X
        c = be.zeros((self.l,), torch.float64)
        for i, blk in enumerate(X.blocks):
            be.csr_kernel_colsum(blk, X.d, self.pack, self.l, self.gamma, c, first=i == 0)
        X.comm.allreduce_sum_(c)
        return c.cpu().numpy()

    def keep_block(self):
        from sklearn.metrics.pairwise import rbf_kernel

        return rbf_kernel(self.keep.astype(np.float64), gamma=self.gamma)

    def embed(self, W):
        be, X = self.be, self.X
        k = int(W.shape[1])
        dt = torch.float32 if X.dtype == torch.float32 else torch.float64
        Wd = torch.as_tensor(np.ascontiguousarray(W, dtype=np.float64)).to(be.device)
        out = []
        for blk in X.blocks:
            e = _embedding_buffer(be, int(blk[3]), k, dt)
            if int(blk[3]):
                be.csr_nystrom_embed(blk, X.d, self.pack, self.l, self.gamma, Wd, e)
            out.append(e)
        return out


def _host_parts(X):
    """(rows, host block) per block of X: numpy rows, or a scipy CSR for sparse X."""
    if isinstance(X, _SparseData):
        for crow, col, val, n in X.blocks:
            yield int(n), scipy.sparse.csr_matrix((val.cpu().numpy(), col.cpu().numpy(), crow.cpu().numpy()),
                                                  shape=(int(n), X.d))
        return
    for x in X.chunks:
        yield int(x.shape[0]), (x.float() if x.dtype == torch.bfloat16 else x).cpu().numpy()


class _CallablePasses(object):
    """A user kernel ``metric(X_keep, Y=None, **params)``: evaluated per chunk (numpy rows, or scipy CSR blocks for
    sparse X), reduced in float64 torch."""

    def __init__(self, X, X_keep, metric, params):
        self.X, self.be = X, X.backend
        self.X_keep, self.metric, self.params = X_keep, metric, params
        self.l = int(X_keep.shape[0])

    def _block(self, xh):
        """K(keep, x) as a float64 (l, m) tensor on the device, for the host block ``xh``."""
        K = self.metric(self.X_keep, xh, **self.params)
        if isinstance(K, ChunkedArray):
            K = [b if isinstance(b, torch.Tensor) else torch.as_tensor(np.asarray(b)) for b in K.blocks]
            K = torch.cat([b.to(self.be.device) for b in K], dim=0)
        elif not isinstance(K, torch.Tensor):
            K = torch.as_tensor(np.asarray(K))
        return K.to(device=self.be.device, dtype=torch.float64)

    def colsum(self):
        c = self.be.zeros((self.l,), torch.float64)
        for m, xh in _host_parts(self.X):
            if m:
                c += self._block(xh).sum(1)
        self.X.comm.allreduce_sum_(c)
        return c.cpu().numpy()

    def keep_block(self):
        K = self.metric(self.X_keep, **self.params)
        if isinstance(K, ChunkedArray):
            K = K.compute()
        if isinstance(K, torch.Tensor):
            K = K.cpu().numpy()
        return np.asarray(K, dtype=np.float64)

    def embed(self, W):
        dt = torch.float64 if self.X.dtype == torch.float64 else torch.float32
        Wd = torch.as_tensor(np.ascontiguousarray(W)).to(self.be.device)
        out = []
        for m, xh in _host_parts(self.X):
            e = _embedding_buffer(self.be, m, int(W.shape[1]), dt)
            if m:
                v = self._block(xh).T @ Wd
                e.copy_(v / torch.sqrt((v * v).sum(1, keepdim=True)))
            out.append(e)
        return out
