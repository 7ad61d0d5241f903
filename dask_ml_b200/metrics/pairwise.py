"""GPU versions of the three distance operators the KMeans path uses
(dask_ml/metrics/pairwise.py:18-52, 55-66, 69-97).  Only the euclidean metric exists on this
path; every result is a device-resident ``ChunkedArray`` with the reference's dtypes.  ``pairwise_distances_argmin_min``
and ``euclidean_distances`` also take sparse CSR X (any form ``KMeans`` takes) against a dense Y."""
import numpy as np
import torch

from ..chunked import ChunkedArray


def _prep(X, Y):
    from ..cluster.k_means import _to_device_data

    X = _to_device_data(X, check_finite=False)
    Y = np.asarray(Y)
    if Y.ndim != 2 or Y.shape[1] != X.d:
        raise ValueError(
            "Incompatible dimension for X and Y matrices: X.shape[1] == %d while Y.shape[1] == %d"
            % (X.d, Y.shape[1] if Y.ndim == 2 else -1)
        )
    be = X.backend
    C = torch.as_tensor(np.ascontiguousarray(Y, dtype=np.float64)).to(be.device)
    pack = be.pack_centers(C, X.dtype)
    return X, be, pack, int(Y.shape[0])


def _sparse_x(X):
    """``_SparseData`` for sparse X, else None."""
    from .._sparse import _SparseData, _sparse_data

    return X if isinstance(X, _SparseData) else _sparse_data(X)


def _sparse_prep(X, Y):
    """Sparse X against dense Y: (X, backend, the sparse pack of Y, len(Y), Y's dtype)."""
    Y = np.asarray(Y)
    if Y.ndim != 2 or Y.shape[1] != X.d:
        raise ValueError(
            "Incompatible dimension for X and Y matrices: X.shape[1] == %d while Y.shape[1] == %d"
            % (X.d, Y.shape[1] if Y.ndim == 2 else -1)
        )
    be = X.backend
    C = torch.as_tensor(np.ascontiguousarray(Y, dtype=np.float64)).to(be.device)
    return be, be.sparse_pack_centers(C), int(Y.shape[0]), Y.dtype


def pairwise_distances_argmin_min(X, Y, axis=1, metric="euclidean", batch_size=None, metric_kwargs=None):
    """Per row of X: index of and distance to the nearest row of Y (pairwise.py:18-52).

    Returns ``(argmins int64, mins float64)`` like the reference (pairwise.py:41-49).  ``mins`` is
    the euclidean distance, or its square with ``metric_kwargs={'squared': True}``.
    """
    if type(Y).__module__.startswith("dask"):
        raise TypeError("`Y` must be a numpy array")
    if metric not in ("euclidean", "sqeuclidean", "l2"):
        raise NotImplementedError("only the euclidean metric is on the GPU KMeans path, got %r" % (metric,))
    if axis != 1:
        raise NotImplementedError("axis must be 1")
    squared = bool((metric_kwargs or {}).get("squared", False)) or metric == "sqeuclidean"
    Xs = _sparse_x(X)
    if Xs is not None:
        be, pack, k, _ = _sparse_prep(Xs, Y)
        argmins, mins = [], []
        for blk in Xs.blocks:
            n = int(blk[3])
            lab = be.empty((n,), torch.int32)
            mn = be.empty((n,), torch.float64)
            be.csr_assign_chunk(blk, Xs.d, pack, k, labels=lab, min_dist=mn, squared=squared)
            argmins.append(lab.to(torch.int64))
            mins.append(mn)
        return ChunkedArray(argmins), ChunkedArray(mins)
    X, be, pack, k = _prep(X, Y)
    acc = be.zeros((1,), torch.float64)
    argmins, mins = [], []
    for x in X.chunks:
        n = int(x.shape[0])
        lab = be.empty((n,), torch.int32)
        mn = be.empty((n,), X.out_dtype)
        be.assign_chunk(x, pack, k, lab, mn, squared, acc)
        argmins.append(lab.to(torch.int64))
        mins.append(mn.to(torch.float64))
    return ChunkedArray(argmins), ChunkedArray(mins)


def pairwise_distances(X, Y, metric="euclidean", n_jobs=None, **kwargs):
    """Full (n, len(Y)) euclidean distance blocks (pairwise.py:55-66)."""
    if type(Y).__module__.startswith("dask"):
        raise TypeError("`Y` must be a numpy array")
    if metric != "euclidean":
        raise NotImplementedError("only the euclidean metric is on the GPU KMeans path, got %r" % (metric,))
    return euclidean_distances(X, Y)


def _distance_blocks(X, Y, mode, gamma=0.0):
    """(n_i, len(Y)) blocks of distances / squared distances / rbf values, one per chunk of X.  Y wider than 256 rows is
    cut into column blocks of 256 (the width of the tensor-path kernel); every block is one pass of the chunk."""
    be = X.backend
    Y64 = np.ascontiguousarray(Y, dtype=np.float64)
    k = int(Y64.shape[0])
    step = 256
    outs = [be.empty((m, k), X.dtype) for m in X.chunk_rows]
    for c0 in range(0, k, step):
        c1 = min(k, c0 + step)
        C = torch.as_tensor(Y64[c0:c1]).to(be.device)
        pack = be.pack_centers(C, X.dtype)
        for x, out in zip(X.chunks, outs):
            if int(x.shape[0]):
                be.transform_chunk(x, pack, c1 - c0, out[:, c0:c1], mode=mode, gamma=gamma)
    return outs


def _as_device(X):
    from ..cluster.k_means import _to_device_data
    from ..engine import DeviceData

    X = _to_device_data(X, check_finite=False)
    if X.dtype == torch.bfloat16:
        # the full distance matrix of bf16 rows is produced in float32 (no bf16 transform kernel)
        X = DeviceData([c.to(torch.float32) for c in X.chunks], X.backend, X.comm)
    return X


def euclidean_distances(X, Y=None, Y_norm_squared=None, squared=False, X_norm_squared=None):
    """sqrt(max(||x||^2 - 2 x.y + ||y||^2, 0)) for every (row of X, row of Y)  (pairwise.py:69-97).

    The result has the dtype of X (float64 when Y is float64, like ``-2 * dot(X, Y.T) + XX + YY`` in the reference).
    ``Y=None`` means X against itself.  The kernels compute the row norms themselves; when ``X_norm_squared`` /
    ``Y_norm_squared`` are passed they are validated AND used as the reference uses them (pairwise.py:72-91): the
    difference to the true norms is added to the squared distances before the clamp / square root.
    """
    from ..engine import DeviceData

    Xs = _sparse_x(X)
    if Xs is not None:
        if X_norm_squared is not None or Y_norm_squared is not None:
            raise NotImplementedError("X_norm_squared / Y_norm_squared are not supported for sparse X")
        if Y is None:
            raise NotImplementedError("sparse X needs a dense Y")
        be, pack, k, ydt = _sparse_prep(Xs, Y)
        # dtype of -2 * dot(X, Y.T) + XX + YY: float32 only when both are float32
        odt = torch.float32 if Xs.dtype == torch.float32 and ydt == np.float32 else torch.float64
        outs = []
        for blk in Xs.blocks:
            out = be.empty((int(blk[3]), k), odt)
            be.csr_assign_chunk(blk, Xs.d, pack, k, out=out, mode=2 if squared else 1)
            outs.append(out)
        return ChunkedArray(outs)
    X = _as_device(X)
    if Y is None:
        Y = X.to_host()
    Y = np.asarray(Y)
    if Y.ndim != 2 or Y.shape[1] != X.d:
        raise ValueError(
            "Incompatible dimension for X and Y matrices: X.shape[1] == %d while Y.shape[1] == %d"
            % (X.d, Y.shape[1] if Y.ndim == 2 else -1)
        )
    if X.dtype == torch.float32 and Y.dtype == np.float64:
        # result dtype follows numpy promotion of (X, Y) like -2*dot(X, Y.T)+XX+YY in the reference
        X = DeviceData([c.to(torch.float64) for c in X.chunks], X.backend, X.comm)
    k = int(Y.shape[0])
    XXg = YYg = None
    if X_norm_squared is not None:
        XXg = np.asarray(X_norm_squared)
        if XXg.shape == (1, X.n_local):
            XXg = XXg.T
        elif XXg.shape != (X.n_local, 1):
            raise ValueError("Incompatible dimensions for X and X_norm_squared")
    if Y_norm_squared is not None:
        YYg = np.asarray(Y_norm_squared)
        if YYg.ndim < 2:
            YYg = YYg[np.newaxis, :]
        if YYg.shape == (k, 1):
            YYg = YYg.T
        if YYg.shape != (1, k):
            raise ValueError("Incompatible dimensions for Y and Y_norm_squared")
    if XXg is None and YYg is None:
        return ChunkedArray(_distance_blocks(X, Y, 1 if squared else 0))
    # caller-supplied norms: start from the true squared distances and swap the norm terms
    outs = _distance_blocks(X, Y, 1)
    be = X.backend
    Yd = torch.as_tensor(np.ascontiguousarray(Y, dtype=np.float64)).to(be.device)
    yy_true = (Yd * Yd).sum(1)
    off = 0
    res = []
    for x, out in zip(X.chunks, outs):
        n = int(x.shape[0])
        d2 = out.to(torch.float64)
        if XXg is not None:
            xx_true = (x.to(torch.float64) ** 2).sum(1)
            d2 = d2 + (torch.as_tensor(np.asarray(XXg[off:off + n, 0], dtype=np.float64)).to(be.device) - xx_true)[:, None]
        if YYg is not None:
            d2 = d2 + (torch.as_tensor(np.asarray(YYg[0], dtype=np.float64)).to(be.device) - yy_true)[None, :]
        d2 = torch.clamp(d2, min=0.0)
        res.append((d2 if squared else torch.sqrt(d2)).to(X.dtype))
        off += n
    return ChunkedArray(res)


def check_pairwise_arrays(X, Y, precomputed=False):
    """Shape validation of pairwise.py:100-118 (Y=None means X against itself)."""
    Xs = X.shape
    if Y is None:
        Y = X
    Ys = Y.shape
    if precomputed:
        if Xs[1] != Ys[0]:
            raise ValueError(
                "Precomputed metric requires shape (n_queries, n_indexed). Got (%d, %d) for %d indexed."
                % (Xs[0], Xs[1], Ys[0])
            )
    elif Xs[1] != Ys[1]:
        raise ValueError(
            "Incompatible dimension for X and Y matrices: X.shape[1] == %d while Y.shape[1] == %d" % (Xs[1], Ys[1])
        )
    return X, Y


def rbf_kernel(X, Y=None, gamma=None):
    """exp(-gamma * ||x - y||^2) (pairwise.py:131-139); ``gamma`` defaults to 1 / n_features.  One fused pass: the
    distance kernel's epilogue applies the exponential (mode 2 of ``bkm_transform_chunk``)."""
    Xd = _as_device(X)
    if Y is None:
        Y = Xd.to_host()
    Y = np.asarray(Y)
    if Y.ndim != 2 or Y.shape[1] != Xd.d:
        raise ValueError(
            "Incompatible dimension for X and Y matrices: X.shape[1] == %d while Y.shape[1] == %d"
            % (Xd.d, Y.shape[1] if Y.ndim == 2 else -1)
        )
    if gamma is None:
        gamma = 1.0 / Xd.d
    return ChunkedArray(_distance_blocks(Xd, Y, 2, float(gamma)))


def pairwise_kernels(X, Y=None, metric="linear", filter_params=False, n_jobs=1, **kwds):
    """pairwise.py:172-195; only the kernel built on the distance path ('rbf') runs on the engine."""
    if metric == "precomputed":
        X, _ = check_pairwise_arrays(X, Y, precomputed=True)
        return X
    if metric == "rbf":
        if filter_params:
            kwds = dict((k, kwds[k]) for k in kwds if k in ("gamma",))
        return rbf_kernel(X, Y, **kwds)
    if metric in ("linear", "polynomial", "sigmoid"):
        raise NotImplementedError("kernel %r is outside the KMeans hot path of the GPU engine" % metric)
    raise ValueError("Unknown kernel %r" % metric)
