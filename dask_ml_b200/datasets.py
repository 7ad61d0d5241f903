"""The generators of dask_ml.datasets: ``make_blobs`` (dask_ml/datasets.py:76-202) and ``make_classification``,
``make_regression``, ``make_counts`` (datasets.py:24-73, 205-378).

make_blobs

The reference builds prototype centres from ONE scikit-learn call with the user's seed (the per-cluster means of a
first-block-sized sample, datasets.py:160-176) and then generates every block independently with
``sklearn.datasets.make_blobs(n_block, centers=prototype, random_state=block_index)`` (datasets.py:178-189).

* ``device=None`` (default): exactly that, block by block on the host -> bit-identical to the reference for the
  same scikit-learn version (BASELINE config C1: 100k x 16 float64, 8 blocks).  Returns host ``ChunkedArray``s.
* ``device='cuda'``: the same prototype centres, but every block is generated ON THE GPU by ``bkm_make_blobs_chunk``
  (Philox streams keyed by the block index, so a block is reproducible whatever GPU generates it).  numpy's
  Mersenne-Twister stream cannot be reproduced on the device: the blocks are statistically equivalent, not identical
  (labels are i.i.d. uniform instead of an exact equal split).  Returns device-resident ``ChunkedArray``s.

make_classification, make_regression, make_counts
  The reference draws X and the response from dask's per-block streams, which cannot be reproduced.  These three use
  the package's own stream, defined in include/bkm_b200.h (``bkm_make_glm_chunk``): the parameters (the Philox key,
  the informative indices and coefficients, make_regression's ``coef``) are drawn on the host from a numpy
  ``RandomState``, and every element from Philox4x32-10 counters built from the GLOBAL row index.  ``device='cuda'``
  runs the kernel; ``device=None`` runs the numpy restatement below.  The dataset therefore does not depend on
  ``chunks``, and the two paths agree (X to rounding of the math library, y except within ~1e-12 of a decision).
"""
from numbers import Integral

import numpy as np

from .chunked import ChunkedArray

_TAG_X, _TAG_RESPONSE, _TAG_NOISE = 0, 1, 2
_LOGISTIC, _NORMAL, _POISSON = 0, 1, 2
_POISSON_LAM_MAX = 9.223372006484771e18          # numpy's POISSON_LAM_MAX: int64 max - 10 sqrt(int64 max)
_W32 = np.uint64(0xFFFFFFFF)


def _normalize_chunks(chunks, n_samples, n_features):
    """Row block sizes from the forms datasets.py:133-139 accepts (blocksize, blockshape, explicit sizes)."""
    if chunks is None:
        return [int(n_samples)]
    if isinstance(chunks, Integral):
        c = int(chunks)
    elif isinstance(chunks, (tuple, list)) and len(chunks) and isinstance(chunks[0], (tuple, list)):
        if len(chunks) > 1 and len(chunks[1]) > 1:
            raise ValueError("Can only generate arrays partitioned along the first axis. Specifying a larger chunksize "
                             "for the second axis.")
        sizes = [int(v) for v in chunks[0]]
        if sum(sizes) != n_samples:
            raise ValueError("chunks do not add up to n_samples")
        return sizes
    else:
        if len(chunks) > 1 and int(chunks[1]) < n_features:
            raise ValueError("Can only generate arrays partitioned along the first axis. Specifying a larger chunksize "
                             "for the second axis.")
        c = int(chunks[0])
    c = max(1, c)
    return [c] * (n_samples // c) + ([n_samples % c] if n_samples % c else [])


def make_blobs(n_samples=100, n_features=2, centers=None, cluster_std=1.0, center_box=(-10.0, 10.0), shuffle=True,
               random_state=None, chunks=None, device=None, dtype=None):
    """Generate isotropic Gaussian blobs for clustering, one row block at a time (datasets.py:76-202).

    Returns ``(X, y)``: ``ChunkedArray`` of shape (n_samples, n_features) float64 and (n_samples,) int64 like the
    reference (``dtype`` lets the device generator write float32 directly)."""
    import sklearn.datasets

    sizes = _normalize_chunks(chunks, int(n_samples), int(n_features))
    if centers is None:
        centers = 3
    if isinstance(centers, Integral):
        # prototype centres: per-cluster means of one first-block-sized sample drawn with the user's seed
        n_centers = int(centers)
        Xp, yp = sklearn.datasets.make_blobs(n_samples=sizes[0], n_features=n_features, centers=n_centers,
                                             shuffle=shuffle, cluster_std=cluster_std, center_box=center_box,
                                             random_state=random_state)
        centers = np.zeros((n_centers, n_features))
        for i in range(n_centers):
            centers[i] = Xp[yp == i].mean(0)
    centers = np.asarray(centers, dtype=np.float64)
    if device is None:
        Xs, ys = [], []
        for i, m in enumerate(sizes):
            Xb, yb = sklearn.datasets.make_blobs(n_samples=m, n_features=n_features, centers=centers,
                                                 cluster_std=cluster_std, shuffle=shuffle, center_box=center_box,
                                                 random_state=i)
            Xs.append(Xb if dtype is None else Xb.astype(dtype))
            ys.append(yb.astype(np.int64))
        return ChunkedArray(Xs), ChunkedArray(ys)

    import torch

    from .engine import CudaBackend

    be = CudaBackend(torch.device(device) if not isinstance(device, torch.device) else device)
    tdt = torch.float64 if dtype is None else {np.dtype("float32"): torch.float32, np.dtype("float64"): torch.float64}[np.dtype(dtype)]
    k = int(centers.shape[0])
    std = np.broadcast_to(np.asarray(cluster_std, dtype=np.float64), (k,)).copy()
    Cd = torch.as_tensor(centers).to(be.device)
    Sd = torch.as_tensor(std).to(be.device)
    Xs, ys = [], []
    for i, m in enumerate(sizes):
        Xb = torch.empty((m, int(n_features)), dtype=tdt, device=be.device)
        yb = torch.empty((m,), dtype=torch.int64, device=be.device)
        be.make_blobs_chunk(Xb, yb, Cd, Sd, i)
        Xs.append(Xb)
        ys.append(yb)
    return ChunkedArray(Xs), ChunkedArray(ys)


# ---------------------------------------------------------------------------------------------------------------------
# the stream of make_classification / make_regression / make_counts (include/bkm_b200.h), restated in numpy
# ---------------------------------------------------------------------------------------------------------------------
def _philox4(key, row, j, tag):
    """Philox4x32-10 under the 64-bit ``key`` at counters (row lo, row hi, j, tag): four uint64 arrays of 32-bit words."""
    row, j = np.broadcast_arrays(np.asarray(row, dtype=np.uint64), np.asarray(j, dtype=np.uint64))
    M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
    c0, c1 = row & _W32, row >> np.uint64(32)
    c2, c3 = j & _W32, np.full(row.shape, tag, dtype=np.uint64)
    k0, k1 = int(key) & 0xFFFFFFFF, (int(key) >> 32) & 0xFFFFFFFF
    for _ in range(10):
        p0, p1 = M0 * c0, M1 * c2
        c0, c1, c2, c3 = ((p1 >> np.uint64(32)) ^ c1 ^ np.uint64(k0), p1 & _W32,
                          (p0 >> np.uint64(32)) ^ c3 ^ np.uint64(k1), p0 & _W32)
        k0, k1 = (k0 + 0x9E3779B9) & 0xFFFFFFFF, (k1 + 0xBB67AE85) & 0xFFFFFFFF
    return c0, c1, c2, c3


def _u53(a, b):
    """The 53-bit uniform in [0, 1) of two 32-bit words (numpy's construction)."""
    return ((a >> np.uint64(5)).astype(np.float64) * 67108864.0 + (b >> np.uint64(6)).astype(np.float64)) \
        * (1.0 / 9007199254740992.0)


def _sincospi(t):
    """(sin(pi t), cos(pi t)) for t in [0, 2): the quadrant is split off exactly, so only pi * r rounds."""
    q = np.rint(2.0 * t)
    r = t - 0.5 * q                                           # exact, in [-0.25, 0.25]
    s, c = np.sin(np.pi * r), np.cos(np.pi * r)
    qi = q.astype(np.int64) & 3
    sn = np.choose(qi, [s, c, -s, -c])
    cs = np.choose(qi, [c, -s, -c, s])
    return sn, cs


def _normal_pair(w0, w1):
    """The Box-Muller pair of two 32-bit words (the normals of make_blobs_kernel)."""
    u1 = (w0.astype(np.float64) + 1.0) * (1.0 / 4294967296.0)
    u2 = w1.astype(np.float64) * (1.0 / 4294967296.0)
    rad = np.sqrt(-2.0 * np.log(u1))
    sn, cs = _sincospi(2.0 * u2)
    return rad * cs, rad * sn


def _x_block(key, row0, m, d, dtype):
    """Rows row0 .. row0 + m - 1 of X, in ``dtype``."""
    pairs = (d + 1) // 2
    rows = (np.uint64(row0) + np.arange(m, dtype=np.uint64))[:, None]
    w0, w1, _, _ = _philox4(key, rows, np.arange(pairs, dtype=np.uint64)[None, :], _TAG_X)
    n0, n1 = _normal_pair(w0, w1)
    X = np.empty((m, 2 * pairs), dtype=np.float64)
    X[:, 0::2] = n0
    X[:, 1::2] = n1
    return np.ascontiguousarray(X[:, :d]).astype(dtype)


def _linear(Xb, info, t):
    """z of target t: the float64 sum in list order of x_f * c[f, t] over the informative list, x_f as stored."""
    z = np.zeros(Xb.shape[0], dtype=np.float64)
    for row in info:
        z = z + Xb[:, int(row[0])].astype(np.float64) * row[1 + t]
    return z


_LOGGAM_A = (8.333333333333333e-02, -2.777777777777778e-03, 7.936507936507937e-04, -5.952380952380952e-04,
             8.417508417508418e-04, -1.917526917526918e-03, 6.410256410256410e-03, -2.955065359477124e-02,
             1.796443723749843e-01, -1.39243221690590e+00)


def _loggam(x):
    """numpy's random_loggam, elementwise."""
    x = np.asarray(x, dtype=np.float64)
    n = np.where(x < 7.0, (7.0 - x).astype(np.int64), 0)
    x0 = x + n.astype(np.float64)
    r = 1.0 / x0
    x2 = r * r
    gl0 = np.full(x.shape, _LOGGAM_A[9])
    for k in range(8, -1, -1):
        gl0 = gl0 * x2 + _LOGGAM_A[k]
    gl = gl0 / x0 + 0.5 * 1.8378770664093453e+00 + (x0 - 0.5) * np.log(x0) - x0
    for k in range(1, int(n.max(initial=0)) + 1):
        s = n >= k
        gl[s] = gl[s] - np.log(x0[s] - 1.0)
        x0[s] = x0[s] - 1.0
    return np.where((x == 1.0) | (x == 2.0), 0.0, gl)


def _rel(a, b):
    return np.abs(a - b) / np.maximum(np.abs(b), 1e-300)


def _poisson(lam, key, rows, margin=False):
    """numpy's legacy Poisson draw of every rate, attempt j of row r taking the response uniforms at (r, j).

    With ``margin=True`` also returns, per row, the smallest relative distance of a comparison the draw made to its
    decision boundary: a row whose margin is below the math library's rounding can come out differently elsewhere."""
    lam = np.asarray(lam, dtype=np.float64)
    y = np.zeros(lam.shape, dtype=np.int64)
    mg = np.full(lam.shape, np.inf)
    # multiplication method, lam < 10
    idx = np.flatnonzero((lam > 0.0) & (lam < 10.0))
    enlam = np.exp(-lam[idx])
    prod = np.ones(idx.size)
    cnt = np.zeros(idx.size, dtype=np.int64)
    att = 0
    while idx.size:
        w0, w1, _, _ = _philox4(key, rows[idx], att, _TAG_RESPONSE)
        prod = prod * _u53(w0, w1)
        if margin:
            mg[idx] = np.minimum(mg[idx], _rel(prod, enlam))
        go = prod > enlam
        y[idx[~go]] = cnt[~go]
        idx, enlam, prod, cnt = idx[go], enlam[go], prod[go], cnt[go] + 1
        att += 1
    # PTRS, lam >= 10
    idx = np.flatnonzero(lam >= 10.0)
    lm = lam[idx]
    slam, loglam = np.sqrt(lm), np.log(lm)
    b = 0.931 + 2.53 * slam
    a = -0.059 + 0.02483 * b
    invalpha = 1.1239 + 1.1328 / (b - 3.4)
    vr = 0.9277 - 3.6224 / (b - 2.0)
    att = 0
    with np.errstate(divide="ignore", invalid="ignore"):
        while idx.size:
            w0, w1, w2, w3 = _philox4(key, rows[idx], att, _TAG_RESPONSE)
            U = _u53(w0, w1) - 0.5
            V = _u53(w2, w3)
            us = 0.5 - np.abs(U)
            t = (2.0 * a / us + b) * U + lm + 0.43
            ft = np.floor(t)
            k = np.where(np.isfinite(ft), ft, -1.0).astype(np.int64)
            done = (us >= 0.07) & (V <= vr)
            rest = ~done & ~((k < 0) | ((us < 0.013) & (V > us)))
            lhs = np.log(V) + np.log(invalpha) - np.log(a / (us * us) + b)
            kf = np.maximum(k, 0).astype(np.float64)                # rhs is only read where k >= 0
            rhs = -lm + kf * loglam - _loggam(kf + 1.0)
            done |= rest & (lhs <= rhs)
            if margin:
                frac = np.minimum(t - ft, ft + 1.0 - t) / np.maximum(np.abs(t), 1.0)
                m = np.minimum(np.minimum(_rel(us, 0.07), _rel(V, vr)), np.where(np.isfinite(t), frac, np.inf))
                m = np.minimum(m, np.where(us < 0.02, _rel(us, 0.013), np.inf))
                m = np.minimum(m, np.where(rest, np.abs(lhs - rhs) / np.maximum(np.abs(rhs), 1.0), np.inf))
                mg[idx] = np.minimum(mg[idx], m)
            y[idx[done]] = k[done]
            keep = ~done
            idx, lm, slam, loglam, a, b, invalpha, vr = (v[keep] for v in (idx, lm, slam, loglam, a, b, invalpha, vr))
            att += 1
    return (y, mg) if margin else y


def _response_host(Xb, family, info, key, row0, n_targets=1, bias=0.0, noise=0.0):
    """y of one block from its stored X (the host half of bkm_make_glm_chunk)."""
    m = Xb.shape[0]
    rows = np.uint64(row0) + np.arange(m, dtype=np.uint64)
    if family == _NORMAL:
        y = np.empty((m, n_targets), dtype=np.float64)
        for t in range(n_targets):
            yt = _linear(Xb, info, t) + bias
            if noise > 0:
                w0, w1, _, _ = _philox4(key, rows, t, _TAG_NOISE)
                yt = yt + noise * _normal_pair(w0, w1)[0]
            y[:, t] = yt
        return y
    z = _linear(Xb, info, 0)
    if family == _LOGISTIC:
        w0, w1, _, _ = _philox4(key, rows, 0, _TAG_RESPONSE)
        return (_u53(w0, w1) < 1.0 / (1.0 + np.exp(-z))).astype(np.int64)
    with np.errstate(over="ignore"):
        lam = np.exp(z)
    if not np.all(lam <= _POISSON_LAM_MAX):
        raise ValueError("lam value too large")
    return _poisson(lam, key, rows)


# ---------------------------------------------------------------------------------------------------------------------
# make_classification, make_regression, make_counts
# ---------------------------------------------------------------------------------------------------------------------
def _row_chunks(chunks, n_samples, n_features):
    """Row block sizes of a (n_samples, n_features) array chunked by any form dask's ``normalize_chunks`` takes for it
    (a block size, a block shape, explicit sizes); a split of the columns raises the reference's ValueError
    (``_check_axis_partitioning``, datasets.py:12-21).  ``chunks=None`` is one block."""
    if chunks is None:
        return [n_samples]
    if isinstance(chunks, Integral):
        rows, cols = chunks, chunks
    elif isinstance(chunks, (tuple, list)) and len(chunks) == 2:
        rows, cols = chunks
    else:
        raise ValueError("chunks must be an int, a (rows, columns) block shape or explicit block sizes")
    if isinstance(cols, (tuple, list)):
        c = int(cols[0])
    else:
        c = n_features if cols is None or int(cols) == -1 else min(int(cols), n_features)
    if c != n_features:
        raise ValueError("Can only generate arrays partitioned along the first axis. Specifying a larger chunksize "
                         "for the second axis.\n\n\tchunk size: {}\n\tn_features: {}".format(c, n_features))
    if isinstance(rows, (tuple, list)):
        sizes = [int(v) for v in rows]
        if sum(sizes) != n_samples:
            raise ValueError("chunks do not add up to n_samples")
        return sizes
    r = n_samples if rows is None or int(rows) == -1 else max(1, int(rows))
    return [r] * (n_samples // r) + ([n_samples % r] if n_samples % r else []) or [n_samples]


def _out_dtype(dtype):
    dt = np.dtype(np.float64 if dtype is None else dtype)
    if dt not in (np.dtype(np.float32), np.dtype(np.float64)):
        raise ValueError("dtype must be float32 or float64, got %s" % dt)
    return dt


def _draw_key(rng):
    """The 64-bit Philox key: the first 8 bytes of the 624-word state dask's ``random_state_data`` draws."""
    return int(np.frombuffer(rng.bytes(624 * 4)[:8], dtype="<u8")[0])


def _informative(rng, n_features, n_informative, scale):
    """idx (with replacement, the default of ``choice``), then beta = (U - 1) * scale in [-scale, 0); the list
    [(idx_k, beta[idx_k])] in idx order."""
    idx = rng.choice(n_features, n_informative)
    beta = (rng.random_sample(n_features) - 1) * scale
    return np.column_stack([idx.astype(np.float64), beta[idx]]).reshape(-1, 2)


def _generate(sizes, d, dtype, family, info, key, device, n_targets=1, bias=0.0, noise=0.0):
    """X and y block by block, on the host (device=None) or by ``bkm_make_glm_chunk``."""
    dt = _out_dtype(dtype)
    if device is None:
        Xs, ys, row0 = [], [], 0
        for m in sizes:
            Xb = _x_block(key, row0, m, d, dt)
            Xs.append(Xb)
            ys.append(_response_host(Xb, family, info, key, row0, n_targets, bias, noise))
            row0 += m
    else:
        import torch

        from .engine import CudaBackend

        be = CudaBackend(torch.device(device) if not isinstance(device, torch.device) else device)
        tdt = torch.float32 if dt == np.dtype(np.float32) else torch.float64
        ydt = torch.float64 if family == _NORMAL else torch.int64
        Xs, ys, row0 = [], [], 0
        info_d = torch.as_tensor(np.ascontiguousarray(info, dtype=np.float64)).to(be.device)
        flag = torch.zeros(1, dtype=torch.int32, device=be.device)
        for m in sizes:
            Xb = torch.empty((m, d), dtype=tdt, device=be.device)
            yb = torch.empty((m, n_targets) if family == _NORMAL else (m,), dtype=ydt, device=be.device)
            be.make_glm_chunk(Xb, yb, row0, family, info_d, n_targets, bias, noise, key, flag)
            Xs.append(Xb)
            ys.append(yb)
            row0 += m
        if family == _POISSON and int(flag.item()):
            raise ValueError("lam value too large")
    if family == _NORMAL and n_targets == 1:
        ys = [yb.reshape(-1) for yb in ys]
    return ChunkedArray(Xs), ChunkedArray(ys)


def _normal_panel(key, m, d, device):
    """Rows 0 .. m - 1 of the stream's X under ``key`` as a float64 (m, d) tensor on ``device``: ``bkm_make_glm_chunk``
    on a CUDA device, the numpy restatement ``_x_block`` otherwise (the two agree to rounding of the math library).
    TruncatedSVD's Gaussian test matrix on sparse X."""
    import torch

    device = torch.device(device)
    if device.type != "cuda":
        return torch.from_numpy(_x_block(key, 0, m, d, np.float64))
    from .engine import CudaBackend

    be = CudaBackend(device)
    X = torch.empty((m, d), dtype=torch.float64, device=device)
    y = torch.empty((m,), dtype=torch.int64, device=device)       # the (unused) logistic response of the same call
    if m:
        be.make_glm_chunk(X, y, 0, _LOGISTIC, None, 1, 0.0, 0.0, key)
    return X


def make_counts(n_samples=1000, n_features=100, n_informative=2, scale=1.0, chunks=100, random_state=None,
                device=None, dtype=None):
    """A dummy dataset for modelling count data (datasets.py:24-73): X i.i.d. N(0, 1), y ~ Poisson(exp(z)) with
    z = X[:, idx] . beta[idx] (see ``make_classification`` for idx and beta).

    ``chunks`` is the number of rows per block.  Returns ``(X, y)``: ``ChunkedArray`` of shape (n_samples,
    n_features) in ``dtype`` (float64 by default) and (n_samples,) int64; host numpy blocks for ``device=None``,
    device tensors otherwise.  A rate numpy's ``RandomState.poisson`` rejects raises its ``ValueError``."""
    import sklearn.utils

    n, d = int(n_samples), int(n_features)
    sizes = _normalize_chunks(chunks, n, d)
    rng = sklearn.utils.check_random_state(random_state)
    key = _draw_key(rng)
    info = _informative(rng, d, n_informative, scale)
    return _generate(sizes, d, dtype, _POISSON, info, key, device)


def make_classification(n_samples=100, n_features=20, n_informative=2, n_redundant=2, n_repeated=0, n_classes=2,
                        n_clusters_per_class=2, weights=None, flip_y=0.01, class_sep=1.0, hypercube=True, shift=0.0,
                        scale=1.0, shuffle=True, random_state=None, chunks=None, device=None, dtype=None):
    """A binary classification problem from a logistic model (datasets.py:340-378).

    X is i.i.d. N(0, 1).  ``idx = rng.choice(n_features, n_informative)`` is drawn WITH replacement (a repeated index
    counts twice), ``beta = (rng.random_sample(n_features) - 1) * scale`` lies in [-scale, 0), and
    ``y = U < 1 / (1 + exp(-z))`` with ``z = X[:, idx] . beta[idx]``, as int64.  As in the reference, only
    ``n_classes == 2`` is supported and every other shape parameter (``n_redundant``, ``n_repeated``,
    ``n_clusters_per_class``, ``weights``, ``flip_y``, ``class_sep``, ``hypercube``, ``shift``, ``shuffle``) is
    accepted and ignored.  Returns ``(X, y)`` as ``make_counts`` does."""
    import sklearn.utils

    n, d = int(n_samples), int(n_features)
    sizes = _row_chunks(chunks, n, d)
    if n_classes != 2:
        raise NotImplementedError("n_classes != 2 is not yet supported.")
    rng = sklearn.utils.check_random_state(random_state)
    key = _draw_key(rng)
    info = _informative(rng, d, n_informative, scale)
    return _generate(sizes, d, dtype, _LOGISTIC, info, key, device)


def make_regression(n_samples=100, n_features=100, n_informative=10, n_targets=1, bias=0.0, effective_rank=None,
                    tail_strength=0.5, noise=0.0, shuffle=True, coef=False, random_state=None, chunks=None,
                    device=None, dtype=None):
    """A random linear regression problem (datasets.py:205-337).

    ``coef`` is the one of ``sklearn.datasets.make_regression(n_samples=<first block's size>, ..., coef=True,
    random_state=rng)`` with ``rng = sklearn.utils.check_random_state(random_state)``, bit-identical to the
    reference's (``effective_rank`` and ``tail_strength`` only shape that discarded sample).  X is i.i.d. N(0, 1) and
    ``y = X . coef + bias (+ noise * N(0, 1))`` in float64, of shape (n_samples,) for one target.  Returns
    ``(X, y, coef)`` when ``coef is True``, else ``(X, y)``."""
    import sklearn.datasets
    import sklearn.utils

    n, d = int(n_samples), int(n_features)
    sizes = _row_chunks(chunks, n, d)
    rng = sklearn.utils.check_random_state(random_state)
    return_coef = coef is True
    _, _, w = sklearn.datasets.make_regression(
        n_samples=sizes[0], n_features=d, n_informative=n_informative, n_targets=n_targets, bias=bias,
        effective_rank=effective_rank, tail_strength=tail_strength, noise=noise, shuffle=shuffle, coef=True,
        random_state=rng)
    key = _draw_key(rng)
    nt = int(n_targets)
    w2 = np.asarray(w, dtype=np.float64).reshape(d, nt)
    nz = np.flatnonzero(np.any(w2 != 0, axis=1))
    info = np.column_stack([nz.astype(np.float64), w2[nz]]).reshape(-1, 1 + nt)
    X, y = _generate(sizes, d, dtype, _NORMAL, info, key, device, nt, float(bias), float(noise))
    return (X, y, w) if return_coef else (X, y)
