"""KMeans with the dask_ml.cluster.KMeans API, executed by the H100 engine.

Mirrors dask_ml/cluster/k_means.py (reference @ 0310a90):
  KMeans                      :26-233     k_means            :236-275
  k_init                      :291-369    init_pp            :372-384
  init_random                 :387-393    init_scalable      :396-463
  evaluate_cost/_sample_points :466-491   _kmeans_single_lloyd :499-569
The host loop keeps the reference's control flow (including its quirks Q1-Q6, DESIGN.md (a));
all arithmetic over X runs in the CUDA kernels behind include/bkm_b200.h.
"""
import logging
from numbers import Integral

import numpy as np
import scipy.sparse
import torch
from sklearn.base import BaseEstimator, TransformerMixin
from sklearn.utils.validation import check_is_fitted

from ..chunked import ChunkedArray, as_chunked, is_dask_array, is_dask_dataframe, _is_torch
from .._sparse import _SparseData, _sparse_data, check_label_sum_classes
from ..engine import Comm, CudaBackend, DeviceData, _NP_TO_TORCH
from ..utils import _timed, _timer, check_array

logger = logging.getLogger(__name__)

# Replaced by tests that exercise the host loop on CPU with a checker backend.
_BACKEND_FACTORY = CudaBackend


def _get_backend():
    return _BACKEND_FACTORY()


# ---------------------------------------------------------------------------------------
# input handling
# ---------------------------------------------------------------------------------------
_NONFINITE_MSG = "Input contains NaN, infinity or a value too large for dtype('float64')."


def _to_blocks(X):
    """ndarray / torch tensor / ChunkedArray / dask array -> list of 2-D blocks."""
    if isinstance(X, ChunkedArray):
        return X.blocks
    if is_dask_array(X):
        return as_chunked(X).blocks
    return [X]


def _block_np_dtype(b):
    from ..chunked import block_dtype

    return block_dtype(b)


def _to_device_data(X, backend=None, comm=None, check_finite=True):
    """Validated array-like -> DeviceData (rows resident on the device), or ``_SparseData`` for sparse X."""
    if isinstance(X, (DeviceData, _SparseData)):
        return X
    sp = _sparse_data(X)
    if sp is not None:
        if check_finite:
            sp.check_finite()
        return sp
    backend = backend or _get_backend()
    blocks = _to_blocks(X)
    from ..chunked import is_bf16_block

    if all(is_bf16_block(b) for b in blocks):
        tdt = torch.bfloat16                # engine extension: bf16 rows stay bf16 (BASELINE config C5)
    else:
        dt = _block_np_dtype(blocks[0])
        if dt == np.dtype("int32") or dt == np.dtype("float16"):
            dt = np.dtype("float32")            # k_means.py:171-172
        elif dt == np.dtype("int64"):
            dt = np.dtype("float64")            # k_means.py:173-174
        elif dt not in (np.dtype("float32"), np.dtype("float64")):
            dt = np.dtype("float64")
        tdt = _NP_TO_TORCH[dt]
    chunks = [backend.to_device(b, tdt) for b in blocks]
    data = DeviceData(chunks, backend, comm)
    if check_finite:
        flag = backend.check_finite(chunks)
        comm_ = data.comm
        flag_f = flag.to(torch.float64)
        comm_.allreduce_sum_(flag_f)
        if float(flag_f.item()) != 0.0:
            raise ValueError(_NONFINITE_MSG)    # k_means.py:179-185
    return data


class KMeans(TransformerMixin, BaseEstimator):
    """Scalable KMeans for clustering (API of dask_ml.cluster.KMeans, k_means.py:26-152).

    Parameters
    ----------
    n_clusters : int, default 8
    init : {'k-means||', 'k-means++', 'random'} or ndarray of shape (n_clusters, n_features)
    oversampling_factor : int, default 2
        Oversampling factor ``l`` of k-means|| (Bahmani et al. 2012, Alg. 2).
    max_iter : int
        Maximum number of EM (Lloyd) iterations.
    init_max_iter : int
        Number of k-means|| rounds; default ``round(log(cost))``.
    tol : float
        Convergence threshold on ``||C - C'||_F^2`` (raw, as in the reference, k_means.py:555-559).
    random_state : int, RandomState or None
    precompute_distances, copy_x, n_jobs, algorithm :
        Accepted for scikit-learn signature compatibility and ignored, as in the reference
        (k_means.py:148-152).

    Attributes
    ----------
    cluster_centers_ : np.ndarray (n_clusters, n_features), dtype of X
    labels_ : ChunkedArray (n_samples,) int32 — device-resident, ``.compute()`` gives numpy
    inertia_ : np.float64
    n_iter_ : int
    """

    def __init__(
        self,
        n_clusters=8,
        init="k-means||",
        oversampling_factor=2,
        max_iter=300,
        tol=0.0001,
        precompute_distances="auto",
        random_state=None,
        copy_x=True,
        n_jobs=1,
        algorithm="full",
        init_max_iter=None,
    ):
        self.n_clusters = n_clusters
        self.init = init
        self.oversampling_factor = oversampling_factor
        self.random_state = random_state
        self.max_iter = max_iter
        self.init_max_iter = init_max_iter
        self.algorithm = algorithm
        self.tol = tol
        self.precompute_distances = precompute_distances
        self.n_jobs = n_jobs
        self.copy_x = copy_x

    @_timed(_logger=logger)
    def _check_array(self, X):
        """Validation of k_means.py:154-186, ending with X resident on the device."""
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
        X = check_array(
            X,
            accept_dask_dataframe=False,
            accept_unknown_chunks=False,
            accept_sparse=False,
        )
        return _to_device_data(X)

    def __sklearn_tags__(self):
        tags = super().__sklearn_tags__()
        tags.input_tags.sparse = True           # sparse CSR blocks run through the sparse passes
        return tags

    def fit(self, X, y=None):
        X = self._check_array(X)
        labels, centroids, inertia, n_iter = k_means(
            X,
            self.n_clusters,
            oversampling_factor=self.oversampling_factor,
            random_state=self.random_state,
            init=self.init,
            return_n_iter=True,
            max_iter=self.max_iter,
            init_max_iter=self.init_max_iter,
            tol=self.tol,
        )
        self.cluster_centers_ = centroids
        self.labels_ = labels
        self.inertia_ = inertia
        self.n_iter_ = n_iter
        self.n_features_in_ = centroids.shape[1]
        return self

    def _check_n_features(self, X):
        d = X.d if isinstance(X, (DeviceData, _SparseData)) else X.shape[1]
        n_in = getattr(self, "n_features_in_", self.cluster_centers_.shape[1])
        if d != n_in:
            raise ValueError(
                "X has {} features, but {} is expecting {} features as input.".format(d, type(self).__name__, n_in)
            )

    def transform(self, X, y=None):
        check_is_fitted(self, "cluster_centers_")
        X = self._check_array(X)
        self._check_n_features(X)
        from ..metrics.pairwise import euclidean_distances

        return euclidean_distances(X, self.cluster_centers_)

    def predict(self, X):
        """Index of the closest centre for every row (k_means.py:212-233); int32 labels."""
        check_is_fitted(self, "cluster_centers_")
        X = self._check_array(X)
        self._check_n_features(X)
        from ..metrics.pairwise import pairwise_distances_argmin_min

        labels = pairwise_distances_argmin_min(X, self.cluster_centers_)[0].astype(np.int32)
        return labels


def k_means(
    X,
    n_clusters,
    init="k-means||",
    precompute_distances="auto",
    n_init=1,
    max_iter=300,
    verbose=False,
    tol=1e-4,
    random_state=None,
    copy_x=True,
    n_jobs=-1,
    algorithm="full",
    return_n_iter=False,
    oversampling_factor=2,
    init_max_iter=None,
):
    """K-means clustering, functional form (k_means.py:236-275)."""
    labels, inertia, centers, n_iter = _kmeans_single_lloyd(
        X,
        n_clusters,
        max_iter=max_iter,
        init=init,
        verbose=verbose,
        tol=tol,
        random_state=random_state,
        oversampling_factor=oversampling_factor,
        init_max_iter=init_max_iter,
    )
    if return_n_iter:
        return labels, centers, inertia, n_iter
    else:
        return labels, centers, inertia


# ---------------------------------------------------------------------------------------
# Initialisation
# ---------------------------------------------------------------------------------------
def _as_random_state(random_state, comm):
    """Same stream on every rank: ints/None seed a RandomState (None -> rank 0 draws the seed)."""
    if isinstance(random_state, np.random.RandomState):
        return random_state
    if random_state is None:
        seed = comm.bcast_obj(int(np.random.randint(0, 2 ** 31 - 1)))
        return np.random.RandomState(seed)
    return np.random.RandomState(int(random_state))


def k_init(
    X,
    n_clusters,
    init="k-means||",
    random_state=None,
    max_iter=None,
    oversampling_factor=2,
    weighted=False,
):
    """Choose the initial centres (k_means.py:291-369).  Returns np.ndarray (k, d)."""
    n_features = X.d if isinstance(X, (DeviceData, _SparseData)) else X.shape[1]
    if isinstance(init, np.ndarray):
        K, P = init.shape

        if K != n_clusters:
            msg = "Number of centers in provided 'init' ({}) does not match 'n_clusters' ({})"
            raise ValueError(msg.format(K, n_clusters))

        if P != n_features:
            msg = "Number of features in the provided 'init' ({}) do not match the number of features in 'X'"
            raise ValueError(msg.format(P, n_features))

        return init

    elif not isinstance(init, str):
        raise TypeError("'init' must be an array or str, got {}".format(type(init)))

    valid = {"k-means||", "k-means++", "random"}
    if init not in valid:
        raise ValueError("'init' must be one of {}, got {}".format(valid, init))

    X = _to_device_data(X, check_finite=False)
    if weighted and isinstance(X, _SparseData):
        raise NotImplementedError("weighted k-means|| is not implemented for sparse X")
    if isinstance(random_state, Integral) or random_state is None:
        random_state = _as_random_state(random_state, X.comm)

    if init == "k-means||":
        return init_scalable(X, n_clusters, random_state, max_iter, oversampling_factor, weighted=weighted)
    elif init == "k-means++":
        return init_pp(X, n_clusters, random_state)
    else:
        return init_random(X, n_clusters, random_state)


def init_pp(X, n_clusters, random_state):
    """k-means++ through scikit-learn on the host, like the reference (k_means.py:372-384):
    the whole dataset is brought into host memory (single-process only)."""
    from sklearn.cluster import kmeans_plusplus

    if X.comm.world != 1:
        raise NotImplementedError("init='k-means++' loads all of X on one host; use 'k-means||' when distributed")
    logger.info("Initializing with k-means++")
    Xh = X.to_host()
    with _timer("initialization of %2d centers" % n_clusters, _logger=logger):
        centers, _ = kmeans_plusplus(Xh, n_clusters, random_state=random_state)
    return centers


@_timed(_logger=logger)
def init_random(X, n_clusters, random_state):
    """Centres = randomly chosen rows (k_means.py:387-393)."""
    logger.info("Initializing randomly")
    idx = sorted(random_state.randint(0, X.n_global, size=n_clusters))
    rows = X.global_rows(idx)
    return rows.toarray() if scipy.sparse.issparse(rows) else rows


class _AssignPass(object):
    """One E-step-only sweep over all local chunks against a fixed set of centres."""

    def __init__(self, X):
        self.X = X
        self.be = X.backend

    def run(self, centers64, want_labels=False, want_min=False, squared=True):
        be, X = self.be, self.X
        k = centers64.shape[0]
        C = torch.as_tensor(np.ascontiguousarray(centers64, dtype=np.float64)).to(be.device)
        pack = be.pack_centers(C, X.dtype)
        acc = be.zeros((1,), torch.float64)
        labels, mins = [], []
        for x in X.chunks:
            n = x.shape[0]
            lab = be.empty((n,), torch.int32) if want_labels else None
            mn = be.empty((n,), X.out_dtype) if want_min else None
            be.assign_chunk(x, pack, k, lab, mn, squared, acc)
            labels.append(lab)
            mins.append(mn)
        X.comm.allreduce_sum_(acc)
        return labels, mins, acc

    def cost(self, centers64):
        """phi = sum of min squared distances, as a checked host float."""
        _, _, acc = self.run(centers64, squared=True)
        v = float(acc.item())
        _check_engine(self.be, v, "the k-means|| cost")
        return v


class _SparseAssignPass(_AssignPass):
    """``_AssignPass`` over sparse CSR blocks (``bkm_csr_assign_chunk``): the centres (dense, or the sparse candidate
    rows of k-means||) are densified on the device into the sparse pack; the minimum is float64."""

    def run(self, centers64, want_labels=False, want_min=False, squared=True):
        be, X = self.be, self.X
        C = _dense_centres(centers64, X.d, be)
        k = int(C.shape[0])
        pack = be.sparse_pack_centers(C)
        acc = be.zeros((1,), torch.float64)
        labels, mins = [], []
        for blk in X.blocks:
            n = int(blk[3])
            lab = be.empty((n,), torch.int32) if want_labels else None
            mn = be.empty((n,), torch.float64) if want_min else None
            be.csr_assign_chunk(blk, X.d, pack, k, labels=lab, min_dist=mn, squared=squared, dist_sum=acc)
            labels.append(lab)
            mins.append(mn)
        X.comm.allreduce_sum_(acc)
        return labels, mins, acc


def _dense_centres(C, d, be):
    """(k, d) float64 device centres from an array or a host scipy CSR (densified on the device)."""
    if not scipy.sparse.issparse(C):
        return torch.as_tensor(np.ascontiguousarray(C, dtype=np.float64)).to(be.device)
    C = scipy.sparse.csr_matrix(C)
    out = be.zeros((C.shape[0], d), torch.float64)
    rows = np.repeat(np.arange(C.shape[0], dtype=np.int64), np.diff(C.indptr))
    if len(rows):
        out[torch.as_tensor(rows).to(be.device), torch.as_tensor(C.indices.astype(np.int64)).to(be.device)] = \
            torch.as_tensor(C.data.astype(np.float64)).to(be.device)
    return out


def _assign_pass(X):
    return _SparseAssignPass(X) if isinstance(X, _SparseData) else _AssignPass(X)


def _sweep_rows(X):
    """Candidates per k-means|| sweep: 256 (the tensor path's limit); for sparse X also at most 32 MB of pack."""
    if isinstance(X, _SparseData):
        return int(max(1, min(256, (1 << 22) // max(1, X.d))))
    return 256


@_timed(_logger=logger)
def init_scalable(X, n_clusters, random_state=None, max_iter=None, oversampling_factor=2, weighted=False):
    """k-means|| (Bahmani et al. 2012, Alg. 2) following k_means.py:396-463.

    Each round is one distance sweep on the device over the NEW candidates only (``bkm_assign_chunk``: min d^2 per
    row), folded into the running minimum and summed to the cost phi by ``bkm_min_fold_chunk``, followed by the
    Bernoulli draw kernel (``bkm_sample_chunk``).  The reference draws U with dask's per-chunk RandomState
    (k_means.py:487); here U comes from a counter-based Philox stream keyed by a per-round seed and the global row
    index, so a run is reproducible for a given ``random_state`` independent of chunking and of the number of GPUs
    (k-means|| sampling parity with the reference is therefore distributional, not bit-exact: DESIGN.md (c)).

    The final reduce of the candidates to ``n_clusters`` centres (k_means.py:457-463: an in-memory scikit-learn KMeans,
    unweighted) runs on the GPU through this engine (``_reduce_candidates``).  ``weighted=True`` gives every candidate
    the number of points it attracts, as the paper's step 7 does and the reference omits.
    """
    logger.info("Initializing with k-means||")
    be, comm = X.backend, X.comm
    rs = random_state if isinstance(random_state, np.random.RandomState) else _as_random_state(random_state, comm)
    c_idx = _scalable_candidates(X, rs, max_iter, oversampling_factor)
    sweep = _AssignPass(X)
    # sorted, like the reference (k_means.py:432-435); fetched once, after the last round.  Sparse X: a CSR of the rows
    centers = X.global_rows(c_idx)

    if centers.shape[0] < n_clusters:
        logger.warning("Found fewer than %d clusters in init.", n_clusters)
        # supplement with random rows (k_means.py:445-455).  The reference permutes all n row indices for this
        # (random_state.choice(arange(n), replace=False)): O(n) host work for a handful of rows.  Same distribution in
        # O(need): draw, de-duplicate, repeat.
        need = n_clusters - centers.shape[0]
        n = int(X.n_global)
        chosen = set()
        while len(chosen) < need:
            for v in rs.randint(0, n, size=2 * (need - len(chosen)) + 8):
                if len(chosen) < need:
                    chosen.add(int(v))
        locs = sorted(chosen)
        extra = X.global_rows(locs)
        if scipy.sparse.issparse(centers):
            return np.vstack([centers.toarray(), extra.toarray()])
        return np.vstack([centers, extra])
    else:
        # Steps 7, 8 (k_means.py:457-463): reduce the candidates to n_clusters centres
        weights = None
        if weighted:
            lab, _, _ = sweep.run(centers.astype(np.float64), want_labels=True)
            wt = be.zeros((len(centers),), torch.float64)
            for l in lab:
                wt += torch.bincount(l.long(), minlength=len(centers)).to(torch.float64)
            comm.allreduce_sum_(wt)
            weights = wt.cpu().numpy()
        rng2 = int(rs.randint(0, 2 ** 32 - 1, dtype=np.int64))
        return _reduce_candidates(centers, n_clusters, rng2, be, weights)


def _scalable_candidates(X, rs, max_iter, oversampling_factor):
    """Steps 1-6 of k-means|| (k_means.py:406-435): the sorted global row indices of the candidate centres."""
    be, comm = X.backend, X.comm
    sweep = _assign_pass(X)

    # Step 1: first centre = global row 0 (k_means.py:406-408)
    idx = 0
    centers = X.global_rows([idx])
    c_idx = {idx}

    # Step 2: initial cost (k_means.py:411-420)
    cost = sweep.cost(centers.astype(np.float64))
    if cost == 0:
        n_iter = 0
    else:
        n_iter = int(np.round(np.log(cost)))
    if max_iter is not None:
        n_iter = min(max_iter, n_iter)

    # Steps 3-6: oversampling rounds (k_means.py:423-435).  The reference re-evaluates the distances to ALL
    # candidates every round; min_j d(x, c_j) over a growing set is the running minimum of the per-round minima, so
    # each round only sweeps the candidates that are new (in blocks of <= 256: the tensor path's limit) and folds
    # them into the per-chunk running minimum kept on the device.
    run_min = None
    swept = set()
    for i in range(n_iter):
        with _timer("init iteration %2d/%2d , %2d centers" % (i + 1, n_iter, len(c_idx)), _logger=logger):
            seed = int(rs.randint(0, 2 ** 31 - 1)) | (int(rs.randint(0, 2 ** 31 - 1)) << 32)
            fresh = sorted(c_idx - swept)
            phi_t = be.zeros((1,), torch.float64)
            step = _sweep_rows(X)
            blocks = [fresh[b0:b0 + step] for b0 in range(0, len(fresh), step)]
            for bi, blk in enumerate(blocks):
                block = X.global_rows(blk).astype(np.float64)
                _, mins_b, _ = sweep.run(block, want_min=True, squared=True)
                last = bi == len(blocks) - 1
                if run_min is None:
                    run_min = mins_b
                    if last:
                        for a in run_min:
                            be.min_fold(a, None, phi_t)
                else:
                    for a, b in zip(run_min, mins_b):
                        be.min_fold(a, b, phi_t if last else None)      # phi from the fully folded minimum only
            if not blocks:
                for a in run_min:
                    be.min_fold(a, None, phi_t)
            swept |= set(fresh)
            mins = run_min
            comm.allreduce_sum_(phi_t)
            phi = float(phi_t.item())
            _check_engine(be, phi, "the k-means|| cost")
            new_idxs = set()
            if phi > 0:
                cap = max(1024, 8 * int(oversampling_factor) + 1024)
                while True:
                    picked = be.empty((cap,), torch.int64)
                    n_picked = be.zeros((1,), torch.int32)
                    off = X.row_offset
                    for rows, mn in zip(X.chunk_rows, mins):
                        be.sample_chunk(mn, oversampling_factor / phi, seed, off, picked, n_picked)
                        off += int(rows)
                    m = int(n_picked.item())
                    if m <= cap:
                        break
                    cap = m
                local = picked[:m].cpu().numpy().tolist()
                for part in comm.allgather_obj(local):
                    new_idxs |= set(int(v) for v in part)
            c_idx |= new_idxs
    return sorted(c_idx)


def _reduce_candidates(cand, n_clusters, seed, be, weights=None, n_init=10, max_iter=300, tol=1e-4):
    """KMeans on the (few) k-means|| candidates, on the GPU: the stand-in for the in-memory scikit-learn KMeans of
    k_means.py:457-463 (``n_init`` restarts of k-means++ seeding + Lloyd, best inertia wins, scikit-learn's
    variance-scaled tolerance).  Runs identically on every rank (same candidates, same seed): no collective.
    Distances go through ``bkm_assign_chunk`` / the fused Lloyd kernels; the D^2 sampling and, for the weighted
    variant only, the weighted centre update are a few vector operations on the (m,) / (m, d) candidate arrays."""
    from ..engine import Comm, DeviceData
    from .._sparse import _csr_block

    sparse = scipy.sparse.issparse(cand)
    if sparse:
        # the candidates stay a CSR block and run through the sparse passes
        cand = scipy.sparse.csr_matrix(cand)
        m, d = cand.shape
        Xc = _SparseData([_csr_block(cand, be.device)], d, be, _LocalComm())
        c64 = cand.astype(np.float64)
        var = np.asarray(c64.multiply(c64).mean(axis=0)).ravel() - np.asarray(c64.mean(axis=0)).ravel() ** 2
        var_tol = float(np.mean(var) * tol)                                          # sklearn's _tolerance
        sweep = _SparseAssignPass(Xc)

        def dist_to(i):
            return sweep.run(cand[i], want_min=True)[1][0]
    else:
        cand = np.ascontiguousarray(cand)
        m, d = cand.shape
        dt = torch.float64 if cand.dtype == np.float64 else torch.float32
        Xc = DeviceData([be.to_device(cand, dt)], be, _LocalComm())
        x = Xc.chunks[0]
        var_tol = float(np.mean(np.var(cand.astype(np.float64), axis=0)) * tol)       # sklearn's _tolerance
    g = torch.Generator(device=be.device)
    g.manual_seed(int(seed) & 0x7FFFFFFFFFFFFFFF)
    w = None if weights is None else torch.as_tensor(np.asarray(weights, dtype=np.float64)).to(be.device).clamp_(min=0.0)
    best = None
    for _ in range(int(n_init)):
        # ---- k-means++ seeding (D^2 sampling) over the candidates
        first = int(torch.randint(0, m, (1,), generator=g, device=be.device).item()) if w is None else \
            int(torch.multinomial(w / w.sum(), 1, generator=g).item())
        chosen = [first]
        if sparse:
            closest = dist_to([first])
        else:
            closest = be.empty((m,), Xc.out_dtype)
            c1 = x[first:first + 1].to(torch.float64)
            be.assign_chunk(x, be.pack_centers(c1.contiguous(), dt), 1, None, closest, True, None)
        for _j in range(1, n_clusters):
            p = closest.to(torch.float64)
            if w is not None:
                p = p * w
            tot = float(p.sum().item())
            nxt = int(torch.multinomial(p / tot, 1, generator=g).item()) if tot > 0 else \
                int(torch.randint(0, m, (1,), generator=g, device=be.device).item())
            chosen.append(nxt)
            if sparse:
                newd = dist_to([nxt])
            else:
                newd = be.empty((m,), Xc.out_dtype)
                be.assign_chunk(x, be.pack_centers(x[nxt:nxt + 1].to(torch.float64).contiguous(), dt), 1, None, newd,
                                True, None)
            be.min_fold(closest, newd, None)
        if sparse:
            C0 = cand[chosen].toarray().astype(np.float64)
        else:
            C0 = x[torch.as_tensor(chosen, device=be.device)].to(torch.float64).cpu().numpy()
        # ---- Lloyd on the candidates
        if w is None:
            st = _lloyd_state(Xc, C0)
            lloyd_loop(st, max_iter, var_tol)
            inertia = float(st.relabel(squared=True).item())
            C = st.C.cpu().numpy()
        else:
            C = torch.as_tensor(C0).to(be.device)
            lab = be.empty((m,), torch.int32)
            inertia = None
            for _it in range(max_iter):
                be.assign_chunk(x, be.pack_centers(C.contiguous(), dt), n_clusters, lab, None, True, None)
                l64 = lab.long()
                sums = torch.zeros((n_clusters, d), dtype=torch.float64, device=be.device).index_add_(
                    0, l64, x.to(torch.float64) * w[:, None])
                cw = torch.zeros((n_clusters,), dtype=torch.float64, device=be.device).index_add_(0, l64, w)
                Cn = torch.where(cw[:, None] > 0, sums / cw.clamp(min=1e-300)[:, None], C)
                shift = float(((C - Cn) ** 2).sum().item())
                C = Cn
                if shift <= var_tol:
                    break
            dmin = be.empty((m,), Xc.out_dtype)
            be.assign_chunk(x, be.pack_centers(C.contiguous(), dt), n_clusters, lab, dmin, True, None)
            inertia = float((dmin.to(torch.float64) * w).sum().item())
            C = C.cpu().numpy()
        if best is None or inertia < best[0]:
            best = (inertia, C)
    return best[1]


class _LocalComm(object):
    """Single-rank communicator for work every rank repeats identically (the candidate reduce)."""

    rank, world = 0, 1

    def allreduce_sum_(self, t):
        return t

    def allgather_obj(self, obj):
        return [obj]

    def bcast_obj(self, obj, src=0):
        return obj


def evaluate_cost(X, centers):
    """phi_X(C) = sum_i min_j ||x_i - c_j||^2 (k_means.py:466-469); X is DeviceData."""
    X = _to_device_data(X, check_finite=False)
    _, _, acc = _assign_pass(X).run(np.asarray(centers, dtype=np.float64), squared=True)
    return float(acc.item())


# ---------------------------------------------------------------------------------------
# EM steps
# ---------------------------------------------------------------------------------------
class LloydState(object):
    """Device-resident state of the Lloyd loop (k_means.py:522-560).

    Two ways to drive it:
      * ``run(max_iter, tol)`` — the DEVICE-RESIDENT loop (CUDA backend): per iteration one fused E+M call per chunk
        (the first one overwrites the accumulators, no memsets), one all-reduce of ``[k*d sums | k counts | inertia]``
        when distributed, and ``bkm_finalize_step`` (centre update + shift + stop test + the next iteration's centre
        pack in one kernel).  The stop test runs on the device; the host enqueues ``sync_every`` iterations at a time
        and reads the 40-byte loop state once per batch; iterations enqueued after convergence are no-ops.
      * ``step()`` / ``accept()`` — one iteration with the shift left on the device (the CPU checker backend of the
        tests and ``lloyd_iteration_host`` use the same arithmetic through ``finalize``).
    """

    def __init__(self, X, centers):
        be = X.backend
        self.X, self.be = X, be
        k, d = centers.shape
        self.k, self.d = int(k), int(d)
        # private copies: the state is updated in place and must never alias the caller's `init`.
        # Two centre buffers: iteration i reads Cb[cur] and writes Cb[cur ^ 1].
        c0 = torch.from_numpy(np.array(centers, dtype=np.float64, order="C", copy=True)).to(be.device)
        self.Cb = [c0, be.empty((k, d), torch.float64)]
        self.cur = 0
        # one buffer so that the per-iteration collective is a single all-reduce
        self.red = be.zeros((k * d + k + 1,), torch.float64)
        self.sums = self.red[: k * d]
        self.counts_f = self.red[k * d: k * d + k]
        self.inertia = self.red[k * d + k:]
        self.counts = be.zeros((k,), torch.int64)
        self.shift = be.zeros((1,), torch.float64)
        self.labels = [be.empty((m,), torch.int32) for m in X.chunk_rows]
        self.pack = None
        self.device_loop = hasattr(be, "finalize_step")
        self.kernel_event_hook = None        # bench.py: () -> (start_event, end_event) around the chunk kernels
        self.sync_every = 8

    # the current centres / the other buffer
    @property
    def C(self):
        return self.Cb[self.cur]

    @property
    def C_new(self):
        return self.Cb[self.cur ^ 1]

    def step(self, kernel_events=None):
        be, X, k = self.be, self.X, self.k
        self.pack = be.pack_centers(self.C, X.dtype, out=self.pack)
        self.red.zero_()
        self.counts.zero_()
        if kernel_events is not None:       # bench.py: CUDA events around the fused chunk kernel(s)
            kernel_events[0].record()
        for x, lab in zip(X.chunks, self.labels):
            # per-row distances are not needed inside the loop: the inertia is produced by relabel()
            be.lloyd_chunk(x, self.pack, k, lab, None, self.sums, self.counts, None)
        if kernel_events is not None:
            kernel_events[1].record()
        if X.comm.world > 1:
            self.counts_f.copy_(self.counts)
            X.comm.allreduce_sum_(self.red)
            self.counts.copy_(self.counts_f.round())
        be.finalize(self.sums, self.counts, self.C, self.C_new, self.shift)

    def accept(self):
        self.cur ^= 1

    def run(self, max_iter, tol):
        """The device-resident loop.  Returns ``(shift, index of the last iteration, accepted)`` like ``lloyd_loop``."""
        be, X, k = self.be, self.X, self.k
        state, hist = be.loop_state_new(tol, max_iter)
        self.pack = be.pack_centers(self.C, X.dtype, out=self.pack)       # iteration 0's pack; later ones come from finalize_step
        resident = isinstance(X.chunks, list)
        work = [(x, lab) for x, lab in zip(X.chunks, self.labels) if int(x.shape[0]) > 0] if resident else None
        base = self.cur
        issued = 0
        done = n_iter = 0
        shift = None
        logged = 0
        while issued < max_iter and not done:
            for _ in range(min(self.sync_every, max_iter - issued)):
                c_in, c_out = self.Cb[(base + issued) & 1], self.Cb[(base + issued + 1) & 1]
                ev = self.kernel_event_hook() if self.kernel_event_hook is not None else None
                if ev is not None:
                    ev[0].record()
                if X.n_local == 0:
                    self.red.zero_()                  # a rank without rows still takes part in the all-reduce
                first = True
                # resident chunks: the prepared list; host-resident data: one streamed sweep per iteration
                for x, lab in (work if resident else zip(X.chunks, self.labels)):
                    if int(x.shape[0]) == 0:
                        continue
                    be.lloyd_chunk(x, self.pack, k, lab, None, self.sums, self.counts_f, None, first=first,
                                   loop_state=state)
                    first = False
                if ev is not None:
                    ev[1].record()
                X.comm.allreduce_sum_(self.red)
                be.finalize_step(self.red, c_in, c_out, state, self.pack, X.dtype)
                issued += 1
            done, n_iter, shift = be.loop_state_read(state)      # the only host synchronisation of the batch
            _check_engine(be, shift, "the centre shift")
            if logger.isEnabledFor(logging.INFO):
                for v in hist[logged:n_iter].cpu().numpy().tolist():
                    logger.info("Lloyd loop %2d. Shift: %0.4f", logged, v)
                    logged += 1
        if shift is None:
            return None, -1, False
        # converged in iteration n_iter - 1: its update was NOT taken over (Q3) -> the centres it read are current
        self.cur = (base + n_iter - 1) & 1 if done else (base + n_iter) & 1
        self.shift.fill_(shift)
        return shift, n_iter - 1, not done

    def relabel(self, squared):
        """E-step only against the current centres; returns the summed min distance tensor."""
        be, X, k = self.be, self.X, self.k
        self.pack = be.pack_centers(self.C, X.dtype, out=self.pack)
        acc = be.zeros((1,), torch.float64)
        for x, lab in zip(X.chunks, self.labels):
            be.assign_chunk(x, self.pack, k, lab, None, squared, acc)
        X.comm.allreduce_sum_(acc)
        return acc


class _SparseLloydState(object):
    """``LloydState`` on sparse CSR blocks.  The centres live in a sparse pack (``bkm_sparse_pack_centers``): CT (d, k),
    the transposed centres, then their squared norms; two packs, iteration i reads packs[cur] and writes the other.

    One iteration on each rank: the assign pass (labels and counts) over every block, the label-sum pass
    (sumsT (d, k) = X^T onehot(labels)) over every block's transpose, one all-reduce of ``[d*k sumsT | k counts |
    inertia]``, then ``bkm_sparse_finalize_step`` (centre update + shift + stop test + the next pack).  Memory: the two
    packs and the reduced buffer, 3 * 8 d k bytes.
      * ``run(max_iter, tol)`` — the device-resident loop, as ``LloydState.run``.
      * ``step()`` / ``accept()`` — one iteration with the shift left in ``shift`` (the CPU checker backend)."""

    def __init__(self, X, centers):
        be = X.backend
        self.X, self.be = X, be
        k, d = centers.shape
        self.k, self.d = int(k), int(d)
        c0 = torch.from_numpy(np.array(centers, dtype=np.float64, order="C", copy=True)).to(be.device)
        self.packs = [be.sparse_pack_centers(c0), be.empty((d * k + k,), torch.float64)]
        self.cur = 0
        self.red = be.zeros((d * k + k + 1,), torch.float64)
        self.sums = self.red[: d * k].view(d, k)
        self.counts_f = self.red[d * k: d * k + k]
        self.shift = be.zeros((1,), torch.float64)
        self.labels = [be.empty((int(b[3]),), torch.int32) for b in X.blocks]
        self.device_loop = hasattr(be, "sparse_finalize_step") and hasattr(be, "loop_state_new")
        self.kernel_event_hook = None
        self.sync_every = 8

    @property
    def C(self):
        """The current centres, (k, d) float64 (a view of the pack's CT)."""
        return self.packs[self.cur][: self.d * self.k].view(self.d, self.k).t()

    def _sweep(self, pack, state=None):
        """The two passes of one iteration into ``red`` (before the all-reduce)."""
        be, X, k, d = self.be, self.X, self.k, self.d
        work = [(b, c, lab) for b, c, lab in zip(X.blocks, X.transposes(), self.labels) if int(b[3]) > 0]
        if not work:
            self.red.zero_()                  # a rank without rows still takes part in the all-reduce
        for i, (b, _c, lab) in enumerate(work):
            be.csr_assign_chunk(b, d, pack, k, labels=lab, counts=self.counts_f, first=i == 0, loop_state=state)
        for i, (_b, c, lab) in enumerate(work):
            be.csc_label_sums_chunk(c, d, lab, k, self.sums, first=i == 0, loop_state=state)

    def step(self):
        self._sweep(self.packs[self.cur])
        self.X.comm.allreduce_sum_(self.red)
        self.be.sparse_finalize(self.red, self.packs[self.cur], self.packs[self.cur ^ 1], self.shift, self.k, self.d)

    def accept(self):
        self.cur ^= 1

    def run(self, max_iter, tol):
        """The device-resident loop.  Returns ``(shift, index of the last iteration, accepted)`` like ``lloyd_loop``."""
        be, X, k, d = self.be, self.X, self.k, self.d
        state, hist = be.loop_state_new(tol, max_iter)
        base = self.cur
        issued = 0
        done = n_iter = 0
        shift = None
        logged = 0
        while issued < max_iter and not done:
            for _ in range(min(self.sync_every, max_iter - issued)):
                p_in, p_out = self.packs[(base + issued) & 1], self.packs[(base + issued + 1) & 1]
                ev = self.kernel_event_hook() if self.kernel_event_hook is not None else None
                if ev is not None:
                    ev[0].record()
                self._sweep(p_in, state)
                if ev is not None:
                    ev[1].record()
                X.comm.allreduce_sum_(self.red)
                be.sparse_finalize_step(self.red, p_in, p_out, state, k, d)
                issued += 1
            done, n_iter, shift = be.loop_state_read(state)
            _check_engine(be, shift, "the centre shift")
            if logger.isEnabledFor(logging.INFO):
                for v in hist[logged:n_iter].cpu().numpy().tolist():
                    logger.info("Lloyd loop %2d. Shift: %0.4f", logged, v)
                    logged += 1
        if shift is None:
            return None, -1, False
        # converged in iteration n_iter - 1: its pack was NOT taken over (Q3) -> the pack it read is current
        self.cur = (base + n_iter - 1) & 1 if done else (base + n_iter) & 1
        self.shift.fill_(shift)
        return shift, n_iter - 1, not done

    def relabel(self, squared):
        """E-step only against the current centres; returns the summed min distance tensor."""
        be, X, k = self.be, self.X, self.k
        acc = be.zeros((1,), torch.float64)
        for b, lab in zip(X.blocks, self.labels):
            be.csr_assign_chunk(b, X.d, self.packs[self.cur], k, labels=lab, squared=squared, dist_sum=acc)
        X.comm.allreduce_sum_(acc)
        return acc


def _lloyd_state(X, centers):
    return _SparseLloydState(X, centers) if isinstance(X, _SparseData) else LloydState(X, centers)


def _check_engine(be, value, what):
    """A poisoned step (NaN shift / cost, see bkm_debug_abort_code) becomes an error."""
    if value == value and abs(value) != float("inf"):
        return
    code = be.abort_code() if hasattr(be, "abort_code") else 0
    if code:
        be.reset_abort()
        raise RuntimeError("KMeans engine: a pipeline wait inside the tensor kernel timed out (abort code 0x%08x) "
                           "while computing %s; the results of this call are invalid" % (code, what))
    raise RuntimeError("KMeans engine: non-finite %s (%r) — X or the centres hold values outside the range of "
                       "their dtype" % (what, value))


def lloyd_loop(st, max_iter, tol):
    """The Lloyd iterations of k_means.py:522-560 over a ``LloydState``.  ``bench.py`` times this very function.
    CUDA backend: ``LloydState.run`` (device-resident stop test, one host read of the loop state per batch of
    iterations).  Checker backend of the CPU tests: one ``step()`` and one host read of the shift per iteration.
    Returns ``(shift, index of the last iteration, accepted)``; ``accepted`` tells whether ``st.C`` already holds the
    centres computed by the last iteration (False after the convergence ``break``, Q3)."""
    if getattr(st, "device_loop", False):
        with _timer("Lloyd loop (device-resident, %d iterations at most)" % max_iter, _logger=logger):
            return st.run(max_iter, tol)
    shift = None
    i = -1
    accepted = False
    for i in range(max_iter):
        with _timer("Lloyd loop %2d." % i, _logger=logger):
            st.step()
            shift = float(st.shift.item())       # the one host sync per iteration (k_means.py:552)
            _check_engine(st.be, shift, "the centre shift")
            logger.info("Shift: %0.4f", shift)
            accepted = False
            if shift < tol:
                break                            # Q3: break BEFORE centers = new_centers
            st.accept()
            accepted = True
    return shift, i, accepted


def _kmeans_single_lloyd(
    X,
    n_clusters,
    max_iter=300,
    init="k-means||",
    verbose=False,
    x_squared_norms=None,
    random_state=None,
    tol=1e-4,
    precompute_distances=True,
    oversampling_factor=2,
    init_max_iter=None,
):
    """Lloyd iterations with the reference's exact control flow (k_means.py:499-569)."""
    X = _to_device_data(X)
    if isinstance(X, _SparseData):
        check_label_sum_classes(n_clusters, "clusters")
    centers = k_init(
        X,
        n_clusters,
        init=init,
        oversampling_factor=oversampling_factor,
        random_state=random_state,
        max_iter=init_max_iter,
    )
    dt = X.np_dtype
    st = _lloyd_state(X, np.asarray(centers))
    shift, i, accepted = lloyd_loop(st, max_iter, tol)

    if shift is None:
        raise ValueError("max_iter must be at least 1, got %r" % (max_iter,))

    if shift > 1e-7:
        # Q4: re-label against the current centres with the default (non-squared) metric
        inertia = float(st.relabel(squared=False).item())
        _check_engine(st.be, inertia, "the inertia")
    else:
        # Q4, other side: inertia = sum of the SQUARED distances of the last E-step, i.e. against the
        # centres that E-step used.  The loop does not keep per-row distances, so they are produced here
        # by one E-step-only pass against those same centres (labels are identical).
        if accepted:
            st.accept()                          # back to the centres of the last E-step
        inertia = float(st.relabel(squared=True).item())
        _check_engine(st.be, inertia, "the inertia")
        if accepted:
            st.accept()

    labels = ChunkedArray(st.labels)
    centers = st.C.cpu().numpy().astype(dt)
    return labels, np.float64(inertia), centers, i + 1


def lloyd_iteration_host(X_host, centers, backend=None, comm=None, block_rows=1 << 20):
    """One Lloyd iteration (k_means.py:523-555) over a HOST-resident row chunk.

    ``X_host`` is a (n, d) float32/float64 torch CPU tensor (pinned memory makes the copies
    asynchronous) or numpy array.  Row blocks are streamed host->device through two device buffers
    on a copy stream while the fused E+M kernel consumes the previous block, so X crosses PCIe exactly
    once per iteration; then the all-reduce, the centre update and a device->host read of the result.
    Returns ``(new_centers float64 (k,d), inertia float64, shift float64)`` on the host.
    This is the ingestion path for data that is not (or does not fit) resident in HBM.
    """
    be = backend or _get_backend()
    comm = comm or Comm()
    if not _is_torch(X_host):
        X_host = torch.from_numpy(np.ascontiguousarray(X_host))
    n, d = int(X_host.shape[0]), int(X_host.shape[1])
    dt = X_host.dtype
    centers = np.ascontiguousarray(centers, dtype=np.float64)
    k = int(centers.shape[0])
    cache = getattr(be, "_host_iter_cache", None)
    key = (block_rows, d, dt, k)
    if cache is None or cache["key"] != key:
        cache = {
            "key": key,
            "bufs": [be.empty((block_rows, d), dt) for _ in range(2)],
            "copy_stream": torch.cuda.Stream(device=be.device),
            "red": be.zeros((k * d + k + 1,), torch.float64),
            "counts": be.zeros((k,), torch.int64),
            "C": be.empty((k, d), torch.float64),
            "C_new": be.empty((k, d), torch.float64),
            "shift": be.zeros((1,), torch.float64),
            "pack": None,
            "out_host": torch.empty((k * d + 2,), dtype=torch.float64).pin_memory(),
        }
        be._host_iter_cache = cache
    bufs, cs = cache["bufs"], cache["copy_stream"]
    red, counts = cache["red"], cache["counts"]
    sums, counts_f, inertia = red[: k * d], red[k * d: k * d + k], red[k * d + k:]
    main = torch.cuda.current_stream(be.device)
    cache["C"].copy_(torch.from_numpy(centers), non_blocking=True)
    cache["pack"] = be.pack_centers(cache["C"], dt, out=cache["pack"])
    red.zero_()
    counts.zero_()
    copied = [None, None]
    consumed = [None, None]
    nblk = (n + block_rows - 1) // block_rows
    for b in range(nblk):
        s0 = b * block_rows
        m = min(block_rows, n - s0)
        slot = b & 1
        with torch.cuda.stream(cs):
            if consumed[slot] is not None:
                cs.wait_event(consumed[slot])
            bufs[slot][:m].copy_(X_host[s0:s0 + m], non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(cs)
            copied[slot] = ev
        main.wait_event(copied[slot])
        be.lloyd_chunk(bufs[slot][:m], cache["pack"], k, None, None, sums, counts, inertia)
        ev = torch.cuda.Event()
        ev.record(main)
        consumed[slot] = ev
    if comm.world > 1:
        counts_f.copy_(counts)
        comm.allreduce_sum_(red)
        counts.copy_(counts_f.round())
    be.finalize(sums, counts, cache["C"], cache["C_new"], cache["shift"])
    out = cache["out_host"]
    out[: k * d].copy_(cache["C_new"].view(-1), non_blocking=True)
    out[k * d: k * d + 1].copy_(inertia, non_blocking=True)
    out[k * d + 1:].copy_(cache["shift"], non_blocking=True)
    main.synchronize()
    res = out.numpy()
    return res[: k * d].reshape(k, d).copy(), float(res[k * d]), float(res[k * d + 1])
