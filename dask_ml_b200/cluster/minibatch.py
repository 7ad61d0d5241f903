"""PartialMiniBatchKMeans with the dask_ml.cluster.PartialMiniBatchKMeans API, executed by the H100 engine.

Mirrors dask_ml/cluster/minibatch.py and the block-wise fit of dask_ml/_partial.py:39-100 (reference @ 0310a90): a
scikit-learn ``MiniBatchKMeans`` whose ``fit`` calls ``partial_fit`` once per row block, in the order
``check_random_state(None).shuffle`` gives, continuing from whatever state is already learned.

``partial_fit`` follows the installed scikit-learn's ``MiniBatchKMeans.partial_fit`` (sklearn/cluster/_kmeans.py)
step for step.  The work over the rows of a batch runs in CUDA: one fused E+M pass (``bkm_lloyd_chunk``: labels,
float64 sums and counts), then ``bkm_minibatch_step`` (``_minibatch_update_dense``: the centre and weight-sum update
and the next centre pack).  The host reads k weight sums and the batch inertia once per batch: the reassignment
decision and the random draws of scikit-learn depend on them, and run on the host in numpy with the estimator's
RandomState, so the RNG stream is scikit-learn's.

Sparse CSR batches (any form ``KMeans`` takes) run scikit-learn's ``_minibatch_update_sparse`` the same way on the
transposed centres: per block the CSR arg-min pass, the block's transpose and the label-indexed column sums, then
``bkm_sparse_minibatch_step``.
"""
import logging
import warnings

import numpy as np
import scipy.sparse
import torch
from sklearn.base import _fit_context
from sklearn.cluster import MiniBatchKMeans, kmeans_plusplus
from sklearn.utils import check_array as _sk_check_array
from sklearn.utils import check_random_state
from sklearn.utils.validation import _is_arraylike_not_scalar, check_is_fitted

from .._sparse import _SparseData, check_label_sum_classes
from ..chunked import ChunkedArray
from ..engine import StreamedChunks, single_process
from . import k_means as _km
from .k_means import KMeans

logger = logging.getLogger(__name__)

_partial_deprecation = (
    "'{cls.__name__}' is deprecated. Use "
    "'dask_ml.wrappers.Incremental({base.__name__}(), **kwargs)' "
    "instead."
)


def _single_process():
    single_process("PartialMiniBatchKMeans")


class _Shape(object):
    """Stands in for X in scikit-learn helpers that only read ``X.shape``."""

    def __init__(self, n, d):
        self.shape = (n, d)


class _MiniBatchState(object):
    """Device state between batches: float64 centres and weight sums (ping-pong pairs, ``[cur]`` is current), the
    ``[k*d sums | k counts | inertia]`` buffer of one batch and the centre pack of the current centres."""

    def __init__(self, be, centers, weight_sums, dtype):
        k, d = centers.shape
        self.k, self.d = int(k), int(d)
        c0 = torch.from_numpy(np.array(centers, dtype=np.float64, order="C", copy=True)).to(be.device)
        w0 = torch.from_numpy(np.array(weight_sums, dtype=np.float64, copy=True)).to(be.device)
        self.Cb = [c0, be.empty((k, d), torch.float64)]
        self.Wb = [w0, be.empty((k,), torch.float64)]
        self.cur = 0
        self.red = be.zeros((k * d + k + 1,), torch.float64)
        self.sums = self.red[: k * d]
        self.counts = self.red[k * d: k * d + k]
        self.inertia = self.red[k * d + k:]
        self.dtype = dtype
        self.pack = be.pack_centers(self.C, dtype)
        cuda = be.device.type == "cuda"
        self.host = torch.empty((k + 1,), dtype=torch.float64, pin_memory=cuda)
        self.read_done = None

    @property
    def C(self):
        return self.Cb[self.cur]

    @property
    def W(self):
        return self.Wb[self.cur]

    def step(self, be, chunks, dtype):
        """Enqueue one batch: the fused E+M pass over its chunks, then the centre / weight-sum update and the pack."""
        if dtype != self.dtype:                 # a batch of another dtype than the previous one
            self.dtype = dtype
            self.pack = be.pack_centers(self.C, dtype, out=self.pack)
        first = True
        for x in chunks:
            # a chunk without rows launches nothing, so it cannot be the one that overwrites the previous batch's sums
            if int(x.shape[0]) == 0:
                continue
            be.lloyd_chunk(x, self.pack, self.k, None, None, self.sums, self.counts, self.inertia, first=first)
            first = False
        be.minibatch_step(self.red, self.Cb[self.cur], self.Wb[self.cur], self.Cb[self.cur ^ 1], self.Wb[self.cur ^ 1],
                          self.pack, self.dtype)
        self.cur ^= 1

    def start_read(self):
        """Enqueue the copy of the weight sums and the batch inertia to the host."""
        self.host[: self.k].copy_(self.W, non_blocking=True)
        self.host[self.k:].copy_(self.inertia, non_blocking=True)
        if self.W.is_cuda:
            self.read_done = torch.cuda.Event()
            self.read_done.record(torch.cuda.current_stream(self.W.device))

    def finish_read(self):
        """(weight sums float64 (k,), batch inertia): waits for the copies of ``start_read`` only."""
        if self.read_done is not None:
            self.read_done.synchronize()
            self.read_done = None
        v = self.host.numpy()
        return v[: self.k].copy(), float(v[self.k])


def _rows(x):
    """Rows of a dense chunk or of a sparse (crow, col, val, n) block."""
    return int(x[3]) if isinstance(x, tuple) else int(x.shape[0])


class _SparseMiniBatchState(object):
    """``_MiniBatchState`` for sparse CSR batches: two sparse packs (``bkm_sparse_pack_centers``: the centres transposed,
    (d, k), then their squared norms) and two float64 weight-sum vectors, ping-pong pairs with ``[cur]`` current, and
    the ``[d*k sumsT | k counts | inertia]`` buffer of one batch.  Memory: 3 * 8 d k bytes, as for sparse ``KMeans``.

    Each block's transpose is built for its step and dropped after it; its canonical-CSR flag is added on the device
    and read with the weight sums."""

    def __init__(self, be, centers, weight_sums):
        k, d = centers.shape
        self.k, self.d = int(k), int(d)
        c0 = torch.from_numpy(np.array(centers, dtype=np.float64, order="C", copy=True)).to(be.device)
        w0 = torch.from_numpy(np.array(weight_sums, dtype=np.float64, copy=True)).to(be.device)
        self.packs = [be.sparse_pack_centers(c0), be.empty((d * k + k,), torch.float64)]
        self.Wb = [w0, be.empty((k,), torch.float64)]
        self.cur = 0
        self.red = be.zeros((d * k + k + 1,), torch.float64)
        self.sums = self.red[: d * k].view(d, k)
        self.counts = self.red[d * k: d * k + k]
        self.inertia = self.red[d * k + k:]
        self.bad = be.zeros((1,), torch.float64)
        cuda = be.device.type == "cuda"
        self.host = torch.empty((k + 2,), dtype=torch.float64, pin_memory=cuda)
        self.read_done = None

    @property
    def C(self):
        """The current centres, (k, d) float64 (a view of the current pack)."""
        return self.packs[self.cur][: self.d * self.k].view(self.d, self.k).t()

    @property
    def W(self):
        return self.Wb[self.cur]

    def step(self, be, blocks, dtype=None):
        """Enqueue one batch: per block with rows the assign pass (labels, counts, the batch inertia), the block's
        transpose and the label sums; then the centre / weight-sum update and the next pack."""
        k, d = self.k, self.d
        pack = self.packs[self.cur]
        self.bad.zero_()
        first = True
        for blk in blocks:
            n = _rows(blk)
            if n == 0:
                continue
            lab = be.empty((n,), torch.int32)
            be.csr_assign_chunk(blk, d, pack, k, labels=lab, counts=self.counts, dist_sum=self.inertia, first=first)
            csc = be.csr_transpose_chunk(blk, d)
            self.bad += csc[3][0]
            be.csc_label_sums_chunk(csc, d, lab, k, self.sums, first=first)
            first = False
        be.sparse_minibatch_step(self.red, pack, self.Wb[self.cur], self.packs[self.cur ^ 1], self.Wb[self.cur ^ 1], k, d)
        self.cur ^= 1

    def undo(self):
        """Back to the state before the last step (its inputs are still in the other halves of the pairs)."""
        self.cur ^= 1

    def set_centres(self, be, C):
        """Repack the current pack from the float64 centres C (k, d)."""
        self.packs[self.cur] = be.sparse_pack_centers(C.contiguous(), out=self.packs[self.cur])

    def start_read(self):
        """Enqueue the copy of the weight sums, the batch inertia and the canonical-CSR flag to the host."""
        self.host[: self.k].copy_(self.W, non_blocking=True)
        self.host[self.k: self.k + 1].copy_(self.inertia, non_blocking=True)
        self.host[self.k + 1:].copy_(self.bad, non_blocking=True)
        if self.W.is_cuda:
            self.read_done = torch.cuda.Event()
            self.read_done.record(torch.cuda.current_stream(self.W.device))

    def finish_read(self):
        """(weight sums float64 (k,), batch inertia, non-canonical blocks)."""
        if self.read_done is not None:
            self.read_done.synchronize()
            self.read_done = None
        v = self.host.numpy()
        return v[: self.k].copy(), float(v[self.k]), float(v[self.k + 1])


def _new_state(be, X, centers, weight_sums):
    if isinstance(X, _SparseData):
        return _SparseMiniBatchState(be, centers, weight_sums)
    return _MiniBatchState(be, centers, weight_sums, X.dtype)


class PartialMiniBatchKMeans(MiniBatchKMeans):
    """Mini-batch k-means over the row blocks of X (API of dask_ml.cluster.PartialMiniBatchKMeans).

    .. deprecated:: 0.6.0 (in dask-ml)
       Use the :class:`dask_ml.wrappers.Incremental` meta-estimator instead.

    ``fit`` passes the row blocks of X, in a random order, to ``partial_fit``, one block per mini-batch step: each
    block is read once, so this is the estimator for data larger than device memory
    (``dask_ml_b200.engine.host_resident``).  Parameters, ``get_params``, ``clone`` and their validation are
    scikit-learn's ``MiniBatchKMeans``'s.

    X may also be sparse (a ChunkedArray of torch CSR blocks, one torch CSR tensor or a scipy.sparse matrix): each
    step then keeps the centres transposed in a sparse pack, 3 * 8 n_features n_clusters bytes of device memory.  Dense
    and sparse batches may follow each other; they continue from the same float64 state.

    Differences from scikit-learn: centres and weight sums are kept in float64 on the device whatever the dtype of X
    (scikit-learn keeps float32 for float32 X, whose counters stop counting exactly above 2^24 rows per cluster);
    ``sample_weight`` is not supported (the fused kernels add rows unweighted); ``labels_`` is a device-resident int32
    ``ChunkedArray``.  A pickled estimator keeps the float64 centres and weight sums, so an unpickled one continues
    exactly where the original would.

    Attributes
    ----------
    cluster_centers_ : np.ndarray (n_clusters, n_features), dtype of X (float32 for bfloat16 rows)
    labels_ : ChunkedArray (n_samples of the last batch,) int32, with ``compute_labels``
    inertia_ : float, squared distances of the last batch to the new centres, with ``compute_labels``
    n_steps_ : int, number of mini-batch steps (blocks) processed so far
    """

    def __init__(self, **kwargs):
        self._deprecated()
        super().__init__(**kwargs)

    @classmethod
    def _deprecated(cls):
        for base in cls.mro():
            if base.__module__.startswith("sklearn"):
                break
        warnings.warn(_partial_deprecation.format(cls=cls, base=base), FutureWarning)

    @classmethod
    def _get_param_names(cls):
        # __init__ takes **kwargs: the parameters are those of the scikit-learn class
        for base in cls.mro():
            if base.__module__.startswith("sklearn"):
                return base._get_param_names()

    def __getstate__(self):
        # the device buffers are pickled as float64 host arrays (cluster_centers_ and _counts are rounded to X's dtype)
        # and moved back to the device by the next step
        state = dict(self.__dict__)
        st = state.pop("_mb", None)
        if st is not None:
            state["_mb_host"] = (st.C.cpu().numpy(), st.W.cpu().numpy())
        return state

    _check_array = KMeans._check_array
    predict = KMeans.predict
    transform = KMeans.transform

    def _check_n_features(self, X):
        if X.d != self.n_features_in_:
            raise ValueError("X has {} features, but {} is expecting {} features as input.".format(
                X.d, type(self).__name__, self.n_features_in_))

    def score(self, X, y=None, sample_weight=None):
        """Opposite of the sum of squared distances of the rows of X to their closest centre."""
        if sample_weight is not None:
            raise NotImplementedError("sample_weight is not supported")
        check_is_fitted(self, "cluster_centers_")
        X = self._check_array(X)
        self._check_n_features(X)
        return -_km.evaluate_cost(X, self.cluster_centers_)

    @_fit_context(prefer_skip_nested_validation=True)
    def fit(self, X, y=None, compute=True):
        """One ``partial_fit`` step per row block, in the order ``check_random_state(None).shuffle`` gives (the global
        numpy RNG), continuing from the state already learned.  Host-resident data is streamed block by block, each
        block once; the labels and inertia of the last block are computed after the last step only (every earlier
        value would be overwritten)."""
        if not compute:
            raise NotImplementedError("compute=False: PartialMiniBatchKMeans.fit runs eagerly, there is no lazy result")
        _single_process()
        X = self._check_array(X)
        order = list(range(len(X.chunk_rows)))
        check_random_state(None).shuffle(order)
        if isinstance(X, _SparseData):
            blocks = (X.blocks[i] for i in order)
        elif isinstance(X.chunks, StreamedChunks):
            blocks = X.chunks.iter_order(order)
        else:
            blocks = (X.chunks[i] for i in order)
        nxt = next(blocks, None)
        for pos, i in enumerate(order):
            x, off = nxt, int(X.chunk_offsets[i])
            reassign = self._step_begin(X, [x], off)
            # streamed data: the next block's host->device copy is enqueued before the host waits for this step
            nxt = next(blocks, None)
            self._step_end(X, [x], off, reassign, self.compute_labels and pos == len(order) - 1)
        self._publish(X)
        return self

    @_fit_context(prefer_skip_nested_validation=True)
    def partial_fit(self, X, y=None, sample_weight=None):
        """Update the centres with one mini-batch X (scikit-learn's ``MiniBatchKMeans.partial_fit``)."""
        if sample_weight is not None:
            raise NotImplementedError("sample_weight is not supported: the fused kernels add rows unweighted")
        _single_process()
        X = self._check_array(X)
        chunks = X.blocks if isinstance(X, _SparseData) else X.chunks
        reassign = self._step_begin(X, chunks, 0)
        self._step_end(X, chunks, 0, reassign, self.compute_labels)
        self._publish(X)
        return self

    # -----------------------------------------------------------------------------------------------------------
    def _check_batch_params(self, n):
        """The parts of ``MiniBatchKMeans._check_params_vs_input`` that ``partial_fit`` uses (``_tol`` is not)."""
        if n < self.n_clusters:
            raise ValueError(f"n_samples={n} should be >= n_clusters={self.n_clusters}.")
        if self.n_init == "auto":
            self._n_init = 1 if (isinstance(self.init, str) and self.init == "k-means++") or \
                _is_arraylike_not_scalar(self.init) else 3
        else:
            self._n_init = self.n_init
        if _is_arraylike_not_scalar(self.init) and self._n_init != 1:
            warnings.warn(
                "Explicit initial center position passed: performing only"
                f" one init in {self.__class__.__name__} instead of "
                f"n_init={self._n_init}.",
                RuntimeWarning,
                stacklevel=3,
            )
            self._n_init = 1
        self._batch_size = min(self.batch_size, n)
        self._init_size = self.init_size
        if self._init_size is None:
            self._init_size = 3 * self._batch_size
            if self._init_size < self.n_clusters:
                self._init_size = 3 * self.n_clusters
        elif self._init_size < self.n_clusters:
            warnings.warn(
                f"init_size={self._init_size} should be larger than "
                f"n_clusters={self.n_clusters}. Setting it to "
                "min(3*n_clusters, n_samples)",
                RuntimeWarning,
                stacklevel=3,
            )
            self._init_size = 3 * self.n_clusters
        self._init_size = min(self._init_size, n)

    @staticmethod
    def _host_rows(X, idx):
        """Local rows of X on the host: numpy, or a scipy CSR for sparse X."""
        return X._local_csr(idx) if isinstance(X, _SparseData) else X.local_rows(idx)

    @staticmethod
    def _dense_rows(X, idx):
        """Local rows of X as a float64-able numpy array (sparse rows densified, as scikit-learn's ``toarray()``)."""
        return X._local_csr(idx).toarray() if isinstance(X, _SparseData) else X.local_rows(idx)

    def _init_centroids_host(self, X, off, n):
        """``_BaseKMeans._init_centroids`` on ``init_size`` rows of the batch, gathered to the host."""
        rs = self._random_state
        init = self.init
        if _is_arraylike_not_scalar(init):
            init = _sk_check_array(init, dtype=X.np_dtype, copy=True, order="C")
            self._validate_center_shape(_Shape(n, X.d), init)
        idx = np.arange(n)
        if self._init_size < n:
            idx = rs.randint(0, n, self._init_size)
        if isinstance(init, str) and init == "k-means++":
            centers, _ = kmeans_plusplus(self._host_rows(X, off + idx), self.n_clusters, random_state=rs)
        elif isinstance(init, str) and init == "random":
            sw = np.ones(len(idx), dtype=X.np_dtype)
            seeds = rs.choice(len(idx), size=self.n_clusters, replace=False, p=sw / sw.sum())
            centers = self._dense_rows(X, off + idx[seeds])
        elif _is_arraylike_not_scalar(init):
            centers = init
        else:
            centers = init(self._host_rows(X, off + idx), self.n_clusters, random_state=rs)
            if scipy.sparse.issparse(centers):
                centers = centers.toarray()
            centers = _sk_check_array(centers, dtype=X.np_dtype, copy=False, order="C")
            self._validate_center_shape(_Shape(n, X.d), centers)
        return centers

    @staticmethod
    def _batch_rows(X, chunks):
        return int(sum(_rows(x) for x in chunks)) if isinstance(chunks, list) else X.n_local

    def _step_begin(self, X, chunks, off):
        """First half of ``partial_fit`` on the batch made of the rows ``off, off + 1, ...`` of X that ``chunks``
        (device tensors, or the streamed chunks of X) hold: validation, the initialisation on the first call, the
        reassignment decision, and the step enqueued on the device.  Returns the reassignment decision."""
        be = X.backend
        n = self._batch_rows(X, chunks)
        st = getattr(self, "_mb", None)
        has_centers = st is not None or hasattr(self, "cluster_centers_")
        if n == 0:
            raise ValueError("Found array with 0 sample(s) (shape=(0, %d)) while a minimum of 1 is required by %s."
                             % (X.d, type(self).__name__))
        if has_centers:
            self._check_n_features(X)
        elif isinstance(X, _SparseData):
            check_label_sum_classes(self.n_clusters, "clusters")
        self._random_state = getattr(self, "_random_state", check_random_state(self.random_state))
        self.n_steps_ = getattr(self, "n_steps_", 0)

        if not has_centers:
            self._check_batch_params(n)
            centers = self._init_centroids_host(X, off, n)
            self._counts = np.zeros(self.n_clusters, dtype=X.np_dtype)
            self._n_since_last_reassign = 0
            self.n_features_in_ = X.d
            st = self._mb = _new_state(be, X, centers, self._counts)
        elif st is None:                        # unpickled: the float64 state, or the published attributes
            centers, weight_sums = self.__dict__.pop("_mb_host", (self.cluster_centers_, self._counts))
            st = self._mb = _new_state(be, X, centers, weight_sums)
        elif isinstance(st, _SparseMiniBatchState) != isinstance(X, _SparseData):
            # a sparse batch after a dense one, or the reverse: the same float64 state in the other layout
            st = self._mb = _new_state(be, X, st.C.cpu().numpy(), st.W.cpu().numpy())

        random_reassign = self._random_reassign()
        st.step(be, chunks, X.dtype)
        st.start_read()
        return random_reassign

    def _step_end(self, X, chunks, off, random_reassign, compute_labels):
        """Second half: the one host read of the step, scikit-learn's reassignment, and the labels and inertia of the
        batch against the new centres."""
        be, st = X.backend, self._mb
        n = self._batch_rows(X, chunks)
        sparse = isinstance(st, _SparseMiniBatchState)
        if sparse:
            w, batch_inertia, bad = st.finish_read()
            if bad != 0.0:
                st.undo()
                raise ValueError("Sparse input must be canonical CSR: the column indices of a block of the batch are "
                                 "not strictly increasing within each row, or not in [0, %d)" % X.d)
        else:
            w, batch_inertia = st.finish_read()
        _km._check_engine(be, batch_inertia, "the batch inertia")

        # scikit-learn's _mini_batch_step after _minibatch_update_dense, on the weight sums in X's dtype
        if random_reassign and self.reassignment_ratio > 0:
            weight_sums = w.astype(X.np_dtype)
            to_reassign = weight_sums < self.reassignment_ratio * weight_sums.max()
            if to_reassign.sum() > 0.5 * n:
                indices_dont_reassign = np.argsort(weight_sums)[int(0.5 * n):]
                to_reassign[indices_dont_reassign] = False
            n_reassigns = to_reassign.sum()
            if n_reassigns:
                new_centers = self._random_state.choice(n, replace=False, size=n_reassigns)
                if self.verbose:
                    print(f"[MiniBatchKMeans] Reassigning {n_reassigns} cluster centers.")
                # streamed data: the rows come from the host copy of the batch, which stays valid
                rows = torch.from_numpy(self._dense_rows(X, off + new_centers)).to(device=st.C.device,
                                                                                    dtype=torch.float64)
                where = torch.as_tensor(np.where(to_reassign)[0], device=st.C.device)
                if sparse:
                    C = st.C.contiguous()
                    C[where] = rows
                    st.set_centres(be, C)
                else:
                    st.C[where] = rows
                    st.pack = be.pack_centers(st.C, st.dtype, out=st.pack)
            w[to_reassign] = np.min(w[~to_reassign])
            st.W.copy_(torch.from_numpy(w))
        self._counts = w.astype(X.np_dtype)

        if compute_labels:
            acc = be.zeros((1,), torch.float64)
            labels = []
            for x in chunks:
                lab = be.empty((_rows(x),), torch.int32)
                if sparse:
                    be.csr_assign_chunk(x, st.d, st.packs[st.cur], st.k, labels=lab, dist_sum=acc)
                else:
                    be.assign_chunk(x, st.pack, st.k, lab, None, True, acc)
                labels.append(lab)
            self.labels_ = ChunkedArray(labels)
            self.inertia_ = float(acc.item())
            _km._check_engine(be, self.inertia_, "the inertia")
        self.n_steps_ += 1
        self._n_features_out = st.k

    def _publish(self, X):
        self.cluster_centers_ = self._mb.C.cpu().numpy().astype(X.np_dtype)
