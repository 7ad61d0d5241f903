"""The shared intake and reduction of the scoring metrics.

``y_true`` / ``y_pred`` (/ ``sample_weight``) come in every form ``GaussianNB.fit`` takes y.  When their row chunks agree
the blocks are reduced pairwise where they are; otherwise each is flattened to one block (``naive_bayes._y_flat``).  A
pair with a CUDA block is reduced on that device by ``bkm_metric_chunk`` (a host partner is uploaded); a pair of host
blocks is reduced by the numpy statement of the same sums below.  With ``torch.distributed`` initialised the sums of all
ranks are added in one all-reduce, so every rank returns the global score.
"""
import numpy as np

from .. import _lib
from ..chunked import ChunkedArray, _is_torch, as_chunked, block_to_numpy, is_dask_array
from ..naive_bayes import _y_flat

EQ, ERR, LOGLOSS = _lib.METRIC_EQ, _lib.METRIC_ERR, _lib.METRIC_LOGLOSS


def _block_list(a):
    if isinstance(a, ChunkedArray):
        return list(a.blocks)
    if is_dask_array(a):
        return list(as_chunked(a).blocks)
    if _is_torch(a):
        return [a.detach()]
    return [np.asarray(a)]


def _trailing(blocks, what):
    if blocks[0].ndim not in (1, 2):
        raise ValueError("%s must be 1-D or 2-D; got %d dimensions" % (what, blocks[0].ndim))
    return tuple(int(s) for s in blocks[0].shape[1:])


def aligned_blocks(arrays, names):
    """[(block of array 0, block of array 1, ...), ...] with equal rows per tuple; an array that is None stays None."""
    lists = [None if a is None else _block_list(a) for a in arrays]
    tails = [None if b is None else _trailing(b, nm) for b, nm in zip(lists, names)]
    rows = [None if b is None else tuple(int(x.shape[0]) for x in b) for b in lists]
    totals = [sum(r) for r in rows if r is not None]
    if len(set(totals)) > 1:
        raise ValueError("Found input variables with inconsistent numbers of samples: %r" % totals)
    if len({r for r in rows if r is not None}) > 1:                       # different chunking: one block each
        lists = [None if a is None else [_y_flat(a, nm).reshape((-1,) + tl)]
                 for a, nm, tl in zip(arrays, names, tails)]
    n_blocks = len(next(b for b in lists if b is not None))
    return [tuple(None if b is None else b[i] for b in lists) for i in range(n_blocks)]


def _device_of(blocks):
    for b in blocks:
        if _is_torch(b) and b.is_cuda:
            return b.device
    return None


def _to_device(b, device, dtype=None):
    import torch

    from ..engine import _METRIC_CODE

    t = b if _is_torch(b) else torch.as_tensor(np.ascontiguousarray(b))
    t = t.to(device)
    if dtype is not None:
        t = t.to(dtype)
    elif t.dtype not in _METRIC_CODE:
        t = t.to(torch.float64 if t.is_floating_point() else torch.int64)
    return t.contiguous()


def _host(b):
    return np.asarray(block_to_numpy(b) if _is_torch(b) else b)


def _as2d(x):
    return x.reshape(x.shape[0], -1)


def host_sums(mode, a, b, w=None, shift=None, eps=0.0):
    """The sums of ``bkm_metric_chunk`` for one pair of host blocks, in numpy float64."""
    if mode == EQ:
        a2, b2 = _as2d(a), _as2d(b)
        if a2.dtype.kind in "biu" and b2.dtype.kind in "biu":
            eq = (a2.astype(np.int64) == b2.astype(np.int64)).all(1)
        else:
            eq = (a2.astype(np.float64) == b2.astype(np.float64)).all(1)
        wt = np.ones(len(eq)) if w is None else w.astype(np.float64)
        return np.array([np.sum(wt * eq), np.sum(wt)])
    if mode == ERR:
        a2, b2 = _as2d(a).astype(np.float64), _as2d(b).astype(np.float64)
        dl, t = b2 - a2, a2 - shift
        return np.stack([(dl * dl).sum(0), np.abs(dl).sum(0), t.sum(0), (t * t).sum(0)])
    q = np.clip(_as2d(b).astype(np.float64), eps, 1.0 - eps)
    if q.shape[1] == 1:
        q = np.hstack([1.0 - q, q])
    cls = a.astype(np.int64)
    ok = (cls >= 0) & (cls < q.shape[1])
    pick = np.where(ok, q[np.arange(len(cls)), np.where(ok, cls, 0)], np.nan)
    wt = np.ones(len(cls)) if w is None else w.astype(np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.array([np.sum(-wt * np.log(pick / q.sum(1))), np.sum(wt)])


def first_row_shift(tuples, m, comm):
    """The first local row of y_true in float64, rank 0's on every rank: the origin of r2's sums of squares (the
    cancellation guard of the scalers' statistics pass)."""
    shift = np.zeros(m)
    for t in tuples:
        if int(t[0].shape[0]):
            shift = _host(t[0][:1]).astype(np.float64).reshape(m)
            break
    shift = np.where(np.isfinite(shift), shift, 0.0)
    return np.asarray(comm.bcast_obj(shift))


def reduce_sums(mode, tuples, m, shift=None, eps=0.0, comm=None):
    """Add the sums of every (a, b[, w]) tuple and all-reduce them.  Returns (sums, n): float64 numpy of shape (4, m)
    for ERR and (2,) otherwise, and the global number of rows."""
    import torch

    from ..engine import Comm

    comm = comm or Comm()
    shape = (4, m) if mode == ERR else (2,)
    host = np.zeros(shape)
    dev_acc = {}
    n = 0
    for tup in tuples:
        a, b = tup[0], tup[1]
        w = tup[2] if len(tup) > 2 else None
        rows = int(b.shape[0])
        n += rows
        if rows == 0:
            continue
        device = _device_of(tup)
        if device is None:
            host += host_sums(mode, _host(a), _host(b), None if w is None else _host(w), shift, eps)
            continue
        from ..model_selection._split import _backend

        be = _backend(device)
        acc = dev_acc.get(device)
        first = acc is None
        if first:
            acc = dev_acc[device] = torch.empty(shape, dtype=torch.float64, device=device)
            if shift is not None:
                dev_acc[device, "shift"] = torch.as_tensor(shift).to(device)
        be.metric_chunk(_to_device(a, device), _to_device(b, device), mode, acc,
                        w=None if w is None else _to_device(w, device, torch.float64),
                        shift=dev_acc.get((device, "shift")), eps=eps, first=first)
    devices = [k for k in dev_acc if not isinstance(k, tuple)]
    total = host + sum(dev_acc[d].cpu().numpy() for d in devices)
    red = torch.as_tensor(np.concatenate([total.reshape(-1), [float(n)]]))
    if comm.world > 1:
        if devices:                                   # a device process group (NCCL) reduces device tensors only
            red = red.to(devices[0])
        comm.allreduce_sum_(red)
    out = red.cpu().numpy()
    return out[:-1].reshape(shape), int(round(out[-1]))
