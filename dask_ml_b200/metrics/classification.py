"""accuracy_score and log_loss with the dask_ml.metrics API (dask_ml/metrics/classification.py:11-150), reduced where the
arrays live: one ``bkm_metric_chunk`` pass per pair of device blocks, numpy for host blocks (metrics/_scoring.py)."""
import types

import numpy as np

from ..chunked import _is_torch
from ..naive_bayes import _local_unique, class_indices
from . import _scoring as sc


def accuracy_score(y_true, y_pred, normalize=True, sample_weight=None, compute=True):
    """Accuracy classification score; for 2-D label indicators the subset accuracy (a row counts when every label
    matches).  ``normalize=False`` returns the (weighted) number of matching rows.  The result is always concrete
    (``compute`` is accepted for the reference's signature)."""
    tuples = sc.aligned_blocks([y_true, y_pred, sample_weight], ["y_true", "y_pred", "sample_weight"])
    if len(tuples[0][0].shape) != len(tuples[0][1].shape) or tuples[0][0].shape[1:] != tuples[0][1].shape[1:]:
        raise ValueError("y_true and y_pred must have the same shape; got trailing shapes %r and %r"
                         % (tuple(tuples[0][0].shape[1:]), tuple(tuples[0][1].shape[1:])))
    m = int(tuples[0][0].shape[1]) if len(tuples[0][0].shape) == 2 else 1
    (hit, total), _ = sc.reduce_sums(sc.EQ, tuples, m)
    if normalize:
        with np.errstate(divide="ignore", invalid="ignore"):
            return float(np.float64(hit) / np.float64(total))
    return float(hit) if sample_weight is not None else int(round(hit))


def _classes_of(tuples, labels, comm):
    if labels is not None:
        classes = np.unique(np.asarray(labels))
    else:
        local = [_local_unique(t[0].reshape(-1) if _is_torch(t[0]) else np.asarray(t[0]).reshape(-1))
                 for t in tuples if int(t[0].shape[0])]
        parts = [p for ps in comm.allgather_obj(local) for p in ps if len(p)]
        classes = np.unique(np.concatenate(parts)) if parts else np.zeros(0)
    if len(classes) < 2:
        if labels is None:
            raise ValueError("y_true contains only one label ({}). Please provide the true labels explicitly through "
                             "the labels argument.".format(classes[0] if len(classes) else None))
        raise ValueError("The labels array needs to contain at least two labels for log_loss, got {}.".format(classes))
    return classes


def log_loss(y_true, y_pred, eps=1e-15, normalize=True, sample_weight=None, labels=None):
    """Log loss (cross-entropy).  ``y_pred`` holds (n, K) probabilities, columns in the sorted order of the labels, or
    (n,) probabilities of the larger of two labels.  Probabilities are clipped to [eps, 1 - eps] and each row is
    renormalised.  Unlike the reference, which averages per-block losses and infers the labels per block, this is the
    exact mean (``normalize=False``: sum) over all rows, with the labels taken from all of ``y_true`` (or ``labels``).
    A ``y_true`` value that is not a label makes the result NaN."""
    from ..engine import Comm

    comm = Comm()
    tuples = sc.aligned_blocks([y_true, y_pred, sample_weight], ["y_true", "y_pred", "sample_weight"])
    if len(tuples[0][0].shape) != 1:
        raise ValueError("y_true must be 1-D for log_loss")
    classes = _classes_of(tuples, labels, comm)
    K = len(classes)
    m = int(tuples[0][1].shape[1]) if len(tuples[0][1].shape) == 2 else 1
    if (m == 1 and K != 2) or (m > 1 and m != K):
        raise ValueError("y_true and y_pred contain different number of classes {}, {}. Classes found in y_true: {}"
                         .format(K, 2 if m == 1 else m, classes))
    coded = []
    for t, p, w in tuples:
        device = sc._device_of((t, p, w))
        if device is not None and int(t.shape[0]):
            from ..model_selection._split import _backend

            shim = types.SimpleNamespace(backend=_backend(device), chunk_offsets=[0, int(t.shape[0])])
            cls = class_indices(t, classes, shim)[0]
        else:
            h = sc._host(t)
            pos = np.clip(np.searchsorted(classes, h), 0, K - 1)
            cls = np.where(classes[pos] == h, pos, -1).astype(np.int32)
        coded.append((cls, p, w))
    (loss, total), _ = sc.reduce_sums(sc.LOGLOSS, coded, m, eps=float(eps), comm=comm)
    if normalize:
        with np.errstate(divide="ignore", invalid="ignore"):
            return float(np.float64(loss) / np.float64(total))
    return float(loss)
