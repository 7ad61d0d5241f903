"""mean_squared_error, mean_absolute_error and r2_score with the dask_ml.metrics API (dask_ml/metrics/regression.py:8-92):
one ``bkm_metric_chunk`` pass per pair of device blocks gives every sum the three scores need, r2's denominator
included (its sums of squares are taken about the first row of ``y_true``, so no second pass and no cancellation)."""
import numpy as np

from . import _scoring as sc


def _check_sample_weight(sample_weight):
    if sample_weight is not None:
        raise ValueError("'sample_weight' is not supported.")


def _err_sums(y_true, y_pred):
    from ..engine import Comm

    comm = Comm()
    tuples = sc.aligned_blocks([y_true, y_pred], ["y_true", "y_pred"])
    t0, p0 = tuples[0][0], tuples[0][1]
    m = int(t0.shape[1]) if len(t0.shape) == 2 else 1
    if (int(p0.shape[1]) if len(p0.shape) == 2 else 1) != m:
        raise ValueError("y_true and y_pred have different number of output ({}!={})"
                         .format(m, int(p0.shape[1]) if len(p0.shape) == 2 else 1))
    shift = sc.first_row_shift(tuples, m, comm)
    sums, n = sc.reduce_sums(sc.ERR, tuples, m, shift=shift, comm=comm)
    return sums, n


def _mean_error(y_true, y_pred, sample_weight, multioutput, row):
    _check_sample_weight(sample_weight)
    sums, n = _err_sums(y_true, y_pred)
    with np.errstate(divide="ignore", invalid="ignore"):
        output_errors = sums[row] / np.float64(n)
    if isinstance(multioutput, str):
        if multioutput == "raw_values":
            return output_errors
    else:
        raise ValueError("Weighted 'multioutput' not supported.")
    return float(output_errors.mean())


def mean_squared_error(y_true, y_pred, sample_weight=None, multioutput="uniform_average", compute=True):
    """Mean squared error; ``multioutput="raw_values"`` returns the error of every output as a numpy array."""
    return _mean_error(y_true, y_pred, sample_weight, multioutput, 0)


def mean_absolute_error(y_true, y_pred, sample_weight=None, multioutput="uniform_average", compute=True):
    """Mean absolute error; ``multioutput="raw_values"`` returns the error of every output as a numpy array."""
    return _mean_error(y_true, y_pred, sample_weight, multioutput, 1)


def r2_score(y_true, y_pred, sample_weight=None, multioutput="uniform_average", compute=True):
    """R^2, the mean over the outputs.  An output whose numerator and denominator are both zero scores 1, one whose
    denominator alone is zero scores 0 (the reference's rule)."""
    _check_sample_weight(sample_weight)
    if multioutput != "uniform_average":
        raise NotImplementedError("'multioutput' must be 'uniform_average'")
    sums, n = _err_sums(y_true, y_pred)
    numerator = sums[0]
    with np.errstate(all="ignore"):
        denominator = sums[3] - sums[2] * sums[2] / np.float64(n)
        nonzero_denominator = denominator != 0
        nonzero_numerator = numerator != 0
        valid = nonzero_denominator & nonzero_numerator
        scores = np.ones(len(numerator))
        scores[valid] = 1 - numerator[valid] / denominator[valid]
        scores[nonzero_numerator & ~nonzero_denominator] = 0.0
    return float(scores.mean())
