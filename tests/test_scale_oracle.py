"""Power-of-two equivariance of the reference's Lloyd loop (CPU, through the oracle's scikit-learn path).

The reference's E-step runs in float64, so on X' = 2^p X with initial centres 2^p C and tol' = 4^p tol it gives the
same labels and n_iter, centres multiplied by exactly 2^p and an inertia multiplied by 4^p.  tests/test_gpu_scale.py
demands the same of the CUDA engine; this pins that it is the reference's behaviour.

The inertia branch of the reference (Q4: re-label with the non-squared metric when the final shift exceeds an
ABSOLUTE 1e-7) is not scale-invariant, so the data is chosen for a loop that ends on a zero shift (the labels stop
changing), where every p takes the squared branch.
"""
import numpy as np
import pytest

from _util import blob_seeds, grid_blobs

P_FIT = [-100, -64, 0, 64, 96]


@pytest.fixture(scope="module")
def data():
    X, blob = grid_blobs(3000, 13, 20, 7, 2.0 ** -12, 2.0 ** 5, std=0.02, return_blob=True)
    return X.astype(np.float32), blob_seeds(X, blob, 20)


def _fit(oracle, X, C, p):
    blocks = oracle.to_blocks(np.ldexp(X, p), 1000)
    lab, inertia, cen, n_iter = oracle.kmeans_single_lloyd(blocks, C.shape[0], init=np.ldexp(C, p).astype(np.float64),
                                                           tol=1e-4 * 4.0 ** p, max_iter=30)
    return np.concatenate(lab), inertia, cen, n_iter


def test_scale_data_is_exact(data):
    X, C = data
    for p in (-112, 96):
        assert np.array_equal(np.ldexp(np.ldexp(X, p), -p), X)
        assert np.abs(np.ldexp(X, p)[X != 0]).min() >= np.finfo(np.float32).tiny


@pytest.mark.parametrize("p", P_FIT)
def test_reference_lloyd_is_power_of_two_equivariant(oracle, data, p):
    X, C = data
    lab0, in0, cen0, it0 = _fit(oracle, X, C, 0)
    assert it0 < 30, "the base fit must converge to a zero shift"
    lab, inertia, cen, n_iter = _fit(oracle, X, C, p)
    assert n_iter == it0
    np.testing.assert_array_equal(lab, lab0)
    assert cen.dtype == np.float32
    np.testing.assert_array_equal(cen, np.ldexp(cen0, p))
    assert np.isfinite(inertia)
    assert abs(inertia - 4.0 ** p * in0) <= 1e-12 * 4.0 ** p * in0
