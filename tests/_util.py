"""Helpers shared by the parity tests."""
import ctypes

import numpy as np

TC_ARGMIN, TC_XFORM, TC_COLSUM, TC_EMBED = 0, 1, 2, 3      # the epilogues of the fp32 tensor-core kernel (bkm_tc.cu)


def tc_layout(lib, d, k, epi, mstep=0, kw=0):
    """(KS, N, S, shared-memory bytes) of the fp32 tensor-core kernel variant that runs a (d, k) call of epilogue
    ``epi``: S slots of its X ring, each refilled once the tile it holds is done."""
    out = (ctypes.c_int * 4)()
    rc = lib.bkm_debug_tc_layout(int(d), int(k), int(epi), int(mstep), int(kw), out)
    assert rc == 0, rc
    return tuple(out)


def sm_count(lib, device=0):
    """The device's SM count: the tensor-core kernel's grid (one CTA per SM, tiles dealt round-robin)."""
    v = ctypes.c_int(0)
    assert lib.bkm_device_info(int(device), ctypes.byref(v), None, None) == 0
    return int(v.value)


def d2_f64(X, C):
    X = np.asarray(X, dtype=np.float64)
    C = np.asarray(C, dtype=np.float64)
    return ((X[:, None, :] - C[None, :, :]) ** 2).sum(-1) if X.shape[0] * C.shape[0] * X.shape[1] < 5e7 else \
        np.maximum((X * X).sum(1)[:, None] - 2 * X @ C.T + (C * C).sum(1)[None, :], 0)


def grid_blobs(n, d, k_true, seed, step, bound, spread=0.6, std=0.05, return_blob=False):
    """float64 blob rows on the grid ``step`` with |x| < ``bound``.  On a grid of 2^-12 below 2^5 (float32) or 2^-4
    below 2^4 (bfloat16) every row, and every power-of-two multiple of it that stays a normal float, is exact in that
    type, so results on 2^p X can be compared with results on X exactly.  ``return_blob``: also the blob of each row."""
    rng = np.random.RandomState(seed)
    cent = rng.uniform(-spread * bound, spread * bound, size=(k_true, d))
    blob = rng.randint(0, k_true, size=n)
    X = cent[blob] + rng.standard_normal((n, d)) * (std * bound)
    X = np.clip(np.round(X / step) * step, step - bound, bound - step)
    return (X, blob) if return_blob else X


def blob_seeds(X, blob, k):
    """One row of each of the first k blobs: initial centres from which Lloyd settles in a few iterations and stops on
    a zero shift."""
    return np.stack([X[np.nonzero(blob == j)[0][0]] for j in range(k)])


def distinct_rows(X, k, seed):
    """k distinct rows of X (centres that scale exactly with X)."""
    U = np.unique(X, axis=0)
    return U[np.random.RandomState(seed).choice(len(U), k, replace=False)]


def assert_labels_match(got, want, X, C, rtol=1e-9, max_frac=1e-3):
    """Labels must be identical except on float64 near-ties: rows where the two chosen centres are
    equidistant to `rtol` relative to (||x||^2+||c||^2).  This is the documented tie-breaking."""
    got = np.asarray(got).astype(np.int64)
    want = np.asarray(want).astype(np.int64)
    assert got.shape == want.shape
    bad = np.nonzero(got != want)[0]
    if len(bad) == 0:
        return 0
    Xb = np.asarray(X, dtype=np.float64)[bad]
    C = np.asarray(C, dtype=np.float64)
    dg = ((Xb - C[got[bad]]) ** 2).sum(1)
    dw = ((Xb - C[want[bad]]) ** 2).sum(1)
    scale = (Xb ** 2).sum(1) + (C ** 2).sum(1).max()
    rel = np.abs(dg - dw) / scale
    assert rel.max() <= rtol, "label mismatch that is not a float64 near-tie: rel margin %g at row %d" % (
        rel.max(), bad[rel.argmax()])
    assert len(bad) <= max(1, max_frac * len(got)), "%d near-tie mismatches of %d rows" % (len(bad), len(got))
    return len(bad)
