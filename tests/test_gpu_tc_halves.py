"""The fp32 tensor-core kernel's arg-min decided one column half at a time at N = 256 (run with -m gpu).

For N = 256 the kernel finds the minimum of columns 0..127, counts that half's columns within the near-tie bound of
it, then does the same for columns 128..255 in the same registers, and keeps the first half's count only where the
overall minimum does not move it out of the bound.  Rows here put their best and second-best columns on either side
of the halves' border (and inside one half) in every order:

* cross-above: the best column j + 128 in the second half, column j within the bound of it;
* cross-below: the best column j in the first half, column j + 128 within the bound;
* cross-equal: columns j and j + 128 at exactly equal distances (the float64 re-check takes j);
* inner-first / inner-second: a near-tie between columns j, j + 1 of one half, the other half far;
* far rows labelled in either half, so that the second half's minimum often drops the first half's count.

The centres are 0/1 vectors (the bits of the column index in features 0..7) and the near-tie rows are dyadic, so
every distance the split-fp16 product forms for them is exact and the near-tie rows are deferred for certain; the far
rows are at least 0.5 from every other centre.  Labels must equal the float64 arg-min, the deferred count must be the
number of near-tie rows, and the sums must equal the order-exact reference bit for bit: the deferred rows go to
clusters of their own, whose float64 sums are exact in any order.  Row counts sit at the wrap points of the M-step
variants' 5-slot ring."""
import numpy as np
import pytest

import msum_ref as mr
from _util import TC_ARGMIN, sm_count, tc_layout

pytestmark = pytest.mark.gpu

FORCE_TC = 2
DELTA = 2.0 ** -18                     # offset of a near-tie row from the midpoint: distance gap 2 DELTA = 2^-17
TAU_TC = lambda d: (8.0 * np.sqrt(3.0 * ((d + 7) // 8)) + 16.0) * 2.0 ** -24      # bkm_api.cu tau_for, family 1
KINDS = ("cross-above", "cross-below", "cross-equal", "inner-first", "inner-second")

SHAPES = [(64, 256), (64, 200), (20, 129)]
ROWS = {
    "64GS-37": lambda G, S: 64 * G * S - 37,                # the ring never wraps
    "64GS+64": lambda G, S: 64 * G * S + 64,                # only CTA 0 refills
    "64G(S+1)+1": lambda G, S: 64 * G * (S + 1) + 1,        # every CTA refills once
    "64G2S+1": lambda G, S: 64 * G * 2 * S + 1,             # CTA 0 reaches the second phase flip of slot 0
    "64G(3S+2)+29": lambda G, S: 64 * G * (3 * S + 2) + 29,
}


@pytest.fixture(scope="module")
def be():
    from dask_ml_b200.engine import CudaBackend

    return CudaBackend()


def _centres(k, d):
    C = np.zeros((k, d))
    for b in range(8):
        C[:, b] = (np.arange(k) >> b) & 1
    return C


def _design(n, d, k, seed):
    """(X32 as float64, float64 labels, near-tie mask): a near-tie row about every 37 rows."""
    rng = np.random.RandomState(seed)
    C = _centres(k, d)
    # the near-tie rows' pairs (j, j + 128 across the halves; j, j + 1 inside a half, j even) and their labels
    cross = [j for j in (0, 3, 42, 77, 127) if j + 128 < k]
    inner1 = [j for j in (8, 100) if j + 1 < 128]
    inner2 = [j for j in (130, 198, 250) if j + 1 < k]
    tie_cols = set(cross) | {j + 128 for j in cross} | set(inner1) | {j + 1 for j in inner1} | set(inner2) | \
        {j + 1 for j in inner2}
    free = np.array([j for j in range(k) if j not in tie_cols])
    # far rows: their centre plus noise of at most 0.25 per feature that fills the low bits of the fp32 sums
    lab = free[rng.randint(0, len(free), n)]
    X = C[lab] + 0.25 * 2.0 ** -rng.uniform(0, 12, size=(n, 1)) * rng.uniform(-1, 1, size=(n, d))
    tie = np.zeros(n, dtype=bool)
    rows = np.arange(rng.randint(0, 37), n, 37)
    kinds = [kd for kd in KINDS if kd != "inner-second" or inner2]        # k = 129: no pair inside the second half
    for i, r in enumerate(rows):
        kind = kinds[i % len(kinds)]
        if kind.startswith("cross"):
            j = cross[(i // len(kinds)) % len(cross)]
            x, f = C[j].copy(), 7                                       # columns j, j + 128 differ in feature 7 only
            x[f] = 0.5 + {"cross-above": DELTA, "cross-below": -DELTA, "cross-equal": 0.0}[kind]
        else:
            js = inner1 if kind == "inner-first" else inner2
            j = js[(i // len(kinds)) % len(js)]
            x, f = C[j].copy(), 0                                       # columns j, j + 1 differ in feature 0 only
            x[f] = 0.5 - DELTA if (i // len(kinds)) % 2 else 0.5 + DELTA
        X[r] = x
        tie[r] = True
    X32 = X.astype(np.float32).astype(np.float64)
    # d^2 - ||x||^2 = ||c||^2 - 2 x.c, exact in float64 here (x.c adds at most 8 fp32 values below 1.25)
    e = (C * C).sum(1)[None, :] - 2.0 * (X32 @ C.T)
    want = e.argmin(1)                                                  # lowest index on exact ties
    two = np.partition(e, 1, axis=1)[:, :2]
    gap = two[:, 1] - two[:, 0]
    bound = TAU_TC(d) * ((X32 * X32).sum(1) + (C * C).sum(1).max())
    # the design: near-tie rows well inside the bound, every other row far outside it
    assert (gap[tie] <= 0.5 * bound[tie]).all() and (gap[~tie] >= 0.25).all()
    assert np.array_equal(want[~tie], lab[~tie]) and not np.isin(want[~tie], list(tie_cols)).any()
    return X32, C, want, tie


@pytest.mark.parametrize("rows", list(ROWS))
@pytest.mark.parametrize("d,k", SHAPES, ids=["d%d-k%d" % s for s in SHAPES])
def test_halves_argmin_and_sums(be, d, k, rows):
    import torch

    G = sm_count(be.lib, be.device.index or 0)
    ks, N, S, _ = tc_layout(be.lib, d, k, TC_ARGMIN, mstep=1)
    assert N == 256 and S == 5
    n = ROWS[rows](G, S)
    X32, C, want, tie = _design(n, d, k, n + 31 * k + d)
    n_tie = int(tie.sum())
    # fused rows in the order-exact per-CTA partials; the deferred rows' float64 sums are exact in any order and land
    # in clusters no fused row has
    want_sums = mr.reduce_partials(mr.tc_partials(X32.astype(np.float32), want, k, G, keep=~tie))
    np.add.at(want_sums, want[tie], X32[tie])
    want_cnt = np.bincount(want, minlength=k)
    be.flags = FORCE_TC
    try:
        assert be.kernel_family(d, k, torch.float32) == 1
        x = be.to_device(X32.astype(np.float32), torch.float32)
        pack = be.pack_centers(torch.as_tensor(C).to(be.device), torch.float32)
        for want_dist in (False, True):
            labels = be.empty((n,), torch.int32)
            sums, counts = be.zeros((k * d,), torch.float64), be.zeros((k,), torch.int64)
            be.lloyd_chunk(x, pack, k, labels, be.empty((n,), torch.float32) if want_dist else None, sums, counts,
                           be.zeros((1,), torch.float64) if want_dist else None)
            torch.cuda.synchronize()
            assert be.deferred_rows(n, d, k, torch.float32) == n_tie, "want_dist=%s" % want_dist
            np.testing.assert_array_equal(labels.cpu().numpy(), want)
            np.testing.assert_array_equal(counts.cpu().numpy(), want_cnt)
            got = sums.cpu().numpy().reshape(k, d)
            bad = got.view(np.uint64) != want_sums.view(np.uint64)
            assert not bad.any(), "want_dist=%s: %d sums differ from the order-exact reference, first at %s" % (
                want_dist, int(bad.sum()), np.argwhere(bad)[0].tolist())
        labels = be.empty((n,), torch.int32)
        be.assign_chunk(x, pack, k, labels, None, True, None)
        torch.cuda.synchronize()
        assert be.deferred_rows(n, d, k, torch.float32) == n_tie, "assign"
        np.testing.assert_array_equal(labels.cpu().numpy(), want)
    finally:
        be.flags = 0
