"""Family 1's arg-min epilogue on designed rows (run with -m gpu).

The fused kernel decides a row from its minimum m and the columns whose value lies within the near-tie bound of m:
exactly one such column is the label, more than one defers the row to the float64 re-check, which takes the lowest
index on exact ties.  The rows here tie exactly in fp32 between columns held by the same lane, by different lanes of
a quad and by the two column halves of N = 256, three ways, and between a centre pair's midpoint; the other rows are
far from every tie and must be labelled in the fused kernel, with every column index as a label.  Shapes with padded
columns (k < N, down to k = 1) check that a padded column never counts as a second candidate."""
import numpy as np
import pytest

import msum_ref as mr

pytestmark = pytest.mark.gpu

FORCE_TC = 2

# (d, k, duplicated centre groups, midpoint pairs): N = 256 (two column halves), N = 128 (C3's shape, 28 padded
# columns), N = 32 and N = 16 with padded columns.  Columns j and j' sit in the same lane iff j // 2 == j' // 2 (mod 4).
CASES = [
    (64, 256, [(0, 2), (4, 5), (9, 15), (127, 128), (3, 200), (20, 22, 150), (251, 253, 255)],
     [(32, 33), (32, 34), (64, 72), (1, 129), (96, 224)]),
    (41, 100, [(0, 6), (10, 11), (30, 32, 99)], [(16, 17), (16, 18), (64, 68)]),
    (16, 31, [(1, 3, 5)], [(8, 9), (8, 10)]),
    (3, 2, [], [(0, 1)]),
    (3, 1, [], []),
]


def _design(d, k, groups, pairs, seed):
    rng = np.random.RandomState(seed)
    C = mr.lattice_centres(k, d, spacing=10.0, offset=-10.0)
    for g in groups:
        C[list(g[1:])] = C[g[0]]
    # every column is the nearest centre of 40 rows (integer noise keeps the rows exact in fp32 and far from any tie)
    pattern = np.repeat(np.arange(k), 40)
    X = C[pattern] + rng.randint(-1, 2, size=(len(pattern), d))
    mids = [0.5 * (C[a] + C[b]) for a, b in pairs for _ in range(24)]
    if mids:
        X = np.concatenate([X, np.array(mids)])
    X = X[rng.permutation(len(X))]
    # float64 distances are exact here (multiples of 1/4 far below 2^53)
    d2 = ((X[:, None, :] - C[None, :, :]) ** 2).sum(-1)
    want = d2.argmin(1)                                     # lowest index on exact ties
    srt = np.sort(d2, axis=1)
    tied = srt[:, 1] == srt[:, 0] if k > 1 else np.zeros(len(X), dtype=bool)
    if k > 1:
        # the design: a row is an exact tie, or its best two are far apart (far beyond the near-tie bound)
        assert (tied | (srt[:, 1] - srt[:, 0] >= 10.0)).all()
    return X, C, want, int(tied.sum())


@pytest.fixture(scope="module")
def be():
    from dask_ml_b200.engine import CudaBackend

    return CudaBackend()


@pytest.mark.parametrize("d,k,groups,pairs", CASES, ids=["d%d-k%d" % c[:2] for c in CASES])
def test_family1_argmin_ties(be, d, k, groups, pairs):
    import torch

    X64, C, want, n_tied = _design(d, k, groups, pairs, d * 1000 + k)
    n = len(X64)
    assert n_tied == 40 * sum(len(g) for g in groups) + 24 * len(pairs) * (k > 1)
    be.flags = FORCE_TC
    try:
        assert be.kernel_family(d, k, torch.float32) == 1
        x = be.to_device(X64, torch.float32)
        pack = be.pack_centers(torch.as_tensor(C).to(be.device), torch.float32)
        lab = torch.as_tensor(want).to(be.device)
        want_sums = torch.zeros((k, d), dtype=torch.float64, device=be.device).index_add_(
            0, lab, torch.as_tensor(X64).to(be.device))
        for want_dist in (False, True):
            labels = be.empty((n,), torch.int32)
            sums, counts = be.zeros((k * d,), torch.float64), be.zeros((k,), torch.int64)
            be.lloyd_chunk(x, pack, k, labels, be.empty((n,), torch.float32) if want_dist else None, sums, counts,
                           be.zeros((1,), torch.float64) if want_dist else None)
            torch.cuda.synchronize()
            assert be.deferred_rows(n, d, k, torch.float32) == n_tied, "want_dist=%s" % want_dist
            np.testing.assert_array_equal(labels.cpu().numpy(), want)
            assert torch.equal(counts, torch.bincount(lab, minlength=k))
            assert torch.equal(sums.view(k, d), want_sums)          # half-integer rows: every order is exact
        labels = be.empty((n,), torch.int32)
        be.assign_chunk(x, pack, k, labels, None, True, None)
        torch.cuda.synchronize()
        assert be.deferred_rows(n, d, k, torch.float32) == n_tied, "assign"
        np.testing.assert_array_equal(labels.cpu().numpy(), want)
    finally:
        be.flags = 0
