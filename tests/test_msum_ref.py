"""CPU self-tests of the order-exact M-step references (tests/msum_ref.py): they restate the kernels' orders correctly,
and the order-sensitive data of the bit-exact GPU tests (test_gpu_msum.py) changes its sums when the order changes."""
import numpy as np
import pytest

import msum_ref as mr


def _naive_tc_partials(X32, labels, keep, k, grid):
    P = np.zeros((grid, k, X32.shape[1]), dtype=np.float32)
    n = X32.shape[0]
    ntiles = -(-n // 64)
    for b in range(grid):
        for tile in range(b, ntiles, grid):
            for r in range(tile * 64, min(n, tile * 64 + 64)):
                if keep[r]:
                    for f in range(X32.shape[1]):
                        P[b, labels[r], f] = np.float32(P[b, labels[r], f] + X32[r, f])
    return P


def _naive_reduce(P, first, old):
    flat = P.reshape(P.shape[0], -1)
    out = np.empty(flat.shape[1])
    for i in range(flat.shape[1]):
        s = [0.0] * 8
        for g in range(flat.shape[0]):
            s[g % 8] = s[g % 8] + float(flat[g, i])
        t = s[0]
        for y in range(1, 8):
            t = t + s[y]
        out[i] = t if first else old.reshape(-1)[i] + t
    return out.reshape(P.shape[1:])


def _bits_equal(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))


@pytest.mark.parametrize("n,k,d,sm", [(1, 3, 2, 4), (300, 5, 3, 4), (1000, 7, 5, 3), (64 * 9 + 5, 4, 2, 9)])
def test_family1_partials_and_fold_match_naive(n, k, d, sm):
    rng = np.random.RandomState(n + k)
    X32 = (100.0 + rng.standard_normal((n, d)) * 2.0 ** -rng.uniform(0, 12, (n, 1))).astype(np.float32)
    labels = rng.randint(0, k, n)
    keep = rng.uniform(size=n) > 0.1
    grid = mr.tc_grid(n, sm)
    P = mr.tc_partials(X32, labels, k, sm, keep=keep)
    assert _bits_equal(P, _naive_tc_partials(X32, labels, keep, k, grid))
    old = rng.standard_normal((k, d))
    for first in (True, False):
        assert _bits_equal(mr.reduce_partials(P, first, old), _naive_reduce(P, first, old))


@pytest.mark.parametrize("n,k,d,sm", [(1, 40, 16, 132), (4097, 300, 64, 132), (3 * 4096 + 1, 1024, 128, 5),
                                      (20 * 4096, 257, 128, 7)])
def test_family3_partials_match_naive(n, k, d, sm):
    rng = np.random.RandomState(k)
    X32 = rng.standard_normal((n, d)).astype(np.float32)
    labels = rng.randint(0, k, n)
    rb, tpb = mr.rowpass_blocks(n, k, d, sm)
    assert rb <= max(1, sm // mr.tc2_slices(k, d)) and (rb - 1) * tpb < -(-n // mr.RP_TILE) <= rb * tpb
    P = mr.rowpass_partials(X32, labels, k, sm)
    want = np.zeros_like(P)
    for r in range(n):                                  # row blocks are runs of whole tiles, rows in order
        b = r // mr.RP_TILE // tpb
        want[b, labels[r]] = want[b, labels[r]] + X32[r]
    assert _bits_equal(P, want)


def test_slices_and_blocks():
    # DS: the (k / DS) x d_padded fp32 sums of one slice (+ 40 KB) fit 210 KB
    assert [mr.tc2_slices(k, 128) for k in (40, 257, 300, 512, 1024, 4096)] == [1, 1, 1, 2, 4, 16]
    assert mr.tc2_slices(300, 64) == 1 and mr.tc2_slices(512, 96) == 2
    assert mr.rowpass_blocks(1, 1024, 128, 132) == (1, 1)
    assert mr.rowpass_blocks(300_000, 1024, 128, 132) == (25, 3)       # 74 tiles, 33 row-block slots
    assert mr.rowpass_blocks(4096 * 200, 40, 16, 132) == (100, 2)


def test_centres_are_separated():
    for k, d in [(16, 3), (255, 48), (1024, 128), (2, 3), (31, 16)]:
        C = mr.lattice_centres(k, d)
        D = ((C[:, None, :] - C[None, :, :]) ** 2).sum(-1) + np.eye(k) * 1e9
        assert D.min() >= 32.0 ** 2
        assert (C[:, mr.zero_features(d)] == 0).all()


def _final(X32, labels, k, sm, **kw):
    fold = kw.pop("fold", tuple(range(8)))
    return mr.reduce_partials(mr.tc_partials(X32, labels, k, sm, **kw), fold=fold)


def test_order_changes_are_visible():
    """Each of these changes of order changes at least 1 % of the sums of the designed data, so a bit-exact test
    against the reference sees a kernel that adds in another order."""
    sm, k, d = 132, 64, 20
    n = 64 * sm * 4 + 77
    rng = np.random.RandomState(0)
    pattern = np.where(rng.uniform(size=n) < 0.5, 0, rng.randint(0, k, n))        # one dominant cluster
    X32 = mr.designed_rows(pattern, mr.lattice_centres(k, d), 1).astype(np.float32)
    ref = _final(X32, pattern, k, sm)
    grid = mr.tc_grid(n, sm)
    rows = np.arange(n)
    lt, pos = rows // 64 // grid, rows % 64
    variants = {
        "odd tile before even tile": dict(rank_key=(lt ^ 1) * 64 + pos),
        "grid - 1": dict(grid=grid - 1),
        "grid + 1": dict(grid=grid + 1),
        "rows reversed in each tile": dict(rank_key=lt * 64 + 63 - pos),
        "chains folded 7 -> 0": dict(fold=tuple(range(7, -1, -1))),
    }
    for name, kw in variants.items():
        frac = float(np.mean(_final(X32, pattern, k, sm, **kw) != ref))
        assert frac >= 0.01, (name, frac)
