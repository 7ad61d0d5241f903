"""The fused fp32 M-step's four class lists, exactly (run with -m gpu).

Family 1 (tc_chunk_kernel, bkm_tc.cu) gives warp q of each warpgroup the clusters c with c % 4 == q and every thread a
feature pair.  On designed data whose labels are known in advance and whose sums change with the order of the
additions, the library's sums must equal the order-exact reference (tests/msum_ref.py) bit for bit: tiles whose 64 rows
all fall in one class (one label, or several labels of the class), class lists of every length around the batches of
8, and k of 4, 5, 100 and 256 with an odd d whose last feature pair straddles d."""
import numpy as np
import pytest

import msum_ref as mr

pytestmark = pytest.mark.gpu

FORCE_TC = 2


@pytest.fixture(scope="module")
def be():
    from dask_ml_b200.engine import CudaBackend

    return CudaBackend()


def _sm(be):
    import torch

    return torch.cuda.get_device_properties(be.device).multi_processor_count


def _tile_labels(t, k, rng):
    """Labels of the 64 rows of tile t: a tile of one class, one label of one class, class lists of 1 .. 63 rows, or
    uniform labels, in turn; the class q = t % 4 (mod k when k < 4) moves from tile to tile."""
    q = t % min(4, k)
    mine = np.arange(q, k, 4)
    rest = np.setdiff1d(np.arange(k), mine)
    kind = (t // 4) % 4
    if kind == 0:                                       # all 64 rows in class q, labels drawn from it
        return rng.choice(mine, 64)
    if kind == 1:                                       # one label: every batch of 8 repeats it
        return np.full(64, mine[(t // 16) % len(mine)])
    if kind == 2 and len(rest):                         # class q list of 1, 7, 8, 9, 15, 16, 17 or 63 rows
        sel = np.zeros(64, dtype=bool)
        sel[rng.permutation(64)[:(1, 7, 8, 9, 15, 16, 17, 63)[(t // 16) % 8]]] = True
        return np.where(sel, rng.choice(mine, 64), rng.choice(rest, 64))
    return rng.randint(0, k, 64)


def _pattern(n, k, seed):
    rng = np.random.RandomState(seed)
    return np.concatenate([_tile_labels(t, k, rng) for t in range(-(-n // 64))])[:n].astype(np.int64)


SHAPES = [(d, k) for k in (4, 5, 100, 256) for d in (2, 41, 63, 64)]
# n = a * sm_count + b: one row, fewer tiles than CTAs, tile pairs with a short last tile, a chunk of ~300k rows
ROWS = [(0, 1), (0, 261), (128, 77), (0, 300_007)]


@pytest.mark.parametrize("a,b", ROWS, ids=["%dsm%+d" % r if r[0] else str(r[1]) for r in ROWS])
@pytest.mark.parametrize("d,k", SHAPES)
def test_class_lists_sums_bit_exact(be, d, k, a, b):
    import torch

    sm = _sm(be)
    n = a * sm + b
    be.flags = FORCE_TC if k * d < 512 else 0
    try:
        assert be.kernel_family(d, k, torch.float32) == 1
        pattern = _pattern(n, k, n + 7 * k + d)
        C = mr.lattice_centres(k, d)
        X32 = mr.designed_rows(pattern, C, n + d).astype(np.float32)
        x = be.to_device(X32, torch.float32)
        pack = be.pack_centers(torch.as_tensor(C).to(be.device), torch.float32)
        want = np.ascontiguousarray(mr.reduce_partials(mr.tc_partials(X32, pattern, k, sm)), dtype=np.float64)
        for want_dist in (True, False):
            labels = be.empty((n,), torch.int32)
            sums, counts = be.zeros((k * d,), torch.float64), be.zeros((k,), torch.int64)
            be.lloyd_chunk(x, pack, k, labels, be.empty((n,), torch.float32) if want_dist else None, sums, counts,
                           be.zeros((1,), torch.float64) if want_dist else None)
            torch.cuda.synchronize()
            assert be.deferred_rows(n, d, k, torch.float32) == 0
            np.testing.assert_array_equal(labels.cpu().numpy(), pattern)
            got = np.ascontiguousarray(sums.cpu().numpy(), dtype=np.float64)
            bad = got.view(np.uint64) != want.reshape(got.shape).view(np.uint64)
            assert not bad.any(), "want_dist=%s: %d of %d sums differ, first at %s" % (
                want_dist, int(bad.sum()), bad.size, np.argwhere(bad)[0].tolist())
            np.testing.assert_array_equal(counts.cpu().numpy(), np.bincount(pattern, minlength=k))
    finally:
        be.flags = 0
