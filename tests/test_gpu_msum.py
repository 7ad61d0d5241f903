"""The M-step sums of every kernel family, exactly (run with -m gpu).

* Bit-exact: families 1 and 3 promise sums formed in a fixed order (tests/msum_ref.py restates it).  On designed data
  whose labels are known in advance and whose sums change with the order of the additions, the library's float64 sums
  must equal the reference bit for bit: for every class-list shape of the fused M-step (one parity list of 64 rows and
  the other empty, a label repeated in every batch of 8, runs, repeats at list distance 7 and 8, the padding rows of
  k == N, ...), every grid tail, both Lloyd variants, two launches, float64 counts and a two-chunk accumulation.
* Exact arithmetic: small-integer rows keep every partial sum below 2^24, so any order gives the exact answer; the
  sums must equal the float64 sums of the same labels exactly.  This sees any lost, repeated or misrouted row in the
  families whose order is not observable (0 and 2) and in the float64 re-check of deferred rows."""
import numpy as np
import pytest

import msum_ref as mr

pytestmark = pytest.mark.gpu

FORCE_SIMT, FORCE_TC = 1, 2


@pytest.fixture(scope="module")
def be():
    from dask_ml_b200.engine import CudaBackend

    return CudaBackend()


def _sm(be):
    """The SM count the library sizes its grids with (cudaDevAttrMultiProcessorCount)."""
    import torch

    return torch.cuda.get_device_properties(be.device).multi_processor_count


def _assert_bits_equal(got, want, what):
    got = np.ascontiguousarray(got, dtype=np.float64)
    want = np.ascontiguousarray(want, dtype=np.float64).reshape(got.shape)
    bad = got.view(np.uint64) != want.view(np.uint64)
    if bad.any():
        diff = np.abs(got - want)[bad]
        raise AssertionError("%s: %d of %d sums differ from the order-exact reference (max |diff| %g, first at %s)"
                             % (what, int(bad.sum()), bad.size, float(diff.max()), np.argwhere(bad)[0].tolist()))


# ------------------------------------------------------------------------------------------------ family 1
def _tile_labels(kind, k, t, rng):
    """Labels of the 64 rows of tile t for one class-list shape (k >= 2)."""
    ev, od = np.arange(0, k, 2), np.arange(1, k, 2)
    i = np.arange(64)
    if kind == "one even label":                        # one parity list of 64 entries, the other empty
        return np.full(64, ev[t % len(ev)])
    if kind == "one odd label":
        return np.full(64, od[t % len(od)])
    if kind == "alternating":                           # two labels of the same parity: every batch repeats
        return np.where(i % 2 == 0, ev[t % len(ev)], ev[(t + 1) % len(ev)])
    if kind == "distinct":                              # no batch repeats (k >= 64)
        return rng.permutation(k)[:64] if k >= 64 else i % k
    if kind == "runs":
        out = []
        while len(out) < 64:
            out += [rng.randint(k)] * (1, 2, 3, 7, 8, 9)[len(out) % 6]
        return np.array(out[:64])
    if kind == "repeat at distance 7 and 8":            # one even list: list position == row
        lab = ev[(i + t) % len(ev)]
        lab[7] = lab[0]                                 # same batch
        lab[15] = lab[8]
        lab[16] = lab[8]                                # next batch
        return lab
    if kind == "list lengths":                          # even list of 1, 7, 8, 9, 31, 32, 33 or 63 entries
        even = np.zeros(64, dtype=bool)
        even[rng.permutation(64)[:(1, 7, 8, 9, 31, 32, 33, 63)[t % 8]]] = True
        return np.where(even, rng.choice(ev, 64), rng.choice(od, 64))
    if kind == "top labels":                            # k - 1, k - 2: next to the spare rows N, N + 1 when k == N
        return np.where(rng.uniform(size=64) < 0.8, k - 1 - rng.randint(0, 2, 64), rng.randint(0, k, 64))
    assert kind == "dominant"
    return np.where(rng.uniform(size=64) < 0.9, k // 3, rng.randint(0, k, 64))


KINDS = ("one even label", "one odd label", "alternating", "distinct", "runs", "repeat at distance 7 and 8",
         "list lengths", "top labels", "dominant")


def _f1_pattern(n, k, seed):
    rng = np.random.RandomState(seed)
    tiles = [_tile_labels(KINDS[t % len(KINDS)], k, t, rng) for t in range(-(-n // 64))]
    return np.concatenate(tiles)[:n].astype(np.int64)


# (d, k): N = 16, 32, 64, 128, 256 and KS = 1..4, with k == N, odd k and k = 2
F1_SHAPES = [(3, 16), (24, 2), (16, 31), (20, 64), (41, 100), (33, 128), (48, 255), (64, 129), (64, 256)]
# n = a * sm_count + b: one row, fewer tiles than CTAs, a last tile of 1 or 63 rows, warpgroup 1 without a tile, odd and
# even numbers of tile pairs, and a chunk of ~300k rows
F1_ROWS = [(0, 1), (0, 63), (0, 65), (64, -1), (64, 1), (128, 5), (192, 77), (0, 300_007)]


@pytest.mark.parametrize("a,b", F1_ROWS, ids=["%dsm%+d" % r if r[0] else str(r[1]) for r in F1_ROWS])
@pytest.mark.parametrize("d,k", F1_SHAPES)
def test_family1_sums_bit_exact(be, d, k, a, b):
    import torch

    sm = _sm(be)
    n = a * sm + b
    be.flags = FORCE_TC if k * d < 512 else 0
    try:
        assert be.kernel_family(d, k, torch.float32) == 1
        pattern = _f1_pattern(n, k, n + 7 * k + d)
        C = mr.lattice_centres(k, d)
        X32 = mr.designed_rows(pattern, C, n + d).astype(np.float32)
        x = be.to_device(X32, torch.float32)
        pack = be.pack_centers(torch.as_tensor(C).to(be.device), torch.float32)
        want = mr.reduce_partials(mr.tc_partials(X32, pattern, k, sm))
        wcnt = np.bincount(pattern, minlength=k)

        def call(xc, rows, sums, counts, labels=None, mind2=None, inertia=None, first=False):
            be.lloyd_chunk(xc, pack, k, labels, mind2, sums, counts, inertia, first=first)
            torch.cuda.synchronize()
            assert be.deferred_rows(rows, d, k, torch.float32) == 0          # every row in the fused M-step

        for want_dist in (True, False):
            for launch in range(2):
                labels = be.empty((n,), torch.int32)
                sums, counts = be.zeros((k * d,), torch.float64), be.zeros((k,), torch.int64)
                call(x, n, sums, counts, labels, be.empty((n,), torch.float32) if want_dist else None,
                     be.zeros((1,), torch.float64) if want_dist else None)
                np.testing.assert_array_equal(labels.cpu().numpy(), pattern)
                _assert_bits_equal(sums.cpu().numpy(), want, "want_dist=%s launch %d" % (want_dist, launch))
                np.testing.assert_array_equal(counts.cpu().numpy(), wcnt)
        sums, counts = be.zeros((k * d,), torch.float64), be.zeros((k,), torch.float64)     # FLAG_COUNTS_F64
        call(x, n, sums, counts)
        _assert_bits_equal(sums.cpu().numpy(), want, "float64 counts")
        np.testing.assert_array_equal(counts.cpu().numpy(), wcnt.astype(np.float64))
        if n >= 2:
            # two chunks of one iteration: the first overwrites (NaN before), the second adds
            m = max(1, n // 3)
            sums = torch.full((k * d,), float("nan"), dtype=torch.float64, device=be.device)
            counts = torch.full((k,), -7, dtype=torch.int64, device=be.device)
            call(x[:m], m, sums, counts, first=True)
            w1 = mr.reduce_partials(mr.tc_partials(X32[:m], pattern[:m], k, sm))
            _assert_bits_equal(sums.cpu().numpy(), w1, "first chunk")
            np.testing.assert_array_equal(counts.cpu().numpy(), np.bincount(pattern[:m], minlength=k))
            call(x[m:], n - m, sums, counts)
            w2 = mr.reduce_partials(mr.tc_partials(X32[m:], pattern[m:], k, sm), first=False, old=w1)
            _assert_bits_equal(sums.cpu().numpy(), w2, "second chunk")
            np.testing.assert_array_equal(counts.cpu().numpy(), wcnt)
    finally:
        be.flags = 0


# ------------------------------------------------------------------------------------------------ family 3
F3_SHAPES = [(16, 40), (64, 300), (96, 512), (128, 257), (128, 1024)]     # FPL 1, 2, 4; DS = 1, 1, 2, 1, 4
F3_ROWS = [1, 4095, 4096, 4097, 200_003]                                   # 4097: fewer tiles than the RB cap


@pytest.mark.parametrize("n", F3_ROWS)
@pytest.mark.parametrize("d,k", F3_SHAPES)
def test_family3_sums_bit_exact(be, d, k, n):
    """The row pass adds each cluster's rows in row order whatever its balance table says: absent, present, stale."""
    import torch

    sm = _sm(be)
    assert be.kernel_family(d, k, torch.bfloat16) == 3
    rng = np.random.RandomState(n + k)
    pattern = np.where(rng.uniform(size=n) < 0.5, k // 3, rng.randint(0, k, n)).astype(np.int64)
    C = mr.lattice_centres(k, d)
    Xb = torch.as_tensor(mr.designed_rows(pattern, C, n + d)).to(be.device).to(torch.bfloat16)
    X32 = Xb.float().cpu().numpy()                       # bf16 -> fp32 is exact
    x = be.to_device(Xb, torch.bfloat16)
    pack = be.pack_centers(torch.as_tensor(C).to(be.device), torch.bfloat16)
    want = mr.reduce_partials(mr.rowpass_partials(X32, pattern, k, sm))
    wcnt = np.bincount(pattern, minlength=k)

    ws = be._workspace(n, d, k, torch.bfloat16)

    def check(state, table_k):
        # header of the balance table (WsLayout::off_bal = 0): {magic, k, cluster slices, 0}
        assert int(ws[:16].view(torch.int32)[1]) == table_k, state
        labels = be.empty((n,), torch.int32)
        sums, counts = be.zeros((k * d,), torch.float64), be.zeros((k,), torch.int64)
        be.lloyd_chunk(x, pack, k, labels, None, sums, counts, None)
        torch.cuda.synchronize()
        assert be._workspace(n, d, k, torch.bfloat16) is ws
        np.testing.assert_array_equal(labels.cpu().numpy(), pattern)
        _assert_bits_equal(sums.cpu().numpy(), want, "balance table " + state)
        np.testing.assert_array_equal(counts.cpu().numpy(), wcnt)

    ws[:8192].zero_()                                            # no table left by earlier calls
    check("absent", 0)
    check("present", k)
    k2 = k // 2 + 1                                              # a call with another k leaves its table behind
    pack2 = be.pack_centers(torch.as_tensor(mr.lattice_centres(k2, d)).to(be.device), torch.bfloat16)
    be.lloyd_chunk(x, pack2, k2, None, None, be.zeros((k2 * d,), torch.float64), be.zeros((k2,), torch.int64), None)
    torch.cuda.synchronize()
    check("stale", k2)


# ------------------------------------------------------------------------------------------------ exact arithmetic
# (id, dtype, d, k, flags, row pitch or None, n, expected family)
EXACT = [
    ("f0-fp32-smem", "float32", 64, 256, FORCE_SIMT, None, 300_000, 0),
    ("f0-fp32-smallk", "float32", 13, 20, FORCE_SIMT, None, 400_000, 0),
    ("f0-fp32-global-128x300", "float32", 128, 300, 0, None, 400_000, 0),
    ("f0-fp32-global-64x512", "float32", 64, 512, 0, None, 400_000, 0),
    ("f0-fp64-smem", "float64", 16, 8, 0, None, 400_000, 0),
    ("f0-fp64-global", "float64", 64, 256, 0, None, 300_000, 0),
    ("f0-fp32-wide", "float32", 784, 10, 0, None, 20_000, 0),
    ("f2-stream2-pitch13", "float32", 13, 20, 0, 13, 400_000, 2),
    ("f2-stream2-pitch16", "float32", 13, 20, 0, 16, 400_000, 2),
    ("f2-v1-k31", "float32", 16, 31, 0, 16, 400_000, 2),
    ("f2-v1-pitch40", "float32", 5, 8, 0, 40, 400_000, 2),
]


def _int_rows(pattern, C, seed):
    """Small-integer rows (|x| <= 21): every partial sum of up to ~800k rows stays below 2^24, so it is exact in fp32."""
    return C[pattern] + np.random.RandomState(seed).randint(-1, 2, size=(len(pattern), C.shape[1]))


def _check_exact(be, X64, labels, sums, counts, k, want_labels):
    import torch

    d = X64.shape[1]
    np.testing.assert_array_equal(labels.cpu().numpy(), want_labels)
    lab = labels.long()
    x64 = torch.as_tensor(X64).to(be.device)
    want = torch.zeros((k, d), dtype=torch.float64, device=be.device).index_add_(0, lab, x64)
    got = sums.view(k, d)
    assert torch.equal(got, want), "%d sums differ, max |diff| %g" % (int((got != want).sum()), float((got - want).abs().max()))
    assert torch.equal(counts, torch.bincount(lab, minlength=k))
    assert torch.equal(got.sum(0), x64.sum(0))            # no row lost or counted twice


@pytest.mark.parametrize("case", EXACT, ids=[c[0] for c in EXACT])
def test_exact_arithmetic_sums(be, case):
    import torch

    _, dtype_name, d, k, flags, pitch, n, family = case
    dt = getattr(torch, dtype_name)
    be.flags = flags
    try:
        assert be.kernel_family(d, k, dt) == family
        rng = np.random.RandomState(d * k)
        pattern = np.where(rng.uniform(size=n) < 0.9, k // 3, rng.randint(0, k, n))      # one dominant cluster
        C = mr.lattice_centres(k, d, spacing=10.0, offset=-10.0)
        X64 = _int_rows(pattern, C, n)
        if pitch is None:
            x = be.to_device(X64, dt)
        else:
            buf = torch.full((n, pitch), 7.5e4, dtype=dt, device=be.device)        # the padding must never be added
            buf[:, :d] = torch.as_tensor(X64, dtype=dt).to(be.device)
            x = buf[:, :d]
        pack = be.pack_centers(torch.as_tensor(C).to(be.device), dt)
        labels = be.empty((n,), torch.int32)
        sums, counts = be.zeros((k * d,), torch.float64), be.zeros((k,), torch.int64)
        be.lloyd_chunk(x, pack, k, labels, None, sums, counts, None)
        torch.cuda.synchronize()
        _check_exact(be, X64, labels, sums, counts, k, pattern)
    finally:
        be.flags = 0


def _tied_data(k, d, n, seed, big_rows):
    """Integer rows of a pattern with a dominant cluster over centres of which some are duplicates: the rows of a
    duplicate tie exactly and take the lower index.  ``big_rows`` rows get an entry of 2^19."""
    rng = np.random.RandomState(seed)
    pattern = np.where(rng.uniform(size=n) < 0.6, k // 3, rng.randint(0, k, n))
    C = mr.lattice_centres(k, d, spacing=10.0, offset=-10.0)
    dup = {k - 1: 0, k - 2: 1, k // 2: k // 3}                   # higher index -> the centre it duplicates
    first = np.arange(k)
    for j, i in dup.items():
        C[j] = C[i]
        first[j] = i
    X64 = _int_rows(pattern, C, seed + 1)
    want = first[pattern]
    big = rng.choice(n, big_rows, replace=False)
    X64[big, 0] = 2.0 ** 19
    for r in big:
        want[r] = int(np.argmin(((X64[r] - C) ** 2).sum(1)))            # float64 arg-min, lowest index on ties
    return X64, C, want, int(np.isin(pattern, list(dup)).sum()) + big_rows


@pytest.mark.parametrize("d,k", [(3, 16), (41, 100), (64, 256)])
def test_family1_deferred_rows_exact(be, d, k):
    """Deferred rows (whole clusters tied with a duplicate centre, entries beyond fp16's range) leave holes in the class
    lists and are added by the float64 re-check: the sums stay exact."""
    import torch

    n = 300_000
    X64, C, want_labels, n_tied = _tied_data(k, d, n, d + k, 5)
    be.flags = FORCE_TC
    try:
        x = be.to_device(X64, torch.float32)
        pack = be.pack_centers(torch.as_tensor(C).to(be.device), torch.float32)
        for want_dist in (False, True):
            labels = be.empty((n,), torch.int32)
            sums, counts = be.zeros((k * d,), torch.float64), be.zeros((k,), torch.int64)
            be.lloyd_chunk(x, pack, k, labels, be.empty((n,), torch.float32) if want_dist else None, sums, counts,
                           be.zeros((1,), torch.float64) if want_dist else None)
            torch.cuda.synchronize()
            assert be.deferred_rows(n, d, k, torch.float32) >= n_tied
            _check_exact(be, X64, labels, sums, counts, k, want_labels)
    finally:
        be.flags = 0


@pytest.mark.parametrize("d,k", [(16, 40), (128, 1024)])
def test_family3_tied_centres_exact(be, d, k):
    import torch

    n = 300_000
    X64, C, want_labels, _ = _tied_data(k, d, n, d + k, 0)
    x = be.to_device(torch.as_tensor(X64).to(be.device).to(torch.bfloat16), torch.bfloat16)      # integers: exact
    pack = be.pack_centers(torch.as_tensor(C).to(be.device), torch.bfloat16)
    labels = be.empty((n,), torch.int32)
    sums, counts = be.zeros((k * d,), torch.float64), be.zeros((k,), torch.int64)
    be.lloyd_chunk(x, pack, k, labels, None, sums, counts, None)
    torch.cuda.synchronize()
    _check_exact(be, X64, labels, sums, counts, k, want_labels)
