"""The X ring of the fp32 tensor-core kernel (bkm_tc.cu) in all four epilogues, at the row counts where it wraps.

Each CTA streams its tiles through S shared-memory slots filled by TMA; tile lt + S is loaded into the slot of tile lt
once that is done, and the slot's barrier parity flips on every pass.  With G SMs and 64-row tiles a CTA holds more than
S tiles only past 64 G S rows, and S depends on the variant (bkm_debug_tc_layout, tests/test_tc_layout_host.py).  Here
every entry point on that kernel runs at row counts derived from G and S: below, at and past the first refill, at the
second phase flip, and for about 20 passes of the ring.

Rows are a view X = buf[3:3 + n, :d] of a buffer whose other rows and padding columns hold a poison (a finite value in
the data's range, or NaN); every output must be bit-identical to the same call on the clean copy that
``CudaBackend.to_device`` makes, and must match float64 on the device.  The data are well separated blobs on a 2^-12
grid around a lattice of centres: no row is a float64 near-tie (so none is deferred to the float64 re-check, and
nothing depends on the order of its float64 atomics), and every sum of the M-step is reproducible to the bit."""
import contextlib

import numpy as np
import pytest
import torch

from _util import TC_ARGMIN, TC_COLSUM, TC_EMBED, TC_XFORM, sm_count, tc_layout
from dask_ml_b200 import _lib

pytestmark = pytest.mark.gpu

R0 = 3                                  # first row of the view in its buffer
SPARE = 64                              # rows of the buffer outside the view (3 before, 61 after)
POISONS = (0.375, float("nan"))
GRID = 2.0 ** -12
KWS = (1, 7, 32, 33, 64)                # embedding widths: S = 8, 8, 6, 6, 4 at N = 256
TAU_TC = lambda d: (8.0 * np.sqrt(3.0 * ((d + 7) // 8)) + 16.0) * 2.0 ** -24      # bkm_api.cu tau_for, family 1
TAU_SIMT = lambda d: 8.0 * (np.sqrt(d) + 2.0) * 2.0 ** -24                          # CUDA-core kernels

# Row counts as functions of the SM count G and the ring depth S of the variant under test
ROWS = {
    "1": lambda G, S: 1,
    "63": lambda G, S: 63,
    "64": lambda G, S: 64,
    "65": lambda G, S: 65,
    "64G-1": lambda G, S: 64 * G - 1,                       # one tile per CTA, the last one partial
    "64G+1": lambda G, S: 64 * G + 1,                       # CTA 0 takes a second, one-row tile
    "64GS": lambda G, S: 64 * G * S,                        # every CTA exactly fills its ring, no refill
    "64GS+64": lambda G, S: 64 * G * S + 64,                # only CTA 0 refills (its slot 0)
    "64G(S+1)-1": lambda G, S: 64 * G * (S + 1) - 1,        # every CTA refills once, the last tile partial
    "64G(S+1)+1": lambda G, S: 64 * G * (S + 1) + 1,
    "64G2S+1": lambda G, S: 64 * G * 2 * S + 1,             # CTA 0 reaches the second phase flip of slot 0
    "20-passes": lambda G, S: 64 * G * S * 20 + 64 * (G // 3) + 29,   # ... then a third of the CTAs one more tile
}
BELOW, ABOVE = "64GS-37", "64G(S+2)+37"
ROWS[BELOW] = lambda G, S: 64 * G * S - 37                  # the ring never wraps; the last tile partial
ROWS[ABOVE] = lambda G, S: 64 * G * (S + 2) + 37            # every CTA refills twice, CTA 0 three times


@pytest.fixture(scope="module")
def be():
    from dask_ml_b200.engine import CudaBackend

    return CudaBackend()


@pytest.fixture(scope="module")
def G(be):
    return sm_count(be.lib, be.device.index or 0)


@contextlib.contextmanager
def _flags(be, flags):
    old = be.flags
    be.flags = flags
    try:
        yield
    finally:
        be.flags = old


# ---------------------------------------------------------------------------------------------- data and references
_CENTRES = {}


def _centres(d, k):
    """k distinct points of the lattice {-1, -0.75, ..., 1}^d (float64 on the device): 0.25 apart at least, so that
    rows within 0.0125 (one standard deviation) of one are far from a near-tie with any other."""
    if (d, k) not in _CENTRES:
        rng = np.random.RandomState(1000 * d + k)
        rows = {}
        while len(rows) < k:
            rows.setdefault(tuple(rng.randint(-4, 5, size=d) * 0.25), None)
        _CENTRES[(d, k)] = torch.tensor(list(rows), dtype=torch.float64, device="cuda")
    return _CENTRES[(d, k)]


class _Rows:
    """n rows around the centres of (d, k), exact in fp32: the clean copy, the pack and the poisoned views."""

    def __init__(self, be, d, k, n):
        self.d, self.k, self.n = d, k, n
        self.C = _centres(d, k)
        g = torch.Generator(device=be.device).manual_seed(n * 257 + d * 31 + k)
        lab = torch.randint(0, k, (n,), device=be.device, generator=g)
        noise = torch.round(torch.randn((n, d), device=be.device, generator=g, dtype=torch.float64) * (0.0125 / GRID))
        self.X = (self.C[lab] + noise * GRID).float().contiguous()
        self.x = be.to_device(self.X, torch.float32)
        assert self.x.stride(0) % 4 == 0 and self.x.data_ptr() % 16 == 0
        self.pack = be.pack_centers(self.C, torch.float32)
        self.gamma = 1.0 / d

    def poisoned(self):
        """(name, view) for the two row pitches and the two poisons; every element outside the view is poison."""
        p0 = (self.d + 3) // 4 * 4
        for pitch in (p0, p0 + 8):
            for poison in POISONS:
                buf = torch.full((self.n + SPARE, pitch), poison, device="cuda")
                buf[R0:R0 + self.n, :self.d] = self.X
                yield "pitch %d, poison %r" % (pitch, poison), buf[R0:R0 + self.n, :self.d]

    def blocks(self, rows=1 << 17):
        """(start, end, rows as float64, float64 d^2 to every centre) in row blocks."""
        cc = (self.C * self.C).sum(1)
        for s in range(0, self.n, rows):
            xb = self.X[s:s + rows].double()
            d2 = torch.clamp((xb * xb).sum(1, keepdim=True) + cc[None, :] - 2.0 * xb @ self.C.T, min=0.0)
            yield s, s + xb.shape[0], xb, d2


def _labels_f64(d2):
    """float64 arg-min of a block and the margin of the second best."""
    if d2.shape[1] == 1:
        return torch.zeros(d2.shape[0], dtype=torch.int64, device=d2.device), torch.ones_like(d2[:, 0])
    top = torch.topk(d2, 2, dim=1, largest=False)
    return top.indices[:, 0], top.values[:, 1] - top.values[:, 0]


def _bits(t):
    return t.view(torch.int64) if t.dtype == torch.float64 else t.view(torch.int32) if t.dtype == torch.float32 else t


def _assert_same(got, want, what):
    """Bit-identical outputs (NaN included)."""
    for key in want:
        assert torch.equal(_bits(got[key]), _bits(want[key])), "%s: %s differs" % (what, key)


# ---------------------------------------------------------------------------------------------- the entry points
def _run_lloyd(be, r, x):
    n, k, d = r.n, r.k, r.d
    o = dict(labels=be.empty((n,), torch.int32), min_d2=be.empty((n,), torch.float32),
             sums=be.zeros((k * d,), torch.float64), counts=be.zeros((k,), torch.int64),
             inertia=be.zeros((1,), torch.float64), labels_nd=be.empty((n,), torch.int32),
             sums_nd=be.zeros((k * d,), torch.float64), counts_nd=be.zeros((k,), torch.int64),
             labels_a=be.empty((n,), torch.int32))
    with _flags(be, _lib.FLAG_FORCE_TC):
        be.lloyd_chunk(x, r.pack, k, o["labels"], o["min_d2"], o["sums"], o["counts"], o["inertia"])
        dfr = [be.deferred_rows(n, d, k, torch.float32)]
        be.lloyd_chunk(x, r.pack, k, o["labels_nd"], None, o["sums_nd"], o["counts_nd"], None)
        dfr.append(be.deferred_rows(n, d, k, torch.float32))
        be.assign_chunk(x, r.pack, k, o["labels_a"], None, True, None)
    o["deferred"] = torch.tensor(dfr)
    return o


def _check_lloyd(r, o):
    k, d = r.k, r.d
    got = o["labels"].long()
    ref = torch.zeros((k, d), dtype=torch.float64, device="cuda")
    cmax = float((r.C * r.C).sum(1).max())
    exact_sum, scale_sum = 0.0, 0.0
    for s, e, xb, d2 in r.blocks():
        want, margin = _labels_f64(d2)
        bad = got[s:e] != want
        if bool(bad.any()):
            xs = (xb * xb).sum(1)[bad] + cmax
            assert bool((margin[bad] <= 1e-9 * xs).all()), int(bad.sum())
        ref.index_add_(0, got[s:e], xb)
        exact = ((xb - r.C[got[s:e]]) ** 2).sum(1)
        scale = (xb * xb).sum(1) + cmax
        assert float(((o["min_d2"][s:e].double() - exact).abs() / scale).max()) < 2e-6
        exact_sum += float(exact.sum()); scale_sum += float(scale.sum())
    assert torch.equal(o["counts"], torch.bincount(got, minlength=k))
    assert float((o["sums"].view(k, d) - ref).abs().max()) <= 2e-6 * float(ref.abs().max()) + 1e-9
    assert abs(float(o["inertia"][0]) - exact_sum) <= 1e-5 * exact_sum + 2e-6 * scale_sum
    # without distances: the same labels, counts and (same M-step order) the same sums; assign agrees with Lloyd
    assert torch.equal(o["labels_nd"], o["labels"]) and torch.equal(o["counts_nd"], o["counts"])
    assert torch.equal(o["sums_nd"], o["sums"])
    assert torch.equal(o["labels_a"], o["labels"])
    assert int(o["deferred"].sum()) == 0           # no near-ties here: a read NaN would show up as a deferred row


def _run_assign(be, r, x):
    n, k, d = r.n, r.k, r.d
    o = dict(labels=be.empty((n,), torch.int32), dist2=be.empty((n,), torch.float32), dsum=be.zeros((1,), torch.float64),
             labels_r=be.empty((n,), torch.int32), dist=be.empty((n,), torch.float32),
             labels_only=be.empty((n,), torch.int32))
    with _flags(be, _lib.FLAG_FORCE_TC):
        be.assign_chunk(x, r.pack, k, o["labels"], o["dist2"], True, o["dsum"])
        dfr = [be.deferred_rows(n, d, k, torch.float32)]
        be.assign_chunk(x, r.pack, k, o["labels_r"], o["dist"], False, None)
        dfr.append(be.deferred_rows(n, d, k, torch.float32))
        be.assign_chunk(x, r.pack, k, o["labels_only"], None, True, None)
        dfr.append(be.deferred_rows(n, d, k, torch.float32))
    o["deferred"] = torch.tensor(dfr)
    return o


def _check_assign(r, o):
    got = o["labels"].long()
    cmax = float((r.C * r.C).sum(1).max())
    exact_sum, scale_sum = 0.0, 0.0
    for s, e, xb, d2 in r.blocks():
        want, margin = _labels_f64(d2)
        bad = got[s:e] != want
        if bool(bad.any()):
            xs = (xb * xb).sum(1)[bad] + cmax
            assert bool((margin[bad] <= 1e-9 * xs).all()), int(bad.sum())
        exact = ((xb - r.C[got[s:e]]) ** 2).sum(1)
        scale = (xb * xb).sum(1) + cmax
        assert float(((o["dist2"][s:e].double() - exact).abs() / scale).max()) < 2e-6
        assert float(((o["dist"][s:e].double() ** 2 - exact).abs() / scale).max()) < 4e-6
        exact_sum += float(exact.sum()); scale_sum += float(scale.sum())
    assert abs(float(o["dsum"][0]) - exact_sum) <= 1e-5 * exact_sum + 2e-6 * scale_sum
    assert torch.equal(o["labels_r"], o["labels"]) and torch.equal(o["labels_only"], o["labels"])
    assert int(o["deferred"].sum()) == 0


def _run_transform(be, r, x):
    o = {}
    with _flags(be, _lib.FLAG_FORCE_TC):
        for mode in (0, 1, 2):
            o["mode%d" % mode] = be.empty((r.n, r.k), torch.float32)
            be.transform_chunk(x, r.pack, r.k, o["mode%d" % mode], mode=mode, gamma=r.gamma)
    return o


def _check_transform(r, o):
    """test_transform_tensor_path's bounds: error relative to ||x||^2 + ||c||^2."""
    cc = (r.C * r.C).sum(1)
    for s, e, xb, d2 in r.blocks():
        scale = (xb * xb).sum(1, keepdim=True) + cc[None, :]
        g0, g1, g2 = (o["mode%d" % m][s:e].double() for m in (0, 1, 2))
        assert float(((g0 * g0 - d2).abs() / scale).max()) < 2e-6
        assert float(((g1 - d2).abs() / scale).max()) < 2e-6
        assert float((g2 - torch.exp(-r.gamma * d2)).abs().max()) / (r.gamma * float(scale.max())) < 2e-6


def _run_colsum(be, r, x):
    c = be.zeros((r.k,), torch.float64)
    with _flags(be, _lib.FLAG_FORCE_TC):
        be.kernel_colsum(x, r.pack, r.k, r.gamma, c, first=True)
        first = c.clone()
        be.kernel_colsum(x, r.pack, r.k, r.gamma, c, first=False)
    return dict(first=first, second=c)


def _check_colsum(r, o):
    """test_colsum_matches_float64's bounds; the second call adds the same column sums."""
    tau = TAU_TC(r.d)
    cmax = float((r.C * r.C).sum(1).max())
    want = torch.zeros((r.k,), dtype=torch.float64, device="cuda")
    bound = torch.zeros_like(want)
    for s, e, xb, d2 in r.blocks():
        v = torch.exp(-r.gamma * d2)
        want += v.sum(0)
        bound += (v * (r.gamma * tau * ((xb * xb).sum(1)[:, None] + cmax) + 4e-6)).sum(0)
    got = o["first"]
    err = (got - want).abs()
    assert bool((err <= bound + 1e-6 * want).all()), float((err / want).max())
    assert float((err / want).max()) < 2e-5
    assert torch.equal(o["second"], 2.0 * got)


def _embedding(r, kw):
    """(gamma, W) of an embedding of width kw.  One output is the sign of e: there the gamma is sharp enough that a row's
    own centre (kernel value 1) outweighs all others together (each below exp(-200 * 0.0375)), and the weights have
    random signs and magnitudes of at least 0.5, so that the sign follows the row's centre and |e| is far from 0."""
    g = torch.Generator(device="cuda").manual_seed(r.k * 100 + kw)
    W = torch.randn((r.k, kw), device="cuda", generator=g)
    if kw > 1:
        return r.gamma, W
    return 200.0, torch.where(W < 0, W - 0.5, W + 0.5)


def _run_embed(be, r, x, kw):
    gamma, W = _embedding(r, kw)
    out = be.zeros((r.n, kw), torch.float32)
    with _flags(be, _lib.FLAG_FORCE_TC):
        be.nystrom_embed(x, r.pack, r.k, gamma, W, out)
    return dict(out=out)


def _check_embed(r, o, kw):
    """test_embed_matches_float64's bound."""
    gamma, W = _embedding(r, kw)
    W = W.double()
    for s, e, xb, d2 in r.blocks():
        m = d2.min(1, keepdim=True).values
        v = torch.exp(-gamma * (d2 - m)) @ W
        want = v / torch.sqrt((v * v).sum(1, keepdim=True))
        assert float((o["out"][s:e].double() - want).abs().max()) < 1e-4


def _jobs(be, d, k):
    """(name, the variant's (KS, N, S), run, check) of every entry point on the tensor-core kernel."""
    lay = lambda epi, mstep=0, kw=0: tc_layout(be.lib, d, k, epi, mstep, kw)[:3]
    yield "lloyd", lay(TC_ARGMIN, 1), _run_lloyd, _check_lloyd
    yield "assign", lay(TC_ARGMIN), _run_assign, _check_assign
    yield "transform", lay(TC_XFORM), _run_transform, _check_transform
    yield "colsum", lay(TC_COLSUM), _run_colsum, _check_colsum
    for kw in KWS:
        yield ("embed kw=%d" % kw, lay(TC_EMBED, kw=kw), lambda be, r, x, kw=kw: _run_embed(be, r, x, kw),
               lambda r, o, kw=kw: _check_embed(r, o, kw))


def _exercise(be, G, d, k, row_kind):
    """Every entry point at the row count `row_kind` of its own variant's S, on the clean rows (against float64, and
    a repeat bit-identical) and on every poisoned view (bit-identical to the clean rows)."""
    before = int(be.lib.bkm_debug_fallback_count())
    by_n = {}
    for name, (ks, nn, S), run, check in _jobs(be, d, k):
        assert ks == (d + 15) // 16
        by_n.setdefault(ROWS[row_kind](G, S), []).append((name, run, check))
    for n, jobs in sorted(by_n.items()):
        r = _Rows(be, d, k, n)
        clean = {}
        for name, run, check in jobs:
            clean[name] = run(be, r, r.x)
            torch.cuda.synchronize()
            check(r, clean[name])
            _assert_same(run(be, r, r.x), clean[name], "%s, n=%d, repeated" % (name, n))
        for what, xp in r.poisoned():
            for name, run, check in jobs:
                _assert_same(run(be, r, xp), clean[name], "%s, n=%d, %s" % (name, n, what))
        del r, clean
    assert be.lib.bkm_debug_abort_code() == 0
    # FORCE_TC makes a fallback an error; the counter confirms that none happened
    assert int(be.lib.bkm_debug_fallback_count()) == before


# ---------------------------------------------------------------------------------------------- row counts
@pytest.mark.parametrize("row_kind", [kind for kind in ROWS if kind not in (BELOW, ABOVE)])
@pytest.mark.parametrize("d,k", [(64, 256), (29, 30), (5, 200)])
def test_ring_row_counts(be, G, d, k, row_kind):
    """The whole row-count sweep on three shapes: N = 256 with every ring depth (5, 8, 6, 4), N = 32 with padded
    pitches (KS = 2), and N = 256 at KS = 1 with padded pitches."""
    _exercise(be, G, d, k, row_kind)


# ---------------------------------------------------------------------------------------------- instances
INSTANCE_K = [(10, 16), (30, 32), (60, 64), (100, 128), (129, 256), (200, 256), (256, 256)]
INSTANCE_D = [(5, 1), (29, 2), (47, 3), (64, 4)]


@pytest.mark.parametrize("row_kind", [BELOW, ABOVE])
@pytest.mark.parametrize("k,N", INSTANCE_K)
@pytest.mark.parametrize("d,KS", INSTANCE_D)
def test_ring_instances(be, G, d, KS, k, N, row_kind):
    """Every (N, KS) instance of every epilogue, just below the first refill and past it; k = 129 and 256 are the M-step
    variants with an odd ring (S = 5)."""
    for name, (ks, nn, S), _, _ in _jobs(be, d, k):
        assert (ks, nn) == (KS, N), name
        assert (S == 5) == (name == "lloyd" and N == 256), (name, S)
    _exercise(be, G, d, k, row_kind)


# ---------------------------------------------------------------------------------------------- output layouts
SENTINEL = -1234.5


def _window_outputs(be, r, k_out, call):
    """The output written through three layouts of a sentinel-filled buffer: an even pitch on an aligned base (vector
    stores), an odd pitch, a base one float off 8-byte alignment (scalar stores).  Returns the three (n, k_out) blocks
    after checking that nothing outside them changed, rows past n included."""
    n = r.n
    even = k_out + 2 + k_out % 2
    odd = k_out + 3 - k_out % 2
    bufs = [torch.full((n + 4, even), SENTINEL, device="cuda"), torch.full((n + 4, odd), SENTINEL, device="cuda")]
    flat = torch.full(((n + 4) * even + 1,), SENTINEL, device="cuda")
    bufs.append(flat[1:].view(n + 4, even))
    assert bufs[0].data_ptr() % 8 == 0 and bufs[2].data_ptr() % 8 == 4 and bufs[1].stride(0) % 2 == 1
    outs = []
    for b in bufs:
        call(b[:n, :k_out])
        torch.cuda.synchronize()
        keep = torch.ones(b.shape, dtype=torch.bool, device="cuda")
        keep[:n, :k_out] = False
        assert bool((b[keep] == SENTINEL).all())
        outs.append(b[:n, :k_out].clone())
    assert float(flat[0]) == SENTINEL
    return outs


@pytest.mark.parametrize("row_kind", ["65", "64GS+64", ABOVE])
@pytest.mark.parametrize("d,k", [(29, 30), (47, 129), (64, 256)])
def test_output_layouts(be, G, d, k, row_kind):
    """The transform and embedding outputs go to any row pitch and base: the same bits every way as into a plain
    (n, k) tensor, and no store outside the (n, k) window."""
    before = int(be.lib.bkm_debug_fallback_count())
    S = tc_layout(be.lib, d, k, TC_XFORM)[2]
    r = _Rows(be, d, k, ROWS[row_kind](G, S))
    with _flags(be, _lib.FLAG_FORCE_TC):
        for mode in (0, 1, 2):
            plain = be.empty((r.n, k), torch.float32)
            be.transform_chunk(r.x, r.pack, k, plain, mode=mode, gamma=r.gamma)
            for o in _window_outputs(be, r, k, lambda o: be.transform_chunk(r.x, r.pack, k, o, mode=mode, gamma=r.gamma)):
                assert torch.equal(o.view(torch.int32), plain.view(torch.int32)), mode
        for kw in (7, 33):
            gamma, W = _embedding(r, kw)
            plain = be.empty((r.n, kw), torch.float32)
            be.nystrom_embed(r.x, r.pack, k, gamma, W, plain)
            for o in _window_outputs(be, r, kw, lambda o: be.nystrom_embed(r.x, r.pack, k, gamma, W, o)):
                assert torch.equal(o.view(torch.int32), plain.view(torch.int32)), kw
    _check_embed(r, {"out": plain}, 33)
    assert int(be.lib.bkm_debug_fallback_count()) == before


# ---------------------------------------------------------------------------------------------- alignment fallback
@pytest.mark.parametrize("d,k", [(29, 30), (64, 256)])
def test_unaligned_rows_fall_back_to_the_cuda_cores(be, d, k):
    """Rows whose base is 4 bytes off 16-byte alignment cannot be read by TMA: each entry point runs on a CUDA-core
    kernel instead, counts the fallback, and matches float64 within the CUDA-core bounds; under FORCE_TC it refuses."""
    r = _Rows(be, d, k, 20_000)
    pitch = (d + 1 + 3) // 4 * 4
    buf = torch.full((r.n, pitch), POISONS[0], device="cuda")
    buf[:, 1:d + 1] = r.X
    x = buf[:, 1:d + 1]
    assert x.data_ptr() % 16 == 4 and x.stride(0) % 4 == 0
    assert be.kernel_family(d, k, torch.float32) == 1
    n, kw = r.n, 7
    gamma, W = _embedding(r, kw)
    counter = lambda: int(be.lib.bkm_debug_fallback_count())
    calls = []

    def fell_back(fn):
        c0 = counter()
        out = fn()
        torch.cuda.synchronize()
        assert counter() == c0 + 1
        calls.append(fn)
        return out

    # Lloyd and assign
    lab, md = be.empty((n,), torch.int32), be.empty((n,), torch.float32)
    sums, counts, inertia = be.zeros((k * d,), torch.float64), be.zeros((k,), torch.int64), be.zeros((1,), torch.float64)
    fell_back(lambda: be.lloyd_chunk(x, r.pack, k, lab, md, sums, counts, inertia))
    lab2, dist = be.empty((n,), torch.int32), be.empty((n,), torch.float32)
    fell_back(lambda: be.assign_chunk(x, r.pack, k, lab2, dist, False, None))
    got = lab.long()
    cmax = float((r.C * r.C).sum(1).max())
    (_, _, xb, d2), = r.blocks()
    want, margin = _labels_f64(d2)
    bad = got != want
    if bool(bad.any()):
        assert bool((margin[bad] <= 1e-9 * ((xb * xb).sum(1)[bad] + cmax)).all()), int(bad.sum())
    assert torch.equal(lab2, lab)
    assert torch.equal(counts, torch.bincount(got, minlength=k))
    ref = torch.zeros((k, d), dtype=torch.float64, device="cuda").index_add_(0, got, xb)
    assert float((sums.view(k, d) - ref).abs().max()) <= 2e-6 * float(ref.abs().max()) + 1e-9
    exact = ((xb - r.C[got]) ** 2).sum(1)
    scale = (xb * xb).sum(1) + cmax
    assert float(((md.double() - exact).abs() / scale).max()) < 2e-6
    assert float(((dist.double() ** 2 - exact).abs() / scale).max()) < 4e-6
    assert abs(float(inertia[0]) - float(exact.sum())) <= 1e-5 * float(exact.sum()) + 2e-6 * float(scale.sum())
    # transform (test_transform_chunk's CUDA-core bound), column sums and embedding (the CUDA-core bounds of
    # test_colsum_matches_float64 and test_embed_matches_float64)
    out = be.empty((n, k), torch.float32)
    fell_back(lambda: be.transform_chunk(x, r.pack, k, out, mode=1, gamma=r.gamma))
    scale2 = (xb * xb).sum(1, keepdim=True) + (r.C * r.C).sum(1)[None, :]
    assert float(((out.double() - d2).abs() / scale2).max()) < 1e-5
    c = be.zeros((k,), torch.float64)
    fell_back(lambda: be.kernel_colsum(x, r.pack, k, r.gamma, c, first=True))
    v = torch.exp(-r.gamma * d2)
    wc = v.sum(0)
    bound = (v * (r.gamma * TAU_SIMT(d) * ((xb * xb).sum(1)[:, None] + cmax) + 4e-6)).sum(0) + 1e-6 * wc
    assert bool(((c - wc).abs() <= bound).all()) and float(((c - wc).abs() / wc).max()) < 2e-5
    e = be.zeros((n, kw), torch.float32)
    fell_back(lambda: be.nystrom_embed(x, r.pack, k, gamma, W, e))
    _check_embed(r, {"out": e}, kw)
    # FORCE_TC: an error instead of the fallback, and no count
    with _flags(be, _lib.FLAG_FORCE_TC):
        for fn in calls:
            c0 = counter()
            with pytest.raises(RuntimeError, match="pointer alignment"):
                fn()
            assert counter() == c0
