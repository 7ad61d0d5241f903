"""The CUDA-core chunk kernels (the generic kernel of bkm_simt.cu and the streaming kernels of bkm_stream.cu) at their
limits, on data whose every result is exact (run with -m gpu).  The cases and the data come from tests/core_cases.py,
whose restated geometry test_core_cases_host.py pins against the library's layout query.

Rows live in pitch-padded buffers whose padding holds 7.5e4 or NaN; outputs are filled with poison before each call
(labels -1, distances NaN, sums NaN) and so are the workspace's per-CTA partial records (0xff bytes).  Each call must
give, bit for bit:

* labels equal to numpy's float64 arg-min, lowest index on exact ties (duplicate centres in one J block, across J
  blocks, j and j + 256, across warps) and on the near-ties only float64 can decide;
* squared and plain distances equal to the exact distance rounded to the row type, inertia and distance sums exact;
* float64 sums and counts equal to numpy's, so that no row is lost or counted twice;
* the grid the launch picked (the per-CTA distance records that are no longer poison) equal to the restated clamp, and
  the fallback counter moving exactly when a family-1 / family-2 shape ran on the generic kernel.

test_ring_wraps runs the streaming kernels on row counts chosen from the grid they launch, so that every warp holds 1
to 2 NSTG + 1 tiles with the partial last tile at every ring stage; test_grid_tails does the same for the generic
kernel's tile loop.  test_near_ties_need_the_recheck shows that the near-tie data depends on the float64 re-check, and
test_nonfinite_row_gets_label_0 that a row with a NaN or infinite entry gets label 0 on every CUDA-core kernel.
"""
import numpy as np
import pytest

import core_cases as cc
from _util import sm_count

pytestmark = pytest.mark.gpu

CASES = {c["id"]: c for c in cc.cases()}


@pytest.fixture(scope="module")
def backends():
    from dask_ml_b200.engine import CudaBackend

    made = {}

    def get(flags):
        if flags not in made:
            made[flags] = CudaBackend(flags=flags)
        return made[flags]

    return get


@pytest.fixture(scope="module")
def sms(backends):
    be = backends(0)
    return sm_count(be.lib, be.device.index or 0)


def _tdt(dtype):
    import torch

    return torch.float32 if dtype == cc.F32 else torch.float64


def _npdt(dtype):
    return np.float32 if dtype == cc.F32 else np.float64


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view({4: np.uint32, 8: np.uint64}[a.dtype.itemsize])


def _assert_bits(got, want, what):
    got, want = np.asarray(got), np.asarray(want)
    bad = _bits(got) != _bits(want)
    assert not bad.any(), "%s: %d values differ, first at %s (got %r, want %r)" % (
        what, int(bad.sum()), np.argwhere(bad)[0].tolist(), got[bad][0], want[bad][0])


def _rows(be, X, dtype, pitch, base_off=0, pad="big"):
    """X as an (n, d) view of a padded buffer: row pitch ``pitch``, base ``base_off`` elements into an allocation,
    padding 7.5e4 ("big") or NaN."""
    import torch

    n, d = X.shape
    flat = torch.empty(n * pitch + 16, dtype=_tdt(dtype), device=be.device)
    flat.fill_(float("nan") if pad == "nan" else 7.5e4)
    buf = flat[base_off:base_off + n * pitch].view(n, pitch)
    buf[:, :d] = torch.from_numpy(np.ascontiguousarray(X)).to(be.device, _tdt(dtype))
    x = buf[:, :d]
    assert x.stride(0) == pitch and (x.data_ptr() % 16 == 0) == (base_off == 0)
    return x


def _pack(be, C, dtype):
    import torch

    return be.pack_centers(torch.as_tensor(C, dtype=torch.float64).to(be.device), _tdt(dtype))


def _poison_ws(be, x, k, dtype, sms):
    n, d = x.shape
    W = cc.ws_layout(n, d, k, dtype, sms)
    ws = be._workspace(n, d, k, _tdt(dtype))
    ws[W["psum"]:W["total"]].fill_(255)
    return ws, W


def _grid_used(ws, W):
    """CTAs that wrote their distance-sum record: the launched grid."""
    pin = ws[W["pin"]:W["pin"] + 8 * W["part_slots"]].cpu().numpy().view(np.uint64)
    written = pin != np.uint64(0xFFFFFFFFFFFFFFFF)
    g = int(written.sum())
    assert written[:g].all(), "records written out of CTA order"
    return g


def _lloyd(be, x, pack, k, dtype, sms):
    import torch

    n, d = x.shape
    labels = be.empty((n,), torch.int32).fill_(-1)
    md = be.empty((n,), _tdt(dtype)).fill_(float("nan"))
    sums = be.empty((k * d,), torch.float64).fill_(float("nan"))
    counts = be.empty((k,), torch.int64).fill_(-1)
    inertia = be.empty((1,), torch.float64).fill_(float("nan"))
    ws, W = _poison_ws(be, x, k, dtype, sms)
    before = int(be.lib.bkm_debug_fallback_count())
    be.lloyd_chunk(x, pack, k, labels, md, sums, counts, inertia, first=True)
    torch.cuda.synchronize()
    return dict(labels=labels.cpu().numpy(), md=md.cpu().numpy(), sums=sums.cpu().numpy().reshape(k, d),
                counts=counts.cpu().numpy(), inertia=float(inertia[0]), grid=_grid_used(ws, W),
                fallback=int(be.lib.bkm_debug_fallback_count()) - before)


def _assign(be, x, pack, k, dtype, sms, squared=True):
    import torch

    n, d = x.shape
    labels = be.empty((n,), torch.int32).fill_(-1)
    md = be.empty((n,), _tdt(dtype)).fill_(float("nan"))
    ds = be.zeros((1,), torch.float64)
    ws, W = _poison_ws(be, x, k, dtype, sms)
    before = int(be.lib.bkm_debug_fallback_count())
    be.assign_chunk(x, pack, k, labels, md, squared, ds)
    torch.cuda.synchronize()
    return dict(labels=labels.cpu().numpy(), md=md.cpu().numpy(), dist_sum=float(ds[0]), grid=_grid_used(ws, W),
                fallback=int(be.lib.bkm_debug_fallback_count()) - before)


def _check_labels(got, lab, where):
    bad = np.nonzero(got != lab)[0]
    assert len(bad) == 0, "%s: %d labels differ, first row %d: %d for %d" % (where, len(bad), bad[0], got[bad[0]],
                                                                             lab[bad[0]])


def _grids(p, d, k, n, dtype, mstep, sms):
    return {cc.grid(p, d, k, n, dtype, mstep, sms, occ) for occ in range(1, 9)}


def _run_case(backends, sms, c, X, C, lab, d2, check_grid=None):
    """Both entry points on the case's rows; every check.  Returns the two grids."""
    dtype, d, k, n = c["dtype"], c["d"], c["k"], c["n"]
    be = backends(c["flags"])
    T = _npdt(dtype)
    x = _rows(be, X, dtype, c["pitch"], c["base_off"], c["pad"])
    pack = _pack(be, C, dtype)
    fam = cc.kernel_family(d, k, dtype, c["flags"])
    sums, counts = cc.sums_ref(X, lab, k)
    grids = {}
    # assign first (labels only are written): a label out of range stops the test before an M-step uses it
    for squared in (True, False):
        a = _assign(be, x, pack, k, dtype, sms, squared)
        w = "%s assign squared=%s" % (c["id"], squared)
        _check_labels(a["labels"], lab, w)
        _assert_bits(a["md"], (d2 if squared else np.sqrt(d2)).astype(T), w + " distances")
        if squared:
            assert a["dist_sum"] == float(d2.sum()), (w, a["dist_sum"], float(d2.sum()))
        else:
            assert abs(a["dist_sum"] - float(np.sqrt(d2).sum())) <= 1e-12 * float(np.sqrt(d2).sum()) + 1e-300, w
        p = cc.plan(d, k, c["pitch"], dtype, c["flags"], False, c["base_off"] == 0)
        assert a["fallback"] == int(fam in (1, 2) and p["kernel"] == cc.GENERIC), (w, a["fallback"])
        assert a["grid"] in _grids(p, d, k, n, dtype, False, sms), (w, a["grid"], p)
        grids["assign"] = a["grid"]
    lo = _lloyd(be, x, pack, k, dtype, sms)
    w = c["id"] + " lloyd"
    _check_labels(lo["labels"], lab, w)
    _assert_bits(lo["md"], d2.astype(T), w + " min_d2")
    np.testing.assert_array_equal(lo["counts"], counts, err_msg=w)
    _assert_bits(lo["sums"], sums, w + " sums")
    assert np.array_equal(lo["sums"].sum(0), X.sum(0)), w            # every row counted once
    assert lo["inertia"] == float(d2.sum()), (w, lo["inertia"], float(d2.sum()))
    p = cc.plan(d, k, c["pitch"], dtype, c["flags"], True, c["base_off"] == 0)
    assert lo["fallback"] == int(fam in (1, 2) and p["kernel"] == cc.GENERIC), (w, lo["fallback"])
    assert lo["grid"] in _grids(p, d, k, n, dtype, True, sms), (w, lo["grid"], p)
    grids["lloyd"] = lo["grid"]
    return grids


@pytest.mark.parametrize("cid", list(CASES))
def test_case(backends, sms, cid):
    c = CASES[cid]
    X, C, near = cc.design(c)
    lab, d2 = cc.reference(X, C)
    _run_case(backends, sms, c, X, C, lab, d2)


NEAR = [cid for cid, c in CASES.items() if c["data"] == "near"]


@pytest.mark.parametrize("cid", NEAR)
def test_near_ties_need_the_recheck(backends, sms, cid):
    """With BKM_FLAG_NO_RECHECK the fp32 arithmetic decides alone: at least one designed near-tie row gets a
    different label, so the exact labels of test_case come from the float64 re-check."""
    c = CASES[cid]
    X, C, near = cc.design(c)
    lab, d2 = cc.reference(X, C)
    be = backends(c["flags"] | cc.NO_RECHECK)
    x = _rows(be, X, c["dtype"], c["pitch"])
    a = _assign(be, x, _pack(be, C, c["dtype"]), c["k"], c["dtype"], sms)
    assert ((a["labels"] != lab) & near).any(), cid
    assert ((a["labels"] >= 0) & (a["labels"] < c["k"])).all()


def _random_rows(n, d, seed):
    rng = np.random.RandomState(seed)
    return rng.standard_normal((n, d)) * rng.uniform(0.1, 10.0, size=d)


REPRO = [("s2", 13, 20, 16, cc.F32, 0), ("s1", 13, 28, 16, cc.F32, 0), ("smallk", 13, 20, 16, cc.F32, cc.FORCE_SIMT),
         ("smem-f32", 100, 40, 100, cc.F32, 0), ("smem-f64", 40, 30, 40, cc.F64, 0), ("rt2-f64", 7125, 4, 7125, cc.F64, 0)]


@pytest.mark.parametrize("name,d,k,pitch,dtype,flags", REPRO, ids=[r[0] for r in REPRO])
def test_two_launches_same_bits(backends, sms, name, d, k, pitch, dtype, flags):
    """Random, non-exact rows: two Lloyd calls give the same bits (SMEM mode and the streaming kernels fold their
    partials in a fixed order)."""
    n = 20_000 if d < 1000 else 300
    X = _random_rows(n, d, d + k)
    C = X[:k].copy()
    be = backends(flags)
    x = _rows(be, X, dtype, pitch)
    pack = _pack(be, C, dtype)
    p = cc.plan(d, k, pitch, dtype, flags, True)
    r1, r2 = _lloyd(be, x, pack, k, dtype, sms), _lloyd(be, x, pack, k, dtype, sms)
    for key in ("labels", "md", "counts"):
        _assert_bits(r1[key], r2[key], "%s %s" % (name, key))
    if not p["GLOBAL"]:                        # GLOBAL mode: float64 atomics in no fixed order
        _assert_bits(r1["sums"], r2["sums"], name + " sums")
    assert r1["inertia"] == r2["inertia"]


# ------------------------------------------------------------------------------------------------ grid-chosen row counts
def _measure_full_grid(backends, sms, c, rows_per_tile, mstep):
    """The grid of a call with more tiles than any occupancy can take, and the occupancy it implies."""
    p = cc.plan(c["d"], c["k"], c["pitch"], c["dtype"], c["flags"], mstep)
    tiles = sms * 8 * (cc.SW if p["kernel"] != cc.GENERIC else 1) + 1
    n = rows_per_tile * tiles
    X, C = cc.lattice(c["d"], c["k"], n, 5, R=2, r=1)
    be = backends(c["flags"])
    x = _rows(be, X, c["dtype"], c["pitch"])
    pack = _pack(be, C, c["dtype"])
    g = (_lloyd if mstep else _assign)(be, x, pack, c["k"], c["dtype"], sms)["grid"]
    occ = g // sms
    assert g % sms == 0 and 1 <= occ <= 8 and g == cc.grid(p, c["d"], c["k"], n, c["dtype"], mstep, sms, occ), (g, p)
    assert occ <= 228 * 1024 // (p["smem"] + 1024), (occ, p["smem"])
    return g, occ


RING = [("two-row", 13, 20, 16), ("one-row", 13, 28, 16), ("two-row-d3-L4", 3, 12, 4)]


@pytest.mark.parametrize("name,d,k,pitch", RING, ids=[r[0] for r in RING])
def test_ring_wraps(backends, sms, name, d, k, pitch):
    """Warps holding 1 to 2 NSTG + 1 tiles, the partial last tile at every ring stage, n = T * rows + (-1, 0, 1)."""
    c = cc._c(name, d, k, 0, pitch=pitch)
    p = cc.plan(d, k, pitch, cc.F32, 0, True)
    assert p["kernel"] in (cc.ONE_ROW, cc.TWO_ROW)
    R, nstg = p["rows"], p["stages"]
    G, occ = _measure_full_grid(backends, sms, c, R, True)
    nw = G * cc.SW
    top = (2 * nstg) * nw + nw // 2 + 1
    X, C = cc.lattice(d, k, top * R + 1, 11, R=2, r=1)
    lab_all, d2_all = cc.reference(X, C)
    for m in range(1, 2 * nstg + 2):
        T = (m - 1) * nw + nw // 2
        for n in (T * R - 1, T * R, T * R + 1):
            cn = dict(c, n=n, id="%s m=%d n=%d" % (name, m, n))
            grids = _run_case(backends, sms, cn, X[:n], C, lab_all[:n], d2_all[:n])
            want = cc.grid(p, d, k, n, cc.F32, True, sms, occ)
            assert grids["lloyd"] == want and grids["assign"] == want, (cn["id"], grids, want)
            assert (cc._cdiv(n, R) - 1) // nw == m - 1         # the last tile is its warp's m-th


TAILS = [("f32", 20, 17, cc.F32), ("f64", 20, 9, cc.F64), ("f32-global", 96, 400, cc.F32)]


@pytest.mark.parametrize("name,d,k,dtype", TAILS, ids=[t[0] for t in TAILS])
def test_grid_tails(backends, sms, name, d, k, dtype):
    """The generic kernel on G - 1, G and G + 1 row tiles (G its full grid) and on every row count around them."""
    c = cc._c(name, d, k, 0, dtype)
    p = cc.plan(d, k, d, dtype, 0, True)
    assert p["kernel"] == cc.GENERIC
    G, occ = _measure_full_grid(backends, sms, c, p["rt"], True)
    rt = p["rt"]
    X, C = cc.lattice(d, k, (G + 1) * rt + 1, 13, R=2, r=1)
    lab_all, d2_all = cc.reference(X, C)
    for n in ((G - 1) * rt, G * rt - 1, G * rt, G * rt + 1, (G + 1) * rt):
        cn = dict(c, n=n, id="%s n=%d" % (name, n))
        grids = _run_case(backends, sms, cn, X[:n], C, lab_all[:n], d2_all[:n])
        assert grids["lloyd"] == cc.grid(p, d, k, n, dtype, True, sms, occ), (cn["id"], grids)


# ------------------------------------------------------------------------------------------------ non-finite rows
NONFINITE = [("generic-d13-k20", 13, 20, 16, cc.FORCE_SIMT), ("generic-d100-k40", 100, 40, 100, 0),
             ("generic-d20-k300", 20, 300, 20, 0), ("s2-d13-k20", 13, 20, 16, 0), ("s1-d13-k28", 13, 28, 16, 0)]


@pytest.mark.parametrize("entry", ["assign", "lloyd"])
@pytest.mark.parametrize("name,d,k,pitch,flags", NONFINITE, ids=[t[0] for t in NONFINITE])
def test_nonfinite_row_gets_label_0(backends, sms, entry, name, d, k, pitch, flags):
    """fp32 rows with a NaN, +inf or -inf entry (the float64 re-check finds no finite distance): label 0 and a
    non-finite distance, as on the bf16 path; every other row exact, the M-step adds the rows to cluster 0."""
    n = 700
    X, C = cc.lattice(d, k, n, 3)
    lab, d2 = cc.reference(X, C)
    bad = {5: np.nan, 64: np.inf, 301: -np.inf, n - 1: np.nan}
    Xb = X.copy()
    for i, v in bad.items():
        Xb[i, (3 * i) % d] = v
    rows = np.array(sorted(bad))
    lab[rows] = 0
    be = backends(flags)
    x = _rows(be, Xb, cc.F32, pitch)
    pack = _pack(be, C, cc.F32)
    out = (_assign if entry == "assign" else _lloyd)(be, x, pack, k, cc.F32, sms)
    _check_labels(out["labels"], lab, "%s %s" % (name, entry))
    ok = np.ones(n, dtype=bool)
    ok[rows] = False
    assert not np.isfinite(out["md"][rows]).any()
    _assert_bits(out["md"][ok], d2[ok].astype(np.float32), name + " distances")
    if entry == "lloyd":
        sums, counts = cc.sums_ref(X[ok], lab[ok], k)
        counts[0] += len(rows)
        np.testing.assert_array_equal(out["counts"], counts)
        _assert_bits(out["sums"][1:], sums[1:], name + " sums")
