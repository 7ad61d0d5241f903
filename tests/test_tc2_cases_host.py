"""The large-shape tensor path's geometry and designed data without a GPU (tests/tc2_cases.py).

* The host restatement equals the library's own layout query (bkm_debug_tc2_layout) for every d in 1..128, a dense
  set of k in 1..4096 and several row counts, at 132 and 114 SMs and a few odd counts; the workspace total equals
  bkm_workspace_bytes.
* The cases reach every limit of the path at both SM counts: every MMA width, padded and full, every slice count with
  a one-column and a full last slice, one and two K-blocks and partial last K-steps, every DS transition at every
  features-per-lane width, NB = RP_MAXB, the row counts around the tile groups, the binning kernel's second turn and
  the re-check's turn boundaries.
* The designed data is what it claims: bf16-exact, labels equal to the float64 arg-min, near-tie gaps strictly inside
  the bound, exact ties at 0, every other gap at least 16x outside it, partial sums on the 2^-18 grid below 2^6.
"""
import ctypes

import numpy as np
import pytest

import msum_ref as mr
import tc2_cases as tc

BF16 = 2
EUNSUPPORTED, EINVAL = -3, -1


@pytest.fixture(scope="module")
def lib():
    from dask_ml_b200 import _lib

    return _lib.load()


def _query(lib, d, k, n, sms):
    out = (ctypes.c_int * len(tc.LAYOUT_FIELDS))()
    rc = lib.bkm_debug_tc2_layout(int(d), int(k), int(n), int(sms), out)
    return rc, tuple(out)


K_DENSE = sorted(set(range(1, 66)) | set(range(66, 4097, 29)) | {256 * s + o for s in range(1, 16) for o in (0, 1)} |
                 {kt + o for dp in (32, 64, 128) for kt in tc.ds_transitions(dp) for o in (-1, 0)} | {4096})


@pytest.mark.parametrize("sms", [132, 114])
def test_layout_equals_library(lib, sms):
    ns = (1, 63, 5000, 4 * sms * tc.RP_TILE + 1)
    for d in range(1, 129):
        for k in K_DENSE:
            for n in (ns[(d + k) % len(ns)], ns[(d + 2 * k + 1) % len(ns)]):
                rc, got = _query(lib, d, k, n, sms)
                want = tc.layout(d, k, n, sms)
                assert want is not None and rc == 0 and got == want, (d, k, n, sms, rc, got, want)


@pytest.mark.parametrize("sms", [1, 7, 15, 16, 33, 200])
def test_layout_equals_library_odd_sm_counts(lib, sms):
    for d in (1, 9, 64, 65, 128):
        for k in (1, 17, 256, 257, 1349, 2697, 3841, 4096):
            for n in (1, 64 * 7 + 3, 300_000):
                rc, got = _query(lib, d, k, n, sms)
                want = tc.layout(d, k, n, sms)
                if want is None:          # more slices than SMs
                    assert rc == EUNSUPPORTED and tc.tc2_geom(k, d)["S"] > sms, (d, k, n, sms, rc)
                else:
                    assert rc == 0 and got == want, (d, k, n, sms, rc, got, want)


def test_layout_rejects(lib):
    assert _query(lib, 129, 10, 100, 132)[0] == EUNSUPPORTED
    assert _query(lib, 128, 4097, 100, 132)[0] == EUNSUPPORTED
    assert _query(lib, 0, 10, 100, 132)[0] == EUNSUPPORTED
    assert _query(lib, 64, 10, 0, 132)[0] == EINVAL
    assert _query(lib, 64, 10, 100, 0)[0] == EINVAL
    assert lib.bkm_debug_tc2_layout(64, 10, 100, 132, None) == EINVAL


def test_workspace_equals_library(lib):
    """bkm_workspace_bytes sizes for the device's SM count, or 132 without a device."""
    v = ctypes.c_int(0)
    sms = v.value if lib.bkm_device_info(0, ctypes.byref(v), None, None) == 0 else 132
    for d in (1, 8, 64, 128):
        for k in (1, 100, 256, 257, 1024, 4096):
            for n in (1, 4095, 4097, 100_000):
                got = ctypes.c_size_t(0)
                assert lib.bkm_workspace_bytes(n, d, k, BF16, ctypes.byref(got)) == 0
                assert got.value == tc.ws_layout(n, d, k, sms)["total"], (n, d, k)


# ------------------------------------------------------------------------------------------------ reach
@pytest.mark.parametrize("sms", tc.SM_COUNTS)
def test_cases_reach_every_limit(sms):
    cs = tc.cases(sms)
    L = {c["id"]: tc.lay(c["d"], c["k"], c["n"], sms) for c in cs}
    assert all(v is not None for v in L.values())
    # every MMA width, with padded columns (real columns of the slice < N) and full; NS < N where N allows it
    def real(c):
        return min(c["k"], tc.tc2_geom(c["k"], c["d"])["NS"])
    for N in (16, 32, 64, 128, 256):
        of_n = [c for c in cs if L[c["id"]]["N"] == N]
        assert any(real(c) < N for c in of_n) and any(real(c) == N for c in of_n), N
        if N >= 64:
            assert any(L[c["id"]]["NS"] < N for c in of_n), N
    # every S, with a last slice of one real column and with full slices; k = 4096
    for S in range(1, 17):
        ks = {c["k"] for c in cs if L[c["id"]]["S"] == S}
        assert 256 * S in ks and (S == 1 or 256 * (S - 1) + 1 in ks), S
    # a last slice of one real column: only k = 3841 (S = 16, NS = 256) has one
    last_real = {k: k - (tc.tc2_geom(k, 64)["S"] - 1) * tc.tc2_geom(k, 64)["NS"] for k in range(257, 4097)}
    assert [k for k, r in last_real.items() if r == 1] == [3841]
    assert any(c["k"] == 3841 for c in cs)
    # KB = 1 and 2, partial last K-steps, every d of the list
    assert {L[c["id"]]["KB"] for c in cs} == {1, 2}
    assert {1, 8, 9, 16, 63, 64, 65, 100, 127, 128} <= {c["d"] for c in cs}
    assert any(c["d"] % 16 for c in cs if L[c["id"]]["KB"] == 2)
    # every DS transition at every FPL, both sides; DS = 16 gives NB = RP_MAXB
    for dpad, fpl in ((32, 1), (64, 2), (128, 4)):
        for kt in tc.ds_transitions(dpad):
            for k in (kt - 1, kt):
                assert any(c["d"] == dpad and c["k"] == k and L[c["id"]]["FPL"] == fpl for c in cs), (dpad, k)
    assert tc.ds_transitions(128) == [338, 675, 1349, 2697]
    assert all(L[c["id"]]["NB"] == tc.RP_MAXB for c in cs if L[c["id"]]["DS"] == 16)
    assert {L[c["id"]]["DS"] for c in cs} == {1, 2, 4, 8, 16}
    # row counts: 1, 63, tiles = G - 1, G, G + 1, 2G, 2G + 1 (an idle warpgroup in group 0's last pair), with an S that
    # leaves SMs idle
    for d, k in ((128, 1280), (40, 200)):
        G = tc.lay(d, k, 1 << 30, sms)["G"]
        tiles = {-(-c["n"] // 64) for c in cs if (c["d"], c["k"]) == (d, k) and c["id"].startswith("rows")}
        assert {1, G - 1, G, G + 1, 2 * G, 2 * G + 1} <= tiles, (d, k, G, tiles)
    assert sms % tc.tc2_geom(1280, 128)["S"] != 0
    # the binning kernel's second turn holds exactly one row
    big = [c for c in cs if c["id"] == "bin-turn2"][0]
    Lb = L["bin-turn2"]
    assert Lb["bin_grid"] == 4 * sms and -(-big["n"] // tc.RP_TILE) == 4 * sms + 1 and big["n"] % tc.RP_TILE == 1
    # deferred counts at the re-check's turn boundaries, for S = 1 and S > 1
    R = tc.lay(64, 300, 10_000, sms)["recheck_grid"]
    for S in (1, 16):
        nds = {c["n_defer"] for c in cs if c["n_defer"] is not None and tc.tc2_geom(c["k"], c["d"])["S"] == S}
        assert {0, 1, 16, 17, 16 * R - 1, 16 * R, 16 * R + 1} <= nds, (S, nds)
    # ... the S = 16 ones with a duplicate at every reduction level of the re-check
    dup = {(a, b) for a, b, kind in tc.centres(4096, 64)[1] if kind == "dup"}
    assert dup == {(48, 49), (50, 82), (52, 308), (54, 3894)}


@pytest.mark.parametrize("sms", tc.SM_COUNTS)
def test_tile_dealing(sms):
    """The restated dealing stages every (slice, tile) exactly once, and at 2G + 1 tiles group 0's last pair has
    warpgroup 1 idle.  This checks the restatement; the GPU cases at those tile counts check the kernel's own
    dealing."""
    for d, k in ((128, 1280), (40, 200), (128, 4096)):
        G = tc.lay(d, k, 1 << 30, sms)["G"]
        S = tc.tc2_geom(k, d)["S"]
        for tiles in (1, G - 1, G, G + 1, 2 * G, 2 * G + 1):
            n = 64 * tiles - 5
            deal = tc.dealing(d, k, n, sms)
            seen = sorted((s, row0) for _, s, _, _, _, _, row0 in deal)
            assert seen == sorted((s, 64 * t) for s in range(S) for t in range(tiles)), (d, k, tiles)
            if tiles == 2 * G + 1:
                g0 = [x for x in deal if x[2] == 0 and x[1] == 0]
                assert len(g0) == 3 and g0[-1][4] == 0 and g0[-1][5] == 1      # pair 1: warpgroup 0 only


# ------------------------------------------------------------------------------------------------ designed data
def _bf16_exact(a):
    a32 = np.asarray(a, dtype=np.float32)
    return np.array_equal(a32.view(np.uint32) & 0xFFFF, np.zeros(a32.shape, dtype=np.uint32)) and \
        np.array_equal(a32.astype(np.float64), np.asarray(a))


DESIGNS = [(128, 4096), (64, 3841), (128, 1280), (128, 257), (100, 300), (65, 129), (9, 128), (8, 64), (16, 33),
           (1, 2), (128, 1), (64, 17)]


@pytest.mark.parametrize("d,k", DESIGNS, ids=["d%d-k%d" % s for s in DESIGNS])
def test_design_is_exact(d, k):
    n = 700
    X, C, lab, deferred, kinds = tc.design(d, k, n, seed=d + k)
    assert X.shape == (n, d) and C.shape == (k, d)
    # bf16-exact rows and centres; -2 c is its own bf16 hi, so lo = 0
    assert _bf16_exact(X) and _bf16_exact(C) and _bf16_exact(-2.0 * C)
    assert set(np.unique(X)) <= {0.0, 0.5, 1.0, 2.0 ** -10, 2.0 ** -9}
    assert set(np.unique(C)) <= {0.0, 1.0, 2.0 ** -9}
    # every product and partial sum of x (-2 c), and ||c||^2 - 2 x.c, on the 2^-18 grid below 2^6
    cn = (C * C).sum(1)
    assert np.all(np.mod(cn * 2.0 ** 18, 1.0) == 0) and cn.max() < 64
    rows = np.concatenate([np.nonzero(kinds != "far")[0][:48], np.nonzero(kinds == "far")[0][:16]])
    for j0 in range(0, k, 256):                           # in column blocks: the products of 64 rows
        P = X[rows, None, :] * (-2.0 * C[None, j0:j0 + 256, :])
        part = np.cumsum(P, axis=2)
        for v in (P, part, cn[None, j0:j0 + 256] + part[:, :, -1]):
            assert np.all(np.abs(v) < 64) and np.all(np.mod(v * 2.0 ** 18, 1.0) == 0)
    e = cn[None, :] - 2.0 * (X @ C.T)
    # labels = the float64 arg-min (lowest index on exact ties) of the direct distances
    d2 = np.stack([((X - C[j]) ** 2).sum(1) for j in range(k)], 1)
    assert np.array_equal(lab, d2.argmin(1))
    assert np.array_equal(lab, e.argmin(1))
    # the kernel rules on every row agree with the design's far-row shortcut
    g = tc.tc2_geom(k, d)
    lab2, def2 = tc.decide(X, C, k, d, g["NS"], g["S"])
    assert np.array_equal(lab2, lab) and np.array_equal(def2, deferred)
    bound = tc.tau(d) * ((X * X).sum(1) + (C * C).sum(1).max())
    srt = np.sort(e, axis=1)
    gap = srt[:, 1] - srt[:, 0] if k > 1 else np.full(n, np.inf)
    near = np.isin(kinds, ["near-a", "near-b"])
    tie = np.isin(kinds, ["equal", "dup"])
    assert np.all((gap[near] > 0) & (gap[near] < bound[near]))
    assert np.all(gap[near] == 2.0 ** -18)
    assert np.all(gap[tie] == 0)
    far = ~(near | tie) & (kinds != "inner-losing")
    assert np.all(gap[far] >= 16 * bound[far]) and np.all(gap[far] >= 1)
    assert np.array_equal(deferred, near | tie)
    # inner-losing rows: the winner alone by >= 1, and a near-tie in the slice that holds the pair
    il = kinds == "inner-losing"
    assert np.all(gap[il] >= 16 * bound[il])
    if g["S"] > 1 and k >= 257 and d >= 64:
        assert il.any() and (near.sum() > 0) and tie.any()
    assert bound.max() < 1e-3 and tc.tau(d) > 2.0 ** -17


def test_design_slice_kinds():
    """At k = 4096 the special rows include, for every slice border, near-ties in both orders and the exact tie;
    the last column's pair with slice 0; inner-losing rows; and duplicates at every re-check reduction level."""
    d, k = 128, 4096
    C, plan, bits, E, T = tc.centres(k, d)
    NS = tc.tc2_geom(k, d)["NS"]
    pairs = {(a, b) for a, b, kind in plan if kind == "pair"}
    for s in range(1, 16):
        assert (s * NS - 1, s * NS) in pairs
    assert (1, k - 1) in pairs
    for N in (256,):
        assert (N // 2 - 1, N // 2) in pairs
    assert {(a, b) for a, b, kind in plan if kind == "dup"} == {(48, 49), (50, 82), (52, 308), (54, 3894)}
    X, C, lab, deferred, kinds = tc.design(d, k, 4000, 3)
    for kind in ("near-a", "near-b", "equal", "dup", "inner-losing"):
        assert (kinds == kind).sum() > 0, kind


def test_dist_sum_reference():
    """dist_sum_ref adds exact values exactly, and its fold order is visible on values that round."""
    v = np.arange(5000) * 0.25
    assert tc.dist_sum_ref(v, 132) == float(v.sum())
    w = np.zeros(5000)
    w[0], w[1], w[2] = 1.0, 2.0 ** 53, -(2.0 ** 53)       # warps 0, 1, 2 of CTA 0: (1 + 2^53) - 2^53 = 0
    assert tc.dist_sum_ref(w, 132) == 0.0


@pytest.mark.parametrize("sms", tc.SM_COUNTS)
def test_slice_cases_label_every_column(sms):
    """Every slice-count case has a far row, decided on the tensor path, at every column but the duplicates' (the
    last slice's single column at k = 3841 included), and at k = 3841 that column is paired with slice 0."""
    for c in tc.cases(sms):
        if not c["id"].startswith("S"):
            continue
        X, C, lab, deferred, kinds = tc.design(c["d"], c["k"], c["n"], seed=1)
        dup = {x for a, b, kind in tc.centres(c["k"], c["d"])[1] if kind == "dup" for x in (a, b)}
        far = (kinds == "far") & ~deferred
        assert set(lab[far].tolist()) == set(range(c["k"])) - dup, c["id"]
    plan = tc._pair_plan(3841, 128)
    assert (1, 3840, "pair") in plan and not any(3840 in p[:2] for p in plan if p[:2] != (1, 3840))
    X, C, lab, deferred, kinds = tc.design(128, 3841, 4000, seed=2)
    for kind in ("near-a", "near-b", "equal"):
        assert ((kinds == kind) & np.isin(lab, [1, 3840])).any(), kind
