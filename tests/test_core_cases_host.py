"""The CUDA-core chunk kernels' geometry and designed data without a GPU (tests/core_cases.py).

* The host restatement equals the library's own layout query (bkm_debug_core_layout) over a sweep of d, k, row pitch,
  dtype, flags, entry point and base alignment that crosses every mode, row-tile and kernel switch; the workspace
  offsets equal bkm_workspace_bytes.
* The cases reach every limit: every streaming-kernel instance, every M-step pair stride, the k = 24 / 25 and pitch
  32 / 33 switches and the fallbacks, J padding, SMALLK, both sides of the SMEM / GLOBAL boundary of both entries, the
  row tiles, and exact ties at every level of the re-check.
* The designed data is what it claims: in the lattice cases every product and partial sum the fp32 kernels form is an
  integer below 2^24; in the near-tie cases the two best distances are small integers 1 apart, exact in float64 and in
  the fp32 direct form, inside the re-check bound, every other centre is far outside it, and on the generic kernel the
  fp32 E-step without the re-check (emulated bit for bit) mislabels at least one of them.
"""
import ctypes

import numpy as np
import pytest

import core_cases as cc

EUNSUPPORTED, EINVAL, EDTYPE = -3, -1, -2


@pytest.fixture(scope="module")
def lib():
    from dask_ml_b200 import _lib

    return _lib.load()


def _query(lib, d, k, ldx, dtype, flags, mstep, aligned16):
    out = (ctypes.c_int * len(cc.FIELDS))()
    rc = lib.bkm_debug_core_layout(int(d), int(k), int(ldx), int(dtype), int(flags), int(mstep), int(aligned16), out)
    return rc, tuple(out)


def _check(lib, d, k, ldx, dtype, flags, mstep, aligned16):
    rc, got = _query(lib, d, k, ldx, dtype, flags, mstep, aligned16)
    want = cc.layout(d, k, ldx, dtype, flags, mstep, aligned16)
    if want is None:
        assert rc == EUNSUPPORTED, (d, k, ldx, dtype, flags, mstep, aligned16, rc)
    else:
        assert rc == 0 and got == want, (d, k, ldx, dtype, flags, mstep, aligned16, rc, got, want)
    return want


def test_layout_equals_library_small(lib):
    """Every d <= 20, k <= 40 at every pitch up to 70, both dtypes, both entries, aligned or not, with and without
    FORCE_SIMT: every streaming instance and fallback, J, SMALLK."""
    kinds = set()
    for d in range(1, 21):
        for k in range(1, 41):
            for ldx in sorted({d, d + 1, (d + 3) // 4 * 4, 32, 33, 56, 57, 64, 65, 70} - set(range(d))):
                for dtype in (cc.F32, cc.F64):
                    for flags in (0, cc.FORCE_SIMT):
                        for mstep in (1, 0):
                            w = _check(lib, d, k, ldx, dtype, flags, mstep, (d + k + ldx) % 5 != 0)
                            if w:
                                kinds.add(w[0])
    assert kinds == {cc.GENERIC, cc.ONE_ROW, cc.TWO_ROW}


def test_layout_equals_library_wide(lib):
    """Wide rows and many centres: every row-tile step from 256 down to 1, both sides of the SMEM / GLOBAL boundary."""
    rts = {cc.F32: set(), cc.F64: set()}
    modes = set()
    for dtype in (cc.F32, cc.F64):
        for d in list(range(60, 2000, 7)) + list(range(2000, 30001, 397)):
            for k in (1, 4, 9, 33):
                w = _check(lib, d, k, d, dtype, 0, (d + k) % 2, 1)
                if w:
                    rts[dtype].add(w[4])
        for d in (65, 96, 128, 300):
            for k in range(1, 1200, 13):
                for mstep in (1, 0):
                    w = _check(lib, d, k, d, dtype, 0, mstep, 1)
                    modes.add((dtype, mstep, w[2]))
            for mstep in (1, 0):
                kb = cc.global_boundary(d, dtype, mstep)
                for k in (kb - 1, kb):
                    _check(lib, d, k, d, dtype, 0, mstep, 1)
    for dtype in rts:
        assert {256, 224, 192, 160, 128, 96, 64, 32, 16, 8, 4, 2, 1} <= rts[dtype], sorted(rts[dtype])
    assert {(t, m, g) for t in (0, 1) for m in (0, 1) for g in (0, 1)} == modes


def test_layout_rejects(lib):
    assert _query(lib, 64, 256, 64, cc.F32, 0, 1, 1)[0] == EUNSUPPORTED          # tensor path
    assert _query(lib, 13, 20, 16, cc.F32, cc.FORCE_TC, 1, 0)[0] == EUNSUPPORTED  # forced tensor path: no fallback
    assert _query(lib, 64, 256, 64, cc.F32, 0, 1, 0)[0] == 0                      # ... misaligned: the generic kernel
    assert _query(lib, 16, 10, 16, 2, 0, 1, 1)[0] == EUNSUPPORTED                 # bf16 rows
    assert _query(lib, 16, 10, 16, 7, 0, 1, 1)[0] == EDTYPE
    assert _query(lib, 16, 10, 15, cc.F32, 0, 1, 1)[0] == EINVAL
    assert _query(lib, 0, 10, 16, cc.F32, 0, 1, 1)[0] == EINVAL
    assert lib.bkm_debug_core_layout(16, 10, 16, 0, 0, 1, 1, None) == EINVAL


def test_workspace_equals_library(lib):
    v = ctypes.c_int(0)
    sms = v.value if lib.bkm_device_info(0, ctypes.byref(v), None, None) == 0 else 132
    for dtype in (cc.F32, cc.F64):
        for d in (1, 13, 100, 20000):
            for k in (1, 20, 300, 1000):
                for n in (1, 4097, 100_000):
                    got = ctypes.c_size_t(0)
                    assert lib.bkm_workspace_bytes(n, d, k, dtype, ctypes.byref(got)) == 0
                    assert got.value == cc.ws_layout(n, d, k, dtype, sms)["total"], (n, d, k, dtype)


# ------------------------------------------------------------------------------------------------ reach
def _plans(c):
    return {m: cc.plan(c["d"], c["k"], c["pitch"], c["dtype"], c["flags"], m, c["base_off"] == 0) for m in (1, 0)}


def test_cases_reach_every_limit():
    cs = cc.cases()
    assert len({c["id"] for c in cs}) == len(cs)
    P = {c["id"]: _plans(c) for c in cs}
    assert all(p is not None for ps in P.values() for p in ps.values())
    lloyd = [(c, P[c["id"]][1]) for c in cs]
    assign = [(c, P[c["id"]][0]) for c in cs]
    # every streaming instance, both entries
    for entries in (lloyd, assign):
        two = {(p["DH"], p["KB"]) for c, p in entries if p["kernel"] == cc.TWO_ROW}
        one = {(p["DH"], p["KB"]) for c, p in entries if p["kernel"] == cc.ONE_ROW}
        assert two == {(dh, kc) for dh in (2, 4, 6, 7, 8) for kc in range(4, 25, 4)}
        assert one == {(dh, kpt) for dh in (2, 4, 6, 7, 8) for kpt in range(2, 17, 2)}
    # every msS class, pitches 4, 12, 20, 28 at k <= 24
    mss = {p["msS"] for c, p in lloyd if p["kernel"] == cc.TWO_ROW}
    assert mss == {1, 2, 4, 8, 16}
    assert {4, 12, 20, 28} <= {c["pitch"] for c, p in lloyd if p["kernel"] == cc.TWO_ROW and c["k"] <= 24}
    # the switches and fallbacks
    kern = {c["id"]: p["kernel"] for c, p in lloyd}
    assert kern["k24-L16"] == cc.TWO_ROW and kern["k25-L16"] == cc.ONE_ROW
    assert kern["d13-k20-L32"] == cc.TWO_ROW and kern["d13-k20-L33"] == cc.ONE_ROW
    assert kern["d13-k20-L56"] == cc.GENERIC and kern["d13-k20-L65"] == cc.GENERIC   # ring too large, pitch > 64
    assert kern["misaligned-d13-k20"] == cc.GENERIC and kern["misaligned-d41-k100"] == cc.GENERIC
    assert {c["k"] for c in cs if cc.kernel_family(c["d"], c["k"], c["dtype"], c["flags"]) == 2} >= {1}
    # generic: both dtypes, k = 0, 1, J - 1 mod J for J = 8 and 16, SMALLK both sides
    gen = [(c, p) for c, p in lloyd if p["kernel"] == cc.GENERIC]
    for dtype in (cc.F32, cc.F64):
        for J in ((8, 16) if dtype == cc.F32 else (8,)):
            ks = {c["k"] % J for c, p in gen if p["J"] == J and c["dtype"] == dtype and c["k"] > J}
            # fp32 takes J = 16 only where it pads no more than J = 8: k = 1 mod 16 runs on J = 8 blocks
            assert ({0, 1, J - 1} if J == 8 else {0, J - 1}) <= ks, (dtype, J, ks)
        if dtype == cc.F32:
            assert {p["J"] for c, p in gen if c["dtype"] == dtype and c["k"] % 16 == 1 and c["k"] > 16} == {8}
        sk = {(c["d"], c["k"]): p["SMALLK"] for c, p in gen if c["dtype"] == dtype}
        assert sk[(16, 32)] == 1 and sk[(16, 33)] == 0 and sk[(17, 32)] == 0
        for entries, m in ((lloyd, 1), (assign, 0)):
            kb = cc.global_boundary(96, dtype, m)
            g = {c["k"]: p["GLOBAL"] for c, p in entries if c["d"] == 96 and c["dtype"] == dtype
                 and c["id"].startswith("global")}
            assert g.get(kb - 1) == 0 and g.get(kb) == 1, (dtype, m, g)
        rts = {p["rt"] for c, p in assign if p["kernel"] == cc.GENERIC and c["dtype"] == dtype}
        assert {256, 160, 32, 16, 2, 1} <= rts, rts
    # rt < 4 with an odd pitch: the flat 16-byte staging holds for some tiles and not for others
    for c, p in assign:
        if p["kernel"] == cc.GENERIC and p["rt"] < 4 and c["id"].startswith("rt"):
            esz = 8 if c["dtype"] == cc.F64 else 4
            flat = {(r0 * c["pitch"] * esz) % 16 == 0 for r0 in range(0, c["n"], p["rt"])}
            if p["rt"] * esz < 16:
                assert c["pitch"] % 2 == 1 and flat == {True, False}, c["id"]
    # FORCE_SIMT on a family-1 and a family-2 shape
    assert cc.kernel_family(64, 256, cc.F32) == 1 and cc.kernel_family(13, 20, cc.F32) == 2
    assert {"force-simt-d64-k256", "force-simt-d13-k20"} <= set(P)
    # ties at every level of the generic re-check (k = 300, J = 16 for fp32, 8 for float64)
    t = dict(cc.GENERIC_TIES)
    assert t[3] == 5 and 6 // 16 != 21 // 16 and 40 // 32 != 140 // 32 and 263 - 256 == 7
    assert (261 - 256) // 32 < 100 // 32
    # near-tie cases on every kernel
    near = {P[c["id"]][1]["kernel"] for c in cs if c["data"] == "near"}
    assert near == {cc.GENERIC, cc.ONE_ROW, cc.TWO_ROW}


# ------------------------------------------------------------------------------------------------ designed data
def _fp32_direct(X, C, lab):
    """sum (x - c)^2 in fp32, feature by feature"""
    s = np.zeros(X.shape[0], dtype=np.float32)
    for i in range(X.shape[1]):
        df = X[:, i].astype(np.float32) - C[lab, i].astype(np.float32)
        s = (s + df * df).astype(np.float32)
    return s


@pytest.mark.parametrize("cid", [c["id"] for c in cc.cases()])
def test_design_is_exact(cid):
    c = {c["id"]: c for c in cc.cases()}[cid]
    X, C, near = cc.design(c)
    n, d, k = c["n"], c["d"], c["k"]
    assert X.shape == (n, d) and C.shape == (k, d)
    assert np.array_equal(X, np.round(X)) and np.array_equal(C, np.round(C))
    lab, d2 = cc.reference(X, C)
    # the float64 reference is exact: it equals the direct form on every row
    rows = np.arange(n)[:: max(1, n // 300)]
    for i in rows:
        e = ((X[i] - C) ** 2).sum(1)
        assert e.argmin() == lab[i] and e[lab[i]] == d2[i], (cid, i)
    assert np.array_equal(_fp32_direct(X, C, lab).astype(np.float64), d2)
    for a, b in c["ties"]:
        if b < k:
            assert np.array_equal(C[a], C[b]) and (lab == a).any() and not (lab == b).any(), (a, b)
    absX, absC = np.abs(X), np.abs(C)
    if c["data"] == "lattice":
        # every product x_i c_i, every partial dot product, ||x||^2, ||c||^2, every distance and every column sum of a
        # cluster: integers below 2^24 (exact in fp32 in any order)
        lim = 2.0 ** 24
        assert (absX @ absC.T).max() < lim and (absX ** 2).sum(1).max() < lim and (absC ** 2).sum(1).max() < lim
        assert d2.max() < lim and absX.sum(0).max() < lim
    else:
        cn = (C * C).sum(1)
        scale = (X * X).sum(1) + cn.max()
        assert scale.min() >= 2.0 ** 25
        bound = cc.tau(d) * scale
        srt = np.sort(np.stack([((X[i] - C) ** 2).sum(1) for i in range(n)]), 1)
        gap = srt[:, 1] - srt[:, 0]
        pair_rows = near & (srt[:, 1] > 0)
        assert pair_rows.sum() >= 16 * len(c["pairs"]) and np.all(gap[pair_rows] == 1)
        # rows with their own fp32 rounding (w in {-1, 0, 1}^(d - 1): fewer of them at d = 3)
        assert len(np.unique(X[pair_rows], axis=0)) >= min(12, 3 ** (d - 1) // 2) * len(c["pairs"])
        assert np.all(gap[pair_rows] < bound[pair_rows] / 16)
        # the winner of a near-tie row is the higher index of its pair
        for a, b in c["pairs"]:
            assert (pair_rows & (lab == b)).any() and not (pair_rows & (lab == a)).any()
        # every row's two best centres are a designed pair or duplicate (gap far inside the bound) or alone (far
        # outside it), and the third is far outside it
        third = srt[:, 2] if k > 2 else np.full(n, np.inf)
        assert np.all((gap < bound / 16) | (gap > 16 * bound)) and np.all(third - srt[:, 0] > 16 * bound)
        # the data depends on the re-check: the generic kernel's fp32 E-step alone gets a near-tie row wrong
        if cc.plan(d, k, c["pitch"], c["dtype"], c["flags"], False)["kernel"] == cc.GENERIC:
            assert (cc.generic_fp32_argmin(X, C)[pair_rows] != lab[pair_rows]).any(), cid
        # sums of the rows stay below 2^24 in fp32 (every partial of a cluster)
        assert absX.sum(0).max() < 2.0 ** 24
