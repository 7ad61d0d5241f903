"""The CUDA-core Nystrom and transform cases and the numpy restatement of their host rules (tests/simt_pass_cases.py),
without a GPU: the limits each case reaches for an H100 SXM (132 SMs) and an H100 PCIe (114 SMs), so that an edit to the
cases cannot quietly lose one; the exact-data claims; and the restated routing against the library's own answer where
it gives one without a device."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import simt_pass_cases as sc  # noqa: E402

DTS = ("f32", "f64")


def _embed(dt, sms, n=1):
    return {name: (d, l, kw, sc.nystrom_geom(1, n, d, l, kw, dt, sms)) for name, d, l, kw in sc.embed_shapes(dt)}


def _colsum(dt, sms, n=1):
    return {name: (d, l, sc.nystrom_geom(0, n, d, l, 0, dt, sms)) for name, d, l in sc.colsum_shapes(dt)}


# ---------------------------------------------------------------------------------------------------------------------
# the restated rules
# ---------------------------------------------------------------------------------------------------------------------
def test_budget_edges_and_rounding():
    # nw = 8: 25600 bytes per warp, 3200 fp64 or 6400 fp32 elements; an odd fp64 total rounds up by 8 bytes
    assert sc.first_blocked_total("f64") == 3201 and sc.first_blocked_total("f32") == 6401
    assert sc.nystrom_smem(1, 8, 3191, 4, 4, 8) == sc.nystrom_smem(1, 8, 3192, 4, 4, 8) == sc.BUDGET
    assert sc.nystrom_smem(1, 8, 6393, 4, 1, 4) == sc.nystrom_smem(1, 8, 6395, 4, 1, 4) == sc.BUDGET
    assert sc.nystrom_smem(1, 8, 6396, 4, 1, 4) == sc.BUDGET + 8 * 16
    # d4 rounds d up to 4; the COLSUM sums add nw lb float64 elements, rounded to 16 bytes
    assert [sc.d4_of(d) for d in (1, 4, 5, 8, 9)] == [4, 4, 8, 8, 12]
    assert sc.nystrom_smem(0, 1, 33, 4, 0, 8) == 272 + sc.nystrom_smem(1, 1, 33, 4, 0, 8)
    # each row tile at its first d4: 64 rows up to d4 = 396 (fp64) / 796 (fp32), then halving with every doubling of d4
    assert [sc.first_d_of_tr(t, "f64") for t in (32, 16, 8, 4, 2, 1)] == [400, 800, 1600, 3200, 6400, 12800]
    assert [sc.first_d_of_tr(t, "f32") for t in (32, 16, 8, 4, 2, 1)] == [800, 1600, 3200, 6400, 12800, 25600]
    for dt in DTS:
        for t in (32, 16, 8, 4, 2, 1):
            d = sc.first_d_of_tr(t, dt)
            assert sc.transform_geom(1, d - 4, 1, dt, 132).TR == 2 * t and sc.transform_geom(1, d, 1, dt, 132).ok
    # the widest rows either pass supports: the transform at TR = 1 and EMBED at nw = 1, lb = 32 stay within 227 KB
    assert sc.transform_geom(1, 58104, 1, "f32", 132).ok and not sc.transform_geom(1, 58105, 1, "f32", 132).ok
    assert sc.transform_geom(1, 29052, 1, "f64", 132).ok and not sc.transform_geom(1, 29053, 1, "f64", 132).ok
    assert not sc.nystrom_geom(1, 1, 29040, 300, 3, "f64", 132).ok


@pytest.mark.parametrize("sms", sc.SMS)
def test_grid_and_turns(sms):
    for nw in (8, 4, 2, 1):
        d = sc.d_for_nw(1, "f64", nw, 300, 3)
        for n in sc.row_counts(nw, sms):
            g = sc.nystrom_geom(1, n, d, 300, 3, "f64", sms)
            assert g.nw == nw
            if n <= 4 * sms * nw:
                assert g.grid == -(-n // nw) and g.turns == 1
            else:
                assert g.grid == 4 * sms and g.turns == 2 and g.last_turn == 1
        assert sc.row_counts(nw, sms)[:-1] == sorted({1, max(nw - 1, 1), nw + 1})


# ---------------------------------------------------------------------------------------------------------------------
# the cases reach every limit
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sms", sc.SMS)
@pytest.mark.parametrize("dt", DTS)
def test_embed_cases_reach_every_limit(dt, sms):
    t = sc.first_blocked_total(dt)
    c = _embed(dt, sms)
    for kw in (1, 32, 33, 65):
        d, l, _, g = c["fits_kw%d" % kw]
        assert sc.d4_of(d) + l + kw == t - 1 and g.one and g.nw == 8
        d, l, _, g = c["blocked_kw%d" % kw]
        assert sc.d4_of(d) + l + kw == t and not g.one and g.nw == 8 and g.blocks == 2
    d, l, kw, g = c["lb1024_last1"]
    assert (g.nw, g.lb, g.blocks, g.last) == (8, 1024, 3, 1)
    for r in (31, 32, 33):
        # lb = 1024 after five halvings, 31 full blocks and a last block of r rows; one output fewer and the chain stops
        # at 2016
        d, l, kw, g = c["lb1024_last%d" % r]
        assert (g.nw, g.lb, g.blocks, g.last) == (8, 1024, 32, r)
        assert sc.lb1024_chain(l) == [l, 15904, 7968, 4000, 2016, 1024]
        assert sc.nystrom_geom(1, 1, d, l, kw - 1, dt, sms).lb == 2016
        d, l, kw, g = c["nw1_last%d" % r]
        assert g.last == r and g.lb < 1024 and g.nw == 1 and g.blocks == 2
    assert {g.nw for _, _, _, g in c.values()} == {8, 4, 2, 1}
    for nw in (4, 2, 1):
        assert c["nw%d" % nw][3].nw == nw and c["nw%d" % nw][3].one
    d, l, kw, g = c["nw1_halved"]
    assert g.nw == 1 and g.lb < l < 1024 and not g.one
    assert all(g.ok for _, _, _, g in c.values())
    # the exact data stays exact: every squared distance and norm below 2^24
    for d, l, kw, g in c.values():
        assert sc.exact_bound(sc.keep_radius(l, d), d) < 2 ** 24
    # every n at its grid: one row, a partial and a full CTA, and one row in the second grid turn
    for d, l, kw, g in c.values():
        ns = sc.row_counts(g.nw, sms)
        turns = [sc.nystrom_geom(1, n, d, l, kw, dt, sms) for n in ns]
        assert turns[-1].turns == 2 and turns[-1].last_turn == 1 and turns[-1].grid == 4 * sms
        assert ns[0] == 1


@pytest.mark.parametrize("sms", sc.SMS)
@pytest.mark.parametrize("dt", DTS)
def test_colsum_cases_reach_every_limit(dt, sms):
    c = _colsum(dt, sms)
    launches = {name: g.launches for name, (_, _, g) in c.items()}
    assert launches["one"] == 1 and launches["two"] == 2 and launches["many"] >= 16
    assert c["last1"][2].last == 1 and c["last1"][2].launches == 3
    assert {g.nw for _, _, g in c.values()} == {8, 4, 2, 1}
    g = c["nw1_two"][2]
    assert g.nw == 1 and g.launches == 2
    for d, l, g in c.values():
        assert g.ok and sc.exact_bound(sc.keep_radius(l, d), d) < 2 ** 24
        last = sc.nystrom_geom(0, sc.row_counts(g.nw, sms)[-1], d, l, 0, dt, sms)
        assert last.turns == 2 and last.last_turn == 1


@pytest.mark.parametrize("sms", sc.SMS)
@pytest.mark.parametrize("dt", DTS)
def test_transform_cases_reach_every_tile(dt, sms):
    shapes = sc.transform_shapes(dt)
    tiles = set()
    for name, d, k in shapes:
        g = sc.transform_geom(1, d, k, dt, sms)
        n = sc.transform_rows(g.TR, sms)
        g = sc.transform_geom(n, d, k, dt, sms)
        tiles.add(g.TR)
        assert g.ok and g.last_rows == 1 and g.ntiles > g.grid == 4 * sms and k % 4
        assert 36 * d < 2 ** 24                                    # exact: integers in [-3, 3]
    assert tiles == {64, 32, 16, 8, 4, 2, 1}
    assert {d % 4 for _, d, _ in shapes} == {0, 1}


def test_reference_matrices_stay_small():
    """The random-data tests hold n x l float64 matrices: near 100 MiB at most."""
    import test_gpu_simt_passes as t

    for c in t.COLSUM_REF:
        assert c[1] * c[3] * 8 <= 100 * 2 ** 20
    for c in t.EMBED_REF:
        assert c[1] * c[3] * 8 <= 100 * 2 ** 20
    for c in t.TRANSFORM_REF:
        assert c[1] * c[3] * 8 <= 100 * 2 ** 20


# ---------------------------------------------------------------------------------------------------------------------
# the exact data
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d,l", [(4, 3000), (5, 300), (40, 200), (2104, 60)])
def test_exact_rows(d, l):
    keep = sc.keep_rows(l, d, seed=1)
    X, kind, j = sc.exact_rows(keep, 700, seed=2)
    assert keep.dtype == np.int8 and (keep % 2 == 0).all() and len(np.unique(keep, axis=0)) == l
    K, Xf = keep.astype(np.float64), X.astype(np.float64)
    d2 = (Xf * Xf).sum(1)[:, None] - 2.0 * Xf @ K.T + (K * K).sum(1)[None]
    kk = (K * K).sum(1)[:, None] - 2.0 * K @ K.T + (K * K).sum(1)[None]
    assert kk[~np.eye(l, dtype=bool)].min() >= 4                     # distinct keep rows: at least 4 apart
    m = d2.min(1)
    assert (m[kind == sc.COPY] == 0).all() and (m[kind == sc.NEAR] == 1).all() and (m[kind == sc.ODD] >= d).all()
    assert (d2[kind == sc.COPY, j[kind == sc.COPY]] == 0).all()
    # COLSUM at GAMMA_COUNT: 1 for a copy, an underflow for every other pair, in fp32 and fp64
    assert np.exp(np.float32(-sc.GAMMA_COUNT)) == 0 and np.exp(-sc.GAMMA_COUNT) == 0
    # EMBED: gamma m either side of 745.13 at m = 1, and nothing but the nearest keep rows survive the shift
    assert sc.GAMMA_LO * 1.0 <= 745.13 < sc.GAMMA_HI * 1.0
    assert np.exp(-sc.GAMMA_LO * 3.0) == 0 and np.exp(np.float32(-sc.GAMMA_LO)) == 0
    W = sc.signed_one_hot(l, 7, seed=3)
    assert (np.abs(W).sum(1) == 1).all()
    assert X[0].tobytes() == keep[-1].tobytes() and X[-1].tobytes() == keep[0].tobytes()


# ---------------------------------------------------------------------------------------------------------------------
# routing
# ---------------------------------------------------------------------------------------------------------------------
def test_routing():
    assert sc.route("transform", "f32", 64, 256) == ("tc", False)
    assert sc.route("transform", "f32", 65, 7) == ("simt", False)
    assert sc.route("colsum", "f32", 64, 257) == ("simt", False)
    assert sc.route("embed", "f32", 64, 256, kw=64) == ("tc", False)
    assert sc.route("embed", "f32", 64, 256, kw=65) == ("simt", False)
    assert sc.route("colsum", "f64", 4, 7) == ("simt", False)
    assert sc.route("colsum", "f32", 5, 7, ldx=5) == ("simt", True)
    assert sc.route("transform", "f32", 5, 7, base_bytes=4, ldx=8) == ("simt", True)
    assert sc.route("embed", "f32", 5, 7, kw=3, force_simt=True, ldx=5) == ("simt", False)
    # every exact-data case runs on the CUDA cores
    for dt in DTS:
        for _, d, l, kw in sc.embed_shapes(dt):
            assert sc.route("embed", dt, d, l, kw=kw)[0] == "simt"
        for _, d, l in sc.colsum_shapes(dt):
            assert sc.route("colsum", dt, d, l)[0] == "simt"


def test_routing_matches_the_library():
    """bkm_kernel_family under FORCE_TC answers tc_supported for fp32 without a device."""
    from dask_ml_b200 import _lib

    try:
        lib = _lib.load()
    except (RuntimeError, OSError):
        pytest.skip("the library is not built")
    for d in (1, 4, 5, 63, 64, 65, 800):
        for k in (1, 7, 255, 256, 257, 6000):
            fam = lib.bkm_kernel_family(d, k, _lib.BKM_F32, _lib.FLAG_FORCE_TC)
            assert (fam == 1) == sc.tc_supported(d, k, "f32"), (d, k, fam)
            assert lib.bkm_kernel_family(d, k, _lib.BKM_F64, _lib.FLAG_FORCE_TC) < 0
