"""The column-block cases and the numpy restatement of their host rules and fold (tests/colpass_cases.py), without a GPU:
the limits each case reaches for an H100 SXM (132 SMs) and an H100 PCIe (114 SMs), the exact-square property and the
order sensitivity of every case (the restated fold gives other bits with the row groups or the CTAs reversed), the
fold against the existing numpy backends of the scalers, the imputer and the metrics, and the workspace sizes."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import colpass_cases as cc  # noqa: E402

SMS = [132, 114]


def _differs(a, b):
    return np.asarray(a).tobytes() != np.asarray(b).tobytes()


# ---------------------------------------------------------------------------------------------------------------------
# limits
# ---------------------------------------------------------------------------------------------------------------------
def test_widths_reach_every_column_block_with_and_without_spare_threads():
    cbs = {cc.col_block(d) for d in cc.WIDTHS}
    assert sorted(cbs) == [32, 64, 96, 128, 160, 192, 224, 256]
    assert {cb for cb in cbs if cc.spare(cb)} == {96, 160, 192, 224}
    # every block at its full width and one column past the block below it
    for cb in cbs:
        assert cb in cc.WIDTHS and (cb == 32 or cb - 31 in cc.WIDTHS)
    # one, two and three column passes
    assert {cc.cdiv(d, cc.col_block(d)) for d in cc.WIDTHS} == {1, 2, 3}
    # d = 65: CB = 96, G = 2, 64 spare threads; CB = 160 / 192 / 224: G = 1
    assert [(cc.KT // cc.col_block(d), cc.spare(cc.col_block(d))) for d in (65, 160, 192, 224)] == \
        [(2, 64), (1, 96), (1, 64), (1, 32)]


def test_metric_widths():
    gs = {cc.KT // cc.metric_cb(m, "err") for m in cc.METRIC_M}
    assert max(gs) == 256 and min(gs) == 1 and {128, 85, 51, 36, 3, 2} <= gs
    assert {cc.metric_cb(m, "err") % 32 for m in cc.METRIC_M} - {0}              # odd blocks
    assert cc.cdiv(257, cc.metric_cb(257, "err")) == 2 and 257 - 256 == 1          # a one-column second pass
    assert all(cc.metric_cb(m, "eq") == 1 for m in cc.METRIC_ROW_M)


@pytest.mark.parametrize("sms", SMS)
def test_row_counts_reach_the_grid_limits(sms):
    for cap in (4, 8):
        capn = cap * sms
        for G in (1, 2, 3, 4, 8, 36, 51, 85, 128, 256):
            rows = cc.reduce_rows(G, cap, sms)
            grids = {lab: cc.reduce_grid(n, G, cap, sms) for lab, n in rows.items()}
            assert grids["0"] == grids["1"] == 1 and grids["16G+1"] == 2
            assert grids["cap-1"] == capn - 1 and grids["cap"] == capn == grids["past"]
            used, empty, last = cc.grid_facts(rows["cap"], G, capn)
            assert used == capn and last == 16 * G
            used, empty, last = cc.grid_facts(rows["past"], G, capn)
            if 16 * G < capn - 1:
                assert empty > 0, (G, cap)
            if "tail1" in rows:
                g = grids["tail1"]
                assert g <= capn and cc.grid_facts(rows["tail1"], G, g)[2] == 1
            else:
                assert 16 * G > capn
    # the example of a layout with one row group past the cap: 26 empty CTAs at 132 SMs
    assert cc.grid_facts(10033, 1, cc.reduce_grid(10033, 1, 4, 132))[1] == 26
    assert cc.grid_facts(cc.reduce_rows(1, 4, 132)["past"], 1, 528)[1] == 31


@pytest.mark.parametrize("sms", SMS)
def test_element_pass_rows_reach_the_cap(sms):
    for d in cc.WIDTHS:
        rows = cc.pass_rows(d, sms)
        assert cc.col_pass_grid(rows["1"], d, sms) == 1 and cc.col_pass_grid(rows["8G+1"], d, sms) == 2
        assert cc.col_pass_grid(rows["cap"], d, sms) == 8 * sms == cc.col_pass_grid(rows["past"], d, sms)
        assert rows["past"] % (8 * sms) != 0


QT_NQ = {"f32": [1365, 1366, 341, 342, 682, 683], "bf16": [1365, 1366, 341, 342, 682, 683],
         "f64": [2457, 2458, 614, 615, 1228, 1229]}


def qt_ds(dt):
    cs = cc.QCS[dt]
    return [cs - 1, cs, cs + 1, 1001]


@pytest.mark.parametrize("sms", SMS)
@pytest.mark.parametrize("dt", ["f32", "f64", "bf16"])
def test_quantile_transform_geometry(dt, sms):
    nq = QT_NQ[dt]
    geo = [cc.qtransform_geom(10 ** 6, 9, q, dt, sms) for q in nq]
    assert [g[1] for g in geo] == [True, False, True, True, True, True]           # the staged limit
    assert [g[2] for g in geo] == [2, 8, 8, 4, 4, 2]                              # the per-SM steps
    cs = cc.QCS[dt]
    assert [cc.qtransform_geom(10 ** 6, d, 100, dt, sms)[3] for d in qt_ds(dt)] == [1, 1, 2, cc.cdiv(1001, cs)]
    # gy: clamped by the rows (>= 8 per thread), by the per-SM budget, never below 1
    assert cc.qtransform_geom(1, 9, 100, dt, sms)[4] == 1
    assert cc.qtransform_geom(1000, 9, 100, dt, sms)[4] == cc.cdiv(1000, (256 // cs) * 8)
    g = cc.qtransform_geom(10 ** 7, 9, 100, dt, sms)
    assert g[4] == cc.cdiv(8 * sms, g[3])


def test_workspace_sizes():
    assert cc.partials_bytes(1, 7) == 256 + 256
    assert cc.partials_bytes(528, 7 * 513) == cc.cdiv(528 * 7 * 513 * 8, 256) * 256 + 256
    assert cc.pack_ws(8448, 257, 132) == 2304 + cc.partials_bytes(528, 514)
    assert cc.pack_ws(1, 1, 132) == 256 + 512
    assert cc.partials_bytes(cc.metric_grid(10 ** 7, 1, "eq", 132), 4) == cc.cdiv(1056 * 32, 256) * 256 + 256


# ---------------------------------------------------------------------------------------------------------------------
# exact squares and order sensitivity
# ---------------------------------------------------------------------------------------------------------------------
def _order_checks(run, G, grid, n):
    """Two operands add the same in either order: an order shows from three row groups, or three CTAs, with rows."""
    base = run()
    used = cc.grid_facts(n, G, grid)[0]
    if G >= 3 and cc.cta_rows(n, grid)[2] >= 3:
        assert _differs(base, run(rev_groups=True)), "row-group order not seen"
    if used >= 3:
        assert _differs(base, run(rev_ctas=True)), "CTA order not seen"
    return base


@pytest.mark.parametrize("shifted", [False, True], ids=["wide", "shifted"])
@pytest.mark.parametrize("dt", ["f32", "f64", "bf16"])
def test_colstats_and_impute_cases(dt, shifted):
    sms = 132
    for d in cc.WIDTHS:
        G = cc.KT // cc.col_block(d)
        for lab, n in cc.reduce_rows(G, 4, sms).items():
            if n * d > 3 * 10 ** 6 or n < 2:
                continue
            X, s = cc.stat_case(n, d, dt, sms, 4, seed=n + d, shifted=shifted)
            grid = cc.reduce_grid(n, G, 4, sms)
            assert cc.short_ok(X - (0.0 if s is None else s))
            if shifted:                          # squares of short integers round in their last bits only
                cc.colstats_fold(X, s, G, grid)
            else:
                _order_checks(lambda **kw: cc.colstats_fold(X, s, G, grid, **kw)[:2], G, grid, n)
            if not shifted:                      # the imputer's sums of short integers are exact in any order
                _order_checks(lambda **kw: cc.impute_fold(X, s, True, 0.0, G, grid, **kw)[3], G, grid, n)


@pytest.mark.parametrize("dt", ["f32", "f64", "bf16"])
def test_metric_err_cases(dt):
    sms = 132
    for m in cc.METRIC_M:
        G = cc.KT // cc.metric_cb(m, "err")
        for lab, n in cc.reduce_rows(G, 8, sms).items():
            if n < 2 or n * m > 2 * 10 ** 6:
                continue
            A, B = metric_err_case(n, m, dt, seed=n + m)
            grid = cc.metric_grid(n, m, "err", sms)
            assert cc.short_ok(B - A) and cc.short_ok(A)
            _order_checks(lambda **kw: cc.metric_err_fold(A, B, None, G, grid, **kw), G, grid, n)


def metric_err_case(n, m, dt, seed):
    """a = m1 2^k, b = m2 2^k on one exponent per element: b - a is short."""
    rng = np.random.RandomState(seed)
    k = rng.randint(-30, 31, (n, m))
    top = 1 << cc.MBITS[dt]
    A = np.ldexp(rng.randint(-top + 1, top, (n, m)).astype(np.float64), k)
    B = np.ldexp(rng.randint(-top + 1, top, (n, m)).astype(np.float64), k)
    return A, B


def test_metric_row_cases():
    sms = 132
    for m in cc.METRIC_ROW_M:
        for lab, n in cc.reduce_rows(256, 8, sms).items():
            if n < 2 or n * m > 4 * 10 ** 6:
                continue
            w = cc.wide(np.random.RandomState(n), n, "f64")
            grid = cc.metric_grid(n, m, "eq", sms)
            A = np.zeros((n, m))
            t = cc.eq_terms(A, A, w)
            _order_checks(lambda **kw: cc.metric_row_fold(t, w, 256, grid, **kw), 256, grid, n)


@pytest.mark.parametrize("sms", SMS)
def test_pack_cases(sms):
    for k in cc.PACK_K:
        G = cc.KT // cc.col_block(k)
        rows = cc.pack_rows(k, sms)
        assert cc.pack_grid_sparse(rows["cap"], k, sms) == 4 * sms
        if sms != 132:
            continue
        for lab, p in rows.items():
            if p * k > 10 ** 6 or p < 2:
                continue
            c = cc.pack_case(p, k, sms, seed=p + k)
            assert cc.short_ok(c.new) and cc.short_ok(c.ct_in - c.new) and cc.short_ok(c.C)
            grid = cc.pack_grid_sparse(p, k, sms)
            if k >= 32:                          # one column of positive sums can round alike in both orders
                _order_checks(lambda **kw: cc.pack_fold(c.new, c.ct_in, G, grid, **kw), G, grid, p)


# ---------------------------------------------------------------------------------------------------------------------
# the fold against the existing numpy backends
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", [1, 65, 193])
def test_fold_agrees_with_the_numpy_backends(d):
    from test_impute_host import ImputeOracleBackend
    from test_preprocessing_host import PPOracleBackend

    from dask_ml_b200.metrics import _scoring

    sms, n = 132, 5000
    G = cc.KT // cc.col_block(d)
    grid = cc.reduce_grid(n, G, 4, sms)
    X, s = cc.stat_case(n, d, "f64", sms, 4, seed=d, shifted=True)
    x = torch.from_numpy(X)
    sh = torch.from_numpy(s)
    acc, mm = torch.empty(5, d, dtype=torch.float64), torch.empty(2, d, dtype=torch.float64)
    PPOracleBackend().colstats_chunk(x, sh, acc, mm, first=True)
    v = cc.colstats_fold(X, s, G, grid)
    np.testing.assert_allclose(v[:5], acc.numpy(), rtol=1e-13)
    np.testing.assert_array_equal(v[5:], mm.numpy())
    acc4 = torch.empty(4, d, dtype=torch.float64)
    ImputeOracleBackend().impute_stats_chunk(x, False, -1.0, sh, acc4, first=True)
    np.testing.assert_allclose(cc.impute_fold(X, s, False, -1.0, G, grid), acc4.numpy(), rtol=1e-13)
    A, B = metric_err_case(n, d, "f64", seed=d)
    Gm = cc.KT // cc.metric_cb(d, "err")
    want = _scoring.host_sums(_scoring.ERR, A, B, shift=np.zeros(d))
    got = cc.metric_err_fold(A, B, None, Gm, cc.metric_grid(n, d, "err", sms))
    np.testing.assert_allclose(got, want, rtol=1e-12)
    w = np.ldexp(1.0, np.random.RandomState(d).randint(-4, 5, n))
    cls = np.random.RandomState(d).randint(0, 3, n).astype(np.int32)
    P = np.random.RandomState(d + 1).uniform(0, 1, (n, 3))
    lg = cc.metric_row_fold(cc.logloss_terms(cls, P, w, 1e-15), w, 256, cc.metric_grid(n, 3, "log", sms), sub=True)
    np.testing.assert_allclose(lg[:, 0], _scoring.host_sums(_scoring.LOGLOSS, cls, P, w=w, eps=1e-15), rtol=1e-12)
    eq = cc.metric_row_fold(cc.eq_terms(A[:, :1], B[:, :1], w), w, 256, cc.metric_grid(n, 1, "eq", sms))
    np.testing.assert_allclose(eq[:, 0], _scoring.host_sums(_scoring.EQ, A[:, :1], B[:, :1], w=w), rtol=1e-12)


def test_device_fmin_fmax_order_signed_zeros():
    """CUDA's fmin / fmax put -0.0 below +0.0 whatever the order; np.fmin / np.fmax return their first argument."""
    p, m = np.array([0.0]), np.array([-0.0])
    for a, b in ((p, m), (m, p)):
        assert np.signbit(cc.dev_fmin(a, b))[0] and not np.signbit(cc.dev_fmax(a, b))[0]
    assert not np.signbit(np.fmin(p, m))[0] and np.signbit(np.fmax(m, p))[0]
    assert cc.dev_fmin(np.array([np.nan]), m)[0] == 0.0 and cc.dev_fmax(np.array([3.0]), np.array([np.nan]))[0] == 3.0


def test_store_rules():
    v = np.array([[1.0], [2.0], [0.0], [0.0], [0.0], [-0.0], [3.0]])
    acc, mm = cc.colstats_store(None, v, True)
    acc2, mm2 = cc.colstats_store((acc, mm), np.array([[1.0], [1.0], [0], [0], [0], [-1.0], [2.0]]), False)
    np.testing.assert_array_equal(acc2[:2, 0], [2.0, 3.0])
    np.testing.assert_array_equal(mm2[:, 0], [-1.0, 3.0])
