"""The dense cases and the numpy restatement of the dense passes' host rules (tests/dense_cases.py), without a GPU: the
limits each case reaches for an H100 SXM (132 SMs) and an H100 PCIe (114 SMs), so that an edit to the cases cannot
quietly lose one, and the exact-data claim itself: every reference, summed in two orders, gives the same bits."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import dense_cases as dc  # noqa: E402


def _same(a, b):
    for x, y in zip(a, b):
        x, y = np.asarray(x), np.asarray(y)
        assert x.tobytes() == y.tobytes()


# ---------------------------------------------------------------------------------------------------------------------
# GaussianNB jll
# ---------------------------------------------------------------------------------------------------------------------
# the largest class block of every path, with the log-probability output and without it
KB_TABLE = {("f32", 8, False): (86, 1285), ("f32", 16, False): (78, 668), ("f32", 32, False): (64, 318),
            ("f32", 64, False): (43, 131), ("f32", 32, True): (46, 109), ("f64", 8, False): (78, 665),
            ("f64", 16, False): (64, 316), ("f64", 32, False): (42, 130), ("f64", 32, True): (25, 44)}


def test_jll_paths_and_block_sizes():
    assert {(dt, fc, ch) for dt, _, fc, ch in dc.jll_paths()} == set(KB_TABLE)
    for dt, d, fc, ch in dc.jll_paths():
        assert dc.jll_path(dt, d) == (fc, ch)
        assert (dc.jll_kb_max(dt, d, True), dc.jll_kb_max(dt, d, False)) == KB_TABLE[(dt, fc, ch)]
        for out in (False, True):
            kb = dc.jll_kb_max(dt, d, out)
            es = 8 if dt == "f64" else 4
            assert dc.jll_smem(es, kb, fc, fc, ch, out) <= dc.JBUDGET
            # K = kb stays resident; kb + 1 and 2 kb + 1 run two and three blocks of kb
            blocks = [(K + dc.jll_kb(dt, d, K, out) - 1) // dc.jll_kb(dt, d, K, out) for K in dc.jll_ks(dt, d, out)]
            assert blocks == [1, 2, 3]
    # the d of each path: partial and full register widths, several chunks with a partial last one
    assert {d % fc for dt, d, fc, ch in dc.jll_paths() if not ch} > {0}
    assert all(d > 64 and d % dc.JC for dt, d, fc, ch in dc.jll_paths() if ch)


@pytest.mark.parametrize("dt,d,fc,ch", dc.jll_paths())
@pytest.mark.parametrize("out", [False, True])
def test_jll_cases_are_exact_and_reach_their_blocks(dt, d, fc, ch, out):
    kb = dc.jll_kb_max(dt, d, out)
    for K in dc.jll_ks(dt, d, out):
        for nan in (None, K - 1) if K > 2 * kb else (None,):
            c = dc.jll_case(dt, d, K, kb, seed=K, nan_class=nan)
            r1, r2 = dc.jll_ref(c), dc.jll_ref(c, -1)
            _same(r1, r2)
            jll, lab, ties, lp = r1
            if nan is not None:
                assert nan // kb == 2 and (lab == nan).all() and ties == 0
                continue
            # every jll a multiple of 1/4, every fp32 sum exact, and the fp32 bound E far below half that step
            assert (jll * 4 == np.round(jll * 4)).all()
            assert (np.abs(c.x - c.theta[:1]).max() ** 2 * c.w.max() * d) < 2 ** 24
            assert 2 * dc.fp32_bound(c) < 0.25
            a, b = c.tie
            assert (lab[c.tie_rows] == a).all() and ties >= len(c.tie_rows)
            if K > kb:
                assert a // kb == 0 and b // kb == 1                 # the tie straddles the first block boundary
            if c.last is not None:
                assert (lab[c.last_rows] == K - 1).all() and len(c.last_rows) > 0
            assert np.isfinite(lp).all()


# ---------------------------------------------------------------------------------------------------------------------
# linear jll and projection
# ---------------------------------------------------------------------------------------------------------------------
def test_linear_and_projection_geometries():
    assert {dc.linear_geom(K)[0] for K in dc.LIN_K} == {1, 2, 4}
    assert {dc.linear_geom(K)[2] for K in dc.LIN_K} == {1, 2, 3}
    for sms in dc.SMS:
        g = [dc.project_geom(dc.project_case(k, 31).x.shape[0], k, sms) for k in dc.LIN_K]
        assert {x[0] for x in g} == {1, 2, 4} and {x[2] for x in g} == {1, 2, 3}
        assert all(x[3] > 1 for x in g)                             # several row tiles, on several CTAs
    # one feature step short of 32, exactly 32, and one feature into the second step
    assert sorted((d + 31) // 32 for d in dc.LIN_D) == [1, 1, 2] and 32 in dc.LIN_D


@pytest.mark.parametrize("K", dc.LIN_K)
@pytest.mark.parametrize("d", dc.LIN_D)
def test_linear_and_projection_cases_are_exact(K, d):
    c = dc.linear_case(K, d, seed=K + d, binarize=1.5 if d == 33 else None)
    r = dc.linear_ref(c)
    _same(r, dc.linear_ref(c, -1))
    jll, lab, _ = r
    a, b = c.tie
    _, cw, nblk = dc.linear_geom(K)
    assert (lab[c.tie_rows] == a).all() and (jll[c.tie_rows, a] == jll[c.tie_rows, b]).all()
    if nblk > 1:
        assert a // cw == 0 and b // cw == 1
    if c.last is not None:
        assert (lab[c.zero_rows] == K - 1).all()
    p = dc.project_case(K, d, seed=K * d)
    out, rec = dc.project_ref(p)
    _same((out, rec), dc.project_ref(p, -1))
    # every column's largest |out| is held by two rows of opposite sign: the record takes the lower one
    top = np.abs(out) == rec[:, 0][None]
    assert (top.sum(0) >= 2).all() and (out[top] != 0).all()
    assert (out == out.astype(np.float32)).all()                    # the fp32 output is exact too


# ---------------------------------------------------------------------------------------------------------------------
# Gram
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sms", dc.SMS)
def test_gram_cases_reach_the_split_limits(sms):
    t = dc.gram_one_split_d(sms)
    assert t == {132: 1409, 114: 1281}[sms]
    ds = dc.gram_ds(sms)
    big = 10 ** 6
    assert dc.gram_geom(big, t - 1, sms).splits == 2 and dc.gram_geom(big, t, sms).splits == 1
    assert dc.gram_geom(big, 2049, sms).splits == 1
    assert {d % 64 for d in ds} >= {0, 1, 63}
    for d in ds:
        c = dc.gram_case(d, sms)
        gA, gB = (dc.gram_geom(x.shape[0], d, sms) for x in c.xs)
        if gA.splits > 1:
            assert c.xs[0].shape[0] - (gA.splits - 1) * gA.rows_per_split == 1   # one row in the last split
        assert c.xs[0].shape[0] != c.xs[1].shape[0]
        if d < t:
            assert gA.splits > 1 and (gA.splits, gA.rows_per_split) != (gB.splits, gB.rows_per_split)
    # the bulk and the plain-load path of every dtype, and a base one element off alignment
    for dt, es in dc.ES.items():
        assert dc.bulk_ok(0, t - 1, t - 1, dt) and not dc.bulk_ok(es, t - 1, t - 1, dt)
        assert not dc.bulk_ok(0, t, t, dt)


@pytest.mark.parametrize("d", sorted(set(dc.gram_ds(132) + dc.gram_ds(114))))
def test_gram_cases_are_exact(d):
    c = dc.gram_case(d, 132 if d in dc.gram_ds(132) else 114, seed=d)
    _same(dc.gram_ref(c), dc.gram_ref(c, -1))


# ---------------------------------------------------------------------------------------------------------------------
# moments and class counts
# ---------------------------------------------------------------------------------------------------------------------
def test_moments_cases_reach_the_slice_limits():
    assert [dc.mom_ks(d) for d in dc.MOM_D] == [48, 47, 47, 47]
    assert [dc.mom_geom(1, d, 1, 132).nf for d in dc.MOM_D] == [1, 1, 2, 3]
    for sms in dc.SMS:
        for d in dc.MOM_D:
            ks = dc.mom_ks(d)
            for K, nk in ((ks, 1), (ks + 1, 2)):
                gA, gB = (dc.mom_geom(n, d, K, sms) for n in (600, 300))
                assert gA.nk == nk and gA.splits == 3 and gB.splits == 2


@pytest.mark.parametrize("d", dc.MOM_D)
def test_moments_cases_are_exact(d):
    ks = dc.mom_ks(d)
    for K in (ks, ks + 1):
        c = dc.mom_case(d, K, seed=d + K)
        for bz in (None, 0.5):
            _same(dc.mom_ref(c, binarize=bz), dc.mom_ref(c, -1, binarize=bz))
        assert (c.cls[0] == K - 1).any() and (c.cls[0] == -1).any() and (c.cls[0] == K).any()


# ---------------------------------------------------------------------------------------------------------------------
# GLM
# ---------------------------------------------------------------------------------------------------------------------
def test_glm_cases_reach_every_column_block():
    cb = [dc.glm_phase_b(d) for d in dc.GLM_D]
    assert {x[0] for x in cb} == {32, 64, 96, 128, 160, 192, 224, 256}
    assert {x[1] for x in cb} == {1, 2, 4, 8} and max(x[2] for x in cb) == 3
    for dt, es in dc.ES.items():
        vec = {dc.bulk_ok(0, d, d, dt) for d in dc.GLM_D}
        assert vec == {True, False}
        assert not any(dc.bulk_ok(es, d, d, dt) for d in dc.GLM_D)
    for sms in dc.SMS:
        c = dc.glm_case(31, sms)
        nA, nB = (x.shape[0] for x in c.xs)
        gA, gB = dc.glm_grid(nA, sms), dc.glm_grid(nB, sms)
        assert gA == 3 * sms and (nA + 31) // 32 > gA and gB < gA     # some CTAs walk two tiles; B another grid
        assert nA % 32 and nB % 32


@pytest.mark.parametrize("d", dc.GLM_D)
def test_glm_normal_cases_are_exact(d):
    c = dc.glm_case(d, 132, seed=d)
    g1, h1, w1, m1, _, _ = dc.glm_ref(c)
    g2, h2, w2, m2, _, _ = dc.glm_ref(c, -1)
    _same((g1, h1) + tuple(m1), (g2, h2) + tuple(m2))
