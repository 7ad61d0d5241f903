"""The column-block passes on the H100 at their layout and grid limits (tests/colpass_cases.py), against the fold restated
in the kernel's order.

The reductions (the scalers' statistics, the imputer's statistics, the metrics' ERR / EQ sums and the sparse KMeans
pack) are held byte for byte, signs of zero included, to ``colpass_cases.fold``: on the cases' data a fold that took
the row groups or the CTAs in another order gives other bits.  Each runs as a chain over the layout's row counts, the
first call overwriting and every later one, on another grid, accumulating; the chain runs twice and must give the same
bits.  LOGLOSS's log term goes through CUDA's log and is held to a tolerance; its sum of weights is exact.  The element
passes write into outputs of a larger pitch pre-filled with NaN: the affine pass is bit-identical to numpy's two-step
expression for every op pair, the imputer's fill and inverse to numpy's restatement of scikit-learn's transform with an
exact NaN / inf count, and the quantile transform to ``transform_restated`` (uniform) or within NORMAL_TOL (normal).
The SM count is the device's, and the workspace queries are checked against the restatement."""
import os
import sys
import warnings

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import colpass_cases as cc  # noqa: E402

pytestmark = pytest.mark.gpu

TD = {"f32": torch.float32, "f64": torch.float64, "bf16": torch.bfloat16}
MISS = -1.0


@pytest.fixture(scope="module")
def be():
    from dask_ml_b200.engine import CudaBackend

    return CudaBackend()


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _rows(X, dt, pad):
    """X on the device in dtype dt, as a view of row pitch d + pad."""
    n, d = X.shape
    buf = torch.zeros((n, d + pad), dtype=TD[dt], device="cuda")
    if n:
        buf[:, :d] = torch.from_numpy(X).to(TD[dt]).cuda()
    return buf[:, :d]


def _dev(a, dt=torch.float64):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dt).cuda()


def _host(*ts):
    torch.cuda.synchronize()
    return [t.cpu().numpy().copy() for t in ts]


def _same(got, want, what):
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    if got.tobytes() != want.tobytes():
        bad = np.argwhere(got.view(np.int64) != want.view(np.int64))
        raise AssertionError("%s: %d elements differ, first %s: %r vs %r" % (
            what, len(bad), bad[0], got[tuple(bad[0])], want[tuple(bad[0])]))


def _bits(got, want, what):
    """Bit-identical in the output's own dtype, signs of zero included; a NaN matches any NaN (numpy keeps an input
    NaN's payload, the device's arithmetic writes its canonical NaN)."""
    got, want = np.ascontiguousarray(got), np.ascontiguousarray(want, dtype=got.dtype)
    u = np.uint32 if got.dtype == np.float32 else np.uint64
    nan = np.isnan(got) & np.isnan(want)
    if (got.view(u)[~nan] != want.view(u)[~nan]).any() or (np.isnan(got) != np.isnan(want)).any():
        bad = np.argwhere((got.view(u) != want.view(u)) & ~nan)
        raise AssertionError("%s: %d elements differ, first %s: %r vs %r" % (
            what, len(bad), bad[0], got[tuple(bad[0])], want[tuple(bad[0])]))


def _query(be, name, *args):
    return be._query(name, *[int(a) for a in args])


def _chain(run_once):
    """run_once() twice: the same bits at every step."""
    a, b = run_once(), run_once()
    for x, y in zip(a, b):
        for u, v in zip(x, y):
            assert u.tobytes() == v.tobytes()
    return a


# ---------------------------------------------------------------------------------------------------------------------
# scalers' and imputer's statistics
# ---------------------------------------------------------------------------------------------------------------------
def _stat_chain(d, dt, sms, shifted):
    G = cc.KT // cc.col_block(d)
    out = []
    for i, (lab, n) in enumerate(cc.reduce_rows(G, 4, sms).items()):
        X, s = cc.stat_case(n, d, dt, sms, 4, seed=1000 * d + i, shifted=shifted, miss=MISS)
        Xh = torch.from_numpy(X).to(TD[dt]).double().numpy()            # the values the device sees
        out.append((lab, n, X, s, Xh))
    return G, out


@pytest.mark.parametrize("dt", ["f32", "f64", "bf16"])
@pytest.mark.parametrize("d", cc.WIDTHS)
def test_colstats_and_impute_stats(be, sms, d, dt):
    for shifted in ((False, True) if dt == "f32" else (False,)):
        G, chain = _stat_chain(d, dt, sms, shifted)
        want_cs, want_im, prev_cs, prev_im = [], [], None, None
        for i, (lab, n, X, s, Xh) in enumerate(chain):
            grid = cc.reduce_grid(n, G, 4, sms)
            assert _query(be, "bkm_colstats_workspace_bytes", n, d) == cc.partials_bytes(grid, 7 * d)
            assert _query(be, "bkm_impute_stats_workspace_bytes", n, d) == cc.partials_bytes(grid, 4 * d)
            prev_cs = cc.colstats_store(prev_cs, cc.colstats_fold(Xh, s, G, grid), i == 0)
            miss_nan = i % 2 == 0
            prev_im = cc.sum_store(prev_im, cc.impute_fold(Xh, s, miss_nan, MISS, G, grid), i == 0)
            want_cs.append(prev_cs)
            want_im.append(prev_im)
        xs = [(_rows(X, dt, 3 + 2 * (i % 2)), None if s is None else _dev(s)) for i, (_, _, X, s, _) in enumerate(chain)]

        def run():
            acc = torch.full((5, d), np.nan, dtype=torch.float64, device="cuda")
            mm = torch.full((2, d), np.nan, dtype=torch.float64, device="cuda")
            acc4 = torch.full((4, d), np.nan, dtype=torch.float64, device="cuda")
            steps = []
            for i, (x, sh) in enumerate(xs):
                be.colstats_chunk(x, sh, acc, mm, first=i == 0)
                be.impute_stats_chunk(x, i % 2 == 0, MISS, sh, acc4, first=i == 0)
                steps.append(_host(acc, mm, acc4))
            return steps

        got = _chain(run)
        for i, ((a, m, a4), (wa, wm), wi) in enumerate(zip(got, want_cs, want_im)):
            what = "d=%d %s %s rows %s" % (d, dt, "shifted" if shifted else "wide", chain[i][0])
            _same(a, wa, "colstats acc " + what)
            _same(m, wm, "colstats min/max " + what)
            _same(a4, wi, "impute stats " + what)


# ---------------------------------------------------------------------------------------------------------------------
# metrics
# ---------------------------------------------------------------------------------------------------------------------
def _err_case(n, m, dt, sms, seed):
    rng = np.random.RandomState(seed)
    k = rng.randint(-30, 31, (n, m))
    top = 1 << cc.MBITS[dt]
    A = np.ldexp(rng.randint(-top + 1, top, (n, m)).astype(np.float64), k)
    B = np.ldexp(rng.randint(-top + 1, top, (n, m)).astype(np.float64), k)
    G = cc.KT // cc.metric_cb(m, "err")
    grid = cc.metric_grid(n, m, "err", sms)
    cc.plant(A, n, G, grid, 2.0 ** 60, True)
    cc.plant(B, n, G, grid, 2.0 ** 60, True)
    return A, B


@pytest.mark.parametrize("dt", ["f32", "f64", "bf16"])
@pytest.mark.parametrize("m", cc.METRIC_M)
def test_metric_err(be, sms, m, dt):
    G = cc.KT // cc.metric_cb(m, "err")
    cases, want, prev = [], [], None
    for i, (lab, n) in enumerate(cc.reduce_rows(G, 8, sms).items()):
        A, B = _err_case(n, m, dt, sms, seed=100 * m + i)
        assert cc.short_ok(B - A) and cc.short_ok(A)
        shift = None                                   # a - s stays short only for s = 0 on wide exponents
        grid = cc.metric_grid(n, m, "err", sms)
        assert _query(be, "bkm_metric_workspace_bytes", n, m, 1) == cc.partials_bytes(grid, 4 * m)
        prev = cc.sum_store(prev, cc.metric_err_fold(A, B, shift, G, grid), i == 0)
        want.append(prev)
        cases.append((_dev(A, TD[dt]), _dev(B, TD[dt]), None if shift is None else _dev(shift), lab))

    def run():
        acc = torch.full((4, m), np.nan, dtype=torch.float64, device="cuda")
        steps = []
        for i, (a, b, s, _) in enumerate(cases):
            s = s if s is not None else torch.zeros(m, dtype=torch.float64, device="cuda")
            be.metric_chunk(a, b, 1, acc, shift=s, first=i == 0)
            steps.append(_host(acc))
        return steps

    for (g,), w, c in zip(_chain(run), want, cases):
        _same(g, w, "ERR m=%d %s rows %s" % (m, dt, c[3]))


@pytest.mark.parametrize("m", cc.METRIC_ROW_M)
def test_metric_eq_and_logloss(be, sms, m):
    cases, weq, wlog, tlog, pe, pl, pt = [], [], [], [], None, None, None
    for i, (lab, n) in enumerate(cc.reduce_rows(256, 8, sms).items()):
        if n * m > 5 * 10 ** 6:
            continue                                   # the cap at m = 40: 170M elements
        rng = np.random.RandomState(7 * m + i)
        w = cc.wide(rng, n, "f64", kspan=20)
        grid = cc.metric_grid(n, m, "eq", sms)
        cc.plant(w[:, None], n, 256, grid, 2.0 ** 60, True)
        A = rng.randint(0, 3, (n, m)).astype(np.float64)
        B = A.copy()
        B[rng.rand(n) < 0.3, m - 1] += 1.0
        cls = rng.randint(0, max(m, 2), n).astype(np.int32)
        P = rng.uniform(0.0, 1.0, (n, m))
        assert _query(be, "bkm_metric_workspace_bytes", n, m, 0) == cc.partials_bytes(grid, 4)
        pe = cc.sum_store(pe, cc.metric_row_fold(cc.eq_terms(A, B, w), w, 256, grid), i == 0)
        ll = cc.logloss_terms(cls, P, w, 1e-7)
        pl = cc.sum_store(pl, cc.metric_row_fold(ll, w, 256, grid, sub=True), i == 0)
        pt = cc.sum_store(pt, cc.metric_row_fold(np.abs(ll), np.abs(w), 256, grid), i == 0)
        weq.append(pe)
        wlog.append(pl)
        tlog.append(pt)
        cases.append([_dev(x, t) for x, t in ((A, torch.float32), (B, torch.float32), (w, torch.float64),
                                              (cls, torch.int32), (P, torch.float64))] + [lab])

    def run():
        eq = torch.full((2,), np.nan, dtype=torch.float64, device="cuda")
        lg = torch.full((2,), np.nan, dtype=torch.float64, device="cuda")
        steps = []
        for i, (a, b, w, cls, P, _) in enumerate(cases):
            be.metric_chunk(a, b, 0, eq, w=w, first=i == 0)
            be.metric_chunk(cls, P if m > 1 else P[:, 0].contiguous(), 2, lg, w=w, eps=1e-7, first=i == 0)
            steps.append(_host(eq, lg))
        return steps

    for (e, lgot), we, wl, tl, c in zip(_chain(run), weq, wlog, tlog, cases):
        _same(e, we[:, 0], "EQ m=%d rows %s" % (m, c[5]))
        _same(lgot[1], wl[1, 0], "LOGLOSS sum w m=%d rows %s" % (m, c[5]))
        if np.isnan(wl[0, 0]):
            assert np.isnan(lgot[0])
        else:
            assert abs(lgot[0] - wl[0, 0]) <= 1e-13 * tl[0, 0], (lgot[0], wl[0, 0], tl[0, 0])


# ---------------------------------------------------------------------------------------------------------------------
# sparse KMeans pack
# ---------------------------------------------------------------------------------------------------------------------
def _pack_call(be, name, args, k, p):
    from dask_ml_b200 import _lib

    nb = _query(be, "bkm_sparse_pack_workspace_bytes", k, p)
    ws = torch.full((nb,), 0xFF, dtype=torch.uint8, device="cuda")
    _lib.call(name, *args, ws.data_ptr(), nb, torch.cuda.current_stream().cuda_stream)
    return ws[: 8 * k].view(torch.float64)


@pytest.mark.parametrize("k", cc.PACK_K)
def test_sparse_pack(be, sms, k):
    G = cc.KT // cc.col_block(k)
    for lab, p in cc.pack_rows(k, sms).items():
        grid = cc.pack_grid_sparse(p, k, sms)
        assert _query(be, "bkm_sparse_pack_workspace_bytes", k, p) == cc.pack_ws(p, k, sms)
        c = cc.pack_case(p, k, sms, seed=p + k)
        v0 = cc.pack_fold(c.C.T, None, G, grid)
        v1 = cc.pack_fold(c.new, c.ct_in, G, grid)
        shift = 0.0
        for j in range(k):
            shift += v1[0, j]
        C64, red = _dev(c.C), _dev(c.red)
        pack_in = _dev(np.concatenate([c.ct_in.ravel(), np.zeros(k)]))

        def run():
            pack = torch.full((p * k + k,), np.nan, dtype=torch.float64, device="cuda")
            sc0 = _pack_call(be, "bkm_sparse_pack_centers", (C64.data_ptr(), k, p, pack.data_ptr()), k, p)
            out = torch.full((p * k + k,), np.nan, dtype=torch.float64, device="cuda")
            state, hist = be.loop_state_new(0.0, 4)
            sc1 = _pack_call(be, "bkm_sparse_finalize_step", (red.data_ptr(), pack_in.data_ptr(), out.data_ptr(),
                                                               state.data_ptr(), k, p), k, p)
            return [_host(pack, sc0, out, sc1, hist)]

        (pack, sc0, out, sc1, hist), = _chain(run)
        what = "k=%d p=%d (%s)" % (k, p, lab)
        _same(pack[: p * k], c.C.T.ravel(), "pack CT " + what)
        _same(pack[p * k:], v0[1], "pack cn " + what)
        _same(sc0, v0[0], "pack shift terms " + what)
        _same(out[: p * k], c.new.ravel(), "step CT " + what)
        _same(out[p * k:], v1[1], "step cn " + what)
        _same(sc1, v1[0], "step shift terms " + what)
        _same(hist[0], shift, "step shift " + what)


# ---------------------------------------------------------------------------------------------------------------------
# affine
# ---------------------------------------------------------------------------------------------------------------------
AFFINE_TYPES = [("f32", "f32"), ("bf16", "f32"), ("f32", "f64"), ("f64", "f64"), ("bf16", "f64")]
OPS = [(o1, o2) for o1 in range(3) for o2 in range(3)]


def _affine_ref(Xh, a, b, op1, op2, odt):
    C = np.float32 if odt == "f32" else np.float64
    x = Xh.astype(C)
    ac, bc = a.astype(C), b.astype(C)
    with np.errstate(all="ignore"):
        if op1 == 1:
            x = x - ac
        elif op1 == 2:
            x = x * ac
        if op2 == 1:
            x = x / bc
        elif op2 == 2:
            x = x + bc
    return x


@pytest.mark.parametrize("types", AFFINE_TYPES, ids=["%s-%s" % t for t in AFFINE_TYPES])
@pytest.mark.parametrize("d", cc.WIDTHS)
def test_affine(be, sms, d, types):
    xdt, odt = types
    G = cc.KT // cc.col_block(d)
    rng = np.random.RandomState(d)
    a = cc.wide(rng, d, "f64", kspan=8)
    b = cc.wide(rng, d, "f64", kspan=8)
    for i, (lab, n) in enumerate(cc.pass_rows(d, sms).items()):
        X = cc.wide(rng, (n, d), xdt, kspan=20)
        cc.place_specials(X, cc.special_rows(n, G, cc.col_pass_grid(n, d, sms)), MISS, i)
        x = _rows(X, xdt, 1 + 2 * i)
        Xh = x.float().cpu().numpy() if xdt == "bf16" else x.cpu().numpy()
        for op1, op2 in (OPS if lab == "8G+1" else [(1, 1), (2, 2)]):
            buf = torch.full((n, d + 5), np.nan, dtype=TD[odt], device="cuda")
            be.affine_chunk(x, _dev(a), _dev(b), op1, op2, buf[:, :d])
            (got,) = _host(buf)
            want = _affine_ref(Xh, a, b, op1, op2, odt)
            _bits(got[:, :d], want, "d=%d %s rows %s ops %d %d" % (d, types, lab, op1, op2))
            assert np.isnan(got[:, d:]).all()


# ---------------------------------------------------------------------------------------------------------------------
# the imputer's fill pass and its inverse
# ---------------------------------------------------------------------------------------------------------------------
def _fill_layout(T):
    """(d, keep, ind, check) for T = n_keep + n_ind + n_check tasks."""
    nk = (T + 1) // 2
    ni = T // 4
    nc = T - nk - ni
    return nk + nc, list(range(nk)), list(range(0, nk, 2))[:ni], list(range(nk, nk + nc))


@pytest.mark.parametrize("dt", ["f32", "f64", "bf16"])
@pytest.mark.parametrize("T", cc.WIDTHS)
def test_impute_fill_and_inverse(be, sms, T, dt):
    C = np.float64 if dt == "f64" else np.float32
    odt = torch.float64 if dt == "f64" else torch.float32
    d, keep, ind, chk = _fill_layout(T)
    assert len(keep) + len(ind) + len(chk) == T
    G = cc.KT // cc.col_block(T)
    rng = np.random.RandomState(T)
    stats = cc.wide(rng, d, dt, kspan=8)
    cols = _dev(np.array(keep + ind + chk), torch.int32)
    for i, (lab, n) in enumerate(cc.pass_rows(T, sms).items()):
        X = cc.wide(rng, (n, d), dt, kspan=20)
        cc.place_specials(X, cc.special_rows(n, G, cc.col_pass_grid(n, T, sms)), MISS, i)
        X[rng.rand(n, d) < 0.05] = MISS
        X[rng.rand(n, d) < 0.02] = np.nan
        X[rng.rand(n, d) < 0.01] = np.inf
        x = _rows(X, dt, 2 + i)
        v = x.float().cpu().numpy() if dt == "bf16" else x.cpu().numpy()
        for miss_nan in (False, True):
            m = np.isnan(v) if miss_nan else v == MISS
            want = np.hstack([np.where(m[:, keep], stats[keep].astype(C), v[:, keep].astype(C)),
                              m[:, ind].astype(C)])
            seen = v[:, keep + chk]
            bad = [float(np.isnan(seen).sum()), float(np.isinf(seen).sum())]
            w = len(keep) + len(ind)
            outs = []
            for _ in range(2):
                buf = torch.full((n, w + 3), np.nan, dtype=odt, device="cuda")
                inv = torch.zeros(2, dtype=torch.float64, device="cuda")
                be.impute_chunk(x, miss_nan, MISS, _dev(stats), cols, len(keep), len(ind), len(chk), False,
                                buf[:, :w], invalid=inv)
                outs.append(_host(buf, inv))
            assert outs[0][0].tobytes() == outs[1][0].tobytes()
            (buf, inv) = outs[0]
            what = "T=%d %s rows %s miss %s" % (T, dt, lab, "nan" if miss_nan else MISS)
            _bits(buf[:, :w], want, what)
            assert np.isnan(buf[:, w:]).all()
            assert inv.tolist() == bad, (what, inv.tolist(), bad)
        # the inverse: T output columns from T source and T indicator columns (-1: none)
        src = [o % d if o % 7 else -1 for o in range(T)]
        isrc = [(o % d) if o % 3 else -1 for o in range(T)]
        Xi = np.where(rng.rand(n, d) < 0.5, 0.0, X)
        Xi[:, ::2] = (rng.rand(n, (d + 1) // 2) < 0.3).astype(np.float64)
        xi = _rows(Xi, dt, 1)
        vi = xi.float().cpu().numpy() if dt == "bf16" else xi.cpu().numpy()
        want = np.zeros((n, T), dtype=C)
        for o in range(T):
            if src[o] >= 0:
                want[:, o] = vi[:, src[o]]
            if isrc[o] >= 0:
                want[vi[:, isrc[o]] != 0, o] = C(MISS)
        buf = torch.full((n, T + 3), np.nan, dtype=odt, device="cuda")
        be.impute_chunk(xi, False, MISS, None, _dev(np.array(src + isrc), torch.int32), T, T, 0, True, buf[:, :T])
        (buf,) = _host(buf)
        _bits(buf[:, :T], want, "inverse T=%d %s rows %s" % (T, dt, lab))
        assert np.isnan(buf[:, T:]).all()


# ---------------------------------------------------------------------------------------------------------------------
# quantile transform
# ---------------------------------------------------------------------------------------------------------------------
QT_NQ = {"f32": [1365, 1366, 341, 342, 682, 683], "bf16": [1365, 1366, 341, 342, 682, 683],
         "f64": [2457, 2458, 614, 615, 1228, 1229]}


@pytest.mark.parametrize("dt", ["f32", "f64", "bf16"])
@pytest.mark.parametrize("i", range(6))
def test_quantile_transform(be, sms, dt, i):
    from scipy import stats
    from sklearn.preprocessing._data import BOUNDS_THRESHOLD
    from test_gpu_quantile import NORMAL_TOL, normal_error
    from test_quantile_host import transform_restated

    nq = QT_NQ[dt][i]
    CS = cc.QCS[dt]
    ref = np.linspace(0.0, 1.0, nq)
    eps = BOUNDS_THRESHOLD - np.spacing(1)
    for d in (CS - 1, CS, CS + 1, 1001):
        rng = np.random.RandomState(nq + d)
        q = np.sort(np.round(rng.standard_normal((nq, d)) * 4, 2), axis=0)      # ties among the quantiles
        qT = _dev(q.T)
        geo = cc.qtransform_geom(10 ** 9, d, nq, dt, sms)
        n_big = geo[4] * (cc.KT // CS) * 8 + 5
        for n in ((700, n_big) if d == CS + 1 else (700,)):
            X = rng.standard_normal((n, d)) * 5
            X[::13, 0] = np.nan
            X[1::17, d - 1] = -0.0
            X[2::19, d // 2] = 0.0
            U = np.clip(rng.uniform(-0.1, 1.1, (n, d)), 0, 1)
            U[::11, d - 1] = np.nan
            for dist, inverse in (("uniform", False), ("uniform", True), ("normal", False), ("normal", True)):
                if dist == "normal" and (n == n_big or d == 1001):
                    continue
                src = (stats.norm.ppf(U) if dist == "normal" else U) if inverse else X
                x = _rows(src, dt, 3)
                xh = x.float().cpu().numpy() if dt == "bf16" else x.cpu().numpy()
                D = stats.norm if dist == "normal" else stats.uniform
                lo, hi = (0.0, 0.0) if inverse else (float(D.ppf(eps)), float(D.ppf(1 - eps)))
                buf = torch.full((n, d + 3), np.nan, dtype=torch.float64, device="cuda")
                be.quantile_transform_chunk(x, qT, _dev(ref), inverse, int(dist == "normal"), lo, hi, buf[:, :d])
                (got,) = _host(buf)
                want = transform_restated(xh, q, ref, inverse, dist)
                assert np.isnan(got[:, d:]).all()
                if dist == "uniform":
                    _bits(got[:, :d], want, "uniform d=%d nq=%d n=%d inverse=%s" % (d, nq, n, inverse))
                else:
                    assert normal_error(got[:, :d], want, q, ref) <= NORMAL_TOL


# ---------------------------------------------------------------------------------------------------------------------
# end to end at the spare-thread widths
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", [70, 150])
def test_estimators_at_spare_thread_widths(d):
    import sklearn.impute
    import sklearn.preprocessing as skp

    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.impute import SimpleImputer
    from dask_ml_b200.preprocessing import MinMaxScaler, StandardScaler

    rng = np.random.RandomState(d)
    X = rng.standard_normal((20000, d)) * rng.uniform(0.5, 4, d) + rng.uniform(-5, 5, d)
    C = ChunkedArray([torch.from_numpy(X[i:i + 7000]).cuda() for i in range(0, len(X), 7000)])
    s, ws = StandardScaler().fit(C), skp.StandardScaler().fit(X)
    np.testing.assert_allclose(s.mean_, ws.mean_, rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(s.var_, ws.var_, rtol=1e-9)
    np.testing.assert_allclose(s.transform(C).compute(), ws.transform(X), rtol=1e-10, atol=1e-12)
    mm, wm = MinMaxScaler().fit(C), skp.MinMaxScaler().fit(X)
    np.testing.assert_array_equal(mm.data_min_, wm.data_min_)
    np.testing.assert_array_equal(mm.data_max_, wm.data_max_)
    np.testing.assert_allclose(mm.transform(C).compute(), wm.transform(X), rtol=1e-12, atol=1e-12)
    Xm = X.copy()
    Xm[rng.rand(*X.shape) < 0.1] = np.nan
    Xm[:, 3] = X[:, 3]                                                    # a column with nothing missing
    Cm = ChunkedArray([torch.from_numpy(Xm[i:i + 7000]).cuda() for i in range(0, len(Xm), 7000)])
    for strategy in ("mean", "median"):
        est = SimpleImputer(strategy=strategy, add_indicator=True).fit(Cm)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            want = sklearn.impute.SimpleImputer(strategy=strategy, add_indicator=True).fit(Xm)
        np.testing.assert_allclose(est.statistics_, want.statistics_, rtol=1e-12)
        np.testing.assert_array_equal(est.indicator_.features_, want.indicator_.features_)
        want.statistics_ = est.statistics_.copy()
        out = est.transform(Cm)
        np.testing.assert_array_equal(out.compute(), want.transform(Xm))
        np.testing.assert_array_equal(est.inverse_transform(out).compute(), want.inverse_transform(want.transform(Xm)))
