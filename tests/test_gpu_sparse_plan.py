"""Every CSR pass on the H100 on blocks built to reach the transpose plan's segment and Gram-run limits, skewed rows,
rows at the row gather's batch edges and every column-tile shape (tests/sparse_cases.py).

Each pass runs twice and must give the same bits.  Each accumulating pass runs as a first call on one block and an
accumulating call on a second block of the same width with a different plan, sharing the workspace.  The transpose and
the plain-add label sums are held bit for bit to the numpy restatement; the fma passes to 1e-13 of the scale of each
output (|X|ᵀ|v|, |X||W|, ...).  With integer values and dyadic operands (the 'int' cases) every one of those sums is
exact, so the bound is then zero in effect."""
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import sparse_cases as sc  # noqa: E402

pytestmark = pytest.mark.gpu

DT = {"f32": np.float32, "f64": np.float64}
# (value dtype, values): integers in float32 (exact sums), standard normal in float64
COMBOS = [("f32", "int"), ("f64", "rand")]
COLUMN_CASES = sorted(sc.column_cases())
_cache = {}


@pytest.fixture(scope="module")
def be():
    from dask_ml_b200.engine import CudaBackend

    return CudaBackend()


def _pair(kind, name, dt, values):
    key = (kind, name, dt, values)
    if key not in _cache:
        if len(_cache) > 6:
            _cache.clear()
        _cache[key] = (sc.column_cases if kind == "col" else sc.row_cases)(DT[dt], values)[name]()
    return _cache[key]


def _dev(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _blk(m):
    return (_dev(m.indptr.astype(np.int64)), _dev(m.indices.astype(np.int64)), _dev(m.data), m.shape[0])


def _host(*ts):
    torch.cuda.synchronize()
    return [t.cpu().numpy().copy() for t in ts]


def _operand(rng, shape, values):
    """Dyadic values for the integer cases (every product and sum exact), standard normal otherwise."""
    if values == "int":
        return rng.randint(-8, 9, shape) / 8.0
    return rng.standard_normal(shape)


def _f64(m):
    return sp.csr_matrix(m, dtype=np.float64)


def _close(got, want, scale, what):
    err = np.abs(got - want)
    bound = 1e-13 * scale
    bad = np.argwhere(~(err <= bound))
    assert len(bad) == 0, "%s: %d elements off, first %s: %r vs %r (bound %g)" % (
        what, len(bad), bad[0], got[tuple(bad[0])], want[tuple(bad[0])], bound[tuple(bad[0])])


def _twice(run):
    """run() twice: the same bits."""
    a, b = run(), run()
    for x, y in zip(a, b):
        assert x.tobytes() == y.tobytes()
    return a


# ---------------------------------------------------------------------------------------------------------------------
# the transpose and its plan
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", ["f32", "f64"])
@pytest.mark.parametrize("kind,name", [("col", c) for c in COLUMN_CASES] + [("row", "rows"), ("row", "skewed")])
def test_transpose_and_plan(be, kind, name, dt):
    for m in _pair(kind, name, dt, "int"):
        d = m.shape[1]
        P = sc.plan(m, d)
        blk = _blk(m)
        colptr, rows, vals, plan = _twice(lambda: _host(*be.csr_transpose_chunk(blk, d)))
        assert colptr.tobytes() == P.colptr.tobytes()
        assert rows.tobytes() == P.rows.tobytes()
        assert vals.tobytes() == P.vals.tobytes()
        nw = len(P.words)
        assert plan[:nw].tobytes() == P.words.tobytes()
        assert plan[nw:].view(np.int32)[:len(P.seg_col)].tobytes() == P.seg_col.tobytes()


# ---------------------------------------------------------------------------------------------------------------------
# the column passes
# ---------------------------------------------------------------------------------------------------------------------
def _transposes(be, pair):
    d = pair[0].shape[1]
    return [(_blk(m), be.csr_transpose_chunk(_blk(m), d), sc.plan(m, d)) for m in pair]


@pytest.mark.parametrize("dt,values", COMBOS)
@pytest.mark.parametrize("name", COLUMN_CASES)
def test_csc_matvec(be, name, dt, values):
    pair = _pair("col", name, dt, values)
    d = pair[0].shape[1]
    (_, c1, _), (_, c2, _) = _transposes(be, pair)
    rng = np.random.RandomState(1)
    v = [[_operand(rng, m.shape[0], values) for _ in range(2)] for m in pair]
    vd = [[_dev(x) for x in vv] for vv in v]

    def run(two):
        o1 = torch.full((d,), 7.0, dtype=torch.float64, device="cuda")
        o2 = torch.full((d,), 7.0, dtype=torch.float64, device="cuda")
        be.csc_matvec_chunk(c1, d, vd[0][0], o1, v2=vd[0][1] if two else None, out2=o2 if two else None, first=True)
        f = _host(o1, o2)
        be.csc_matvec_chunk(c2, d, vd[1][0], o1, v2=vd[1][1] if two else None, out2=o2 if two else None)
        return f + _host(o1, o2)

    X1, X2 = _f64(pair[0]), _f64(pair[1])
    for two in (False, True):
        f1, f2, a1, a2 = _twice(lambda: run(two))
        for q, (fst, acc) in enumerate(((f1, a1), (f2, a2))[: 1 + two]):
            _close(fst, X1.T @ v[0][q], abs(X1).T @ abs(v[0][q]), "first call, vector %d" % q)
            _close(acc, X1.T @ v[0][q] + X2.T @ v[1][q], abs(X1).T @ abs(v[0][q]) + abs(X2).T @ abs(v[1][q]),
                   "accumulated, vector %d" % q)
        if not two:
            assert (f2 == 7.0).all() and (a2 == 7.0).all()


@pytest.mark.parametrize("dt", ["f32", "f64"])
@pytest.mark.parametrize("d", sc.GRAM_D)
def test_gram_weighted_csr(be, d, dt):
    """Gram widths of 8, 8, 7 and 3 warps, each with columns of 1 to 4 runs: exact on integer values and dyadic
    weights."""
    pair = _pair("col", "edges" if d == 18 else "gram%d" % d, dt, "int")
    assert pair[0].shape[1] == d
    tr = _transposes(be, pair)
    rng = np.random.RandomState(2)
    w = [rng.randint(1, 9, m.shape[0]) / 4.0 for m in pair]
    wd = [_dev(x) for x in w]

    def run():
        G = torch.full((d, d), 7.0, dtype=torch.float64, device="cuda")
        out = []
        for i, (blk, csc, P) in enumerate(tr):
            be.gram_weighted_csr_chunk(blk, csc, d, wd[i], G, int(P.status[2]), first=i == 0)
            out += _host(G)
        return out

    g1, g2 = _twice(run)
    X1, X2 = _f64(pair[0]), _f64(pair[1])
    want1 = (X1.T @ sp.diags(w[0]) @ X1).toarray()
    np.testing.assert_array_equal(g1, want1)
    want1 += (X2.T @ sp.diags(w[1]) @ X2).toarray()
    np.testing.assert_array_equal(g2, want1)


def _panel_params():
    out = []
    for name in COLUMN_CASES + ["rows"]:
        for l in sc.L_PANEL:
            if name in ("packed", "rows") or l <= 65:
                out += [(name, l, dt, v) for dt, v in COMBOS]
    return out


@pytest.mark.parametrize("name,l,dt,values", _panel_params())
def test_csc_panel(be, name, l, dt, values):
    pair = _pair("row" if name == "rows" else "col", name, dt, values)
    d = pair[0].shape[1]
    (_, c1, _), (_, c2, _) = _transposes(be, pair)
    rng = np.random.RandomState(l)
    Ps = [_operand(rng, (m.shape[0], l), values) for m in pair]
    Pd = [_dev(x) for x in Ps]

    def run():
        out = torch.full((d, l), 7.0, dtype=torch.float64, device="cuda")
        be.csc_panel_chunk(c1, d, Pd[0], out, first=True)
        f = _host(out)
        be.csc_panel_chunk(c2, d, Pd[1], out)
        return f + _host(out)

    first, acc = _twice(run)
    X1, X2 = _f64(pair[0]), _f64(pair[1])
    s1 = np.asarray(abs(X1).T @ abs(Ps[0]))
    _close(first, np.asarray(X1.T @ Ps[0]), s1, "first call")
    _close(acc, np.asarray(X1.T @ Ps[0]) + np.asarray(X2.T @ Ps[1]), s1 + np.asarray(abs(X2).T @ abs(Ps[1])),
           "accumulated")


@pytest.mark.parametrize("dt,values", COMBOS)
@pytest.mark.parametrize("name,k", [(n, k) for n in ("edges", "packed", "gram1537") for k in sc.K_LABEL
                                    if k <= 3201 and (n != "gram1537" or k <= 33)] + [("packed", 25600)])
def test_csc_label_sums(be, name, k, dt, values):
    """Bit for bit against the restatement in the kernel's order, at 8, 7 and 1 warps per CTA."""
    pair = _pair("col", name, dt, values)
    d = pair[0].shape[1]
    (_, c1, P1), (_, c2, P2) = _transposes(be, pair)
    rng = np.random.RandomState(k)
    labs = [rng.randint(0, k, m.shape[0]).astype(np.int32) for m in pair]
    ld = [_dev(x) for x in labs]

    def run():
        out = torch.full((d, k), 7.0, dtype=torch.float64, device="cuda")
        be.csc_label_sums_chunk(c1, d, ld[0], k, out, first=True)
        f = _host(out)
        be.csc_label_sums_chunk(c2, d, ld[1], k, out)
        return f + _host(out)

    first, acc = _twice(run)
    want = sc.label_sums(P1, labs[0], k)
    assert first.tobytes() == want.tobytes()
    want = sc.label_sums(P2, labs[1], k, prev=want)
    assert acc.tobytes() == want.tobytes()
    if values == "int":
        X1, X2 = _f64(pair[0]), _f64(pair[1])
        np.testing.assert_array_equal(acc, (X1.T @ sc.onehot(labs[0], k) + X2.T @ sc.onehot(labs[1], k)).toarray())


@pytest.mark.parametrize("dt,values", COMBOS)
@pytest.mark.parametrize("binarize", [None, 0.5])
@pytest.mark.parametrize("name,K", [("edges", 1), ("edges", 33), ("packed", 33), ("packed", 3201)])
def test_csc_class_counts(be, name, K, binarize, dt, values):
    """Weighted (dyadic weights) and binarising, labels outside [0, K) left out: bit for bit."""
    pair = _pair("col", name, dt, values)
    d = pair[0].shape[1]
    (_, c1, P1), (_, c2, P2) = _transposes(be, pair)
    rng = np.random.RandomState(K + 1)
    labs = [rng.randint(-1, K, m.shape[0]).astype(np.int32) for m in pair]
    ws = [rng.randint(1, 9, pair[0].shape[0]) / 4.0, None]
    ld = [_dev(x) for x in labs]
    wd = [_dev(ws[0]), None]

    def run():
        out = torch.full((d, K), 7.0, dtype=torch.float64, device="cuda")
        be.csc_class_counts_chunk(c1, d, ld[0], K, out, w=wd[0], binarize=binarize, first=True)
        f = _host(out)
        be.csc_class_counts_chunk(c2, d, ld[1], K, out, w=wd[1], binarize=binarize)
        return f + _host(out)

    first, acc = _twice(run)
    want = sc.label_sums(P1, labs[0], K, w=ws[0], binarize=binarize)
    assert first.tobytes() == want.tobytes()
    want = sc.label_sums(P2, labs[1], K, binarize=binarize, prev=want)
    assert acc.tobytes() == want.tobytes()


def test_label_sums_bound(be):
    """k = 25600 is the widest label-sum pass (one warp per CTA); k = 25601 is refused by both entry points."""
    m = _pair("col", "packed", "f32", "int")[0]
    d = m.shape[1]
    blk = _blk(m)
    csc = be.csr_transpose_chunk(blk, d)
    lab = torch.zeros(m.shape[0], dtype=torch.int32, device="cuda")
    out = torch.empty((d, 25601), dtype=torch.float64, device="cuda")
    be.csc_label_sums_chunk(csc, d, lab, 25600, out[:, :25600].contiguous(), first=True)
    with pytest.raises(RuntimeError, match="bkm_csc_label_sums_chunk"):
        be.csc_label_sums_chunk(csc, d, lab, 25601, out, first=True)
    with pytest.raises(RuntimeError, match="bkm_csc_class_counts_chunk"):
        be.csc_class_counts_chunk(csc, d, lab, 25601, out, first=True)
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------------------
# the row passes
# ---------------------------------------------------------------------------------------------------------------------
ROW_CASES = ["rows", "skewed", "edges", "mean6+0", "mean6+1", "mean12+0", "mean12+1", "mean24+0", "mean24+1"]


@pytest.mark.parametrize("dt,values", COMBOS)
@pytest.mark.parametrize("name", ROW_CASES)
def test_glm_csr_pass(be, name, dt, values):
    """The normal family in all four modes at G = 4, 8, 16 and 32 (each threshold from both sides), a row of 10^5
    entries in a G = 4 block, and rows of 0 to 2048 entries."""
    from test_glm_host import glm_terms

    pair = _pair("row", name, dt, values)
    d = pair[0].shape[1]
    rng = np.random.RandomState(5)
    beta = _operand(rng, d + 1, values)
    ys = [_operand(rng, m.shape[0], values) for m in pair]
    bd, yd = _dev(beta), [_dev(y) for y in ys]
    blks = [_blk(m) for m in pair]

    def run():
        grad = torch.full((d + 2,), 7.0, dtype=torch.float64, device="cuda")
        hrow = torch.full((d + 1,), 7.0, dtype=torch.float64, device="cuda")
        out = []
        for i, (blk, m) in enumerate(zip(blks, pair)):
            n = m.shape[0]
            r = torch.empty(n, dtype=torch.float64, device="cuda")
            w = torch.empty(n, dtype=torch.float64, device="cuda")
            r0 = torch.empty(n, dtype=torch.float64, device="cuda")
            g0 = torch.full((d + 2,), 7.0, dtype=torch.float64, device="cuda")
            mu = torch.empty(n, dtype=torch.float64, device="cuda")
            lab = torch.empty(n, dtype=torch.uint8, device="cuda")
            be.glm_csr_pass_chunk(blk, d, yd[i], bd, 1, 1, r=r, w=w, grad=grad, hrow=hrow, first=i == 0)
            be.glm_csr_pass_chunk(blk, d, yd[i], bd, 1, 0, r=r0, grad=g0, first=True)
            be.glm_csr_pass_chunk(blk, d, None, bd, 1, 2, out=mu)
            be.glm_csr_pass_chunk(blk, d, None, bd, 1, 3, out=lab)
            out += _host(r, w, r0, g0, mu, lab, grad, hrow)
        return out

    got = _twice(run)
    tot = np.zeros(3)
    for i, m in enumerate(pair):
        r, w, r0, g0, mu, lab, grad, hrow = got[8 * i: 8 * i + 8]
        X = _f64(m)
        eta = X @ beta[:-1] + beta[-1]
        esc = abs(X) @ abs(beta[:-1]) + abs(beta[-1])
        mw, lw, rw, ww = glm_terms(1, eta, ys[i])
        _close(mu, mw, esc, "mu")
        _close(r, rw, 2 * (esc + abs(ys[i])), "r")
        np.testing.assert_array_equal(w, ww)
        assert r0.tobytes() == r.tobytes()
        sure = np.abs(eta - 0.5) > 1e-12 * (esc + 1)
        np.testing.assert_array_equal(lab.astype(bool)[sure], (mw > 0.5)[sure])
        np.testing.assert_array_equal(lab.astype(bool), mu > 0.5)
        s = np.array([rw.sum(), lw.sum(), ww.sum()])
        tot += s
        got_s = np.array([grad[d], grad[d + 1], hrow[d]])
        scale = np.array([np.abs(rw).sum(), lw.sum(), ww.sum()]) if i == 0 else None
        if i == 0:
            assert (np.abs(got_s - s) <= 1e-12 * (scale + 1)).all()
            assert np.array([g0[d], g0[d + 1]]).tobytes() == got_s[:2].tobytes()
        else:
            assert (np.abs(got_s - tot) <= 1e-12 * (np.abs(tot) + np.abs(rw).sum() + 1)).all()


def _row_params(widths, small=33):
    out = []
    for name in ("rows", "skewed", "edges", "mean24+1", "mean6+0"):
        for l in widths:
            if name in ("skewed", "edges") and l > small:
                continue
            out += [(name, l, dt, v) for dt, v in COMBOS]
    return out


@pytest.mark.parametrize("name,l,dt,values", _row_params(sc.L_PANEL))
def test_csr_panel(be, name, l, dt, values):
    """X W and the ColMax record at C = 1, 2, 4 and up to three blockIdx.y tiles; the record folded over two blocks."""
    pair = _pair("row", name, dt, values)
    d = pair[0].shape[1]
    rng = np.random.RandomState(l + 3)
    W = _operand(rng, (d, l), values)
    Wd = _dev(W)
    blks = [_blk(m) for m in pair]
    n1 = pair[0].shape[0]

    def run():
        rec = be.colmax_new(l)
        out = []
        for i, blk in enumerate(blks):
            o = torch.full((pair[i].shape[0], l), 7.0, dtype=torch.float64, device="cuda")
            be.csr_panel_chunk(blk, d, Wd, out=o, colmax=rec, row_offset=0 if i == 0 else n1)
            out += _host(o, rec)
        return out

    o1, r1, o2, r2 = _twice(run)
    for i, o in enumerate((o1, o2)):
        X = _f64(pair[i])
        _close(o, np.asarray(X @ W), np.asarray(abs(X) @ abs(W)), "X W")
    # the record: per column the largest |t| over both blocks, its lowest global row and its signed value
    for rec, both in ((r1, o1), (r2, np.vstack([o1, o2]))):
        a = np.abs(both)
        row = np.argmax(a, axis=0)
        np.testing.assert_array_equal(rec[:, 0], a.max(axis=0))
        np.testing.assert_array_equal(rec[:, 1].view(np.int64), row)
        np.testing.assert_array_equal(rec[:, 2], both[row, np.arange(l)])


def _centres(be, rng, k, d, values):
    C = _operand(rng, (k, d), values)
    return C, be.sparse_pack_centers(_dev(C))


def _d2(X, C):
    xn = np.asarray(X.multiply(X).sum(1)).ravel()
    cn = (C * C).sum(1)
    d2 = np.maximum(xn[:, None] - 2.0 * np.asarray(X @ C.T) + cn[None, :], 0.0)
    return d2, xn[:, None] + 2.0 * np.asarray(abs(X) @ abs(C).T) + cn[None, :]


@pytest.mark.parametrize("name,k,dt,values", _row_params(sc.K_ASSIGN))
def test_csr_assign(be, name, k, dt, values):
    """The arg-min, distance and squared-distance modes; labels, minima, counts and the distance sum over two
    blocks."""
    pair = _pair("row", name, dt, values)
    d = pair[0].shape[1]
    C, pack = _centres(be, np.random.RandomState(k), k, d, values)
    blks = [_blk(m) for m in pair]

    def run():
        ds = torch.full((1,), 7.0, dtype=torch.float64, device="cuda")
        cnt = torch.full((k,), 7.0, dtype=torch.float64, device="cuda")
        out = []
        for i, blk in enumerate(blks):
            n = pair[i].shape[0]
            lab = torch.empty(n, dtype=torch.int32, device="cuda")
            mn = torch.empty(n, dtype=torch.float64, device="cuda")
            d2 = torch.empty((n, k), dtype=torch.float64, device="cuda")
            dist = torch.empty((n, k), dtype=torch.float64, device="cuda")
            be.csr_assign_chunk(blk, d, pack, k, labels=lab, min_dist=mn, dist_sum=ds, counts=cnt, first=i == 0)
            be.csr_assign_chunk(blk, d, pack, k, out=d2, mode=2)
            be.csr_assign_chunk(blk, d, pack, k, out=dist, mode=1)
            out += _host(lab, mn, d2, dist, ds, cnt)
        return out

    got = _twice(run)
    labs, mins = [], []
    for i in range(2):
        lab, mn, d2, dist, ds, cnt = got[6 * i: 6 * i + 6]
        want, scale = _d2(_f64(pair[i]), C)
        _close(d2, want, scale, "d2")
        assert dist.tobytes() == np.sqrt(d2).tobytes()
        np.testing.assert_array_equal(lab, np.argmin(d2, axis=1))           # ties to the lowest centre
        np.testing.assert_array_equal(mn, d2[np.arange(len(lab)), lab])
        labs.append(lab)
        mins.append(mn)
        allc = np.concatenate(labs)
        np.testing.assert_array_equal(cnt, np.bincount(allc, minlength=k).astype(np.float64))
        s = np.concatenate(mins)
        assert abs(ds[0] - s.sum()) <= 1e-13 * s.sum() * 4 + 1e-300


@pytest.mark.parametrize("binarize", [None, 0.5])
@pytest.mark.parametrize("name,K,dt,values", _row_params(sc.K_NB))
def test_nb_csr_jll(be, name, K, dt, values, binarize):
    from dask_ml_b200._lib import NB_JLL, NB_LOG_PROBA, NB_PROBA

    pair = _pair("row", name, dt, values)
    m = pair[0]
    d, n = m.shape[1], m.shape[0]
    rng = np.random.RandomState(K)
    WT, b = _operand(rng, (d, K), values), _operand(rng, K, values)
    WTd, bd = _dev(WT), _dev(b)
    blk = _blk(m)

    def run():
        out = []
        for mode in (NB_JLL, NB_LOG_PROBA, NB_PROBA):
            lab = torch.empty(n, dtype=torch.int32, device="cuda")
            o = torch.empty((n, K), dtype=torch.float64, device="cuda")
            be.nb_csr_jll_chunk(blk, d, WTd, bd, labels=lab, out=o, out_mode=mode, binarize=binarize)
            out += _host(lab, o)
        return out

    lab, jll, lab2, lp, lab3, pr = _twice(run)
    A = _f64(m)
    if binarize is not None:
        A = (A > binarize).astype(np.float64)
    want = np.asarray(A @ WT) + b
    scale = np.asarray(abs(A) @ abs(WT)) + abs(b)
    _close(jll, want, scale, "jll")
    np.testing.assert_array_equal(lab, np.argmax(jll, axis=1))               # the first maximum
    np.testing.assert_array_equal(lab2, lab)
    np.testing.assert_array_equal(lab3, lab)
    mx = want.max(axis=1, keepdims=True)
    lse = mx + np.log(np.exp(want - mx).sum(axis=1, keepdims=True))
    rs = scale.max(axis=1, keepdims=True) + 1.0
    assert (np.abs(lp - (want - lse)) <= 1e-12 * rs).all()
    assert (np.abs(pr - np.exp(want - lse)) <= 1e-12 * rs).all()


@pytest.mark.parametrize("dt,values", COMBOS)
@pytest.mark.parametrize("name,l", [(n, l) for n in ("mean24+1", "rows") for l in sc.L_COLSUM])
def test_csr_kernel_colsum(be, name, l, dt, values):
    """The colsum epilogue in 1, 2 and 3 windows of keep rows, over two blocks."""
    pair = _pair("row", name, dt, values)
    d = pair[0].shape[1]
    C, pack = _centres(be, np.random.RandomState(l), l, d, values)
    d2s = [_d2(_f64(m), C) for m in pair]
    gamma = 1.0 / np.median(d2s[0][0])
    blks = [_blk(m) for m in pair]

    def run():
        cs = torch.full((l,), 7.0, dtype=torch.float64, device="cuda")
        out = []
        for i, blk in enumerate(blks):
            be.csr_kernel_colsum(blk, d, pack, l, gamma, cs, first=i == 0)
            out += _host(cs)
        return out

    got = _twice(run)
    want, tol = np.zeros(l), np.zeros(l)
    for i, (d2, scale) in enumerate(d2s):
        e = np.exp(-gamma * d2)
        want = want + e.sum(axis=0)
        tol = tol + (e * (gamma * 1e-13 * scale + 1e-15)).sum(axis=0)      # each d2 within 1e-13 of its scale
        assert (np.abs(got[i] - want) <= 4 * tol + 1e-12 * want).all()


@pytest.mark.parametrize("kw", [7, 40])
@pytest.mark.parametrize("dt,values", COMBOS)
@pytest.mark.parametrize("name,l", [(n, l) for n in ("mean24+1", "rows") for l in sc.L_EMBED])
def test_csr_nystrom_embed(be, name, l, dt, values, kw):
    """The embed epilogue over several tiles of keep rows (the first sweep for the row minimum, then per tile)."""
    m = _pair("row", name, dt, values)[0]
    d, n = m.shape[1], m.shape[0]
    rng = np.random.RandomState(l + kw)
    C, pack = _centres(be, rng, l, d, values)
    W = rng.standard_normal((l, kw))
    d2, scale = _d2(_f64(m), C)
    gamma = 1.0 / np.median(d2)
    blk, Wd = _blk(m), _dev(W)

    def run():
        o = torch.empty((n, kw), dtype=torch.float64, device="cuda")
        be.csr_nystrom_embed(blk, d, pack, l, gamma, Wd, o)
        return _host(o)

    (got,) = _twice(run)
    e = np.exp(-gamma * (d2 - d2.min(axis=1, keepdims=True))) @ W
    want = e / np.linalg.norm(e, axis=1, keepdims=True)
    np.testing.assert_allclose(got, want, rtol=1e-9, atol=1e-10)


# ---------------------------------------------------------------------------------------------------------------------
# the SGD row tile
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.filterwarnings("ignore::FutureWarning")
@pytest.mark.parametrize("penalty", ["l2", "elasticnet"])
def test_sgd_rows_at_the_row_tile(penalty):
    """Rows of 1023 to 2048 entries around the 1024-entry row tile of the CSR epoch (kTile, bkm_sgd.cu): bit-identical
    to scikit-learn."""
    from sklearn.linear_model import SGDClassifier

    from dask_ml_b200.linear_model import PartialSGDClassifier

    lens = [1024, 1025, 2048, 1023, 5, 0, 2047, 1024, 33] * 4
    ours = PartialSGDClassifier(classes=np.arange(3), random_state=4, penalty=penalty)
    ref = SGDClassifier(random_state=4, penalty=penalty)
    for i in range(2):
        X = sc.rows_at(lens, 2100, seed=20 + i, values="rand")
        y = np.random.RandomState(i).randint(0, 3, X.shape[0])
        ours.partial_fit(X, torch.from_numpy(y).cuda(), classes=np.arange(3))
        ref.partial_fit(X, y, classes=np.arange(3))
    np.testing.assert_array_equal(ours.coef_, ref.coef_)
    np.testing.assert_array_equal(ours.intercept_, ref.intercept_)
    assert ours.t_ == ref.t_
