"""The dense row-chunk passes on the H100 at their class-block, split, slice and column-group limits, on exact integer
data (tests/dense_cases.py).

Every case holds values whose every partial sum is exact, so numpy's float64 result is a bit-exact reference at every
geometry: the Gram, column sums and weighted Gram, the projection and its arg-max records, the normal-family GLM grad,
hrow and w, the moments, squared deviations and class counts, the raw linear jll and every label (exact ties resolve to
the lowest index, as np.argmax) are held bit for bit.  Outputs that go through exp or log (log-softmax, softmax, the
logistic and Poisson families) are held to a stated tolerance.  Each pass runs twice and must give the same bits; each
accumulating pass runs a first call and then an accumulating call on a block with another geometry.  The SM count is
the device's, and where a pass sizes its workspace from its geometry the test checks that size against the
restatement."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import dense_cases as dc  # noqa: E402

pytestmark = pytest.mark.gpu

TD = {"f32": torch.float32, "f64": torch.float64, "bf16": torch.bfloat16}
POISON = 12345.0
PAD = 3
# (row dtype, d): every jll path; bf16 rows run the fp32 kernels
JLL = [(dt, d) for prec, d, fc, ch in dc.jll_paths() for dt in (("f32", "bf16") if prec == "f32" else ("f64",))]


@pytest.fixture(scope="module")
def be():
    from dask_ml_b200.engine import CudaBackend

    return CudaBackend()


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _dev(a, dt=torch.float64):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dt).cuda()


def _x(h, dt, layout="aligned"):
    """Rows on the device: a fresh allocation, or a base one element past it ("offset")."""
    t = torch.from_numpy(np.ascontiguousarray(h)).to(TD[dt])
    if layout == "aligned":
        return t.cuda()
    n, d = h.shape
    big = torch.zeros(n * d + 1, dtype=TD[dt], device="cuda")
    v = big[1:].view(n, d)
    v.copy_(t)
    return v


def _base(x):
    return x.data_ptr() % 256


def _host(*ts):
    torch.cuda.synchronize()
    return [t.cpu().numpy().copy() for t in ts]


def _twice(run):
    """run() twice: the same bits."""
    a, b = run(), run()
    for x, y in zip(a, b):
        assert x.tobytes() == y.tobytes()
    return a


def _eq(got, want, what):
    got, want = np.asarray(got), np.asarray(want, dtype=got.dtype)
    bad = np.argwhere(~((got == want) | (np.isnan(got) & np.isnan(want))))
    assert len(bad) == 0, "%s: %d elements differ, first %s: %r vs %r" % (
        what, len(bad), bad[0], got[tuple(bad[0])], want[tuple(bad[0])])


def _close(got, want, tol, what):
    err = np.abs(got - want)
    bad = np.argwhere(~(err <= tol))
    assert len(bad) == 0, "%s: %d elements off, first %s: %r vs %r" % (
        what, len(bad), bad[0], got[tuple(bad[0])], want[tuple(bad[0])])


def _ws(be, name, *args):
    return be._query(name, *[int(a) for a in args])


# ---------------------------------------------------------------------------------------------------------------------
# GaussianNB jll
# ---------------------------------------------------------------------------------------------------------------------
def _jll(be, x, c, out, exp_out=False):
    """(labels, n_deferred, the (n, K + PAD) output buffer) of one call; the output is a view of pitch K + PAD whose
    padding holds POISON."""
    n, K = x.shape[0], c.K
    dev = [_dev(a) for a in (c.theta, c.w, c.logc)]
    lab = torch.full((n,), -7, dtype=torch.int32, device="cuda")
    nd = torch.zeros(1, dtype=torch.int32, device="cuda")
    buf = torch.full((n, K + PAD), POISON, dtype=torch.float64, device="cuda")
    be.nb_jll_chunk(x, *dev, labels=lab, out=buf[:, :K] if out else None, exp_out=exp_out, n_deferred=nd)
    return _host(lab, nd, buf)


def _lp_tol(lp, jll, K):
    vmax = np.abs(np.nanmax(jll, 1, keepdims=True))
    return 4e-12 * (1.0 + np.abs(lp) + vmax) + 1e-15 * K


@pytest.mark.parametrize("out", [False, True], ids=["labels", "out"])
@pytest.mark.parametrize("dt,d", JLL)
def test_jll_class_blocks(be, dt, d, out):
    prec = "f64" if dt == "f64" else "f32"
    kb = dc.jll_kb_max(prec, d, out)
    for i, K in enumerate(dc.jll_ks(prec, d, out)):
        assert -(-K // dc.jll_kb(prec, d, K, out)) == i + 1           # one, two and three class blocks
        c = dc.jll_case(prec, d, K, kb, seed=K)
        jll, lab, ties, lp = dc.jll_ref(c)
        x = _x(c.x, dt)
        glab, nd, buf = _twice(lambda: _jll(be, x, c, out))
        _eq(glab, lab, "labels K=%d" % K)
        # the fp32 path defers exactly the tied rows (every other row's margin is far above its bound) and re-decides
        # them in float64; the float64 path defers nothing
        assert int(nd[0]) == (ties if prec == "f32" else 0), (int(nd[0]), ties)
        assert (buf[:, K:] == POISON).all()
        if out:
            _close(buf[:, :K], lp, _lp_tol(lp, jll, K), "log-softmax K=%d" % K)
        else:
            assert (buf == POISON).all()
        if i < 2:
            continue
        if out:                                                       # exp_out, across the blocks
            _, _, p = _twice(lambda: _jll(be, x, c, True, exp_out=True))
            ep = np.exp(lp)
            _close(p[:, :K], ep, _lp_tol(lp, jll, K) * 1.01 * ep + 1e-300, "softmax K=%d" % K)
            assert (p[:, K:] == POISON).all()
        # a NaN log-prior in the last block: the first NaN class on every row, NaN log-probabilities
        cn = dc.jll_case(prec, d, K, kb, seed=K, nan_class=K - 1)
        _, labn, _, _ = dc.jll_ref(cn)
        assert (labn == K - 1).all()
        glab, nd, buf = _twice(lambda: _jll(be, x, cn, out))
        _eq(glab, labn, "labels with a NaN class")
        assert int(nd[0]) == 0
        if out:
            assert np.isnan(buf[:, :K]).all() and (buf[:, K:] == POISON).all()


# ---------------------------------------------------------------------------------------------------------------------
# linear jll
# ---------------------------------------------------------------------------------------------------------------------
def _lin(be, x, c, mode, labels=True):
    n, K = x.shape[0], c.K
    lab = torch.full((n,), -7, dtype=torch.int32, device="cuda")
    buf = torch.full((n, K + PAD), POISON, dtype=torch.float64, device="cuda")
    be.nb_linear_jll_chunk(x, _dev(c.W), _dev(c.b), labels=lab if labels else None,
                           out=buf[:, :K] if mode is not None else None, out_mode=mode or 0, binarize=c.binarize)
    return _host(lab, buf)


@pytest.mark.parametrize("dt", ["f32", "f64", "bf16"])
@pytest.mark.parametrize("d", dc.LIN_D)
@pytest.mark.parametrize("K", dc.LIN_K)
def test_linear_jll_blocks(be, K, d, dt):
    c = dc.linear_case(K, d, seed=K + d, binarize=1.5 if d == 33 else None)
    jll, lab, lp = dc.linear_ref(c)
    x = _x(c.x, dt)
    glab, _ = _twice(lambda: _lin(be, x, c, None))
    _eq(glab, lab, "labels")
    glab, raw = _twice(lambda: _lin(be, x, c, 0))
    _eq(glab, lab, "labels with jll")
    _eq(raw[:, :K], jll, "raw jll")
    assert (raw[:, K:] == POISON).all()
    tol = 4e-12 * (1.0 + np.abs(lp) + np.abs(jll).max(1, keepdims=True)) + 1e-15 * K
    gl, o = _twice(lambda: _lin(be, x, c, 1, labels=False))
    assert (gl == -7).all() and (o[:, K:] == POISON).all()
    _close(o[:, :K], lp, tol, "log-softmax")
    _, o = _twice(lambda: _lin(be, x, c, 2))
    ep = np.exp(lp)
    _close(o[:, :K], ep, 1.01 * tol * ep + 1e-300, "softmax")


# ---------------------------------------------------------------------------------------------------------------------
# projection
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", ["f32", "f64", "bf16"])
@pytest.mark.parametrize("d", dc.LIN_D)
@pytest.mark.parametrize("k", dc.LIN_K)
def test_projection_column_blocks(be, sms, k, d, dt):
    A = dc.project_case(k, d, seed=k * d)
    B = dc.project_case(k, d, seed=k * d, n=2 * k + 70)                # the same W and shift, another grid
    assert dc.project_geom(A.x.shape[0], k, sms)[3] != dc.project_geom(B.x.shape[0], k, sms)[3]
    nA = A.x.shape[0]
    outA, recA = dc.project_ref(A)
    outB, recB = dc.project_ref(B, row_offset=nA)
    rec = dc.colmax_merge(recA, recB)
    odt = torch.float32 if dt == "f32" else torch.float64
    xs = [_x(A.x, dt), _x(B.x, dt, "offset")]
    W, s = _dev(A.W), _dev(A.shift)

    def run():
        cm = be.colmax_new(k)
        bufs = []
        for x, off in zip(xs, (0, nA)):
            buf = torch.full((x.shape[0], k + PAD), POISON, dtype=odt, device="cuda")
            be.project_chunk(x, s, W, out=buf[:, :k], colmax=cm, row_offset=off)
            bufs.append(buf)
        return _host(*bufs, cm)

    bA, bB, cm = _twice(run)
    for buf, want in ((bA, outA), (bB, outB)):
        _eq(buf[:, :k].astype(np.float64), want, "projection")
        assert (buf[:, k:] == POISON).all()
    _eq(cm[:, 0], rec[:, 0], "colmax |out|")
    _eq(cm[:, 1].view(np.int64), rec[:, 1].astype(np.int64), "colmax row")
    _eq(cm[:, 2], rec[:, 2], "colmax value")


# ---------------------------------------------------------------------------------------------------------------------
# Gram and weighted Gram
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("weighted", [False, True], ids=["gram", "weighted"])
@pytest.mark.parametrize("dt", ["f32", "f64", "bf16"])
@pytest.mark.parametrize("i", range(len(dc.gram_ds(132))))
def test_gram_splits(be, sms, i, dt, weighted):
    d = dc.gram_ds(sms)[i]
    c = dc.gram_case(d, sms, seed=d)
    geo = [dc.gram_geom(x.shape[0], d, sms) for x in c.xs]
    for x, g in zip(c.xs, geo):
        assert _ws(be, "bkm_gram_workspace_bytes", x.shape[0], d) == g.total
    if d >= dc.gram_one_split_d(sms):
        assert geo[0].splits == 1
    else:
        assert geo[0].splits > 1 and c.xs[0].shape[0] - (geo[0].splits - 1) * geo[0].rows_per_split == 1
    cs, G, H = dc.gram_ref(c)
    shift = _dev(c.shift)
    ws = [_dev(w) for w in c.ws]
    for layouts in (("aligned", "offset"), ("offset", "aligned")):
        xs = [_x(x, dt, lay) for x, lay in zip(c.xs, layouts)]
        bulk = [dc.bulk_ok(_base(x), d, d, dt) for x in xs]
        assert bulk[layouts.index("offset")] is False
        if d % (16 // dc.ES[dt]) == 0:
            assert bulk[layouts.index("aligned")] is True

        def run():
            g = torch.full((d, d), np.nan, dtype=torch.float64, device="cuda")
            s = torch.full((d,), np.nan, dtype=torch.float64, device="cuda")
            for j, x in enumerate(xs):
                if weighted:
                    be.gram_weighted_chunk(x, ws[j], g, first=j == 0)
                else:
                    be.gram_chunk(x, shift, s, g, first=j == 0)
            return _host(g, s)

        g, s = _twice(run)
        if weighted:
            _eq(g, H, "weighted Gram %s" % (layouts,))
        else:
            _eq(g, G, "Gram %s" % (layouts,))
            _eq(s, cs, "colsum %s" % (layouts,))


# ---------------------------------------------------------------------------------------------------------------------
# moments and class counts
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", ["f32", "f64", "bf16"])
@pytest.mark.parametrize("kslice", ["ks", "ks+1"])
@pytest.mark.parametrize("d", dc.MOM_D)
def test_moments_and_counts_slices(be, sms, d, kslice, dt):
    ks = dc.mom_ks(d)
    K = ks + (kslice == "ks+1")
    c = dc.mom_case(d, K, seed=d + K)
    for x in c.xs:
        g = dc.mom_geom(x.shape[0], d, K, sms)
        assert g.nk == 1 + (K > ks) and g.nf == -(-d // 256) and g.splits > 1
        assert _ws(be, "bkm_nb_workspace_bytes", x.shape[0], d, K) == g.total
    S, C, Q, F, CC = dc.mom_ref(c)
    _, _, _, Fb, _ = dc.mom_ref(c, binarize=0.5)
    xs = [_x(c.xs[0], dt), _x(c.xs[1], dt, "offset")]
    cls = [_dev(y, torch.int32) for y in c.cls]
    ws = [_dev(w) for w in c.ws]
    theta = _dev(c.theta)

    def run():
        outs = []
        for th in (None, theta):
            s = torch.full((K, d), np.nan, dtype=torch.float64, device="cuda")
            n = torch.full((K,), np.nan, dtype=torch.float64, device="cuda")
            for j in range(2):
                be.class_moments_chunk(xs[j], cls[j], K, s, n if th is None else None, theta=th, first=j == 0)
            outs += [s, n]
        for bz in (None, 0.5):
            f = torch.full((K, d), np.nan, dtype=torch.float64, device="cuda")
            n = torch.full((K,), np.nan, dtype=torch.float64, device="cuda")
            for j in range(2):
                be.class_counts_chunk(xs[j], cls[j], K, f, n, w=ws[j], binarize=bz, first=j == 0)
            outs += [f, n]
        return _host(*outs)

    gS, gC, gQ, _, gF, gCC, gFb, gCCb = _twice(run)
    _eq(gS, S, "sums")
    _eq(gC, C, "counts")
    _eq(gQ, Q, "squared deviations")
    _eq(gF, F, "weighted feature counts")
    _eq(gFb, Fb, "binarised feature counts")
    _eq(gCC, CC, "weighted class counts")
    _eq(gCCb, CC, "weighted class counts (binarised)")


# ---------------------------------------------------------------------------------------------------------------------
# GLM
# ---------------------------------------------------------------------------------------------------------------------
def _glm_run(be, c, xs, ys, beta, mode, family):
    d = c.d
    grad = torch.full((d + 2,), np.nan, dtype=torch.float64, device="cuda")
    hrow = torch.full((d + 1,), np.nan, dtype=torch.float64, device="cuda")
    ws = [torch.full((x.shape[0],), np.nan, dtype=torch.float64, device="cuda") for x in xs]
    for j, x in enumerate(xs):
        be.glm_pass_chunk(x, ys[j], beta, family, mode, grad=grad, hrow=hrow if mode == 1 else None,
                          w=ws[j] if mode == 1 else None, first=j == 0)
    return _host(grad, hrow, *ws)


@pytest.mark.parametrize("dt", ["f32", "f64", "bf16"])
@pytest.mark.parametrize("d", dc.GLM_D)
def test_glm_column_blocks(be, sms, d, dt):
    c = dc.glm_case(d, sms, seed=d, family=1)
    for x in c.xs:
        assert _ws(be, "bkm_glm_workspace_bytes", x.shape[0], d) == dc.glm_ws(x.shape[0], d, sms)
    grad, hrow, wref, mus, _, _ = dc.glm_ref(c)
    ys = [_dev(y) for y in c.ys]
    beta = _dev(c.beta)
    for layouts in (("aligned", "offset"), ("offset", "aligned")):
        xs = [_x(x, dt, lay) for x, lay in zip(c.xs, layouts)]
        vec = [dc.bulk_ok(_base(x), d, d, dt) for x in xs]
        assert vec[layouts.index("offset")] is False
        g, h, w0, w1 = _twice(lambda: _glm_run(be, c, xs, ys, beta, 1, 1))
        _eq(g, grad, "Newton grad %s" % (layouts,))
        _eq(h, hrow, "hrow %s" % (layouts,))
        _eq(w0, wref[0], "w")
        _eq(w1, wref[1], "w")
        g, h, _, _ = _twice(lambda: _glm_run(be, c, xs, ys, beta, 0, 1))
        _eq(g, grad, "grad %s" % (layouts,))
        assert np.isnan(h).all()
        for x, mu in zip(xs, mus):
            o = torch.full((x.shape[0],), np.nan, dtype=torch.float64, device="cuda")

            def predict(x=x, o=o):
                be.glm_pass_chunk(x, None, beta, 1, 2, out=o)
                return _host(o)

            (got,) = _twice(predict)
            _eq(got, mu, "mu")


@pytest.mark.parametrize("family", [0, 2], ids=["logistic", "poisson"])
@pytest.mark.parametrize("d", [31, 129, 200, 513])
def test_glm_families(be, sms, d, family):
    """The logistic and Poisson families go through exp and log1p: grad, hrow and w to 1e-13 of the scale of each sum
    (sum |r| |x|, sum |w| |x|), with block A aligned and block B one element off alignment (element loads)."""
    c = dc.glm_case(d, sms, seed=d + 7, family=family)
    grad, hrow, wref, _, gs, hs = dc.glm_ref(c)
    xs = [_x(c.xs[0], "f64"), _x(c.xs[1], "f64", "offset")]
    g, h, w0, w1 = _twice(lambda: _glm_run(be, c, xs, [_dev(y) for y in c.ys], _dev(c.beta), 1, family))
    _close(g, grad, 1e-13 * gs + 1e-300, "grad")
    _close(h, hrow, 1e-13 * hs + 1e-300, "hrow")
    _close(w0, wref[0], 1e-14 * np.abs(wref[0]) + 1e-300, "w")
    _close(w1, wref[1], 1e-14 * np.abs(wref[1]) + 1e-300, "w")
